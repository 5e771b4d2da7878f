"""The group-major schedule of the wgmma mask + cross-fade kernel (dsd_tc.cu) at its edges, with the clip sizes derived
from the device's SM count.

Work item w = group * m_tiles + tile; CTA c of min(SMs, items) takes [c n / ctas, (c + 1) n / ctas).  The producer
stages a group's B rows, fade-table entries and Nyquist bin only when its range enters that group, and streams the A
tile of every item from the pre-split image, so the edges are where a range starts (on a group's last tile, or
mid-group), how many group boundaries it crosses, a last group only partly inside the clip, and fewer items than SMs.
`schedule` reproduces the kernel's partition, and every case asserts the edges it is sized for.

- Stems (Ŝ) mode through dcs_dsd_mask_f32 against the float64 per-element bound of test_gpu_mask_views.py, at F = 129
  (one tile plus the producer's Nyquist bin), 513 and 2049 (a 1 MB A image), with 3 decoders and with 4 (the stereo net:
  two mixture channels, one call each): twice with identical bits, the NaN sentinels around and between the output
  planes untouched.
- Masks mode through dcs_separate_masks: twice with identical bits into a NaN-filled buffer whose pad columns, plane
  gaps and tail stay NaN, and M * X equal to the stems call's spectrum tap bit for bit (test_gpu_masks.check_bits), which
  ties the masks to the Ŝ mode checked above."""
import os
import sys

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_mask_views as mv  # noqa: E402
import test_gpu_masks as tm  # noqa: E402
from oracle import pipeline  # noqa: E402


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def schedule(F, T, ndec):
    """(m_tiles, frames per group, CTA ranges) of the launch dsd_tc.cu makes for F bins and T frames"""
    frames = 8 if ndec == 3 else 4
    nyq = F > 128 and (F - 1) % 128 == 0
    m = (F - 1) // 128 if nyq else -(-F // 128)
    n = m * -(-T // frames)
    ctas = min(sms(), n)
    return m, frames, [(c * n // ctas, (c + 1) * n // ctas) for c in range(ctas)]


def edges(F, T, ndec):
    """the schedule edges a launch reaches"""
    m, frames, rng = schedule(F, T, ndec)
    spans = [(e - 1) // m - b // m + 1 for b, e in rng]      # groups a range touches
    out = set()
    if m > 1 and any(b % m == m - 1 for b, _ in rng):
        out.add("starts_on_last_tile")
    if any(0 < b % m < m - 1 for b, _ in rng):
        out.add("starts_mid_group")
    if 2 in spans:
        out.add("crosses_one_boundary")
    if max(spans) >= 3:
        out.add("crosses_several")
    if T % frames:
        out.add("partial_last_group")
    if m * -(-T // frames) < sms():
        out.add("fewer_items_than_sms")
    return out


# name -> (F, ndec, frames T as a function of the SM count S, the edges the case is sized for)
S_CASES = {
    "F129_dec3": (129, 3, lambda S: 8 * (3 * S + 3) - 3, {"crosses_several", "partial_last_group"}),
    "F513_dec3": (513, 3, lambda S: 8 * (S + S // 2 + 1) - 5,
                  {"starts_on_last_tile", "starts_mid_group", "crosses_one_boundary", "crosses_several", "partial_last_group"}),
    "F2049_dec3_long": (2049, 3, lambda S: 8 * (S // 8 + 3) - 1, {"starts_mid_group", "crosses_one_boundary", "partial_last_group"}),
    "F2049_dec3_few": (2049, 3, lambda S: 8 * max(1, S // 16 - 1) - 3, {"fewer_items_than_sms", "partial_last_group"}),
    "F129_dec4": (129, 4, lambda S: 4 * (4 * S + 1) - 2, {"crosses_several", "partial_last_group"}),
    "F513_dec4": (513, 4, lambda S: 4 * (S + 7) - 1,
                  {"starts_on_last_tile", "starts_mid_group", "crosses_one_boundary", "partial_last_group"}),
    "F2049_dec4": (2049, 4, lambda S: 4 * (S // 4 + 1) - 3,
                   {"starts_on_last_tile", "starts_mid_group", "crosses_one_boundary", "partial_last_group"}),
}


@pytest.fixture(scope="module")
def ctx():
    from deepconvsep_b200.engine import Context
    return Context(0)


def test_cases_cover_every_edge():
    reached = set()
    for F, ndec, T_of, want in S_CASES.values():
        got = edges(F, T_of(sms()), ndec)
        assert want <= got, (F, ndec, want - got)
        reached |= got
    assert reached == {"starts_on_last_tile", "starts_mid_group", "crosses_one_boundary", "crosses_several",
                       "partial_last_group", "fewer_items_than_sms"}


@pytest.mark.parametrize("name", list(S_CASES))
def test_stems_mode_matches_float64(ctx, name):
    F, ndec, T_of, _ = S_CASES[name]
    case = mv.dsd_case("group_major_" + name, F, T_of(sms()), 30, 25, ndec=ndec)
    case["engine"] = "tc"
    b = mv.Buffers(case)
    Sb = mv._run(ctx, case, b, mv.ENGINES["tc"])
    assert np.array_equal(Sb, mv._run(ctx, case, b, mv.ENGINES["tc"])), "two runs gave different bits"

    T, ldf = case["T"], case["ldf"]
    body = Sb[2 * mv.SLACK:2 * mv.SLACK + 2 * b.nplanes * b.sp].reshape(b.nplanes, b.sp, 2)
    written = np.zeros((b.nplanes, b.sp), bool)
    written[:, :T * ldf].reshape(b.nplanes, T, ldf)[:, :, :F] = True
    assert (Sb[:2 * mv.SLACK] == mv.S_SENTINEL).all() and (Sb[2 * mv.SLACK + 2 * b.nplanes * b.sp:] == mv.S_SENTINEL).all()
    assert (body[~written] == mv.S_SENTINEL).all(), "S elements outside the written frames and bins changed"
    vals = body[:, :T * ldf].reshape(b.nplanes, T, ldf, 2).view(np.float32)[:, :, :F]
    assert np.isfinite(vals).all()
    S = vals[..., 0] + 1j * vals[..., 1].astype(np.float64)

    frames = np.arange(T)
    pm = mv._plane_map(case)
    worst, fails, wf = 0.0, [], 1.0
    for mset in sorted(set(m for _, m, _ in pm)):
        ref = mv.reference_masks(case, frames, mset)
        wf = min(wf, mv.well_fraction(ref))
        idx = [i for i, (_, m, _) in enumerate(pm) if m == mset]
        wo, fa = mv.evaluate(ref, S[idx], case["X"][mset])
        worst = max(worst, wo)
        fails += fa
    mv.record("mask_group_major:" + name, F=F, T=T, ndec=ndec, well_conditioned=wf, worst_error_over_bound=worst)
    assert not fails, (name, fails)
    assert wf >= 0.99, (name, wf)
    assert worst <= 1.0, (name, worst)


# name -> (arch, N, hop, patcher, frames T as a function of the SM count S)
M_CASES = {
    "dsd_N256": ("dsd", 256, 128, "standalone", lambda S: 8 * (2 * S + 1) - 3),
    "dsd_N1024": ("dsd", 1024, 512, "standalone", lambda S: 8 * (S + S // 2 + 1) - 5),
    "dsd_ild_N1024": ("dsd_ild", 1024, 512, "util", lambda S: 4 * (S + 7) - 1),
}


@pytest.mark.parametrize("name", list(M_CASES))
def test_masks_mode_bits_and_fences(name):
    arch, N, hop, patcher, T_of = M_CASES[name]
    _, sep = tm.separator(arch, N, hop, seed=9, patcher=patcher)
    L = (T_of(sms()) - 2) * hop                                   # T = ceil(L / hop) + 2 frames
    T, F, ldf = sep.stft.num_frames(L), sep.model.F, sep.stft.ldf
    ndec = 4 if arch == "dsd_ild" else 3
    assert T == T_of(sms()) and sep.num_patches(T) > 0 and "partial_last_group" in edges(F, T, ndec)
    a, _ = pipeline.synth_mixture(L / 44100.0, 90 + N)
    a = a[:L]
    if arch == "dsd_ild":
        b, _ = pipeline.synth_mixture(L / 44100.0, 91 + N)
        audio = np.stack([a, 0.4 * a + 0.6 * b[:L]], axis=1).astype(np.float32)
        x = torch.tensor(np.ascontiguousarray(audio.T), device="cuda")
    else:
        audio = a.astype(np.float32)
        x = torch.tensor(audio, device="cuda")
    nplanes = sep.nsrc * (2 if arch == "dsd_ild" else 1)
    m_stride = T * ldf + 29
    outs = []
    for _ in range(2):
        buf = torch.full((nplanes * m_stride + 64,), float("nan"), dtype=torch.float32, device="cuda")
        tm.raw_call(sep, x, buf, m_stride)
        h = buf.cpu().numpy()
        planes = np.stack([h[p * m_stride:p * m_stride + T * ldf].reshape(T, ldf) for p in range(nplanes)])
        assert np.isfinite(planes[:, :, :F]).all() and np.isnan(planes[:, :, F:]).all()
        for p in range(nplanes):
            assert np.isnan(h[p * m_stride + T * ldf:(p + 1) * m_stride]).all()
        assert np.isnan(h[nplanes * m_stride:]).all()
        outs.append(h)
    assert tm.same_bits(outs[0], outs[1])
    tm.check_bits(sep, audio)
