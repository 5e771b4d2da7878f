"""The masks output (dcs_separate_masks, dcs_separate_masks_score, dcs_separate_masks_notes; Separator.separate_masks):
the network's blended soft masks, from a pipeline that stops before the inverse STFT.

- bit for bit against the stems path of every family: the masks M and the mixture STFT X (Stft.forward) give the
  spectrum tap of the stems call as view_as_real(X) * M[..., None] in fp32 (up to the sign of a zero, see same_values),
  and Stft.inverse of that gives its stems bit for bit -- on both engines (DCS_DEBUG_SIMT_GEMM=1 routes the mask stage to the FFMA twins);
- against the float64 blended masks of tests/masks_oracle.py, the max-pool and 1x1 routing adopted from the routing tap;
- fences: NaN-filled buffers keep their pad columns, gaps and sentinels; determinism; short clips; dcs_set_wiener;
- refusals before anything is queued, and the workspace the mode saves."""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from oracle import dsp, nets, pipeline  # noqa: E402
import masks_oracle as mo  # noqa: E402
import score1x1_oracle as s1  # noqa: E402
from parity import record  # noqa: E402

TOL = 1e-4
MASK_MAX = 1.0 + 2.0 ** -20


def score_filters(T, F, seed=4):
    """synthetic filters with filterSpec's structure: 1 on note bins, 1e-18 elsewhere, normalised over the sources"""
    rng = np.random.default_rng(seed)
    raw = np.full((4, T, F), 1e-18, dtype=np.float32)
    for j in range(4):
        for _ in range(6 + T // 40):
            t0, b0 = rng.integers(0, max(1, T - 40)), rng.integers(1, F - 24)
            raw[j, t0:t0 + 40, b0:b0 + 20] = 1.0
    return (raw / raw.sum(axis=0)).astype(np.float32)


def melody_table(T, F, seed=3, nnotes=12, nh=3):
    """a note table [4, nnotes, 3 + 2 nh]: first frame, last frame, MIDI number, (lo, hi) bin pairs"""
    rng = np.random.default_rng(seed)
    m = np.zeros((4, nnotes, 3 + 2 * nh))
    for j in range(4):
        for p in range(nnotes):
            n0 = float(rng.integers(0, T))
            m[j, p, :3] = (n0, n0 + float(rng.integers(5, 60)), float(rng.integers(40, 90)))
            for k in range(nh):
                lo = int(rng.integers(0, F - 30))
                m[j, p, 3 + 2 * k:5 + 2 * k] = (lo, lo + int(rng.integers(2, 30)))
    return m


def separator(arch, N, hop, seed=5, overlap=25, patcher="standalone", win="hanning", tc=None, params=None, **kw):
    from deepconvsep_b200.engine import Separator
    F = N // 2 + 1
    if params is None:
        params = s1.make_synthetic_params_1x1(seed=seed) if arch == "bach10_score_1x1" else nets.make_synthetic_params(arch, F, seed=seed)
    return params, Separator(params, arch=arch, frame_size=N, hop=hop, window=win, overlap=overlap, patcher=patcher,
                             feat_size=F, time_context=tc, **kw)


def same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def same_values(a, b):
    """bit for bit, except that a zero may carry either sign: the strided-conv1 nets' tensor-core kernel stores +0 for
    the frames no patch covers (the standalone patcher's tail), where mask 0 times a negative X component is -0"""
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    diff = a.view(np.uint32) != b.view(np.uint32)
    return bool(np.all((a == 0) & (b == 0) | ~diff))


def device_masks(sep, audio, **kw):
    """separate_masks on the device, pad columns zero: [nplanes, T, ldf]"""
    x = torch.tensor(np.ascontiguousarray(np.asarray(audio, dtype=np.float32).T), device="cuda")
    T = sep.stft.num_frames(x.shape[-1])
    nplanes = sep.nsrc * (2 if sep.model.arch == "dsd_ild" else 1)
    out = torch.zeros((nplanes, T, sep.stft.ldf), dtype=torch.float32, device="cuda")
    got = sep.separate_masks(x, out=out, **kw)
    assert got is out
    return out


def mixture_stft(sep, audio):
    """X of each channel as the device computes it: complex64 cuda [nch, T, ldf]"""
    a = np.asarray(audio, dtype=np.float32)
    chans = [a] if a.ndim == 1 else [a[:, c] for c in range(a.shape[1])]
    return torch.stack([sep.stft.forward(torch.tensor(np.ascontiguousarray(c), device="cuda"), want_mag=False)[0] for c in chans])


def check_bits(sep, audio, masks_kw=None, tapped_kw=None, masks_audio=None):
    """M * X against the spectrum tap of the stems call and iSTFT(M * X) against its stems, bit for bit.  masks_audio:
    the clip the masks are taken from (the downmix for keep-channels), planes (source, channel) in both calls."""
    M = device_masks(sep, audio if masks_audio is None else masks_audio, **(masks_kw or {}))
    stems, tap = sep.separate_tapped(audio, **(tapped_kw or {}))
    X = mixture_stft(sep, audio)
    nch = X.shape[0]
    Mx = M.repeat_interleave(nch, dim=0) if M.shape[0] * nch == tap.shape[0] and M.shape[0] == sep.nsrc else M
    Xp = X.repeat(Mx.shape[0] // nch, 1, 1)                                # plane (s, c) -> X of channel c
    MX = torch.view_as_real(Xp) * Mx[..., None]
    F = sep.model.F
    assert same_values(MX[:, :, :F].cpu().numpy(), np.ascontiguousarray(tap).view(np.float32).reshape(MX[:, :, :F].shape))
    L = np.asarray(audio).shape[0]
    want = sep.stft.inverse(torch.view_as_complex(MX.contiguous()), num_out=L).cpu().numpy()
    got = np.asarray(stems)
    if got.ndim == 3:                                                        # [L, nsrc, 2] -> planes (source, channel)
        got = np.ascontiguousarray(got.transpose(1, 2, 0).reshape(-1, L))
    assert same_bits(got, want)
    Mh = M[:, :, :F].cpu().numpy()
    assert Mh.min() >= 0 and Mh.max() <= MASK_MAX and Mh.std() > 0.01
    return M


# ---------------------------------------------------------------------------------------------- 1. bit for bit
@pytest.mark.parametrize("simt", ["0", "1"])
@pytest.mark.parametrize("N", [1024, 2048])
def test_dsd_bits(N, simt, monkeypatch):
    monkeypatch.setenv("DCS_DEBUG_SIMT_GEMM", simt)
    _, sep = separator("dsd", N, 512, seed=N + 1)
    mix, _ = pipeline.synth_mixture(2.0, 11 + N)
    check_bits(sep, mix)


@pytest.mark.parametrize("arch", ["ikala", "ikala_nopool"])
def test_ikala_bits(arch):
    _, sep = separator(arch, 1024, 512, overlap=20)
    mix, _ = pipeline.synth_mixture(2.0, 13)
    mix[20000:40000] = 0.0
    check_bits(sep, mix)


@pytest.mark.parametrize("simt", ["0", "1"])
def test_bach10_bits(simt, monkeypatch):
    monkeypatch.setenv("DCS_DEBUG_SIMT_GEMM", simt)
    _, sep = separator("bach10", 256, 128, win="blackmanharris")
    mix, _ = pipeline.synth_mixture(1.0, 21)
    check_bits(sep, mix)


@pytest.mark.parametrize("arch", ["bach10_score", "bach10_score_1x1"])
def test_score_bits_filters_and_notes(arch):
    N, hop = (256, 128) if arch == "bach10_score" else (512, 256)
    _, sep = separator(arch, N, hop, win="blackmanharris", patcher="util", scale_factor=0.2)
    mix, _ = pipeline.synth_mixture(1.5, 23)
    T, F = dsp.num_frames(mix.size, hop), N // 2 + 1
    check_bits(sep, mix, {"filters": score_filters(T, F)}, {"filters": score_filters(T, F)})
    mel = melody_table(T + 40, F)
    for frame0 in (0, 17):
        check_bits(sep, mix, {"melody": mel, "frame0": frame0}, {"melody": mel, "frame0": frame0})


def test_score_1x1_bits_across_decoder_chunks():
    """P > 128 patches: the masks of every decoder chunk's frames"""
    N, hop, overlap, tc = 512, 256, 25, 30
    _, sep = separator("bach10_score_1x1", N, hop, seed=9, win="blackmanharris", patcher="util", scale_factor=0.2, tc=tc)
    mix, _ = pipeline.synth_mixture(4.0, 5)
    T = dsp.num_frames(mix.size, hop)
    assert sep.num_patches(T) > 128
    f = score_filters(T, N // 2 + 1)
    check_bits(sep, mix, {"filters": f}, {"filters": f})


def test_ild_bits():
    _, sep = separator("dsd_ild", 1024, 512, patcher="util")
    a, _ = pipeline.synth_mixture(2.0, 31)
    b, _ = pipeline.synth_mixture(2.0, 32)
    check_bits(sep, np.stack([a, 0.3 * a + 0.7 * b], axis=1).astype(np.float32))


@pytest.mark.parametrize("N", [1024, 2048])
def test_keep_channels_from_the_downmix_masks(N):
    _, sep = separator("dsd", N, 512, seed=7)
    a, _ = pipeline.synth_mixture(2.0, 41)
    b, _ = pipeline.synth_mixture(2.0, 42)
    audio = np.stack([0.7 * a + 0.3 * b, 0.4 * a + 0.6 * np.roll(b, 11)], axis=1).astype(np.float32)
    mono = (audio[:, 0] + audio[:, 1]) * np.float32(0.5)
    check_bits(sep, audio, None, {"keep_channels": True, "wiener": 0}, masks_audio=mono)


# ---------------------------------------------------------------------------------------------- 2. against float64
def compare(name, got, want, mag, kmap, silent_max=None):
    """got float32 / want float64 [nsrc, T, F], mag [T, F] (|X| up to a scale), kmap flagged bins [T, F]"""
    keep = ~kmap
    w2 = (np.asarray(mag, dtype=np.float64) ** 2)[keep]
    d = got.astype(np.float64) - want
    wrel = [float(np.sqrt((w2 * d[s][keep] ** 2).sum() / max((w2 * want[s][keep] ** 2).sum(), 1e-300))) for s in range(len(got))]
    rel = [float(np.linalg.norm(d[s][keep]) / max(np.linalg.norm(want[s][keep]), 1e-300)) for s in range(len(got))]
    mx = [float(np.abs(d[s][keep]).max()) for s in range(len(got))]
    rec = dict(kind="masks", weighted_rel_l2=wrel, rel_l2=rel, max_abs=mx, flagged_bins=int(kmap.sum()), total_bins=int(kmap.size))
    silent = (np.asarray(mag) == 0) & keep
    if silent_max is not None:
        rec["silent_bins"] = int(silent.sum())
        rec["silent_max_abs"] = float(np.abs(d[:, silent]).max())
    record(name, **rec)
    assert got.min() >= 0 and got.max() <= MASK_MAX
    assert int(kmap.sum()) <= 1e-4 * kmap.size + 8
    for s in range(len(got)):
        assert wrel[s] <= TOL, (name, s, wrel[s])
    if silent_max is not None:
        assert silent.sum() > 1000 and rec["silent_max_abs"] <= silent_max, rec


def host_masks(sep, audio, **kw):
    return sep.separate_masks(np.asarray(audio, dtype=np.float32) if np.asarray(audio).ndim == 1 else audio, **kw)


@pytest.mark.parametrize("arch,N,hop,win,winfn,overlap,patcher", [
    ("dsd", 1024, 512, "hanning", np.hanning, 25, "standalone"),
    ("ikala_nopool", 1024, 512, "hanning", np.hanning, 20, "util"),
    ("bach10", 256, 128, "blackmanharris", dsp.blackmanharris, 25, "standalone")])
def test_single_channel_nets_match_float64(arch, N, hop, win, winfn, overlap, patcher):
    params, sep = separator(arch, N, hop, seed=6, overlap=overlap, patcher=patcher, win=win)
    mix, _ = pipeline.synth_mixture(1.5, 61)
    got = host_masks(sep, mix)
    want, mag, _, kmap = mo.separate_masks(mix, params, arch, frameSize=N, hopSize=hop, window=winfn, overlap=overlap,
                                           patcher=patcher)
    assert got.shape == want.shape == (sep.nsrc,) + mag.shape and got.dtype == np.float32
    compare("masks_%s_N%d" % (arch, N), got, want, mag, kmap)


def test_ikala_pooled_with_silence_matches_float64():
    """|X| = 0 over a silent segment: the masks are defined there and must match to 1e-4 absolute"""
    params, sep = separator("ikala", 1024, 512, seed=5, overlap=20)
    mix, _ = pipeline.synth_mixture(3.0, 70 + 513)
    mix[20000:40000] = 0.0
    _, _, bits = sep.separate_tapped(mix, pool=True)
    got = host_masks(sep, mix)
    want, mag, _, kmap = mo.separate_masks(mix, params, "ikala", overlap=20, pool_bits=bits)
    compare("masks_ikala_silence", got, want, mag, kmap, silent_max=1e-4)


def test_score_build_ca_matches_float64():
    params, sep = separator("bach10_score", 256, 128, seed=8, win="blackmanharris", patcher="util", scale_factor=0.2)
    mix, _ = pipeline.synth_mixture(1.5, 63)
    f = score_filters(dsp.num_frames(mix.size, 128), 129)
    got = host_masks(sep, mix, filters=f)
    want, chsum, _, kmap = mo.separate_score_masks(mix, f, params, frameSize=256, hopSize=128)
    compare("masks_bach10_score", got, want, chsum, kmap)


def test_score_1x1_matches_float64():
    params, sep = separator("bach10_score_1x1", 512, 256, seed=7, win="blackmanharris", patcher="util", scale_factor=0.2)
    mix, _ = pipeline.synth_mixture(1.5, 91)
    f = score_filters(dsp.num_frames(mix.size, 256), 257)
    _, _, codes = sep.separate_tapped(mix, f, pool=True)
    got = host_masks(sep, mix, filters=f)
    want, chsum, _, kmap = mo.separate_score_1x1_masks(mix, f, params, frameSize=512, hopSize=256, gate_codes_dev=codes)
    compare("masks_bach10_score_1x1", got, want, chsum, kmap)


def test_ild_matches_float64():
    params, sep = separator("dsd_ild", 1024, 512, seed=5, patcher="util")
    a, _ = pipeline.synth_mixture(1.5, 3)
    b, _ = pipeline.synth_mixture(1.5, 4)
    audio = np.stack([a, 0.5 * a + 0.5 * b], axis=1)
    got = sep.separate_masks(audio)
    want, mag, _, kmaps = mo.separate_stereo_masks(audio, params)
    assert got.shape == want.shape and got.dtype == np.float32
    for c in range(2):
        compare("masks_dsd_ild_ch%d" % c, got[:, c], want[:, c], mag[c], kmaps[c])


# ---------------------------------------------------------------------------------------------- 3. fences
def raw_call(sep, x, buf, m_stride, **kw):
    from deepconvsep_b200 import _lib
    from deepconvsep_b200.engine import _ptr
    L = x.shape[-1]
    stride = x.stride(0) if x.dim() == 2 else L
    return _lib.check(sep.lib.dcs_separate_masks(sep.ctx.handle, sep.model.handle, sep.stft.handle, _ptr(x), stride, L,
                                                 C.c_float(sep.scale_factor), sep.overlap, sep.patcher, _ptr(buf), m_stride,
                                                 None))


@pytest.mark.parametrize("arch", ["dsd", "dsd_ild"])
def test_fences_determinism_wiener_and_short_clips(arch):
    _, sep = separator(arch, 1024, 512, patcher="util" if arch == "dsd_ild" else "standalone")
    a, _ = pipeline.synth_mixture(2.0, 81)
    b, _ = pipeline.synth_mixture(2.0, 82)
    audio = np.stack([a, 0.5 * (a + b)]) if arch == "dsd_ild" else a[None]
    x = torch.tensor(audio.astype(np.float32), device="cuda").squeeze(0)
    L, F, ldf = audio.shape[-1], sep.model.F, sep.stft.ldf
    T = sep.stft.num_frames(L)
    nplanes = sep.nsrc * (2 if arch == "dsd_ild" else 1)
    m_stride = T * ldf + 37
    outs = []
    for wiener in (0, 0, 2):
        sep.ctx.set_wiener(wiener)
        buf = torch.full((nplanes * m_stride + 64,), float("nan"), dtype=torch.float32, device="cuda")
        raw_call(sep, x, buf, m_stride)
        h = buf.cpu().numpy()
        planes = np.stack([h[p * m_stride:p * m_stride + T * ldf].reshape(T, ldf) for p in range(nplanes)])
        assert np.isfinite(planes[:, :, :F]).all() and np.isnan(planes[:, :, F:]).all()
        for p in range(nplanes):
            assert np.isnan(h[p * m_stride + T * ldf:(p + 1) * m_stride]).all()          # gaps and the sentinels
        assert np.isnan(h[nplanes * m_stride:]).all()
        outs.append(h)
    assert same_bits(outs[0], outs[1]) and same_bits(outs[0], outs[2])
    sep.ctx.set_wiener(0)
    # the device planes of separate_masks are those bits
    got = sep.separate_masks(x)
    assert same_bits(got[:, :, :F].cpu().numpy(), np.stack([outs[0][p * m_stride:p * m_stride + T * ldf].reshape(T, ldf)[:, :F]
                                                            for p in range(nplanes)]))
    # shorter than one patch: all-zero masks, the pads untouched
    xs = x[..., :5000].contiguous()
    Ts = sep.stft.num_frames(5000)
    buf = torch.full((nplanes * Ts * ldf,), float("nan"), dtype=torch.float32, device="cuda")
    raw_call(sep, xs, buf, Ts * ldf)
    h = buf.cpu().numpy().reshape(nplanes, Ts, ldf)
    assert sep.num_patches(Ts) == 0 and (h[:, :, :F] == 0).all() and np.isnan(h[:, :, F:]).all()


# ---------------------------------------------------------------------------------------------- 4. refusals
def test_refusals_queue_nothing():
    from deepconvsep_b200 import _lib
    from deepconvsep_b200.engine import Model, Stft, _ptr
    _, sep = separator("dsd", 1024, 512)
    ctx, lib = sep.ctx, sep.lib
    mix, _ = pipeline.synth_mixture(1.0, 5)
    L = mix.size
    T, ldf = sep.stft.num_frames(L), sep.stft.ldf
    x = torch.tensor(mix.astype(np.float32), device="cuda")
    buf = torch.zeros((4 * T * ldf,), dtype=torch.float32, device="cuda")
    filt = torch.zeros((4, T, ldf), dtype=torch.float32, device="cuda")
    mel = melody_table(T, 513)
    score = Model(ctx, nets.make_synthetic_params("bach10_score", 513, seed=3), arch="bach10_score", feat_size=513)
    other_plan = Stft(ctx, 2048, 512, "hanning")
    ref = sep.separate_masks(x).clone()

    def masks(model=sep.model, plan=sep.stft, audio=x, out=buf, m_stride=T * ldf):
        return lib.dcs_separate_masks(ctx.handle, model.handle, plan.handle, _ptr(audio), L, L, C.c_float(0.3), 25, 0,
                                      _ptr(out), m_stride, None)

    def masks_score(model, f=filt):
        return lib.dcs_separate_masks_score(ctx.handle, model.handle, sep.stft.handle, _ptr(x), L, _ptr(f), C.c_float(0.2),
                                            25, 1, _ptr(buf), T * ldf, None)

    def masks_notes(model, m_stride=T * ldf):
        return lib.dcs_separate_masks_notes(ctx.handle, model.handle, sep.stft.handle, _ptr(x), L, mel.ctypes.data,
                                            mel.shape[1], mel.shape[2], 0, C.c_float(0.2), 25, 1, _ptr(buf), m_stride, None)
    refused = {
        "score net on dcs_separate_masks": lambda: masks(model=score),
        "dsd net on dcs_separate_masks_score": lambda: masks_score(sep.model),
        "dsd net on dcs_separate_masks_notes": lambda: masks_notes(sep.model),
        "m_stride < T * ldf": lambda: masks(m_stride=T * ldf - 1),
        "notes, m_stride < T * ldf": lambda: masks_notes(score, m_stride=T * ldf - 1),
        "NULL audio": lambda: masks(audio=None),
        "NULL masks": lambda: masks(out=None),
        "NULL filters": lambda: masks_score(score, f=None),
        "plan F != model F": lambda: masks(plan=other_plan),
    }
    for name, call in refused.items():
        torch.cuda.synchronize()
        n0 = ctx.launch_count()
        with pytest.raises(_lib.DcsError):
            _lib.check(call())
        assert ctx.launch_count() == n0, name
    with pytest.raises(ValueError):
        sep.separate_masks(mix, melody=mel)
    with pytest.raises(ValueError):
        sep.separate_masks(mix, filters=np.zeros((4, T, 513), dtype=np.float32))
    assert same_bits(sep.separate_masks(x)[:, :, :513].cpu().numpy(), ref[:, :, :513].cpu().numpy())


# ---------------------------------------------------------------------------------------------- 5. workspace
def test_workspace_holds_no_spectra():
    """180 s at N = 2048: the masks call's workspace is smaller than the stems call's by at least the spectra"""
    N, L = 2048, 180 * 44100
    params = nets.make_synthetic_params("dsd", N // 2 + 1, seed=1)
    x = torch.tensor(np.random.default_rng(0).uniform(-0.3, 0.3, L).astype(np.float32), device="cuda")
    _, a = separator("dsd", N, 512, params=params)
    _, b = separator("dsd", N, 512, params=params)
    a.separate_masks(x)
    b.separate_device(x)
    torch.cuda.synchronize()
    T, ldf = a.stft.num_frames(L), a.stft.ldf
    wm, ws = a.ctx.workspace_bytes(), b.ctx.workspace_bytes()
    record("masks_workspace_N2048_180s", masks_bytes=wm, stems_bytes=ws, spectra_bytes=4 * T * ldf * 8)
    assert ws - wm >= 4 * T * ldf * 8, (wm, ws)
