"""C-channel stems (dcs_separate_audio_channels, dcs_apply_masks; Separator.separate_channels / apply_masks): the
downmix's masks applied to each channel's STFT inside the inverse STFT.

- bit for bit: one channel against separate() for every single-channel family, two channels against
  separate_keep_channels (DSD100), apply_masks(separate_masks(downmix)) against separate_channels at C = 6;
- C = 6 on a 15 s clip against the float64 oracle of tests/channels_oracle.py at the plain bars (1e-4 relative L2, 0.01 dB
  SDR), the oracle adopting the device's mask -- read bit-exact from separate_masks on the same downmix -- at the bins
  its kink map flags, after checking 0 <= M <= 1, and only there (the rule of tests/parity.py with the mask in place of
  the spectrum tap);
- short clips, the workspace (independent of C, no masked spectra), the spectrum-tap refusal, the launch count, the
  argument refusals before anything is queued."""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from oracle import nets, pipeline  # noqa: E402
import channels_oracle as co  # noqa: E402
from parity import record, rel, istft_rows  # noqa: E402

TOL = 1e-4
MB = 1 << 20


def separator(arch, N, hop=512, seed=5, overlap=25, patcher="standalone", win="hanning", params=None):
    from deepconvsep_b200.engine import Separator
    F = N // 2 + 1
    if params is None:
        params = nets.make_synthetic_params(arch, F, seed=seed)
    return params, Separator(params, arch=arch, frame_size=N, hop=hop, window=win, overlap=overlap, patcher=patcher, feat_size=F)


def same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def channels(seconds, nch, seed):
    """nch channels of different gains and delays of two sources"""
    a, _ = pipeline.synth_mixture(seconds, seed)
    b, _ = pipeline.synth_mixture(seconds, seed + 1)
    rng = np.random.default_rng(seed)
    cols = []
    for c in range(nch):
        g, h = rng.uniform(-1.0, 1.0, 2)
        cols.append(g * np.roll(a, int(rng.integers(0, 60))) + h * np.roll(b, int(rng.integers(0, 60))))
    return (0.5 * np.stack(cols, axis=1)).astype(np.float32)


def rounded(nbytes):
    return (nbytes + MB - 1) // MB * MB


# ---------------------------------------------------------------------------------------------- 1. bit for bit
@pytest.mark.parametrize("arch,N,win,overlap", [("dsd", 1024, "hanning", 25), ("dsd", 2048, "hanning", 25),
                                                ("bach10", 4096, "blackmanharris", 25), ("ikala", 1024, "hanning", 20),
                                                ("ikala_nopool", 1024, "hanning", 20)])
def test_one_channel_is_the_mono_call(arch, N, win, overlap):
    _, sep = separator(arch, N, overlap=overlap, win=win)
    mix, _ = pipeline.synth_mixture(2.0, 11 + N)
    a = mix.astype(np.float32)
    want = sep.separate(a)                                   # [nsrc, L]
    got = sep.separate_channels(a[:, None])                  # [L, nsrc, 1]
    assert got.shape == (a.size, sep.nsrc, 1) and np.abs(want).max() > 0
    assert same_bits(got[:, :, 0].T, want)


@pytest.mark.parametrize("N", [1024, 2048])
def test_two_channels_are_keep_channels(N):
    _, sep = separator("dsd", N, seed=7)
    audio = channels(2.0, 2, 41)
    want = sep.separate_keep_channels(audio)
    got = sep.separate_channels(audio)
    assert got.shape == want.shape == (audio.shape[0], 4, 2) and same_bits(got, want)
    x = torch.tensor(np.ascontiguousarray(audio.T), device="cuda")
    assert same_bits(sep.separate_channels(x).cpu().numpy(), sep.separate_keep_channels(x).cpu().numpy())


@pytest.mark.parametrize("arch,N,win", [("dsd", 2048, "hanning"), ("bach10", 4096, "blackmanharris")])
def test_apply_masks_of_the_downmix_masks_is_separate_channels(arch, N, win):
    _, sep = separator(arch, N, win=win)
    audio = channels(2.0, 6, 51)
    x = torch.tensor(np.ascontiguousarray(audio.T), device="cuda")
    mono = x[0]
    for c in range(1, 6):
        mono = mono + x[c]
    masks = sep.separate_masks((mono * float(np.float32(1.0) / np.float32(6.0))).contiguous())     # 1.0f / nx, in fp32
    want = sep.separate_channels(x)
    got = sep.apply_masks(x, masks)
    assert tuple(got.shape) == (sep.nsrc * 6, audio.shape[0]) and float(want.abs().max()) > 0
    assert same_bits(got.cpu().numpy(), want.cpu().numpy())
    # the numpy layouts of both calls
    h = sep.apply_masks(audio, masks[:, :, :sep.model.F].cpu().numpy())
    assert same_bits(h, sep.separate_channels(audio))
    assert same_bits(h, want.cpu().numpy().reshape(sep.nsrc, 6, -1).transpose(2, 0, 1))
    # edited masks, a source count of the caller's own
    one = sep.apply_masks(x, torch.ones_like(masks[:1]))
    assert tuple(one.shape) == (6, audio.shape[0]) and rel(one.cpu().numpy(), audio.T.astype(np.float64)) < 1e-5


# ---------------------------------------------------------------------------------------------- 2. against float64
def sdr_db(ref, est):
    return 10.0 * np.log10(np.sum(ref ** 2) / max(np.sum((ref - est) ** 2), 1e-300))


def test_six_channels_match_float64():
    N, hop, nch = 1024, 512, 6
    params, sep = separator("dsd", N, seed=6)
    audio = channels(15.0, nch, 61)
    L = audio.shape[0]
    got = sep.separate_channels(audio)                                     # [L, nsrc, C]
    stems, mags, phs, mms, masks, kmap = co.separate_channels(audio, params, frameSize=N, hopSize=hop)
    T, F = kmap.shape
    # the device's masks of the same downmix, bit-exact
    x = torch.tensor(np.ascontiguousarray(audio.T), device="cuda")
    mono = x[0]
    for c in range(1, nch):
        mono = mono + x[c]
    Mdev = sep.separate_masks((mono * float(np.float32(1.0) / np.float32(nch))).contiguous())[:, :, :F].cpu().numpy().astype(np.float64)
    nflag = int(kmap.sum())
    assert nflag <= 1e-4 * kmap.size + 8
    tt, ff = np.nonzero(kmap)
    assert np.all(Mdev[:, tt, ff] >= 0) and np.all(Mdev[:, tt, ff] <= 1 + 2.0 ** -20)
    rows = sorted(set(int(t) for t in tt))
    win = np.hanning(N)
    errs, raws, dsdr = [], [], []
    for c in range(nch):
        Xc = (mags[c].astype(np.float64) / 0.3) * np.sqrt(N) * np.exp(1j * phs[c])
        for s in range(sep.nsrc):
            want = stems[:, s, c]
            raws.append(rel(got[:, s, c], want))
            if nflag:
                S_or = (mms[c][s, :T] / 0.3) * np.sqrt(N) * np.exp(1j * phs[c])
                D = np.zeros((T, F), dtype=np.complex128)
                D[tt, ff] = Mdev[s, tt, ff] * Xc[tt, ff] - S_or[tt, ff]
                want = want + istft_rows(D, rows, win, hop, N, L)
            errs.append(rel(got[:, s, c], want))
            # SDR of the stem against a reference signal, device versus oracle
            ref = audio[:, c].astype(np.float64)
            dsdr.append(abs(sdr_db(ref, got[:, s, c].astype(np.float64)) - sdr_db(ref, want)))
    record("channels_dsd_N1024_C6_15s", kind="channels", channels=nch, seconds=L / 44100.0, flagged_bins=nflag,
           total_bins=int(kmap.size), rel_l2=errs, rel_l2_unmodified=raws, sdr_diff_db=dsdr, tol=TOL)
    assert max(errs) <= TOL, (max(errs), max(raws), nflag)
    assert max(dsdr) <= 0.01, max(dsdr)


# ---------------------------------------------------------------------------------------------- 3. pipeline rules
def test_clip_shorter_than_one_patch_gives_zeros():
    _, sep = separator("dsd", 1024)
    audio = channels(0.1, 3, 71)
    assert sep.num_patches(sep.stft.num_frames(audio.shape[0])) == 0
    got = sep.separate_channels(audio)
    assert got.shape == (audio.shape[0], 4, 3) and not got.any()


def test_workspace_is_independent_of_the_channel_count_and_the_tap_is_refused():
    from deepconvsep_b200 import _lib
    N, L = 2048, 30 * 44100
    params = nets.make_synthetic_params("dsd", N // 2 + 1, seed=1)
    rng = np.random.default_rng(0)
    x6 = torch.tensor(rng.uniform(-0.3, 0.3, (6, L)).astype(np.float32), device="cuda")
    ws = {}
    for name, call in (("masks", lambda s: s.separate_masks(x6[0].contiguous())), ("c6", lambda s: s.separate_channels(x6)),
                       ("c2", lambda s: s.separate_channels(x6[:2].contiguous())),
                       ("keep", lambda s: s.separate_keep_channels(x6[:2].contiguous()))):
        _, sep = separator("dsd", N, params=params)
        call(sep)
        torch.cuda.synchronize()
        ws[name] = sep.ctx.workspace_bytes()
    T, ldf = sep.stft.num_frames(L), sep.stft.ldf
    plane = T * ldf
    # the masks call's buffers (magnitude, network) + the downmix, ONE mixture STFT plane and the nsrc mask planes
    assert ws["c6"] == ws["masks"] + rounded(4 * L) + rounded(8 * plane) + rounded(4 * 4 * plane), ws
    assert ws["c6"] == ws["c2"] == ws["keep"]              # keep-channels is the C = 2 path
    record("channels_workspace_N2048_30s", **ws)
    # a spectrum tap on the ctx: refused before anything is queued
    tap = torch.zeros((4, T, ldf), dtype=torch.complex64, device="cuda")
    _lib.check(sep.lib.dcs_set_spectrum_tap(sep.ctx.handle, tap.data_ptr(), tap.numel()))
    n0 = sep.ctx.launch_count()
    try:
        with pytest.raises(_lib.DcsError, match="spectrum tap"):
            sep.separate_channels(x6)
    finally:
        _lib.check(sep.lib.dcs_set_spectrum_tap(sep.ctx.handle, None, 0))
    assert sep.ctx.launch_count() == n0


@pytest.mark.parametrize("nch", [1, 2, 6])
def test_launch_count(nch):
    _, sep = separator("dsd", 1024)
    audio = channels(2.0, nch, 81)
    x = torch.tensor(np.ascontiguousarray(audio.T), device="cuda")
    sep.separate_masks(x[0].contiguous())                 # warm: buffers allocated
    n0 = sep.ctx.launch_count()
    sep.separate_masks(x[0].contiguous())
    masks_launches = sep.ctx.launch_count() - n0
    sep.separate_channels(x)
    n1 = sep.ctx.launch_count()
    sep.separate_channels(x)
    assert sep.ctx.launch_count() - n1 == masks_launches + 1 + 2 * nch


def test_wiener_setting_is_ignored():
    _, sep = separator("dsd", 1024)
    audio = channels(2.0, 2, 91)
    want = sep.separate_channels(audio)
    sep.ctx.set_wiener(2)
    try:
        assert same_bits(sep.separate_channels(audio), want)
    finally:
        sep.ctx.set_wiener(0)


def test_refusals_queue_nothing():
    from deepconvsep_b200 import _lib
    from deepconvsep_b200.engine import Model, Stft, _ptr
    _, sep = separator("dsd", 1024)
    ctx, lib = sep.ctx, sep.lib
    L = 30000
    T, ldf = sep.stft.num_frames(L), sep.stft.ldf
    x = torch.zeros((3, L), dtype=torch.float32, device="cuda")
    out = torch.zeros((12, L), dtype=torch.float32, device="cuda")
    masks = torch.zeros((4, T, ldf), dtype=torch.float32, device="cuda")
    score = Model(ctx, nets.make_synthetic_params("bach10_score", 513, seed=3), arch="bach10_score", feat_size=513)
    ild = Model(ctx, nets.make_synthetic_params("dsd_ild", 513, seed=3), arch="dsd_ild", feat_size=513)
    other_plan = Stft(ctx, 2048, 512, "hanning")

    def chans(model=sep.model, plan=sep.stft, audio=x, nx=3, stride=L, n=L, overlap=25, patcher=0, o=out, ostride=L):
        return lib.dcs_separate_audio_channels(ctx.handle, model.handle, plan.handle, _ptr(audio), nx, stride, n, C.c_float(0.3),
                                               overlap, patcher, _ptr(o), ostride, None)

    def apply(plan=sep.stft, audio=x, nx=3, stride=L, n=L, m=masks, nsrc=4, m_stride=T * ldf, o=out, ostride=L, mp=None):
        return lib.dcs_apply_masks(ctx.handle, plan.handle, _ptr(audio), nx, stride, n, _ptr(m) if mp is None else mp, nsrc,
                                   m_stride, _ptr(o), ostride, None)
    refused = {
        "score net": (lambda: chans(model=score), "dcs_apply_masks"), "stereo net": (lambda: chans(model=ild), "dcs_separate_masks"),
        "nx 0": (lambda: chans(nx=0), "nx"), "nx 17": (lambda: chans(nx=17), "nx"), "NULL audio": (lambda: chans(audio=None), "NULL"),
        "NULL stems": (lambda: chans(o=None), "NULL"), "audio_stride < L": (lambda: chans(stride=L - 1), "stride"),
        "stem_stride < L": (lambda: chans(ostride=L - 1), "stride"), "no samples": (lambda: chans(n=0), "length"),
        "overlap": (lambda: chans(overlap=30), "overlap"), "patcher": (lambda: chans(patcher=7), "patcher"),
        "plan F != model F": (lambda: chans(plan=other_plan), "bins"),
        "apply: nx 0": (lambda: apply(nx=0), "nx"), "apply: nx 17": (lambda: apply(nx=17), "nx"),
        "apply: nsrc 0": (lambda: apply(nsrc=0), "nsrc"), "apply: NULL masks": (lambda: apply(m=None), "NULL"),
        "apply: NULL audio": (lambda: apply(audio=None), "NULL"), "apply: m_stride": (lambda: apply(m_stride=T * ldf - 1), "m_stride"),
        "apply: masks misaligned": (lambda: apply(mp=masks.data_ptr() + 2), "d_masks"),
        "apply: audio_stride < L": (lambda: apply(stride=L - 1), "stride"), "apply: stem_stride < L": (lambda: apply(ostride=L - 1), "stride"),
        "apply: no samples": (lambda: apply(n=0), "length"),
    }
    torch.cuda.synchronize()
    for name, (call, word) in refused.items():
        n0 = ctx.launch_count()
        assert call() == -1, name
        assert word in lib.dcs_last_error().decode(), (name, lib.dcs_last_error())
        assert ctx.launch_count() == n0, name
    assert chans() == 0 and apply() == 0
    torch.cuda.synchronize()
