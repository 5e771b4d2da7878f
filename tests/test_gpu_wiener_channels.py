"""The C-channel Wiener post-filter on the GPU (dcs_wiener_channels, dcs_separate_audio_channels_wiener;
engine.wiener_channels, Separator.separate_channels(wiener=...)) against the float64 oracle of
tests/wiener_channels_oracle.py:

- spectra: C in {3, 6, 8}, nsrc in {1, 2, 4}, K in {1, 2, 3}, radius in {0, 1, 3}, F in {513, 1025}, a partial last
  chunk, per-plane relative L2 <= 1e-5 (the bar of test_gpu_wiener.py); NaN in pad bins and plane gaps untouched,
  all-zero frames stay 0, the same bytes on a second run;
- exact: nx = 2 is dcs_wiener_stereo_windowed, radius >= n-1 is radius 0, a chunk does not see frames more than K*W
  chunks away;
- structure at C = 6: equal channels give the closed form, permuting the channels permutes the output;
- bookkeeping: 2K + 1 launches, refusals queue nothing;
- pipeline: wiener 0 is separate_channels, C = 2 DSD is keep-channels with the filter, C = 2 iKala and C = 6 (DSD,
  iKala) on 15 s against float64, the spectrum tap, the workspace formula of dcs.h, a 180 s C = 8 run."""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from oracle import dsp, nets, pipeline  # noqa: E402
import wiener_channels_oracle as wco  # noqa: E402
from parity import record  # noqa: E402

SPEC_BAR, STEM_BAR = 1e-5, 1e-4
MB = 1 << 20
NAN = complex(float("nan"), float("nan"))


def rel(a, b):
    return float(np.linalg.norm(np.asarray(a, np.complex128) - b) / max(np.linalg.norm(b), 1e-30))


def rounded(nbytes):
    return (nbytes + MB - 1) // MB * MB


def spectra(nx, nsrc, T, F, seed, silent=()):
    """X [nx, T, F] and soft-mask stems [nsrc, nx, T, F] (complex128, float32-representable): nsrc sources, each
    reaching channel c with its own gain and delay (a phase ramp over the bins), so R_j has complex off-diagonal terms.
    Frames in `silent` have every stem zero."""
    rng = np.random.default_rng(seed)
    src = (rng.standard_normal((nsrc, T, F)) + 1j * rng.standard_normal((nsrc, T, F))) \
        * rng.uniform(0.01, 1.0, (nsrc, 1, F)) * rng.gamma(0.3, 1.0, (nsrc, T, F))
    gain = rng.uniform(0.1, 1.0, (nsrc, nx, 1, 1))
    delay = rng.uniform(0.0, 40.0, (nsrc, nx, 1, 1))
    img = gain * np.exp(-1j * np.pi * np.arange(F) * delay / (F - 1)) * src[:, None] * 40.0
    X = img.sum(axis=0).astype(np.complex64)
    mag = np.abs(img).sum(axis=1) * rng.uniform(1.0, 1.8, (nsrc, T, F))
    Y = ((mag / mag.sum(axis=0))[:, None] * X[None]).astype(np.complex64)
    Y[:, :, list(silent)] = 0
    return X.astype(np.complex128), Y.astype(np.complex128)


def planes(a, ldf, gap):
    """a [n, T, F] -> a device view [n, T, ldf] of planes T * ldf + gap apart, with NaN in the pad bins and gaps, and
    the buffer under it"""
    n, T, F = a.shape
    buf = torch.full((n, T * ldf + gap), NAN, dtype=torch.complex64, device="cuda")
    v = buf[:, :T * ldf].view(n, T, ldf)
    v[:, :, :F] = torch.tensor(a.astype(np.complex64), device="cuda")
    return v, buf


def filt(ctx, X, S, K, F, radius):
    from deepconvsep_b200.engine import wiener_channels
    wiener_channels(ctx, X, S, K, num_bins=F, radius=radius)
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------- 1. spectra
CASES = [(3, 1, 1, 0, 513), (3, 2, 2, 1, 1025), (3, 4, 3, 3, 513), (6, 1, 2, 3, 1025), (6, 2, 3, 0, 513),
         (6, 4, 1, 1, 1025), (8, 1, 3, 1, 513), (8, 2, 1, 3, 1025), (8, 4, 2, 0, 1025)]


@pytest.mark.parametrize("nx,nsrc,K,radius,F", CASES)
def test_spectra_match_the_oracle(nx, nsrc, K, radius, F):
    from deepconvsep_b200.engine import Context
    T, ldf, gap = 700, F + 7, 24                            # 5 full chunks and one of 60 frames
    silent = range(650, 700)
    X, Y = spectra(nx, nsrc, T, F, seed=nx * 100 + nsrc * 10 + K, silent=silent)
    ctx = Context(0)
    Xd, Xbuf = planes(X, ldf, gap)
    Sd, Sbuf = planes(Y.reshape(nsrc * nx, T, F), ldf, gap)
    S0 = Sbuf.clone()
    n0 = ctx.launch_count()
    filt(ctx, Xd, Sd, K, F, radius)
    assert ctx.launch_count() - n0 == 2 * K + 1
    got = Sd[:, :, :F].cpu().numpy()
    want = wco.wiener(X, Y, K, radius).reshape(nsrc * nx, T, F)
    errs = [rel(got[p], want[p]) for p in range(nsrc * nx)]
    record("wiener_channels_C%d_nsrc%d_K%d_W%d_F%d" % (nx, nsrc, K, radius, F), max_rel=max(errs), per_plane=errs)
    assert max(errs) <= SPEC_BAR, errs
    assert not got[:, 650:].any()                                           # all-zero frames stay 0
    assert all(rel(got[p], Y.reshape(-1, T, F)[p]) > 1e-4 for p in range(nsrc * nx) if nsrc > 1)   # it did filter
    # pad bins and the gaps between planes: never touched (NaN stays NaN, bit for bit)
    a, b = S0.view(torch.float32).view(torch.int32), Sbuf.view(torch.float32).view(torch.int32)
    assert torch.equal(a[:, T * ldf * 2:], b[:, T * ldf * 2:])
    pa = a[:, :T * ldf * 2].view(-1, T, ldf, 2)[:, :, F:]
    pb = b[:, :T * ldf * 2].view(-1, T, ldf, 2)[:, :, F:]
    assert torch.equal(pa, pb)
    # the same bytes on a second run
    Sd2, Sbuf2 = planes(Y.reshape(nsrc * nx, T, F), ldf, gap)
    filt(ctx, Xd, Sd2, K, F, radius)
    assert torch.equal(Sbuf2.view(torch.int64), Sbuf.view(torch.int64))


# ---------------------------------------------------------------------------------------------- 2. exact
@pytest.mark.parametrize("radius", [0, 2])
def test_two_channels_are_the_stereo_filter(radius):
    from deepconvsep_b200.engine import Context, wiener_stereo
    T, F, ldf = 600, 513, 520
    X, Y = spectra(2, 4, T, F, seed=3 + radius)
    ctx = Context(0)
    Xd, _ = planes(X, ldf, 0)
    Sa, _ = planes(Y.reshape(8, T, F), ldf, 0)
    Sb = Sa.clone()
    filt(ctx, Xd, Sa, 2, F, radius)
    wiener_stereo(ctx, Xd, Sb, 2, num_bins=F, radius=radius)
    torch.cuda.synchronize()
    assert torch.equal(Sa.view(torch.int64), Sb.view(torch.int64))


def test_radius_covering_the_clip_is_radius_zero_and_windows_are_local():
    from deepconvsep_b200.engine import Context
    T, F, ldf, nx, K, W = 128 * 8, 513, 520, 6, 2, 1
    X, Y = spectra(nx, 2, T, F, seed=17)
    ctx = Context(0)
    Xd, _ = planes(X, ldf, 0)
    Y = Y.reshape(2 * nx, T, F)
    runs = {}
    for radius in (0, 7, 30):
        Sd, _ = planes(Y, ldf, 0)
        filt(ctx, Xd, Sd, K, F, radius)
        runs[radius] = Sd.view(torch.int64).clone()
    assert torch.equal(runs[7], runs[0]) and torch.equal(runs[30], runs[0])
    # change chunk 7 (mixture and stems): chunks 0 .. 7 - K*W - 1 keep their bytes, and the change does reach chunk 6
    Sd, _ = planes(Y, ldf, 0)
    filt(ctx, Xd, Sd, K, F, W)
    before = Sd.view(torch.int64).clone()
    X2, Y2 = X.copy(), Y.copy()
    X2[:, 7 * 128:] *= 3.0
    Y2[:, 7 * 128:] *= np.linspace(0.5, 1.5, F)
    Xd2, _ = planes(X2, ldf, 0)
    Sd2, _ = planes(Y2, ldf, 0)
    filt(ctx, Xd2, Sd2, K, F, W)
    after = Sd2.view(torch.int64)
    keep = (7 - K * W) * 128
    assert torch.equal(after[:, :keep], before[:, :keep])
    assert not torch.equal(after[:, 6 * 128:7 * 128], before[:, 6 * 128:7 * 128])


# ---------------------------------------------------------------------------------------------- 3. structure at C = 6
def test_equal_channels_give_the_closed_form():
    from deepconvsep_b200.engine import Context
    T, F, ldf, nx = 400, 513, 520, 6
    X2, Y2 = spectra(1, 4, T, F, seed=23)
    a, b = X2[0], Y2[:, 0]
    X = np.repeat(a[None], nx, axis=0)
    Y = np.repeat(b[:, None], nx, axis=1)
    ctx = Context(0)
    Xd, _ = planes(X, ldf, 0)
    Sd, _ = planes(Y.reshape(4 * nx, T, F), ldf, 0)
    filt(ctx, Xd, Sd, 2, F, 0)
    got = Sd[:, :, :F].cpu().numpy().reshape(4, nx, T, F)
    want = wco.equal_channels(a, b, nx, 2)
    errs = [rel(got[j, c], want[j]) for j in range(4) for c in range(nx)]
    record("wiener_channels_equal_C6", errs=errs)
    assert max(errs) <= 1e-6, errs


def test_permuting_the_channels_permutes_the_output():
    from deepconvsep_b200.engine import Context
    T, F, ldf, nx = 400, 513, 520, 6
    X, Y = spectra(nx, 4, T, F, seed=29)
    perm = [4, 2, 0, 5, 1, 3]
    ctx = Context(0)
    out = []
    for x, y in ((X, Y), (X[perm], Y[:, perm])):
        Xd, _ = planes(x, ldf, 0)
        Sd, _ = planes(y.reshape(4 * nx, T, F), ldf, 0)
        filt(ctx, Xd, Sd, 2, F, 1)
        out.append(Sd[:, :, :F].cpu().numpy().reshape(4, nx, T, F))
    errs = [rel(out[1][j, c], out[0][j, perm[c]]) for j in range(4) for c in range(nx)]
    assert max(errs) <= 1e-6, errs


# ---------------------------------------------------------------------------------------------- 4. bookkeeping
def test_refusals_queue_nothing():
    from deepconvsep_b200 import _lib
    from deepconvsep_b200.engine import Context, _ptr
    ctx = Context(0)
    lib = ctx.lib
    T, ldf, F = 300, 520, 513
    X = torch.zeros((9, T, ldf), dtype=torch.complex64, device="cuda")
    S = torch.zeros((36, T, ldf), dtype=torch.complex64, device="cuda")

    def call(x=X, nx=3, x_plane=T * ldf, s=S, src_stride=T * ldf, nsrc=4, t=T, ld=ldf, f=F, k=1, radius=0, sp=None):
        return lib.dcs_wiener_channels(ctx.handle, _ptr(x), nx, x_plane, _ptr(s) if sp is None else sp, src_stride, nsrc, t, ld,
                                       f, k, radius, None)
    refused = {
        "nx 1": lambda: call(nx=1), "nx 9": lambda: call(nx=9), "nx 0": lambda: call(nx=0),
        "negative iterations": lambda: call(k=-1), "negative radius": lambda: call(radius=-1),
        "nsrc 5": lambda: call(nsrc=5), "nsrc 0": lambda: call(nsrc=0),
        "x plane stride < T * ldf": lambda: call(x_plane=T * ldf - 1), "source stride < T * ldf": lambda: call(src_stride=T * ldf - 8),
        "T = 0": lambda: call(t=0), "F > ldf": lambda: call(f=ldf + 1), "NULL spectra": lambda: call(x=None),
        "misaligned stems": lambda: call(sp=S.data_ptr() + 4),
    }
    torch.cuda.synchronize()
    for name, fn in refused.items():
        n0 = ctx.launch_count()
        with pytest.raises(_lib.DcsError):
            _lib.check(fn())
        assert ctx.launch_count() == n0, name
    n0 = ctx.launch_count()
    assert call(k=0) == 0 and ctx.launch_count() == n0                     # 0 iterations: nothing to do
    for K in (1, 3):
        n0 = ctx.launch_count()
        assert call(nx=8, nsrc=4, k=K, radius=1) == 0
        assert ctx.launch_count() - n0 == 2 * K + 1
    torch.cuda.synchronize()
    # the pipeline entry: refusals before anything is queued
    sep = separator("dsd", 1024, 7)
    L = 30000
    x = torch.zeros((9, L), dtype=torch.float32, device="cuda")
    out = torch.zeros((36, L), dtype=torch.float32, device="cuda")

    def chans(nx=3, k=1, radius=0):
        return lib.dcs_separate_audio_channels_wiener(sep.ctx.handle, sep.model.handle, sep.stft.handle, _ptr(x), nx, L, L,
                                                      C.c_float(0.3), 25, 0, k, radius, _ptr(out), L, None)
    for name, fn in {"nx 1": lambda: chans(nx=1), "nx 9": lambda: chans(nx=9), "negative iterations": lambda: chans(k=-1),
                     "negative radius": lambda: chans(radius=-1), "nx 17 unfiltered": lambda: chans(nx=17, k=0)}.items():
        n0 = sep.ctx.launch_count()
        with pytest.raises(_lib.DcsError):
            _lib.check(fn())
        assert sep.ctx.launch_count() == n0, name
    for name, fn in {"python nx 1": lambda: sep.separate_channels(x[:1], wiener=1),
                     "python nx 9": lambda: sep.separate_channels(x, wiener=1),
                     "python orphan radius": lambda: sep.separate_channels(x[:3], wiener_radius=1)}.items():
        n0 = sep.ctx.launch_count()
        with pytest.raises(ValueError):
            fn()
        assert sep.ctx.launch_count() == n0, name


# ---------------------------------------------------------------------------------------------- 5. pipeline
OVERLAP = {"dsd": 25, "ikala": 20}


def separator(arch, N, seed):
    from deepconvsep_b200.engine import Separator
    params = nets.make_synthetic_params(arch, N // 2 + 1, seed=seed)
    return Separator(params, arch=arch, frame_size=N, hop=min(512, N // 2), window="hanning", overlap=OVERLAP[arch],
                     feat_size=N // 2 + 1)


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


def downmix_masks(sep, x):
    """the device masks of the fp32 downmix (((a_0 + a_1) + a_2) + ...) * (1.0f / nx), [nsrc, T, ldf]"""
    nx = x.shape[0]
    mono = x[0]
    for c in range(1, nx):
        mono = mono + x[c]
    return sep.separate_masks((mono * float(np.float32(1.0) / np.float32(nx))).contiguous())


def same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def test_wiener_zero_is_separate_channels_and_two_channels_are_keep_channels():
    sep = separator("dsd", 1024, 31)
    audio6 = channels(3.0, 6, 5)
    assert same_bits(sep.separate_channels(audio6, wiener=0), sep.separate_channels(audio6))
    audio = channels(8.0, 2, 7)                               # 690 frames: 6 chunks, so that W = 2 is a window
    for K in (1, 2):
        for W in (0, 2):
            want = sep.separate_keep_channels(audio, wiener=K, wiener_radius=W)
            got = sep.separate_channels(audio, wiener=K, wiener_radius=W)
            assert same_bits(got, want), (K, W)
            assert not same_bits(got, sep.separate_channels(audio))


def sdr_db(ref, est):
    return 10.0 * np.log10(np.sum(ref ** 2) / max(np.sum((ref - est) ** 2), 1e-300))


@pytest.mark.parametrize("arch,nx", [("ikala", 2), ("dsd", 6), ("ikala", 6)])
def test_15s_matches_float64(arch, nx):
    N, K, W = 1024, 2, 1
    sep = separator(arch, N, 61 + nx)
    hop = sep.hop
    audio = channels(15.0, nx, 71 + nx)
    L = audio.shape[0]
    F = N // 2 + 1
    got = sep.separate_channels(audio, wiener=K, wiener_radius=W)              # [L, nsrc, C]
    x = torch.tensor(np.ascontiguousarray(audio.T), device="cuda")
    M = downmix_masks(sep, x)[:, :, :F].cpu().numpy().astype(np.float64)      # bit-exact device masks
    win = np.hanning(N)
    X = np.stack([dsp.stft_norm(audio[:, c].astype(np.float64), win, hop, N) for c in range(nx)])
    T = X.shape[1]
    assert M.shape == (sep.nsrc, T, F)
    Y = wco.wiener(X, M[:, None] * X[None], K, W)
    errs, dsdr = [], []
    for j in range(sep.nsrc):
        for c in range(nx):
            want = dsp.istft_norm(Y[j, c], win, hopsize=hop, nfft=N)[:L]
            g = got[:, j, c].astype(np.float64)
            errs.append(float(np.linalg.norm(g - want) / np.linalg.norm(want)))
            ref = audio[:, c].astype(np.float64)
            dsdr.append(abs(sdr_db(ref, g) - sdr_db(ref, want)))
    record("wiener_channels_%s_C%d_15s" % (arch, nx), K=K, radius=W, rel_l2=errs, sdr_diff_db=dsdr)
    assert max(errs) <= STEM_BAR, errs
    assert max(dsdr) <= 0.01, dsdr
    plain = sep.separate_channels(audio)
    assert min(rel(got[:, j, c], plain[:, j, c]) for j in range(sep.nsrc) for c in range(nx)) > 1e-3    # the filter acted


def test_spectrum_tap_is_wiener_channels_of_the_masked_spectra():
    from deepconvsep_b200 import _lib
    from deepconvsep_b200.engine import wiener_channels
    nx, K, W = 4, 2, 1
    sep = separator("dsd", 1024, 41)
    audio = channels(6.0, nx, 43)
    L = audio.shape[0]
    x = torch.tensor(np.ascontiguousarray(audio.T), device="cuda")
    T, ldf, F = sep.stft.num_frames(L), sep.stft.ldf, sep.stft.F
    tap = torch.zeros((4 * nx, T, ldf), dtype=torch.complex64, device="cuda")
    _lib.check(sep.lib.dcs_set_spectrum_tap(sep.ctx.handle, tap.data_ptr(), tap.numel()))
    try:
        sep.separate_channels(x, wiener=K, wiener_radius=W)
        torch.cuda.synchronize()
    finally:
        _lib.check(sep.lib.dcs_set_spectrum_tap(sep.ctx.handle, None, 0))
    M = downmix_masks(sep, x)
    Xd = torch.stack([sep.stft.forward(x[c].contiguous(), want_mag=False)[0] for c in range(nx)])
    S = torch.empty((4, nx, T, ldf, 2), dtype=torch.float32, device="cuda")
    S[:] = torch.view_as_real(Xd)[None] * M[:, None, :, :, None]           # M_s * X_c componentwise in fp32
    S = torch.view_as_complex(S).reshape(4 * nx, T, ldf)
    wiener_channels(sep.ctx, Xd.contiguous(), S, K, num_bins=F, radius=W)
    torch.cuda.synchronize()
    assert torch.equal(tap[:, :, :F].view(torch.int64), S[:, :, :F].view(torch.int64))


def wiener_bytes(nsrc, nx, T, F, radius):
    """the filter's workspace stated in include/dcs.h (dcs_wiener_channels)"""
    n = -(-T // 128)
    P = nsrc * nx * nx * F
    q = n if radius > 0 else 1
    b = 128 if nx == 2 else 32
    return 8 * (n * P + q * P + n * -(-F // b) + q)


@pytest.mark.parametrize("seconds,nx,radius", [(30.0, 6, 0), (180.0, 8, 2)])
def test_workspace_formula(seconds, nx, radius):
    N, L = 2048, int(seconds * 44100)
    params = nets.make_synthetic_params("dsd", N // 2 + 1, seed=1)
    rng = np.random.default_rng(0)
    x = torch.tensor(rng.uniform(-0.3, 0.3, (nx, L)).astype(np.float32), device="cuda")
    from deepconvsep_b200.engine import Separator
    ws = {}
    outs = {}
    for K in (0, 2):
        sep = Separator(params, arch="dsd", frame_size=N, hop=512, window="hanning", overlap=25, feat_size=N // 2 + 1)
        outs[K] = sep.separate_channels(x, wiener=K, wiener_radius=radius if K else 0)
        torch.cuda.synchronize()
        ws[K] = sep.ctx.workspace_bytes()
        if K:
            assert bool(torch.isfinite(outs[K]).all())
            assert not torch.equal(outs[K], outs[0])
    T, ldf, F = sep.stft.num_frames(L), sep.stft.ldf, N // 2 + 1
    plane = T * ldf
    want = ws[0] - rounded(8 * plane) + rounded(8 * nx * plane) + rounded(8 * 4 * nx * plane) + rounded(wiener_bytes(4, nx, T, F, radius))
    record("wiener_channels_workspace_C%d_%ds" % (nx, int(seconds)), plain=ws[0], filtered=ws[2], formula=want)
    assert ws[2] == want, (ws, want)
