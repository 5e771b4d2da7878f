"""Polyphase resampling on the device (dcs_resample; engine.Resampler, Separator(..., sample_rate=)):

- the kernel element by element against the float64 direct formula of tests/resample_oracle.py (run on the fp32 input
  widened), for every rate of the policy's table in both directions, 1 and 6 planes with gaps, NaN wherever the kernel
  must not read, NaN-payload sentinels around every output plane, under the bound
  |y_dev - y| <= 2^-24 |y| + 2 ceil(K/up) 2^-53 sum|h x|, and the same bits on two runs;
- every argument class the C ABI refuses, with nothing queued and the ctx still working;
- composition: each stems call with sample_rate=fs is, bit for bit, Resampler in -> the 44.1 kHz call -> Resampler back;
  at 44100 it is the call without the keyword, with the same launch count;
- end to end against float64: resample_poly -> the oracle pipeline -> resample_poly back, mono and C = 6."""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import resample_oracle as ro  # noqa: E402
from parity import record, rel, istft_rows  # noqa: E402

NAN_IN = np.uint32(0x7fc0beef)      # NaN payloads: what the kernel must not read, and must not write
NAN_OUT = np.uint32(0x7fc0dead)


@pytest.fixture(scope="module")
def ctx():
    from deepconvsep_b200.engine import Context
    return Context(0)


def _resampler(ctx, rate_in, rate_out):
    from deepconvsep_b200.engine import Resampler
    return Resampler(ctx, rate_in, rate_out)


def _run(rs, x, num_out, gap_in=37, gap_out=29, pad=64):
    """x float32 [P, L] through rs into sentinel-fenced planes -> (y [P, num_out], the fences intact)"""
    P, L = x.shape
    si, so = L + gap_in, num_out + gap_out
    ibuf = torch.from_numpy(np.full(P * si, NAN_IN, dtype=np.uint32).view(np.float32)).cuda()
    iv = ibuf.view(P, si)[:, :L]
    iv.copy_(torch.from_numpy(x))
    obuf = torch.from_numpy(np.full(2 * pad + P * so, NAN_OUT, dtype=np.uint32).view(np.float32)).cuda()
    ov = obuf[pad:pad + P * so].view(P, so)[:, :num_out]
    rs.resample(iv, num_out=num_out, out=ov)
    torch.cuda.synchronize()
    raw = obuf.cpu().numpy().view(np.uint32)
    planes = raw[pad:pad + P * so].reshape(P, so)
    fences = np.concatenate([raw[:pad], raw[pad + P * so:], planes[:, num_out:].ravel()])
    return planes[:, :num_out].view(np.float32).copy(), bool(np.all(fences == NAN_OUT))


@pytest.mark.parametrize("direction", ["in", "back"])
@pytest.mark.parametrize("rate", ro.TABLE_RATES)
def test_kernel_against_float64(ctx, rate, direction):
    rate_in, rate_out = (rate, ro.MODEL_RATE) if direction == "in" else (ro.MODEL_RATE, rate)
    rs = _resampler(ctx, rate_in, rate_out)
    up, down = rs.up, rs.down
    h = ro.taps(up, down)
    Q = -(-h.size // up)
    rng = np.random.default_rng(rate * 2 + (direction == "back"))
    worst = 0.0
    for P in (1, 6):
        for L in (1, 7, max(8, h.size // 3), 10 * rate_in):
            x = rng.uniform(-1.0, 1.0, (P, L)).astype(np.float32)
            n = ro.length(L, up, down)
            got, fenced = _run(rs, x, n)
            assert fenced, (rate, direction, P, L)
            y = ro.direct(x.astype(np.float64), up, down, h)
            bound = 2.0 ** -24 * np.abs(y) + 2 * Q * 2.0 ** -53 * ro.direct(np.abs(x.astype(np.float64)), up, down, np.abs(h))
            err = np.abs(got.astype(np.float64) - y)
            assert np.all(np.isfinite(got)) and np.all(err <= bound), (rate, direction, P, L, float(np.max(err - bound)))
            worst = max(worst, float(np.max(err / np.maximum(bound, 1e-300))))
            again, _ = _run(rs, x, n, gap_in=3, gap_out=5)
            assert again.tobytes() == got.tobytes()
            # a shorter num_out is the head of the whole output
            if n > 3:
                head, fenced = _run(rs, x, n - 3)
                assert fenced and head.tobytes() == got[:, :n - 3].tobytes()
    record("resample_%d_%s" % (rate, direction), kind="resample", up=up, down=down, taps_per_phase=Q,
           worst_error_over_bound=worst)


def test_refusals_queue_nothing(ctx):
    from deepconvsep_b200 import _lib
    lib = ctx.lib
    h = ro.taps(160, 147)
    hp = h.ctypes.data
    out = C.c_void_p()
    n0 = ctx.launch_count()
    bad_create = [(None, 160, 147, hp, h.size), (ctx.handle, 0, 147, hp, h.size), (ctx.handle, 160, 0, hp, h.size),
                  (ctx.handle, 320, 294, hp, h.size), (ctx.handle, 160, 147, hp, h.size - 1),
                  (ctx.handle, 160, 147, hp, 0), (ctx.handle, 160, 147, None, h.size)]
    for args in bad_create:
        assert lib.dcs_resampler_create(*args, C.byref(out)) == -1, args
    assert lib.dcs_resampler_create(ctx.handle, 160, 147, hp, h.size, None) == -1
    big = ro.taps(44100, 44099)                                   # a 7 MB bank
    assert lib.dcs_resampler_create(ctx.handle, 44100, 44099, big.ctypes.data, big.size, C.byref(out)) == -1
    assert b"bank" in lib.dcs_last_error()
    rs = _resampler(ctx, 44100, 48000)
    L, n = 1000, ro.length(1000, 160, 147)
    x = torch.zeros((2, L + 8), device="cuda")
    y = torch.zeros((2, n + 8), device="cuda")
    xp, yp = x.data_ptr(), y.data_ptr()
    bad = [(None, xp, 1, L, L, yp, n, n), (rs.handle, None, 1, L, L, yp, n, n), (rs.handle, xp, 1, L, L, None, n, n),
           (rs.handle, xp, 0, L, L, yp, n, n), (rs.handle, xp, 1, L, 0, yp, n, n), (rs.handle, xp, 1, L, L, yp, n, 0),
           (rs.handle, xp, 1, L, L, yp, n, n + 1), (rs.handle, xp, 2, L - 1, L, yp, n, n),
           (rs.handle, xp, 2, L, L, yp, n - 1, n), (rs.handle, xp, 1, -1, L, yp, n, n),
           (rs.handle, xp + 2, 1, L, L, yp, n, n), (rs.handle, xp, 1, L, L, yp + 1, n, n)]
    for args in bad:
        assert lib.dcs_resample(*args, None) == -1, args
    torch.cuda.synchronize()
    assert ctx.launch_count() == n0 and not y.any()
    # the ctx and the resampler still work
    src = torch.rand((2, L), device="cuda")
    got = rs.resample(src)
    want = ro.direct(src.cpu().numpy().astype(np.float64), 160, 147, rs.taps)
    assert ctx.launch_count() == n0 + 1 and np.max(np.abs(got.cpu().numpy() - want)) < 1e-5
    with pytest.raises(_lib.DcsError):
        rs.resample(src, num_out=n + 1)
    with pytest.raises(ValueError, match="44099"):
        _resampler(ctx, 44099, 44100)


# ---------------------------------------------------------------------------------------------- composition
def _separator(arch, seed=5):
    from deepconvsep_b200.engine import Separator
    from oracle import nets
    params = nets.make_synthetic_params(arch, 513, seed=seed)
    return params, Separator(params, arch=arch, frame_size=1024, hop=512, window="hanning", overlap=25, feat_size=513)


def _channels(seconds, rate, nch, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(int(seconds * rate)) / rate
    cols = [0.3 * np.sin(2 * np.pi * (110 * (c + 1) + 40 * t) * t) + 0.1 * rng.standard_normal(t.size) for c in range(nch)]
    return np.stack(cols, axis=1).astype(np.float32)


def _same(a, b):
    a = a.cpu().numpy() if hasattr(a, "cpu") else a
    b = b.cpu().numpy() if hasattr(b, "cpu") else b
    return a.shape == b.shape and np.ascontiguousarray(a).tobytes() == np.ascontiguousarray(b).tobytes()


@pytest.fixture(scope="module")
def seps():
    return {"dsd": _separator("dsd")[1], "dsd_ild": _separator("dsd_ild")[1]}


CALLS = [("separate", "dsd", 1, {}), ("separate_keep_channels", "dsd", 2, {}),
         ("separate_keep_channels", "dsd", 2, {"wiener": 2, "wiener_radius": 1}), ("separate_stereo", "dsd_ild", 2, {}),
         ("separate_channels", "dsd", 6, {}), ("separate_channels", "dsd", 6, {"wiener": 2})]


@pytest.mark.parametrize("rate", [48000, 96000])
@pytest.mark.parametrize("name,arch,nch,kw", CALLS)
def test_sample_rate_is_the_composition_of_public_pieces(seps, name, arch, nch, kw, rate):
    from deepconvsep_b200.engine import Resampler
    sep = seps[arch]
    method = getattr(sep, name)
    audio = _channels(1.5, rate, nch, seed=rate + nch)
    a = audio[:, 0] if nch == 1 else audio
    L = audio.shape[0]
    x = torch.tensor(np.ascontiguousarray(audio.T), device="cuda")        # [C, L]
    down, back = Resampler(sep.ctx, rate, 44100), Resampler(sep.ctx, 44100, rate)
    x44 = down.resample(x)
    s44 = sep.separate_device(x44[0]) if nch == 1 else method(x44, **kw)
    want = back.resample(s44, num_out=L)                                   # [nsrc * C, L]
    assert float(want.abs().max()) > 0
    got_dev = method(x[0] if nch == 1 else x, sample_rate=rate, **kw)
    assert _same(got_dev, want)
    got = method(a, sample_rate=rate, **kw)                               # numpy in -> the numpy layout
    w = want.cpu().numpy()
    assert _same(got, w if nch == 1 else np.ascontiguousarray(w.reshape(sep.nsrc, nch, L).transpose(2, 0, 1)))
    # at 44100 the keyword changes nothing: the same call, bits and launch count
    a44 = (_channels(1.5, 44100, nch, seed=7)[:, 0] if nch == 1 else _channels(1.5, 44100, nch, seed=7))
    n0 = sep.ctx.launch_count()
    plain = method(a44, **kw)
    n1 = sep.ctx.launch_count()
    keyed = method(a44, sample_rate=44100, **kw)
    assert _same(plain, keyed) and sep.ctx.launch_count() - n1 == n1 - n0
    # one launch each way on top of the 44.1 kHz call
    n0 = sep.ctx.launch_count()
    method(x44[0] if nch == 1 else x44, **kw) if nch > 1 else sep.separate_device(x44[0])
    n1 = sep.ctx.launch_count()
    method(x[0] if nch == 1 else x, sample_rate=rate, **kw)
    assert sep.ctx.launch_count() - n1 == (n1 - n0) + 2


def test_score_and_masks_calls_refuse_other_rates(seps):
    sep = seps["dsd"]
    a = np.zeros(44100, dtype=np.float32)
    with pytest.raises(ValueError, match="Resampler"):
        sep.separate_masks(a, sample_rate=48000)
    with pytest.raises(ValueError, match="Resampler"):
        sep.apply_masks(a[:, None], np.zeros((4, 89, 513), dtype=np.float32), sample_rate=48000)
    with pytest.raises(ValueError, match="44099"):
        sep.separate(a, sample_rate=44099)


# ---------------------------------------------------------------------------------------------- against float64
def test_mono_48k_matches_float64():
    from scipy.signal import resample_poly
    from oracle import pipeline
    from deepconvsep_b200.engine import Resampler
    params, sep = _separator("dsd", seed=2)
    mix, _ = pipeline.synth_mixture(10.0 * 48000 / 44100, 1001)       # 10 s of samples, read as 48 kHz
    a = mix.astype(np.float32)
    L = a.size
    got = sep.separate(a, sample_rate=48000)
    x44 = resample_poly(a.astype(np.float64), 147, 160)
    stems44, mag, ph, mm = pipeline.separate(x44, params, "dsd", frameSize=1024, overlap=25, return_spec=True,
                                             count_kinks=True)
    kmap = pipeline.separate.last_kink_map
    # the device's spectra at the 44.1 kHz stage of the composed call, for the flagged bins
    x44_dev = Resampler(sep.ctx, 48000, 44100).resample(torch.tensor(a[None], device="cuda"))[0].cpu().numpy()
    _, S_dev = sep.separate_tapped(x44_dev)
    T, F = ph.shape
    nflag = int(kmap.sum())
    assert nflag <= 1e-4 * kmap.size + 8
    want44 = stems44.copy()
    if nflag:
        tt, ff = np.nonzero(kmap)
        rows = sorted(set(int(t) for t in tt))
        S_or = (mm[:, :T] / 0.3) * np.sqrt(1024) * np.exp(1j * ph)[None]
        for s in range(sep.nsrc):
            D = np.zeros((T, F), dtype=np.complex128)
            D[tt, ff] = S_dev[s][tt, ff] - S_or[s][tt, ff]
            want44[s] = want44[s] + istft_rows(D, rows, np.hanning(1024), 512, 1024, stems44.shape[1])
    want = resample_poly(want44, 160, 147, axis=1)[:, :L]
    errs = [rel(got[s], want[s]) for s in range(sep.nsrc)]
    record("resample_dsd_mono_48k_10s", kind="resample_e2e", flagged_bins=nflag, rel_l2=errs, tol=1e-4)
    assert max(errs) <= 1e-4, (errs, nflag)


def test_six_channels_48k_match_float64():
    from scipy.signal import resample_poly
    import channels_oracle as co
    from deepconvsep_b200.engine import Resampler
    params, sep = _separator("dsd", seed=6)
    nch = 6
    audio = _channels(10.0, 48000, nch, seed=61)
    L = audio.shape[0]
    got = sep.separate_channels(audio, sample_rate=48000)                 # [L, nsrc, C]
    x44 = resample_poly(audio.astype(np.float64), 147, 160, axis=0)
    stems, mags, phs, mms, masks, kmap = co.separate_channels(x44, params, frameSize=1024, hopSize=512)
    T, F = kmap.shape
    L44 = x44.shape[0]
    # the device's masks of its own downmix at the 44.1 kHz stage, for the flagged bins
    x = Resampler(sep.ctx, 48000, 44100).resample(torch.tensor(np.ascontiguousarray(audio.T), device="cuda"))
    mono = x[0]
    for c in range(1, nch):
        mono = mono + x[c]
    Mdev = sep.separate_masks((mono * float(np.float32(1.0) / np.float32(nch))).contiguous())[:, :, :F].cpu().numpy()
    nflag = int(kmap.sum())
    assert nflag <= 1e-4 * kmap.size + 8
    tt, ff = np.nonzero(kmap)
    rows = sorted(set(int(t) for t in tt))
    errs = []
    for c in range(nch):
        Xc = (mags[c].astype(np.float64) / 0.3) * np.sqrt(1024) * np.exp(1j * phs[c])
        for s in range(sep.nsrc):
            w44 = stems[:, s, c]
            if nflag:
                S_or = (mms[c][s, :T] / 0.3) * np.sqrt(1024) * np.exp(1j * phs[c])
                D = np.zeros((T, F), dtype=np.complex128)
                D[tt, ff] = Mdev[s, tt, ff].astype(np.float64) * Xc[tt, ff] - S_or[tt, ff]
                w44 = w44 + istft_rows(D, rows, np.hanning(1024), 512, 1024, L44)
            want = resample_poly(w44, 160, 147)[:L]
            errs.append(rel(got[:, s, c], want))
    record("resample_dsd_C6_48k_10s", kind="resample_e2e", flagged_bins=nflag, rel_l2=errs, tol=1e-4)
    assert max(errs) <= 1e-4, (max(errs), nflag)
