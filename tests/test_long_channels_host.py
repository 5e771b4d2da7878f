"""Long C-channel recordings without a GPU (dcs_long_segments, Separator.separate_long_channels / long_segments):

- the planner, over a grid of lengths, cores, N/hop 2 and 8, overlaps 25 and 20, without and with the Wiener reach
  K * W, at 44.1 kHz and every accepted rate: the cores tile the recording once, each model range is
  longclip.plan_segments' bound for its core, and the in and exact ranges are the supports of resample_oracle.direct;
- a float64 stitching check: direct -> channels_oracle (-> wiener_channels_oracle) -> direct, segment by segment and
  stitched, against the whole recording, at 44.1 and 48 kHz;
- the Python method against a stand-in library: marshalling, and every refusal made before any library call."""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest

import channels_oracle as co
import resample_oracle as ro
import wiener_channels_oracle as wco
from deepconvsep_b200 import _lib, engine, longclip
from deepconvsep_b200.engine import Separator
from oracle import dsp, nets, pipeline

CHUNK = _lib.WIENER_CHUNK_FRAMES


def _lib_or_skip():
    from deepconvsep_b200 import build
    build.build()
    return _lib.load()


def _plan(lib, L, K, N, H, tc, ov, reach=0, up=1, down=1, ntaps=1):
    args = (L, K, N, H, tc, ov, reach, up, down, ntaps, ntaps)
    n = lib.dcs_long_segments(*args, None, 0)
    assert n == -(-L // K)
    segs = (_lib.Segment * n)()
    assert lib.dcs_long_segments(*args, segs, n) == n
    return [(s.in_start, s.in_stop, s.model_start, s.model_stop, s.out_start, s.out_stop) for s in segs]


def _support(up, down, m, num_in):
    """[lo, hi] of the inputs output m reads in resample_oracle.direct (its own index arithmetic), clipped to the input"""
    K = 20 * max(up, down) + 1
    half = (K - 1) // 2
    t = m * down + half
    j0, ph = t // up, t % up
    js = [j0 - i for i in range(-(-K // up)) if ph + i * up < K]
    return max(0, min(js)), min(num_in - 1, max(js))


def _longclip_bounds(L, o0, o1, first, last, N, H, tc, ov, reach):
    """longclip.plan_segments' model range for the core [o0, o1) (hop multiples) of a clip of L samples, read off plans
    of clips 2 o0 and 2 o1 long cut in two, where the cut falls on o0 and o1 (the right bound does not depend on the
    segment's start: it is a multiple of the hop, and of lcm(step, CHUNK) with the filter)"""
    s0 = 0
    if not first:
        segs = longclip.plan_segments(2 * o0, 2, N, H, tc, ov, reach)
        assert len(segs) == 2 and segs[1].out_start == o0
        s0 = segs[1].in_start
    s1 = L
    if not last:
        segs = longclip.plan_segments(2 * o1, 2, N, H, tc, ov, reach)
        assert len(segs) == 2 and segs[0].out_stop == o1 and segs[0].in_stop < 2 * o1
        s1 = min(L, segs[0].in_stop)
    return s0, s1


GEOMETRIES = [(1024, 512, 30, 25), (1024, 512, 30, 20), (2048, 256, 30, 25), (2048, 256, 30, 20)]


@pytest.mark.parametrize("N,H,tc,ov", GEOMETRIES)
@pytest.mark.parametrize("reach", [0, 2])
def test_planner_matches_longclip_at_441(N, H, tc, ov, reach):
    lib = _lib_or_skip()
    left, right = longclip.margins(N, H, tc, ov, reach)
    K = -(-2 * (left + right) // H) * H + 7 * H        # hop-aligned cores long enough for plan_segments to cut there
    for L in (1, 777, K - 1, K, K + 1, 2 * K + 1, 3 * K + 13 * H + 5, 5 * K):
        segs = _plan(lib, L, K, N, H, tc, ov, reach)
        assert segs[0][4] == 0 and segs[-1][5] == L
        for a, b in zip(segs, segs[1:]):
            assert a[5] == b[4]
        for i, (i0, i1, m0, m1, o0, o1) in enumerate(segs):
            assert (i0, i1) == (m0, m1)
            assert 0 <= m0 <= o0 < o1 <= m1 <= L and o1 - o0 <= K
            assert m0 % H == 0 and (m0 // H) % ((tc - ov) * CHUNK // np.gcd(tc - ov, CHUNK) if reach else tc - ov) == 0
            assert (m0, m1) == _longclip_bounds(L, o0, o1, i == 0, i == len(segs) - 1, N, H, tc, ov, reach), (L, i)
    # a last core of one sample, and cores of one sample
    segs = _plan(lib, 2 * K + 1, K, N, H, tc, ov, reach)
    assert segs[-1][4:] == (2 * K, 2 * K + 1) and segs[-1][3] == 2 * K + 1
    segs = _plan(lib, 5, 1, N, H, tc, ov, reach)
    assert [s[4:] for s in segs] == [(i, i + 1) for i in range(5)] and all(s[2:4] == (0, 5) for s in segs)


def test_planner_refuses_bad_arguments():
    lib = _lib_or_skip()
    for bad in ((0, 10, 1024, 512, 30, 25), (10, 0, 1024, 512, 30, 25), (10, 10, 1024, 512, 30, 30),
                (10, 10, 1024, 0, 30, 25), (10, 10, 1024, 512, 30, -1)):
        assert lib.dcs_long_segments(*bad, 0, 1, 1, 1, 1, None, 0) == -1
    assert lib.dcs_long_segments(10, 5, 1024, 512, 30, 25, -1, 1, 1, 1, 1, None, 0) == -1
    assert lib.dcs_long_segments(10, 5, 1024, 512, 30, 25, 0, 1, 1, 1, 1, None, 1) == -1   # out NULL with room asked


@pytest.mark.parametrize("rate", ro.TABLE_RATES)
@pytest.mark.parametrize("reach", [0, 2])
def test_planner_ranges_follow_the_resampler_supports(rate, reach):
    lib = _lib_or_skip()
    up, down = ro.ratio(rate, ro.MODEL_RATE)
    N, H, tc, ov = 2048, 256, 30, 25
    K = int(rate * (60 if reach else 9)) + 3
    for L in (1, K - 1, K, K + 1, 3 * K + 1):
        Lm = ro.length(L, up, down)
        segs = _plan(lib, L, K, N, H, tc, ov, reach, up, down, 20 * max(up, down) + 1)
        assert segs[0][4] == 0 and segs[-1][5] == L
        for a, b in zip(segs, segs[1:]):
            assert a[5] == b[4]
        for i, (i0, i1, m0, m1, o0, o1) in enumerate(segs):
            # the exact range at 44.1 kHz: what the way back reads for the core, inside the model range
            e0, e1 = _support(down, up, o0, Lm)[0], _support(down, up, o1 - 1, Lm)[1] + 1
            assert 0 <= m0 <= e0 < e1 <= m1 <= Lm
            assert i < len(segs) - 1 or m1 == Lm
            # the in range: exactly what the way in reads for the model range
            assert (i0, i1) == (_support(up, down, m0, L)[0], _support(up, down, m1 - 1, L)[1] + 1), (rate, L, i)
            # and the model range is longclip's bound for the exact range
            if reach == 0 and i not in (0, len(segs) - 1):
                q = -(-(N // 2) // H)
                s_v = -(-q // (tc - ov)) * (tc - ov)
                g0 = ((e0 - N // 2) // H - s_v - ov) // (tc - ov) * (tc - ov)
                assert m0 == max(g0, 0) * H
                assert m1 == min(Lm, m0 + (-(-(e1 - m0 + N // 2) // H) + q + tc - 1) * H)


# ------------------------------------------------------------------------------------ float64 stitching
def _stems_oracle(audio, params, N, H, ov, patcher, wiener=(0, 0)):
    """float64 [L, C] -> [L, nsrc, C]: channels_oracle, and the C-channel Wiener filter on its spectra when wiener[0]"""
    stems, mags, phs, mms, _, _ = co.separate_channels(audio, params, "dsd", frameSize=N, hopSize=H, overlap=ov, patcher=patcher)
    if not wiener[0]:
        return stems
    sf = 0.3
    X = np.stack([m.astype(np.float64) / sf * np.exp(1j * p) for m, p in zip(mags, phs)])
    T = X.shape[1]
    Y = np.stack([np.stack([mm[j, :T] / sf * np.exp(1j * phs[c]) for c, mm in enumerate(mms)]) for j in range(mms[0].shape[0])])
    Y = wco.wiener(X, Y, wiener[0], wiener[1])
    L = audio.shape[0]
    out = np.zeros_like(stems)
    for j in range(Y.shape[0]):
        for c in range(Y.shape[1]):
            out[:, j, c] = dsp.compute_inverse(np.abs(Y[j, c]), np.angle(Y[j, c]), frameSize=N, hopSize=H, window=np.hanning)[:L]
    return out


def _at_rate(audio, params, rate, N, H, ov, patcher, wiener):
    """the oracle route at `rate`: direct to 44.1 kHz, the stems oracle, direct back to the recording's length"""
    if rate == ro.MODEL_RATE:
        return _stems_oracle(audio, params, N, H, ov, patcher, wiener)
    up, down = ro.ratio(rate, ro.MODEL_RATE)
    planes = ro.direct(audio.T, up, down, ro.taps(up, down))
    st = _stems_oracle(planes.T, params, N, H, ov, patcher, wiener)
    return np.moveaxis(ro.direct(np.moveaxis(st, 0, -1), down, up, ro.taps(down, up), num_out=audio.shape[0]), -1, 0)


@pytest.mark.parametrize("rate,wiener", [(44100, (0, 0)), (48000, (0, 0)), (44100, (1, 1))])
def test_stitched_oracle_equals_the_whole_recording(rate, wiener):
    N, H, ov, patcher = 1024, 512, 25, "util"
    params = nets.make_synthetic_params("dsd", N // 2 + 1, seed=3)
    seconds = 24.0 if wiener[0] else 6.0          # the filter's margins are K W chunks of 128 frames to either side
    a, _ = pipeline.synth_mixture(seconds, 5)
    b, _ = pipeline.synth_mixture(seconds, 9)
    rec = np.stack([a, 0.5 * b - 0.25 * a], axis=1)
    if rate != ro.MODEL_RATE:
        rec = rec[:int(len(rec) * rate / ro.MODEL_RATE)]   # the same material read as a 48 kHz recording
    L = rec.shape[0]
    lib = _lib_or_skip()
    K = L // 3 + 11
    up, down = ro.ratio(rate, ro.MODEL_RATE)
    ntaps = 1 if rate == ro.MODEL_RATE else 20 * max(up, down) + 1
    segs = _plan(lib, L, K, N, H, 30, ov, wiener[0] * wiener[1], up, down, ntaps)
    assert len(segs) == 3 and any(s[2] > 0 for s in segs)     # some segment starts past the recording's start
    whole = _at_rate(rec, params, rate, N, H, ov, patcher, wiener)
    got = np.zeros_like(whole)
    for (i0, i1, m0, m1, o0, o1) in segs:
        if rate == ro.MODEL_RATE:
            piece = _stems_oracle(rec[i0:i1], params, N, H, ov, patcher, wiener)
            got[o0:o1] = piece[o0 - i0:o1 - i0]
            continue
        h_to, h_from = ro.taps(up, down), ro.taps(down, up)
        # the model range of the whole recording's resampling from the staged samples only, placed at their offsets
        staged = np.zeros((L, rec.shape[1]))
        staged[i0:i1] = rec[i0:i1]
        planes = ro.direct(staged.T, up, down, h_to)[:, m0:m1]
        assert np.array_equal(planes, ro.direct(rec.T, up, down, h_to)[:, m0:m1])
        st = _stems_oracle(planes.T, params, N, H, ov, patcher, wiener)
        placed = np.zeros((ro.length(L, up, down),) + st.shape[1:])
        placed[m0:m1] = st
        back = np.moveaxis(ro.direct(np.moveaxis(placed, 0, -1), down, up, h_from, num_out=L), -1, 0)
        got[o0:o1] = back[o0:o1]
    scale = np.abs(whole).max()
    assert np.abs(got - whole).max() <= 1e-13 * scale, np.abs(got - whole).max() / scale


# ------------------------------------------------------------------------------------ the Python method
NSRC = 4
CT = {np.dtype(np.int16): C.c_int16, np.dtype(np.int32): C.c_int32, np.dtype(np.float32): C.c_float}
DTYPES = {0: np.int16, 1: np.int32, 2: np.float32}


def _arr(ptr, n, dtype):
    return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(CT[np.dtype(dtype)])), shape=(n,))


class FakeLib(object):
    """source s = the recording's samples over (s + 1), cast to the output dtype"""

    def __init__(self):
        self.calls = []

    def dcs_separate_long_channels_host(self, ctx, model, plan, to, back, fin, fout, h_in, L, ch, iters, radius, core, scale,
                                        overlap, patcher, h_out, out_stride, stream):
        self.calls.append((ctx, model, plan, to, back, fin, fout, L, ch, iters, radius, core, scale, overlap, patcher,
                           out_stride, stream))
        a = _arr(h_in, L * ch, DTYPES[fin]).reshape(L, ch)
        o = _arr(h_out, NSRC * out_stride * ch, DTYPES[fout]).reshape(NSRC, out_stride, ch)
        for s in range(NSRC):
            o[s, :L] = (a.astype(np.float64) / (s + 1)).astype(DTYPES[fout])
        return 0

    def __getattr__(self, name):
        raise AssertionError("unexpected library call %s" % name)


class FakeResampler(object):
    def __init__(self, ctx, rate_in, rate_out):
        engine.check_resample_rates(rate_in, rate_out)
        self.handle = "h%d-%d" % (int(rate_in), int(rate_out))


@pytest.fixture
def sep(monkeypatch):
    monkeypatch.setattr(engine, "_stream_ptr", lambda stream=None, device=None: None)
    monkeypatch.setattr(engine, "Resampler", FakeResampler)
    lib = FakeLib()
    s = object.__new__(Separator)
    s.lib, s.nsrc, s.scale_factor, s.overlap, s.patcher = lib, NSRC, 0.3, 25, 1
    s.ctx = SimpleNamespace(handle=1, device=0, lib=lib)
    s.model = SimpleNamespace(arch="dsd", handle=2, tc=30)
    s.stft = SimpleNamespace(handle=3)
    s.frame_size, s.hop = 2048, 512
    s._resamplers = {}
    return s


@pytest.mark.parametrize("dtype,out_dtype", [(np.int16, None), (np.int32, np.float32), (np.float32, np.int16)])
def test_separate_long_channels_marshals(sep, dtype, out_dtype):
    rng = np.random.default_rng(0)
    rec = (rng.standard_normal((5000, 6)) * 1000).astype(dtype)
    out = sep.separate_long_channels(rec, out_dtype=out_dtype, wiener=2, wiener_radius=2, sample_rate=48000,
                                     segment_seconds=0.5)
    od = np.dtype(dtype if out_dtype is None else out_dtype)
    assert out.shape == (NSRC, 5000, 6) and out.dtype == od
    for s in range(NSRC):
        assert np.array_equal(out[s], (rec.astype(np.float64) / (s + 1)).astype(od))
    (call,) = sep.lib.calls
    fmt = {np.dtype(np.int16): 0, np.dtype(np.int32): 1, np.dtype(np.float32): 2}
    assert call == (1, 2, 3, "h48000-44100", "h44100-48000", fmt[np.dtype(dtype)], fmt[od], 5000, 6, 2, 2, 24000, 0.3, 25, 1,
                    5000, None)
    # 44.1 kHz: no resamplers; into a caller's array
    o2 = np.zeros((NSRC, 5000, 6), dtype=od)
    assert sep.separate_long_channels(rec, out=o2, out_dtype=out_dtype) is o2
    assert sep.lib.calls[-1][3:5] == (None, None) and sep.lib.calls[-1][11] == 120 * 44100


def test_separate_long_channels_refusals(sep):
    rec = np.zeros((100, 2), dtype=np.int16)
    bad = [
        dict(recording=np.zeros((100,), dtype=np.int16)),                  # not [L, C]
        dict(recording=np.zeros((100, 2), dtype=np.float64)),              # not a sample format
        dict(recording=np.zeros((100, 17), dtype=np.int16)),               # 17 channels
        dict(recording=np.zeros((100, 1), dtype=np.int16), wiener=1),      # the filter on one channel
        dict(recording=rec, wiener=-1),
        dict(recording=rec, wiener_radius=1),                              # a radius without the filter
        dict(recording=rec, sample_rate=7999),
        dict(recording=rec, sample_rate=44100.5),
        dict(recording=rec, segment_seconds=0),
        dict(recording=rec, segment_seconds=-1.0),
        dict(recording=rec, segment_seconds="120"),
        dict(recording=rec, segment_seconds=float("inf")),
        dict(recording=rec, segment_seconds=float("nan")),
        dict(recording=rec, out_dtype=np.float64),
        dict(recording=rec, out_dtype="nonsense"),
        dict(recording=rec, out=np.zeros((NSRC, 99, 2), dtype=np.int16)),
        dict(recording=rec, out=np.zeros((NSRC, 100, 2), dtype=np.int32)),
    ]
    for kw in bad:
        with pytest.raises(ValueError):
            sep.separate_long_channels(**kw)
    assert sep.lib.calls == []
    sep.model.arch = "dsd_ild"
    with pytest.raises(ValueError):
        sep.separate_long_channels(rec)
    assert sep.lib.calls == []


def test_long_segments_is_the_librarys_plan(sep):
    lib = _lib_or_skip()
    sep.lib = lib
    L = 44100 * 300 + 17
    got = sep.long_segments(L, wiener=2, wiener_radius=2)
    assert got == [engine.LongSegment(*s) for s in _plan(lib, L, 120 * 44100, 2048, 512, 30, 25, 4)]
    got = sep.long_segments(L, sample_rate=48000, segment_seconds=60)
    assert got == [engine.LongSegment(*s) for s in _plan(lib, L, 60 * 48000, 2048, 512, 30, 25, 0, 147, 160, 3201)]
    for kw in (dict(segment_seconds=0), dict(segment_seconds=float("inf")), dict(wiener=-1), dict(wiener_radius=2),
               dict(wiener=2, wiener_radius=-1), dict(sample_rate=7999)):
        with pytest.raises(ValueError):
            sep.long_segments(L, **kw)


@pytest.mark.parametrize("reach", [0, 4])
@pytest.mark.parametrize("rate", [44100, 48000])
def test_model_ranges_are_bounded_by_the_core(rate, reach):
    """every model range is its exact range plus longclip.margins and under (align + 1) hops of grid rounding per end,
    whatever the recording's length (include/dcs.h, the workspace bound)"""
    lib = _lib_or_skip()
    N, H, tc, ov = 2048, 512, 30, 25
    step = tc - ov
    align = step * CHUNK // np.gcd(step, CHUNK) if reach else step
    left, right = longclip.margins(N, H, tc, ov, reach)
    up, down = ro.ratio(rate, ro.MODEL_RATE)
    ntaps = 1 if rate == ro.MODEL_RATE else 20 * max(up, down) + 1
    K = 20 * rate + 3
    Lm_core = -(-K * up // down) + 2 * (ntaps // up + 1)                 # a core's exact range at 44.1 kHz, at most
    bound = Lm_core + left + right + 2 * (align + 1) * H
    for L in (3 * K + 1, 7 * K + 12345, 11 * K + 999, 20 * K - 7):
        segs = _plan(lib, L, K, N, H, tc, ov, reach, up, down, ntaps)
        assert max(s[3] - s[2] for s in segs) <= bound, (L, max(s[3] - s[2] for s in segs), bound)
