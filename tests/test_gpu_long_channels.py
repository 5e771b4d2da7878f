"""Long C-channel recordings through the multi-clip scheduler (dcs_separate_long_channels_host,
Separator.separate_long_channels) and the windowed conversions it runs at other rates (dcs_channels_decode_range,
dcs_channels_encode_range).

- range entries, every format, 8 / 22.05 / 32 / 48 / 96 / 192 kHz, C in {1, 2, 6, 16} (the channel-group decode at
  192 kHz, C = 16): windows at both ends, of one sample, across tile edges and at every out_first mod up (48 kHz), each
  against the slice of dcs_channels_decode / _encode on the whole signal (values, -0 equal to +0), the staged range
  the window's exact support;
- the pipeline byte for byte against the contract of include/dcs.h, segment by segment: all nine format pairs at
  48 kHz, a subset at 44.1 kHz and other rates; the DSD network at N = 1024 and 2048, iKala, both patchers, the Wiener
  filter with K = 2 and W = 1, 2 at C = 2 and 6; L <= core, L = core +- 1, a last core of one sample;
- against the whole-recording batch with float32 stems (1e-4 relative L2 per stem and channel), without and with the
  Wiener filter (K = 2, W = 2) at 44.1 and 48 kHz;
- output pitches over the 2-D copy limit (2^31 - 1 bytes) and over 2^32;
- launch count, the workspace formula and its independence of the recording's length; refusals with nothing queued."""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import channels_formats_oracle as fo  # noqa: E402
import resample_oracle as ro  # noqa: E402
from test_gpu_channels_formats import audio_clip, separator, rounded  # noqa: E402

FORMATS = (fo.I16, fo.I32, fo.F32)


def _lib():
    from deepconvsep_b200 import _lib
    return _lib


def _support(up, down, m_first, m_last, num_in):
    ntaps = 20 * max(up, down) + 1
    half = (ntaps - 1) // 2
    lo = -((-(m_first * down + half - ntaps + 1)) // up)
    hi = (m_last * down + half) // up
    return max(0, lo), min(num_in - 1, hi)


def _dev(a):
    t = torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).ravel().copy()).cuda()
    assert t.data_ptr() % 16 == 0
    return t


def decode_whole(ctx, rs, pcm, fmt):
    L, nch = pcm.shape
    n = rs.length(L)
    out = torch.empty((nch + 1) * n, dtype=torch.float32, device="cuda")
    _lib().check(ctx.lib.dcs_channels_decode(ctx.handle, rs.handle, fmt, _dev(pcm).data_ptr(), L, nch, out.data_ptr(), n, None))
    return out.cpu().numpy().reshape(nch + 1, n)


def decode_range(ctx, rs, pcm, fmt, i0, i1, o0, n):
    """outputs [o0, o0 + n) of the whole recording's decode from its samples [i0, i1)"""
    L, nch = pcm.shape
    out = torch.full(((nch + 1) * n + 64,), float("nan"), dtype=torch.float32, device="cuda")
    _lib().check(ctx.lib.dcs_channels_decode_range(ctx.handle, rs.handle, fmt, _dev(pcm[i0:i1]).data_ptr(), L, i0, i1 - i0, nch,
                                                   out.data_ptr(), o0, n, None))
    h = out.cpu().numpy()
    assert np.isnan(h[(nch + 1) * n:]).all()
    return h[:(nch + 1) * n].reshape(nch + 1, n)


def encode_whole(ctx, rs, stems, nsrc, fmt, L):
    P, Lm = stems.shape
    nch = P // nsrc
    out = torch.zeros(nsrc * nch * L * 4, dtype=torch.uint8, device="cuda")
    _lib().check(ctx.lib.dcs_channels_encode(ctx.handle, rs.handle, fmt, _dev(stems).data_ptr(), Lm, nsrc, nch, Lm,
                                             out.data_ptr(), L, nch * L, None))
    return out.cpu().numpy().view(fo.DTYPES[fmt])[:nsrc * nch * L].reshape(nsrc, L, nch)


def encode_range(ctx, rs, stems, nsrc, fmt, Lm, i0, o0, n):
    """outputs [o0, o0 + n) of the encode of a 44.1 kHz signal of Lm samples whose stems at [i0, i0 + width) are given"""
    P, width = stems.shape
    nch = P // nsrc
    b = np.dtype(fo.DTYPES[fmt]).itemsize
    out = torch.full((nsrc * nch * n * b + 64,), 0x5A, dtype=torch.uint8, device="cuda")
    _lib().check(ctx.lib.dcs_channels_encode_range(ctx.handle, rs.handle, fmt, _dev(stems).data_ptr(), Lm, i0, width, nsrc,
                                                   nch, out.data_ptr(), o0, n, nch * n, None))
    h = out.cpu().numpy()
    assert (h[nsrc * nch * n * b:] == 0x5A).all()
    return h[:nsrc * nch * n * b].view(fo.DTYPES[fmt]).reshape(nsrc, n, nch)


def _same_values(a, b):
    """equal values, -0 equal to +0 (NaN payloads compared as bits)"""
    if a.dtype.kind == "f":
        return np.array_equal(a, b) or (np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(a[~np.isnan(a)], b[~np.isnan(b)]))
    return np.array_equal(a, b)


@pytest.fixture(scope="module")
def ctx():
    from deepconvsep_b200.engine import Context
    return Context(0)


@pytest.fixture(scope="module")
def resamplers(ctx):
    from deepconvsep_b200.engine import Resampler
    made = {}

    def get(rate_in, rate_out):
        if (rate_in, rate_out) not in made:
            made[rate_in, rate_out] = Resampler(ctx, rate_in, rate_out)
        return made[rate_in, rate_out]
    return get


def _windows(n, up, tile, every_residue):
    """(first, count) windows of outputs [0, n): both ends, one sample, across the first tiles' edges, and out_first at
    residues mod up"""
    w = {(0, 1), (n - 1, 1), (0, n), (n // 3, n // 3), (tile - 3, 7), (2 * tile - 1, 3)}
    residues = range(up) if every_residue else (1, up // 2, up - 1)
    base = (n // 2) // up * up
    w |= {(base + r, 1 + r % 5) for r in residues}
    return sorted((f, min(c, n - f)) for f, c in w if 0 <= f < n and c >= 1)


@pytest.mark.parametrize("fmt", FORMATS, ids=["i16", "i32", "f32"])
@pytest.mark.parametrize("rate", [8000, 22050, 32000, 48000, 96000, 192000])
def test_decode_range_is_a_slice_of_the_whole(ctx, resamplers, rate, fmt):
    rs = resamplers(rate, ro.MODEL_RATE)
    rng = np.random.default_rng(rate + 7 * fmt)
    for nch in (1, 2, 6, 16):
        pcm = fo.random_clip(rng, int(rate * 0.25) + 11 * nch, nch, fmt)
        L = pcm.shape[0]
        whole = decode_whole(ctx, rs, pcm, fmt)
        n = whole.shape[1]
        tile = fo.pcm_plan(rs.up, rs.down, nch, False, fmt)[0] * rs.up
        for o0, cnt in _windows(n, rs.up, tile, rate == 48000 and nch == 6):
            i0, i1 = _support(rs.up, rs.down, o0, o0 + cnt - 1, L)
            got = decode_range(ctx, rs, pcm, fmt, i0, i1 + 1, o0, cnt)
            assert _same_values(got, whole[:, o0:o0 + cnt]), (rate, fmt, nch, o0, cnt)
        # a staged range wider than the support gives the same values
        got = decode_range(ctx, rs, pcm, fmt, 0, L, n // 4, n // 2)
        assert _same_values(got, whole[:, n // 4:n // 4 + n // 2])


@pytest.mark.parametrize("fmt", FORMATS, ids=["i16", "i32", "f32"])
@pytest.mark.parametrize("rate", [8000, 22050, 32000, 48000, 96000, 192000])
def test_encode_range_is_a_slice_of_the_whole(ctx, resamplers, rate, fmt):
    rs = resamplers(ro.MODEL_RATE, rate)
    rng = np.random.default_rng(3 * rate + fmt)
    for k, nch in enumerate((1, 2, 6, 16)):
        nsrc = 1 + k % 4
        L = int(rate * 0.25) + 5 * nch
        Lm = ro.length(L, rs.down, rs.up)
        stems = (rng.standard_normal((nsrc * nch, Lm)) * 0.5).astype(np.float32)
        whole = encode_whole(ctx, rs, stems, nsrc, fmt, L)
        tile = fo.pcm_plan(rs.up, rs.down, nch, True, fmt)[0] * rs.up
        for o0, cnt in _windows(L, rs.up, tile, rate == 48000 and nch == 6):
            i0, i1 = _support(rs.up, rs.down, o0, o0 + cnt - 1, Lm)
            got = encode_range(ctx, rs, np.ascontiguousarray(stems[:, i0:i1 + 1]), nsrc, fmt, Lm, i0, o0, cnt)
            assert _same_values(got, whole[:, o0:o0 + cnt]), (rate, fmt, nch, o0, cnt)


def test_range_entries_against_the_oracle(ctx, resamplers):
    """one decode window and one encode window against resample_oracle.direct in float64"""
    rate = 48000
    to, back = resamplers(rate, ro.MODEL_RATE), resamplers(ro.MODEL_RATE, rate)
    rng = np.random.default_rng(1)
    pcm = fo.random_clip(rng, 24000, 2, fo.F32)
    o0, n = 9001, 777
    i0, i1 = _support(to.up, to.down, o0, o0 + n - 1, pcm.shape[0])
    got = decode_range(ctx, to, pcm, fo.F32, i0, i1 + 1, o0, n)
    want = ro.direct(pcm.T.astype(np.float64), to.up, to.down, ro.taps(to.up, to.down))[:, o0:o0 + n]
    assert np.abs(got[1:] - want).max() <= 1e-6 * np.abs(want).max()
    stems = (rng.standard_normal((2, 22050)) * 0.5).astype(np.float32)
    o0, n = 5003, 1001
    i0, i1 = _support(back.up, back.down, o0, o0 + n - 1, stems.shape[1])
    got = encode_range(ctx, back, np.ascontiguousarray(stems[:, i0:i1 + 1]), 1, fo.F32, stems.shape[1], i0, o0, n)
    want = ro.direct(stems.astype(np.float64), back.up, back.down, ro.taps(back.up, back.down))[:, o0:o0 + n]
    assert np.abs(got[0].T - want).max() <= 1e-6 * np.abs(want).max()


# ---------------------------------------------------------------------------------------------- pipeline
def contract(sep, rec, fin, fout, rate, wiener, radius, core):
    """the stems the byte contract of include/dcs.h gives, segment by segment -> [nsrc, L, C] of fout"""
    L, nch = rec.shape
    segs = sep.long_segments(L, wiener, radius, rate, segment_seconds=core / rate)
    out = np.zeros((sep.nsrc, L, nch), dtype=fo.DTYPES[fout])
    for sg in segs:
        if rate == ro.MODEL_RATE:
            clip = np.ascontiguousarray(rec[sg.in_start:sg.in_stop])
            got = sep.separate_channels_batch([clip], out_dtype=fo.DTYPES[fout], wiener=wiener, wiener_radius=radius)[0]
            out[:, sg.out_start:sg.out_stop] = got[:, sg.out_start - sg.in_start:sg.out_stop - sg.in_start]
            continue
        to, back = sep.resampler(rate, ro.MODEL_RATE), sep.resampler(ro.MODEL_RATE, rate)
        Sm = sg.model_stop - sg.model_start
        planes = decode_range(sep.ctx, to, rec, fin, sg.in_start, sg.in_stop, sg.model_start, Sm)
        x = torch.from_numpy(np.ascontiguousarray(planes[1:])).cuda()
        stems = sep.separate_channels(x, wiener=wiener, wiener_radius=radius).cpu().numpy().reshape(sep.nsrc * nch, Sm)
        out[:, sg.out_start:sg.out_stop] = encode_range(sep.ctx, back, stems, sep.nsrc, fout, to.length(L), sg.model_start,
                                                        sg.out_start, sg.out_stop - sg.out_start)
    return out, segs


def check(sep, rec, fin, fout, rate, core, wiener=0, radius=0, min_segments=2):
    got = sep.separate_long_channels(rec, out_dtype=fo.DTYPES[fout], wiener=wiener, wiener_radius=radius, sample_rate=rate,
                                     segment_seconds=core / rate)
    want, segs = contract(sep, rec, fin, fout, rate, wiener, radius, core)
    assert len(segs) >= min_segments
    assert got.shape == want.shape and got.dtype == want.dtype
    assert fo.same_bits(got, want), (fin, fout, rate, rec.shape, core, int(np.sum(got != want)))
    assert np.abs(got.astype(np.float64)).sum() > 0
    return got, segs


@pytest.mark.parametrize("N", [1024, 2048])
def test_every_format_pair_at_48k(N):
    sep = separator("dsd", N, seed=60)
    rate, core = 48000, 2 * 48000 + 17
    for fin in FORMATS:
        rec = audio_clip(int(6.3 * rate) + fin, 6, 800 + fin, fin)
        for fout in FORMATS:
            _, segs = check(sep, rec, fin, fout, rate, core, min_segments=4)
            assert any(s.model_start > 0 for s in segs)


@pytest.mark.parametrize("rate", [44100, 22050, 96000, 192000])
def test_rates_channels_and_edge_lengths(rate):
    sep = separator("dsd", 1024, seed=61, patcher="util")
    core = int(1.5 * rate) + 3
    for k, (nch, fmt) in enumerate(((1, fo.I16), (2, fo.I32), (6, fo.F32), (16, fo.I32))):
        # L <= core, L = core +- 1, a last core of one sample, several cores
        for L in ((core - 1, core, core + 1, 2 * core + 1, int(4.2 * core)) if k == 1 else (2 * core + 1, int(3.3 * core))):
            check(sep, audio_clip(L, nch, 810 + k + L % 97, fmt), fmt, fmt if k % 2 else fo.I16, rate, core, min_segments=1)


def test_ikala_and_overlap_20():
    sep = separator("ikala", 1024, seed=62, overlap=20)
    for rate in (44100, 48000):
        check(sep, audio_clip(int(5.5 * rate), 2, 820, fo.I16), fo.I16, fo.I16, rate, int(1.7 * rate))


@pytest.mark.parametrize("nch", [2, 6])
@pytest.mark.parametrize("radius", [1, 2])
def test_wiener(nch, radius):
    sep = separator("dsd", 1024, seed=63)
    for rate, fin, fout in ((44100, fo.I16, fo.I16), (48000, fo.I32, fo.F32)):
        core = 10 * rate + 1
        rec = audio_clip(int(32 * rate), nch, 830 + nch + radius, fin)
        _, segs = check(sep, rec, fin, fout, rate, core, wiener=2, radius=radius, min_segments=4)
        assert any(s.model_start > 0 for s in segs)


def test_one_segment_is_the_whole_batch():
    sep = separator("dsd", 2048, seed=64)
    for rate, fin, fout, wiener in ((44100, fo.I32, fo.I16, 0), (48000, fo.F32, fo.I32, 1), (192000, fo.I32, fo.I32, 0)):
        rec = audio_clip(int(2.1 * rate), 16 if rate == 192000 else 3, 840, fin)
        for core in (rec.shape[0], rec.shape[0] + 1000):
            got = sep.separate_long_channels(rec, out_dtype=fo.DTYPES[fout], wiener=wiener, sample_rate=rate,
                                             segment_seconds=core / rate)
            want = sep.separate_channels_batch([rec], out_dtype=fo.DTYPES[fout], wiener=wiener, sample_rate=rate)[0]
            assert fo.same_bits(got, want), (rate, fin, fout)


@pytest.mark.parametrize("rate,wiener", [(44100, 0), (48000, 0), (44100, 2), (48000, 2)])
def test_close_to_the_whole_recording(rate, wiener):
    """float32 stems against the whole-recording batch: the kept samples differ only by the GEMMs' summation order.
    With the filter (K = 2, W = 2) the margins reach K W = 4 chunks of 128 frames to either side."""
    sep = separator("dsd", 1024, seed=5)
    nch = 6
    seconds, core = (40.0, 10.0) if wiener else (9.5, 2.0)
    radius = 2 if wiener else 0
    rec = audio_clip(int(seconds * rate), nch, 1001, fo.F32)
    whole = sep.separate_channels_batch([rec], wiener=wiener, wiener_radius=radius, sample_rate=rate)[0]
    got = sep.separate_long_channels(rec, wiener=wiener, wiener_radius=radius, sample_rate=rate, segment_seconds=core)
    segs = sep.long_segments(rec.shape[0], wiener, radius, sample_rate=rate, segment_seconds=core)
    assert len(segs) == int(np.ceil(seconds / core)) and any(sg.model_start > 0 for sg in segs)
    for s in range(sep.nsrc):
        for c in range(nch):
            ref = np.linalg.norm(whole[s, :, c])
            assert ref > 0 and np.linalg.norm(got[s, :, c] - whole[s, :, c]) <= 1e-4 * ref, (s, c)


@pytest.mark.parametrize("rate", [44100, 48000])
def test_output_pitch_past_the_copy_limit(rate):
    """a source-to-source output pitch over the devices' 2-D copy limit (cudaDevAttrMaxPitch, 2^31 - 1 bytes), and over
    2^32: the stems of a long multichannel recording.  The output rows are far apart in a sparse mapping that reserves
    no memory; the kept bytes are those of the same call into a compact array, and the bytes around each row untouched"""
    import mmap
    from deepconvsep_b200 import _lib
    sep = separator("dsd", 1024, seed=67)
    nch, core = 16, int(1.2 * rate)
    rec = audio_clip(int(3.3 * rate), nch, 870, fo.F32)
    L = rec.shape[0]
    w = nch * 4
    want = sep.separate_long_channels(rec, sample_rate=rate, segment_seconds=core / rate)
    pre = (None, None) if rate == 44100 else (sep.resampler(rate, 44100).handle, sep.resampler(44100, rate).handle)
    for pitch_min in (1 << 31, 1 << 32):
        stride = pitch_min // w + 1001
        size = (sep.nsrc - 1) * stride * w + L * w + 4096
        # 0x4000: MAP_NORESERVE on Linux (the mmap module does not name it on every version)
        buf = mmap.mmap(-1, size, flags=mmap.MAP_PRIVATE | mmap.MAP_ANONYMOUS | getattr(mmap, "MAP_NORESERVE", 0x4000))
        out = np.frombuffer(buf, dtype=np.uint8)
        _lib.check(sep.lib.dcs_separate_long_channels_host(
            sep.ctx.handle, sep.model.handle, sep.stft.handle, *pre, fo.F32, fo.F32, rec.ctypes.data, L, nch, 0, 0, core,
            C.c_float(sep.scale_factor), sep.overlap, sep.patcher, out.ctypes.data, stride, None))
        for s in range(sep.nsrc):
            row = out[s * stride * w:s * stride * w + L * w]
            assert row.tobytes() == want[s].tobytes(), (pitch_min, s)
            assert not out[s * stride * w + L * w:s * stride * w + L * w + 4096].any(), (pitch_min, s)
        del out, row
        buf.close()


def test_launch_count_and_workspace():
    nch, rate = 6, 44100
    core = 3 * rate + 5
    rec = audio_clip(int(11.2 * rate), nch, 850, fo.I16)
    sep = separator("dsd", 2048, seed=65)
    segs = sep.long_segments(rec.shape[0], 2, 1, rate, segment_seconds=core / rate)
    n0 = sep.ctx.launch_count()
    sep.separate_long_channels(rec, wiener=2, wiener_radius=1, segment_seconds=core / rate)
    n_long = sep.ctx.launch_count() - n0
    per = 0
    for sg in segs:
        n0 = sep.ctx.launch_count()
        sep.separate_channels_batch([np.ascontiguousarray(rec[sg.in_start:sg.in_stop])], wiener=2, wiener_radius=1)
        per += sep.ctx.launch_count() - n0
    assert n_long == per, (n_long, per)
    # the workspace formula; and two lengths with the same core whose longest segments fall alike on the frame grid take
    # the same workspace (in general the workspace is bounded by the core, not constant)
    for fin, fout, r in ((fo.I16, fo.I16, 44100), (fo.I32, fo.F32, 48000)):
        c = 3 * r + 5
        wss = []
        for seconds in (41.2, 63.9):          # long enough for a segment whose margins reach neither end
            x = audio_clip(int(seconds * r), nch, 851, fin)
            fresh = separator("dsd", 2048, seed=65)
            fresh.separate_long_channels(x, out_dtype=fo.DTYPES[fout], wiener=2, wiener_radius=1, sample_rate=r,
                                         segment_seconds=c / r)
            ss = fresh.long_segments(x.shape[0], 2, 1, r, segment_seconds=c / r)
            Sw = max(s.model_stop - s.model_start for s in ss)
            Smax = max(s.in_stop - s.in_start for s in ss)
            Kmax = max(s.out_stop - s.out_start for s in ss)
            single = separator("dsd", 2048, seed=65)
            single.separate_channels(torch.zeros((nch, Sw), dtype=torch.float32, device="cuda"), wiener=2, wiener_radius=1)
            bi, bo = (np.dtype(fo.DTYPES[f]).itemsize for f in (fin, fout))
            want = (single.ctx.workspace_bytes() - rounded(4 * Sw) + rounded(4 * (nch + 1) * Sw) + rounded(4 * 4 * nch * Sw)
                    + 2 * rounded(bi * nch * Smax) + 2 * rounded(bo * 4 * nch * Kmax))
            assert fresh.ctx.workspace_bytes() == want, (r, seconds, fresh.ctx.workspace_bytes(), want)
            wss.append(fresh.ctx.workspace_bytes())
        assert wss[0] == wss[1], wss


def test_refusals_queue_nothing():
    from deepconvsep_b200 import _lib
    sep = separator("dsd", 1024, seed=66)
    ctx, lib = sep.ctx, sep.lib
    rate, nch = 48000, 3
    rec = audio_clip(5 * rate, nch, 860, fo.I32)
    L = rec.shape[0]
    to, back, to96 = sep.resampler(rate, 44100), sep.resampler(44100, rate), sep.resampler(96000, 44100)
    out = np.full((4, L, nch), 0x5A5A5A5A, dtype=np.int32)
    sep.separate_long_channels(np.zeros((rate, nch), np.int32), sample_rate=rate, segment_seconds=0.5)
    ws = ctx.workspace_bytes()

    def call(pair=(to, back), fin=1, fout=1, channels=nch, iterations=0, radius=0, core=rate, out_stride=L, h_in=True,
             h_out=True, n=L, overlap=25, patcher=0):
        h = [None if r is None else r.handle for r in pair]
        return lib.dcs_separate_long_channels_host(
            ctx.handle, sep.model.handle, sep.stft.handle, h[0], h[1], fin, fout, rec.ctypes.data if h_in else None, n,
            channels, iterations, radius, core, C.c_float(0.3), overlap, patcher, out.ctypes.data if h_out else None,
            out_stride, None)

    refused = {
        "in format 3": (lambda: call(fin=3), "unknown sample format"),
        "out format -1": (lambda: call(fout=-1), "unknown sample format"),
        "NULL to_model": (lambda: call(pair=(None, back)), "NULL resampler"),
        "not inverse": (lambda: call(pair=(to96, back)), "not inverse"),
        "channels 17": (lambda: call(channels=17), "channels 17"),
        "filter on 9 channels": (lambda: call(channels=9, iterations=1), "Wiener"),
        "iterations -1": (lambda: call(iterations=-1), "iterations"),
        "core 0": (lambda: call(core=0), "core_samples"),
        "out_stride < L": (lambda: call(out_stride=L - 1), "out_stride"),
        "num_samples 0": (lambda: call(n=0), "num_samples"),
        "NULL in": (lambda: call(h_in=False), "NULL"),
        "NULL out": (lambda: call(h_out=False), "NULL"),
        "radius 0 over segments": (lambda: call(iterations=1, radius=0), "radius"),
        "overlap 30": (lambda: call(overlap=30), "overlap"),
        "patcher 5": (lambda: call(patcher=5), "patcher"),
    }
    for name, (fn, msg) in refused.items():
        torch.cuda.synchronize()
        n0 = ctx.launch_count()
        with pytest.raises(_lib.DcsError) as e:
            _lib.check(fn())
        assert ctx.launch_count() == n0 and ctx.workspace_bytes() == ws, name
        assert msg in str(e.value), (name, str(e.value))
        assert (out == 0x5A5A5A5A).all(), name
    # one segment with radius 0 is the whole recording: accepted
    _lib.check(call(iterations=1, radius=0, core=L))
    out[...] = 0x5A5A5A5A
    # taps set on the ctx
    tap = torch.zeros(1 << 20, dtype=torch.complex64, device="cuda")
    for setter in ("dcs_set_spectrum_tap", "dcs_set_pool_tap"):
        _lib.check(getattr(lib, setter)(ctx.handle, tap.data_ptr(), tap.numel()))
        n0 = ctx.launch_count()
        with pytest.raises(_lib.DcsError) as e:
            _lib.check(call())
        assert "tap" in str(e.value) and ctx.launch_count() == n0 and (out == 0x5A5A5A5A).all()
        _lib.check(getattr(lib, setter)(ctx.handle, None, 0))
    # the range entries
    d = torch.zeros(4 * nch * 4 * L + 64, dtype=torch.float32, device="cuda")
    p = d.data_ptr()
    n = to.length(L)
    lo, hi = _support(to.up, to.down, 1000, 1999, L)
    blo, bhi = _support(back.up, back.down, 1000, 1999, n)
    bad = [lambda: lib.dcs_channels_decode_range(ctx.handle, None, 1, p, L, lo, hi + 1 - lo, nch, p, 1000, 1000, None),
           lambda: lib.dcs_channels_decode_range(ctx.handle, to.handle, 3, p, L, lo, hi + 1 - lo, nch, p, 1000, 1000, None),
           lambda: lib.dcs_channels_decode_range(ctx.handle, to.handle, 1, p, L, lo + 1, hi - lo, nch, p, 1000, 1000, None),
           lambda: lib.dcs_channels_decode_range(ctx.handle, to.handle, 1, p, L, lo, hi - lo, nch, p, 1000, 1000, None),
           lambda: lib.dcs_channels_decode_range(ctx.handle, to.handle, 1, p, L, lo, hi + 1 - lo, nch, p, n - 5, 6, None),
           lambda: lib.dcs_channels_decode_range(ctx.handle, to.handle, 1, p, L, L - 5, 6, nch, p, n - 5, 5, None),
           lambda: lib.dcs_channels_decode_range(ctx.handle, to.handle, 1, p, L, lo, hi + 1 - lo, 17, p, 1000, 1000, None),
           lambda: lib.dcs_channels_encode_range(ctx.handle, back.handle, 1, p, n, blo + 1, bhi - blo, 4, nch, p, 1000, 1000,
                                                 nch * 1000, None),
           lambda: lib.dcs_channels_encode_range(ctx.handle, back.handle, 1, p, n, blo, bhi - blo, 4, nch, p, 1000, 1000,
                                                 nch * 1000, None),
           lambda: lib.dcs_channels_encode_range(ctx.handle, back.handle, 1, p, n, blo, bhi + 1 - blo, 4, nch, p, 1000, 1000,
                                                 nch * 1000 + 1, None),
           lambda: lib.dcs_channels_encode_range(ctx.handle, back.handle, 1, p, n, blo, bhi + 1 - blo, 4, nch, p + 2, 1000, 1000,
                                                 nch * 1000, None)]
    torch.cuda.synchronize()
    n0 = ctx.launch_count()
    for k, fn in enumerate(bad):
        assert fn() == -1, k
    assert ctx.launch_count() == n0 and not d.any()
    got = sep.separate_long_channels(rec, sample_rate=rate, segment_seconds=1.0)
    want, _ = contract(sep, rec, fo.I32, fo.I32, rate, 0, 0, rate)
    assert fo.same_bits(got, want)
