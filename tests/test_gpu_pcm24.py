"""Packed 24-bit PCM (DCS_SAMPLE_I24, engine.PCM24) on the device: its conversion kernels element by element, and the
multi-clip scheduler and the long-recording path byte for byte, against tests/pcm24_oracle.py and against the int32
route carrying the same 24-bit values (v << 8 in, the int32 stems >> 8 out).

- plain kernels (pcm24_decode_channels_kernel, pcm24_encode_channels_kernel): C 1..16, lengths 1, 255, 256, 257 and
  4099, every source and destination offset modulo 16 bytes, NaN payloads between the stem planes, sentinel bytes
  around every output, every case twice;
- fused and windowed kernels (resample_decode_kernel / resample_encode_kernel<DCS_SAMPLE_I24>): the decode's planes are
  the I32 instantiation's on v << 8 and the encode's bytes the I32 encode's shifted right by 8, at every rate class,
  at odd addresses, and at 192 kHz with C = 16 (channel groups and one more downmix launch);
- batch: the 7 format pairs with I24 against encode_out(separate_channels(decode_in(clip))) at 44.1 and 48 kHz, the
  ties to int32, the Wiener filter, launch counts, the workspace formula with b = 3;
- long recordings: the per-segment byte contract of include/dcs.h, one segment as the batch, a wav_samples memmap.
- code 3 stays refused."""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import channels_formats_oracle as fo  # noqa: E402
import pcm24_oracle as p24  # noqa: E402
import resample_oracle as ro  # noqa: E402
from oracle import nets, pipeline  # noqa: E402

I24 = p24.I24
NAN_IN = np.uint32(0x7fc0beef)
NAN_OUT = np.uint32(0x7fc0dead)
SENT = 0x5A
PADB = 256                      # sentinel bytes before and after every buffer
MB = 1 << 20


def _lib():
    from deepconvsep_b200 import _lib
    return _lib


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


def _twice(fn):
    a, fa = fn()
    b, fb = fn()
    assert fa and fb, "a fence changed"
    assert a.tobytes() == b.tobytes(), "two runs differ"
    return a


def _bytes_at(raw, off):
    """device bytes: PADB sentinels, `off` more, raw, PADB sentinels; (tensor, pointer of raw[0])"""
    buf = np.full(2 * PADB + off + len(raw), SENT, dtype=np.uint8)
    buf[PADB + off:PADB + off + len(raw)] = np.frombuffer(raw, np.uint8)
    d = torch.from_numpy(buf).cuda()
    assert d.data_ptr() % 16 == 0
    return d, d.data_ptr() + PADB + off


def _planes_out(n):
    return torch.from_numpy(np.full(2 * 64 + n, NAN_OUT, dtype=np.uint32).view(np.int32)).cuda()


def decode(ctx, pcm, fmt, off=0, rs=None, num_out=None):
    """[L, C] of fmt at `off` bytes past a 16-byte boundary -> (uint32 bits [C + 1, num_out], fences intact)"""
    L, nch = pcm.shape
    n = L if num_out is None else num_out
    keep, pin = _bytes_at(np.ascontiguousarray(pcm).tobytes(), off)
    out = _planes_out((nch + 1) * n)
    _lib().check(ctx.lib.dcs_channels_decode(ctx.handle, rs.handle if rs else None, fmt, pin, L, nch,
                                             out.data_ptr() + 4 * 64, n, None))
    raw = out.cpu().numpy().view(np.uint32)
    fenced = bool(np.all(raw[:64] == NAN_OUT) and np.all(raw[64 + (nch + 1) * n:] == NAN_OUT))
    return raw[64:64 + (nch + 1) * n].reshape(nch + 1, n).copy(), fenced


def encode(ctx, stems, nsrc, fmt, off, rs=None, num_out=None, gap=0):
    """stem planes float32 [nsrc * C, num_in], NaN payloads in the gaps -> (bytes [nsrc, num_out * C * b], fences
    intact); the output starts `off` bytes past a 16-byte boundary"""
    P, Lin = stems.shape
    nch = P // nsrc
    n = Lin if num_out is None else num_out
    stride = Lin + gap
    sbuf = np.full(64 + P * stride + 64, NAN_IN, dtype=np.uint32)
    sbuf[64:64 + P * stride].reshape(P, stride)[:, :Lin] = np.ascontiguousarray(stems, dtype=np.float32).view(np.uint32)
    ds = torch.from_numpy(sbuf.view(np.int32)).cuda()
    b = 3 if fmt == I24 else np.dtype(fo.DTYPES[fmt]).itemsize
    total = nsrc * nch * n * b
    dout, pout = _bytes_at(b"\x5a" * total, off)
    _lib().check(ctx.lib.dcs_channels_encode(ctx.handle, rs.handle if rs else None, fmt, ds.data_ptr() + 4 * 64, Lin, nsrc,
                                             nch, stride, pout, n, nch * n, None))
    raw = dout.cpu().numpy()
    k0 = PADB + off
    fenced = bool(np.all(raw[:k0] == SENT) and np.all(raw[k0 + total:] == SENT))
    return raw[k0:k0 + total].reshape(nsrc, -1).copy(), fenced


def _v3_bytes(a):
    return np.ascontiguousarray(a).view(np.uint8).reshape(a.shape[0], -1)


def _i32_top3(a):
    """int32 samples [...] -> the bytes of their top 24 bits, packed"""
    return np.ascontiguousarray(a, dtype=np.int32).view(np.uint8).reshape(-1, 4)[:, 1:].reshape(-1)


# ---------------------------------------------------------------------------------------------- 1. plain kernels
LENGTHS = (1, 255, 256, 257, 4099)


def test_plain_decode_every_offset(ctx):
    rng = np.random.default_rng(1)
    for nch in range(1, 17):
        v = p24.values24()
        clips = [p24.random_clip(rng, L, nch) for L in LENGTHS]
        clips.append(p24.pack(np.resize(rng.permutation(v), (-(-v.size // nch), nch))))
        for k, pcm in enumerate(clips):
            want = np.ascontiguousarray(p24.decode_channels(pcm)).view(np.uint32)
            for off in (range(16) if pcm.shape[0] in (255, 257, 4099) else ((k + nch) % 16, 15 - (k + nch) % 16)):
                got = _twice(lambda: decode(ctx, pcm, I24, off))
                assert got.tobytes() == want.tobytes(), (nch, pcm.shape, off, np.argwhere(got != want)[:4].tolist())


def test_plain_encode_every_offset(ctx):
    rng = np.random.default_rng(2)
    vals = p24.stem_values()
    k = 0
    for nch in range(1, 17):
        for off in range(16):
            for L in (1, 7, 255, 256, 257, 513):
                nsrc = 1 + k % 4
                k += 1
                stems = rng.choice(vals, (nsrc * nch, L)).astype(np.float32)
                got = _twice(lambda: encode(ctx, stems, nsrc, I24, off, gap=1 + k % 9))
                want = _v3_bytes(p24.interleave(stems, nsrc).reshape(nsrc, -1))
                assert np.array_equal(got, want), (nch, nsrc, L, off, np.argwhere(got != want)[:4].tolist())
        stems = np.resize(rng.permutation(vals), (2 * nch, -(-vals.size // (2 * nch)))).astype(np.float32)
        got = _twice(lambda: encode(ctx, stems, 2, I24, nch % 16, gap=5))
        i32 = _twice(lambda: encode(ctx, stems, 2, fo.I32, 0, gap=5))
        assert np.array_equal(got.reshape(-1), _i32_top3(i32.view(np.int32)))      # the int32 encode >> 8, on the device


# ---------------------------------------------------------------------------------------------- 2. fused kernels
def _channel_set(rate):
    return range(1, 17) if rate in (48000, 192000) else (1, 2, 5, 16)


@pytest.mark.parametrize("rate", ro.TABLE_RATES)
def test_fused_decode_is_int32s(ctx, resamplers, rate):
    rs = resamplers(rate, ro.MODEL_RATE)
    rng = np.random.default_rng(rate)
    for nch in _channel_set(rate):
        groups = fo.pcm_plan(rs.up, rs.down, nch, False, I24)[2]
        for k, (Lin, Lout) in enumerate(fo.fused_lengths(rs.up, rs.down, nch, False, fo.I32)):
            pcm = p24.random_clip(rng, Lin, nch)
            n0 = ctx.launch_count()
            got = _twice(lambda: decode(ctx, pcm, I24, (k + nch) % 16, rs, Lout))
            assert ctx.launch_count() - n0 == 2 * (1 + (groups > 1)), (rate, nch, groups)
            want, fenced = decode(ctx, p24.to_i32(pcm), fo.I32, 0, rs, Lout)
            assert fenced and got.tobytes() == want.tobytes(), (rate, nch, Lin, Lout, np.argwhere(got != want)[:4].tolist())


@pytest.mark.parametrize("rate", ro.TABLE_RATES)
def test_fused_encode_is_int32s_shifted(ctx, resamplers, rate):
    rs = resamplers(ro.MODEL_RATE, rate)
    rng = np.random.default_rng(3 * rate)
    for nch in _channel_set(rate):
        for k, (Lin, Lout) in enumerate(fo.fused_lengths(rs.up, rs.down, nch, True, fo.I32)):
            nsrc = 1 + (k + nch) % 4
            stems = p24.decode(p24.random_clip(rng, Lin, nsrc * nch)).T.copy() * np.float32(1.2)   # past full scale
            got = _twice(lambda: encode(ctx, stems, nsrc, I24, (k + nch) % 16, rs, Lout))
            i32, fenced = encode(ctx, stems, nsrc, fo.I32, 0, rs, Lout)
            assert fenced and np.array_equal(got.reshape(-1), _i32_top3(i32.view(np.int32))), (rate, nch, nsrc, Lin, Lout)
            y32 = rs.resample(torch.from_numpy(stems).cuda(), num_out=Lout).cpu().numpy()
            assert np.array_equal(got, _v3_bytes(p24.interleave(y32, nsrc).reshape(nsrc, -1)))


def test_channel_groups_at_192k(ctx, resamplers):
    rs = resamplers(192000, ro.MODEL_RATE)
    assert fo.decode_groups(192000, 16, I24) > 1
    pcm = p24.random_clip(np.random.default_rng(4), 9001, 16)
    n0 = ctx.launch_count()
    got, fenced = decode(ctx, pcm, I24, 5, rs, rs.length(9001))
    n1 = ctx.launch_count()
    want, _ = decode(ctx, p24.to_i32(pcm), fo.I32, 0, rs, rs.length(9001))
    assert fenced and n1 - n0 == ctx.launch_count() - n1 == 2 and got.tobytes() == want.tobytes()


@pytest.mark.parametrize("rate", [22050, 48000, 192000])
def test_windowed_kernels_are_int32s(ctx, resamplers, rate):
    """dcs_channels_decode_range / _encode_range at odd addresses: the I32 windows' planes and bytes >> 8"""
    to, back = resamplers(rate, ro.MODEL_RATE), resamplers(ro.MODEL_RATE, rate)
    rng = np.random.default_rng(rate + 7)
    L = int(0.4 * rate) + 3
    Lm = to.length(L)
    for nch in (1, 6, 16):
        pcm = p24.random_clip(rng, L, nch)
        i0, i1 = L // 5, L - L // 7
        o0, n = to.length(i0) + 40, to.length(i1) - to.length(i0) - 200
        outs = []
        for fmt, rec, off in ((I24, pcm, 3), (fo.I32, p24.to_i32(pcm), 0)):
            keep, pin = _bytes_at(np.ascontiguousarray(rec[i0:i1]).tobytes(), off)
            out = _planes_out((nch + 1) * n)
            _lib().check(ctx.lib.dcs_channels_decode_range(ctx.handle, to.handle, fmt, pin, L, i0, i1 - i0, nch,
                                                           out.data_ptr() + 4 * 64, o0, n, None))
            outs.append(out.cpu().numpy())
        assert outs[0].tobytes() == outs[1].tobytes(), (rate, nch)
        nsrc = 2
        stems = p24.decode(p24.random_clip(rng, n, nsrc * nch)).T.copy() * np.float32(1.1)
        ds = torch.from_numpy(stems).cuda()
        e0 = back.length(o0 + 200)                       # 200 stems of margin: more than any rate's filter reaches
        en = back.length(o0 + n - 200) - e0
        got = []
        for fmt, b, off in ((I24, 3, 11), (fo.I32, 4, 0)):
            dout, pout = _bytes_at(b"\x5a" * (nsrc * nch * en * b), off)
            _lib().check(ctx.lib.dcs_channels_encode_range(ctx.handle, back.handle, fmt, ds.data_ptr(), Lm, o0, n, nsrc, nch,
                                                           pout, e0, en, nch * en, None))
            raw = dout.cpu().numpy()
            assert np.all(raw[:PADB + off] == SENT) and np.all(raw[PADB + off + nsrc * nch * en * b:] == SENT)
            got.append(raw[PADB + off:PADB + off + nsrc * nch * en * b])
        assert np.array_equal(got[0], _i32_top3(got[1].view(np.int32))), (rate, nch)


# ---------------------------------------------------------------------------------------------- 3. batch
def separator(arch="dsd", N=1024, seed=5, overlap=25, patcher="standalone"):
    from deepconvsep_b200.engine import Separator
    F = N // 2 + 1
    return Separator(nets.make_synthetic_params(arch, F, seed=seed), arch=arch, frame_size=N, hop=512, window="hanning",
                     overlap=overlap, patcher=patcher, feat_size=F)


def audio24(L, nch, seed):
    """[L, nch] V3 at full scale: two sources at different gains and delays per channel, clipped at both ends"""
    n = max(L, 4410) + 64
    a, _ = pipeline.synth_mixture(n / 44100.0, seed)
    b, _ = pipeline.synth_mixture(n / 44100.0, seed + 1)
    rng = np.random.default_rng(seed)
    cols = []
    for c in range(nch):
        g, h = rng.uniform(-1.0, 1.0, 2)
        cols.append(g * np.roll(a, int(rng.integers(0, 60))) + h * np.roll(b, int(rng.integers(0, 60))))
    x = np.stack(cols, axis=1)[:L]
    x = 1.25 * x / max(np.abs(x).max(), 1e-9)
    return p24.pack(np.clip(np.round(x * 2 ** 23), -2 ** 23, 2 ** 23 - 1).astype(np.int64))


FMTS = {fo.I16: np.dtype(np.int16), fo.I32: np.dtype(np.int32), fo.F32: np.dtype(np.float32), I24: p24.PCM24}


def as_fmt(clip24, fmt):
    """the same audio in fmt: int32 and float32 carry the 24-bit values exactly, int16 their top 16 bits"""
    v = p24.unpack(clip24).astype(np.int64)
    return {I24: clip24, fo.I32: (v << 8).astype(np.int32), fo.F32: (v / 2.0 ** 23).astype(np.float32),
            fo.I16: (v >> 8).astype(np.int16)}[fmt]


def float_route(sep, clip, fin, fout, rate=44100, wiener=0, wiener_radius=0):
    planes = p24.decode(clip) if fin == I24 else fo.decode(clip, fin)
    x = torch.from_numpy(np.ascontiguousarray(planes.T)).cuda()
    stems = sep.separate_channels(x, wiener=wiener, wiener_radius=wiener_radius, sample_rate=rate).cpu().numpy()
    L, nch = clip.shape
    stems = stems.reshape(sep.nsrc * nch, L)
    return p24.interleave(stems, sep.nsrc) if fout == I24 else fo.interleave(stems, sep.nsrc, fout)


@pytest.mark.parametrize("rate", [44100, 48000])
def test_every_pair_with_i24(rate):
    sep = separator("dsd", 1024, seed=40)
    nch = 6
    base = [audio24(int(0.9 * rate), nch, 800), audio24(3001, nch, 801)]
    pairs = [(I24, f) for f in FMTS] + [(f, I24) for f in (fo.I16, fo.I32, fo.F32)]
    assert len(pairs) == 7
    got = {}
    for fin, fout in pairs:
        clips = [as_fmt(c, fin) for c in base]
        got[fin, fout] = sep.separate_channels_batch(clips, out_dtype=FMTS[fout], sample_rate=rate)
        for g, c in zip(got[fin, fout], clips):
            assert g.shape == (sep.nsrc, c.shape[0], nch) and g.dtype == FMTS[fout]
            assert fo.same_bits(g, float_route(sep, c, fin, fout, rate)), (rate, fin, fout, c.shape)
    # the ties to int32: 24-bit in is int32 (v << 8) in, 24-bit out is int32 out >> 8
    i32_f32 = sep.separate_channels_batch([as_fmt(c, fo.I32) for c in base], out_dtype=np.float32, sample_rate=rate)
    i32_i32 = sep.separate_channels_batch([as_fmt(c, fo.I32) for c in base], out_dtype=np.int32, sample_rate=rate)
    for k in range(2):
        assert fo.same_bits(got[I24, fo.F32][k], i32_f32[k])
        assert fo.same_bits(got[I24, fo.I32][k], i32_i32[k])
        assert np.array_equal(_v3_bytes(got[I24, I24][k].reshape(-1, 1)).reshape(-1), _i32_top3(i32_i32[k]))
        assert np.array_equal(_v3_bytes(got[fo.I32, I24][k].reshape(-1, 1)).reshape(-1), _i32_top3(i32_i32[k]))
    assert np.abs(p24.unpack(got[I24, I24][0]).astype(np.int64)).sum() > 0


def test_wiener_and_launch_counts():
    sep = separator("dsd", 1024, seed=45)
    rate = 48000
    clip = audio24(3 * rate, 6, 820)
    got = sep.separate_channels_batch([clip], wiener=2, wiener_radius=2, sample_rate=rate)[0]
    assert fo.same_bits(got, float_route(sep, clip, I24, I24, rate, 2, 2))
    counts = {}
    for rate in (44100, 48000, 192000):
        for fmt in (fo.I32, I24):
            clips = [as_fmt(audio24(int(s * rate), 16 if rate == 192000 else 6, 830 + k), fmt) for k, s in enumerate((0.5, 0.3))]
            sep.separate_channels_batch(clips, sample_rate=rate)
            n0 = sep.ctx.launch_count()
            sep.separate_channels_batch(clips, sample_rate=rate)
            counts[rate, fmt] = sep.ctx.launch_count() - n0
        assert counts[rate, fo.I32] == counts[rate, I24], counts


@pytest.mark.parametrize("rate,nch,fin,fout", [(44100, 6, I24, I24), (48000, 8, I24, fo.F32), (96000, 3, fo.I16, I24)])
def test_workspace_formula(rate, nch, fin, fout):
    clips = [as_fmt(audio24(int(s * rate), nch, 840 + k), fin) for k, s in enumerate((1.7, 3.3, 2.1))]
    Lmax = max(c.shape[0] for c in clips)
    batch = separator("dsd", 2048, seed=47)
    batch.separate_channels_batch(clips, out_dtype=FMTS[fout], sample_rate=rate)
    Lm = batch.resampler(rate, 44100).length(Lmax) if rate != 44100 else Lmax
    single = separator("dsd", 2048, seed=47)
    single.separate_channels(torch.zeros((nch, Lm), dtype=torch.float32, device="cuda"))
    rounded = lambda x: (x + MB - 1) // MB * MB   # noqa: E731
    bi, bo = FMTS[fin].itemsize, FMTS[fout].itemsize
    want = (single.ctx.workspace_bytes() - rounded(4 * Lm) + rounded(4 * (nch + 1) * Lm) + rounded(4 * batch.nsrc * nch * Lm)
            + 2 * rounded(bi * nch * Lmax) + 2 * rounded(bo * batch.nsrc * nch * Lmax))
    assert batch.ctx.workspace_bytes() == want


# ---------------------------------------------------------------------------------------------- 4. long recordings
def contract24(sep, rec, rate, core):
    """the per-segment byte contract of include/dcs.h with I24 in and out -> [nsrc, L, C] V3"""
    L, nch = rec.shape
    segs = sep.long_segments(L, 0, 0, rate, segment_seconds=core / rate)
    out = np.zeros((sep.nsrc, L, nch), dtype=p24.PCM24)
    ctx = sep.ctx
    for sg in segs:
        if rate == ro.MODEL_RATE:
            clip = np.ascontiguousarray(rec[sg.in_start:sg.in_stop])
            got = sep.separate_channels_batch([clip])[0]
            out[:, sg.out_start:sg.out_stop] = got[:, sg.out_start - sg.in_start:sg.out_stop - sg.in_start]
            continue
        to, back = sep.resampler(rate, ro.MODEL_RATE), sep.resampler(ro.MODEL_RATE, rate)
        Sm = sg.model_stop - sg.model_start
        keep, pin = _bytes_at(np.ascontiguousarray(rec[sg.in_start:sg.in_stop]).tobytes(), 0)
        planes = torch.empty((nch + 1, Sm), dtype=torch.float32, device="cuda")
        _lib().check(ctx.lib.dcs_channels_decode_range(ctx.handle, to.handle, I24, pin, L, sg.in_start,
                                                       sg.in_stop - sg.in_start, nch, planes.data_ptr(), sg.model_start, Sm,
                                                       None))
        stems = sep.separate_channels(planes[1:].contiguous()).reshape(sep.nsrc * nch, Sm).contiguous()
        n = sg.out_stop - sg.out_start
        dout = torch.zeros(sep.nsrc * nch * n * 3, dtype=torch.uint8, device="cuda")
        _lib().check(ctx.lib.dcs_channels_encode_range(ctx.handle, back.handle, I24, stems.data_ptr(), to.length(L),
                                                       sg.model_start, Sm, sep.nsrc, nch, dout.data_ptr(), sg.out_start, n,
                                                       nch * n, None))
        out[:, sg.out_start:sg.out_stop] = dout.cpu().numpy().view(p24.PCM24).reshape(sep.nsrc, n, nch)
    return out, segs


@pytest.mark.parametrize("rate", [44100, 48000])
def test_long_segment_contract(rate):
    sep = separator("dsd", 1024, seed=50)
    rec = audio24(int(7.3 * rate), 6, 850)
    core = int(2.5 * rate)
    got = sep.separate_long_channels(rec, sample_rate=rate, segment_seconds=core / rate)
    want, segs = contract24(sep, rec, rate, core)
    assert len(segs) >= 3 and got.dtype == p24.PCM24 and fo.same_bits(got, want)
    # the long path's ties to int32, and one segment is the batch
    i32 = sep.separate_long_channels(as_fmt(rec, fo.I32), out_dtype=np.int32, sample_rate=rate, segment_seconds=core / rate)
    assert np.array_equal(_v3_bytes(got.reshape(-1, 1)).reshape(-1), _i32_top3(i32))
    one = sep.separate_long_channels(rec, sample_rate=rate, segment_seconds=rec.shape[0] / rate + 1)
    assert fo.same_bits(one, sep.separate_channels_batch([rec], sample_rate=rate)[0])


def test_long_from_a_wav_memmap(tmp_path):
    from deepconvsep_b200 import util
    sep = separator("dsd", 1024, seed=51)
    rec = audio24(int(5.1 * 48000), 6, 860)
    util.write_wav(str(tmp_path / "r.wav"), 48000, rec)
    rate, mm = util.wav_samples(str(tmp_path / "r.wav"))
    assert isinstance(mm, np.memmap) and rate == 48000
    got = sep.separate_long_channels(mm, sample_rate=rate, segment_seconds=2.0)
    assert fo.same_bits(got, sep.separate_long_channels(np.array(rec), sample_rate=rate, segment_seconds=2.0))
    util.write_wav(str(tmp_path / "s.wav"), rate, got[1])
    assert fo.same_bits(util.wav_samples(str(tmp_path / "s.wav"))[1], got[1])


def test_code_3_refused():
    sep = separator("dsd", 1024, seed=52)
    ctx, lib = sep.ctx, sep.lib
    rec = audio24(4000, 2, 870)
    out = np.empty((sep.nsrc, 4000, 2), dtype=p24.PCM24)
    sep.separate_long_channels(rec)
    n0 = ctx.launch_count()
    for fin, fout in ((3, I24), (I24, 3)):
        with pytest.raises(_lib().DcsError, match="unknown sample format"):
            _lib().check(lib.dcs_separate_long_channels_host(
                ctx.handle, sep.model.handle, sep.stft.handle, None, None, fin, fout, rec.ctypes.data, 4000, 2, 0, 0, 4000,
                C.c_float(sep.scale_factor), sep.overlap, sep.patcher, out.ctypes.data, 4000, None))
    d = torch.zeros(4096, dtype=torch.uint8, device="cuda")
    assert lib.dcs_channels_decode(ctx.handle, None, 3, d.data_ptr() + 1, 10, 2, d.data_ptr() + 1024, 10, None) == -1
    assert ctx.launch_count() == n0 and not d.any()
