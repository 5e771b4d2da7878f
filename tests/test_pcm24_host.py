"""Packed 24-bit PCM (DCS_SAMPLE_I24, engine.PCM24) without a GPU:

- the numpy rules of tests/pcm24_oracle.py against scipy.io.wavfile's int32 read of hand-built 24-bit WAV files and
  against the int32 encode shifted right by 8, with explicit values at full scale, NaN and infinities;
- Separator.separate_channels_batch / separate_long_channels against a stand-in library: V3 clips and out_dtype PCM24
  pass code 4, shapes and dtypes, refusals before any library call;
- the fused kernels' tile plan for I24: int32's, over every accepted rate and C = 1..16;
- util.wav_samples / write_wav: round trips in all four formats, plain and WAVE_FORMAT_EXTENSIBLE headers, what scipy
  reads of them, RF64 per EBU Tech 3306 on a hand-built header and on write, and the refusals."""
import ctypes as C
import struct
from types import SimpleNamespace

import numpy as np
import pytest
import scipy.io.wavfile

import channels_formats_oracle as fo
import pcm24_oracle as p24
import resample_oracle as ro
from deepconvsep_b200 import engine, util, _lib
from deepconvsep_b200.engine import Separator

NSRC = 4
GUID_TAIL = b"\x00\x00\x00\x00\x10\x00\x80\x00\x00\xaa\x00\x38\x9b\x71"


def wav_bytes(data, C, rate, bits, tag=1, extensible=False, valid=None, rf64=False, extra=b""):
    """a WAV file built field by field: fmt (plain or EXTENSIBLE), an optional chunk before data, the data chunk"""
    b = bits // 8
    if extensible:
        fmt = struct.pack("<HHIIHHHHI", 0xFFFE, C, rate, rate * C * b, C * b, bits, 22, valid or bits, 0)
        fmt += struct.pack("<H", tag) + GUID_TAIL
    else:
        fmt = struct.pack("<HHIIHH", tag, C, rate, rate * C * b, C * b, bits)
    body = b"fmt " + struct.pack("<I", len(fmt)) + fmt + extra
    body += b"data" + struct.pack("<I", 0xFFFFFFFF if rf64 else len(data)) + data + b"\x00" * (len(data) & 1)
    if rf64:
        ds64 = b"ds64" + struct.pack("<IQQQI", 28, 4 + 36 + len(body), len(data), len(data) // (C * b), 0)
        return b"RF64" + struct.pack("<I", 0xFFFFFFFF) + b"WAVE" + ds64 + body
    return b"RIFF" + struct.pack("<I", 4 + len(body)) + b"WAVE" + body


# ---------------------------------------------------------------------------------------------- 1. the rules
@pytest.mark.parametrize("extensible", [False, True])
def test_decode_is_the_int32_route_on_scipys_read(tmp_path, extensible):
    rng = np.random.default_rng(1)
    for nch in (1, 2, 6):
        v = p24.values24()
        rows = v.size // nch
        pcm = p24.random_clip(rng, rows + 1001, nch)
        pcm[:rows] = p24.pack(v[:rows * nch].reshape(rows, nch))
        path = tmp_path / ("x%d.wav" % nch)
        path.write_bytes(wav_bytes(pcm.tobytes(), nch, 48000, 24, extensible=extensible, extra=b"LIST\x04\x00\x00\x00abcd"))
        rate, i32 = scipy.io.wavfile.read(str(path))
        i32 = i32.reshape(len(i32), -1)
        assert rate == 48000 and i32.dtype == np.int32
        assert np.array_equal(i32, p24.to_i32(pcm))
        assert fo.same_bits(p24.decode(pcm), fo.decode(i32, fo.I32))
        assert fo.same_bits(p24.decode_channels(pcm), fo.decode_channels(i32, fo.I32))
        rate2, mm = util.wav_samples(str(path))
        assert rate2 == 48000 and mm.dtype == engine.PCM24 and fo.same_bits(mm, pcm)


def test_encode_is_the_int32_encode_shifted():
    y = p24.stem_values()
    got = p24.unpack(p24.encode(y)).astype(np.int64)
    assert np.array_equal(got, fo.encode(y, fo.I32).astype(np.int64) >> 8)
    assert np.array_equal(p24.encode(y).view(np.uint8).reshape(-1, 3),
                          fo.encode(y, fo.I32).view(np.uint8).reshape(-1, 4)[:, 1:])      # the top 3 bytes
    pins = {1.0: b"\xff\xff\x7f", -1.0: b"\x00\x00\x80", np.nan: b"\x00\x00\x00", np.inf: b"\xff\xff\x7f",
            -np.inf: b"\x00\x00\x80", 3e9: b"\xff\xff\x7f", -3e9: b"\x00\x00\x80", -0.0: b"\x00\x00\x00",
            0.5: b"\xff\xff\x3f", 2.0 ** -23: b"\x00\x00\x00", -2.0 ** -23: b"\xff\xff\xff",   # -255 >> 8 floors to -1
            np.float32(1.0 + 2 ** -23): b"\xff\xff\x7f"}
    for v, want in pins.items():
        assert p24.encode(np.float32(v)).tobytes() == want, v


def test_pack_unpack():
    v = p24.values24()
    assert np.array_equal(p24.unpack(p24.pack(v)), v)
    assert p24.pack([-1, 1, -2 ** 23]).tobytes() == b"\xff\xff\xff\x01\x00\x00\x00\x00\x80"


# ---------------------------------------------------------------------------------------------- 2. the Python methods
DT = {0: np.dtype(np.int16), 1: np.dtype(np.int32), 2: np.dtype(np.float32), 4: p24.PCM24}


def _view(ptr, n, dtype):
    return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_uint8)), shape=(n * dtype.itemsize,)).view(dtype)


def _fill(a, fout, s):
    """the stand-in separation: the clip as int32 (V3 shifted left by 8) over (s + 1), in fout (V3: shifted right by 8)"""
    x = p24.to_i32(a) if a.dtype == p24.PCM24 else a
    y = (x.astype(np.float64) / (s + 1))
    return p24.pack(y.astype(np.int32) >> 8) if DT[fout] == p24.PCM24 else y.astype(DT[fout])


class FakeLib(object):
    def __init__(self):
        self.calls = []

    def dcs_separate_batch_channels_host(self, ctx, model, plan, to, back, fin, fout, n, pin, lens, ch, iters, radius,
                                         scale, overlap, patcher, pout, strides, stream):
        Ls = _view(lens, n, np.dtype(np.int64))
        self.calls.append(("batch", to, back, fin, fout, n, ch))
        for i in range(n):
            a = _view(pin[i], Ls[i] * ch, DT[fin]).reshape(Ls[i], ch)
            o = _view(pout[i], NSRC * ch * Ls[i], DT[fout]).reshape(NSRC, Ls[i], ch)
            for s in range(NSRC):
                o[s] = _fill(a, fout, s)
        return 0

    def dcs_separate_long_channels_host(self, ctx, model, plan, to, back, fin, fout, h_in, L, ch, iters, radius, core, scale,
                                        overlap, patcher, h_out, out_stride, stream):
        self.calls.append(("long", to, back, fin, fout, L, ch))
        a = _view(h_in, L * ch, DT[fin]).reshape(L, ch)
        o = _view(h_out, NSRC * out_stride * ch, DT[fout]).reshape(NSRC, out_stride, ch)
        for s in range(NSRC):
            o[s, :L] = _fill(a, fout, s)
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


def test_codes():
    assert _lib.SAMPLE_I24 == 4 and engine.PCM24 == np.dtype("V3") and engine.PCM24.itemsize == 3
    assert 3 not in (_lib.SAMPLE_I16, _lib.SAMPLE_I32, _lib.SAMPLE_F32, _lib.SAMPLE_I24)


@pytest.mark.parametrize("din,dout", [(p24.PCM24, None), (p24.PCM24, np.int32), (p24.PCM24, np.float32),
                                      (p24.PCM24, np.int16), (np.int32, p24.PCM24), (np.float32, p24.PCM24),
                                      (np.int16, p24.PCM24)])
def test_batch_codes_shapes_and_dtypes(sep, din, dout):
    rng = np.random.default_rng(2)
    nch = 6
    if din is p24.PCM24:
        clips = [p24.random_clip(rng, L, nch) for L in (700, 1)]
    else:
        clips = [fo.random_clip(rng, L, nch, {np.int16: fo.I16, np.int32: fo.I32, np.float32: fo.F32}[din])
                 for L in (700, 1)]
    want_out = np.dtype(din if dout is None else dout)
    code = {v: k for k, v in DT.items()}
    for rate in (44100, 48000):
        got = sep.separate_channels_batch(clips, out_dtype=dout, sample_rate=rate)
        hs = (None, None) if rate == 44100 else ("h48000-44100", "h44100-48000")
        assert sep.lib.calls[-1] == ("batch",) + hs + (code[np.dtype(din)], code[want_out], 2, nch)
        for g, c in zip(got, clips):
            assert g.shape == (NSRC, c.shape[0], nch) and g.dtype == want_out and g.flags.c_contiguous
            for s in range(NSRC):
                assert fo.same_bits(g[s], _fill(c, code[want_out], s))


def test_long_takes_a_wav_memmap(sep, tmp_path):
    rng = np.random.default_rng(3)
    pcm = p24.random_clip(rng, 5000, 6)
    util.write_wav(str(tmp_path / "r.wav"), 48000, pcm)
    rate, mm = util.wav_samples(str(tmp_path / "r.wav"))
    assert isinstance(mm, np.memmap) and not mm.flags.writeable
    for dout, code in ((None, 4), (np.int32, 1), (p24.PCM24, 4)):
        out = sep.separate_long_channels(mm, out_dtype=dout, sample_rate=rate)
        assert sep.lib.calls[-1] == ("long", "h48000-44100", "h44100-48000", 4, code, 5000, 6)
        assert out.shape == (NSRC, 5000, 6) and out.dtype == DT[code]
        assert fo.same_bits(out[2], _fill(pcm, code, 2))
    out = np.empty((NSRC, 5000, 6), dtype=p24.PCM24)
    assert sep.separate_long_channels(pcm, out=out) is out and sep.lib.calls[-1][3:5] == (4, 4)


def test_refusals_before_any_library_call(sep):
    rng = np.random.default_rng(4)
    v3 = p24.random_clip(rng, 500, 6)
    i32 = p24.to_i32(v3)
    bad = {
        "V3 with int32": (dict(clips=[v3, i32]), "same dtype"),
        "int32 with V3": (dict(clips=[i32, v3]), "same dtype"),
        "1-D V3": (dict(clips=[v3[:, 0]]), "clips \\[L, C\\]"),
        "V6 clip": (dict(clips=[np.zeros((10, 2), dtype="V6")]), "int16 or int32 or float32"),
        "uint8 clip": (dict(clips=[np.zeros((10, 3), dtype=np.uint8)]), "int16 or int32 or float32"),
        "out V6": (dict(clips=[v3], out_dtype="V6"), "V6"),
        "out 'pcm24'": (dict(clips=[v3], out_dtype="pcm24"), "not a dtype"),
        "17 channels": (dict(clips=[p24.random_clip(rng, 50, 17)]), "16 channels"),
        "wiener on nine channels": (dict(clips=[p24.random_clip(rng, 50, 9)], wiener=1), None),
        "44 099 Hz": (dict(clips=[v3], sample_rate=44099), "44099"),
    }
    for name, (kw, msg) in bad.items():
        with pytest.raises(ValueError, match=msg):
            sep.separate_channels_batch(**kw)
    for kw in (dict(recording=v3[:, 0]), dict(recording=v3, out_dtype="V6"), dict(recording=v3, out_dtype="pcm24"),
               dict(recording=v3, out=np.empty((NSRC, 500, 6), dtype=np.int32))):
        with pytest.raises(ValueError):
            sep.separate_long_channels(**kw)
    assert sep.lib.calls == []


# ---------------------------------------------------------------------------------------------- 3. tile plans
def test_i24_plans_are_int32s_at_every_accepted_rate():
    lo, hi = engine.RESAMPLE_RATES
    rates = [r for r in range(lo, hi + 1) if ro.accepted(r) and r != ro.MODEL_RATE]
    assert len(rates) == 7379
    for rate in rates:
        for d in ((rate, 44100), (44100, rate)):
            up, down = ro.ratio(*d)
            for nch in range(1, 17):
                for enc in (False, True):
                    plan = fo.pcm_plan(up, down, nch, enc, p24.I24)
                    assert plan is not None and plan == fo.pcm_plan(up, down, nch, enc, fo.I32), (d, nch, enc)
    assert fo.decode_groups(192000, 16, p24.I24) > 1


# ---------------------------------------------------------------------------------------------- 4. WAV helpers
def _samples(rng, dtype, L, nch):
    if dtype == p24.PCM24:
        return p24.random_clip(rng, L, nch)
    if dtype == np.float32:
        return rng.uniform(-1.5, 1.5, (L, nch)).astype(np.float32)
    info = np.iinfo(dtype)
    return rng.integers(info.min, info.max, (L, nch), endpoint=True).astype(dtype)


@pytest.mark.parametrize("dtype", [np.int16, p24.PCM24, np.int32, np.float32], ids=["i16", "i24", "i32", "f32"])
@pytest.mark.parametrize("extensible", [False, True])
def test_wav_round_trip_and_scipy(tmp_path, dtype, extensible):
    rng = np.random.default_rng(5)
    for nch, L in ((1, 1001), (2, 7), (6, 4099), (16, 3)):
        x = _samples(rng, np.dtype(dtype), L, nch)
        path = str(tmp_path / "w.wav")
        util.write_wav(path, 96000, x, extensible=extensible)
        with open(path, "rb") as f:
            raw = f.read()
        assert raw[:4] == b"RIFF" and struct.unpack("<I", raw[4:8])[0] == len(raw) - 8
        assert struct.unpack("<H", raw[20:22])[0] == (0xFFFE if extensible else (3 if dtype == np.float32 else 1))
        rate, y = util.wav_samples(path)
        assert rate == 96000 and y.dtype == np.dtype(dtype) and y.shape == (L, nch) and fo.same_bits(y, x)
        rate, z = scipy.io.wavfile.read(path)
        z = z.reshape(L, nch)
        assert rate == 96000
        if dtype == p24.PCM24:
            assert z.dtype == np.int32 and np.array_equal(z, p24.to_i32(x))
        else:
            assert fo.same_bits(z, x)
    util.write_wav(str(tmp_path / "m.wav"), 8000, x[:, 0])            # [L] is one channel
    assert util.wav_samples(str(tmp_path / "m.wav"))[1].shape == (3, 1)


def test_wav_header_choice_and_odd_data(tmp_path):
    path = str(tmp_path / "o.wav")
    util.write_wav(path, 44100, p24.pack(np.arange(-3, 2)[:, None]))  # 15 bytes: one pad byte
    raw = open(path, "rb").read()
    assert len(raw) % 2 == 0 and raw[20:22] == b"\xfe\xff"            # > 16 bits: EXTENSIBLE by default
    assert np.array_equal(p24.unpack(util.wav_samples(path)[1][:, 0]), np.arange(-3, 2))
    util.write_wav(path, 44100, np.zeros((4, 2), np.int16))
    assert open(path, "rb").read()[20:22] == b"\x01\x00"
    util.write_wav(path, 44100, np.zeros((4, 3), np.int16))
    assert open(path, "rb").read()[20:22] == b"\xfe\xff"
    util.write_wav(path, 44100, np.arange(6, dtype=">i4").reshape(3, 2))   # big-endian input, little-endian file
    assert np.array_equal(util.wav_samples(path)[1], np.arange(6).reshape(3, 2))


def test_rf64_read_hand_built(tmp_path):
    """EBU Tech 3306: RF64 id, RIFF size 0xFFFFFFFF, a ds64 chunk first holding the RIFF and data sizes, data size
    0xFFFFFFFF in the data chunk"""
    rng = np.random.default_rng(6)
    for dtype, bits, tag in ((p24.PCM24, 24, 1), (np.int16, 16, 1), (np.float32, 32, 3)):
        x = _samples(rng, np.dtype(dtype), 777, 6)
        path = tmp_path / "r.wav"
        path.write_bytes(wav_bytes(x.tobytes(), 6, 48000, bits, tag=tag, extensible=True, rf64=True))
        rate, y = util.wav_samples(str(path))
        assert rate == 48000 and y.dtype == np.dtype(dtype) and fo.same_bits(y, x)


def test_rf64_write_past_four_gigabytes(tmp_path, monkeypatch):
    """RF64 is written when the file would pass 2^32 - 1 bytes: the threshold lowered here so that a small file crosses
    it; the layout is the one the hand-built header has"""
    rng = np.random.default_rng(7)
    x = p24.random_clip(rng, 1000, 16)
    path = str(tmp_path / "big.wav")
    monkeypatch.setattr(util, "_RIFF_LIMIT", 40000)
    util.write_wav(path, 48000, x)
    raw = open(path, "rb").read()
    assert raw[:4] == b"RF64" and raw[4:8] == b"\xff\xff\xff\xff" and raw[12:16] == b"ds64"
    riff, data, count = struct.unpack("<QQQ", raw[20:44])
    assert riff == len(raw) - 8 and data == x.nbytes and count == 1000
    assert raw.index(b"data") + 8 + x.nbytes == len(raw)
    assert raw[raw.index(b"data") + 4:raw.index(b"data") + 8] == b"\xff\xff\xff\xff"
    assert fo.same_bits(util.wav_samples(path)[1], x)
    monkeypatch.setattr(util, "_RIFF_LIMIT", 0xFFFFFFFF)
    util.write_wav(path, 48000, x)                                     # below the real limit: RIFF
    assert open(path, "rb").read()[:4] == b"RIFF"


def test_wav_refusals(tmp_path):
    path = tmp_path / "bad.wav"
    cases = {
        "8-bit": (wav_bytes(b"\x00" * 8, 2, 8000, 8), "0x0001 with 8-bit"),
        "64-bit float": (wav_bytes(b"\x00" * 16, 1, 8000, 64, tag=3), "0x0003 with 64-bit"),
        "A-law": (wav_bytes(b"\x00" * 8, 1, 8000, 8, tag=6), "0x0006"),
        "extensible A-law": (wav_bytes(b"\x00" * 8, 1, 8000, 8, tag=6, extensible=True), "0x0006"),
        "24-bit float": (wav_bytes(b"\x00" * 6, 1, 8000, 24, tag=3), "0x0003 with 24-bit"),
        "valid 28 of 24": (wav_bytes(b"\x00" * 6, 1, 8000, 24, extensible=True, valid=28), "28 valid"),
        "not WAVE": (b"RIFX" + b"\x00" * 40, "not a RIFF"),
        "no data": (wav_bytes(b"", 1, 8000, 16)[:36], "no data"),
        "truncated": (wav_bytes(b"\x00" * 64, 2, 8000, 16)[:-10], "claims 64 bytes"),
    }
    for name, (raw, msg) in cases.items():
        path.write_bytes(raw)
        with pytest.raises(ValueError, match=msg):
            util.wav_samples(str(path))
    # 20-bit samples in a 3-byte container use the 24-bit rule
    path.write_bytes(wav_bytes(b"\x10\x00\x80" * 2, 1, 8000, 24, extensible=True, valid=20))
    assert util.wav_samples(str(path))[1].dtype == p24.PCM24
    for x in (np.zeros((4, 2), np.float64), np.zeros((4, 2), np.uint8), np.zeros((4, 2), "V6"), np.zeros((2, 2, 2), np.int16)):
        with pytest.raises(ValueError, match="write_wav takes"):
            util.write_wav(str(tmp_path / "o.wav"), 8000, x)
