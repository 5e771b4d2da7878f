"""Separator.separate_channels_batch without a GPU, and the host restatements of the int32 / float32 sample formats:

- against a stand-in library: the format codes passed for each clip dtype and out_dtype, 44.1 kHz and other rates
  reaching dcs_separate_batch_channels_host with NULL or the separator's resamplers, output shapes and dtypes, and every
  refusal raised before any library call;
- the fused kernels' tile plan with 4-byte staging, enumerated over every accepted rate, C = 1..16 and both sides: a
  plan always exists, and the pairs whose decode takes channel groups (one more launch) are the ones include/dcs.h
  names;
- numpy restatements of the int32 and float32 rules against the host routes they promise the bits of."""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest

import channels_formats_oracle as fo
import pcm16_oracle as po
import resample_oracle as ro
from deepconvsep_b200 import engine
from deepconvsep_b200.engine import Separator

NSRC = 4
CT = {np.dtype(np.int16): C.c_int16, np.dtype(np.int32): C.c_int32, np.dtype(np.float32): C.c_float,
      np.dtype(np.int64): C.c_int64}


def _arr(ptr, n, dtype):
    return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(CT[np.dtype(dtype)])), shape=(n,))


class FakeLib(object):
    """source s of clip i = the clip's samples over (s + 1), cast to the output dtype, in the interleaved layout"""

    def __init__(self):
        self.calls = []

    def dcs_separate_batch_channels_host(self, ctx, model, plan, to, back, fin, fout, n, pin, lens, ch, iters, radius,
                                         scale, overlap, patcher, pout, strides, stream):
        Ls = tuple(int(v) for v in _arr(lens, n, np.int64))
        st = tuple(int(v) for v in _arr(strides, n, np.int64))
        self.calls.append((ctx, model, plan, to, back, fin, fout, n, ch, iters, radius, scale, overlap, patcher, Ls, st,
                           stream))
        din, dout = fo.DTYPES[fin], fo.DTYPES[fout]
        for i in range(n):
            a = _arr(pin[i], Ls[i] * ch, din).reshape(Ls[i], ch)
            o = _arr(pout[i], NSRC * ch * st[i], dout).reshape(NSRC, st[i], ch)
            for s in range(NSRC):
                o[s, :Ls[i]] = (a.astype(np.float64) / (s + 1)).astype(dout)
        return 0

    def __getattr__(self, name):
        raise AssertionError("unexpected library call %s" % name)


class FakeResampler(object):
    made = []

    def __init__(self, ctx, rate_in, rate_out):
        engine.check_resample_rates(rate_in, rate_out)
        self.handle = "h%d-%d" % (int(rate_in), int(rate_out))
        FakeResampler.made.append((int(rate_in), int(rate_out)))


@pytest.fixture
def sep(monkeypatch):
    monkeypatch.setattr(engine, "_stream_ptr", lambda stream=None, device=None: None)
    monkeypatch.setattr(engine, "Resampler", FakeResampler)
    FakeResampler.made = []
    lib = FakeLib()
    s = object.__new__(Separator)
    s.lib, s.nsrc, s.scale_factor, s.overlap, s.patcher = lib, NSRC, 0.3, 25, 1
    s.ctx = SimpleNamespace(handle=1, device=0, lib=lib)
    s.model = SimpleNamespace(arch="dsd", handle=2)
    s.stft = SimpleNamespace(handle=3)
    s._resamplers = {}
    return s


def _clips(dtype, nch, lengths, seed=0):
    rng = np.random.default_rng(seed)
    fmt = {np.int16: fo.I16, np.int32: fo.I32, np.float32: fo.F32}[dtype]
    return [fo.random_clip(rng, L, nch, fmt) for L in lengths]


# ---------------------------------------------------------------------------------------------- 1. the Python method
@pytest.mark.parametrize("din", [np.int16, np.int32, np.float32])
@pytest.mark.parametrize("dout", [None, np.int16, np.int32, np.float32])
def test_format_codes_shapes_and_dtypes(sep, din, dout):
    nch = 6
    clips = _clips(din, nch, (700, 1300, 1), seed=3)
    got = sep.separate_channels_batch(clips, out_dtype=dout, wiener=2, wiener_radius=3)
    want_out = np.dtype(din if dout is None else dout)
    call = sep.lib.calls[-1]
    codes = {np.dtype(np.int16): 0, np.dtype(np.int32): 1, np.dtype(np.float32): 2}
    assert call[:11] == (1, 2, 3, None, None, codes[np.dtype(din)], codes[want_out], 3, nch, 2, 3)
    assert abs(call[11] - 0.3) < 1e-7 and call[12:14] == (25, 1)
    assert call[14] == call[15] == (700, 1300, 1) and call[16] is None
    assert FakeResampler.made == []
    for g, c in zip(got, clips):
        assert g.shape == (NSRC, c.shape[0], nch) and g.dtype == want_out and g.flags.c_contiguous
        for s in range(NSRC):
            assert np.array_equal(g[s], (c.astype(np.float64) / (s + 1)).astype(want_out))


@pytest.mark.parametrize("rate,nch,dtype", [(48000, 6, np.int32), (8000, 1, np.float32), (192000, 16, np.int32),
                                            (96000, 2, np.int16)])
def test_other_rates_pass_the_resamplers(sep, rate, nch, dtype):
    clips = _clips(dtype, nch, (900, 5), seed=nch)
    got = sep.separate_channels_batch(clips, out_dtype=np.float32, sample_rate=rate)
    call = sep.lib.calls[-1]
    assert call[3:7] == ("h%d-44100" % rate, "h44100-%d" % rate, {np.int16: 0, np.int32: 1, np.float32: 2}[dtype], 2)
    assert [g.shape for g in got] == [(NSRC, 900, nch), (NSRC, 5, nch)] and all(g.dtype == np.float32 for g in got)
    sep.separate_channels_batch(clips[:1], sample_rate=[rate])
    assert FakeResampler.made == [(rate, 44100), (44100, rate)]
    assert sep.lib.calls[-1][3:7] == ("h%d-44100" % rate, "h44100-%d" % rate, sep.lib.calls[-1][5], sep.lib.calls[-1][5])


def test_outs_and_strided_clips(sep):
    base = _clips(np.int32, 12, (400,), seed=5)[0]
    clip = base[:, ::2]
    outs = [np.zeros((NSRC, 400, 6), dtype=np.float32)]
    got = sep.separate_channels_batch([clip], outs=outs, out_dtype="float32", sample_rate=44100.0)
    assert got[0] is outs[0] and np.array_equal(outs[0][1], (clip.astype(np.float64) / 2).astype(np.float32))
    assert sep.separate_channels_batch([]) == [] and len(sep.lib.calls) == 1


def test_refusals_before_any_library_call(sep):
    six = _clips(np.int32, 6, (500,))[0]
    bad = {
        "float64 clip": (dict(clips=[six.astype(np.float64)]), "int16 or int32 or float32"),
        "uint8 clip": (dict(clips=[six.astype(np.uint8)]), "int16 or int32 or float32"),
        "int64 clip": (dict(clips=[six.astype(np.int64)]), "int16 or int32 or float32"),
        "1-D clip": (dict(clips=[six[:, 0]]), "clips \\[L, C\\]"),
        "mixed dtypes": (dict(clips=[six, six.astype(np.float32)]), "same dtype"),
        "mixed channel counts": (dict(clips=[six, six[:, :4]]), "channel count"),
        "17 channels": (dict(clips=_clips(np.float32, 17, (50,))), "16 channels"),
        "out_dtype float64": (dict(clips=[six], out_dtype=np.float64), "float64"),
        "out_dtype uint16": (dict(clips=[six], out_dtype=np.uint16), "uint16"),
        "out_dtype not a dtype": (dict(clips=[six], out_dtype="pcm24"), "not a dtype"),
        "out_dtype bad, no clips": (dict(clips=[], out_dtype=np.float64), "float64"),
        "44 099 Hz": (dict(clips=[six], sample_rate=44099), "44099"),
        "mixed rates": (dict(clips=[six, six], sample_rate=[48000, 96000]), "one sample rate"),
        "wiener on nine channels": (dict(clips=_clips(np.int16, 9, (50,)), wiener=1), None),
        "negative wiener": (dict(clips=[six], wiener=-1), None),
        "radius without wiener": (dict(clips=[six], wiener_radius=2), None),
    }
    for name, (kw, msg) in bad.items():
        with pytest.raises(ValueError, match=msg):
            sep.separate_channels_batch(**kw)
        assert sep.lib.calls == [] and FakeResampler.made == [], name
    for arch in ("dsd_ild", "bach10_score"):
        sep.model.arch = arch
        with pytest.raises(ValueError, match="separate_masks"):
            sep.separate_channels_batch([six], sample_rate=48000)
    assert sep.lib.calls == [] and FakeResampler.made == []


def test_pcm16_method_keeps_its_messages(sep):
    """separate_pcm16_channels_batch shares the checks; its refusals still name it and int16"""
    with pytest.raises(ValueError, match="separate_pcm16_channels_batch needs int16 clips"):
        sep.separate_pcm16_channels_batch(_clips(np.int32, 2, (10,)))
    with pytest.raises(ValueError, match="separate_pcm16_channels_batch takes 1 to 16 channels"):
        sep.separate_pcm16_channels_batch(_clips(np.int16, 17, (10,)))
    with pytest.raises(ValueError, match="separate_pcm16_channels_batch takes one sample rate"):
        sep.separate_pcm16_channels_batch(_clips(np.int16, 2, (10, 10)), sample_rate=[48000])
    assert sep.lib.calls == []


# ---------------------------------------------------------------------------------------------- 2. tile plans
def accepted_rates():
    """the rates a clip may have other than the networks' 44.1 kHz"""
    lo, hi = engine.RESAMPLE_RATES
    return [r for r in range(lo, hi + 1) if ro.accepted(r) and r != ro.MODEL_RATE]


def test_closed_form_plan_is_the_kernel_loop():
    """the closed form of channels_formats_oracle against pcm16_oracle's loop, where both apply (int16 decode, encode)"""
    for rate in ro.TABLE_RATES:
        for d in ((rate, 44100), (44100, rate)):
            up, down = ro.ratio(*d)
            for C in range(1, 17):
                for enc in (False, True):
                    tp, cn, _ = fo.pcm_plan(up, down, C, enc, fo.I16)
                    assert (tp, cn) == po.pcm_plan(up, down, C, enc), (d, C, enc)


def test_four_byte_plans_over_every_accepted_rate():
    rates = accepted_rates()
    assert len(rates) == 7379
    grouped = []
    for rate in rates:
        for d in ((rate, 44100), (44100, rate)):
            up, down = ro.ratio(*d)
            for C in range(1, 17):
                for enc in (False, True):
                    for fmt in (fo.I16, fo.I32, fo.F32):
                        plan = fo.pcm_plan(up, down, C, enc, fmt)
                        assert plan is not None, (d, C, enc, fmt)
                        tp, cn, groups = plan
                        assert tp >= fo.RS_V and tp % fo.RS_V == 0 and groups * cn >= C > (groups - 1) * cn
                        if not enc:
                            assert fmt != fo.I16 or groups == 1      # the int16 decode never splits
                # the encode stages fp32 stems in every format: one plan
                assert len({fo.pcm_plan(up, down, C, True, f) for f in (fo.I16, fo.I32, fo.F32)}) == 1
        for C in range(1, 17):
            g = fo.decode_groups(rate, C, fo.I32)
            assert g == fo.decode_groups(rate, C, fo.F32)
            if g > 1:
                grouped.append((rate, C))
    # dcs.h: C >= 11 at some rates, 192 kHz at C = 16 among them
    assert len(grouped) == 3179
    assert min(C for _, C in grouped) >= 11 and (192000, 16) in grouped and (48000, 16) not in grouped
    assert all((r, C + 1) in grouped for r, C in grouped if C < 16)     # more channels never fit better


# ---------------------------------------------------------------------------------------------- 3. the rules
def test_int32_decode_is_the_scripts_host_route():
    v = fo.int32_values()
    got = fo.decode(v, fo.I32)
    want = (v.astype(float) / np.iinfo(np.int32).max).astype(np.float32)
    assert fo.same_bits(got, want)
    assert got[v == 2 ** 31 - 1][0] == 1.0 and got[v == -2 ** 31][0] == np.float32(-2.0 ** 31 / fo.I32_MAX)
    # a 24-bit file read by scipy: 0x7fffff -> 2147483392, decoded to just under 1
    assert fo.decode(np.int32([0x7fffff << 8]), fo.I32)[0] == np.float32(2147483392 / fo.I32_MAX) < 1.0


def test_int32_encode_saturates_and_truncates():
    y = fo.i32_stem_values()
    got = fo.encode(y, fo.I32)
    assert got.dtype == np.int32
    finite = np.isfinite(y) & (np.abs(y.astype(np.float64) * fo.I32_MAX) < 2.0 ** 31 - 1)
    want = np.trunc(y[finite].astype(np.float64) * fo.I32_MAX).astype(np.int64)
    assert np.array_equal(got[finite].astype(np.int64), want)
    special = {np.float32(np.inf): 2 ** 31 - 1, np.float32(-np.inf): -2 ** 31, np.float32(3e9): 2 ** 31 - 1,
               np.float32(-3e9): -2 ** 31, np.float32(1.0): 2 ** 31 - 1, np.float32(-1.0): -(2 ** 31 - 1),
               np.float32(1.5): 2 ** 31 - 1, np.float32(-1.5): -2 ** 31}
    for k, v in special.items():
        assert fo.encode(np.float32([k]), fo.I32)[0] == v, k
    assert np.all(fo.encode(y[np.isnan(y)], fo.I32) == 0)
    above = np.nextafter(np.float32(1.0), np.float32(2))
    assert fo.encode(np.float32([above]), fo.I32)[0] == 2 ** 31 - 1            # saturates, never wraps
    # decode then encode gives every 24-bit value back in the top bytes, within one LSB of the 32-bit word
    v = fo.int32_values()
    back = fo.encode(fo.decode(v, fo.I32), fo.I32).astype(np.int64)
    assert np.all(np.abs(back - v) <= 256)


def test_float32_is_a_bit_copy():
    y = fo.stem_values(fo.F32)
    assert fo.same_bits(fo.encode(y, fo.F32), y) and fo.same_bits(fo.decode(y, fo.F32), y)
    assert fo.same_bits(fo.encode(fo.NAN_PAYLOADS, fo.F32), fo.NAN_PAYLOADS)


def test_int16_rules_are_pcm16_oracles():
    v = po.all_int16(3)
    assert fo.same_bits(fo.decode_channels(v, fo.I16), po.decode_channels(v))
    y = po.stem_values()
    assert fo.same_bits(fo.encode(y, fo.I16), po.encode(y))


def test_interleave_and_downmix_in_every_format():
    rng = np.random.default_rng(7)
    for fmt in (fo.I16, fo.I32, fo.F32):
        pcm = fo.random_clip(rng, 33, 5, fmt)
        planes = fo.decode_channels(pcm, fmt)
        assert planes.shape == (6, 33) and planes.dtype == np.float32
        assert fo.same_bits(planes[0], po.downmix(planes[1:]))
        stems = rng.uniform(-2, 2, (2 * 5, 33)).astype(np.float32)
        out = fo.interleave(stems, 2, fmt)
        assert out.shape == (2, 33, 5) and out.dtype == fo.DTYPES[fmt]
        assert fo.same_bits(out[1, :, 3], fo.encode(stems[5 + 3], fmt))
