"""Separator.separate_pcm16_channels_batch(sample_rate=...) without a GPU: the arguments and resampler handles it passes
to dcs_separate_batch_pcm16_channels_resampled_host, that 44.1 kHz still goes to dcs_separate_batch_pcm16_channels_host,
the output shapes at the clips' own length, and the ValueErrors raised before any library call, against a stand-in
library working on host memory."""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest

from deepconvsep_b200 import engine
from deepconvsep_b200.engine import Separator

NSRC = 4


def _i16(ptr, n):
    return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_int16)), shape=(n,))


def _i64(ptr, n):
    return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_int64)), shape=(n,))


def _fill(n, pin, lens, strides, ch, pout):
    """source s of clip i = clip i // (s + 1), value for value, in the interleaved layout"""
    Ls, st = _i64(lens, n).copy(), _i64(strides, n).copy()
    for i in range(n):
        L = int(Ls[i])
        a = _i16(pin[i], L * ch).reshape(L, ch)
        o = _i16(pout[i], NSRC * ch * int(st[i])).reshape(NSRC, int(st[i]), ch)
        for s in range(NSRC):
            o[s, :L] = a // (s + 1)
    return tuple(Ls), tuple(st)


class FakeLib(object):
    def __init__(self):
        self.calls = []

    def dcs_separate_batch_pcm16_channels_host(self, ctx, model, plan, n, pin, lens, ch, iters, radius, scale, overlap,
                                               patcher, pout, strides, stream):
        Ls, st = _fill(n, pin, lens, strides, ch, pout)
        self.calls.append(("44k", ctx, model, plan, n, ch, iters, radius, scale, overlap, patcher, Ls, st, stream))
        return 0

    def dcs_separate_batch_pcm16_channels_resampled_host(self, ctx, model, plan, to, back, n, pin, lens, ch, iters, radius,
                                                         scale, overlap, patcher, pout, strides, stream):
        Ls, st = _fill(n, pin, lens, strides, ch, pout)
        self.calls.append(("rate", ctx, model, plan, to, back, n, ch, iters, radius, scale, overlap, patcher, Ls, st, stream))
        return 0


class FakeResampler(object):
    """stands in for engine.Resampler: checks the rates as the real one does, and records that it was made"""
    made = []

    def __init__(self, ctx, rate_in, rate_out):
        engine.check_resample_rates(rate_in, rate_out)
        self.rate_in, self.rate_out = int(rate_in), int(rate_out)
        self.handle = "h%d-%d" % (self.rate_in, self.rate_out)
        FakeResampler.made.append((self.rate_in, self.rate_out))


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


def _clips(nch, lengths, seed=0):
    rng = np.random.default_rng(seed)
    return [rng.integers(-30000, 30000, (L, nch)).astype(np.int16) for L in lengths]


@pytest.mark.parametrize("rate,nch", [(48000, 6), (8000, 1), (96000, 2), (192000, 16), (64000, 8)])
def test_arguments_handles_and_shapes(sep, rate, nch):
    clips = _clips(nch, (700, 1300, 1), seed=nch)
    k = 2 if 2 <= nch <= 8 else 0
    got = sep.separate_pcm16_channels_batch(clips, wiener=k, wiener_radius=3 if k else 0, sample_rate=rate)
    call = sep.lib.calls[-1]
    assert call[0] == "rate"
    assert call[1:10] == (1, 2, 3, "h%d-44100" % rate, "h44100-%d" % rate, 3, nch, k, 3 if k else 0)
    assert abs(call[10] - 0.3) < 1e-7 and call[11:13] == (25, 1)
    assert call[13] == call[14] == (700, 1300, 1) and call[15] is None
    assert len(got) == 3
    for g, c in zip(got, clips):
        assert g.shape == (NSRC, c.shape[0], nch) and g.dtype == np.int16 and g.flags.c_contiguous
        for s in range(NSRC):
            assert np.array_equal(g[s], c // (s + 1))
    # the separator's resamplers are made once and kept
    sep.separate_pcm16_channels_batch(clips[:1], sample_rate=rate)
    assert FakeResampler.made == [(rate, 44100), (44100, rate)]
    assert sep.lib.calls[-1][3:6] == (3, "h%d-44100" % rate, "h44100-%d" % rate)


def test_model_rate_goes_to_the_44k_entry(sep):
    clips = _clips(6, (500, 300))
    outs = [np.zeros((NSRC, 500, 6), dtype=np.int16), np.zeros((NSRC, 300, 6), dtype=np.int16)]
    for kw in ({}, {"sample_rate": 44100}, {"sample_rate": 44100.0}, {"sample_rate": [44100, 44100]}):
        got = sep.separate_pcm16_channels_batch(clips, outs=outs, **kw)
        assert got[0] is outs[0] and got[1] is outs[1]
        assert sep.lib.calls[-1][0] == "44k" and sep.lib.calls[-1][3:8] == (3, 2, 6, 0, 0)
    assert FakeResampler.made == []
    assert len(sep.lib.calls) == 4


def test_outs_at_another_rate(sep):
    clip = _clips(12, (900,), seed=3)[0][:, ::2]             # a strided view: 6 channels
    outs = [np.zeros((NSRC, 900, 6), dtype=np.int16)]
    got = sep.separate_pcm16_channels_batch([clip], outs=outs, sample_rate=[48000])
    assert got[0] is outs[0] and np.array_equal(outs[0][3], clip // 4)
    assert sep.lib.calls[-1][0] == "rate"


def test_refusals_before_any_library_call(sep):
    six = _clips(6, (500,))[0]
    bad = {
        "44 099 Hz": (dict(clips=[six], sample_rate=44099), "44099"),
        "7 999 Hz": (dict(clips=[six], sample_rate=7999), "7999"),
        "192 001 Hz": (dict(clips=[six], sample_rate=192001), "192001"),
        "fractional rate": (dict(clips=[six], sample_rate=48000.5), "48000.5"),
        "bad rate, no clips": (dict(clips=[], sample_rate=44099), "44099"),
        "mixed rates": (dict(clips=[six, six], sample_rate=[48000, 96000]), "one sample rate"),
        "one rate for two clips": (dict(clips=[six, six], sample_rate=[48000]), "one sample rate"),
        "mixed channel counts": (dict(clips=[six, _clips(4, (500,))[0]], sample_rate=48000), "channel count"),
        "float clip": (dict(clips=[six.astype(np.float32)], sample_rate=48000), "int16"),
        "1-D clip": (dict(clips=[six[:, 0]], sample_rate=48000), "int16"),
        "17 channels": (dict(clips=_clips(17, (500,)), sample_rate=48000), "16 channels"),
        "wiener on nine channels": (dict(clips=_clips(9, (500,)), wiener=1, sample_rate=48000), None),
    }
    for name, (kw, msg) in bad.items():
        with pytest.raises(ValueError, match=msg):
            sep.separate_pcm16_channels_batch(**kw)
        assert sep.lib.calls == [] and FakeResampler.made == [], name
    sep.model.arch = "dsd_ild"
    with pytest.raises(ValueError, match="separate_masks"):
        sep.separate_pcm16_channels_batch([six], sample_rate=48000)
    assert sep.lib.calls == [] and FakeResampler.made == []
