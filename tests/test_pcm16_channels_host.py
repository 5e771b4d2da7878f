"""Separator.separate_pcm16_channels_batch without a GPU: the arguments it passes to
dcs_separate_batch_pcm16_channels_host, the interleaved int16 layouts in and out, and the ValueErrors it raises before
any library call, against a stand-in library working on host memory."""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest

from deepconvsep_b200 import engine
from deepconvsep_b200.engine import Separator

NSRC = 4


def _i16(ptr, n):
    """the n int16 values at address ptr"""
    return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_int16)), shape=(n,))


def _i64(ptr, n):
    return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_int64)), shape=(n,))


class FakeLib(object):
    """source s of clip i = clip i // (s + 1), value for value, in the interleaved layout"""

    def __init__(self):
        self.calls = []

    def dcs_separate_batch_pcm16_channels_host(self, ctx, model, plan, n, pin, lens, ch, iters, radius, scale, overlap,
                                               patcher, pout, strides, stream):
        Ls, st = _i64(lens, n).copy(), _i64(strides, n).copy()
        self.calls.append((ctx, model, plan, n, ch, iters, radius, scale, overlap, patcher, tuple(Ls), tuple(st), stream))
        for i in range(n):
            L = int(Ls[i])
            a = _i16(pin[i], L * ch).reshape(L, ch)
            o = _i16(pout[i], NSRC * ch * int(st[i])).reshape(NSRC, int(st[i]), ch)
            for s in range(NSRC):
                o[s, :L] = a // (s + 1)
        return 0


@pytest.fixture
def sep(monkeypatch):
    monkeypatch.setattr(engine, "_stream_ptr", lambda stream=None, device=None: None)
    lib = FakeLib()
    s = object.__new__(Separator)
    s.lib, s.nsrc, s.scale_factor, s.overlap, s.patcher = lib, NSRC, 0.3, 25, 1
    s.ctx = SimpleNamespace(handle=1, device=0, lib=lib)
    s.model = SimpleNamespace(arch="dsd", handle=2)
    s.stft = SimpleNamespace(handle=3)
    return s


def _clips(nch, lengths, seed=0):
    rng = np.random.default_rng(seed)
    return [rng.integers(-30000, 30000, (L, nch)).astype(np.int16) for L in lengths]


@pytest.mark.parametrize("nch", [1, 2, 6, 16])
def test_arguments_and_layouts(sep, nch):
    clips = _clips(nch, (700, 1300, 50), seed=nch)
    got = sep.separate_pcm16_channels_batch(clips, wiener=2 if 2 <= nch <= 8 else 0,
                                            wiener_radius=3 if 2 <= nch <= 8 else 0)
    k = 2 if 2 <= nch <= 8 else 0
    call = sep.lib.calls[-1]
    assert call[:7] == (1, 2, 3, 3, nch, k, 3 if k else 0)
    assert abs(call[7] - 0.3) < 1e-7 and call[8:10] == (25, 1)
    assert call[10] == call[11] == (700, 1300, 50) and call[12] is None
    assert len(got) == 3
    for g, c in zip(got, clips):
        assert g.shape == (NSRC, c.shape[0], nch) and g.dtype == np.int16 and g.flags.c_contiguous
        for s in range(NSRC):
            assert np.array_equal(g[s], c // (s + 1))


def test_outs_and_non_contiguous_clips(sep):
    base = _clips(12, (900,), seed=3)[0]
    clip = base[:, ::2]                                      # a strided view: 6 channels
    outs = [np.zeros((NSRC, 900, 6), dtype=np.int16)]
    got = sep.separate_pcm16_channels_batch([clip], outs=outs)
    assert got[0] is outs[0]
    assert np.array_equal(outs[0][3], clip // 4)
    assert sep.separate_pcm16_channels_batch([]) == [] and len(sep.lib.calls) == 1


def test_refusals_before_any_library_call(sep):
    six = _clips(6, (500,))[0]
    bad = {
        "mixed channel counts": dict(clips=[six, _clips(4, (500,))[0]]),
        "float clip": dict(clips=[six.astype(np.float32)]),
        "int32 clip": dict(clips=[six.astype(np.int32)]),
        "1-D clip": dict(clips=[six[:, 0]]),
        "3-D clip": dict(clips=[six[None]]),
        "17 channels": dict(clips=_clips(17, (500,))),
        "wiener on one channel": dict(clips=[six[:, :1]], wiener=1),
        "wiener on nine channels": dict(clips=_clips(9, (500,)), wiener=1),
        "negative wiener": dict(clips=[six], wiener=-1),
        "negative radius": dict(clips=[six], wiener=1, wiener_radius=-1),
        "radius without wiener": dict(clips=[six], wiener_radius=2),
    }
    for name, kw in bad.items():
        with pytest.raises(ValueError):
            sep.separate_pcm16_channels_batch(**kw)
        assert sep.lib.calls == [], name
    for arch in ("dsd_ild", "bach10_score", "bach10_score_1x1"):
        sep.model.arch = arch
        with pytest.raises(ValueError, match="separate_masks"):
            sep.separate_pcm16_channels_batch([six])
    assert sep.lib.calls == []
    # the existing keep-channels batch still takes stereo clips only
    sep.model.arch = "dsd"
    with pytest.raises(ValueError, match="stereo"):
        sep.separate_pcm16_batch([six], keep_channels=True)
    assert sep.lib.calls == []
