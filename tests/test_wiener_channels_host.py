"""The C-channel Wiener post-filter without a GPU: the float64 oracle (tests/wiener_channels_oracle.py) against the
two-channel oracles, its algebra (the sources plus the residual give the mixture, channel permutations, the
equal-channel closed form), and the marshalling of engine.wiener_channels and Separator.separate_channels(wiener=...)
against a stand-in library, refusals included."""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest

from oracle import wiener as W
import wiener_channels_oracle as wco
import wiener_local_oracle as wlo

from deepconvsep_b200 import engine
from deepconvsep_b200.engine import Separator


def spectra(C_, nsrc, T, F, seed):
    """a mixture of nsrc sources with complex per-channel gains (so R_j has complex off-diagonal terms), and soft-mask
    stems of it"""
    rng = np.random.default_rng(seed)
    src = (rng.standard_normal((nsrc, T, F)) + 1j * rng.standard_normal((nsrc, T, F))) * rng.gamma(0.5, 1.0, (nsrc, T, F))
    gains = rng.uniform(0.2, 1.0, (nsrc, C_, 1, 1)) * np.exp(1j * rng.uniform(-np.pi, np.pi, (nsrc, C_, 1, F)))
    img = gains * src[:, None] * 30.0
    X = img.sum(axis=0)
    mag = np.abs(img).sum(axis=1) * rng.uniform(1.0, 1.5, (nsrc, T, F))
    Y = (mag / mag.sum(axis=0))[:, None] * X[None]
    return X, Y


def rel(a, b):
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


# ---------------------------------------------------------------------------------------------- the oracle
@pytest.mark.parametrize("K", [1, 2])
def test_two_channels_are_the_stereo_oracles(K):
    X, Y = spectra(2, 4, 300, 24, K)
    assert rel(wco.wiener(X, Y, K), W.wiener(X, Y, K)) <= 1e-12
    for radius in (1, 3):
        assert rel(wco.wiener(X, Y, K, radius), wlo.wiener_windowed(X, Y, K, radius)) <= 1e-12


@pytest.mark.parametrize("C_,radius", [(3, 0), (6, 0), (6, 1)])
def test_sources_and_residual_give_the_mixture(C_, radius):
    X, Y = spectra(C_, 3, 260, 16, C_)
    Y1 = wco.em_step(X, Y, wco._scales(X, radius), radius)
    res = wco.residual(X, Y, radius)
    assert rel(Y1.sum(axis=0) + res, X) <= 1e-12
    assert np.linalg.norm(res) < 0.05 * np.linalg.norm(X)          # the sources take nearly all of it


def test_permuting_the_channels_permutes_the_output():
    X, Y = spectra(5, 2, 200, 12, 9)
    perm = [3, 0, 4, 1, 2]
    want = wco.wiener(X, Y, 2)
    got = wco.wiener(X[perm], Y[:, perm], 2)
    assert rel(got, want[:, perm]) <= 1e-12


@pytest.mark.parametrize("C_", [2, 3, 6])
def test_equal_channels_closed_form(C_):
    rng = np.random.default_rng(C_)
    a = (rng.standard_normal((200, 10)) + 1j * rng.standard_normal((200, 10))) * 20.0
    m = rng.uniform(0.0, 1.0, (4, 200, 10))
    b = m / m.sum(axis=0) * a[None]
    X = np.repeat(a[None], C_, axis=0)
    Y = np.repeat(b[:, None], C_, axis=1)
    got = wco.wiener(X, Y, 2)
    want = wco.equal_channels(a, b, C_, 2)
    for c in range(C_):
        assert rel(got[:, c], want) <= 1e-10


# ---------------------------------------------------------------------------------------------- marshalling
def _host(ptr, n, ctype=C.c_float):
    return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(ctype)), shape=(n,))


class FakeLib(object):
    """the entry points on host memory: the filter scales every stem plane by 2, the pipelines write (s + 1) * channel
    c (and + 100 * iterations + radius with the filter)"""

    def __init__(self):
        self.calls = []

    def dcs_wiener_channels(self, ctx, X, nx, x_plane, S, src_stride, nsrc, T, ldf, F, iterations, radius, stream):
        self.calls.append(("wiener", nx, x_plane, src_stride, nsrc, T, ldf, F, iterations, radius))
        s = _host(S, 2 * nsrc * nx * src_stride)
        s *= 2
        return 0

    def _stems(self, x, nx, stride, L, out, ostride, extra):
        a = _host(x, nx * stride).reshape(nx, stride)
        o = _host(out, 4 * nx * ostride).reshape(4 * nx, ostride)
        for s in range(4):
            for c in range(nx):
                o[s * nx + c, :L] = (s + 1) * a[c, :L] + extra

    def dcs_separate_audio_channels(self, ctx, model, plan, x, nx, stride, L, scale, overlap, patcher, out, ostride, stream):
        self.calls.append(("channels", nx, stride, L, scale, overlap, patcher, ostride))
        self._stems(x, nx, stride, L, out, ostride, 0)
        return 0

    def dcs_separate_audio_channels_wiener(self, ctx, model, plan, x, nx, stride, L, scale, overlap, patcher, iterations, radius,
                                           out, ostride, stream):
        self.calls.append(("channels_wiener", nx, stride, L, scale, overlap, patcher, iterations, radius, ostride))
        self._stems(x, nx, stride, L, out, ostride, 100 * iterations + radius)
        return 0


@pytest.fixture
def torch_host(monkeypatch):
    torch = pytest.importorskip("torch")
    monkeypatch.setattr(engine, "_stream_ptr", lambda stream=None, device=None: None)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))     # host tensors stand for device planes
    return torch


@pytest.fixture
def sep(torch_host, monkeypatch):
    from deepconvsep_b200.engine import Stft
    lib = FakeLib()
    s = object.__new__(Separator)
    s.lib, s.nsrc, s.scale_factor, s.overlap, s.patcher = lib, 4, 0.3, 25, 0
    s.ctx = SimpleNamespace(handle=1, device=0, lib=lib)
    s.model = SimpleNamespace(arch="dsd", handle=2, F=513)
    st = object.__new__(Stft)
    st.ctx, st.lib, st.N, st.hop, st.device, st.F, st.ldf, st.handle = s.ctx, lib, 1024, 512, 0, 513, 520, 3
    monkeypatch.setattr(Stft, "dev", property(lambda self: torch_host.device("cpu")))
    s.stft = st
    return s


@pytest.mark.parametrize("nx", [2, 3, 8])
def test_wiener_channels_arguments(torch_host, nx):
    torch = torch_host
    lib = FakeLib()
    ctx = SimpleNamespace(handle=1, device=0, lib=lib)
    T, ldf = 37, 520
    X = torch.zeros((nx, T, ldf), dtype=torch.complex64)
    S = torch.ones((2 * nx, T, ldf), dtype=torch.complex64)
    assert engine.wiener_channels(ctx, X, S, 3, num_bins=513, radius=2) is S
    assert lib.calls == [("wiener", nx, T * ldf, T * ldf, 2, T, ldf, 513, 3, 2)]
    assert bool((S == 2).all())
    engine.wiener_channels(ctx, X, S, 1)
    assert lib.calls[-1] == ("wiener", nx, T * ldf, T * ldf, 2, T, ldf, ldf, 1, 0)


def test_wiener_channels_refusals(torch_host):
    torch = torch_host
    lib = FakeLib()
    ctx = SimpleNamespace(handle=1, device=0, lib=lib)
    T, ldf = 20, 40

    def z(*shape, dtype=torch.complex64):
        return torch.zeros(shape, dtype=dtype)
    bad = {
        "one channel": (z(1, T, ldf), z(4, T, ldf)),
        "nine channels": (z(9, T, ldf), z(9, T, ldf)),
        "stems not a multiple of nx": (z(3, T, ldf), z(7, T, ldf)),
        "shape mismatch": (z(3, T, ldf), z(6, T + 1, ldf)),
        "float32": (z(3, T, ldf, dtype=torch.float32), z(6, T, ldf, dtype=torch.float32)),
        "strided rows": (z(3, T, 2 * ldf)[:, :, ::2], z(6, T, ldf)),
    }
    for name, (X, S) in bad.items():
        with pytest.raises(ValueError):
            engine.wiener_channels(ctx, X, S, 1)
        assert lib.calls == [], name


@pytest.mark.parametrize("nx", [2, 6, 8])
def test_separate_channels_wiener_arguments(sep, nx):
    torch = pytest.importorskip("torch")
    L = 2000
    audio = np.random.default_rng(nx).uniform(-1, 1, (L, nx))
    plain = sep.separate_channels(audio)
    assert sep.lib.calls[-1] == ("channels", nx, L, L, 0.3, 25, 0, L)
    assert sep.separate_channels(audio, wiener=0).tobytes() == plain.tobytes()        # wiener 0: today's call
    assert sep.lib.calls[-1][0] == "channels"
    got = sep.separate_channels(audio, wiener=2, wiener_radius=3)
    assert sep.lib.calls[-1] == ("channels_wiener", nx, L, L, 0.3, 25, 0, 2, 3, L)
    assert got.shape == (L, 4, nx) and np.array_equal(got, plain + np.float32(203))
    x = torch.as_tensor(np.ascontiguousarray(audio.T.astype(np.float32)))
    planes = sep.separate_channels(x, wiener=1)
    assert sep.lib.calls[-1] == ("channels_wiener", nx, L, L, 0.3, 25, 0, 1, 0, L)
    assert tuple(planes.shape) == (4 * nx, L)


def test_separate_channels_wiener_refusals(sep):
    torch = pytest.importorskip("torch")
    L = 1000
    refused = {
        "one channel": lambda: sep.separate_channels(np.zeros((L, 1)), wiener=1),
        "mono vector": lambda: sep.separate_channels(np.zeros(L), wiener=1),
        "nine channels": lambda: sep.separate_channels(np.zeros((L, 9)), wiener=1),
        "nine device planes": lambda: sep.separate_channels(torch.zeros((9, L)), wiener=1),
        "negative radius": lambda: sep.separate_channels(np.zeros((L, 3)), wiener=1, wiener_radius=-1),
        "orphan radius": lambda: sep.separate_channels(np.zeros((L, 3)), wiener_radius=2),
        "negative iterations": lambda: sep.separate_channels(np.zeros((L, 3)), wiener=-1),
    }
    for name, call in refused.items():
        with pytest.raises(ValueError):
            call()
        assert sep.lib.calls == [], name
    sep.separate_channels(np.zeros((L, 9)))           # without the filter nine channels are fine
    assert sep.lib.calls[-1][:2] == ("channels", 9)
