"""Stems of the mono DSD100 / HHDS network from its masks: at N = 1024 / 2048 (the register inverse STFT) the mask kernel
writes the blended masks and the inverse STFT forms M_s * X as it reads each row, with one X row ring shared by the
groups of the four sources.  Everything here is bit for bit:

- the stems equal the plain inverse STFT (dcs_istft) of the masked spectra the spectrum tap received from the same
  call, for clips shorter than a frame, of a length that is not a multiple of the hop, and of 180 s;
- the tap equals the masks of dcs_separate_masks times the mixture STFT, componentwise in fp32, with zero pad columns;
- the masked inverse STFT (dcs_istft_masked) equals dcs_istft on the same M * X for source counts that fill the
  quads of a CTA exactly, leave groups idle or split into chunks, with one and two channels."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

SR = 44100
_SEPS = {}


def _sep(N, hop):
    from deepconvsep_b200.engine import Separator
    from oracle import nets
    if (N, hop) not in _SEPS:
        params = nets.make_synthetic_params("dsd", N // 2 + 1, seed=3)
        _SEPS[(N, hop)] = Separator(params, frame_size=N, hop=hop, window="hanning", overlap=25, device=0)
    return _SEPS[(N, hop)]


def _clip(L, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    t = torch.arange(L, device="cuda", dtype=torch.float32) / SR
    x = 0.3 * torch.sin(2 * np.pi * 220.0 * t) + 0.1 * torch.randn(L, device="cuda", generator=g)
    return x.clamp(-0.99, 0.99).contiguous()


def _tapped(sep, x):
    """stems and the masked spectra [nsrc, T, ldf] of one separate_device call with the spectrum tap on"""
    from deepconvsep_b200 import _lib
    from deepconvsep_b200.engine import _ptr
    T = sep.stft.num_frames(x.numel())
    tap = torch.full((sep.nsrc, T, sep.stft.ldf), complex(float("nan"), float("nan")), dtype=torch.complex64, device="cuda")
    out = torch.empty((sep.nsrc, x.numel()), dtype=torch.float32, device="cuda")
    _lib.check(sep.lib.dcs_set_spectrum_tap(sep.ctx.handle, _ptr(tap), tap.numel()))
    try:
        n0 = sep.ctx.launch_count()
        sep.separate_device(x, out)
        torch.cuda.synchronize()
        launches = sep.ctx.launch_count() - n0
    finally:
        _lib.check(sep.lib.dcs_set_spectrum_tap(sep.ctx.handle, None, 0))
    return out, tap, launches


# lengths: shorter than a frame, not a multiple of the hop (even, and odd: stems rows of odd length are not 8-byte
# aligned, so that clip keeps the masked spectra in memory), and 180 s
CASES = [(N, hop, L) for N in (1024, 2048) for hop in (512, 256) for L in (N - 200, 3 * SR + 138, 3 * SR + 137)] + [
    (2048, 512, 180 * SR), (1024, 512, 180 * SR)]


@pytest.mark.parametrize("N,hop,L", CASES, ids=["N%d_hop%d_L%d" % c for c in CASES])
def test_stems_equal_istft_of_tap(N, hop, L):
    sep = _sep(N, hop)
    x = _clip(L, N + hop + L)
    got, tap, _ = _tapped(sep, x)
    want = sep.stft.inverse(tap, num_out=L)
    assert torch.equal(got, want), int((got != want).sum())
    # the same clip without the tap: the same stems; from masks, one launch fewer (the tap's elementwise pass)
    again = torch.empty_like(got)
    n0 = sep.ctx.launch_count()
    sep.separate_device(x, again)
    torch.cuda.synchronize()
    assert torch.equal(got, again)
    assert sep.ctx.launch_count() - n0 == _tapped(sep, x)[2] - (L % 2 == 0)


@pytest.mark.parametrize("N,hop,L", [(1024, 512, 5 * SR + 12), (2048, 256, 4 * SR + 302), (2048, 512, 1500)])
def test_tap_is_masks_times_x(N, hop, L):
    sep = _sep(N, hop)
    x = _clip(L, 7 * N + hop)
    _, tap, _ = _tapped(sep, x)
    F = N // 2 + 1
    M = sep.separate_masks(x)                                      # [nsrc, T, ldf] device planes
    X = sep.stft.forward(x, want_mag=False)[0]                     # [T, ldf]
    want = torch.view_as_real(X)[None, :, :F] * M[:, :, :F, None]  # one rounded fp32 product per component
    got = torch.view_as_real(tap)
    assert torch.equal(got[:, :, :F], want)
    assert (got[:, :, F:] == 0).all()


MASKED = [(N, hop, nsrc, nx) for N, hop in ((1024, 256), (2048, 512)) for nsrc in (1, 2, 3, 4, 5, 8) for nx in (1, 2)]


@pytest.mark.parametrize("N,hop,nsrc,nx", MASKED, ids=["N%d_hop%d_nsrc%d_nx%d" % c for c in MASKED])
def test_masked_equals_plain(N, hop, nsrc, nx):
    from deepconvsep_b200.engine import Context, Stft
    ctx = Context(0)
    st = Stft(ctx, N, hop, "hanning")
    T, ldf, F = 700 + 3 * nsrc + nx, st.ldf, N // 2 + 1
    g = torch.Generator(device="cuda").manual_seed(N * 100 + nsrc * 10 + nx)
    X = torch.complex(torch.randn((nx, T, ldf), device="cuda", generator=g), torch.randn((nx, T, ldf), device="cuda", generator=g))
    M = torch.rand((nsrc, T, ldf), device="cuda", generator=g)
    L = st.out_length(T) - 77
    got = st.inverse_masked(X, M, num_out=L)
    S = torch.view_as_complex((torch.view_as_real(X)[None] * M[:, None, :, :, None]).contiguous())   # [nsrc, nx, T, ldf]
    S[..., F:] = 0
    want = st.inverse(S.reshape(nsrc * nx, T, ldf), num_out=L)
    assert torch.equal(got, want), int((got != want).sum())
    st.close()
