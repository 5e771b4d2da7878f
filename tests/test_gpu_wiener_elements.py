"""The Wiener post-filter kernels (csrc/wiener.cu) element by element against float64, one EM iteration at a time, under
the bound of tests/wiener_elements_oracle.py:

- caller spectra, every nx in 2..8 x nsrc in 1..4 at radius 0 and 1, one radius covering the clip, and the shape edges
  (T around one chunk of 128 frames, F around the C-channel tiles of 32 bins and the stereo tiles of 128): nx = 2
  through dcs_wiener_stereo (radius 0) or dcs_wiener_stereo_windowed, with dcs_wiener_channels giving the same bits;
  nx >= 3 through dcs_wiener_channels.  K = 2 is, bit for bit, K = 1 applied twice, and each of the two iterations is
  checked against em_step fed the device's fp32 stems of the iteration before.  Every case: NaN in the pad bins and
  the gaps between planes stays NaN bit for bit, frames with every stem 0 stay exactly 0, a second run gives the same
  bits;
- the masked first pass (dcs_separate_audio_channels_wiener, iKala: 2 sources, DSD: 4; nx 2 .. 8): the iterations = 1
  spectrum tap against em_step of fl32(M_s * X_c), and the iterations = 2 tap is dcs_wiener_channels K = 1 applied to
  it, bit for bit.  The masked first passes of 1 and 3 sources are not run: no network the C-channel path accepts has
  that many sources (iKala 2, the others 4).

The worst err / bound ratio of every case goes to parity.record."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import wiener_elements_oracle as we  # noqa: E402
from parity import record  # noqa: E402
from test_gpu_wiener_channels import channels, downmix_masks, separator  # noqa: E402

NAN_BITS = np.uint32(0x7fc0beef)     # what the filter must neither read into a result nor write


@pytest.fixture(scope="module")
def ctx():
    from deepconvsep_b200.engine import Context
    return Context(0)


def planes(a, ldf, gap):
    """a [n, T, F] -> a device view [n, T, ldf] of planes T * ldf + gap apart with NaN_BITS in the pad bins and gaps,
    and the buffer under it"""
    n, T, F = a.shape
    fill = np.full((n, 2 * (T * ldf + gap)), NAN_BITS, dtype=np.uint32).view(np.complex64)
    buf = torch.from_numpy(fill).cuda()
    v = buf[:, :T * ldf].view(n, T, ldf)
    v[:, :, :F] = torch.from_numpy(np.ascontiguousarray(a, dtype=np.complex64)).cuda()
    return v, buf


def bits(buf):
    return buf.view(torch.int32).cpu().numpy()


def filt(ctx, entry, Xd, S, K, F, radius):
    """S (numpy [nsrc * nx, T, F]) through `entry` in NaN-fenced planes -> (the stems complex64 [nsrc * nx, T, F], the
    buffer's bits)"""
    from deepconvsep_b200 import _lib
    from deepconvsep_b200.engine import _ptr, wiener_channels, wiener_stereo
    T, ldf = Xd.shape[1], Xd.shape[2]
    Sd, buf = planes(S, ldf, 11)
    if entry == "stereo":
        assert radius == 0
        _lib.check(ctx.lib.dcs_wiener_stereo(ctx.handle, _ptr(Xd), Xd.stride(0), _ptr(Sd), Sd.stride(0), Sd.shape[0] // 2, T, ldf,
                                             F, K, None))
    elif entry == "stereo_windowed":
        wiener_stereo(ctx, Xd, Sd, K, num_bins=F, radius=radius)
    else:
        wiener_channels(ctx, Xd, Sd, K, num_bins=F, radius=radius)
    torch.cuda.synchronize()
    return Sd[:, :, :F].cpu().numpy(), bits(buf)


def fences_hold(b, T, ldf, F):
    """the pad bins and the gaps of a buffer from filt still hold NAN_BITS, bit for bit"""
    b = b.reshape(b.shape[0], -1)
    pad = b[:, :2 * T * ldf].reshape(-1, T, ldf, 2)[:, :, F:]
    return bool(np.all(b[:, 2 * T * ldf:] == NAN_BITS) and np.all(pad == NAN_BITS))


def check_iteration(name, X, Y, got, radius):
    nsrc, nx, T, F = Y.shape
    ref, slack = we.reference(X, Y, radius)
    res = we.check(got.reshape(Y.shape), ref, slack, radius)
    record(name, ratio=res["ratio"], where=str(res["where"]), fp64_fraction=res["fp64_fraction"])
    assert res["ok"], (name, res)


@pytest.mark.parametrize("c", we.CASES, ids=we.case_id)
def test_each_iteration_against_float64(c, ctx):
    nx, nsrc, T, F, radius = c
    X, Y = we.make_case(c)
    ldf = F + 3
    Xd, _ = planes(X, ldf, 5)
    entry = "channels" if nx > 2 else ("stereo" if radius == 0 else "stereo_windowed")
    Y0 = Y.reshape(nsrc * nx, T, F)
    y1, b1 = filt(ctx, entry, Xd, Y0, 1, F, radius)
    _, b1_again = filt(ctx, entry, Xd, Y0, 1, F, radius)
    assert np.array_equal(b1, b1_again)                                   # the same bits on a second run
    assert fences_hold(b1, T, ldf, F)
    y2, b2 = filt(ctx, entry, Xd, Y0, 2, F, radius)
    _, b2_composed = filt(ctx, entry, Xd, y1, 1, F, radius)
    assert np.array_equal(b2, b2_composed)                                # K = 2 is K = 1 twice, bit for bit
    assert fences_hold(b2, T, ldf, F)
    if nx == 2:                                                           # the C-channel entry at nx = 2: the same bits
        assert np.array_equal(filt(ctx, "channels", Xd, Y0, 2, F, radius)[1], b2)
    silent = ~Y0.any(axis=(0, 2))
    assert not y1[:, silent].any() and not y2[:, silent].any()             # frames with every stem 0 stay 0
    check_iteration("wiener_elements_%s_K1" % we.case_id(c), X, Y, y1, radius)
    check_iteration("wiener_elements_%s_K2" % we.case_id(c), X, y1.astype(np.complex128).reshape(Y.shape), y2, radius)


@pytest.fixture(scope="module")
def separators():
    cache = {}

    def get(arch):
        if arch not in cache:
            cache[arch] = separator(arch, 1024, 53 if arch == "dsd" else 59)
        return cache[arch]
    return get


def tapped(sep, x, K, radius):
    from deepconvsep_b200 import _lib
    L = x.shape[1]
    T, ldf = sep.stft.num_frames(L), sep.stft.ldf
    tap = torch.zeros((sep.nsrc * x.shape[0], T, ldf), dtype=torch.complex64, device="cuda")
    _lib.check(sep.lib.dcs_set_spectrum_tap(sep.ctx.handle, tap.data_ptr(), tap.numel()))
    try:
        sep.separate_channels(x, wiener=K, wiener_radius=radius)
        torch.cuda.synchronize()
    finally:
        _lib.check(sep.lib.dcs_set_spectrum_tap(sep.ctx.handle, None, 0))
    return tap


# iKala and DSD at nx in {2, 3, 5, 8} and radius 0 and 1, then nx = 4, 6 and 7 once per network, so that every masked
# first pass the networks reach runs
MASKED = [(arch, nx, radius) for arch in ("ikala", "dsd") for nx in (2, 3, 5, 8) for radius in (0, 1)] \
    + [("ikala", 4, 1), ("dsd", 4, 0), ("ikala", 6, 0), ("dsd", 6, 1), ("ikala", 7, 1), ("dsd", 7, 0)]


@pytest.mark.parametrize("arch,nx,radius", MASKED)
def test_masked_first_pass_against_float64(arch, nx, radius, separators):
    from deepconvsep_b200.engine import wiener_channels
    sep = separators(arch)
    nsrc = sep.nsrc
    audio = channels(2.5, nx, 7 * nx + radius)
    x = torch.tensor(np.ascontiguousarray(audio.T), device="cuda")
    F = sep.stft.F
    tap1, tap2 = tapped(sep, x, 1, radius), tapped(sep, x, 2, radius)
    M = np.ascontiguousarray(downmix_masks(sep, x)[:, :, :F].cpu().numpy())        # the device's masks, bitwise
    Xd = torch.stack([sep.stft.forward(x[c].contiguous(), want_mag=False)[0] for c in range(nx)]).contiguous()
    X = np.ascontiguousarray(Xd[:, :, :F].cpu().numpy())
    T = X.shape[1]
    Xr = X.view(np.float32).reshape(nx, T, F, 2)
    Y0 = (M[:, None, :, :, None] * Xr[None]).reshape(nsrc, nx, T, 2 * F).view(np.complex64)   # fl32(M_s * X_c)
    got = tap1[:, :, :F].cpu().numpy().reshape(nsrc, nx, T, F)
    check_iteration("wiener_elements_masked_%s_nx%d_W%d" % (arch, nx, radius), X.astype(np.complex128),
                    Y0.astype(np.complex128), got, radius)
    S = tap1.clone()
    wiener_channels(sep.ctx, Xd, S, 1, num_bins=F, radius=radius)
    torch.cuda.synchronize()
    assert torch.equal(S[:, :, :F].view(torch.int64), tap2[:, :, :F].view(torch.int64))   # masked K = 2 = masked K = 1, then K = 1
