"""The masked inverse STFT (dcs_istft_masked: istft_masked_reg_kernel at N = 1024 / 2048 with hop 256 / 512,
istft_masked_kernel everywhere else): output plane (s * nx + c) = istft_norm(M_s * X_c), the product formed while a
spectrum row is loaded.

- Bit for bit against dcs_istft on S = X * M formed by torch in fp32 (view_as_real(X) * M[..., None]), on every dispatch
  path.  The two kernels of a path share everything after the product, so the reference call is steered onto the same
  path: same output alignment, and a spectrum pointer 8- but not 16-byte aligned where a misaligned mask pointer moves
  the masked call off the register path.
- One case per path against the float64 inverse of tests/stft_views_oracle.py under its per-sample bound, so that the
  equality is tied to the reference and not only to a sibling kernel.
- NaN sits in every element the kernel must not use: pad columns of X and of M, Im of DC and Nyquist, the gaps where
  x_plane, m_stride and out_stride exceed the data, and SLACK elements around the inputs.  Outputs are pre-filled with a
  NaN-payload sentinel that must survive around and between the planes.  Every case runs twice and gives the same bits.
- Every refusal of the header returns DCS_EINVAL with nothing launched."""
import os
import sys
import zlib

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import stft_views_oracle as so  # noqa: E402
from parity import record  # noqa: E402

SLACK = so.SLACK
SENT = np.uint32(0x7FC5A5A5)      # quiet NaN with a payload no kernel produces


@pytest.fixture(scope="module")
def ctx():
    from deepconvsep_b200.engine import Context
    return Context(0)


_PLANS = {}


def _plan(ctx, N, H):
    from deepconvsep_b200.engine import Stft
    if (id(ctx), N, H) not in _PLANS:
        _PLANS[(id(ctx), N, H)] = Stft(ctx, N, H, "hanning")
    return _PLANS[(id(ctx), N, H)]


def _stream(ctx):
    from deepconvsep_b200.engine import _stream_ptr
    return _stream_ptr(None, ctx.device)


def _sentinels(n):
    return torch.from_numpy(np.full(n, SENT, np.uint32).view(np.float32)).cuda()


# name -> (N, hop, path, output offset in floats, mask offset in floats).  The register path needs an 8-byte aligned
# output and 16-byte aligned mask rows; either offset moves the register sizes onto the shared-memory kernel.
PATHS = {
    "reg_1024_256": (1024, 256, "reg", 0, 0), "reg_1024_512": (1024, 512, "reg", 0, 0),
    "reg_2048_256": (2048, 256, "reg", 0, 0), "reg_2048_512": (2048, 512, "reg", 0, 0),
    "smem_256": (256, 128, "smem", 0, 0), "smem_512": (512, 256, "smem", 0, 0), "smem_4096": (4096, 512, "smem", 0, 0),
    "smem_odd_hop": (1024, 186, "smem", 0, 0),
    "smem_forced_by_output": (2048, 512, "smem", 1, 0), "smem_forced_by_mask": (1024, 256, "smem", 0, 1),
}
SHAPES = [(nx, nsrc) for nx in (1, 2, 3) for nsrc in (1, 4)]


def _inputs(N, T, ldf, nx, nsrc, x_plane, m_stride, m_off, rng):
    """NaN everywhere but bins < F of each row (and Im of DC / Nyquist of X) -> device buffers, pointers, host values"""
    F = N // 2 + 1
    xb = np.full((2 * SLACK + nx * x_plane, 2), np.nan, np.float32)
    Xv = (rng.standard_normal((nx, T, F, 2)) * rng.uniform(0.1, 30.0, (nx, T, 1, 1))).astype(np.float32)
    for c in range(nx):
        rows = xb[SLACK + c * x_plane:SLACK + c * x_plane + T * ldf].reshape(T, ldf, 2)
        rows[:, :F] = Xv[c]
        rows[:, 0, 1] = np.nan
        rows[:, F - 1, 1] = np.nan
    mb = np.full(2 * SLACK + m_off + nsrc * m_stride, np.nan, np.float32)
    Mv = rng.uniform(0.0, 1.0, (nsrc, T, F)).astype(np.float32)
    Mv[:, :, ::7] = 0.0                      # exact zeros and ones, as the networks' masks hold them
    Mv[:, :, 3::11] = 1.0
    for s in range(nsrc):
        mb[SLACK + m_off + s * m_stride:SLACK + m_off + s * m_stride + T * ldf].reshape(T, ldf)[:, :F] = Mv[s]
    Xd, Md = torch.from_numpy(xb).cuda(), torch.from_numpy(mb).cuda()
    return Xd, Md, Xd.data_ptr() + 8 * SLACK, Md.data_ptr() + 4 * (SLACK + m_off), Xv, Mv


def _product(Xv, Mv, ldf, s_off):
    """S = X * M by torch in fp32, componentwise: planes (s * nx + c) [T, ldf], pad columns and Im of DC / Nyquist NaN;
    s_off = 1 leaves the spectrum pointer 8- but not 16-byte aligned"""
    nx, T, F = Xv.shape[:3]
    nsrc = Mv.shape[0]
    X, M = torch.from_numpy(Xv).cuda(), torch.from_numpy(Mv).cuda()
    P = (X[None] * M[:, None, :, :, None]).reshape(nsrc * nx, T, F, 2)
    buf = torch.full((s_off + nsrc * nx * T * ldf, 2), float("nan"), dtype=torch.float32, device="cuda")
    S = buf[s_off:].view(nsrc * nx, T, ldf, 2)
    S[:, :, :F] = P
    S[:, :, 0, 1] = float("nan")
    S[:, :, F - 1, 1] = float("nan")
    return buf, buf.data_ptr() + 8 * s_off, P.cpu().numpy()


def masked_case(ctx, name, nx, nsrc, oracle=False):
    N, H, path, o_off, m_off = PATHS[name]
    F, ldf, T = N // 2 + 1, so.padded_bins(N), 41
    st = _plan(ctx, N, H)
    rng = np.random.default_rng(zlib.crc32(("%s/%d/%d" % (name, nx, nsrc)).encode()))
    x_plane, m_stride = T * ldf + 6, T * ldf + 8
    mx = (T - 1) * H + N // 2
    num_out = mx - 3                                   # the last hop is partial, the last group ragged
    out_stride = num_out + (num_out % 2) + 6
    nplanes = nsrc * nx
    Xd, Md, xp, mp, Xv, Mv = _inputs(N, T, ldf, nx, nsrc, x_plane, m_stride, m_off, rng)
    Sbuf, sp, P = _product(Xv, Mv, ldf, 1 if m_off else 0)
    lib, stream = ctx.lib, _stream(ctx)

    def run(masked):
        ob = _sentinels(2 * SLACK + o_off + nplanes * out_stride)
        optr = ob.data_ptr() + 4 * (SLACK + o_off)
        if masked:
            r = lib.dcs_istft_masked(st.handle, xp, nx, x_plane, mp, nsrc, m_stride, T, ldf, optr, num_out, out_stride, stream)
        else:
            r = lib.dcs_istft(st.handle, sp, nplanes, T, ldf, T * ldf, optr, num_out, out_stride, stream)
        assert r == 0, (name, nx, nsrc, masked, r)
        torch.cuda.synchronize()
        return ob.cpu().numpy().view(np.uint32)
    n0 = ctx.launch_count()
    got = run(True)
    assert ctx.launch_count() == n0 + 1                 # one launch over all sources and channels
    assert np.array_equal(got, run(True)), ("two runs gave different bits", name, nx, nsrc)
    want = run(False)
    written = np.zeros(got.size, bool)
    for k in range(nplanes):
        written[SLACK + o_off + k * out_stride:SLACK + o_off + k * out_stride + num_out] = True
    assert (got[~written] == SENT).all(), ("fence / gap elements changed", name, nx, nsrc)
    assert np.isfinite(got[written].view(np.float32)).all(), ("NaN reached the output", name, nx, nsrc)
    diff = got != want
    assert not diff.any(), ("%d samples differ from dcs_istft(X * M)" % int(diff.sum()), name, nx, nsrc, int(np.argmax(diff)))
    assert np.abs(got[written].view(np.float32)).max() > 0
    if not oracle:
        return None
    w = st.window
    cI = so.c_inverse(N, path == "reg")
    worst = 0.0
    for k in range(nplanes):
        Sk = P[k, ..., 0].astype(np.float64) + 1j * P[k, ..., 1].astype(np.float64)
        y, bd = so.istft_ref(Sk, w, w, H, N, cI)
        a0 = SLACK + o_off + k * out_stride
        e = np.abs(got[a0:a0 + num_out].view(np.float32).astype(np.float64) - y[:num_out])
        r = so.ratio(e, bd[:num_out])
        worst = max(worst, float(r.max()))
        assert r.max() <= 1.0, ("error over the float64 bound", name, k, float(r.max()))
    return worst


@pytest.mark.parametrize("name", list(PATHS))
def test_same_bits_as_istft_of_the_product(ctx, name):
    for nx, nsrc in SHAPES:
        masked_case(ctx, name, nx, nsrc)


@pytest.mark.parametrize("name", ["reg_1024_256", "reg_2048_512", "smem_4096", "smem_forced_by_mask"])
def test_matches_float64_inverse_of_the_product(ctx, name):
    worst = masked_case(ctx, name, 2, 4, oracle=True)
    record("istft_masked:" + name, path=PATHS[name][2], worst_error_over_bound=worst)


def test_long_clip_many_groups(ctx):
    """3 channels x 4 sources over 1500 frames: several groups per plane on the register path, whose index decodes
    (channel, hop run, source)"""
    N, H, nx, nsrc, T = 2048, 512, 3, 4, 1500
    ldf = so.padded_bins(N)
    st = _plan(ctx, N, H)
    rng = np.random.default_rng(7)
    Xd, Md, xp, mp, Xv, Mv = _inputs(N, T, ldf, nx, nsrc, T * ldf, T * ldf, 0, rng)
    Sbuf, sp, _ = _product(Xv, Mv, ldf, 0)
    L = (T - 3) * H + 100
    a = torch.empty((nsrc * nx, L), dtype=torch.float32, device="cuda")
    b = torch.empty_like(a)
    assert ctx.lib.dcs_istft_masked(st.handle, xp, nx, T * ldf, mp, nsrc, T * ldf, T, ldf, a.data_ptr(), L, L, _stream(ctx)) == 0
    assert ctx.lib.dcs_istft(st.handle, sp, nsrc * nx, T, ldf, T * ldf, b.data_ptr(), L, L, _stream(ctx)) == 0
    torch.cuda.synchronize()
    assert torch.isfinite(a).all() and torch.equal(a.view(torch.int32), b.view(torch.int32))


def test_python_wrapper(ctx):
    st = _plan(ctx, 1024, 256)
    g = torch.Generator(device="cuda").manual_seed(3)
    X = torch.view_as_complex(torch.randn((2, 30, st.ldf, 2), device="cuda", generator=g))
    M = torch.rand((3, 30, st.ldf), device="cuda", generator=g)
    got = st.inverse_masked(X, M, num_out=5000)
    S = torch.view_as_complex((torch.view_as_real(X)[None] * M[:, None, :, :, None]).reshape(6, 30, st.ldf, 2).contiguous())
    assert got.shape == (6, 5000) and torch.equal(got.view(torch.int32), st.inverse(S, num_out=5000).view(torch.int32))
    with pytest.raises(ValueError):
        st.inverse_masked(X, M[:, :29])
    with pytest.raises(ValueError):
        st.inverse_masked(X, M.double())


def test_refusals_queue_nothing(ctx):
    N, H = 1024, 256
    st = _plan(ctx, N, H)
    F, ldf, T, L = N // 2 + 1, so.padded_bins(N), 12, 9 * H
    plane = T * ldf
    X = _sentinels(2 * (2 * plane + 2 * SLACK))
    M = _sentinels(2 * plane + 2 * SLACK)
    out = _sentinels(4 * L + 2 * SLACK)
    xp, mp, op = X.data_ptr() + 8 * SLACK, M.data_ptr() + 4 * SLACK, out.data_ptr() + 4 * SLACK
    lib, h, stream = ctx.lib, st.handle, _stream(ctx)

    def call(plan=h, x=xp, nx=2, x_plane=plane, m=mp, nsrc=2, m_stride=plane, T_=T, ldf_=ldf, o=op, n=L, o_stride=L):
        return lib.dcs_istft_masked(plan, x, nx, x_plane, m, nsrc, m_stride, T_, ldf_, o, n, o_stride, stream)
    n0 = ctx.launch_count()
    bad = {
        "NULL plan": call(plan=None), "NULL X": call(x=None), "NULL M": call(m=None), "NULL out": call(o=None),
        "no frames": call(T_=0), "nx 0": call(nx=0), "nx 17": call(nx=17), "nsrc 0": call(nsrc=0),
        "ldf < F": call(ldf_=F - 1), "negative x_plane": call(nx=1, x_plane=-1), "negative m_stride": call(nsrc=1, m_stride=-1),
        "negative out_stride": call(o_stride=-1), "channels share rows": call(x_plane=plane - 1),
        "masks share rows": call(m_stride=plane - 1), "planes share samples": call(o_stride=L - 1),
        "num_out too long": call(nx=1, nsrc=1, n=(T - 1) * H + N // 2 + 1, o_stride=1 << 20),
        "X not 8-byte aligned": call(x=xp + 4), "M not 4-byte aligned": call(m=mp + 2),
    }
    torch.cuda.synchronize()
    assert all(r == -1 for r in bad.values()), bad
    assert ctx.launch_count() == n0
    assert b"d_M not 4-byte aligned" in lib.dcs_last_error()      # the message names the argument
    for b in (X, M, out):
        assert (b.cpu().numpy().view(np.uint32) == SENT).all()
