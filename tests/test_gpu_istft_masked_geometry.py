"""Launch geometry of the masked register inverse STFT (istft_masked_reg_kernel, 12 warps a CTA): source counts whose
quads of min(nsrc, groups) groups fill a CTA differently, and clips shorter than one CTA's quads.

At N = 2048 a CTA has 12 groups, at N = 1024 24.  nsrc = 3 and 6 give quads of 3 and 6 groups; nsrc = 5 and 8 leave
groups of a CTA idle (they walk the frames on zeros and store nothing).  Clips of 3, 41 and 600 frames give one partial
CTA up to several CTAs per plane.  On every register path (N 1024 / 2048, hop 256 / 512) and nx 1 and 2:
- the output equals dcs_istft on S = X * M formed by torch in fp32, bit for bit;
- two runs give the same bits;
- the sentinels around and between the output planes are untouched."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

SENT = np.uint32(0x7FC5A5A5)      # quiet NaN with a payload no kernel produces
SLACK = 64
PATHS = [(1024, 256), (1024, 512), (2048, 256), (2048, 512)]


@pytest.fixture(scope="module")
def ctx():
    from deepconvsep_b200.engine import Context
    return Context(0)


def _sentinels(n):
    return torch.from_numpy(np.full(n, SENT, np.uint32).view(np.float32)).cuda()


def _case(ctx, st, N, H, nx, nsrc, T, seed):
    from deepconvsep_b200.engine import _stream_ptr
    F, ldf = N // 2 + 1, st.ldf
    g = torch.Generator(device="cuda").manual_seed(seed)
    X = torch.full((nx, T, ldf, 2), float("nan"), device="cuda")
    X[:, :, :F] = torch.randn((nx, T, F, 2), device="cuda", generator=g) * 10.0
    M = torch.full((nsrc, T, ldf), float("nan"), device="cuda")
    M[:, :, :F] = torch.rand((nsrc, T, F), device="cuda", generator=g)
    M[:, :, ::7] = 0.0
    M[:, :, 3:F:11] = 1.0
    X[:, :, 0, 1] = float("nan")                     # Im of DC and Nyquist: ignored
    X[:, :, F - 1, 1] = float("nan")
    S = torch.full((nsrc * nx, T, ldf, 2), float("nan"), device="cuda")
    S[:, :, :F] = (X[None, :, :, :F] * M[:, None, :, :F, None]).reshape(nsrc * nx, T, F, 2)
    num_out = (T - 1) * H + N // 2 - 3
    out_stride = num_out + (num_out % 2) + 6
    nplanes = nsrc * nx
    stream = _stream_ptr(None, ctx.device)

    def run(masked):
        ob = _sentinels(2 * SLACK + nplanes * out_stride)
        op = ob.data_ptr() + 4 * SLACK
        if masked:
            r = ctx.lib.dcs_istft_masked(st.handle, X.data_ptr(), nx, T * ldf, M.data_ptr(), nsrc, T * ldf, T, ldf, op,
                                         num_out, out_stride, stream)
        else:
            r = ctx.lib.dcs_istft(st.handle, S.data_ptr(), nplanes, T, ldf, T * ldf, op, num_out, out_stride, stream)
        assert r == 0, (N, H, nx, nsrc, T, masked, r)
        torch.cuda.synchronize()
        return ob.cpu().numpy().view(np.uint32)
    got = run(True)
    assert np.array_equal(got, run(True)), ("two runs gave different bits", N, H, nx, nsrc, T)
    want = run(False)
    written = np.zeros(got.size, bool)
    for k in range(nplanes):
        written[SLACK + k * out_stride:SLACK + k * out_stride + num_out] = True
    assert (got[~written] == SENT).all(), ("fence / gap elements changed", N, H, nx, nsrc, T)
    assert np.isfinite(got[written].view(np.float32)).all(), ("NaN reached the output", N, H, nx, nsrc, T)
    diff = got != want
    assert not diff.any(), ("%d samples differ from dcs_istft(X * M)" % int(diff.sum()), N, H, nx, nsrc, T)


@pytest.mark.parametrize("N,H", PATHS)
@pytest.mark.parametrize("nsrc", [3, 5, 6, 8])
def test_quad_shapes_same_bits_as_istft_of_the_product(ctx, N, H, nsrc):
    from deepconvsep_b200.engine import Stft
    st = Stft(ctx, N, H, "hanning")
    try:
        for nx in (1, 2):
            for T in (3, 41, 600):
                _case(ctx, st, N, H, nx, nsrc, T, seed=N + H + 10 * nsrc + 100 * nx + T)
    finally:
        st.close()
