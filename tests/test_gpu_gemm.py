"""GPU parity of the GEMM building block: the wgmma 3xTF32 kernel (engine 1) and the FFMA
kernel (engine 0) against a float64 matmul.  Tolerance: 2e-6 relative L2 (fp32 accumulate)."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from deepconvsep_b200.engine import Context
    return Context(0)


@pytest.mark.parametrize("engine", [1, 0])
@pytest.mark.parametrize("M,N,K,lda_extra", [(128, 64, 32, 0), (1, 1, 1, 0), (300, 50, 750, 0), (257, 128, 800, 4),
                                             (1000, 150, 129, 3), (130, 2400, 128, 0), (4096, 50, 1025, 7),
                                             # N <= 32 (the BN = 32 kernels of the 30-channel convolutions): A vector
                                             # widths 2 / 1 with split K over 3 / 4 slices, a one-element K tail, width 4
                                             (300, 30, 780, 2), (1000, 32, 1040, 1), (129, 17, 33, 0), (257, 30, 96, 0)])
def test_gemm_matches_float64(ctx, engine, M, N, K, lda_extra):
    rng = np.random.default_rng(M * 7 + N * 3 + K)
    A = rng.standard_normal((M, K + lda_extra)).astype(np.float32)
    B = (rng.standard_normal((K, N)) / np.sqrt(K)).astype(np.float32)
    bias = rng.standard_normal(N).astype(np.float32) * 0.1
    Ad = torch.tensor(A, device="cuda")[:, :K]
    for relu in (False, True):
        C = ctx.gemm(Ad, B, bias, relu=relu, engine=engine).cpu().numpy().astype(np.float64)
        ref = A[:, :K].astype(np.float64) @ B.astype(np.float64) + bias
        if relu:
            ref = np.maximum(ref, 0)
        err = np.linalg.norm(C - ref) / np.linalg.norm(ref)
        assert err < 2e-6, (engine, relu, err)
        assert np.abs(C - ref).max() < 2e-5 * max(1.0, np.abs(ref).max())


@pytest.mark.parametrize("pitch", [50, 52])
def test_tensor_core_gemm_overlapping_rows(ctx, pitch):
    """A rows that overlap (row stride < K): the convolution-as-GEMM view (no im2col copy).
    pitch 52 keeps 16-byte aligned rows (vector loads), pitch 50 only 8-byte ones."""
    rng = np.random.default_rng(1)
    buf = rng.standard_normal(pitch * 400).astype(np.float32)
    K, M, N = 15 * pitch, 300, 50
    d = torch.tensor(buf, device="cuda")
    Ad = torch.as_strided(d, (M, K), (pitch, 1))
    B = (rng.standard_normal((K, N)) / 27.0).astype(np.float32)
    ref = np.lib.stride_tricks.as_strided(buf, (M, K), (4 * pitch, 4)).astype(np.float64) @ B.astype(np.float64)
    for engine in (1, 0):
        C = ctx.gemm(Ad, B, None, engine=engine).cpu().numpy().astype(np.float64)
        assert np.linalg.norm(C - ref) / np.linalg.norm(ref) < 2e-6

