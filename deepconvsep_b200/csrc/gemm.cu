// gemm.cu -- fp32 GEMM with strided / overlapping operand addressing, C = act(A*B + bias).
//
// The encoder/decoder of build_ca() (separate_dsd.py:195-234) is expressed as GEMMs whose A
// operand is a *view* of an activation buffer: convolution rows overlap (row stride < row
// length), K may be split in segments (one per kernel tap), and C may be scattered into a
// zero-padded buffer for the following transposed convolution.  No im2col copy is ever
// materialised in HBM.
//
// This is the exact-fp32 FFMA path (the soft mask amplifies operand rounding ~25x, SURVEY.md
// App. C: plain TF32 gives 1e-2 relative error).  Tile 128x64x16, 256 threads, 8x4 outputs per
// thread, register-prefetched global loads, A tile transposed in shared memory.
#include "common.cuh"

namespace dcs {

constexpr int BM = 128, BN = 64, BK = 16, TM = 8, TN = 4, NTHREADS = 256;

__global__ void __launch_bounds__(NTHREADS)
gemm_f32_kernel(const GemmDesc d) {
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN];
  const int tid = threadIdx.x;
  const int tx = tid % 16, ty = tid / 16;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;

  // A loads: this thread always loads column (tid % 16) of rows (tid / 16) + 16 r
  const int ak = tid % BK;
  int64_t a_row_off[8];
  bool a_row_ok[8];
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    const int m = m0 + tid / BK + 16 * r;
    a_row_ok[r] = (m < d.M) && (m < d.a_valid_rows);
    const int mc = m < d.M ? m : 0;
    a_row_off[r] = (int64_t)(mc / d.m_inner) * d.a_so + (int64_t)((mc % d.m_inner) / d.m_inner2) * d.a_si + (int64_t)(mc % d.m_inner2) * d.a_s2;
  }
  // B loads: column (tid % 64), rows (tid / 64) + 4 r
  const int bn = n0 + tid % BN;
  const bool bn_ok = bn < d.N;

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  float ra[8], rb[4];
  auto gload = [&](int k0) {
    const int k = k0 + ak;
    const bool kok = k < d.K;
    const int kc = kok ? k : 0;
    const int64_t koff = (int64_t)(kc / d.k_seg) * d.k_ss + (kc % d.k_seg);
#pragma unroll
    for (int r = 0; r < 8; ++r) ra[r] = (kok && a_row_ok[r]) ? __ldg(d.A + a_row_off[r] + koff) : 0.f;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int kb = k0 + tid / BN + 4 * r;
      rb[r] = (bn_ok && kb < d.K) ? __ldg(d.B + (int64_t)kb * d.ldb + bn) : 0.f;
    }
  };
  gload(0);
  for (int k0 = 0; k0 < d.K; k0 += BK) {
#pragma unroll
    for (int r = 0; r < 8; ++r) As[ak][tid / BK + 16 * r] = ra[r];
#pragma unroll
    for (int r = 0; r < 4; ++r) Bs[tid / BN + 4 * r][tid % BN] = rb[r];
    __syncthreads();
    if (k0 + BK < d.K) gload(k0 + BK);
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[kk][ty * TM]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[kk][ty * TM + 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[kk][tx * TN]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float bb[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int m = m0 + ty * TM + i;
    if (m >= d.M) continue;
    const int64_t roff = gemm_c_row_offset(d, m);
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int n = n0 + tx * TN + j;
      if (n >= d.N) continue;
      float v = acc[i][j];
      if (d.bias) v += __ldg(d.bias + n);
      if (d.relu) v = fmaxf(v, 0.f);
      d.C[roff + (int64_t)(n / d.n_seg) * d.n_ss + (n % d.n_seg)] = v;
    }
  }
}

GemmDesc gemm_plain(const float* A, int64_t lda, const float* B, int64_t ldb, const float* bias, float* C,
                    int64_t ldc, int M, int N, int K, int relu) {
  GemmDesc d{};
  d.A = A; d.B = B; d.bias = bias; d.C = C;
  d.M = M; d.N = N; d.K = K;
  d.a_valid_rows = M;
  d.m_inner = 1; d.a_so = lda; d.a_si = 0; d.m_inner2 = 1; d.a_s2 = 0;
  d.k_seg = K > 0 ? K : 1; d.k_ss = 0;
  d.ldb = ldb;
  d.cm_inner = 1; d.c_so = ldc; d.c_si = 0; d.cm_inner2 = 1; d.c_s2 = 0;
  d.n_seg = N > 0 ? N : 1; d.n_ss = 0; d.c_col0 = 0;
  d.relu = relu;
  d.kc_rows = 0; d.kc_unit = d.kc_pad = d.kc_n = d.kc_taps = 0;
  return d;
}

int launch_gemm(dcs_ctx* ctx, const GemmDesc& d, cudaStream_t st) {
  if (d.M <= 0 || d.N <= 0) return DCS_OK;
  DCS_REQUIRE(d.K > 0 && d.m_inner > 0 && d.m_inner2 > 0 && d.k_seg > 0 && d.cm_inner > 0 && d.cm_inner2 > 0 && d.n_seg > 0, "bad GEMM descriptor");
  DCS_REQUIRE(gemm_c_view_ok(d), "GEMM: negative C stride or column offset");
  dim3 grid((unsigned)ceil_div64(d.N, BN), (unsigned)ceil_div64(d.M, BM));
  DCS_REQUIRE(grid.y <= 65535u * 16u, "GEMM M=%d too large", d.M);
  if (grid.y > 65535u) {
    // split M (keeps the kernel simple; only enormous clips get here)
    GemmDesc lo = d, hi = d;
    const int half = (int)((int64_t)(grid.y / 2) * BM);
    DCS_REQUIRE(d.m_inner == 1 && d.cm_inner == 1 && d.m_inner2 == 1 && d.cm_inner2 == 1, "GEMM M=%d too large for segmented rows", d.M);
    lo.M = half; if (lo.a_valid_rows > half) lo.a_valid_rows = half;
    hi.M = d.M - half; hi.A = d.A + (int64_t)half * d.a_so; hi.C = d.C + (int64_t)half * d.c_so;
    hi.a_valid_rows = d.a_valid_rows - half;
    DCS_TRY(launch_gemm(ctx, lo, st));
    return launch_gemm(ctx, hi, st);
  }
  gemm_f32_kernel<<<grid, NTHREADS, 0, st>>>(d);
  DCS_CHECK_LAUNCH();
  ctx->launches++;
  return DCS_OK;
}

}  // namespace dcs
