// bsseval.cu -- the O(L) part of BSS-Eval 3.0 `bss_eval_sources` on the device, in float64:
// the auto-/cross-correlation lags the least-squares projection is built from
// (evaluation/bss_eval/bss_eval_sources.m:120-145 computes them with length-2^nextpow2(L+511)
// FFTs; only lags |m| < flen = 512 are ever used, so they are accumulated directly):
//     out[p][li] = sum_t a_p[t + li - (flen-1)] * b_p[t],      li = 0 .. 2*flen-2
// for a list of signal pairs.  The Gram matrix of the delayed sources, the right-hand sides, the
// dense solve and the SDR / SIR / SAR ratios are O(flen^2 .. flen^3) host work
// (deepconvsep_b200/evaluation.py).
//
// One CTA = one pair x one span of 32 x 2048 samples.  Per 2048-sample step the b samples and the
// a window (2048 + 1023 samples) are staged in shared memory as doubles; thread i owns the four
// consecutive lags 4i..4i+3 and slides a 4-register window over a, so one step costs one
// broadcast load, one window load and four DFMAs.  The window is stored by residue mod 4
// (aw[r][q] = a[.. + 4q + r]) so that the 32 lanes of a warp read 32 consecutive doubles.
// Spans are summed in a fixed order by a second kernel: run-to-run deterministic.
#include "common.cuh"

namespace dcs {

constexpr int XC_THREADS = 256;
constexpr int XC_LAGS = 4 * XC_THREADS;      // 1024 >= 2*512-1
constexpr int XC_SUB = 2048;                 // samples per shared-memory step
constexpr int XC_SPAN = 32;                  // steps per CTA
constexpr int XC_AQ = (XC_SUB + XC_LAGS) / 4;

__global__ void __launch_bounds__(XC_THREADS)
xcorr_partial_kernel(const float* const* __restrict__ A, const float* const* __restrict__ B, int64_t L, int flen,
                     double* __restrict__ partial, int nspans) {
  __shared__ double aw[4][XC_AQ + 1];
  __shared__ double bw[XC_SUB];
  const int tid = threadIdx.x, pair = blockIdx.y, span = blockIdx.x;
  const float* __restrict__ a = A[pair];
  const float* __restrict__ b = B[pair];
  double acc0 = 0.0, acc1 = 0.0, acc2 = 0.0, acc3 = 0.0;
  const int64_t tbeg = (int64_t)span * XC_SUB * XC_SPAN;
  for (int sc = 0; sc < XC_SPAN; ++sc) {
    const int64_t t0 = tbeg + (int64_t)sc * XC_SUB;
    if (t0 >= L) break;   // CTA-uniform
    __syncthreads();
    for (int i = tid; i < XC_SUB; i += XC_THREADS) {
      const int64_t t = t0 + i;
      bw[i] = t < L ? (double)__ldg(b + t) : 0.0;
    }
    // window element x <-> a[t0 - (flen-1) + x], x = 0 .. XC_SUB + XC_LAGS - 1
    for (int x = tid; x < XC_SUB + XC_LAGS; x += XC_THREADS) {
      const int64_t t = t0 - (flen - 1) + x;
      aw[x & 3][x >> 2] = (t >= 0 && t < L) ? (double)__ldg(a + t) : 0.0;
    }
    __syncthreads();
    // lag li = 4*tid + j reads window element i + li at step i
    double w0 = aw[0][tid], w1 = aw[1][tid], w2 = aw[2][tid];
#pragma unroll 4
    for (int i = 0; i < XC_SUB; ++i) {
      const int x = i + 3;                              // window element (4*tid + x), residue x & 3
      const double w3 = aw[x & 3][tid + (x >> 2)];
      const double bv = bw[i];
      acc0 = fma(w0, bv, acc0);
      acc1 = fma(w1, bv, acc1);
      acc2 = fma(w2, bv, acc2);
      acc3 = fma(w3, bv, acc3);
      w0 = w1; w1 = w2; w2 = w3;
    }
  }
  double* dst = partial + ((int64_t)pair * nspans + span) * XC_LAGS + 4 * tid;
  dst[0] = acc0; dst[1] = acc1; dst[2] = acc2; dst[3] = acc3;
}

__global__ void xcorr_reduce_kernel(const double* __restrict__ partial, int nspans, int nlags, double* __restrict__ out) {
  const int li = blockIdx.x * blockDim.x + threadIdx.x, pair = blockIdx.y;
  if (li >= nlags) return;
  double s = 0.0;
  for (int sp = 0; sp < nspans; ++sp) s += partial[((int64_t)pair * nspans + sp) * XC_LAGS + li];   // fixed order
  out[(int64_t)pair * nlags + li] = s;
}

int launch_xcorr_lags(dcs_ctx* ctx, const float* const* h_a, const float* const* h_b, int npairs, int64_t L, int flen,
                      double* h_out, cudaStream_t st) {
  DCS_REQUIRE(npairs > 0 && npairs <= 65535 && L > 0, "xcorr: bad pair count / length");
  DCS_REQUIRE(flen >= 1 && 2 * flen - 1 <= XC_LAGS, "xcorr: flen %d out of range (1..%d)", flen, XC_LAGS / 2);
  const int nlags = 2 * flen - 1;
  const int64_t nspans64 = ceil_div64(L, (int64_t)XC_SUB * XC_SPAN);
  DCS_REQUIRE(nspans64 <= 0x7fffffff, "xcorr: signal too long");
  const int nspans = (int)nspans64;
  const size_t ptr_bytes = (size_t)npairs * sizeof(float*);
  DCS_TRY(ctx->net[NET_XC_PTRS].ensure(2 * ptr_bytes + (size_t)npairs * nlags * sizeof(double) + 16, st));
  DCS_TRY(ctx->net[NET_XC_PARTIAL].ensure((size_t)npairs * nspans * XC_LAGS * sizeof(double), st));
  uint8_t* base = ctx->net[NET_XC_PTRS].as<uint8_t>();
  const float** dA = reinterpret_cast<const float**>(base);
  const float** dB = reinterpret_cast<const float**>(base + ptr_bytes);
  double* d_out = reinterpret_cast<double*>(base + (2 * ptr_bytes + 15) / 16 * 16);
  DCS_CUDA(cudaMemcpyAsync(dA, h_a, ptr_bytes, cudaMemcpyHostToDevice, st));
  DCS_CUDA(cudaMemcpyAsync(dB, h_b, ptr_bytes, cudaMemcpyHostToDevice, st));
  double* partial = ctx->net[NET_XC_PARTIAL].as<double>();
  xcorr_partial_kernel<<<dim3((unsigned)nspans, (unsigned)npairs), XC_THREADS, 0, st>>>(dA, dB, L, flen, partial, nspans);
  DCS_CHECK_LAUNCH();
  ctx->launches++;
  xcorr_reduce_kernel<<<dim3((unsigned)ceil_div64(nlags, 256), (unsigned)npairs), 256, 0, st>>>(partial, nspans, nlags, d_out);
  DCS_CHECK_LAUNCH();
  ctx->launches++;
  DCS_CUDA(cudaMemcpyAsync(h_out, d_out, (size_t)npairs * nlags * sizeof(double), cudaMemcpyDeviceToHost, st));
  DCS_CUDA(cudaStreamSynchronize(st));
  return DCS_OK;
}

}  // namespace dcs
