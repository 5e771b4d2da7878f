// sconv.cu -- kernels for the strided-conv1 networks (iKala, Bach10, score-informed Bach10):
//   * max-pool (1,4) over frequency with Theano's tie bookkeeping
//     (examples/ikala/separate_ikala.py:176; InverseLayer(pool) :183,188 routes the value to EVERY
//     position equal to the window maximum -- MaxPoolGrad semantics)
//   * K3s, exact-fp32 FFMA twin of sconv_tc.cu (the DCS_DEBUG_SIMT_GEMM=1 cross-check):
//     InverseLayer(pool) + InverseLayer(conv1) (transposed strided convolution over
//     frequency) + ConcatLayer + bias + ReLU + soft ratio mask + patch cross-fade + phase,
//     fused (separate_ikala.py:183-217, bach10/separate_bach10.py:207-266, :139-169 of each).
//
// Transposed strided conv as STRIDE interleaved FIR filters: output bin b = STRIDE*m + r gets
//   Y[b] = sum_{dd < ND, f < 30} Gu[m - dd][f] * W1[f][KW-1 - r - STRIDE*dd]      (ND = ceil(KW/STRIDE))
// One thread owns one m (STRIDE consecutive bins) so a staged activation value feeds STRIDE FMAs
// per source; the decoder rows of the <= 6 patches covering a frame are staged in shared memory
// one patch at a time (pitch 33: consecutive m -> consecutive banks).  Like the DSD100 kernels,
// no per-patch output tensor exists in HBM.
#include "common.cuh"

namespace dcs {

__global__ void pool4_kernel(const float* __restrict__ H1, float* __restrict__ Hp, uint8_t* __restrict__ tie,
                             int64_t rows, int J, int WP) {
  // H1 [rows][J][32] -> Hp [rows][WP][32], tie [rows][WP][32] (bit r: element 4*jp+r equals the max)
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t total = rows * WP * 32;
  if (i >= total) return;
  const int c = (int)(i & 31);
  const int64_t rj = i >> 5;
  const int jp = (int)(rj % WP);
  const int64_t t = rj / WP;
  const float* src = H1 + (t * J + 4 * jp) * 32 + c;
  const float a0 = src[0], a1 = src[32], a2 = src[64], a3 = src[96];
  const float mx = fmaxf(fmaxf(a0, a1), fmaxf(a2, a3));
  Hp[i] = mx;
  tie[i] = (uint8_t)((a0 == mx) | ((a1 == mx) << 1) | ((a2 == mx) << 2) | ((a3 == mx) << 3));
}

constexpr int SC_TILE = 128;   // m values (threads) per CTA

// CHUNK: as in sconv_mask_tc_kernel (G from patch a.p_base, frames [a.t0, a.t1)); MASKS: the blended masks to M
// (source s at M + s * src_stride), X and S untouched
template <int STRIDE, int ND, int NSRC, int NDEC, int RULE, int POOL, int NW, bool CHUNK = false, bool MASKS = false>
__global__ void __launch_bounds__(SC_TILE)
sconv_mask_kernel(const SconvMaskArgs a, float* __restrict__ M) {
  constexpr int JT = SC_TILE + ND - 1;  // staged activation positions per tile
  extern __shared__ __align__(16) float sm[];
  float* gs = sm;                                   // [NDEC][JT][33]
  float4* ws = reinterpret_cast<float4*>(sm + NDEC * JT * 33 + (4 - (NDEC * JT * 33) % 4) % 4);  // [NW][ND][32]
  const int tid = threadIdx.x;
  // frames on gridDim.x (2^31-1 blocks: any clip length), bin tiles on gridDim.y (a handful)
  const int m0 = blockIdx.y * SC_TILE, m = m0 + tid;
  const int t = (CHUNK ? a.t0 : 0) + blockIdx.x;
  const int p_base = CHUNK ? a.p_base : 0;
  const int step = a.tc - a.overlap;
  // weights: w[dd][f][r] = W1[f][KW-1 - r - STRIDE*dd] (0 where the tap index is negative)
  for (int i = tid; i < NW * ND * 32; i += SC_TILE) ws[i] = reinterpret_cast<const float4*>(a.W)[i];
  int k_hi = t / step;
  if (k_hi > a.P - 1) k_hi = a.P - 1;
  int k_lo = t - a.tc + 1;
  k_lo = k_lo > 0 ? (k_lo + step - 1) / step : 0;
  const float inv_ov1 = a.overlap > 1 ? 1.0f / (float)(a.overlap - 1) : 0.f;
  float macc[NSRC][STRIDE];
#pragma unroll
  for (int o = 0; o < NSRC; ++o)
#pragma unroll
    for (int r = 0; r < STRIDE; ++r) macc[o][r] = 0.f;

  for (int k = k_lo; k <= k_hi; ++k) {
    const int p = t - k * step;
    __syncthreads();
    // stage activations of patch k, frame-in-patch p: positions j in [m0-(ND-1), m0+SC_TILE)
    for (int idx = tid; idx < NDEC * JT * 32; idx += SC_TILE) {
      const int f = idx & 31, jl = (idx >> 5) % JT, d = (idx >> 5) / JT;
      const int j = m0 - (ND - 1) + jl;
      float v = 0.f;
      if (POOL == 0) {
        if (j >= 0 && j < a.J) v = __ldg(a.G + ((((int64_t)(k - p_base) * NDEC + d) * a.tc + p) * a.J + j) * 32 + f);
      } else {
        const int jp = j / POOL;
        if (j >= 0 && jp < a.WP) {
          const uint8_t bits = a.tie[((int64_t)t * a.WP + jp) * 32 + f];
          if ((bits >> (j - jp * POOL)) & 1) v = __ldg(a.G + ((((int64_t)(k - p_base) * NDEC + d) * a.tc + p) * a.WP + jp) * 32 + f);
        }
      }
      gs[(d * JT + jl) * 33 + f] = v;
    }
    __syncthreads();
    float acc[NSRC][STRIDE];
#pragma unroll
    for (int o = 0; o < NSRC; ++o)
#pragma unroll
      for (int r = 0; r < STRIDE; ++r) acc[o][r] = 0.f;
#pragma unroll 1
    for (int dd = 0; dd < ND; ++dd) {
      const float* grow = gs + (tid + ND - 1 - dd) * 33;
#pragma unroll 6
      for (int f = 0; f < 30; ++f) {
        // NW == 1: one filter bank, one decoder per source (iKala, Bach10);
        // NW == NSRC, NDEC == 1: one decoder, one filter bank per source = per input channel
        // of the tied conv1 (score-informed Bach10, trainCNNrwc.py:189,248-251)
        const float4 w0 = ws[dd * 32 + f];
#pragma unroll
        for (int o = 0; o < NSRC; ++o) {
          const float4 w = NW == 1 ? w0 : ws[(o * ND + dd) * 32 + f];
          const float wr[4] = {w.x, w.y, w.z, w.w};
          const float g = grow[(NDEC == 1 ? 0 : o) * JT * 33 + f];
#pragma unroll
          for (int r = 0; r < STRIDE; ++r) acc[o][r] = fmaf(g, wr[r], acc[o][r]);
        }
      }
    }
    // bias + ReLU + ratio mask across the sources + sequential cross-fade
    const float up = k == k_lo ? 1.f : (float)p * inv_ov1;
    const float down = k == k_lo ? 0.f : (float)(a.overlap - 1 - p) * inv_ov1;
#pragma unroll
    for (int r = 0; r < STRIDE; ++r) {
      float pv[NSRC], tot = 0.f;
#pragma unroll
      for (int o = 0; o < NSRC; ++o) {
        pv[o] = fmaxf(acc[o][r] + a.bout[o], 0.f);
        tot += pv[o];
      }
      const bool pos = tot > MASK_TOT_MIN;
      const float rr = pos ? __fdividef(up, tot) : 0.f;
      const float q = (pos || RULE == 1) ? 0.f : up / (float)NSRC;
#pragma unroll
      for (int o = 0; o < NSRC; ++o) macc[o][r] = fmaf(down, macc[o][r], fmaf(pv[o], rr, q));
    }
  }
#pragma unroll
  for (int r = 0; r < STRIDE; ++r) {
    const int b = STRIDE * m + r;
    if (MASKS && b < a.F) {
      const int64_t o = (int64_t)t * a.ldf + b;
#pragma unroll
      for (int s = 0; s < NSRC; ++s) M[o + s * a.src_stride] = macc[s][r];
    } else if (b < a.F) {
      const int64_t o = (int64_t)t * a.ldf + b;
      const float2 x = a.X[o];
#pragma unroll
      for (int s = 0; s < NSRC; ++s) a.S[o + s * a.src_stride] = make_float2(macc[s][r] * x.x, macc[s][r] * x.y);
    }
  }
}

// score-informed input channels: in_ch[t][b] = filter_ch[t][b] * mag[t][b]   (trainCNNrwc.py:388-391)
__global__ void channel_mul_kernel(const float* __restrict__ mag, const float* __restrict__ filt, float* __restrict__ out,
                                   int64_t plane, int nch) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= plane) return;
  const float m = mag[i];
  for (int c = 0; c < nch; ++c) out[c * plane + i] = filt[c * plane + i] * m;
}

int launch_channel_mul(dcs_ctx* ctx, const float* mag, const float* filt, float* out, int64_t plane, int nch, cudaStream_t st) {
  if (plane <= 0) return DCS_OK;
  channel_mul_kernel<<<(unsigned)ceil_div64(plane, 256), 256, 0, st>>>(mag, filt, out, plane, nch);
  DCS_CHECK_LAUNCH();
  ctx->launches++;
  return DCS_OK;
}

int launch_pool4(dcs_ctx* ctx, const float* H1, float* Hp, uint8_t* tie, int64_t rows, int J, int WP, cudaStream_t st) {
  const int64_t total = rows * WP * 32;
  if (total <= 0) return DCS_OK;
  pool4_kernel<<<(unsigned)ceil_div64(total, 256), 256, 0, st>>>(H1, Hp, tie, rows, J, WP);
  DCS_CHECK_LAUNCH();
  ctx->launches++;
  return DCS_OK;
}

template <int STRIDE, int ND, int NSRC, int NDEC, int RULE, int POOL, int NW, bool CHUNK = false>
static int launch_sconv_t(dcs_ctx* ctx, const SconvMaskArgs& a, float* M, cudaStream_t st) {
  constexpr int JT = SC_TILE + ND - 1;
  const size_t smem = (size_t)(NDEC * JT * 33 + 4) * sizeof(float) + NW * ND * 32 * sizeof(float4);
  auto kern = M ? sconv_mask_kernel<STRIDE, ND, NSRC, NDEC, RULE, POOL, NW, CHUNK, true>
                : sconv_mask_kernel<STRIDE, ND, NSRC, NDEC, RULE, POOL, NW, CHUNK, false>;
  DCS_TRY(ensure_smem_attr(kern, (int)smem));
  const int mtot = (a.F + STRIDE - 1) / STRIDE;
  dim3 grid((unsigned)(a.t1 - a.t0), (unsigned)ceil_div64(mtot, SC_TILE));
  kern<<<grid, SC_TILE, smem, st>>>(a, M);
  DCS_CHECK_LAUNCH();
  ctx->launches++;
  return DCS_OK;
}

int launch_sconv_mask(dcs_ctx* ctx, const SconvMaskArgs& a, cudaStream_t st, float* M) {
  if (a.T <= 0 || a.t1 <= a.t0) return DCS_OK;
  const int step = a.tc - a.overlap;
  DCS_REQUIRE(step > 0 && (a.tc + step - 1) / step <= 64, "sconv_mask: bad time_context/overlap");
  DCS_REQUIRE(a.t0 >= 0 && a.t1 <= a.T, "sconv_mask: frame range [%d, %d) outside [0, %d)", a.t0, a.t1, a.T);
  if (a.arch == DCS_ARCH_BACH10) return launch_sconv_t<4, 8, 4, 4, 1, 0, 1>(ctx, a, M, st);
  if (a.arch == DCS_ARCH_BACH10_SCORE) return launch_sconv_t<4, 8, 4, 1, 1, 0, 4>(ctx, a, M, st);
  if (a.arch == DCS_ARCH_BACH10_SCORE_1X1) return launch_sconv_t<2, 3, 4, 1, 1, 0, 4, true>(ctx, a, M, st);
  if (a.arch == DCS_ARCH_IKALA) return launch_sconv_t<3, 10, 2, 2, 0, 4, 1>(ctx, a, M, st);
  if (a.arch == DCS_ARCH_IKALA_NOPOOL) return launch_sconv_t<3, 10, 2, 2, 0, 0, 1>(ctx, a, M, st);
  DCS_REQUIRE(false, "sconv_mask: architecture %d not supported", a.arch);
}

}  // namespace dcs
