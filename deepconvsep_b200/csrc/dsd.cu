// dsd.cu -- K3 for the DSD100 / hiphopss network, exact-fp32 FFMA version: InverseLayer(conv1) +
// ConcatLayer + output bias + ReLU + soft ratio mask + patch cross-fade + mixture-phase re-apply, fused.
// The product path for the reference settings is the wgmma kernel in dsd_tc.cu; this one serves
// (time_context, overlap) settings with more than 6 patches per frame and, under DCS_DEBUG_SIMT_GEMM=1,
// the cross-check of the mask stage (every other layer stays on the tensor cores).
//
// Reference: examples/dsd100/separate_dsd.py:212-234 (l_inverse4x, l_merge, l_out), :258-271 (masks),
// :139-169 (overlapadd_multi), :304 + :36-41 (compute_inverse).  Because conv1 spans the whole
// frequency axis, the transposed conv1 of decoder d at (patch k, frame-in-patch p) is the GEMV
// Y[b] = sum_c G[k][d][p][c] * W1[c,0,0,F-1-b]; every patch covering mixture frame t sees the
// same input frame, each patch output is mask*input and the cross-fade is linear, so the
// blended estimate is (sum_k omega_k mask_{s,k}) * X[t]  (SURVEY.md App. A.1/A.5).  No
// per-patch [P,4,30,F] tensor ever exists in HBM: this kernel reads the tiny G rows and X and
// writes the four masked complex spectra once.
//
// One thread owns one frequency bin (its 50 conv1 weights live in registers) and walks
// `frames_per_cta` frames; the G rows of the <= 6 patches covering a frame are staged in
// shared memory and broadcast.  Bins 0..F-2 map onto 256-thread tiles (F-1 is a power of two);
// the Nyquist bin is handled by lane 0 of an extra warp in tile 0.
#include "common.cuh"

namespace dcs {

constexpr int MASK_TILE = 256;
constexpr int MASK_THREADS = MASK_TILE + 32;
constexpr int MASK_MAXP = 6;

// MASKS: the blended masks themselves to M (source s at M + s * src_stride); X and S are not touched
template <int C1, int NDEC, bool MASKS = false>
__global__ void __launch_bounds__(MASK_THREADS)
dsd_mask_kernel(const DsdMaskArgs a, float* __restrict__ M, int frames_per_cta) {
  constexpr int PITCH = (C1 + 3) / 4 * 4;
  __shared__ __align__(16) float gs[MASK_MAXP][NDEC][PITCH];
  const int tid = threadIdx.x;
  int b = -1;
  if (tid < MASK_TILE) {
    const int bb = blockIdx.y * MASK_TILE + tid;
    if (bb < a.F - 1) b = bb;
  } else if (tid == MASK_TILE && blockIdx.y == 0) {
    b = a.F - 1;
  }
  const bool bok = b >= 0;
  float w[C1];
#pragma unroll
  for (int c = 0; c < C1; ++c) w[c] = bok ? __ldg(a.W1t + (int64_t)c * a.ldw + b) : 0.f;
  const float bo0 = __ldg(a.bout + 0), bo1 = __ldg(a.bout + 1), bo2 = __ldg(a.bout + 2), bo3 = __ldg(a.bout + 3);
  const int step = a.tc - a.overlap;
  const float inv_ov1 = a.overlap > 1 ? 1.0f / (float)(a.overlap - 1) : 0.f;

  const int t0 = blockIdx.x * frames_per_cta;
  for (int f = 0; f < frames_per_cta; ++f) {
    const int t = t0 + f;
    if (t >= a.T) break;
    int k_hi = t / step;
    if (k_hi > a.P - 1) k_hi = a.P - 1;
    int k_lo = t - a.tc + 1;
    k_lo = k_lo > 0 ? (k_lo + step - 1) / step : 0;
    float acc0 = 0.f, acc1 = 0.f, acc2 = 0.f, acc3 = 0.f;
    for (int kc = k_lo; kc <= k_hi; kc += MASK_MAXP) {
      const int np = min(MASK_MAXP, k_hi - kc + 1);
      __syncthreads();
      for (int idx = tid; idx < np * NDEC * C1; idx += MASK_THREADS) {
        const int j = idx / (NDEC * C1), rem = idx - j * NDEC * C1;
        const int d = rem / C1, c = rem - d * C1;
        const int k = kc + j, p = t - k * step;
        gs[j][d][c] = __ldg(a.G + ((int64_t)(k * NDEC + d) * a.tc + p) * a.ldg + c);
      }
      __syncthreads();
      if (bok) {
        for (int j = 0; j < np; ++j) {
          const int k = kc + j, p = t - k * step;
          float y[NDEC];
#pragma unroll
          for (int d = 0; d < NDEC; ++d) {
            float s0 = 0.f, s1 = 0.f;
            const float4* g4 = reinterpret_cast<const float4*>(&gs[j][d][0]);
#pragma unroll
            for (int q = 0; q < C1 / 4; ++q) {
              const float4 g = g4[q];
              s0 = fmaf(w[4 * q + 0], g.x, s0);
              s1 = fmaf(w[4 * q + 1], g.y, s1);
              s0 = fmaf(w[4 * q + 2], g.z, s0);
              s1 = fmaf(w[4 * q + 3], g.w, s1);
            }
#pragma unroll
            for (int c = C1 / 4 * 4; c < C1; ++c) s0 = fmaf(w[c], gs[j][d][c], s0);
            y[d] = s0 + s1;
          }
          // NDEC == 3: l_merge = [dec1, dec2, dec3, dec2] (separate_dsd.py:228 builds source 4 from l_fc12)
          // NDEC == 4: one decoder per source (trainCNN_ILD_DSD100.py:95-100)
          const float p0 = fmaxf(y[0] + bo0, 0.f), p1 = fmaxf(y[1] + bo1, 0.f);
          const float p2 = fmaxf(y[2] + bo2, 0.f), p3 = fmaxf(y[NDEC == 4 ? 3 : 1] + bo3, 0.f);
          const float tot = (p0 + p1) + (p2 + p3);
          float m0, m1, m2, m3;
          if (tot > MASK_TOT_MIN) {
            const float r = 1.0f / tot;
            m0 = p0 * r; m1 = p1 * r; m2 = p2 * r; m3 = p3 * r;
          } else if (NDEC == 3) {  // eps*rand cancels: every source gets 1/4 (separate_dsd.py:258-266)
            m0 = m1 = m2 = m3 = 0.25f;
          } else {                 // prediction / (sum + eps*rand) with prediction == 0 (trainCNN_ILD_DSD100.py:185)
            m0 = m1 = m2 = m3 = 0.f;
          }
          if (k == k_lo) {
            acc0 = m0; acc1 = m1; acc2 = m2; acc3 = m3;
          } else {  // sep = down*sep + up*src on the first `overlap` frames of a later patch
            const float up = (float)p * inv_ov1;
            const float down = (float)(a.overlap - 1 - p) * inv_ov1;
            acc0 = down * acc0 + up * m0;
            acc1 = down * acc1 + up * m1;
            acc2 = down * acc2 + up * m2;
            acc3 = down * acc3 + up * m3;
          }
        }
      }
    }
    if (MASKS && bok) {
      const int64_t o = (int64_t)t * a.ldf + b;
      M[o] = acc0;
      M[o + a.src_stride] = acc1;
      M[o + 2 * a.src_stride] = acc2;
      M[o + 3 * a.src_stride] = acc3;
    } else if (bok) {
      const int64_t o = (int64_t)t * a.ldf + b;
      const float2 x = a.X[o];
      a.S[o] = make_float2(acc0 * x.x, acc0 * x.y);
      a.S[o + a.src_stride] = make_float2(acc1 * x.x, acc1 * x.y);
      a.S[o + 2 * a.src_stride] = make_float2(acc2 * x.x, acc2 * x.y);
      a.S[o + 3 * a.src_stride] = make_float2(acc3 * x.x, acc3 * x.y);
    }
  }
}

int launch_dsd_mask(dcs_ctx* ctx, const DsdMaskArgs& a, cudaStream_t st, float* M) {
  if (a.T <= 0) return DCS_OK;
  DCS_REQUIRE(a.tc > a.overlap && a.overlap >= 0, "time_context %d must exceed overlap %d", a.tc, a.overlap);
  const int fpc = 16;
  // frames on gridDim.x (2^31-1 blocks: any clip length), bin tiles on gridDim.y (a handful)
  dim3 grid((unsigned)ceil_div64(a.T, fpc), (unsigned)ceil_div64(a.F - 1, MASK_TILE));
  if (M && a.ndec == 4) dsd_mask_kernel<50, 4, true><<<grid, MASK_THREADS, 0, st>>>(a, M, fpc);
  else if (M) dsd_mask_kernel<50, 3, true><<<grid, MASK_THREADS, 0, st>>>(a, M, fpc);
  else if (a.ndec == 4) dsd_mask_kernel<50, 4><<<grid, MASK_THREADS, 0, st>>>(a, nullptr, fpc);
  else dsd_mask_kernel<50, 3><<<grid, MASK_THREADS, 0, st>>>(a, nullptr, fpc);
  DCS_CHECK_LAUNCH();
  ctx->launches++;
  return DCS_OK;
}

}  // namespace dcs
