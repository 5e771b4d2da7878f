// dsd_tc.cu -- K3 on the tensor cores: InverseLayer(conv1) for every (patch, decoder) covering a
// frame as ONE wgmma GEMM per tile, with bias + ReLU + soft ratio mask + patch cross-fade +
// mixture-phase re-apply fused into the epilogue.  Same math as dsd.cu (reference:
// separate_dsd.py:212-234, :258-271, :139-169, :304); dsd.cu remains the path for
// (time_context, overlap) settings with more than 6 patches per frame and the DCS_DEBUG_SIMT_GEMM
// cross-check.
//
// GEMM view (D = A * B^T, fp32-accurate 3xTF32):
//   M = frequency bins  (128 per CTA tile, one 64-row half per warpgroup)
//   N = (frame, patch slot, decoder) = 8 x 6 x 3 (or 6 x 6 x 4, the stereo net) = 144 columns per group
//   K = conv1 filters (50, padded to 56 = 7 k-steps; two 32-wide swizzled planes)
//   A = W1t tile [128 bins][K]  (weights; split hi/lo into shared memory ONCE per CTA)
//   B = G rows   [144][K]       (decoder activations of the patches covering the group's frames,
//                                gathered from the patch-major G; empty slots are zero rows)
// Persistent CTAs: a CTA owns one 128-bin tile and a contiguous range of groups.  Per group all
// 256 threads store the (prefetched) B rows split into hi/lo planes, the two warpgroups issue 21
// wgmma m64n144k8 (the 14 small correction products first, then the 7 main ones, so the truncating
// accumulation sees only 7 large addends), park the accumulators in a [144][bins] shared tile, and
// every thread then runs the mask epilogue for one bin and half of the group's frames.  The global
// loads of the next group's B rows are in flight during the MMAs and the epilogue.
#include "common.cuh"
#include "tc.cuh"

namespace dcs {

using namespace tc;

constexpr int MT_BINS = 128;             // bins per CTA tile
constexpr int MT_SLOTS = 6;              // patch slots per frame
constexpr int MT_COLS = 144;             // GEMM columns per group = frames x 6 slots x decoders
constexpr int MT_C1 = 50;
constexpr int MT_KSTEPS = 7;             // ceil(50 / 8)
constexpr int MT_THREADS = 256;          // two warpgroups
constexpr int MT_A_SUB = MT_BINS * ROW_BYTES;      // 16 KB: [128][32] fp32
constexpr int MT_B_SUB = MT_COLS * ROW_BYTES;      // 18 KB: [144][32] fp32
constexpr int MT_A_BYTES = 4 * MT_A_SUB;           // hi k0-31, hi k32-63, lo k0-31, lo k32-63
constexpr int MT_B_BYTES = 4 * MT_B_SUB;           // same four planes
constexpr int MT_DP = MT_BINS + 4;                 // row pitch of the accumulator tile (conflict-free stores)
constexpr int MT_D_OFF = MT_A_BYTES + MT_B_BYTES;
constexpr int MT_SMEM = MT_D_OFF + MT_COLS * MT_DP * 4 + 1024;   // + alignment slack
constexpr int MT_B_CHUNKS = MT_COLS * 16 / MT_THREADS;           // 16-byte pieces of B per thread and group: 9

// NDEC = 3: the DSD100 / hiphopss net (4th output = decoder 2 with its own bias, all-zero bins get 1/4 each,
//           separate_dsd.py:228,258-266), 8 frames per group;
// NDEC = 4: the stereo / ILD net, one launch per input channel (one decoder per source, all-zero bins get 0,
//           trainCNN_ILD_DSD100.py:99-106,183-186), 6 frames per group -- the same 144-column tile either way.
template <int NDEC>
struct MaskTile {
  static constexpr int FRAMES = MT_COLS / (MT_SLOTS * NDEC);    // 8 or 6
  static constexpr int VALS = MT_SLOTS * NDEC;                  // accumulator columns per frame: 18 or 24
};

// B rows of group g: row r = (frame f, slot j, decoder d) = (f * 6 + j) * NDEC + d, 16 float4 per row
// (columns 52..63 are zero).  The patch in slot j of frame t is k_lo(t) + j; an empty slot is a zero row.
template <int NDEC>
__device__ __forceinline__ void mask_load_b(const DsdMaskArgs& a, int g, int tid, float4 (&rb)[MT_B_CHUNKS]) {
  const int step = a.tc - a.overlap;
#pragma unroll
  for (int i = 0; i < MT_B_CHUNKS; ++i) {
    const int idx = i * MT_THREADS + tid, r = idx >> 4, c4 = idx & 15;
    const int f = r / (MT_SLOTS * NDEC), jd = r - f * (MT_SLOTS * NDEC), j = jd / NDEC, d = jd - j * NDEC;
    const int t = g * MaskTile<NDEC>::FRAMES + f;
    int k_lo = t - a.tc + 1;
    k_lo = k_lo > 0 ? (k_lo + step - 1) / step : 0;
    const int k = k_lo + j;
    rb[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c4 < 13 && t < a.T && k < a.P && k * step <= t) {
      const int p = t - k * step;
      rb[i] = __ldg(reinterpret_cast<const float4*>(a.G + ((int64_t)(k * NDEC + d) * a.tc + p) * a.ldg) + c4);
    }
  }
}

template <int NDEC>
__global__ void __launch_bounds__(MT_THREADS, 1)
dsd_mask_tc_kernel(const DsdMaskArgs a, const float4* __restrict__ xtab, int groups_per_cta, int num_groups) {
  using MT = MaskTile<NDEC>;
  constexpr int FRAMES = MT::FRAMES, VALS = MT::VALS;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  uint8_t* sA = smem;
  uint8_t* sB = smem + MT_A_BYTES;
  float* sD = reinterpret_cast<float*>(smem + MT_D_OFF);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wg = warp >> 2, wq = warp & 3;
  const int bin0 = blockIdx.x * MT_BINS;
  const int g_begin = blockIdx.y * groups_per_cta;
  const int g_end = min(num_groups, g_begin + groups_per_cta);

  // A tile: thread = bin row (threads 0..127), W1t is [c][bin] so the reads are coalesced over bins
  if (tid < MT_BINS) {
    const int b = bin0 + tid;
    const bool ok = b < a.F;
#pragma unroll
    for (int c4 = 0; c4 < 16; ++c4) {
      float e[4], hi[4], lo[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int c = 4 * c4 + i;
        e[i] = (ok && c < MT_C1) ? __ldg(a.W1t + (int64_t)c * a.ldw + b) : 0.f;
        split_tf32(e[i], hi[i], lo[i]);
      }
      const uint32_t off = (c4 >> 3) * MT_A_SUB + tile_off(tid, c4 & 7);
      *reinterpret_cast<float4*>(sA + off) = make_float4(hi[0], hi[1], hi[2], hi[3]);
      *reinterpret_cast<float4*>(sA + 2 * MT_A_SUB + off) = make_float4(lo[0], lo[1], lo[2], lo[3]);
    }
  }

  // epilogue ownership: bin = tid % 128, frames [fh * FRAMES/2, (fh + 1) * FRAMES/2)
  const int eb = tid & (MT_BINS - 1), fh = tid >> 7;
  const int b = bin0 + eb;
  const bool bok = b < a.F;
  const float bo0 = __ldg(a.bout + 0), bo1 = __ldg(a.bout + 1), bo2 = __ldg(a.bout + 2), bo3 = __ldg(a.bout + 3);

  float4 rb[MT_B_CHUNKS];
  if (g_begin < g_end) mask_load_b<NDEC>(a, g_begin, tid, rb);
  for (int g = g_begin; g < g_end; ++g) {
    // ---- B planes (the previous group's MMAs and epilogue reads are done: barrier at the loop end)
#pragma unroll
    for (int i = 0; i < MT_B_CHUNKS; ++i) {
      const int idx = i * MT_THREADS + tid, r = idx >> 4, c4 = idx & 15;
      float h[4], l[4];
      split_tf32(rb[i].x, h[0], l[0]); split_tf32(rb[i].y, h[1], l[1]);
      split_tf32(rb[i].z, h[2], l[2]); split_tf32(rb[i].w, h[3], l[3]);
      const uint32_t off = (c4 >> 3) * MT_B_SUB + tile_off(r, c4 & 7);
      *reinterpret_cast<float4*>(sB + off) = make_float4(h[0], h[1], h[2], h[3]);
      *reinterpret_cast<float4*>(sB + 2 * MT_B_SUB + off) = make_float4(l[0], l[1], l[2], l[3]);
    }
    fence_proxy_async();
    __syncthreads();
    if (g + 1 < g_end) mask_load_b<NDEC>(a, g + 1, tid, rb);   // in flight during the MMAs and the epilogue

    // ---- MMAs: warpgroup wg computes bins [64 wg, 64 wg + 64) x 144 columns
    {
      float acc[72];
      const uint32_t a_hi = smem_u32(sA) + wg * 64 * ROW_BYTES, a_lo = a_hi + 2 * MT_A_SUB;
      const uint32_t b_hi = smem_u32(sB), b_lo = b_hi + 2 * MT_B_SUB;
      wgmma_fence();
#pragma unroll
      for (int j = 0; j < MT_KSTEPS; ++j) {
        const uint32_t ao = (j >> 2) * MT_A_SUB + KSTEP_BYTES * (j & 3), bo = (j >> 2) * MT_B_SUB + KSTEP_BYTES * (j & 3);
        wgmma_tf32_n144(acc, make_desc(a_lo + ao), make_desc(b_hi + bo), j != 0);
      }
#pragma unroll
      for (int j = 0; j < MT_KSTEPS; ++j) {
        const uint32_t ao = (j >> 2) * MT_A_SUB + KSTEP_BYTES * (j & 3), bo = (j >> 2) * MT_B_SUB + KSTEP_BYTES * (j & 3);
        wgmma_tf32_n144(acc, make_desc(a_hi + ao), make_desc(b_lo + bo), 1);
      }
#pragma unroll
      for (int j = 0; j < MT_KSTEPS; ++j) {
        const uint32_t ao = (j >> 2) * MT_A_SUB + KSTEP_BYTES * (j & 3), bo = (j >> 2) * MT_B_SUB + KSTEP_BYTES * (j & 3);
        wgmma_tf32_n144(acc, make_desc(a_hi + ao), make_desc(b_hi + bo), 1);
      }
      wgmma_commit();
      wgmma_wait_all();
      // fragment -> sD[column][bin] (tc.cuh: d[4j + 2i + e] = D[16 wq + lane/4 + 8i][8j + 2(lane%4) + e])
#pragma unroll
      for (int j = 0; j < MT_COLS / 8; ++j)
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
          for (int e = 0; e < 2; ++e)
            sD[(8 * j + 2 * (lane & 3) + e) * MT_DP + wg * 64 + wq * 16 + (lane >> 2) + 8 * i] = acc[4 * j + 2 * i + e];
    }
    __syncthreads();

    // ---- epilogue (thread = bin): bias + ReLU + ratio mask + sequential cross-fade + .X
#pragma unroll 1
    for (int ff = fh * (FRAMES / 2); ff < (fh + 1) * (FRAMES / 2); ++ff) {
      const int t = g * FRAMES + ff;
      const float2 x = (bok && t < a.T) ? a.X[(int64_t)t * a.ldf + b] : make_float2(0.f, 0.f);
      float acc0 = 0.f, acc1 = 0.f, acc2 = 0.f, acc3 = 0.f;
#pragma unroll
      for (int j = 0; j < MT_SLOTS; ++j) {
        // (up, down, up/4, -) of (frame, slot) (dsd_xfade_table_kernel): acc <- down*acc + up*mask
        const float4 c = __ldg(xtab + (int64_t)t * MT_SLOTS + j);
        const float* y = sD + (ff * VALS + NDEC * j) * MT_DP + eb;
        const float p0 = fmaxf(y[0] + bo0, 0.f), p1 = fmaxf(y[MT_DP] + bo1, 0.f);
        const float p2 = fmaxf(y[2 * MT_DP] + bo2, 0.f);
        const float p3 = fmaxf(y[(NDEC == 3 ? 1 : 3) * MT_DP] + bo3, 0.f);   // DSD100: decoder 2 again (separate_dsd.py:228)
        const float tot = (p0 + p1) + (p2 + p3);
        const bool pos = tot > 1.2e-38f;
        float rc;
        asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(rc) : "f"(tot));
        const float r = pos ? c.x * rc : 0.f;             // up * mask = p * (up / tot)
        const float q = (pos || NDEC == 4) ? 0.f : c.z;   // all-zero bin: 1/4 each (DSD100 rule); 0 (ILD rule)
        acc0 = fmaf(c.y, acc0, fmaf(p0, r, q));
        acc1 = fmaf(c.y, acc1, fmaf(p1, r, q));
        acc2 = fmaf(c.y, acc2, fmaf(p2, r, q));
        acc3 = fmaf(c.y, acc3, fmaf(p3, r, q));
      }
      if (bok && t < a.T) {
        const int64_t o = (int64_t)t * a.ldf + b;
        a.S[o] = make_float2(acc0 * x.x, acc0 * x.y);
        a.S[o + a.src_stride] = make_float2(acc1 * x.x, acc1 * x.y);
        a.S[o + 2 * a.src_stride] = make_float2(acc2 * x.x, acc2 * x.y);
        a.S[o + 3 * a.src_stride] = make_float2(acc3 * x.x, acc3 * x.y);
      }
    }
    __syncthreads();   // sB and sD are rewritten for the next group
  }
}

// (up, down, up/4, 0) of every (frame, patch slot): the sequential cross-fade of overlapadd_multi
// (separate_dsd.py:139-169) as a per-slot recurrence; frames >= T (padding to whole groups) and slots
// without a patch get (0, 1): they leave the accumulated masks untouched.
__global__ void dsd_xfade_table_kernel(float4* __restrict__ tab, int T, int Tpad, int P, int tc, int overlap) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= Tpad * MT_SLOTS) return;
  const int t = i / MT_SLOTS, j = i - t * MT_SLOTS;
  const int step = tc - overlap;
  const float inv_ov1 = overlap > 1 ? 1.0f / (float)(overlap - 1) : 0.f;
  int k_lo = t - tc + 1;
  k_lo = k_lo > 0 ? (k_lo + step - 1) / step : 0;
  int k_hi = t / step;
  if (k_hi > P - 1) k_hi = P - 1;
  float up = 0.f, down = 1.f;
  if (t < T && k_lo + j <= k_hi) {
    const int p = t - (k_lo + j) * step;
    up = j == 0 ? 1.f : (float)p * inv_ov1;
    down = j == 0 ? 0.f : (float)(overlap - 1 - p) * inv_ov1;
  }
  tab[i] = make_float4(up, down, 0.25f * up, 0.f);
}

bool dsd_mask_tc_supported(const DsdMaskArgs& a) {
  const int step = a.tc - a.overlap;
  return step > 0 && (a.ndec == 3 || a.ndec == 4) && (a.tc + step - 1) / step <= MT_SLOTS && a.ldg % 4 == 0 && a.ldg >= 52 &&
         ((uintptr_t)a.G % 16 == 0);
}

// all F bins; the last 128-bin tile holds only the Nyquist bin (F = 2^k + 1)
template <int NDEC>
static int launch_dsd_mask_tc_t(dcs_ctx* ctx, const DsdMaskArgs& a, cudaStream_t st) {
  using MT = MaskTile<NDEC>;
  DCS_TRY(ensure_smem_attr(dsd_mask_tc_kernel<NDEC>, MT_SMEM));
  const int m_tiles = (a.F + MT_BINS - 1) / MT_BINS;
  const int num_groups = (a.T + MT::FRAMES - 1) / MT::FRAMES;
  int chunks = ctx->num_sms / m_tiles;
  if (chunks < 1) chunks = 1;
  if (chunks > num_groups) chunks = num_groups;
  const int gpc = (num_groups + chunks - 1) / chunks;
  dim3 grid((unsigned)m_tiles, (unsigned)((num_groups + gpc - 1) / gpc));
  const int Tpad = num_groups * MT::FRAMES;
  DCS_TRY(ctx->net[NET_XTAB].ensure((size_t)Tpad * MT_SLOTS * sizeof(float4), st));
  float4* xtab = ctx->net[NET_XTAB].as<float4>();
  dsd_xfade_table_kernel<<<(unsigned)ceil_div64((int64_t)Tpad * MT_SLOTS, 256), 256, 0, st>>>(xtab, a.T, Tpad, a.P, a.tc, a.overlap);
  DCS_CHECK_LAUNCH();
  ctx->launches++;
  dsd_mask_tc_kernel<NDEC><<<grid, MT_THREADS, MT_SMEM, st>>>(a, xtab, gpc, num_groups);
  DCS_CHECK_LAUNCH();
  ctx->launches++;
  return DCS_OK;
}

int launch_dsd_mask_tc(dcs_ctx* ctx, const DsdMaskArgs& a, cudaStream_t st) {
  if (a.T <= 0) return DCS_OK;
  DCS_REQUIRE(dsd_mask_tc_supported(a), "dsd_mask_tc: unsupported shape");
  return a.ndec == 4 ? launch_dsd_mask_tc_t<4>(ctx, a, st) : launch_dsd_mask_tc_t<3>(ctx, a, st);
}

}  // namespace dcs
