// dsd_tc.cu -- K3 on the tensor cores: InverseLayer(conv1) for every (patch, decoder) covering a
// frame as ONE wgmma GEMM per tile, with bias + ReLU + soft ratio mask + patch cross-fade +
// mixture-phase re-apply fused into the epilogue.  Same math as dsd.cu (reference:
// separate_dsd.py:212-234, :258-271, :139-169, :304); dsd.cu remains the path for
// (time_context, overlap) settings with more than 6 patches per frame and the DCS_DEBUG_SIMT_GEMM
// cross-check.
//
// GEMM view (D = A * B^T, fp32-accurate 3xTF32):
//   M = frequency bins  (128 per tile, one 64-row half per warpgroup)
//   N = (frame, patch slot, decoder) per group: 8 x 6 x 3 = 144 columns (DSD100), 4 x 6 x 4 = 96 (stereo net)
//   K = conv1 filters (50, padded to 56 = 7 k-steps; two 32-wide swizzled planes)
//   A = W1t tile [128 bins][K]  (weights; split hi/lo into shared memory once per tile and CTA)
//   B = G rows   [N][K]         (decoder activations of the patches covering the group's frames,
//                                gathered from the patch-major G; empty slots are zero rows)
// The B rows are ordered so that each thread's accumulator fragment holds every value its outputs
// need (2 bins x 2 frames x 18 values, or 2 bins x 1 frame x 24 values): the epilogue runs straight
// from the wgmma registers.
//
// Persistent CTAs, one per SM, each over a contiguous range of (tile, group) work items in tile-major
// order.  B is double-buffered.  Per item, after one barrier: each warpgroup issues the 21 k8 products
// (the 14 small correction products first, then the 7 main ones, so the truncating accumulation sees
// only 7 large addends) on stage s as two commit groups, columns of slots 0-2 and of slots 3-5; while
// they run, every thread issues this item's X loads, splits and stores the prefetched B rows of the next
// item into stage s^1 and issues the global loads of the item after that; then it runs the mask
// epilogue from registers, slots 0-2 as soon as the first commit group has landed.
#include "common.cuh"
#include "tc.cuh"

namespace dcs {

using namespace tc;

constexpr int MT_BINS = 128;             // bins per tile
constexpr int MT_SLOTS = 6;              // patch slots per frame
constexpr int MT_C1 = 50;
constexpr int MT_KSTEPS = 7;             // ceil(50 / 8)
constexpr int MT_THREADS = 256;          // two warpgroups
constexpr int MT_A_SUB = MT_BINS * ROW_BYTES;      // 16 KB: [128][32] fp32
constexpr int MT_A_BYTES = 4 * MT_A_SUB;           // hi k0-31, hi k32-63, lo k0-31, lo k32-63

// NDEC = 3: the DSD100 / hiphopss net (4th output = decoder 2 with its own bias, all-zero bins get 1/4 each,
//           separate_dsd.py:228,258-266), 8 frames per group, 144 columns (two m64n72k8 halves);
// NDEC = 4: the stereo / ILD net, one launch per input channel (one decoder per source, all-zero bins get 0,
//           trainCNN_ILD_DSD100.py:99-106,183-186), 4 frames per group, 96 columns (two m64n48k8 halves).
// NX: mixture channels the cross-faded masks are applied to -- 1, or 2 with NDEC = 3 (stereo stems from the masks of
//     the downmix: the same m times each channel's X; GEMM, gather and cross-fade run once).
// Value v = slot * NDEC + decoder.  Fragment (tc.cuh): d[4j + 2i + e] = D[16w + l/4 + 8i][8j + 2(l%4) + e].
//   NDEC = 3: column 8v + f          -> thread holds frames f = 2(l%4) + e, all v: d[4v + 2i + e]
//   NDEC = 4: column 8(v/2) + 2f + v%2 -> thread holds frame f = l%4, all v:     d[4(v/2) + 2i + v%2]
template <int NDEC>
struct MaskTile {
  static constexpr int FRAMES = NDEC == 3 ? 8 : 4;
  static constexpr int COLS = FRAMES * MT_SLOTS * NDEC;         // 144 or 96
  static constexpr int HCOLS = COLS / 2;                        // columns of slots 0-2 (and of slots 3-5)
  static constexpr int TFRAMES = NDEC == 3 ? 2 : 1;             // frames per thread
  static constexpr int B_SUB = COLS * ROW_BYTES;
  static constexpr int B_BYTES = 4 * B_SUB;                     // one stage: the same four planes as A
  static constexpr int B_CHUNKS = COLS * 16 / MT_THREADS;       // 16-byte pieces of B per thread and group: 9 or 6
  static constexpr int SMEM = MT_A_BYTES + 2 * B_BYTES + 1024;  // + alignment slack
  __device__ static int col_frame(int c) { return NDEC == 3 ? (c & 7) : (c & 7) >> 1; }
  __device__ static int col_value(int c) { return NDEC == 3 ? c >> 3 : 2 * (c >> 3) + (c & 1); }
  // frame of the thread's e-th frame (lane = l)
  __device__ static int thread_frame(int lane, int e) { return NDEC == 3 ? 2 * (lane & 3) + e : lane & 3; }
  // accumulator register of (row half i, thread frame e, value v) in the fragment of the column half holding v
  __host__ __device__ static constexpr int acc(int i, int e, int v) { return NDEC == 3 ? 4 * v + 2 * i + e : 4 * (v >> 1) + 2 * i + (v & 1); }
};

// A tile: thread = bin row (threads 0..127), W1t is [c][bin] so the reads are coalesced over bins
__device__ __forceinline__ void mask_load_a(const DsdMaskArgs& a, int tile, int tid, uint8_t* sA) {
  if (tid >= MT_BINS) return;
  const int b = tile * MT_BINS + tid;
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

// B rows of group g: row r = GEMM column (MaskTile::col_frame / col_value), 16 float4 per row (columns
// 52..63 are zero).  The patch in slot j of frame t is k_lo(t) + j; an empty slot is a zero row.
template <int NDEC>
__device__ __forceinline__ void mask_load_b(const DsdMaskArgs& a, int g, int tid, float4 (&rb)[MaskTile<NDEC>::B_CHUNKS]) {
  using MT = MaskTile<NDEC>;
  const int step = a.tc - a.overlap;
  // chunk i covers row 16 i + tid / 16: the frame (row % 8 decides it) is the same for all of a thread's chunks
  const int t = g * MT::FRAMES + MT::col_frame(tid >> 4), c4 = tid & 15;
  int k_lo = t - a.tc + 1;
  k_lo = k_lo > 0 ? (k_lo + step - 1) / step : 0;
#pragma unroll
  for (int i = 0; i < MT::B_CHUNKS; ++i) {
    const int v = MT::col_value(16 * i + (tid >> 4)), j = v / NDEC, d = v - j * NDEC;
    const int k = k_lo + j;
    rb[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c4 < 13 && t < a.T && k < a.P && k * step <= t) {
      const int p = t - k * step;
      rb[i] = __ldg(reinterpret_cast<const float4*>(a.G + ((int64_t)(k * NDEC + d) * a.tc + p) * a.ldg) + c4);
    }
  }
}

// the prefetched B rows, split into hi/lo planes, into one stage
template <int NDEC>
__device__ __forceinline__ void mask_store_b(uint8_t* sB, int tid, const float4 (&rb)[MaskTile<NDEC>::B_CHUNKS]) {
  using MT = MaskTile<NDEC>;
#pragma unroll
  for (int i = 0; i < MT::B_CHUNKS; ++i) {
    const int idx = i * MT_THREADS + tid, r = idx >> 4, c4 = idx & 15;
    float h[4], l[4];
    split_tf32(rb[i].x, h[0], l[0]); split_tf32(rb[i].y, h[1], l[1]);
    split_tf32(rb[i].z, h[2], l[2]); split_tf32(rb[i].w, h[3], l[3]);
    const uint32_t off = (c4 >> 3) * MT::B_SUB + tile_off(r, c4 & 7);
    *reinterpret_cast<float4*>(sB + off) = make_float4(h[0], h[1], h[2], h[3]);
    *reinterpret_cast<float4*>(sB + 2 * MT::B_SUB + off) = make_float4(l[0], l[1], l[2], l[3]);
  }
}

template <int NDEC, int NX>
__global__ void __launch_bounds__(MT_THREADS, 1)
dsd_mask_tc_kernel(const DsdMaskArgs a, const float4* __restrict__ xtab, int num_groups, int num_items) {
  using MT = MaskTile<NDEC>;
  constexpr int FRAMES = MT::FRAMES, TF = MT::TFRAMES;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  uint8_t* sA = smem;
  uint8_t* sB = smem + MT_A_BYTES;   // two stages of MT::B_BYTES

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wg = warp >> 2, wq = warp & 3;
  // work items w = tile * num_groups + group; this CTA's share [w_begin, w_end) differs from the others' by at most one
  const int w_begin = (int)((int64_t)blockIdx.x * num_items / gridDim.x);
  const int w_end = (int)((int64_t)(blockIdx.x + 1) * num_items / gridDim.x);
  const int row0 = wg * 64 + wq * 16 + (lane >> 2);   // tile rows row0 and row0 + 8 are this thread's bins
  const float bo0 = __ldg(a.bout + 0), bo1 = __ldg(a.bout + 1), bo2 = __ldg(a.bout + 2), bo3 = __ldg(a.bout + 3);

  float4 rb[MT::B_CHUNKS];
  if (w_begin < w_end) {
    mask_load_b<NDEC>(a, w_begin % num_groups, tid, rb);
    mask_store_b<NDEC>(sB, tid, rb);
    fence_proxy_async();
    if (w_begin + 1 < w_end) mask_load_b<NDEC>(a, (w_begin + 1) % num_groups, tid, rb);
  }
  int tile = -1;
  for (int w = w_begin, s = 0; w < w_end; ++w, s ^= 1) {
    const int g = w % num_groups;
    // publishes stage s; every warpgroup has waited for its MMAs of item w - 1, so stage s^1 and A are free
    __syncthreads();
    if (w / num_groups != tile) {
      tile = w / num_groups;
      mask_load_a(a, tile, tid, sA);
      fence_proxy_async();
      __syncthreads();
    }

    // ---- MMAs: warpgroup wg computes bins [64 wg, 64 wg + 64) x MT::COLS columns, as two commit groups:
    //      columns [0, HCOLS) hold slots 0-2, [HCOLS, COLS) slots 3-5
    float acc[2][MT::HCOLS / 2];
    {
      const uint32_t a_hi = smem_u32(sA) + wg * 64 * ROW_BYTES, a_lo = a_hi + 2 * MT_A_SUB;
      wgmma_fence();
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t b_hi = smem_u32(sB + s * MT::B_BYTES) + h * (MT::HCOLS / 8) * SBO, b_lo = b_hi + 2 * MT::B_SUB;
#pragma unroll
        for (int j = 0; j < MT_KSTEPS; ++j) {
          const uint32_t ao = (j >> 2) * MT_A_SUB + KSTEP_BYTES * (j & 3), bo = (j >> 2) * MT::B_SUB + KSTEP_BYTES * (j & 3);
          wgmma_tf32<MT::HCOLS>(acc[h], make_desc(a_lo + ao), make_desc(b_hi + bo), j != 0);
        }
#pragma unroll
        for (int j = 0; j < MT_KSTEPS; ++j) {
          const uint32_t ao = (j >> 2) * MT_A_SUB + KSTEP_BYTES * (j & 3), bo = (j >> 2) * MT::B_SUB + KSTEP_BYTES * (j & 3);
          wgmma_tf32<MT::HCOLS>(acc[h], make_desc(a_hi + ao), make_desc(b_lo + bo), 1);
        }
#pragma unroll
        for (int j = 0; j < MT_KSTEPS; ++j) {
          const uint32_t ao = (j >> 2) * MT_A_SUB + KSTEP_BYTES * (j & 3), bo = (j >> 2) * MT::B_SUB + KSTEP_BYTES * (j & 3);
          wgmma_tf32<MT::HCOLS>(acc[h], make_desc(a_hi + ao), make_desc(b_hi + bo), 1);
        }
        wgmma_commit();
      }
    }

    // ---- while they run: this item's X (of every channel), B of item w + 1 into stage s^1, global loads of item w + 2
    int bin[2];
    bool bok[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      bin[i] = tile * MT_BINS + row0 + 8 * i;
      bok[i] = bin[i] < a.F;
    }
    float2 x[NX][TF][2];
#pragma unroll
    for (int c = 0; c < NX; ++c)
#pragma unroll
      for (int e = 0; e < TF; ++e) {
        const int t = g * FRAMES + MT::thread_frame(lane, e);
#pragma unroll
        for (int i = 0; i < 2; ++i)
          x[c][e][i] = (bok[i] && t < a.T) ? a.X[c * a.x_plane + (int64_t)t * a.ldf + bin[i]] : make_float2(0.f, 0.f);
      }
    if (w + 1 < w_end) {
      mask_store_b<NDEC>(sB + (s ^ 1) * MT::B_BYTES, tid, rb);
      fence_proxy_async();
    }
    if (w + 2 < w_end) mask_load_b<NDEC>(a, (w + 2) % num_groups, tid, rb);

    // ---- epilogue per (bin, frame): bias + ReLU + ratio mask + sequential cross-fade + .X; slots 0-2 run
    //      while the MMAs of slots 3-5 are still in flight
    float m[TF][2][4];   // cross-faded masks of the 4 sources
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (h == 0) {
        wgmma_wait<1>();
        wgmma_fence_acc(acc[0]);
      } else {
        wgmma_wait<0>();
        wgmma_fence_acc(acc[1]);
      }
#pragma unroll
      for (int e = 0; e < TF; ++e) {
        const int t = g * FRAMES + MT::thread_frame(lane, e);
#pragma unroll
        for (int i = 0; i < 2; ++i) {
#pragma unroll
          for (int jj = 0; jj < MT_SLOTS / 2; ++jj) {
            const int j = h * (MT_SLOTS / 2) + jj;
            // (up, down, up/4, -) of (frame, slot) (dsd_xfade_table_kernel): m <- down*m + up*mask
            const float4 c = __ldg(xtab + (int64_t)t * MT_SLOTS + j);
            const float p0 = fmaxf(acc[h][MT::acc(i, e, NDEC * jj + 0)] + bo0, 0.f);
            const float p1 = fmaxf(acc[h][MT::acc(i, e, NDEC * jj + 1)] + bo1, 0.f);
            const float p2 = fmaxf(acc[h][MT::acc(i, e, NDEC * jj + 2)] + bo2, 0.f);
            const float p3 = fmaxf(acc[h][MT::acc(i, e, NDEC * jj + (NDEC == 3 ? 1 : 3))] + bo3, 0.f);   // DSD100: decoder 2 again (separate_dsd.py:228)
            const float tot = (p0 + p1) + (p2 + p3);
            const bool pos = tot > 1.2e-38f;
            float rc;
            asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(rc) : "f"(tot));
            const float r = pos ? c.x * rc : 0.f;             // up * mask = p * (up / tot)
            const float q = (pos || NDEC == 4) ? 0.f : c.z;   // all-zero bin: 1/4 each (DSD100 rule); 0 (ILD rule)
            float* mm = m[e][i];
            mm[0] = fmaf(c.y, j == 0 ? 0.f : mm[0], fmaf(p0, r, q));
            mm[1] = fmaf(c.y, j == 0 ? 0.f : mm[1], fmaf(p1, r, q));
            mm[2] = fmaf(c.y, j == 0 ? 0.f : mm[2], fmaf(p2, r, q));
            mm[3] = fmaf(c.y, j == 0 ? 0.f : mm[3], fmaf(p3, r, q));
          }
        }
      }
    }
    // source s, channel c at S + (s * NX + c) * src_stride
#pragma unroll
    for (int c = 0; c < NX; ++c)
#pragma unroll
      for (int e = 0; e < TF; ++e) {
        const int t = g * FRAMES + MT::thread_frame(lane, e);
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          if (bok[i] && t < a.T) {
            const float2 xx = x[c][e][i];
            const float* mm = m[e][i];
            const int64_t o = (int64_t)t * a.ldf + bin[i] + c * a.src_stride;
            a.S[o] = make_float2(mm[0] * xx.x, mm[0] * xx.y);
            a.S[o + NX * a.src_stride] = make_float2(mm[1] * xx.x, mm[1] * xx.y);
            a.S[o + 2 * NX * a.src_stride] = make_float2(mm[2] * xx.x, mm[2] * xx.y);
            a.S[o + 3 * NX * a.src_stride] = make_float2(mm[3] * xx.x, mm[3] * xx.y);
          }
        }
      }
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
  return step > 0 && (a.ndec == 3 || a.ndec == 4) && (a.nx == 1 || (a.nx == 2 && a.ndec == 3)) && (a.tc + step - 1) / step <= MT_SLOTS && a.ldg % 4 == 0 && a.ldg >= 52 &&
         ((uintptr_t)a.G % 16 == 0);
}

// all F bins; the last 128-bin tile holds only the Nyquist bin (F = 2^k + 1)
template <int NDEC, int NX>
static int launch_dsd_mask_tc_t(dcs_ctx* ctx, const DsdMaskArgs& a, cudaStream_t st) {
  using MT = MaskTile<NDEC>;
  DCS_TRY(ensure_smem_attr(dsd_mask_tc_kernel<NDEC, NX>, MT::SMEM));
  const int m_tiles = (a.F + MT_BINS - 1) / MT_BINS;
  const int num_groups = (a.T + MT::FRAMES - 1) / MT::FRAMES;
  const int num_items = m_tiles * num_groups;
  const int ctas = std::min(ctx->num_sms, num_items);
  const int Tpad = num_groups * MT::FRAMES;
  DCS_TRY(ctx->net[NET_XTAB].ensure((size_t)Tpad * MT_SLOTS * sizeof(float4), st));
  float4* xtab = ctx->net[NET_XTAB].as<float4>();
  dsd_xfade_table_kernel<<<(unsigned)ceil_div64((int64_t)Tpad * MT_SLOTS, 256), 256, 0, st>>>(xtab, a.T, Tpad, a.P, a.tc, a.overlap);
  DCS_CHECK_LAUNCH();
  ctx->launches++;
  dsd_mask_tc_kernel<NDEC, NX><<<(unsigned)ctas, MT_THREADS, MT::SMEM, st>>>(a, xtab, num_groups, num_items);
  DCS_CHECK_LAUNCH();
  ctx->launches++;
  return DCS_OK;
}

int launch_dsd_mask_tc(dcs_ctx* ctx, const DsdMaskArgs& a, cudaStream_t st) {
  if (a.T <= 0) return DCS_OK;
  DCS_REQUIRE(dsd_mask_tc_supported(a), "dsd_mask_tc: unsupported shape");
  if (a.ndec == 4) return launch_dsd_mask_tc_t<4, 1>(ctx, a, st);
  return a.nx == 2 ? launch_dsd_mask_tc_t<3, 2>(ctx, a, st) : launch_dsd_mask_tc_t<3, 1>(ctx, a, st);
}

}  // namespace dcs
