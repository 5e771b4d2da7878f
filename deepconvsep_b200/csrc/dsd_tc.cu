// dsd_tc.cu -- K3 on the tensor cores: InverseLayer(conv1) for every (patch, decoder) covering a
// frame as ONE wgmma GEMM per tile, with bias + ReLU + soft ratio mask + patch cross-fade +
// mixture-phase re-apply fused into the epilogue.  Same math as dsd.cu (reference:
// separate_dsd.py:212-234, :258-271, :139-169, :304); dsd.cu remains the path for
// (time_context, overlap) settings with more than 6 patches per frame and, under DCS_DEBUG_SIMT_GEMM=1,
// the cross-check of this kernel alone.
//
// GEMM view (D = A * B^T, fp32-accurate 3xTF32):
//   M = frequency bins  (128 per tile, one 64-row half per consumer warpgroup)
//   N = (frame, patch slot, decoder) per group: 8 x 6 x 3 = 144 columns (DSD100), 4 x 6 x 4 = 96 (stereo net)
//   K = conv1 filters (50, padded to 56 = 7 k-steps; two 32-wide swizzled planes)
//   A = W1t tile [128 bins][K]  (weights; a pre-split image of every tile, built per launch by dsd_mask_tables_kernel
//                                next to the fade table, bulk-copied into shared memory per item)
//   B = G rows   [N][K]         (decoder activations of the patches covering the group's frames,
//                                gathered from the patch-major G; empty slots are zero rows)
// The B rows are ordered so that each thread's accumulator fragment holds every value its outputs
// need (2 bins x 2 frames x 18 values, or 2 bins x 1 frame x 24 values): the epilogue runs straight
// from the wgmma registers.
//
// Persistent CTAs, one per SM, each over a contiguous range of (group, tile) work items in group-major
// order (w = group * m_tiles + tile), so consecutive items of a CTA share their B rows, with three warpgroups:
//   - the producer (warpgroup 2) bulk-copies the A image of item w into one of two stages, and when its range enters
//     a new group, gathers and splits the group's B rows into the one B stage (the next group's rows are loaded into
//     registers while the current group's tiles run), stages the group's fade-table entries in a ring of two and
//     computes the group's Nyquist bin;
//   - consumers 0 and 1 each issue the 21 k8 products of their 64 bins as one m64n144k8 (m64n96k8) chain --
//     the 14 small correction products first, then the 7 main ones, so the truncating accumulation sees
//     only 7 large addends -- release the A stage (and, after the group's last item, the B stage) once they
//     are complete, and run the mask epilogue from registers.  Two named barriers alternate the issue:
//     consumer 1 issues item w while consumer 0 runs its epilogue of item w, and consumer 0 issues item w + 1
//     while consumer 1 runs its epilogue of item w, so one consumer's epilogue runs under the other's products.
// F = 128 m + 1 (the nets' N / 2 + 1): the tiles cover bins [0, F - 1) and the Nyquist bin, which would
// take a 128-bin tile of its own, is computed by the producer from the fp32 rows it has loaded: an FMA
// chain over each thread's 4 k-values and a fixed xor tree over the 16 threads of a row, then the same
// epilogue arithmetic (mask_slot), by the CTA whose range holds item (g, tile = g mod m).
#include "common.cuh"
#include "tc.cuh"

namespace dcs {

using namespace tc;

constexpr int MT_BINS = 128;             // bins per tile
constexpr int MT_SLOTS = 6;              // patch slots per frame
constexpr int MT_C1 = 50;
constexpr int MT_KSTEPS = 7;             // ceil(50 / 8)
constexpr int MT_CONSUMERS = 256;        // warpgroups 0 and 1: one 64-bin half of the tile each
constexpr int MT_PRODUCER = 128;         // warpgroup 2: A copies, B rows (and the Nyquist bin)
constexpr int MT_THREADS = MT_CONSUMERS + MT_PRODUCER;
constexpr int MT_A_SUB = MT_BINS * ROW_BYTES;      // 16 KB: [128][32] fp32
constexpr int MT_A_BYTES = 4 * MT_A_SUB;           // hi k0-31, hi k32-63, lo k0-31, lo k32-63
// named barriers
constexpr int MT_BAR_TURN1 = 1;          // consumer 1 may issue item w: consumer 0 has issued it
constexpr int MT_BAR_TURN0 = 2;          // consumer 0 may issue item w + 1: consumer 1 has issued item w
constexpr int MT_BAR_PROD = 3;           // the producer's Nyquist dot products are in shared memory

// NDEC = 3: the DSD100 / hiphopss net (4th output = decoder 2 with its own bias, all-zero bins get 1/4 each,
//           separate_dsd.py:228,258-266), 8 frames per group, 144 columns (m64n144k8);
// NDEC = 4: the stereo / ILD net, one launch per input channel (one decoder per source, all-zero bins get 0,
//           trainCNN_ILD_DSD100.py:99-106,183-186), 4 frames per group, 96 columns (m64n96k8).
// Value v = slot * NDEC + decoder.  Fragment (tc.cuh): d[4j + 2i + e] = D[16w + l/4 + 8i][8j + 2(l%4) + e].
//   NDEC = 3: column 8v + f          -> thread holds frames f = 2(l%4) + e, all v: d[4v + 2i + e]
//   NDEC = 4: column 8(v/2) + 2f + v%2 -> thread holds frame f = l%4, all v:     d[4(v/2) + 2i + v%2]
template <int NDEC>
struct MaskTile {
  static constexpr int FRAMES = NDEC == 3 ? 8 : 4;
  static constexpr int COLS = FRAMES * MT_SLOTS * NDEC;         // 144 or 96
  static constexpr int TFRAMES = NDEC == 3 ? 2 : 1;             // frames per thread
  static constexpr int B_SUB = COLS * ROW_BYTES;
  static constexpr int B_BYTES = 4 * B_SUB;                     // one stage: the same four planes as A
  static constexpr int B_CHUNKS = COLS * 16 / MT_PRODUCER;      // 16-byte pieces of B per producer thread and group: 18 or 12
  static constexpr int HCHUNKS = B_CHUNKS / 2;                  // loaded and stored in two halves
  static constexpr int NYQ_BYTES = 2 * COLS * 4;                // two buffers of the Nyquist bin's GEMM values
  static constexpr int XF = FRAMES * MT_SLOTS;                  // fade-table entries of a group
  static constexpr int XF_BYTES = 2 * XF * 16;                  // a ring of two groups' entries
  static constexpr int SMEM = 2 * MT_A_BYTES + B_BYTES + NYQ_BYTES + XF_BYTES + 1024;   // + alignment slack
  __host__ __device__ static constexpr int col_frame(int c) { return NDEC == 3 ? (c & 7) : (c & 7) >> 1; }
  __host__ __device__ static constexpr int col_value(int c) { return NDEC == 3 ? c >> 3 : 2 * (c >> 3) + (c & 1); }
  // the column of (frame f, value v), the inverse of col_frame / col_value
  __host__ __device__ static constexpr int col(int f, int v) { return NDEC == 3 ? 8 * v + f : 8 * (v >> 1) + 2 * f + (v & 1); }
  // frame of the thread's e-th frame (lane = l)
  __device__ static int thread_frame(int lane, int e) { return NDEC == 3 ? 2 * (lane & 3) + e : lane & 3; }
  // accumulator register of (row half i, thread frame e, value v)
  __host__ __device__ static constexpr int acc(int i, int e, int v) { return NDEC == 3 ? 4 * v + 2 * i + e : 4 * (v >> 1) + 2 * i + (v & 1); }
};

// B rows of group g, chunks [I0, I0 + HCHUNKS) of producer thread ptid: row r = GEMM column (MaskTile::col_frame /
// col_value), 16 float4 per row (columns 52..63 are zero).  The patch in slot j of frame t is k_lo(t) + j; an empty
// slot is a zero row.
template <int NDEC, int I0>
__device__ __forceinline__ void mask_load_b(const DsdMaskArgs& a, int g, int ptid, float4 (&rb)[MaskTile<NDEC>::HCHUNKS]) {
  using MT = MaskTile<NDEC>;
  const int step = a.tc - a.overlap;
  // chunk i covers row 8 i + ptid / 16: the frame (row % 8 decides it) is the same for all of a thread's chunks
  const int t = g * MT::FRAMES + MT::col_frame(ptid >> 4), c4 = ptid & 15;
  int k_lo = t - a.tc + 1;
  k_lo = k_lo > 0 ? (k_lo + step - 1) / step : 0;
#pragma unroll
  for (int i = 0; i < MT::HCHUNKS; ++i) {
    const int v = MT::col_value(8 * (I0 + i) + (ptid >> 4)), j = v / NDEC, d = v - j * NDEC;
    const int k = k_lo + j;
    rb[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c4 < 13 && t < a.T && k < a.P && k * step <= t) {
      const int p = t - k * step;
      rb[i] = __ldg(reinterpret_cast<const float4*>(a.G + ((int64_t)(k * NDEC + d) * a.tc + p) * a.ldg) + c4);
    }
  }
}

// chunks [I0, I0 + HCHUNKS) of the loaded B rows, split into hi/lo planes, into one stage
template <int NDEC, int I0>
__device__ __forceinline__ void mask_store_b(uint8_t* sB, int ptid, const float4 (&rb)[MaskTile<NDEC>::HCHUNKS]) {
  using MT = MaskTile<NDEC>;
#pragma unroll
  for (int i = 0; i < MT::HCHUNKS; ++i) {
    const int idx = (I0 + i) * MT_PRODUCER + ptid, r = idx >> 4, c4 = idx & 15;
    float h[4], l[4];
    split_tf32(rb[i].x, h[0], l[0]); split_tf32(rb[i].y, h[1], l[1]);
    split_tf32(rb[i].z, h[2], l[2]); split_tf32(rb[i].w, h[3], l[3]);
    const uint32_t off = (c4 >> 3) * MT::B_SUB + tile_off(r, c4 & 7);
    *reinterpret_cast<float4*>(sB + off) = make_float4(h[0], h[1], h[2], h[3]);
    *reinterpret_cast<float4*>(sB + 2 * MT::B_SUB + off) = make_float4(l[0], l[1], l[2], l[3]);
  }
}

// the Nyquist bin's GEMM value of every column of chunks [I0, I0 + HCHUNKS) from the loaded fp32 B rows: each thread
// an FMA chain over its 4 of the 50 k-values (wn = W1t[k][F - 1]), then a fixed xor tree over the 16 threads of the row
template <int NDEC, int I0>
__device__ __forceinline__ void mask_nyquist_dots(const float4 (&rb)[MaskTile<NDEC>::HCHUNKS], const float (&wn)[4], int ptid,
                                                  float* nyq) {
  using MT = MaskTile<NDEC>;
  const int c4 = ptid & 15;
#pragma unroll
  for (int i = 0; i < MT::HCHUNKS; ++i) {
    float d = rb[i].x * wn[0];
    d = fmaf(rb[i].y, wn[1], d);
    if (c4 < 12) {   // k = 50, 51 of the last chunk are padding
      d = fmaf(rb[i].z, wn[2], d);
      d = fmaf(rb[i].w, wn[3], d);
    }
    d += __shfl_xor_sync(0xffffffffu, d, 8);
    d += __shfl_xor_sync(0xffffffffu, d, 4);
    d += __shfl_xor_sync(0xffffffffu, d, 2);
    d += __shfl_xor_sync(0xffffffffu, d, 1);
    if (c4 == 0) nyq[8 * (I0 + i) + (ptid >> 4)] = d;
  }
}

// one patch slot of the cross-fade: bias + ReLU + soft ratio mask, then mm <- down * mm + up * mask with
// c = (up, down, up/4, -) of (frame, slot) (dsd_mask_tables_kernel).  y3 is the 4th source's GEMM value (DSD100:
// decoder 2 again, separate_dsd.py:228).  The tensor-core bins and the Nyquist bin share it.
template <int NDEC>
__device__ __forceinline__ void mask_slot(const float4 c, float y0, float y1, float y2, float y3, float bo0, float bo1, float bo2,
                                          float bo3, bool first, float (&mm)[4]) {
  const float p0 = fmaxf(y0 + bo0, 0.f);
  const float p1 = fmaxf(y1 + bo1, 0.f);
  const float p2 = fmaxf(y2 + bo2, 0.f);
  const float p3 = fmaxf(y3 + bo3, 0.f);
  const float tot = (p0 + p1) + (p2 + p3);
  const bool pos = tot > MASK_TOT_MIN;
  float rc;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(rc) : "f"(tot));
  const float r = pos ? c.x * rc : 0.f;             // up * mask = p * (up / tot)
  const float q = (pos || NDEC == 4) ? 0.f : c.z;   // all-zero bin: 1/4 each (DSD100 rule); 0 (ILD rule)
  mm[0] = fmaf(c.y, first ? 0.f : mm[0], fmaf(p0, r, q));
  mm[1] = fmaf(c.y, first ? 0.f : mm[1], fmaf(p1, r, q));
  mm[2] = fmaf(c.y, first ? 0.f : mm[2], fmaf(p2, r, q));
  mm[3] = fmaf(c.y, first ? 0.f : mm[3], fmaf(p3, r, q));
}

// the Nyquist bin of frame t from the producer's dot products of its group (f = frame in the group, xf = the group's
// fade-table entries); MASKS: the masks themselves to M (source s at M + s * src_stride), no X read
template <int NDEC, bool MASKS>
__device__ __forceinline__ void mask_nyquist_epilogue(const DsdMaskArgs& a, float* M, const float4* xf, int t, int f, const float* nyq,
                                                      float bo0, float bo1, float bo2, float bo3) {
  using MT = MaskTile<NDEC>;
  if (t >= a.T) return;
  float mm[4];
#pragma unroll
  for (int j = 0; j < MT_SLOTS; ++j) {
    const float4 c = xf[f * MT_SLOTS + j];
    mask_slot<NDEC>(c, nyq[MT::col(f, NDEC * j + 0)], nyq[MT::col(f, NDEC * j + 1)], nyq[MT::col(f, NDEC * j + 2)],
                    nyq[MT::col(f, NDEC * j + (NDEC == 3 ? 1 : 3))], bo0, bo1, bo2, bo3, j == 0, mm);
  }
  const int bin = a.F - 1;
  if constexpr (MASKS) {
    const int64_t o = (int64_t)t * a.ldf + bin;
#pragma unroll
    for (int s = 0; s < 4; ++s) M[o + s * a.src_stride] = mm[s];
  } else {
    const int64_t o = (int64_t)t * a.ldf + bin;
    const float2 xx = a.X[o];
    a.S[o] = make_float2(mm[0] * xx.x, mm[0] * xx.y);
    a.S[o + a.src_stride] = make_float2(mm[1] * xx.x, mm[1] * xx.y);
    a.S[o + 2 * a.src_stride] = make_float2(mm[2] * xx.x, mm[2] * xx.y);
    a.S[o + 3 * a.src_stride] = make_float2(mm[3] * xx.x, mm[3] * xx.y);
  }
}

// nyq_tiles > 0: the tiles cover bins [0, F - 1) and the CTA whose range holds item (g, tile = g % nyq_tiles) also
// computes bin F - 1 of group g on the producer; 0: the tiles cover all F bins.
// MASKS: the cross-faded masks themselves -- the fp32 values the other mode multiplies by X -- go to M, source s at
// M + s * src_stride; X and S are not touched.
template <int NDEC, bool MASKS>
__global__ void __launch_bounds__(MT_THREADS, 1)
dsd_mask_tc_kernel(const DsdMaskArgs a, float* __restrict__ M, const float4* __restrict__ xtab, const uint8_t* __restrict__ aimg,
                   int m_tiles, int num_items, int nyq_tiles) {
  using MT = MaskTile<NDEC>;
  constexpr int FRAMES = MT::FRAMES, TF = MT::TFRAMES;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  __shared__ uint64_t afull[2], aempty[2], bfull, bempty;
  uint8_t* smem = align1024(smem_raw);
  uint8_t* sA = smem;                       // two stages of MT_A_BYTES
  uint8_t* sB = smem + 2 * MT_A_BYTES;      // one stage of MT::B_BYTES
  float* sNyq = reinterpret_cast<float*>(sB + MT::B_BYTES);       // two buffers of MT::COLS
  float4* sXf = reinterpret_cast<float4*>(sNyq + 2 * MT::COLS);   // fade-table entries of the CTA's i-th group at i % 2

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wg = warp >> 2, wq = warp & 3;
  // work items w = group * m_tiles + tile; this CTA's share [w_begin, w_end) differs from the others' by at most one
  const int w_begin = (int)((int64_t)blockIdx.x * num_items / gridDim.x);
  const int w_end = (int)((int64_t)(blockIdx.x + 1) * num_items / gridDim.x);
  const float bo0 = __ldg(a.bout + 0), bo1 = __ldg(a.bout + 1), bo2 = __ldg(a.bout + 2), bo3 = __ldg(a.bout + 3);
  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      mbar_init(&afull[s], 1);                     // the producer's arrival with the copy's byte count
      mbar_init(&aempty[s], MT_CONSUMERS / 32);    // every consumer warp, once its products on the stage are complete
    }
    mbar_init(&bfull, MT_PRODUCER);                // every producer thread, after its stores
    mbar_init(&bempty, MT_CONSUMERS / 32);         // every consumer warp, once its products of the group's last item are complete
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 2) {
    // ---- producer: A of item w into stage (w - w_begin) % 2 once the consumers have released it; the B rows of a
    //      new group into the B stage once the consumers' products of the previous group are complete
    const int ptid = tid - MT_CONSUMERS;
    float wn[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int c = 4 * (ptid & 15) + i;
      wn[i] = (nyq_tiles > 0 && c < MT_C1) ? __ldg(a.W1t + (int64_t)c * a.ldw + a.F - 1) : 0.f;
    }
    // the next group's loads are in flight while the current group's tiles run
    constexpr int H = MT::HCHUNKS;
    float4 r0[H], r1[H], xf = make_float4(0.f, 0.f, 0.f, 0.f);
    const bool xf_thread = ptid < MT::XF;
    if (w_begin < w_end) {
      const int g = w_begin / m_tiles;
      mask_load_b<NDEC, 0>(a, g, ptid, r0);
      mask_load_b<NDEC, H>(a, g, ptid, r1);
      if (xf_thread) xf = __ldg(xtab + (int64_t)g * MT::XF + ptid);
    }
    int nb = 0, gi = -1;
    for (int w = w_begin, it = 0; w < w_end; ++w, ++it) {
      const int s = it & 1;
      if (ptid == 0) {
        if (it >= 2) mbar_wait_relaxed(&aempty[s], ((it >> 1) - 1) & 1);
        mbar_arrive_expect_tx(&afull[s], MT_A_BYTES);
        bulk_copy_g2s(sA + s * MT_A_BYTES, aimg + (int64_t)(w % m_tiles) * MT_A_BYTES, MT_A_BYTES, &afull[s]);
      }
      if (w != w_begin && w % m_tiles != 0) continue;   // the group's B rows are staged
      ++gi;
      const int g = w / m_tiles, gn = g + 1;
      const bool more = (int64_t)gn * m_tiles < w_end;
      const int w_nyq = g * m_tiles + (nyq_tiles > 0 ? g % nyq_tiles : 0);
      const bool nyq_group = nyq_tiles > 0 && w_nyq >= w_begin && w_nyq < w_end;
      float* nq = sNyq + nb * MT::COLS;   // buffer nb was last read before the previous Nyquist group's barrier
      if (gi >= 1) mbar_wait_relaxed(&bempty, (gi - 1) & 1);
      mask_store_b<NDEC, 0>(sB, ptid, r0);
      if (nyq_group) mask_nyquist_dots<NDEC, 0>(r0, wn, ptid, nq);
      if (more) mask_load_b<NDEC, 0>(a, gn, ptid, r0);
      mask_store_b<NDEC, H>(sB, ptid, r1);
      if (nyq_group) mask_nyquist_dots<NDEC, H>(r1, wn, ptid, nq);
      if (more) mask_load_b<NDEC, H>(a, gn, ptid, r1);
      // the consumers' epilogues of group gi - 2, the last readers of this ring slot, precede their release of group gi - 1
      if (xf_thread) sXf[(gi & 1) * MT::XF + ptid] = xf;
      if (xf_thread && more) xf = __ldg(xtab + (int64_t)gn * MT::XF + ptid);
      fence_proxy_async();
      mbar_arrive(&bfull);
      if (nyq_group) {
        nb ^= 1;
        bar_sync(MT_BAR_PROD, MT_PRODUCER);
        if (ptid < FRAMES)
          mask_nyquist_epilogue<NDEC, MASKS>(a, M, sXf + (gi & 1) * MT::XF, g * FRAMES + ptid, ptid, nq, bo0, bo1, bo2, bo3);
      }
    }
    return;
  }

  // ---- consumers, phase-shifted by half an item: consumer 1 issues its products of item w while consumer 0 runs
  //      the epilogue of item w, and consumer 0 issues item w + 1 while consumer 1 runs the epilogue of item w
  const int row0 = wg * 64 + wq * 16 + (lane >> 2);   // tile rows row0 and row0 + 8 are this thread's bins
  int gi = -1;
  for (int w = w_begin, it = 0; w < w_end; ++w, ++it) {
    const int s = it & 1, g = w / m_tiles, tile = w - g * m_tiles;
    if (w == w_begin || tile == 0) ++gi;
    const bool group_end = w + 1 == w_end || tile == m_tiles - 1;
    mbar_wait(&afull[s], (it >> 1) & 1);
    mbar_wait(&bfull, gi & 1);
    if (wg == 1) bar_sync(MT_BAR_TURN1, MT_CONSUMERS);
    else if (it > 0) bar_sync(MT_BAR_TURN0, MT_CONSUMERS);

    // ---- MMAs: bins [64 wg, 64 wg + 64) x MT::COLS columns, the 14 small correction products first, then the 7
    //      main ones, so the truncating accumulation sees only 7 large addends
    float acc[MT::COLS / 2];
    {
      const uint32_t a_hi = smem_u32(sA + s * MT_A_BYTES) + wg * 64 * ROW_BYTES, a_lo = a_hi + 2 * MT_A_SUB;
      const uint32_t b_hi = smem_u32(sB), b_lo = b_hi + 2 * MT::B_SUB;
      wgmma_fence();
#pragma unroll
      for (int j = 0; j < MT_KSTEPS; ++j) {
        const uint32_t ao = (j >> 2) * MT_A_SUB + KSTEP_BYTES * (j & 3), bo = (j >> 2) * MT::B_SUB + KSTEP_BYTES * (j & 3);
        wgmma_tf32<MT::COLS>(acc, make_desc(a_lo + ao), make_desc(b_hi + bo), j != 0);
      }
#pragma unroll
      for (int j = 0; j < MT_KSTEPS; ++j) {
        const uint32_t ao = (j >> 2) * MT_A_SUB + KSTEP_BYTES * (j & 3), bo = (j >> 2) * MT::B_SUB + KSTEP_BYTES * (j & 3);
        wgmma_tf32<MT::COLS>(acc, make_desc(a_hi + ao), make_desc(b_lo + bo), 1);
      }
#pragma unroll
      for (int j = 0; j < MT_KSTEPS; ++j) {
        const uint32_t ao = (j >> 2) * MT_A_SUB + KSTEP_BYTES * (j & 3), bo = (j >> 2) * MT::B_SUB + KSTEP_BYTES * (j & 3);
        wgmma_tf32<MT::COLS>(acc, make_desc(a_hi + ao), make_desc(b_hi + bo), 1);
      }
      wgmma_commit();
    }
    if (wg == 0) bar_arrive(MT_BAR_TURN1, MT_CONSUMERS);
    else if (w + 1 < w_end) bar_arrive(MT_BAR_TURN0, MT_CONSUMERS);

    // ---- while they run: this item's X
    int bin[2];
    bool bok[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      bin[i] = tile * MT_BINS + row0 + 8 * i;
      bok[i] = bin[i] < a.F;
    }
    float2 x[TF][2];
    if constexpr (!MASKS) {
#pragma unroll
      for (int e = 0; e < TF; ++e) {
        const int t = g * FRAMES + MT::thread_frame(lane, e);
#pragma unroll
        for (int i = 0; i < 2; ++i)
          x[e][i] = (bok[i] && t < a.T) ? a.X[(int64_t)t * a.ldf + bin[i]] : make_float2(0.f, 0.f);
      }
    }
    wgmma_wait<0>();
    wgmma_fence_acc(acc);
    if (lane == 0) {
      mbar_arrive(&aempty[s]);
      if (group_end) mbar_arrive(&bempty);
    }

    // ---- epilogue per (bin, frame): bias + ReLU + ratio mask + sequential cross-fade + .X
    float m[TF][2][4];   // cross-faded masks of the 4 sources
#pragma unroll
    for (int e = 0; e < TF; ++e) {
      const float4* xf = sXf + (gi & 1) * MT::XF + MT::thread_frame(lane, e) * MT_SLOTS;   // the frame's (up, down, up/4, -)
#pragma unroll
      for (int i = 0; i < 2; ++i) {
#pragma unroll
        for (int j = 0; j < MT_SLOTS; ++j) {
          const float4 c = xf[j];
          mask_slot<NDEC>(c, acc[MT::acc(i, e, NDEC * j + 0)], acc[MT::acc(i, e, NDEC * j + 1)], acc[MT::acc(i, e, NDEC * j + 2)],
                          acc[MT::acc(i, e, NDEC * j + (NDEC == 3 ? 1 : 3))], bo0, bo1, bo2, bo3, j == 0, m[e][i]);
        }
      }
    }
    if constexpr (MASKS) {   // source s at M + s * src_stride
#pragma unroll
      for (int e = 0; e < TF; ++e) {
        const int t = g * FRAMES + MT::thread_frame(lane, e);
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          if (bok[i] && t < a.T) {
            const int64_t o = (int64_t)t * a.ldf + bin[i];
#pragma unroll
            for (int s = 0; s < 4; ++s) M[o + s * a.src_stride] = m[e][i][s];
          }
        }
      }
    } else {   // source s at S + s * src_stride
#pragma unroll
      for (int e = 0; e < TF; ++e) {
        const int t = g * FRAMES + MT::thread_frame(lane, e);
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          if (bok[i] && t < a.T) {
            const float2 xx = x[e][i];
            const float* mm = m[e][i];
            const int64_t o = (int64_t)t * a.ldf + bin[i];
            a.S[o] = make_float2(mm[0] * xx.x, mm[0] * xx.y);
            a.S[o + a.src_stride] = make_float2(mm[1] * xx.x, mm[1] * xx.y);
            a.S[o + 2 * a.src_stride] = make_float2(mm[2] * xx.x, mm[2] * xx.y);
            a.S[o + 3 * a.src_stride] = make_float2(mm[3] * xx.x, mm[3] * xx.y);
          }
        }
      }
    }
  }
}

// Two tables per launch, one thread per entry of either:
// - (up, down, up/4, 0) of every (frame, patch slot): the sequential cross-fade of overlapadd_multi
//   (separate_dsd.py:139-169) as a per-slot recurrence; frames >= T (padding to whole groups) and slots
//   without a patch get (0, 1): they leave the accumulated masks untouched;
// - the A operand of every 128-bin tile as the kernel's shared-memory image: four 16 KB planes (hi k0-31, hi k32-63,
//   lo k0-31, lo k32-63) of 128 rows, 128B-swizzled (tile_off), split by split_tf32, zero for k >= 50 and bins >= F;
//   thread = (k chunk, bin row) so the reads of W1t[c][bin] are coalesced over bins.
__global__ void dsd_mask_tables_kernel(float4* __restrict__ tab, int T, int Tpad, int P, int tc, int overlap,
                                       const float* __restrict__ W1t, int ldw, int F, int m_tiles, uint8_t* __restrict__ aimg) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < Tpad * MT_SLOTS) {
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
  if (i < m_tiles * 16 * MT_BINS) {
    const int tile = i / (16 * MT_BINS), c4 = (i / MT_BINS) & 15, r = i & (MT_BINS - 1);
    const int b = tile * MT_BINS + r;
    float hi[4], lo[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int c = 4 * c4 + q;
      split_tf32((b < F && c < MT_C1) ? __ldg(W1t + (int64_t)c * ldw + b) : 0.f, hi[q], lo[q]);
    }
    uint8_t* img = aimg + (int64_t)tile * MT_A_BYTES + (c4 >> 3) * MT_A_SUB + tile_off(r, c4 & 7);
    *reinterpret_cast<float4*>(img) = make_float4(hi[0], hi[1], hi[2], hi[3]);
    *reinterpret_cast<float4*>(img + 2 * MT_A_SUB) = make_float4(lo[0], lo[1], lo[2], lo[3]);
  }
}

bool dsd_mask_tc_supported(const DsdMaskArgs& a) {
  const int step = a.tc - a.overlap;
  return step > 0 && (a.ndec == 3 || a.ndec == 4) && (a.tc + step - 1) / step <= MT_SLOTS && a.ldg % 4 == 0 && a.ldg >= 52 &&
         ((uintptr_t)a.G % 16 == 0);
}

// F = 128 m + 1 (the DSD nets' F = N / 2 + 1) with m >= 1: m tiles, and the producer computes the Nyquist bin, which
// would otherwise take a tile of its own; any other F: ceil(F / 128) tiles
template <int NDEC, bool MASKS>
static int launch_dsd_mask_tc_t(dcs_ctx* ctx, const DsdMaskArgs& a, float* M, cudaStream_t st) {
  using MT = MaskTile<NDEC>;
  DCS_TRY(ensure_smem_attr(dsd_mask_tc_kernel<NDEC, MASKS>, MT::SMEM));
  const bool nyq = a.F > MT_BINS && (a.F - 1) % MT_BINS == 0;
  const int m_tiles = nyq ? (a.F - 1) / MT_BINS : (a.F + MT_BINS - 1) / MT_BINS;
  const int num_groups = (a.T + MT::FRAMES - 1) / MT::FRAMES;
  const int num_items = m_tiles * num_groups;
  const int ctas = std::min(ctx->num_sms, num_items);
  const int Tpad = num_groups * MT::FRAMES;
  DCS_TRY(ctx->net[NET_XTAB].ensure((size_t)Tpad * MT_SLOTS * sizeof(float4), st));
  DCS_TRY(ctx->net[NET_AIMG].ensure((size_t)m_tiles * MT_A_BYTES, st));
  float4* xtab = ctx->net[NET_XTAB].as<float4>();
  uint8_t* aimg = ctx->net[NET_AIMG].as<uint8_t>();
  const int64_t nthreads = std::max((int64_t)Tpad * MT_SLOTS, (int64_t)m_tiles * 16 * MT_BINS);
  dsd_mask_tables_kernel<<<(unsigned)ceil_div64(nthreads, 256), 256, 0, st>>>(xtab, a.T, Tpad, a.P, a.tc, a.overlap, a.W1t, a.ldw,
                                                                              a.F, m_tiles, aimg);
  DCS_CHECK_LAUNCH();
  ctx->launches++;
  dsd_mask_tc_kernel<NDEC, MASKS><<<(unsigned)ctas, MT_THREADS, MT::SMEM, st>>>(a, M, xtab, aimg, m_tiles, num_items,
                                                                               nyq ? m_tiles : 0);
  DCS_CHECK_LAUNCH();
  ctx->launches++;
  return DCS_OK;
}

int launch_dsd_mask_tc(dcs_ctx* ctx, const DsdMaskArgs& a, cudaStream_t st, float* M) {
  if (a.T <= 0) return DCS_OK;
  DCS_REQUIRE(dsd_mask_tc_supported(a), "dsd_mask_tc: unsupported shape");
  if (M) return a.ndec == 4 ? launch_dsd_mask_tc_t<4, true>(ctx, a, M, st) : launch_dsd_mask_tc_t<3, true>(ctx, a, M, st);
  return a.ndec == 4 ? launch_dsd_mask_tc_t<4, false>(ctx, a, nullptr, st) : launch_dsd_mask_tc_t<3, false>(ctx, a, nullptr, st);
}

}  // namespace dcs
