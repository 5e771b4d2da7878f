// sconv_tc.cu -- K3s on the tensor cores: InverseLayer(pool) + InverseLayer(conv1) (transposed strided
// convolution over frequency) + ConcatLayer + bias + ReLU + soft ratio mask + patch cross-fade + phase for
// the strided-conv1 networks -- iKala (examples/ikala/separate_ikala.py:183-217), Bach10
// (examples/bach10/separate_bach10.py:207-266), score-informed Bach10
// (examples/bach10_scoreinformed/trainCNNrwc.py:189,248-263).  Same math as sconv.cu's FFMA kernel
// (which stays as the cross-check, DCS_DEBUG_SIMT_GEMM=1).
//
// The transposed strided convolution  Y[STRIDE*m + r] = sum_{dd < ND, f < 30} Gu[m - dd][f] * w[dd][f][r]
// is computed in two steps:
//   1. GEMM on wgmma (fp32-accurate 3xTF32):  Z[j][(dd, r)] = sum_f Gu[j][f] * w[dd][f][r]
//        M = 128 staged positions j (one 64-row half per warpgroup), K = 32 channels (30 + 2 zero),
//        N = NB = 32 columns per filter bank (ND*STRIDE <= 32); A = the activation tile [128 j][32 f] of one
//        decoder -- for the max-pool net gathered through the tie bits of the forward pass (Theano MaxPoolGrad
//        routing) -- split into hi / lo planes; B = the filter bank(s), split once per CTA.
//   2. the accumulators go to a padded [row][column] shared tile; the epilogue thread of output m gathers the
//        ND taps  Y[m][r] = sum_dd Z[m - dd][(dd, r)]  from its neighbours' rows (conflict-free), then bias +
//        ReLU + ratio mask over the sources + the sequential cross-fade recurrence in registers; the masked
//        spectra leave as STRIDE consecutive bins per output position.
// A patch slot's decoders (Bach10: 4, iKala: 2) -- or, score-informed, the 4 filter banks of decoder 1 -- give
// the slot's NSRC x 32 accumulator columns.  CTAs are persistent over a range of frames of one tile of
// 128 - (ND-1) output positions; per slot: operand stores | MMAs | accumulator tile | epilogue, with the global
// loads of the next slot's activations issued before the MMAs of the current one.
#include "common.cuh"
#include "tc.cuh"

namespace dcs {

using namespace tc;

constexpr int ST_ROWS = 128;
constexpr int ST_THREADS = 256;                    // two warpgroups
constexpr int ST_A_TILE = ST_ROWS * ROW_BYTES;     // 16 KB: [128][32] fp32
constexpr int ST_ZP = 129;                         // row pitch of the accumulator tile (floats)

template <int STRIDE, int ND, int NSRC, int NDEC, int NW>
struct SconvTile {
  static constexpr int OUT = ST_ROWS - (ND - 1);     // output positions per tile
  static constexpr int NB = NW * 32;                 // GEMM columns per activation tile
  static constexpr int ITEMS = NDEC;                 // activation tiles per patch slot
  static constexpr int B_PLANE = NB * ROW_BYTES;
  static constexpr int OFF_B = ITEMS * 2 * ST_A_TILE;
  static constexpr int OFF_Z = OFF_B + 2 * B_PLANE;
  static constexpr int SMEM = OFF_Z + ST_ROWS * ST_ZP * 4 + 1024;
  static constexpr int CHUNKS = ITEMS * ST_ROWS * 8 / ST_THREADS;   // float4 of activations per thread and slot
  static_assert(ITEMS * NB == NSRC * 32, "one slot's accumulator columns = 32 per source");
  static_assert(NW == 1 ? NSRC == NDEC : (NDEC == 1 && NSRC == NW), "sources = decoders, or = filter banks of one decoder");
  static_assert(ND * STRIDE <= 32, "taps x stride must fit one 32-column bank");
  static_assert(SMEM <= 227 * 1024, "shared memory");
};

__device__ __forceinline__ void slot_range(int t, int tc, int step, int P, int& k_lo, int& k_hi) {
  k_hi = t / step;
  if (k_hi > P - 1) k_hi = P - 1;
  k_lo = t - tc + 1;
  k_lo = k_lo > 0 ? (k_lo + step - 1) / step : 0;
}

// activation chunk u of slot (t, k): item d, staged row jl, 16-byte channel chunk c4 (k counts from G's first patch).
// Un-pooled nets: G row ((k*NDEC + d)*tc + p) at position j; max-pool net: InverseLayer(pool) -- position j receives G[j / POOL]
// where the forward pass had its window maximum (every tied position does), else 0.  Outside the axis: 0.
template <int POOL>
__device__ __forceinline__ float4 sconv_load(const SconvMaskArgs& a, int t, int k, int p, int d, int ndec, int j, int c4) {
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (j < 0) return v;
  const int64_t row = (int64_t)(k * ndec + d) * a.tc + p;
  if (POOL == 0) {
    if (j < a.J) v = __ldg(reinterpret_cast<const float4*>(a.G + (row * a.J + j) * 32) + c4);
  } else {
    constexpr int PW = POOL ? POOL : 1;
    const int jp = j / PW, rr = j - jp * PW;
    if (jp < a.WP) {
      const uchar4 bits = *reinterpret_cast<const uchar4*>(a.tie + ((int64_t)t * a.WP + jp) * 32 + 4 * c4);
      const float4 g = __ldg(reinterpret_cast<const float4*>(a.G + (row * a.WP + jp) * 32) + c4);
      v.x = ((bits.x >> rr) & 1) ? g.x : 0.f;
      v.y = ((bits.y >> rr) & 1) ? g.y : 0.f;
      v.z = ((bits.z >> rr) & 1) ? g.z : 0.f;
      v.w = ((bits.w >> rr) & 1) ? g.w : 0.f;
    }
  }
  return v;
}

// CHUNK: G holds patches a.p_base.. and the frames [a.t0, a.t1) are written (one decoder chunk of the 1x1 score net);
// otherwise G holds every patch and all a.T frames are written.  MASKS: the blended masks themselves go to M (source s at
// M + s * src_stride); X and S are not touched
template <int STRIDE, int ND, int NSRC, int NDEC, int RULE, int POOL, int NW, bool CHUNK = false, bool MASKS = false>
__global__ void __launch_bounds__(ST_THREADS, 1)
sconv_mask_tc_kernel(const SconvMaskArgs a, float* __restrict__ M, int frames_per_cta) {
  using TL = SconvTile<STRIDE, ND, NSRC, NDEC, NW>;
  constexpr int OUT = TL::OUT, NB = TL::NB, ITEMS = TL::ITEMS, CHUNKS = TL::CHUNKS;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  uint8_t* sA = smem;                                   // item d: hi at d*2*TILE, lo at d*2*TILE + TILE
  uint8_t* sB = smem + TL::OFF_B;                       // hi plane, lo plane
  float* Zs = reinterpret_cast<float*>(smem + TL::OFF_Z);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wg = warp >> 2, wq = warp & 3;
  const int m0 = blockIdx.x * OUT;
  const int j_start = m0 - (ND - 1);
  const int t_begin = (CHUNK ? a.t0 : 0) + blockIdx.y * frames_per_cta;
  const int t_end = min(CHUNK ? a.t1 : a.T, t_begin + frames_per_cta);
  const int p_base = CHUNK ? a.p_base : 0;
  const int step = a.tc - a.overlap;

  // filter banks: B[c = o*32 + dd*STRIDE + r][f] = w[o][dd][f][r] (a.W: float4 [NW][ND][32], .xyzw = r), hi / lo planes
  for (int i = tid; i < NB * 8; i += ST_THREADS) {
    const int c = i >> 3, c4 = i & 7;
    const int o = c >> 5, cc = c & 31, dd = cc / STRIDE, r = cc - dd * STRIDE;
    float hi[4] = {0.f, 0.f, 0.f, 0.f}, lo[4] = {0.f, 0.f, 0.f, 0.f};
    if (dd < ND) {
#pragma unroll
      for (int q = 0; q < 4; ++q) split_tf32(__ldg(a.W + ((int64_t)((o * ND + dd) * 32 + 4 * c4 + q)) * 4 + r), hi[q], lo[q]);
    }
    const uint32_t off = tile_off(c, c4);
    *reinterpret_cast<float4*>(sB + off) = make_float4(hi[0], hi[1], hi[2], hi[3]);
    *reinterpret_cast<float4*>(sB + TL::B_PLANE + off) = make_float4(lo[0], lo[1], lo[2], lo[3]);
  }

  // epilogue ownership: staged row / output position i = tid % 128; the STRIDE sub-bins r with r % 2 == half
  const int i = tid & (ST_ROWS - 1), half = tid >> 7;
  const int m = m0 + i;
  const int mtot = (a.F + STRIDE - 1) / STRIDE;
  const bool mok = i < OUT && m < mtot;
  float bo[NSRC];
#pragma unroll
  for (int o = 0; o < NSRC; ++o) bo[o] = __ldg(a.bout + o);
  const float inv_ov1 = a.overlap > 1 ? 1.0f / (float)(a.overlap - 1) : 0.f;

  // frames no patch covers (past the last patch of the standalone patcher) get zero spectra
  auto zero_frame = [&](int tt) {
    if (!mok) return;
#pragma unroll
    for (int r = 0; r < STRIDE; ++r) {
      const int b = STRIDE * m + r;
      if ((r & 1) == half && b < a.F)
#pragma unroll
        for (int s = 0; s < NSRC; ++s) {
          if (MASKS) M[(int64_t)tt * a.ldf + b + s * a.src_stride] = 0.f;
          else a.S[(int64_t)tt * a.ldf + b + s * a.src_stride] = make_float2(0.f, 0.f);
        }
    }
  };
  // first slot at or after frame tt: (tt, k_lo .. k_hi), or tt = t_end
  auto first_slot = [&](int& tt, int& lo, int& hi) {
    for (; tt < t_end; ++tt) {
      slot_range(tt, a.tc, step, a.P, lo, hi);
      if (lo <= hi) return;
      zero_frame(tt);
    }
  };
  // the slots of this CTA's frames as one sequence: (t, k) advances k, then t
  int t = t_begin, k_lo = 0, k_hi = -1;
  first_slot(t, k_lo, k_hi);
  int k = k_lo;
  float4 ra[CHUNKS];
  auto load_slot = [&](int tt, int kk) {
    const int p = tt - kk * step;
#pragma unroll
    for (int u = 0; u < CHUNKS; ++u) {
      const int idx = u * ST_THREADS + tid, c4 = idx & 7, jl = (idx >> 3) & (ST_ROWS - 1), d = idx >> 10;
      ra[u] = sconv_load<POOL>(a, tt, kk - p_base, p, d, NDEC, j_start + jl, c4);
    }
  };
  if (t < t_end) load_slot(t, k);
  float macc[NSRC][STRIDE];
  while (t < t_end) {
    if (k == k_lo) {
#pragma unroll
      for (int o = 0; o < NSRC; ++o)
#pragma unroll
        for (int r = 0; r < STRIDE; ++r) macc[o][r] = 0.f;
    }
    const int p = t - k * step;
    // ---- activation planes of this slot (the previous slot's MMAs and Z reads finished: barriers below)
#pragma unroll
    for (int u = 0; u < CHUNKS; ++u) {
      const int idx = u * ST_THREADS + tid, c4 = idx & 7, jl = (idx >> 3) & (ST_ROWS - 1), d = idx >> 10;
      float h[4], l[4];
      split_tf32(ra[u].x, h[0], l[0]); split_tf32(ra[u].y, h[1], l[1]);
      split_tf32(ra[u].z, h[2], l[2]); split_tf32(ra[u].w, h[3], l[3]);
      const uint32_t off = d * 2 * ST_A_TILE + tile_off(jl, c4);
      *reinterpret_cast<float4*>(sA + off) = make_float4(h[0], h[1], h[2], h[3]);
      *reinterpret_cast<float4*>(sA + ST_A_TILE + off) = make_float4(l[0], l[1], l[2], l[3]);
    }
    fence_proxy_async();
    __syncthreads();
    // next slot of the sequence; its global loads are in flight during the MMAs and the epilogue
    int tn = t, kn = k + 1, kn_lo = k_lo, kn_hi = k_hi;
    if (kn > k_hi) {
      ++tn;
      first_slot(tn, kn_lo, kn_hi);
      kn = kn_lo;
    }
    if (tn < t_end) load_slot(tn, kn);

    // ---- MMAs: warpgroup wg computes staged rows [64 wg, 64 wg + 64) x (ITEMS x NB) columns
    {
      float acc[ITEMS][NB / 2];
      const uint32_t b_hi = smem_u32(sB), b_lo = b_hi + TL::B_PLANE;
      wgmma_fence();
#pragma unroll
      for (int d = 0; d < ITEMS; ++d) {
        const uint32_t a_hi = smem_u32(sA + d * 2 * ST_A_TILE) + wg * 64 * ROW_BYTES, a_lo = a_hi + ST_A_TILE;
        // corrections first (tiny partial sums), the main product last
#pragma unroll
        for (int j = 0; j < 4; ++j) wgmma_tf32<NB>(acc[d], make_desc(a_hi + KSTEP_BYTES * j), make_desc(b_lo + KSTEP_BYTES * j), j != 0);
#pragma unroll
        for (int j = 0; j < 4; ++j) wgmma_tf32<NB>(acc[d], make_desc(a_lo + KSTEP_BYTES * j), make_desc(b_hi + KSTEP_BYTES * j), 1);
#pragma unroll
        for (int j = 0; j < 4; ++j) wgmma_tf32<NB>(acc[d], make_desc(a_hi + KSTEP_BYTES * j), make_desc(b_hi + KSTEP_BYTES * j), 1);
      }
      wgmma_commit();
      wgmma_wait_all();
      // fragment -> Zs[row][column], column = d*NB + n (tc.cuh: d[4j + 2i + e] = D[16 wq + lane/4 + 8i][8j + 2(lane%4) + e])
#pragma unroll
      for (int d = 0; d < ITEMS; ++d)
#pragma unroll
        for (int j = 0; j < NB / 8; ++j)
#pragma unroll
          for (int ii = 0; ii < 2; ++ii)
#pragma unroll
            for (int e = 0; e < 2; ++e)
              Zs[(wg * 64 + wq * 16 + (lane >> 2) + 8 * ii) * ST_ZP + d * NB + 8 * j + 2 * (lane & 3) + e] = acc[d][4 * j + 2 * ii + e];
    }
    __syncthreads();

    // ---- epilogue: Y[m][r] = sum_dd Z[m - dd][(dd, r)] (staged row of position m - dd is i + ND-1 - dd), then
    // bias + ReLU + ratio mask across the sources + sequential cross-fade (separate_bach10.py:245-266,
    // separate_ikala.py:207-217; overlapadd_multi separate_dsd.py:139-169)
    const float up = k == k_lo ? 1.f : (float)p * inv_ov1;
    const float down = k == k_lo ? 0.f : (float)(a.overlap - 1 - p) * inv_ov1;
    if (i < OUT) {
#pragma unroll
      for (int r = 0; r < STRIDE; ++r) {
        if ((r & 1) != half) continue;
        float pv[NSRC], tot = 0.f;
#pragma unroll
        for (int o = 0; o < NSRC; ++o) {
          float y = 0.f;
#pragma unroll
          for (int dd = 0; dd < ND; ++dd) y += Zs[(i + ND - 1 - dd) * ST_ZP + o * 32 + dd * STRIDE + r];
          pv[o] = fmaxf(y + bo[o], 0.f);
          tot += pv[o];
        }
        const bool pos = tot > MASK_TOT_MIN;
        const float rr = pos ? __fdividef(up, tot) : 0.f;
        const float q = (pos || RULE == 1) ? 0.f : up / (float)NSRC;
#pragma unroll
        for (int o = 0; o < NSRC; ++o) macc[o][r] = fmaf(down, macc[o][r], fmaf(pv[o], rr, q));
      }
    }
    if (k == k_hi && mok) {   // last slot of frame t: the masked spectra of this thread's bins
#pragma unroll
      for (int r = 0; r < STRIDE; ++r) {
        const int b = STRIDE * m + r;
        if (MASKS && (r & 1) == half && b < a.F) {
          const int64_t o = (int64_t)t * a.ldf + b;
#pragma unroll
          for (int s = 0; s < NSRC; ++s) M[o + s * a.src_stride] = macc[s][r];
        } else if ((r & 1) == half && b < a.F) {
          const int64_t o = (int64_t)t * a.ldf + b;
          const float2 x = a.X[o];
#pragma unroll
          for (int s = 0; s < NSRC; ++s) a.S[o + s * a.src_stride] = make_float2(macc[s][r] * x.x, macc[s][r] * x.y);
        }
      }
    }
    t = tn; k = kn; k_lo = kn_lo; k_hi = kn_hi;
  }
}

template <int STRIDE, int ND, int NSRC, int NDEC, int RULE, int POOL, int NW, bool CHUNK = false>
static int launch_sconv_tc_t(dcs_ctx* ctx, const SconvMaskArgs& a, float* M, cudaStream_t st) {
  using TL = SconvTile<STRIDE, ND, NSRC, NDEC, NW>;
  auto kern = M ? sconv_mask_tc_kernel<STRIDE, ND, NSRC, NDEC, RULE, POOL, NW, CHUNK, true>
                : sconv_mask_tc_kernel<STRIDE, ND, NSRC, NDEC, RULE, POOL, NW, CHUNK, false>;
  DCS_TRY(ensure_smem_attr(kern, TL::SMEM));
  const int mtot = (a.F + STRIDE - 1) / STRIDE;
  const int mtiles = (mtot + TL::OUT - 1) / TL::OUT;
  const int nt = a.t1 - a.t0;   // frames this launch writes
  int chunks = ctx->num_sms / mtiles;
  if (chunks < 1) chunks = 1;
  if (chunks > nt) chunks = nt;
  const int fpc = (nt + chunks - 1) / chunks;
  dim3 grid((unsigned)mtiles, (unsigned)((nt + fpc - 1) / fpc));
  kern<<<grid, ST_THREADS, TL::SMEM, st>>>(a, M, fpc);
  DCS_CHECK_LAUNCH();
  ctx->launches++;
  return DCS_OK;
}

bool sconv_mask_tc_supported(const SconvMaskArgs& a) {
  const int step = a.tc - a.overlap;
  return step > 0 && ((uintptr_t)a.G % 16 == 0) && a.t0 >= 0 && a.t0 <= a.t1 && a.t1 <= a.T &&
         (a.arch == DCS_ARCH_BACH10 || a.arch == DCS_ARCH_BACH10_SCORE || a.arch == DCS_ARCH_IKALA || a.arch == DCS_ARCH_IKALA_NOPOOL ||
          a.arch == DCS_ARCH_BACH10_SCORE_1X1);
}

int launch_sconv_mask_tc(dcs_ctx* ctx, const SconvMaskArgs& a, cudaStream_t st, float* M) {
  if (a.T <= 0 || a.t1 <= a.t0) return DCS_OK;
  DCS_REQUIRE(sconv_mask_tc_supported(a), "sconv_mask_tc: unsupported shape");
  if (a.arch == DCS_ARCH_BACH10) return launch_sconv_tc_t<4, 8, 4, 4, 1, 0, 1>(ctx, a, M, st);
  if (a.arch == DCS_ARCH_BACH10_SCORE) return launch_sconv_tc_t<4, 8, 4, 1, 1, 0, 4>(ctx, a, M, st);
  // 1x1 score net: InverseLayer(conv1) of kernel (1,5) stride 2 -- 3 taps per output pair (score1x1.cu)
  if (a.arch == DCS_ARCH_BACH10_SCORE_1X1) return launch_sconv_tc_t<2, 3, 4, 1, 1, 0, 4, true>(ctx, a, M, st);
  if (a.arch == DCS_ARCH_IKALA) return launch_sconv_tc_t<3, 10, 2, 2, 0, 4, 1>(ctx, a, M, st);
  return launch_sconv_tc_t<3, 10, 2, 2, 0, 0, 1>(ctx, a, M, st);
}

}  // namespace dcs
