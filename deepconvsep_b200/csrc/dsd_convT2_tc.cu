// dsd_convT2_tc.cu -- InverseLayer(conv2) of the DSD nets on the tensor cores, built on the layer's own
// structure: the h2 interior rows of one (patch, decoder) pair feed all tc of its output rows, so a block
// of pairs is read from HBM once into shared memory and every GEMM row is a window of it.
//
// GEMM view (D = A * B^T, fp32-accurate 3xTF32, the accumulation plan of gemm_tc.cu):
//   M = (pair, u): 128 rows per work item, Q pairs x U consecutive output positions, pair-major
//   N = 50 filters, padded to 56 (one m64n56k8 per product)
//   K = tap-major, channel pitch 52: k = 52 q + f, K = 52 kh2, in 32-wide stages at absolute multiples of 32
//   A row (pair, u) = the contiguous window of the pair's apad rows starting at row u, i.e. interior float
//       52 (u - (kh2 - 1)) + k; zero outside the interior (the padding rows of apad are never read)
//   B = the tWt2 hi / lo planes (K-major, Kp = 32 ceil(K / 32)), streamed through a ring of swizzled stages
// An item skips the stages outside the union of its U rows' taps; the stages it adds or skips against the
// generic GEMM's tiles are exact zeros for every row, so G is the GEMM path's G as values.
//
// Persistent CTAs, one per SM, each over a contiguous range of items (pair-block-major), 320 threads:
//   - warps 0-7: two consumer warpgroups, one 64-row half of the item each.  Each thread loads its A fragments
//     for a stage from the pair block in shared memory (16 scalar loads, conflict-free: the pair stride is
//     16 floats mod 32 banks), splits them hi / lo in registers, and issues the 12 products of the stage with
//     A from registers.  Epilogue straight from the accumulators into G columns 0..49.
//   - warp 8: the B ring, STAGES deep: cp.async of 28 16-byte pieces per lane and stage; a stage is published
//     (fence.proxy.async + mbarrier arrive) once LAG later stages are in flight.
//   - warp 9: the pair blocks, one bulk copy per pair into a single buffer, when the range enters a new block
//     and the consumers have released the previous one.
#include "common.cuh"
#include "tc.cuh"

namespace dcs {

using namespace tc;

constexpr int CT_C = 50;                     // conv1 = conv2 filters (GEMM N)
constexpr int CT_CP = 52;                    // channel pitch of apad and of K
constexpr int CT_N = 56;                     // N padded to the wgmma width
constexpr int CT_ROWS = 128;                 // GEMM rows per item
constexpr int CT_STAGES = 6;                 // B ring
constexpr int CT_LAG = 4;                    // B stages in flight per producer lane before the oldest is published
constexpr int CT_CONSUMERS = 256;            // warpgroups 0 and 1
constexpr int CT_THREADS = CT_CONSUMERS + 64;   // + the B warp and the activation warp
constexpr int CT_B_PLANE = CT_N * ROW_BYTES;    // 7 KB: one swizzled [56][32] tile
constexpr int CT_B_STAGE = 2 * CT_B_PLANE;      // hi, lo
constexpr int CT_B_PIECES = 2 * CT_N * 8 / 32;  // 16-byte pieces of a stage per producer lane: 28
constexpr int CT_RING = CT_STAGES * CT_B_STAGE;

struct ConvT2Params {
  const float* apad;
  float* G;
  const float* Bhi;
  const float* Blo;
  int Kp, ldg;
  int npairs, tc, kh2, h2;
  int nub;           // u blocks of a pair block: ceil(tc / U)
  int num_items;     // ceil(npairs / Q) * nub
  int pstr;          // floats between two pairs' interiors in shared memory: 52 h2 rounded up to 16 mod 32
};

// floats per pair in shared memory: the interior plus padding to 16 mod 32, so that the two pairs an 8-row
// fragment group touches (U = 4) sit on disjoint banks
static int convT2_pair_stride(int h2) {
  const int n = h2 * CT_CP;
  return n + ((16 - n % 32) + 32) % 32;
}

// stages [kb_lo, kb_hi) of u block ub: the union of the taps q its rows see data through (the clipping rule of
// gemm_tc_kernel, on U rows)
template <int U>
__device__ __forceinline__ void convT2_item_kb(const ConvT2Params& a, int ub, int& kb_lo, int& kb_hi) {
  const int u_min = ub * U, u_max = min(a.tc - 1, u_min + U - 1);
  const int q_lo = max(0, a.kh2 - 1 - u_max), q_hi = min(a.kh2 - 1, a.kh2 + a.h2 - 2 - u_min);
  kb_lo = (CT_CP * q_lo) / KSTAGE;
  kb_hi = (CT_CP * (q_hi + 1) + KSTAGE - 1) / KSTAGE;
}

template <int U>
__global__ void __launch_bounds__(CT_THREADS, 1) dsd_convT2_tc_kernel(const ConvT2Params a) {
  constexpr int Q = CT_ROWS / U;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  float* act = reinterpret_cast<float*>(smem + CT_RING);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + CT_RING + (size_t)Q * a.pstr * 4);
  uint64_t* empty = full + CT_STAGES;
  uint64_t* act_full = empty + CT_STAGES;
  uint64_t* act_empty = act_full + 1;

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;   // warp-uniform role
  const int i0 = (int)((int64_t)a.num_items * blockIdx.x / gridDim.x);
  const int i1 = (int)((int64_t)a.num_items * (blockIdx.x + 1) / gridDim.x);
  if (threadIdx.x == 0) {
    for (int s = 0; s < CT_STAGES; ++s) {
      mbar_init(&full[s], 32);
      mbar_init(&empty[s], CT_CONSUMERS / 32);
    }
    mbar_init(act_full, 1);
    mbar_init(act_empty, CT_CONSUMERS / 32);
    fence_barrier_init();
  }
  __syncthreads();
  if (i0 >= i1) return;

  if (warp == 8) {
    // ------------------------------------------------------------------ B ring
    int g = 0;   // stage sequence number over the whole range
    for (int it = i0; it < i1; ++it) {
      int kb_lo, kb_hi;
      convT2_item_kb<U>(a, it % a.nub, kb_lo, kb_hi);
      for (int kb = kb_lo; kb < kb_hi; ++kb, ++g) {
        const int s = g % CT_STAGES;
        mbar_wait_relaxed(&empty[s], ((g / CT_STAGES) & 1) ^ 1);
        const uint32_t dst = smem_u32(smem + s * CT_B_STAGE);
#pragma unroll
        for (int i = 0; i < CT_B_PIECES; ++i) {
          const int c = i * 32 + lane;                     // 8 lanes cover one 128-byte row
          const int plane = c / (CT_N * 8), rc = c - plane * (CT_N * 8), row = rc >> 3, ch = rc & 7;
          const float* src = (plane ? a.Blo : a.Bhi) + (int64_t)row * a.Kp + kb * KSTAGE + 4 * ch;
          cp_async16(dst + plane * CT_B_PLANE + tile_off(row, ch), src);
        }
        cp_async_commit();
        if (g >= CT_LAG) {   // stage g - LAG has landed: publish it to the async proxy and the consumers
          cp_async_wait<CT_LAG>();
          fence_proxy_async();
          mbar_arrive(&full[(g - CT_LAG) % CT_STAGES]);
        }
      }
    }
    cp_async_wait<0>();
    fence_proxy_async();
    for (int j = max(0, g - CT_LAG); j < g; ++j) mbar_arrive(&full[j % CT_STAGES]);
    return;
  }
  if (warp == 9) {
    // ------------------------------------------------------------------ pair blocks
    if (lane == 0) {
      const uint32_t bytes = (uint32_t)a.h2 * CT_CP * 4;
      const int hp = a.h2 + 2 * (a.kh2 - 1);
      const int b_first = i0 / a.nub, b_last = (i1 - 1) / a.nub;
      for (int b = b_first; b <= b_last; ++b) {
        const int n = b - b_first;
        if (n > 0) mbar_wait_relaxed(act_empty, (n - 1) & 1);
        const int p0 = b * Q, np = min(Q, a.npairs - p0);
        mbar_arrive_expect_tx(act_full, bytes * np);
        for (int p = 0; p < np; ++p)
          bulk_copy_g2s(act + p * a.pstr, a.apad + ((int64_t)(p0 + p) * hp + a.kh2 - 1) * CT_CP, bytes, act_full);
      }
    }
    return;
  }
  // -------------------------------------------------------------------- consumers
  const int wg = warp >> 2, wq = warp & 3, g8 = lane >> 2, t4 = lane & 3;
  int pl[2], jr[2];   // this thread's two fragment rows: pair within the block, offset within the u block
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int r = wg * 64 + wq * 16 + g8 + 8 * i;
    pl[i] = r / U;
    jr[i] = r % U;
  }
  int g = 0, cur = -1, n = -1;
  for (int it = i0; it < i1; ++it) {
    const int b = it / a.nub, ub = it - b * a.nub;
    if (b != cur) {
      cur = b;
      ++n;
      mbar_wait(act_full, n & 1);
    }
    int kb_lo, kb_hi;
    convT2_item_kb<U>(a, ub, kb_lo, kb_hi);
    // element k of row i: interior float x = off + k of its pair, valid for 0 <= x < lim (lim also ends K)
    int off[2], lim[2];
    const float* arow[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int u = ub * U + jr[i];
      off[i] = (u - (a.kh2 - 1)) * CT_CP + t4;
      lim[i] = min(a.h2, u + 1) * CT_CP;
      arow[i] = act + pl[i] * a.pstr;
    }
    float acc[CT_N / 2], corr[CT_N / 2], sum[CT_N / 2];
#pragma unroll
    for (int v = 0; v < CT_N / 2; ++v) sum[v] = 0.f;
    for (int kb = kb_lo; kb < kb_hi; ++kb, ++g) {
      float ahi[4][4], alo[4][4];   // [k-step][fragment register]
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          // a load from a clamped index and a select: no divergent branch between the products
          const int i = q & 1, x = off[i] + kb * KSTAGE + 8 * j + 4 * (q >> 1);
          const bool in = (unsigned)x < (unsigned)lim[i];
          const float e = arow[i][in ? x : 0];
          const float v = in ? e : 0.f;
          split_tf32(v, ahi[j][q], alo[j][q]);
        }
      const int s = g % CT_STAGES;
      mbar_wait(&full[s], (g / CT_STAGES) & 1);
      const uint32_t b_hi = smem_u32(smem + s * CT_B_STAGE), b_lo = b_hi + CT_B_PLANE;
      wgmma_fence();
#pragma unroll
      for (int j = 0; j < KSTAGE / 8; ++j) {
        const uint64_t dbh = make_desc(b_hi + KSTEP_BYTES * j), dbl = make_desc(b_lo + KSTEP_BYTES * j);
        wgmma_tf32_rs_n56(corr, alo[j], dbh, kb != kb_lo || j != 0);
        wgmma_tf32_rs_n56(corr, ahi[j], dbl, 1);
        wgmma_tf32_rs_n56(acc, ahi[j], dbh, j != 0);
      }
      wgmma_commit();
      wgmma_wait_all();
      wgmma_fence_acc(acc);
      wgmma_fence_acc(corr);
      if (lane == 0) mbar_arrive(&empty[s]);
#pragma unroll
      for (int v = 0; v < CT_N / 2; ++v) sum[v] += acc[v];
    }
    // the block's last item in this range: its shared rows are no longer read
    if ((it + 1 == i1 || (it + 1) / a.nub != b) && lane == 0) mbar_arrive(act_empty);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int pair = b * Q + pl[i], u = ub * U + jr[i];
      if (pair >= a.npairs || u >= a.tc) continue;
      float* row = a.G + ((int64_t)pair * a.tc + u) * a.ldg;
#pragma unroll
      for (int j = 0; j < CT_N / 8; ++j) {
        const int c = 8 * j + 2 * t4;
        if (c < CT_C)
          *reinterpret_cast<float2*>(row + c) =
              make_float2(sum[4 * j + 2 * i] + corr[4 * j + 2 * i], sum[4 * j + 2 * i + 1] + corr[4 * j + 2 * i + 1]);
      }
    }
  }
}

bool dsd_convT2_tc_supported(const DsdConvT2Args& a) {
  return a.apad && a.G && a.npairs > 0 && a.tc >= 4 && a.tc <= 64 && a.ldg >= CT_C && a.ldg % 2 == 0 &&
         (int64_t)a.npairs * a.tc < ((int64_t)1 << 31) && (uintptr_t)a.apad % 16 == 0 &&
         (uintptr_t)a.G % 8 == 0;
}

template <int U>
static int launch_convT2_t(dcs_ctx* ctx, const ConvT2Params& p, cudaStream_t st) {
  constexpr int Q = CT_ROWS / U;
  const int smem = CT_RING + Q * p.pstr * 4 + (2 * CT_STAGES + 2) * 8 + 1024;   // + alignment slack
  DCS_TRY(ensure_smem_attr(dsd_convT2_tc_kernel<U>, smem));
  const int ctas = std::min(ctx->num_sms, p.num_items);
  dsd_convT2_tc_kernel<U><<<(unsigned)ctas, CT_THREADS, smem, st>>>(p);
  DCS_CHECK_LAUNCH();
  ctx->launches++;
  return DCS_OK;
}

// U = 4 (Q = 32 pairs per block) up to h2 = 16 (time_context 31), U = 8 (Q = 16) above: the pair block stays
// within 112 KB of shared memory next to the 84 KB B ring
int launch_dsd_convT2_tc(dcs_ctx* ctx, const DsdConvT2Args& a, const TcWeight& w, cudaStream_t st) {
  DCS_REQUIRE(dsd_convT2_tc_supported(a), "dsd_convT2_tc: unsupported shape or alignment");
  const int kh2 = a.tc / 2, h2 = a.tc - kh2 + 1;
  DCS_REQUIRE(w.K == kh2 * CT_CP && w.N == CT_C && w.Np >= CT_N && w.Kp % KSTAGE == 0,
              "dsd_convT2_tc: weight is %dx%d, the layer wants K=%d N=%d", w.K, w.N, kh2 * CT_CP, CT_C);
  ConvT2Params p;
  p.apad = a.apad; p.G = a.G; p.Bhi = w.hi; p.Blo = w.lo; p.Kp = w.Kp; p.ldg = a.ldg;
  p.npairs = a.npairs; p.tc = a.tc; p.kh2 = kh2; p.h2 = h2;
  p.pstr = convT2_pair_stride(h2);
  const int U = h2 <= 16 ? 4 : 8, Q = CT_ROWS / U;
  p.nub = (a.tc + U - 1) / U;
  p.num_items = (int)(ceil_div64(p.npairs, Q) * p.nub);
  return U == 4 ? launch_convT2_t<4>(ctx, p, st) : launch_convT2_t<8>(ctx, p, st);
}

}  // namespace dcs
