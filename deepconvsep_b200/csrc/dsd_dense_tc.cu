// dsd_dense_tc.cu -- the decoder dense layers of the DSD nets on the tensor cores:
//   apad[k][d][kh2 - 1 + i][c] = ReLU(z[k] . Wdec[:, (d h2 + i) 52 + c] + bdec[(d h2 + i) 52 + c]),  i < h2, c < 52
// for every patch k and decoder d, i.e. one GEMM (M = P, K = nfc, N = ndec h2 52) whose columns are scattered into the
// interior rows of the zero-padded apad.  K is short (128 or 256: 4 or 8 stages) and M is a few thousand, so a tile of
// the generic GEMM spends its time filling and draining its pipeline; this kernel keeps each CTA's weight slab resident
// in shared memory and runs over many row blocks.
//
// GEMM view (D = A * B^T, fp32-accurate 3xTF32, the accumulation plan of gemm_tc.cu, so apad is bit-identical to the
// generic GEMM's): K in 32-wide stages at absolute multiples of 32; per k8, lo*hi then hi*lo into one correction
// accumulator over the whole K and hi*hi into a fresh per-stage accumulator added into an fp32 sum after the stage;
// x = sum + corr, x += bias, fmaxf(x, 0).
//
// Grid: N in slabs of 96 columns (m64n96k8), cps CTAs per slab splitting the P rows into equal contiguous ranges
// (2496 columns = 26 slabs x 5 CTAs on 132 SMs at the 180 s clip).  256 threads, no producer warp:
//   - all threads: the slab's tWdec hi / lo planes, K / 32 swizzled [96][32] stage tiles each (96 KB at K = 128),
//     by cp.async, once; the only CTA-wide barrier follows it.
//   - two consumer warpgroups, each over its own 64-row blocks of the range (blocks wg, wg + 2, ...), so one group's
//     products run while the other waits for its stage, splits operands or stores.  Each thread loads its A fragments
//     (8 scalar z elements per row and stage) from global memory -- z is L2-resident -- one stage ahead, splits them
//     hi / lo in registers and issues the stage's 12 products with A from registers.  Epilogue straight from the
//     accumulators into apad: 8-byte stores (N and the segment width h2 52 are even, so a pair never straddles two
//     segments).  Rows past the range read the range's last row and are not stored.
#include "common.cuh"
#include "tc.cuh"

namespace dcs {

using namespace tc;

constexpr int DN_CP = 52;                      // channel pitch of apad (50 filters + 2 zero pad channels)
constexpr int DN_NS = 96;                      // slab width: GEMM N per CTA and per product
constexpr int DN_ROWS = 64;                    // rows per block (one warpgroup's m64)
constexpr int DN_GROUPS = 2;                   // consumer warpgroups
constexpr int DN_THREADS = 128 * DN_GROUPS;
constexpr int DN_TILE = DN_NS * ROW_BYTES;     // 12 KB: one swizzled [96][32] stage tile
constexpr int DN_MAX_K = 256;                  // 2 planes x 8 stage tiles = 192 KB of shared memory

struct DenseParams {
  const float* z;
  const float* bias;
  float* apad;
  const float* Bhi;
  const float* Blo;
  int Kp;
  int P, K, N;
  int nseg;              // h2 * 52: columns per decoder
  int64_t ldc, nss, col0;   // apad floats per patch, per decoder, and to the first interior row
  int cps;               // CTAs per slab
};

// this thread's 16 A elements of stage kb (mma.m16n8k8 tf32 fragments of 4 k-steps, tc.cuh): rows za / zb,
// columns 32 kb + 8 j + t4 (+ 4)
__device__ __forceinline__ void dense_load_stage(float (&raw)[16], const float* za, const float* zb, int kb) {
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int q = 0; q < 4; ++q) raw[4 * j + q] = __ldg((q & 1 ? zb : za) + kb * KSTAGE + 8 * j + 4 * (q >> 1));
}

// one 8-byte store (a float2 store through a pointer is split into two 4-byte ones here); apad is not read by the kernel
__device__ __forceinline__ void st_v2(float* p, float x, float y) {
  asm volatile("st.global.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(x), "f"(y));
}

__global__ void __launch_bounds__(DN_THREADS, 1) dsd_dense_tc_kernel(const DenseParams a) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  const int nst = a.K / KSTAGE;
  const int slab = blockIdx.x / a.cps, part = blockIdx.x - slab * a.cps;
  const int n0 = slab * DN_NS;
  const int r0 = (int)((int64_t)a.P * part / a.cps), r1 = (int)((int64_t)a.P * (part + 1) / a.cps);
  if (r0 >= r1) return;

  // ------------------------------------------------------------------ the weight slab: tile t = plane * nst + kb
  const int pieces = 2 * nst * DN_NS * 8;
  for (int c = threadIdx.x; c < pieces; c += DN_THREADS) {
    const int ch = c & 7, rt = c >> 3, t = rt / DN_NS, row = rt - t * DN_NS;   // 8 threads cover one 128-byte row
    const int plane = t >= nst, kb = t - plane * nst;
    const uint32_t off = t * DN_TILE + tile_off(row, ch);
    if (n0 + row < a.N)
      cp_async16(smem_u32(smem) + off, (plane ? a.Blo : a.Bhi) + (int64_t)(n0 + row) * a.Kp + kb * KSTAGE + 4 * ch);
    else   // past N (the last slab): zero columns, never stored
      *reinterpret_cast<float4*>(smem + off) = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  cp_async_commit();
  cp_async_wait<0>();
  fence_proxy_async();
  __syncthreads();

  // ------------------------------------------------------------------ consumers
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp >> 2, wq = warp & 3, g8 = lane >> 2, t4 = lane & 3;
  const int nblk = (r1 - r0 + DN_ROWS - 1) / DN_ROWS;
  if (wg >= nblk) return;
  // row i (0, 1) of this thread's fragments in block b
  auto row_of = [&](int b, int i) { return r0 + b * DN_ROWS + wq * 16 + g8 + 8 * i; };
  auto zrow = [&](int b, int i) { return a.z + (int64_t)min(row_of(b, i), r1 - 1) * a.K + t4; };
  float raw[16];
  dense_load_stage(raw, zrow(wg, 0), zrow(wg, 1), 0);
  for (int b = wg; b < nblk; b += DN_GROUPS) {
    const float *za = zrow(b, 0), *zb = zrow(b, 1);
    float acc[DN_NS / 2], corr[DN_NS / 2], sum[DN_NS / 2];
#pragma unroll
    for (int v = 0; v < DN_NS / 2; ++v) sum[v] = 0.f;
    for (int kb = 0; kb < nst; ++kb) {
      float ahi[4][4], alo[4][4];   // [k-step][fragment register]
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int q = 0; q < 4; ++q) split_tf32(raw[4 * j + q], ahi[j][q], alo[j][q]);
      // the next stage's A (this block's, or the group's next block's first) in flight under this stage's products;
      // selects, not a branch: a wgmma issue behind a divergent path is serialised.  After the group's last stage
      // this re-reads its last block's first stage, unused.
      {
        const bool same = kb + 1 < nst, nb = !same && b + DN_GROUPS < nblk;
        dense_load_stage(raw, nb ? zrow(b + DN_GROUPS, 0) : za, nb ? zrow(b + DN_GROUPS, 1) : zb, same ? kb + 1 : 0);
      }
      const uint32_t b_hi = smem_u32(smem + kb * DN_TILE), b_lo = smem_u32(smem + (nst + kb) * DN_TILE);
      wgmma_fence();
#pragma unroll
      for (int j = 0; j < KSTAGE / 8; ++j) {
        const uint64_t dbh = make_desc(b_hi + KSTEP_BYTES * j), dbl = make_desc(b_lo + KSTEP_BYTES * j);
        wgmma_tf32_rs_n96(corr, alo[j], dbh, kb != 0 || j != 0);
        wgmma_tf32_rs_n96(corr, ahi[j], dbl, 1);
        wgmma_tf32_rs_n96(acc, ahi[j], dbh, j != 0);
      }
      wgmma_commit();
      wgmma_wait_all();
      wgmma_fence_acc(acc);
      wgmma_fence_acc(corr);
#pragma unroll
      for (int v = 0; v < DN_NS / 2; ++v) sum[v] += acc[v];
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int row = row_of(b, i);
      if (row >= r1) continue;
      float* out = a.apad + (int64_t)row * a.ldc + a.col0;
#pragma unroll
      for (int j = 0; j < DN_NS / 8; ++j) {
        const int n = n0 + 8 * j + 2 * t4;
        if (n >= a.N) continue;
        const int seg = n / a.nseg;
        float x0 = sum[4 * j + 2 * i] + corr[4 * j + 2 * i], x1 = sum[4 * j + 2 * i + 1] + corr[4 * j + 2 * i + 1];
        x0 += __ldg(a.bias + n);
        x1 += __ldg(a.bias + n + 1);
        st_v2(out + seg * a.nss + (n - seg * a.nseg), fmaxf(x0, 0.f), fmaxf(x1, 0.f));
      }
    }
  }
}

bool dsd_dense_tc_supported(const DsdDenseArgs& a) {
  return a.z && a.bias && a.apad && a.P > 0 && a.tc >= 4 && a.tc <= 64 && (a.ndec == 3 || a.ndec == 4) &&
         a.nfc > 0 && a.nfc % KSTAGE == 0 && a.nfc <= DN_MAX_K && (uintptr_t)a.z % 4 == 0 &&
         (uintptr_t)a.bias % 4 == 0 && (uintptr_t)a.apad % 8 == 0;
}

// one launch: ceil(N / 96) slabs x cps CTAs, cps = the SMs per slab (at least 1, at most P)
int launch_dsd_dense_tc(dcs_ctx* ctx, const DsdDenseArgs& a, const TcWeight& w, cudaStream_t st) {
  DCS_REQUIRE(dsd_dense_tc_supported(a), "dsd_dense_tc: unsupported shape or alignment");
  const int kh2 = a.tc / 2, h2 = a.tc - kh2 + 1, hp = h2 + 2 * (kh2 - 1);
  const int N = a.ndec * h2 * DN_CP;
  DCS_REQUIRE(w.K == a.nfc && w.N == N && w.Kp == a.nfc && w.Np >= N,
              "dsd_dense_tc: weight is %dx%d, the layer wants K=%d N=%d", w.K, w.N, a.nfc, N);
  DenseParams p;
  p.z = a.z; p.bias = a.bias; p.apad = a.apad; p.Bhi = w.hi; p.Blo = w.lo; p.Kp = w.Kp;
  p.P = a.P; p.K = a.nfc; p.N = N; p.nseg = h2 * DN_CP;
  p.nss = (int64_t)hp * DN_CP; p.ldc = a.ndec * p.nss; p.col0 = (int64_t)(kh2 - 1) * DN_CP;
  const int nslab = (N + DN_NS - 1) / DN_NS;
  p.cps = std::max(1, std::min(ctx->num_sms / nslab, a.P));
  const int smem = 2 * (a.nfc / KSTAGE) * DN_TILE + 1024;   // + alignment slack
  DCS_TRY(ensure_smem_attr(dsd_dense_tc_kernel, smem));
  dsd_dense_tc_kernel<<<(unsigned)(nslab * p.cps), DN_THREADS, smem, st>>>(p);
  DCS_CHECK_LAUNCH();
  ctx->launches++;
  return DCS_OK;
}

}  // namespace dcs
