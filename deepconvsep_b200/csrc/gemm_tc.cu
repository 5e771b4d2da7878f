// gemm_tc.cu -- fp32-accurate GEMM on the Hopper tensor cores: wgmma.mma_async tf32 with the
// 3xTF32 operand split, accumulators in registers, C = act(A*B + bias).
//
// Same operand model as gemm.cu (GemmDesc): A is a strided / overlapping / K-segmented *view*
// of an fp32 activation buffer in HBM (convolution rows are never materialised); B is a weight
// matrix that was transposed to K-major, zero padded and split into (hi, lo) once at model load
// (TcWeight).  Per CTA: one 128 x BN output tile.
//   warps 0-3   producers: global fp32 -> registers -> hi/lo split -> canonical K-major shared
//               tiles (tc.cuh), fence.proxy.async, mbarrier arrive; the next stage's global loads
//               are in flight while a stage is stored
//   warps 4-11  two consumer warpgroups, one per 64-row half of the tile: 3 wgmma per k-step,
//               then the epilogue straight from the accumulator registers (+bias, ReLU -> global)
// STAGES-deep mbarrier ring (full: 128 producer arrivals, empty: one arrival per consumer warp).
#include "common.cuh"
#include "tc.cuh"

namespace dcs {

using namespace tc;

constexpr int TC_BM = 128;
constexpr int TC_PGROUPS = 1;                       // producer groups of 4 warps (> 1: alternating stages)
constexpr int TC_PWARPS = 4 * TC_PGROUPS;
constexpr int TC_CWARPS = 8;                        // two consumer warpgroups
constexpr int TC_THREADS = (TC_PWARPS + TC_CWARPS) * 32;   // 384: up to 168 registers a thread

template <int BN, int STAGES>
struct TcSmem {
  static constexpr int A_BYTES = TC_BM * ROW_BYTES;  // 16 KB
  static constexpr int B_BYTES = BN * ROW_BYTES;
  static constexpr int STAGE_BYTES = 2 * A_BYTES + 2 * B_BYTES;
  static constexpr int BAR_OFF = STAGES * STAGE_BYTES;
  static constexpr int TOTAL = BAR_OFF + 256 + 1024;  // + alignment slack
};

// Accumulator plan.  The tensor core adds into its fp32 accumulator with truncation, so a chain of
// n sequential accumulations loses ~n * 2^-24 relative.  The main hi*hi term of each 32-wide stage
// (4 k-steps) therefore goes to a fresh accumulator that is added into an fp32 register sum
// (round to nearest) once per stage; the two correction terms (2^-11 smaller, their truncation is
// harmless) share one accumulator over the whole K range.
template <int BN, int STAGES, int AVEC, bool SPLITK, int EPI = 0>
__global__ void __launch_bounds__(TC_THREADS)
gemm_tc_kernel(const GemmDesc d, const float* __restrict__ Bhi, const float* __restrict__ Blo, int Kp,
               int k_splits, float* __restrict__ partial, int ldp) {
  using SM = TcSmem<BN, STAGES>;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + SM::BAR_OFF);
  uint64_t* empty = full + STAGES;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int m0 = blockIdx.x * TC_BM, n0 = blockIdx.y * BN;
  int kb_lo = 0, kb_hi = (d.K + KSTAGE - 1) / KSTAGE;
  if (d.kc_rows > 0) {
    const int u_min = m0 / d.kc_rows, u_max = min(d.M - 1, m0 + TC_BM - 1) / d.kc_rows;
    const int q_lo = max(0, d.kc_pad - u_max), q_hi = min(d.kc_taps - 1, d.kc_pad + d.kc_n - 1 - u_min);
    kb_lo = (d.kc_unit * q_lo) / KSTAGE;
    kb_hi = min(kb_hi, (d.kc_unit * (q_hi + 1) + KSTAGE - 1) / KSTAGE);
    if (kb_hi <= kb_lo) kb_hi = kb_lo + 1;   // keep one (all-zero) block so the accumulators are defined
  }
  if (SPLITK) {   // split-K: this CTA (blockIdx.z) owns a contiguous slice of the k-blocks
    const int per = (kb_hi - kb_lo + k_splits - 1) / k_splits;
    kb_lo += blockIdx.z * per;
    kb_hi = min(kb_hi, kb_lo + per);
    if (kb_hi <= kb_lo) kb_hi = kb_lo + 1;   // cannot happen (the launcher sizes the slices); loads past K are guarded
  }
  const int num_kb = kb_hi - kb_lo;   // k-block i of this tile is global block kb_lo + i

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 128);
      mbar_init(&empty[s], TC_CWARPS);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < TC_PWARPS) {
    // ------------------------------------------------------------------ producers
    // group pg stages k-blocks pg, pg+2, ...: two stage loads are in flight per CTA
    const int pg = warp >> 2;
    const int tid = threadIdx.x & 127, warp = tid >> 5;   // index inside the producer group
    // Each warp-wide load covers whole 128-byte rows (AVEC=4: 4 rows x 8 chunks of 16 B per
    // instruction, AVEC=2: 2 rows x 16 pieces of 8 B, AVEC=1: 1 row x 32 floats) so global reads
    // are coalesced, and the swizzled shared stores of one row hit 8 distinct 16-byte slots.
    constexpr int RPI = AVEC == 4 ? 4 : (AVEC == 2 ? 2 : 1);   // rows per warp instruction
    constexpr int NI = 32 / RPI;                                // instructions per thread per stage (A)
    const int sub = lane / (32 / RPI);                          // row within the instruction
    const int piece = lane % (32 / RPI);                        // piece within the row
    // this thread's A rows: warp w owns rows [32w, 32w+32)
    const float* arow[NI];
    bool row_ok[NI];
#pragma unroll
    for (int i = 0; i < NI; ++i) {
      const int m = m0 + warp * 32 + i * RPI + sub;
      row_ok[i] = (m < d.M) && (m < d.a_valid_rows);
      const int mc = m < d.M ? m : 0;
      arow[i] = d.A + (int64_t)(mc / d.m_inner) * d.a_so + (int64_t)((mc % d.m_inner) / d.m_inner2) * d.a_si + (int64_t)(mc % d.m_inner2) * d.a_s2;
    }
    const bool seg_vec = d.k_seg < d.K;   // only reached with AVEC > 1 when k_seg % KSTAGE == 0 (launcher)
    constexpr int NBI = (2 * BN) / 16;   // B: 2*BN rows (hi+lo planes), 16 rows per pass of 128 threads
    float ra[NI][AVEC];
    float4 rb[NBI];
    auto gload = [&](int kb) {
#pragma unroll
      for (int i = 0; i < NI; ++i) {
        const int k = (kb_lo + kb) * KSTAGE + piece * AVEC;
        // K split in segments (one per convolution tap): with k_seg a multiple of the 32-wide
        // stage a vector never straddles two segments
        const int64_t koff = seg_vec ? (int64_t)(k / d.k_seg) * d.k_ss + (k % d.k_seg) : (int64_t)k;
#pragma unroll
        for (int e = 0; e < AVEC; ++e) ra[i][e] = 0.f;
        if (row_ok[i] && k < d.K) {
          if (AVEC == 4 && k + 4 <= d.K) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(arow[i] + koff));
            ra[i][0] = v.x; ra[i][1] = v.y; ra[i][AVEC > 2 ? 2 : 0] = v.z; ra[i][AVEC > 3 ? 3 : 0] = v.w;
          } else if (AVEC == 2 && k + 2 <= d.K) {
            const float2 v = __ldg(reinterpret_cast<const float2*>(arow[i] + koff));
            ra[i][0] = v.x; ra[i][AVEC > 1 ? 1 : 0] = v.y;
          } else {
#pragma unroll
            for (int e = 0; e < AVEC; ++e) {
              const int kk = k + e;
              if (kk < d.K) ra[i][e] = __ldg(arow[i] + (int64_t)(kk / d.k_seg) * d.k_ss + (kk % d.k_seg));
            }
          }
        }
      }
#pragma unroll
      for (int i = 0; i < NBI; ++i) {
        const int rr = i * 16 + (tid >> 3);          // row in the stacked (hi, lo) B planes
        const int which = rr / BN, rn = rr - which * BN;
        const float* src = (which ? Blo : Bhi) + (int64_t)(n0 + rn) * Kp + (kb_lo + kb) * KSTAGE + 4 * (tid & 7);
        rb[i] = (kb_lo + kb) * KSTAGE < Kp ? ld_stream(reinterpret_cast<const float4*>(src)) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    };
    if (pg < num_kb) gload(pg);
    for (int kb = pg; kb < num_kb; kb += TC_PGROUPS) {
      const int s = kb % STAGES;
      const uint32_t par = (kb / STAGES) & 1;
      mbar_wait_relaxed(&empty[s], par ^ 1);
      uint8_t* st = smem + s * SM::STAGE_BYTES;
#pragma unroll
      for (int i = 0; i < NI; ++i) {
        const int r = warp * 32 + i * RPI + sub;
        const int e0 = piece * AVEC;                 // first fp32 of this piece within the row
        const uint32_t off = tile_off(r, e0 >> 2) + (e0 & 3) * 4;
        float hi[AVEC], lo[AVEC];
#pragma unroll
        for (int e = 0; e < AVEC; ++e) split_tf32(ra[i][e], hi[e], lo[e]);
        if (AVEC == 4) {
          *reinterpret_cast<float4*>(st + off) = make_float4(hi[0], hi[1], hi[AVEC > 2 ? 2 : 0], hi[AVEC > 3 ? 3 : 0]);
          *reinterpret_cast<float4*>(st + SM::A_BYTES + off) = make_float4(lo[0], lo[1], lo[AVEC > 2 ? 2 : 0], lo[AVEC > 3 ? 3 : 0]);
        } else if (AVEC == 2) {
          *reinterpret_cast<float2*>(st + off) = make_float2(hi[0], hi[AVEC > 1 ? 1 : 0]);
          *reinterpret_cast<float2*>(st + SM::A_BYTES + off) = make_float2(lo[0], lo[AVEC > 1 ? 1 : 0]);
        } else {
          *reinterpret_cast<float*>(st + off) = hi[0];
          *reinterpret_cast<float*>(st + SM::A_BYTES + off) = lo[0];
        }
      }
#pragma unroll
      for (int i = 0; i < NBI; ++i) {
        const int rr = i * 16 + (tid >> 3);
        const int which = rr / BN, rn = rr - which * BN;
        *reinterpret_cast<float4*>(st + 2 * SM::A_BYTES + which * SM::B_BYTES + tile_off(rn, tid & 7)) = rb[i];
      }
      fence_proxy_async();
      mbar_arrive(&full[s]);
      if (kb + TC_PGROUPS < num_kb) gload(kb + TC_PGROUPS);
    }
    return;
  }
  // ------------------------------------------------------------------ consumers: one warpgroup per 64-row half
  const int half = (warp - TC_PWARPS) >> 2, wq = warp & 3;
  constexpr int NV = BN / 2;   // accumulator registers per thread (m64 x BN fragment, see tc.cuh)
  float acc[NV], corr[NV], sum[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) { acc[i] = 0.f; corr[i] = 0.f; sum[i] = 0.f; }
  for (int kb = 0; kb < num_kb; ++kb) {
    const int s = kb % STAGES;
    mbar_wait(&full[s], (kb / STAGES) & 1);
    const uint32_t a_hi = smem_u32(smem + s * SM::STAGE_BYTES) + half * 64 * ROW_BYTES;   // 8 KB: keeps the swizzle phase
    const uint32_t a_lo = a_hi + SM::A_BYTES;
    const uint32_t b_hi = smem_u32(smem + s * SM::STAGE_BYTES) + 2 * SM::A_BYTES;
    const uint32_t b_lo = b_hi + SM::B_BYTES;
    wgmma_fence();
#pragma unroll
    for (int j = 0; j < KSTAGE / 8; ++j) {
      const uint64_t dah = make_desc(a_hi + KSTEP_BYTES * j), dal = make_desc(a_lo + KSTEP_BYTES * j);
      const uint64_t dbh = make_desc(b_hi + KSTEP_BYTES * j), dbl = make_desc(b_lo + KSTEP_BYTES * j);
      wgmma_tf32<BN>(corr, dal, dbh, kb != 0 || j != 0);
      wgmma_tf32<BN>(corr, dah, dbl, 1);
      wgmma_tf32<BN>(acc, dah, dbh, j != 0);
    }
    wgmma_commit();
    wgmma_wait_all();
    if (lane == 0) mbar_arrive(&empty[s]);   // this warp's operand reads of the stage are done
#pragma unroll
    for (int i = 0; i < NV; ++i) sum[i] += acc[i];
  }
  // ------------------------------------------------------------------ epilogue from the fragment
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = m0 + half * 64 + wq * 16 + (lane >> 2) + 8 * h;
    if (m >= d.M) continue;
    const int64_t roff = SPLITK ? 0 : gemm_c_row_offset(d, m);
    int64_t groff = 0, gcol = 0;   // EPI_GATE: gate row offset and this row's column offset in the gated layer
    if (EPI & EPI_GATE) {
      groff = (int64_t)(m / d.g_inner) * d.g_so + (int64_t)((m % d.g_inner) / d.g_inner2) * d.g_si;
      gcol = (int64_t)(m % d.g_inner2) * d.g_s2;
    }
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int n = n0 + 8 * j + 2 * (lane & 3) + e;
        if (n >= d.N) continue;
        float x = sum[4 * j + 2 * h + e] + corr[4 * j + 2 * h + e];
        if (EPI) {
          if (EPI & EPI_POST) {
            const float pre = x + __ldg(d.bias + n);
            if (d.code) d.code[(int64_t)m * d.N + n] = pre > 0.f ? 2 : (pre == 0.f ? 1 : 0);
            x = fmaxf(pre, 0.f) + __ldg(d.bias2 + n);
          }
          if (EPI & EPI_GATE) {
            if (gcol + n >= d.g_lim) continue;
            x *= 0.5f * (float)d.gate[groff + gcol + n];
          }
          d.C[roff + (int64_t)(n / d.n_seg) * d.n_ss + (n % d.n_seg)] = x;
        } else if (SPLITK) {   // split-K: raw partial sums, reduced (+bias, activation) by splitk_reduce_kernel
          partial[((int64_t)blockIdx.z * d.M + m) * ldp + n] = x;
        } else {
          if (d.bias) x += __ldg(d.bias + n);
          if (d.relu) x = fmaxf(x, 0.f);
          d.C[roff + (int64_t)(n / d.n_seg) * d.n_ss + (n % d.n_seg)] = x;
        }
      }
    }
  }
}

__global__ void splitk_reduce_kernel(const GemmDesc d, const float* __restrict__ partial, int ldp, int k_splits) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)d.M * d.N) return;
  const int m = (int)(i / d.N), n = (int)(i - (int64_t)m * d.N);
  float x = 0.f;
  for (int z = 0; z < k_splits; ++z) x += partial[((int64_t)z * d.M + m) * ldp + n];   // fixed order: deterministic
  if (d.bias) x += __ldg(d.bias + n);
  if (d.relu) x = fmaxf(x, 0.f);
  const int64_t roff = gemm_c_row_offset(d, m);
  d.C[roff + (int64_t)(n / d.n_seg) * d.n_ss + (n % d.n_seg)] = x;
}

// ---- host side ------------------------------------------------------------------------------
int tc_weight_create(const float* B, int64_t ldb, int K, int N, TcWeight* out, std::vector<void*>* owned) {
  // B[k][n] row-major (ld = ldb) -> K-major Bt[n][k], zero padded to Np x Kp, split hi/lo
  const int Kp = (K + KSTAGE - 1) / KSTAGE * KSTAGE, Np = (N + 63) / 64 * 64;  // the widest tile reads 64 rows
  std::vector<float> hi((size_t)Np * Kp, 0.f), lo((size_t)Np * Kp, 0.f);
  for (int k = 0; k < K; ++k)
    for (int n = 0; n < N; ++n) {
      const float x = B[(size_t)k * ldb + n];
      uint32_t u;
      memcpy(&u, &x, 4);
      u &= 0xFFFFE000u;
      float h;
      memcpy(&h, &u, 4);
      hi[(size_t)n * Kp + k] = h;
      lo[(size_t)n * Kp + k] = x - h;
    }
  out->K = K; out->N = N; out->Kp = Kp; out->Np = Np;
  DCS_CUDA(cudaMalloc((void**)&out->hi, 2 * hi.size() * sizeof(float)));   // one allocation: [hi; lo]
  if (owned) owned->push_back(out->hi);
  out->lo = out->hi + hi.size();
  DCS_CUDA(cudaMemcpy(out->hi, hi.data(), hi.size() * sizeof(float), cudaMemcpyHostToDevice));
  DCS_CUDA(cudaMemcpy(out->lo, lo.data(), lo.size() * sizeof(float), cudaMemcpyHostToDevice));
  return DCS_OK;
}

void tc_weight_destroy(TcWeight* w) {
  if (w->hi) cudaFree(w->hi);
  w->hi = w->lo = nullptr;
}

// the gated epilogues: one launch, no split K (its reduction kernel has the plain epilogue only)
template <int BN, int STAGES, int AVEC, int EPI>
static int launch_tc_epi(dcs_ctx* ctx, const GemmDesc& d, const TcWeight& w, cudaStream_t st) {
  using SM = TcSmem<BN, STAGES>;
  DCS_TRY(ensure_smem_attr(gemm_tc_kernel<BN, STAGES, AVEC, false, EPI>, SM::TOTAL));
  dim3 grid((unsigned)ceil_div64(d.M, TC_BM), (unsigned)ceil_div64(d.N, BN));
  gemm_tc_kernel<BN, STAGES, AVEC, false, EPI><<<grid, TC_THREADS, SM::TOTAL, st>>>(d, w.hi, w.lo, w.Kp, 1, nullptr, 0);
  DCS_CHECK_LAUNCH();
  ctx->launches++;
  return DCS_OK;
}

template <int BN, int STAGES, int AVEC>
static int launch_tc(dcs_ctx* ctx, const GemmDesc& d, const TcWeight& w, cudaStream_t st) {
  using SM = TcSmem<BN, STAGES>;
  DCS_TRY(ensure_smem_attr(gemm_tc_kernel<BN, STAGES, AVEC, false>, SM::TOTAL));
  DCS_TRY(ensure_smem_attr(gemm_tc_kernel<BN, STAGES, AVEC, true>, SM::TOTAL));
  const int m_tiles = (int)ceil_div64(d.M, TC_BM), n_tiles = (int)ceil_div64(d.N, BN);
  const int num_kb = (d.K + KSTAGE - 1) / KSTAGE;
  // skinny GEMMs (few output tiles, long K -- the bottleneck dense layers): split K over otherwise idle SMs
  int splits = 1;
  if ((int64_t)m_tiles * n_tiles * 2 <= ctx->num_sms && num_kb >= 16 && d.kc_rows == 0) {
    splits = (int)std::min<int64_t>(ctx->num_sms / ((int64_t)m_tiles * n_tiles), num_kb / 8);
    if (splits < 2) splits = 1;
    if (splits > 1) {   // no empty slice: every blockIdx.z must own at least one real k-block
      const int per = (num_kb + splits - 1) / splits;
      splits = (num_kb + per - 1) / per;
    }
  }
  float* partial = nullptr;
  const int ldp = (d.N + 3) / 4 * 4;
  if (splits > 1) {
    DCS_TRY(ctx->net[NET_SPLITK].ensure((size_t)splits * d.M * ldp * sizeof(float), st));
    partial = ctx->net[NET_SPLITK].as<float>();
  }
  dim3 grid((unsigned)m_tiles, (unsigned)n_tiles, (unsigned)splits);
  if (splits > 1)
    gemm_tc_kernel<BN, STAGES, AVEC, true><<<grid, TC_THREADS, SM::TOTAL, st>>>(d, w.hi, w.lo, w.Kp, splits, partial, ldp);
  else
    gemm_tc_kernel<BN, STAGES, AVEC, false><<<grid, TC_THREADS, SM::TOTAL, st>>>(d, w.hi, w.lo, w.Kp, 1, nullptr, 0);
  if (splits > 1) {
    DCS_CHECK_LAUNCH();
    ctx->launches++;
    const int64_t tot = (int64_t)d.M * d.N;
    splitk_reduce_kernel<<<(unsigned)ceil_div64(tot, 256), 256, 0, st>>>(d, partial, ldp, splits);
  }
  DCS_CHECK_LAUNCH();
  ctx->launches++;
  return DCS_OK;
}

// vector width the A view allows: every row start and every segment must keep the alignment
static int a_vector_width(const GemmDesc& d) {
  const bool one_seg = d.k_seg >= d.K;
  auto aligned = [&](int v) {
    return ((uintptr_t)d.A % (4 * v) == 0) && d.a_so % v == 0 && d.a_si % v == 0 && d.a_s2 % v == 0 &&
           (one_seg || (d.k_seg % KSTAGE == 0 && d.k_ss % v == 0));
  };
  return aligned(4) ? 4 : (aligned(2) ? 2 : 1);
}

// `d.B` is ignored: the weight comes pre-transposed in `w`.
int launch_gemm_tc(dcs_ctx* ctx, const GemmDesc& d, const TcWeight& w, cudaStream_t st) {
  if (d.M <= 0 || d.N <= 0) return DCS_OK;
  DCS_REQUIRE(d.K == w.K && d.N == w.N, "tc gemm: weight is %dx%d, GEMM wants K=%d N=%d", w.K, w.N, d.K, d.N);
  DCS_REQUIRE(ceil_div64(d.N, 64) <= 65535, "tc gemm: N=%d too large", d.N);
  DCS_REQUIRE(gemm_c_view_ok(d), "tc gemm: negative C stride or column offset");
  const int avec = a_vector_width(d);
  if (d.N <= 32) {   // the 30-channel convolutions of the iKala / Bach10 nets: half the weight traffic and MMA time
    if (avec == 4) return launch_tc<32, 4, 4>(ctx, d, w, st);
    if (avec == 2) return launch_tc<32, 4, 2>(ctx, d, w, st);
    return launch_tc<32, 4, 1>(ctx, d, w, st);
  }
  if (avec == 4) return launch_tc<64, 4, 4>(ctx, d, w, st);
  if (avec == 2) return launch_tc<64, 4, 2>(ctx, d, w, st);
  return launch_tc<64, 4, 1>(ctx, d, w, st);
}

int launch_gemm_tc_epi(dcs_ctx* ctx, const GemmDesc& d, const TcWeight& w, int epi, cudaStream_t st) {
  if (d.M <= 0 || d.N <= 0) return DCS_OK;
  DCS_REQUIRE(d.K == w.K && d.N == w.N, "tc gemm: weight is %dx%d, GEMM wants K=%d N=%d", w.K, w.N, d.K, d.N);
  DCS_REQUIRE(ceil_div64(d.N, 64) <= 65535, "tc gemm: N=%d too large", d.N);
  DCS_REQUIRE(gemm_c_view_ok(d), "tc gemm: negative C stride or column offset");
  DCS_REQUIRE(!(epi & EPI_POST) || (d.bias && d.bias2), "tc gemm: EPI_POST needs both biases");
  DCS_REQUIRE(!(epi & EPI_GATE) || (d.gate && d.g_inner > 0 && d.g_inner2 > 0), "tc gemm: EPI_GATE needs a gate view");
  // float4 operand loads only: the gated layers lay their activations out for it (the scalar-load variant spills)
  DCS_REQUIRE(a_vector_width(d) == 4, "tc gemm: the gated epilogues need a 16-byte aligned A view");
  if (epi == EPI_POST) return launch_tc_epi<64, 4, 4, EPI_POST>(ctx, d, w, st);
  if (epi == EPI_GATE) return launch_tc_epi<64, 4, 4, EPI_GATE>(ctx, d, w, st);
  if (epi == (EPI_POST | EPI_GATE)) return launch_tc_epi<64, 4, 4, EPI_POST | EPI_GATE>(ctx, d, w, st);
  DCS_REQUIRE(false, "tc gemm: unknown epilogue %d", epi);
}

}  // namespace dcs
