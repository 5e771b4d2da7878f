// stft_reg.cu -- STFT (K1) and iSTFT + overlap-add (K4) with the register-resident FFT of
// fft_reg.cuh, for frame sizes 1024 and 2048 (the DSD100 / iKala configurations).  Same reference
// semantics as stft.cu (transform.py:277-396); that file's shared-memory Stockham kernels remain
// the path for the other frame sizes / hops.
//
// K1: one group of T = N/64 threads (a warp for N = 2048) owns a frame: hop-overlapped, windowed
//     samples go from global memory straight into registers, the spectrum is staged once in the
//     group's scratch so that the real-FFT split and the X / mag rows leave fully coalesced.
// K4: a group owns `hops_per_group` consecutive output hops of one source and walks the frames
//     that overlap them IN FRAME ORDER, keeping the overlap-add window (N samples) in registers:
//     after frame n is added, the oldest hop is complete -> divided by sum(win*syn_win), stored
//     coalesced, and the window shifts.  No shared accumulator, no atomics: the summation order
//     is the reference's (ascending frame index) and the result is run-to-run deterministic.
//     N/hop - 1 halo frames are recomputed at the start of each span.  Spectrum (and mask) rows reach shared memory
//     through 2-stage rings filled by bulk async copies on mbarriers, the fetch of frame n+1 in flight while the
//     group waits for frame n; the masked variant shares one X ring among the groups of all sources of a channel.
#include "common.cuh"
#include "fft_reg.cuh"
#include "tc.cuh"

namespace dcs {

constexpr int REG_THREADS = 128;
// K4 runs ONE CTA of 8 warps per SM so that the twiddle table and the synthesis window -- per-thread
// constants re-read for every frame -- sit in shared memory next to the 8 scratch + row buffers.  8 warps
// (not 12) leave up to 255 registers a thread: the 32-value frame, the 32-value overlap-add window and the
// per-slot normalisation stay in registers (at 168 registers ptxas spilled them to local memory on sm_90a).
constexpr int ISTFT_THREADS = 256;

template <int T>
__global__ void __launch_bounds__(REG_THREADS)
stft_reg_kernel(const float* __restrict__ audio, int64_t L, int hop, const float* __restrict__ win,
                const float2* __restrict__ tw, float2* __restrict__ X, float* __restrict__ mag,
                float* __restrict__ phase, int64_t ldf, int64_t nframes, float mag_scale, int frames_per_group) {
  using G = FftGroup<T>;
  constexpr int N2 = G::N2, N = 2 * N2, F = N2 + 1, GPC = REG_THREADS / T;
  extern __shared__ __align__(16) float2 scratch[];
  const int tid = threadIdx.x, b = tid % T, gl = tid / T;
  float2* scr = scratch + gl * G::SCRATCH;
  // shared copies of the twiddle table and of the analysis window (per-thread constants of every frame)
  float2* stw = scratch + GPC * G::SCRATCH;        // tw[0..N2): the real-FFT split twiddles
  float2* stw2 = stw + N2;                         // inter-stage twiddles, lane-contiguous (FftGroup::fill_tw2)
  float2* swin = stw2 + N2;
  for (int i = tid; i < N2; i += REG_THREADS) stw[i] = __ldg(tw + i);
  G::fill_tw2(stw2, tw, tid, REG_THREADS);
  for (int i = tid; i < N2; i += REG_THREADS) swin[i] = __ldg(reinterpret_cast<const float2*>(win) + i);
  __syncthreads();
  const int64_t g = (int64_t)blockIdx.x * GPC + gl;
  const bool audio_aligned8 = (reinterpret_cast<uintptr_t>(audio) & 7) == 0;
  const int64_t warp_first = ((int64_t)blockIdx.x * GPC + (tid / 32) * (32 / T)) * frames_per_group;
  for (int i = 0; i < frames_per_group; ++i) {
    if (warp_first + i >= nframes) break;  // warp-uniform: even the warp's first group is past the end
    const int64_t n = g * frames_per_group + i;
    const bool valid = n < nframes;
    const int64_t base = n * hop - N / 2;
    float2 v[32];
    // frames that lie inside the clip (all but N/hop at either end) take 8-byte loads with no bounds
    // arithmetic: base is even, so the pairs are aligned whenever the buffer is
    if (valid && base >= 0 && base + N <= L && audio_aligned8) {
      const float2* __restrict__ ap = reinterpret_cast<const float2*>(audio + base);
#pragma unroll
      for (int a = 0; a < 32; ++a) {
        const int idx = a * T + b;
        const float2 w = swin[idx], x = __ldg(ap + idx);
        v[a] = make_float2(x.x * w.x, x.y * w.y);
      }
    } else {
#pragma unroll
      for (int a = 0; a < 32; ++a) {
        const int idx = a * T + b;
        const int64_t s = base + 2 * idx;
        const float2 w = swin[idx];
        const float x0 = (valid && s >= 0 && s < L) ? __ldg(audio + s) : 0.f;
        const float x1 = (valid && s + 1 >= 0 && s + 1 < L) ? __ldg(audio + s + 1) : 0.f;
        v[a] = make_float2(x0 * w.x, x1 * w.y);
      }
    }
    G::template forward<true>(v, scr, stw2, b);
#pragma unroll
    for (int q = 0; q < G::Q; ++q)
#pragma unroll
      for (int kb = 0; kb < T; ++kb) scr[(b + T * q) + 32 * kb] = v[q * T + kb];
    __syncwarp();
    if (valid) {
      const int64_t row = n * ldf;
#pragma unroll 4
      for (int m = 0; m < N2 / T; ++m) {
        const int k = b + T * m;
        const float2 xk = real_post_shared<N2>(scr, stw, k);
        if (X) X[row + k] = xk;
        if (mag) mag[row + k] = mag_scale * sqrtf(xk.x * xk.x + xk.y * xk.y);
        if (phase) phase[row + k] = atan2f(xk.y, xk.x);
      }
      if (b == 0) {  // Nyquist bin
        const float2 z0 = scr[0];
        const float vv = z0.x - z0.y;
        if (X) X[row + N2] = make_float2(vv, 0.f);
        if (mag) mag[row + N2] = mag_scale * fabsf(vv);
        if (phase) phase[row + N2] = atan2f(0.f, vv);
      }
      if (b < ldf - F) {  // pad columns
        if (X) X[row + F + b] = make_float2(0.f, 0.f);
        if (mag) mag[row + F + b] = 0.f;
        if (phase) phase[row + F + b] = 0.f;
      }
    }
    __syncwarp();
  }
}

// Shared memory of K4 (bytes): per group its FFT scratch, the twiddle tables and the synthesis window, the spectrum
// row rings (RING stages of ROWP float2 per quad), masked also a mask row ring per group (RING stages of ROWP floats),
// then the ring barriers (full / empty per quad and stage, masked a full barrier per group and stage).
constexpr int ISTFT_RING = 2;
constexpr size_t SM90_SMEM_OPTIN = 232448;   // shared memory a CTA may opt into on sm_90
template <int T>
__host__ __device__ constexpr int istft_rowp() { return (32 * T + 1 + 7) / 8 * 8; }
template <int T>
__host__ __device__ constexpr size_t istft_smem_bytes(int qpc, bool masked) {
  constexpr int GPC = ISTFT_THREADS / T, ROWP = istft_rowp<T>();
  return ((size_t)GPC * FftGroup<T>::SCRATCH + 3 * (size_t)(32 * T) + (size_t)qpc * ISTFT_RING * ROWP) * sizeof(float2) +
         (masked ? (size_t)GPC * ISTFT_RING * ROWP * sizeof(float) : 0) +
         ((size_t)qpc * 2 * ISTFT_RING + (masked ? (size_t)GPC * ISTFT_RING : 0)) * sizeof(uint64_t);
}

// The body of K4 and of its masked variant (MASKED: the spectrum is M_s * X_c, formed as the row is read).
//
// Groups are gathered in QUADS of qw neighbouring groups that walk the same frames (qpc quads per CTA, groups past
// qpc * qw idle: they run the loop on zeros so that every warp reaches the same __syncwarp()s, and store nothing).
// A quad shares one spectrum row ring in shared memory: one elected lane fetches each row with a bulk async copy that
// completes on the stage's `full` mbarrier, and every group of the quad arrives on the stage's `empty` mbarrier once it
// has read the row into registers.  The fetch of frame n+1 is issued at the top of iteration n, before the wait for
// frame n: two rows per quad in flight while the SM waits on HBM.
//   Not masked: qw = 1, a quad is one group and owns hops of plane quad / groups_per_src of S.
//   Masked: S is the mixture STFT (channel c at S + c * src_stride), Mk the masks (source s at Mk + s * m_stride, same
//   ldf), output plane s * nx + c.  The qw groups of a quad apply the masks of qw consecutive sources (one chunk of the
//   nsrc sources, ceil(nsrc / qw) chunks) to the same X rows; each group's mask rows go through a ring of its own the
//   same way (it is their only reader, so no empty barrier).  X is read from HBM once per quad instead of once per group.
template <int T, int HS, bool MASKED>  // HS = hop / 64: window slots (32 float2 each) per hop
__device__ __forceinline__ void
istft_reg_body(const float2* __restrict__ S, int64_t nframes, int64_t ldf, int64_t src_stride,
               const float* __restrict__ wsyn, const float* __restrict__ w2, const float2* __restrict__ tw,
               float* __restrict__ out, int64_t Lout, int64_t out_stride, int hops_per_group, int64_t num_hops,
               int64_t groups_per_src, int64_t total_quads, const float* __restrict__ Mk, int64_t m_stride, int nsrc,
               int nx, int qw, int qpc) {
  using G = FftGroup<T>;
  constexpr int N2 = G::N2, N = 2 * N2, hop = 64 * HS, R = N / hop, C0 = (N / 2) / hop, GPC = ISTFT_THREADS / T;
  constexpr int ROWP = istft_rowp<T>();               // float2 per staged row
  constexpr uint32_t XBYTES = (N2 + 2) / 2 * 16;      // 16-byte pieces covering bins 0..N2
  constexpr uint32_t MBYTES = (N2 + 4) / 4 * 16;      // masked: 16-byte pieces covering bins 0..N2 of a mask row
  extern __shared__ __align__(16) float2 scratch[];
  const int tid = threadIdx.x, b = tid % T, gl = tid / T;
  float2* scr = scratch + gl * G::SCRATCH;
  const int qi = gl / qw, mem = gl - qi * qw;          // quad, member
  const bool in_quad = qi < qpc;
  int64_t gq = (int64_t)blockIdx.x * qpc + (in_quad ? qi : 0);
  bool active = in_quad && gq < total_quads;
  if (gq >= total_quads) gq = total_quads - 1;         // keeps the quad's barriers and the warp convergent; nothing is stored
  int msrc = 0;   // masked: the source whose mask this group applies
  if constexpr (MASKED) {
    const int nchunk = (nsrc + qw - 1) / qw;
    msrc = (int)(gq % nchunk) * qw + mem;
    gq /= nchunk;
    if (msrc >= nsrc) { active = false; msrc = nsrc - 1; }
  }
  const int src = (int)(gq / groups_per_src);   // plane of S (masked: the channel)
  const int64_t h0 = (gq % groups_per_src) * hops_per_group;
  const float inv_n2 = 1.0f / (float)N2;
  float2 acc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = make_float2(0.f, 0.f);
  float* o = out + (int64_t)(MASKED ? msrc * nx + src : src) * out_stride;
  // 1 / sum_r win*syn_win for the interior of the clip (every hop sees the same R frames)
  float2 cinv[G::Q * HS];
#pragma unroll
  for (int q = 0; q < G::Q; ++q)
#pragma unroll
    for (int kb = 0; kb < HS; ++kb) {
      const int e = 2 * ((b + T * q) + 32 * kb);
      float c0 = 0.f, c1 = 0.f;
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const float2 ww = __ldg(reinterpret_cast<const float2*>(w2 + e + r * hop));
        c0 += ww.x;
        c1 += ww.y;
      }
      cinv[q * HS + kb] = make_float2(c0 == 0.f ? 1.f : 1.f / c0, c1 == 0.f ? 1.f : 1.f / c1);
    }

  // shared copies of the twiddle table (N entries, exp(-2 pi i j / N)) and of the synthesis window (as pairs)
  float2* stw = scratch + GPC * G::SCRATCH;             // tw[0..N2): the real-FFT merge twiddles
  float2* stw2 = stw + N2;                              // inter-stage twiddles, lane-contiguous (FftGroup::fill_tw2)
  float2* swsyn = stw2 + N2;
  float2* xring = swsyn + N2 + (in_quad ? qi : 0) * ISTFT_RING * ROWP;            // this quad's spectrum rows
  float* mring = reinterpret_cast<float*>(swsyn + N2 + qpc * ISTFT_RING * ROWP) + gl * ISTFT_RING * ROWP;
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<float*>(swsyn + N2 + qpc * ISTFT_RING * ROWP) +
                                               (MASKED ? GPC * ISTFT_RING * ROWP : 0));
  uint64_t* xfull = bars + (in_quad ? qi : 0) * 2 * ISTFT_RING;   // [stage]: the row landed
  uint64_t* xempty = xfull + ISTFT_RING;                           // [stage]: every group of the quad has read it
  uint64_t* mfull = bars + qpc * 2 * ISTFT_RING + gl * ISTFT_RING;
  for (int i = tid; i < N2; i += ISTFT_THREADS) stw[i] = __ldg(tw + i);
  G::fill_tw2(stw2, tw, tid, ISTFT_THREADS);
  for (int i = tid; i < N2; i += ISTFT_THREADS) swsyn[i] = __ldg(reinterpret_cast<const float2*>(wsyn) + i);
  if (tid < qpc * ISTFT_RING) {
    tc::mbar_init(bars + (tid / ISTFT_RING) * 2 * ISTFT_RING + tid % ISTFT_RING, 1);
    tc::mbar_init(bars + (tid / ISTFT_RING) * 2 * ISTFT_RING + ISTFT_RING + tid % ISTFT_RING, (uint32_t)qw);
  }
  if (MASKED && tid < GPC * ISTFT_RING) tc::mbar_init(bars + qpc * 2 * ISTFT_RING + tid, 1);
  tc::fence_barrier_init();
  __syncthreads();
  const bool xlane = in_quad && mem == 0 && b == 0;   // the quad's producer lane
  const bool glane = in_quad && b == 0;               // the group's lane for its mask rows and its empty arrivals
  const int64_t n_first = h0 + C0 - R + 1, n_last = h0 + hops_per_group - 1 + C0;
  // frame n into stage (n - n_first) % RING; frames outside the clip complete their stage with no bytes
  auto fetch_x = [&](int64_t nn) {
    const int k = (int)(nn - n_first), st = k % ISTFT_RING;
    if (k >= ISTFT_RING)   // the stage held frame nn - RING: wait until every group of the quad has read it
      tc::mbar_wait_relaxed(xempty + st, (uint32_t)((k / ISTFT_RING - 1) & 1));
    if (nn >= 0 && nn < nframes) {
      tc::mbar_arrive_expect_tx(xfull + st, XBYTES);
      tc::bulk_copy_g2s(xring + st * ROWP, S + (int64_t)src * src_stride + nn * ldf, XBYTES, xfull + st);
    } else {
      tc::mbar_arrive(xfull + st);
    }
  };
  auto fetch_m = [&](int64_t nn) {
    const int st = (int)(nn - n_first) % ISTFT_RING;
    if (nn >= 0 && nn < nframes) {
      tc::mbar_arrive_expect_tx(mfull + st, MBYTES);
      tc::bulk_copy_g2s(mring + st * ROWP, Mk + (int64_t)msrc * m_stride + nn * ldf, MBYTES, mfull + st);
    } else {
      tc::mbar_arrive(mfull + st);
    }
  };
  if (xlane) fetch_x(n_first);
  if (MASKED && glane) fetch_m(n_first);
  for (int64_t n = n_first; n <= n_last; ++n) {
    const bool fvalid = in_quad && n >= 0 && n < nframes;
    const int k = (int)(n - n_first), st = k % ISTFT_RING;
    const uint32_t par = (uint32_t)((k / ISTFT_RING) & 1);
    if (n < n_last) {   // frame n+1 goes in flight before this one is waited for
      if (xlane) fetch_x(n + 1);
      if (MASKED && glane) fetch_m(n + 1);
    }
    const float2* srow = xring + st * ROWP;
    const float* smrow = mring + st * ROWP;
    if (in_quad) {
      tc::mbar_wait(xfull + st, par);
      if constexpr (MASKED) tc::mbar_wait(mfull + st, par);
    }
    float2 v[32];
#pragma unroll
    for (int a = 0; a < 32; ++a) {
      const int idx = a * T + b;
      float2 xk = make_float2(0.f, 0.f), xn = xk;
      if (fvalid) {
        xk = srow[idx];
        xn = srow[N2 - idx];
        if constexpr (MASKED) {   // M * X componentwise: two roundings, never contracted into the sums that follow
          const float mk = smrow[idx], mn = smrow[N2 - idx];
          xk = make_float2(__fmul_rn(mk, xk.x), __fmul_rn(mk, xk.y));
          xn = make_float2(__fmul_rn(mn, xn.x), __fmul_rn(mn, xn.y));
        }
      }
      if (idx == 0) { xk.y = 0.f; xn.y = 0.f; }  // irfft ignores Im of DC and Nyquist
      v[a] = real_pre_conj(xk, xn, stw[idx]);
    }
    __syncwarp();                    // every lane has consumed the row
    if (glane) tc::mbar_arrive(xempty + st);
    G::template forward<true>(v, scr, stw2, b);
    // z = conj(V)/N2: samples 2n', 2n'+1 of the frame, n' = (b + T q) + 32 kb  <->  v[q*T + kb]
#pragma unroll
    for (int q = 0; q < G::Q; ++q)
#pragma unroll
      for (int kb = 0; kb < T; ++kb) {
        const int np = (b + T * q) + 32 * kb;
        const float2 w = swsyn[np];
        const float2 r = v[q * T + kb];
        acc[q * T + kb].x = fmaf(w.x, r.x * inv_n2, acc[q * T + kb].x);
        acc[q * T + kb].y = fmaf(w.y, -r.y * inv_n2, acc[q * T + kb].y);
      }
    // the oldest hop of the window is complete: padded samples [n*hop, (n+1)*hop) -> output hop n - C0
    const int64_t h = n - C0;
    if (active && h >= h0 && h < num_hops) {
      const bool interior = (n - (R - 1) >= 0) && (n < nframes);   // all R overlapping frames exist
#pragma unroll
      for (int q = 0; q < G::Q; ++q)
#pragma unroll
        for (int kb = 0; kb < HS; ++kb) {
          const int e = 2 * ((b + T * q) + 32 * kb);  // sample offset inside the hop
          float2 ic = cinv[q * HS + kb];
          if (!interior) {   // clip edges: sum win*syn_win over the frames that exist (transform.py:384-392)
            float c0 = 0.f, c1 = 0.f;
#pragma unroll
            for (int r = 0; r < R; ++r) {
              const int64_t nf = n - r;
              if (nf >= 0 && nf < nframes) {
                const float2 ww = __ldg(reinterpret_cast<const float2*>(w2 + e + r * hop));
                c0 += ww.x;
                c1 += ww.y;
              }
            }
            ic = make_float2(c0 == 0.f ? 1.f : 1.f / c0, c1 == 0.f ? 1.f : 1.f / c1);
          }
          const int64_t oi = h * hop + e;
          const float2 a2 = acc[q * T + kb];
          if (oi + 1 < Lout) {
            *reinterpret_cast<float2*>(o + oi) = make_float2(a2.x * ic.x, a2.y * ic.y);
          } else if (oi < Lout) {
            o[oi] = a2.x * ic.x;
          }
        }
    }
    // shift the window by one hop
#pragma unroll
    for (int q = 0; q < G::Q; ++q) {
#pragma unroll
      for (int kb = 0; kb < T - HS; ++kb) acc[q * T + kb] = acc[q * T + kb + HS];
#pragma unroll
      for (int kb = T - HS; kb < T; ++kb) acc[q * T + kb] = make_float2(0.f, 0.f);
    }
  }
}

template <int T, int HS>
__global__ void __launch_bounds__(ISTFT_THREADS, 1)
istft_reg_kernel(const float2* __restrict__ S, int64_t nframes, int64_t ldf, int64_t src_stride,
                 const float* __restrict__ wsyn, const float* __restrict__ w2, const float2* __restrict__ tw,
                 float* __restrict__ out, int64_t Lout, int64_t out_stride, int hops_per_group, int64_t num_hops,
                 int64_t groups_per_src, int64_t total_groups) {
  istft_reg_body<T, HS, false>(S, nframes, ldf, src_stride, wsyn, w2, tw, out, Lout, out_stride, hops_per_group, num_hops,
                               groups_per_src, total_groups, nullptr, 0, 1, 1, 1, ISTFT_THREADS / T);
}

// K4 on M_s * X_c: X complex [nx][nframes][ldf] (x_plane apart), Mk float [nsrc][nframes][ldf] (m_stride apart); quads
// of qw groups, qpc of them per CTA
template <int T, int HS>
__global__ void __launch_bounds__(ISTFT_THREADS, 1)
istft_masked_reg_kernel(const float2* __restrict__ X, int64_t nframes, int64_t ldf, int64_t x_plane,
                        const float* __restrict__ Mk, int64_t m_stride, int nsrc, int nx, const float* __restrict__ wsyn,
                        const float* __restrict__ w2, const float2* __restrict__ tw, float* __restrict__ out, int64_t Lout,
                        int64_t out_stride, int hops_per_group, int64_t num_hops, int64_t groups_per_plane,
                        int64_t total_quads, int qw, int qpc) {
  istft_reg_body<T, HS, true>(X, nframes, ldf, x_plane, wsyn, w2, tw, out, Lout, out_stride, hops_per_group, num_hops,
                              groups_per_plane, total_quads, Mk, m_stride, nsrc, nx, qw, qpc);
}

int launch_stft_reg(dcs_stft* p, const float* d_audio, int64_t L, float2* d_X, float* d_mag, float* d_phase,
                    float mag_scale, int64_t ldf, int64_t nframes, cudaStream_t st) {
  const int fpg = 4;
  const float ms = mag_scale / sqrtf((float)p->N);
  if (p->N == 2048) {
    using G = FftGroup<32>;
    const int gpc = REG_THREADS / 32;
    const size_t smem = (gpc * G::SCRATCH + 3 * G::N2) * sizeof(float2);   // scratch + twiddles + window
    DCS_TRY(ensure_smem_attr(stft_reg_kernel<32>, (int)smem));
    const unsigned grid = (unsigned)ceil_div64(nframes, (int64_t)gpc * fpg);
    stft_reg_kernel<32><<<grid, REG_THREADS, smem, st>>>(
        d_audio, L, p->hop, p->d_win, p->d_tw, d_X, d_mag, d_phase, ldf, nframes, ms, fpg);
  } else {
    using G = FftGroup<16>;
    const int gpc = REG_THREADS / 16;
    const size_t smem = (gpc * G::SCRATCH + 3 * G::N2) * sizeof(float2);
    DCS_TRY(ensure_smem_attr(stft_reg_kernel<16>, (int)smem));
    const unsigned grid = (unsigned)ceil_div64(nframes, (int64_t)gpc * fpg);
    stft_reg_kernel<16><<<grid, REG_THREADS, smem, st>>>(
        d_audio, L, p->hop, p->d_win, p->d_tw, d_X, d_mag, d_phase, ldf, nframes, ms, fpg);
  }
  DCS_CHECK_LAUNCH();
  p->ctx->launches++;
  return DCS_OK;
}

bool istft_reg_supported(const dcs_stft* p, const float* d_out, int64_t out_stride) {
  // (the caller also guarantees 16-byte aligned spectrum rows: ldf % 2 == 0, see launch_istft)
  return (p->N == 1024 || p->N == 2048) && (p->hop == 512 || p->hop == 256) && ((uintptr_t)d_out % 8 == 0) &&
         out_stride % 2 == 0;
}

// d_M NULL: nsrc planes of d_S.  d_M set: d_S is the mixture STFT of nx channels (src_stride apart), d_M nsrc masks
// (m_stride apart), nsrc * nx output planes
template <int T, int HS>
static int launch_istft_reg_t(dcs_stft* p, const float2* d_S, int nsrc, int64_t nframes, int64_t ldf, int64_t src_stride,
                              float* d_out, int64_t Lout, int64_t out_stride, cudaStream_t st, const float* d_M = nullptr,
                              int64_t m_stride = 0, int nx = 1) {
  constexpr int GPC = ISTFT_THREADS / T;
  const int hop = 64 * HS;
  const int64_t num_hops = ceil_div64(Lout, hop);
  // hops per group: as long as possible (each group recomputes N/hop-1 halo frames) while every SM
  // still gets its resident warps: ONE full wave of equal-sized groups
  const int64_t target_groups = (int64_t)p->ctx->num_sms * (ISTFT_THREADS / 32) * (32 / T);
  const int nplanes = nsrc * nx;
  int64_t hpg = ceil_div64((int64_t)nplanes * num_hops, target_groups);
  if (hpg < 12) hpg = 12;
  if (hpg > 64) hpg = 64;
  const int64_t groups_per_src = ceil_div64(num_hops, hpg);
  if (d_M) {
    // quads of min(nsrc, GPC) groups share an X row ring; as many quads per CTA as fit next to the mask rings:
    // nsrc = 4 at N = 2048 -> 2 quads, 191 KB; every group busy whenever qw divides GPC and the rings fit
    const int qw = nsrc < GPC ? nsrc : GPC;
    int qpc = GPC / qw;
    while (qpc > 1 && istft_smem_bytes<T>(qpc, true) > SM90_SMEM_OPTIN) --qpc;
    const int64_t quads = groups_per_src * nx * ((nsrc + qw - 1) / qw);
    const unsigned grid = (unsigned)ceil_div64(quads, qpc);
    const size_t smem = istft_smem_bytes<T>(qpc, true);   // 191 232 B + barriers at N = 2048, nsrc = 4
    DCS_TRY(ensure_smem_attr(istft_masked_reg_kernel<T, HS>, (int)smem));
    istft_masked_reg_kernel<T, HS><<<grid, ISTFT_THREADS, smem, st>>>(
        d_S, nframes, ldf, src_stride, d_M, m_stride, nsrc, nx, p->d_wsyn, p->d_w2, p->d_tw, d_out, Lout, out_stride,
        (int)hpg, num_hops, groups_per_src, quads, qw, qpc);
  } else {
    const int64_t total = groups_per_src * nplanes;
    const unsigned grid = (unsigned)ceil_div64(total, GPC);
    const size_t smem = istft_smem_bytes<T>(GPC, false);   // a 2-stage row ring per group: 224 KB (N = 2048)
    DCS_TRY(ensure_smem_attr(istft_reg_kernel<T, HS>, (int)smem));
    istft_reg_kernel<T, HS><<<grid, ISTFT_THREADS, smem, st>>>(
        d_S, nframes, ldf, src_stride, p->d_wsyn, p->d_w2, p->d_tw, d_out, Lout, out_stride, (int)hpg, num_hops,
        groups_per_src, total);
  }
  DCS_CHECK_LAUNCH();
  p->ctx->launches++;
  return DCS_OK;
}

int launch_istft_reg(dcs_stft* p, const float2* d_S, int nsrc, int64_t nframes, int64_t ldf, int64_t src_stride,
                     float* d_out, int64_t Lout, int64_t out_stride, cudaStream_t st, const float* d_M, int64_t m_stride,
                     int nx) {
#define DCS_ISTFT_REG_CASE(NN, HOP) \
  if (p->N == NN && p->hop == HOP)  \
    return launch_istft_reg_t<NN / 64, HOP / 64>(p, d_S, nsrc, nframes, ldf, src_stride, d_out, Lout, out_stride, st, d_M, m_stride, nx);
  DCS_ISTFT_REG_CASE(2048, 512)
  DCS_ISTFT_REG_CASE(2048, 256)
  DCS_ISTFT_REG_CASE(1024, 512)
  DCS_ISTFT_REG_CASE(1024, 256)
#undef DCS_ISTFT_REG_CASE
  DCS_REQUIRE(false, "istft_reg: unsupported frame size / hop");
}

}  // namespace dcs
