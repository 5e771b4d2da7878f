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
// K4 runs ONE CTA per SM so that the twiddle tables, the synthesis window and the interior normalisation -- per-thread
// constants re-read for every frame -- sit in shared memory next to the groups' scratch and row rings.  The plain K4 has
// 8 warps (a row ring per group: 226 560 B at N = 2048).  The masked K4 has 12 warps, three per scheduler, to hide more of
// each frame's dependent chain: at most 168 registers a thread hold the 32-value frame and the R - 1 carried hops of the
// overlap-add window, and the groups transpose through half-size scratch so that 12 mask row rings fit.
constexpr int ISTFT_THREADS = 256;
constexpr int ISTFT_MASKED_THREADS = 384;
__host__ __device__ constexpr int istft_threads(bool masked) { return masked ? ISTFT_MASKED_THREADS : ISTFT_THREADS; }

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

// Shared memory of K4 (bytes): per group its FFT scratch (masked: half of it, FftGroup::forward_split), the twiddle
// tables, the synthesis window and the interior normalisation, the spectrum row rings (RING stages of ROWP float2 per
// quad), masked also a mask row ring per group (RING stages of ROWP floats), then the ring barriers (full / empty per
// quad and stage, masked a full barrier per group and stage) and per group the row offsets of its first frame and
// its frame ranges.
constexpr int ISTFT_RING = 2;
constexpr size_t SM90_SMEM_OPTIN = 232448;   // shared memory a CTA may opt into on sm_90
template <int T>
__host__ __device__ constexpr int istft_rowp() { return (32 * T + 1 + 7) / 8 * 8; }
template <int T, int HS>
__host__ __device__ constexpr size_t istft_smem_bytes(int qpc, bool masked) {
  const int gpc = istft_threads(masked) / T, rowp = istft_rowp<T>();
  const int scr = masked ? FftGroup<T>::HALF_SCRATCH : FftGroup<T>::SCRATCH;
  return ((size_t)gpc * scr + 3 * (size_t)(32 * T) + 32 * HS + (size_t)qpc * ISTFT_RING * rowp) * sizeof(float2) +
         (masked ? (size_t)gpc * ISTFT_RING * rowp * sizeof(float) : 0) +
         ((size_t)qpc * 2 * ISTFT_RING + (masked ? (size_t)gpc * ISTFT_RING : 0) + 6 * (size_t)gpc) * sizeof(uint64_t);
}

// 2 * real_pre_conj(xk, xn, twk) without its four halvings: doubling is exact, and the transform that follows is linear
// in exact steps, so its output is 2V to the bit; K4 folds the 1/2 into the synthesis window
__device__ __forceinline__ float2 real_pre_conj_x2(float2 xk, float2 xn, float2 twk) {
  const float2 e = make_float2(xk.x + xn.x, xk.y - xn.y);
  const float2 d = make_float2(xk.x - xn.x, xk.y + xn.y);
  const float2 o = cmul(d, make_float2(twk.x, -twk.y));
  return make_float2(e.x - o.y, -(e.y + o.x));
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
//
// The overlap-add window: frame n covers padded hops n .. n + R - 1.  Hop n is complete once frame n is added, so only
// the R - 1 hops after it are carried in registers, acc[j - 1] for hop n + j.  The completed hop's sums are formed
// straight into `fin`, the carried ones move down one hop and hop n + R - 1 starts from +0.  (Rotating the carried hops
// statically instead of moving them took a branch over R - 1 copies of the accumulation and spilled at 168 registers.)
// Every hop is still the ascending-frame sum starting from +0, as in istft_norm.
template <int T, int HS, bool MASKED>  // HS = hop / 64: window slots (32 float2 each) per hop
__device__ __forceinline__ void
istft_reg_body(const float2* __restrict__ S, int64_t nframes, int64_t ldf, int64_t src_stride,
               const float* __restrict__ wsyn, const float* __restrict__ w2, const float2* __restrict__ tw,
               float* __restrict__ out, int64_t Lout, int64_t out_stride, int hops_per_group, int64_t num_hops,
               int64_t groups_per_src, int64_t total_quads, const float* __restrict__ Mk, int64_t m_stride, int nsrc,
               int nx, int qw, int qpc) {
  using G = FftGroup<T>;
  constexpr int N2 = G::N2, N = 2 * N2, hop = 64 * HS, R = N / hop, C0 = (N / 2) / hop;
  constexpr int THREADS = istft_threads(MASKED), GPC = THREADS / T;
  constexpr int SCR = MASKED ? G::HALF_SCRATCH : G::SCRATCH;
  constexpr int P = R - 1;                            // carried hops
  constexpr int HV = G::Q * HS;                       // float2 of one hop per lane: slot q * HS + kb % HS
  constexpr int ROWP = istft_rowp<T>();               // float2 per staged row
  constexpr uint32_t XBYTES = (N2 + 2) / 2 * 16;      // 16-byte pieces covering bins 0..N2
  constexpr uint32_t MBYTES = (N2 + 4) / 4 * 16;      // masked: 16-byte pieces covering bins 0..N2 of a mask row
  extern __shared__ __align__(16) float2 scratch[];
  const int tid = threadIdx.x, b = tid % T, gl = tid / T;
  float2* scr = scratch + gl * SCR;
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
  float2 acc[P][HV];
#pragma unroll
  for (int p = 0; p < P; ++p)
#pragma unroll
    for (int i = 0; i < HV; ++i) acc[p][i] = make_float2(0.f, 0.f);
  float* o = out + (int64_t)(MASKED ? msrc * nx + src : src) * out_stride;

  // shared copies of the twiddle table (N entries, exp(-2 pi i j / N)), of the synthesis window and of the interior
  // normalisation
  float2* stw = scratch + GPC * SCR;                    // tw[0..N2): the real-FFT merge twiddles
  float2* stw2 = stw + N2;                              // inter-stage twiddles, lane-contiguous (FftGroup::fill_tw2)
  float2* swsyn = stw2 + N2;                            // pairs (w[2np] / N2, -w[2np+1] / N2), signed for forward_split
  float2* scinv = swsyn + N2;                           // 1 / sum_r win*syn_win, pairs of one hop
  float2* xring = scinv + 32 * HS + (in_quad ? qi : 0) * ISTFT_RING * ROWP;       // this quad's spectrum rows
  float* mring = reinterpret_cast<float*>(scinv + 32 * HS + qpc * ISTFT_RING * ROWP) + gl * ISTFT_RING * ROWP;
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<float*>(scinv + 32 * HS + qpc * ISTFT_RING * ROWP) +
                                               (MASKED ? GPC * ISTFT_RING * ROWP : 0));
  uint64_t* xfull = bars + (in_quad ? qi : 0) * 2 * ISTFT_RING;   // [stage]: the row landed
  uint64_t* xempty = xfull + ISTFT_RING;                           // [stage]: every group of the quad has read it
  uint64_t* mfull = bars + qpc * 2 * ISTFT_RING + gl * ISTFT_RING;
  // loop invariants of the group read back from shared memory instead of being held in registers through the loop (at
  // 168 registers the masked K4 spilled them): the rows of frame n_first in S and in Mk (element offsets, read by the
  // fetching lanes, which write them), the ranges of k below, the output hop h0 and the plane's samples from there on
  int64_t* roff = reinterpret_cast<int64_t*>(bars + qpc * 2 * ISTFT_RING + (MASKED ? GPC * ISTFT_RING : 0)) + 6 * gl;
  int* kr = reinterpret_cast<int*>(roff + 2);
  for (int i = tid; i < N2; i += THREADS) stw[i] = __ldg(tw + i);
  G::fill_tw2(stw2, tw, tid, THREADS);
  // z = conj(V)/N2 is summed as fmaf(w / N, 2V.x, a) and fmaf(-w / N, 2V.y, a), where 2V is the transform of
  // real_pre_conj_x2's doubled merge: scaling by powers of two is exact, so the products are those of w * (V / N2)
  // (window values are far from the subnormal range)
  const float inv_n = 1.0f / (float)N;
  for (int i = tid; i < N2; i += THREADS) {
    const float2 w = __ldg(reinterpret_cast<const float2*>(wsyn) + i);
    const bool neg = MASKED && T == 32 && (i & 48) == 48;   // lane bit 4 and odd kb: forward_split's sign
    const float sx = w.x * inv_n, sy = -w.y * inv_n;
    swsyn[i] = neg ? make_float2(-sx, -sy) : make_float2(sx, sy);
  }
  for (int i = tid; i < 32 * HS; i += THREADS) {   // the interior of the clip: every hop sees the same R frames
    float c0 = 0.f, c1 = 0.f;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const float2 ww = __ldg(reinterpret_cast<const float2*>(w2 + 2 * i + r * hop));
      c0 += ww.x;
      c1 += ww.y;
    }
    scinv[i] = make_float2(c0 == 0.f ? 1.f : 1.f / c0, c1 == 0.f ? 1.f : 1.f / c1);
  }
  if (tid < qpc * ISTFT_RING) {
    tc::mbar_init(bars + (tid / ISTFT_RING) * 2 * ISTFT_RING + tid % ISTFT_RING, 1);
    tc::mbar_init(bars + (tid / ISTFT_RING) * 2 * ISTFT_RING + ISTFT_RING + tid % ISTFT_RING, (uint32_t)qw);
  }
  if (MASKED && tid < GPC * ISTFT_RING) tc::mbar_init(bars + qpc * 2 * ISTFT_RING + tid, 1);
  tc::fence_barrier_init();
  __syncthreads();
  const bool xlane = in_quad && mem == 0 && b == 0;   // the quad's producer lane
  const bool glane = in_quad && b == 0;               // the group's lane for its mask rows and its empty arrivals
  // iteration k walks frame n = n_first + k; the ranges of k below are ints (a group walks at most 64 + R - 1 frames)
  const int64_t n_first = h0 + C0 - R + 1;
  if (b == 0) {
    roff[0] = (int64_t)src * src_stride + n_first * ldf;
    roff[1] = (int64_t)msrc * m_stride + n_first * ldf;
  }
  const int nk = hops_per_group + R - 1;
  auto kclamp = [&](int64_t x) { return (int)(x < 0 ? 0 : x > nk ? nk : x); };
  if (b == 0) {
    kr[0] = kclamp(-n_first);                             // kf0, kf1: frames inside the clip, k in [kf0, kf1)
    kr[1] = kclamp(nframes - n_first);
    kr[2] = kclamp(R - 1 - n_first);                      // ki0: all R frames of hop n exist, k in [ki0, kf1)
    kr[3] = active ? kclamp(num_hops - h0 + R - 1) : 0;   // ks1: hops to store, k in [R - 1, ks1)
  }
  __syncwarp();
  if (b == 0) {
    const int64_t lrem = Lout - h0 * hop;
    roff[4] = reinterpret_cast<int64_t>(o + h0 * hop);                   // output hop h0
    roff[5] = lrem > (int64_t)nk * hop ? (int64_t)nk * hop : lrem;       // samples of the plane from there on
  }
  // frame n_first + k into stage k % RING; frames outside the clip complete their stage with no bytes
  auto fetch_x = [&](int k) {
    const int st = k % ISTFT_RING, kf0 = kr[0], kf1 = kr[1];
    if (k >= ISTFT_RING)   // the stage held frame k - RING: wait until every group of the quad has read it
      tc::mbar_wait_relaxed(xempty + st, (uint32_t)((k / ISTFT_RING - 1) & 1));
    if (k >= kf0 && k < kf1) {
      tc::mbar_arrive_expect_tx(xfull + st, XBYTES);
      tc::bulk_copy_g2s(xring + st * ROWP, S + roff[0] + k * ldf, XBYTES, xfull + st);
    } else {
      tc::mbar_arrive(xfull + st);
    }
  };
  auto fetch_m = [&](int k) {
    const int st = k % ISTFT_RING, kf0 = kr[0], kf1 = kr[1];
    if (k >= kf0 && k < kf1) {
      tc::mbar_arrive_expect_tx(mfull + st, MBYTES);
      tc::bulk_copy_g2s(mring + st * ROWP, Mk + roff[1] + k * ldf, MBYTES, mfull + st);
    } else {
      tc::mbar_arrive(mfull + st);
    }
  };
  if (xlane) fetch_x(0);
  if (MASKED && glane) fetch_m(0);
  for (int k = 0; k < nk; ++k) {
    const bool fvalid = in_quad && k >= kr[0] && k < kr[1];
    const int st = k % ISTFT_RING;
    const uint32_t par = (uint32_t)((k / ISTFT_RING) & 1);
    if (k + 1 < nk) {   // frame k+1 goes in flight before this one is waited for
      if (xlane) fetch_x(k + 1);
      if (MASKED && glane) fetch_m(k + 1);
    }
    const float2* srow = xring + st * ROWP;
    const float* smrow = mring + st * ROWP;
    if (in_quad) {
      tc::mbar_wait(xfull + st, par);
      if constexpr (MASKED) tc::mbar_wait(mfull + st, par);
    }
    float2 v[32];
    if (fvalid) {
#pragma unroll
      for (int a = 0; a < 32; ++a) {
        const int idx = a * T + b;
        float2 xk = srow[idx], xn = srow[N2 - idx];
        if constexpr (MASKED) {   // M * X componentwise: two roundings, never contracted into the sums that follow
          const float mk = smrow[idx], mn = smrow[N2 - idx];
          xk = make_float2(__fmul_rn(mk, xk.x), __fmul_rn(mk, xk.y));
          xn = make_float2(__fmul_rn(mn, xn.x), __fmul_rn(mn, xn.y));
        }
        if (idx == 0) { xk.y = 0.f; xn.y = 0.f; }  // irfft ignores Im of DC and Nyquist
        v[a] = real_pre_conj_x2(xk, xn, stw[idx]);
      }
    } else {   // a frame outside the clip adds zeros (of either sign: every hop sum starts from +0, so no output bit moves)
#pragma unroll
      for (int a = 0; a < 32; ++a) v[a] = make_float2(0.f, 0.f);
    }
    __syncwarp();                    // every lane has consumed the row
    if (glane) tc::mbar_arrive(xempty + st);
    if constexpr (MASKED) G::forward_split(v, scr, stw2, b);
    else G::template forward<true>(v, scr, stw2, b);
    // samples 2n', 2n'+1 of the frame, n' = (b + T q) + 32 kb  <->  v[q*T + kb], in hop j = kb / HS of the frame:
    // hop 0 is complete (fin), hops 1 .. R - 2 add to the carried sums, which move down one hop, and hop R - 1 starts
    float2 fin[HV];
#pragma unroll
    for (int q = 0; q < G::Q; ++q)
#pragma unroll
      for (int kb = 0; kb < T; ++kb) {
        const int j = kb / HS, s = q * HS + kb % HS;
        const float2 w = swsyn[(b + T * q) + 32 * kb];
        const float2 r = v[q * T + kb];
        const float2 prev = j == R - 1 ? make_float2(0.f, 0.f) : acc[j][s];
        float2& a = j == 0 ? fin[s] : acc[j - 1][s];
        a = make_float2(fmaf(w.x, r.x, prev.x), fmaf(w.y, r.y, prev.y));
      }
    // padded samples [n*hop, (n+1)*hop) -> output hop n - C0 = h0 + k - (R - 1), divided by sum(win*syn_win)
    const int4 kq = *reinterpret_cast<const int4*>(kr);
    const int kf0 = kq.x, kf1 = kq.y, ki0 = kq.z, ks1 = kq.w;
    if (k >= R - 1 && k < ks1) {
      const int hk = (k - (R - 1)) * hop;
      float* const oh0 = reinterpret_cast<float*>(roff[4]);
      const int lrem = (int)roff[5];
      auto put = [&](int s, int np, float2 ic) {
        const int oi = hk + 2 * np;
        const float2 a2 = fin[s];
        if (oi + 1 < lrem) {
          *reinterpret_cast<float2*>(oh0 + oi) = make_float2(a2.x * ic.x, a2.y * ic.y);
        } else if (oi < lrem) {
          oh0[oi] = a2.x * ic.x;
        }
      };
      if (k >= ki0 && k < kf1 && hk + hop <= lrem) {   // all R overlapping frames exist, the whole hop is in the plane
#pragma unroll
        for (int q = 0; q < G::Q; ++q)
#pragma unroll
          for (int kb = 0; kb < HS; ++kb) {
            const int np = (b + T * q) + 32 * kb;   // sample pair inside the hop
            const float2 a2 = fin[q * HS + kb], ic = scinv[np];
            *reinterpret_cast<float2*>(oh0 + hk + 2 * np) = make_float2(a2.x * ic.x, a2.y * ic.y);
          }
      } else if (k >= ki0 && k < kf1) {   // the plane's last, partial hop
#pragma unroll
        for (int q = 0; q < G::Q; ++q)
#pragma unroll
          for (int kb = 0; kb < HS; ++kb) {
            const int np = (b + T * q) + 32 * kb;
            put(q * HS + kb, np, scinv[np]);
          }
      } else {   // clip edges: sum win*syn_win over the frames that exist (transform.py:384-392)
        // the sums wait in this lane's part of the (idle) scratch: fewer live registers around the reciprocals
#pragma unroll
        for (int s = 0; s < HV; ++s) scr[s * T + b] = fin[s];
#pragma unroll
        for (int q = 0; q < G::Q; ++q)
#pragma unroll
          for (int kb = 0; kb < HS; ++kb) {
            const int np = (b + T * q) + 32 * kb;
            float c0 = 0.f, c1 = 0.f;
#pragma unroll
            for (int r = 0; r < R; ++r) {
              if (k - r >= kf0 && k - r < kf1) {
                const float2 ww = __ldg(reinterpret_cast<const float2*>(w2 + 2 * np + r * hop));
                c0 += ww.x;
                c1 += ww.y;
              }
            }
            fin[q * HS + kb] = scr[(q * HS + kb) * T + b];
            put(q * HS + kb, np, make_float2(c0 == 0.f ? 1.f : 1.f / c0, c1 == 0.f ? 1.f : 1.f / c1));
          }
      }
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
__global__ void __launch_bounds__(ISTFT_MASKED_THREADS, 1)
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
  const bool masked = d_M != nullptr;
  const int threads = istft_threads(masked), gpc = threads / T;
  const int hop = 64 * HS;
  const int64_t num_hops = ceil_div64(Lout, hop);
  // hops per group: as long as possible (each group recomputes N/hop-1 halo frames) while every SM
  // still gets its resident warps: ONE full wave of equal-sized groups
  const int64_t target_groups = (int64_t)p->ctx->num_sms * gpc;
  const int nplanes = nsrc * nx;
  int64_t hpg = ceil_div64((int64_t)nplanes * num_hops, target_groups);
  if (hpg < 12) hpg = 12;
  if (hpg > 64) hpg = 64;
  const int64_t groups_per_src = ceil_div64(num_hops, hpg);
  if (masked) {
    // quads of min(nsrc, gpc) groups share an X row ring; as many quads per CTA as fit next to the mask rings:
    // nsrc = 4 -> 3 quads at N = 2048 (226 208 B at hop 512), 6 at N = 1024 (216 896 B): every group busy
    const int qw = nsrc < gpc ? nsrc : gpc;
    int qpc = gpc / qw;
    while (qpc > 1 && istft_smem_bytes<T, HS>(qpc, true) > SM90_SMEM_OPTIN) --qpc;
    const int64_t quads = groups_per_src * nx * ((nsrc + qw - 1) / qw);
    const unsigned grid = (unsigned)ceil_div64(quads, qpc);
    const size_t smem = istft_smem_bytes<T, HS>(qpc, true);
    DCS_TRY(ensure_smem_attr(istft_masked_reg_kernel<T, HS>, (int)smem));
    istft_masked_reg_kernel<T, HS><<<grid, threads, smem, st>>>(
        d_S, nframes, ldf, src_stride, d_M, m_stride, nsrc, nx, p->d_wsyn, p->d_w2, p->d_tw, d_out, Lout, out_stride,
        (int)hpg, num_hops, groups_per_src, quads, qw, qpc);
  } else {
    const int64_t total = groups_per_src * nplanes;
    const unsigned grid = (unsigned)ceil_div64(total, gpc);
    const size_t smem = istft_smem_bytes<T, HS>(gpc, false);   // a 2-stage row ring per group: 226 560 B (N = 2048)
    DCS_TRY(ensure_smem_attr(istft_reg_kernel<T, HS>, (int)smem));
    istft_reg_kernel<T, HS><<<grid, threads, smem, st>>>(
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
