// stft.cu -- framed STFT (K1) and inverse STFT + overlap-add (K4) for sm_90a.
//
// Reference semantics: transform.py:277-335 (stft_norm), :337-396 (istft_norm), :243-247 and
// :271-273 (magnitude / phase conventions of compute_file / compute_inverse).
//
// K1: one CTA of N/8 threads transforms `frames_per_cta` consecutive frames.  The hop-512
//     overlapped windows are read straight from the audio (each sample is re-read N/hop times,
//     served by L1/L2 -- HBM sees the audio once), multiplied by the window in registers and
//     fed to the first radix-4 pass; the spectrum leaves through coalesced float2 / float
//     stores as X[T][ldf] and mag[T][ldf] = scale*|X|/sqrt(N).
// K4: one CTA owns `hops_per_cta` output hops of one source: it inverse-transforms every frame
//     that overlaps them (N/hop - 1 halo frames are recomputed instead of using atomics, so
//     the sum order is the reference's frame order and the result is deterministic),
//     accumulates window * frame in shared memory, divides by sum(window*analysisWindow) and
//     stores the samples once.
#include "common.cuh"
#include "fft.cuh"

namespace dcs {

template <int N>
__global__ void __launch_bounds__(N / 8)
stft_kernel(const float* __restrict__ audio, int64_t L, int hop, const float* __restrict__ win,
            const float2* __restrict__ tw, float2* __restrict__ X, float* __restrict__ mag,
            float* __restrict__ phase, int64_t ldf, int64_t T, float mag_scale, int frames_per_cta) {
  constexpr int N2 = N / 2, T4 = N2 / 4, F = N2 + 1;
  __shared__ __align__(16) float2 bufA[N2];
  __shared__ __align__(16) float2 bufB[N2];
  const int tid = threadIdx.x;

  float2 w[4];
#pragma unroll
  for (int m = 0; m < 4; ++m) {
    const int idx = 2 * (tid + m * T4);
    w[m] = make_float2(__ldg(win + idx), __ldg(win + idx + 1));
  }
  const int64_t n0 = (int64_t)blockIdx.x * frames_per_cta;
  for (int f = 0; f < frames_per_cta; ++f) {
    const int64_t n = n0 + f;
    if (n >= T) break;  // uniform over the CTA
    const int64_t base = n * hop - N / 2;
    float2 u[4];
#pragma unroll
    for (int m = 0; m < 4; ++m) {
      const int64_t s = base + 2 * (tid + m * T4);
      const float a0 = (s >= 0 && s < L) ? __ldg(audio + s) : 0.f;
      const float a1 = (s + 1 >= 0 && s + 1 < L) ? __ldg(audio + s + 1) : 0.f;
      u[m] = make_float2(a0 * w[m].x, a1 * w[m].y);
    }
    const float2* Z = fft_forward<N2>(u, bufA, bufB, tw, tid);
    const int64_t row = n * ldf;
#pragma unroll
    for (int m = 0; m < 4; ++m) {
      const int k = tid + m * T4;
      const float2 xk = real_post<N2>(Z, tw, k);
      if (X) X[row + k] = xk;
      if (mag) mag[row + k] = mag_scale * sqrtf(xk.x * xk.x + xk.y * xk.y);
      if (phase) phase[row + k] = atan2f(xk.y, xk.x);
    }
    if (tid == 0) {  // Nyquist bin
      const float2 z0 = Z[0];
      const float v = z0.x - z0.y;
      if (X) X[row + N2] = make_float2(v, 0.f);
      if (mag) mag[row + N2] = mag_scale * fabsf(v);
      if (phase) phase[row + N2] = atan2f(0.f, v);
    }
    if (tid < ldf - F) {  // pad columns
      if (X) X[row + F + tid] = make_float2(0.f, 0.f);
      if (mag) mag[row + F + tid] = 0.f;
      if (phase) phase[row + F + tid] = 0.f;
    }
    __syncthreads();  // the next frame's first pass overwrites bufA
  }
}

// The body of K4 and of its masked variant.  Not masked: CTA (x, y) owns span x of plane y of S (or of the polar pair).
// MASKED: S is the mixture STFT (channel c = y at S + c * src_stride), Mk the masks (source s at Mk + s * m_stride, same
// ldf), the spectrum M_s * X_c is formed as the row is read, output plane s * nx + c; x = span * nsrc + s, so the CTAs of
// the nsrc sources that read the same rows of X are launched next to each other.
template <int N, bool MASKED>
__device__ __forceinline__ void
istft_body(const float2* __restrict__ S, const float* __restrict__ pmag, const float* __restrict__ pphase,
           float polar_scale, int64_t T, int64_t ldf, int64_t src_stride, const float* __restrict__ wsyn,
           const float* __restrict__ w2, const float2* __restrict__ tw, float* __restrict__ out, int64_t Lout,
           int64_t out_stride, int hop, int hops_per_cta, const float* __restrict__ Mk, int64_t m_stride, int nsrc, int nx) {
  constexpr int N2 = N / 2, T4 = N2 / 4;
  __shared__ __align__(16) float2 bufA[N2];
  __shared__ __align__(16) float2 bufB[N2];
  extern __shared__ float acc[];  // hops_per_cta * hop
  const int tid = threadIdx.x;
  const int src = blockIdx.y;
  const int span = hops_per_cta * hop;
  // output sample i (after the first N/2 samples are dropped, transform.py:390) <-> padded
  // coordinate q = i + N/2.  This CTA owns q in [q_lo, q_lo + span).
  const int msrc = MASKED ? (int)(blockIdx.x % nsrc) : 0;
  const int64_t q_lo = (int64_t)(MASKED ? blockIdx.x / nsrc : blockIdx.x) * span + N / 2;
  for (int i = tid; i < span; i += T4) acc[i] = 0.f;
  // frames n with n*hop <= q < n*hop + N for some owned q
  int64_t n_lo = (q_lo - N) / hop + 1;  // q_lo >= N/2 > 0; for q_lo < N this is <= 0 -> clamp
  if (q_lo < N) n_lo = 0;
  int64_t n_hi = (q_lo + span - 1) / hop;
  if (n_hi > T - 1) n_hi = T - 1;
  const float inv_n2 = 1.0f / (float)N2;
  __syncthreads();
  for (int64_t n = n_lo; n <= n_hi; ++n) {
    const int64_t row = (int64_t)src * src_stride + n * ldf;
    float2 u[4];
#pragma unroll
    for (int m = 0; m < 4; ++m) {
      const int k = tid + m * T4;
      float2 xk, xn;
      if constexpr (MASKED) {   // M * X componentwise: two roundings, never contracted into the sums that follow
        const float* mrow = Mk + (int64_t)msrc * m_stride + n * ldf;
        const float mk = mrow[k], mn = mrow[N2 - k];
        xk = S[row + k];
        xn = S[row + N2 - k];
        xk = make_float2(__fmul_rn(mk, xk.x), __fmul_rn(mk, xk.y));
        xn = make_float2(__fmul_rn(mn, xn.x), __fmul_rn(mn, xn.y));
      } else if (S) {
        xk = S[row + k];
        xn = S[row + N2 - k];
      } else {
        float sn, cs;
        const float mk = polar_scale * pmag[row + k];
        sincosf(pphase[row + k], &sn, &cs);
        xk = make_float2(mk * cs, mk * sn);
        const float mn = polar_scale * pmag[row + N2 - k];
        sincosf(pphase[row + N2 - k], &sn, &cs);
        xn = make_float2(mn * cs, mn * sn);
      }
      if (k == 0) { xk.y = 0.f; xn.y = 0.f; }  // irfft ignores Im of DC and Nyquist
      u[m] = real_pre_conj(xk, xn, __ldg(tw + k));
    }
    const float2* R = fft_forward<N2>(u, bufA, bufB, tw, tid);
    const int64_t off = n * hop - q_lo;  // local index of sample t=0 of this frame
#pragma unroll
    for (int m = 0; m < 4; ++m) {
      const int mm = tid + m * T4;
      const float2 r = R[mm];
      const int t0 = 2 * mm;
      const int64_t l0 = off + t0;
      // z = conj(R)/N2 ; x[2m] = Re z, x[2m+1] = Im z
      if (l0 >= 0 && l0 < span) acc[l0] += __ldg(wsyn + t0) * (r.x * inv_n2);
      if (l0 + 1 >= 0 && l0 + 1 < span) acc[l0 + 1] += __ldg(wsyn + t0 + 1) * (-r.y * inv_n2);
    }
    __syncthreads();
  }
  float* o = out + (int64_t)(MASKED ? msrc * nx + src : src) * out_stride;
  for (int i = tid; i < span; i += T4) {
    const int64_t q = q_lo + i;
    const int64_t oi = q - N / 2;
    if (oi >= Lout) break;
    // normalisation: sum of window*analysisWindow over all frames covering q (transform.py:384-386)
    int64_t a = (q < N) ? 0 : (q - N) / hop + 1;
    int64_t b = q / hop;
    if (b > T - 1) b = T - 1;
    float c = 0.f;
    for (int64_t n = a; n <= b; ++n) c += __ldg(w2 + (q - n * hop));
    if (c == 0.f) c = 1.f;  // transform.py:392
    o[oi] = acc[i] / c;
  }
}

template <int N>
__global__ void __launch_bounds__(N / 8)
istft_kernel(const float2* __restrict__ S, const float* __restrict__ pmag, const float* __restrict__ pphase,
             float polar_scale, int64_t T, int64_t ldf, int64_t src_stride, const float* __restrict__ wsyn,
             const float* __restrict__ w2, const float2* __restrict__ tw, float* __restrict__ out, int64_t Lout,
             int64_t out_stride, int hop, int hops_per_cta) {
  istft_body<N, false>(S, pmag, pphase, polar_scale, T, ldf, src_stride, wsyn, w2, tw, out, Lout, out_stride, hop,
                       hops_per_cta, nullptr, 0, 1, 1);
}

// K4 on M_s * X_c: X complex [nx][T][ldf] (x_plane apart), Mk float [nsrc][T][ldf] (m_stride apart); grid (spans * nsrc, nx)
template <int N>
__global__ void __launch_bounds__(N / 8)
istft_masked_kernel(const float2* __restrict__ X, int64_t T, int64_t ldf, int64_t x_plane, const float* __restrict__ Mk,
                    int64_t m_stride, int nsrc, int nx, const float* __restrict__ wsyn, const float* __restrict__ w2,
                    const float2* __restrict__ tw, float* __restrict__ out, int64_t Lout, int64_t out_stride, int hop,
                    int hops_per_cta) {
  istft_body<N, true>(X, nullptr, nullptr, 1.f, T, ldf, x_plane, wsyn, w2, tw, out, Lout, out_stride, hop, hops_per_cta, Mk,
                      m_stride, nsrc, nx);
}

__global__ void pcm_decode_kernel(const int16_t* __restrict__ pcm, int64_t L, int channels, int downmix,
                                  float* __restrict__ audio) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= L) return;
  const float maxv = 32767.0f;
  float v;
  if (channels == 1 || downmix == 0) {
    v = (float)pcm[i * channels] / maxv;
  } else {
    // astype(float)/maxv per channel, then (L+R)/2 (separate_dsd.py:282-286) or L+R (iKala)
    const float l = (float)pcm[i * channels] / maxv, r = (float)pcm[i * channels + 1] / maxv;
    v = (downmix == 1) ? (l + r) * 0.5f : (l + r);
  }
  audio[i] = v;
}

__global__ void pcm_encode_kernel(const float* __restrict__ stems, int64_t L, int64_t stem_stride,
                                  int16_t* __restrict__ out, int64_t out_stride) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= L) return;
  const int s = blockIdx.y;
  // (audio_out*maxn).astype('int16'): C truncation toward zero, wraps instead of clipping
  const float v = stems[(int64_t)s * stem_stride + i] * 32767.0f;
  out[(int64_t)s * out_stride + i] = (int16_t)(int)v;
}

// C-channel stems: interleaved [L][C] samples of format FMT -> C + 1 float planes L apart: the downmix, then channel c at
// plane 1 + c.  Each channel is the format's decode (pcm / 32767 for int16) and the downmix is downmix_kernel's
// expression on those planes, so at C = 2 in int16 it is pcm_decode_kernel's downmix 1 and the network sees what the
// mono call would see
template <int FMT>
__global__ void pcm_decode_channels_kernel(const typename SampleFormat<FMT>::T* __restrict__ pcm, int64_t L, int C,
                                           float* __restrict__ planes) {
  using S = SampleFormat<FMT>;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= L) return;
  const typename S::T* row = pcm + i * C;
  float a = S::decode(row[0]);
  planes[L + i] = a;
  for (int c = 1; c < C; ++c) {
    const float v = S::decode(row[c]);
    planes[(int64_t)(1 + c) * L + i] = v;
    a += v;
  }
  planes[i] = a * (1.0f / (float)C);
}

// nx float planes (stride apart) -> (((a_0 + a_1) + a_2) + ...) * (1.0f / nx), summed in that order: the bits of
// pcm_decode_channels_kernel's downmix, the channel itself at nx = 1
__global__ void downmix_kernel(const float* __restrict__ audio, int nx, int64_t stride, int64_t L, float* __restrict__ mono) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= L) return;
  float a = audio[i];
  for (int c = 1; c < nx; ++c) a += audio[c * stride + i];
  mono[i] = a * (1.0f / (float)nx);
}

constexpr int kPcmEncodeRows = 256;   // rows (samples) of one CTA's tile, one per thread
constexpr int kPcmMaxChannels = 16;

// stem planes (source s, channel c) at stems + (s C + c) * stem_stride -> [nsrc][L][C] samples of format FMT (what
// scipy.io.wavfile.write takes for a C-channel stem), source s at out + s C L, the format's encode (for int16 the
// truncation rule of pcm_encode_kernel); grid (ceil(L / 256), nsrc).  A thread's C samples are not an aligned vector
// for most C, so the tile of 256 interleaved rows is staged in shared memory at the byte offset its destination has
// modulo 16: the 16-byte-aligned middle of the destination then meets 16-byte-aligned shared memory, and each warp
// stores 512 contiguous bytes with 16-byte stores.  The up to 16 / b - 1 values (b bytes each) before the first and
// after the last aligned piece (a source's rows start at s C L b bytes, not always a multiple of 16) go out one value
// at a time.  The shift is counted in values: 2-byte units for int16, 4-byte units otherwise (the output is then
// 4-byte aligned).
template <int FMT>
__global__ void __launch_bounds__(kPcmEncodeRows)
pcm_encode_channels_kernel(const float* __restrict__ stems, int64_t L, int C, int64_t stem_stride,
                           typename SampleFormat<FMT>::T* __restrict__ out) {
  using S = SampleFormat<FMT>;
  using T = typename S::T;
  constexpr int kLog2B = sizeof(T) == 2 ? 1 : 2;                    // log2 of the bytes per value
  constexpr int kV = 16 >> kLog2B;                                  // values per 16 bytes
  __shared__ __align__(16) T tile[kPcmEncodeRows * kPcmMaxChannels + kV];
  const int s = blockIdx.y;
  const int64_t i0 = (int64_t)blockIdx.x * kPcmEncodeRows;
  const int rows = (int)(L - i0 < kPcmEncodeRows ? L - i0 : kPcmEncodeRows);
  T* dst = out + ((int64_t)s * L + i0) * C;                         // the tile's first value
  const int shift = (int)(((uintptr_t)dst & 15) >> kLog2B);         // in values
  if ((int)threadIdx.x < rows) {
    const float* src = stems + (int64_t)s * C * stem_stride + i0 + threadIdx.x;
    for (int c = 0; c < C; ++c)
      tile[shift + threadIdx.x * C + c] = S::encode(src[(int64_t)c * stem_stride]);
  }
  __syncthreads();
  const int n = rows * C;                                           // values of the tile
  const int head = min(n, (kV - shift) & (kV - 1));                 // values before the first 16-byte boundary
  const int nvec = (n - head) >> (4 - kLog2B);
  const int tail0 = head + nvec * kV;
  const uint4* vsrc = reinterpret_cast<const uint4*>(tile + shift + head);
  uint4* vdst = reinterpret_cast<uint4*>(dst + head);
  for (int k = threadIdx.x; k < nvec; k += kPcmEncodeRows) vdst[k] = vsrc[k];
  if ((int)threadIdx.x < head) dst[threadIdx.x] = tile[shift + threadIdx.x];
  const int t = tail0 + (int)threadIdx.x;
  if (t < n) dst[t] = tile[shift + t];
}

// Packed 24-bit PCM (DCS_SAMPLE_I24) has no aligned vector of one sample, so both kernels count the tile of 256 rows in
// bytes (768 C, a multiple of 16) and stage it in shared memory at the byte offset its global address has modulo 16:
// the 16-byte-aligned middle then moves with 16-byte loads or stores, and the under 16 bytes before and after it one
// byte at a time.  The global buffer may sit at any address.
constexpr int kPcm24TileBytes = kPcmEncodeRows * kPcmMaxChannels * 3;

// the bytes [0, n) at g <-> tile + shift, shift = g mod 16; kLoad: global -> tile, else tile -> global
template <bool kLoad>
__device__ __forceinline__ void pcm24_move(uint8_t* tile, int shift, uint8_t* g, int n) {
  const int head = min(n, (16 - shift) & 15);
  const int nvec = (n - head) >> 4;
  const int tail0 = head + nvec * 16;
  uint4* vt = reinterpret_cast<uint4*>(tile + shift + head);
  uint4* vg = reinterpret_cast<uint4*>(g + head);
  for (int k = threadIdx.x; k < nvec; k += blockDim.x) {
    if constexpr (kLoad) vt[k] = __ldg(vg + k);
    else vg[k] = vt[k];
  }
  const int t = (int)threadIdx.x < head ? (int)threadIdx.x : tail0 + (int)threadIdx.x - head;
  if ((int)threadIdx.x < head + (n - tail0)) {
    if constexpr (kLoad) tile[shift + t] = g[t];
    else g[t] = tile[shift + t];
  }
}

// pcm_decode_channels_kernel for DCS_SAMPLE_I24: the tile's 768 C bytes staged as above, then each thread decodes its
// row from shared memory and writes the C + 1 planes with the same expressions in the same order
__global__ void __launch_bounds__(kPcmEncodeRows)
pcm24_decode_channels_kernel(const uint8_t* __restrict__ pcm, int64_t L, int C, float* __restrict__ planes) {
  using S = SampleFormat<DCS_SAMPLE_I24>;
  __shared__ __align__(16) uint8_t tile[kPcm24TileBytes + 16];
  const int64_t i0 = (int64_t)blockIdx.x * kPcmEncodeRows;
  const int rows = (int)(L - i0 < kPcmEncodeRows ? L - i0 : kPcmEncodeRows);
  uint8_t* src = const_cast<uint8_t*>(pcm) + i0 * C * 3;
  const int shift = (int)((uintptr_t)src & 15);
  pcm24_move<true>(tile, shift, src, rows * C * 3);
  __syncthreads();
  if ((int)threadIdx.x >= rows) return;
  const int64_t i = i0 + threadIdx.x;
  const Pcm24* row = reinterpret_cast<const Pcm24*>(tile + shift) + threadIdx.x * C;
  float a = S::decode(row[0]);
  planes[L + i] = a;
  for (int c = 1; c < C; ++c) {
    const float v = S::decode(row[c]);
    planes[(int64_t)(1 + c) * L + i] = v;
    a += v;
  }
  planes[i] = a * (1.0f / (float)C);
}

// pcm_encode_channels_kernel for DCS_SAMPLE_I24: each thread encodes its row into the tile, which then goes out as above
__global__ void __launch_bounds__(kPcmEncodeRows)
pcm24_encode_channels_kernel(const float* __restrict__ stems, int64_t L, int C, int64_t stem_stride,
                             uint8_t* __restrict__ out) {
  using S = SampleFormat<DCS_SAMPLE_I24>;
  __shared__ __align__(16) uint8_t tile[kPcm24TileBytes + 16];
  const int s = blockIdx.y;
  const int64_t i0 = (int64_t)blockIdx.x * kPcmEncodeRows;
  const int rows = (int)(L - i0 < kPcmEncodeRows ? L - i0 : kPcmEncodeRows);
  uint8_t* dst = out + ((int64_t)s * L + i0) * C * 3;
  const int shift = (int)((uintptr_t)dst & 15);
  if ((int)threadIdx.x < rows) {
    const float* src = stems + (int64_t)s * C * stem_stride + i0 + threadIdx.x;
    Pcm24* row = reinterpret_cast<Pcm24*>(tile + shift) + threadIdx.x * C;
    for (int c = 0; c < C; ++c) row[c] = S::encode(src[(int64_t)c * stem_stride]);
  }
  __syncthreads();
  pcm24_move<false>(tile, shift, dst, rows * C * 3);
}

template <int N>
static int launch_stft_n(dcs_stft* p, const float* d_audio, int64_t L, float2* d_X, float* d_mag, float* d_phase,
                         float mag_scale, int64_t ldf, int64_t T, cudaStream_t st) {
  const int fpc = 8;
  const unsigned grid = (unsigned)ceil_div64(T, fpc);
  stft_kernel<N><<<grid, N / 8, 0, st>>>(d_audio, L, p->hop, p->d_win, p->d_tw, d_X, d_mag, d_phase, ldf, T,
                                          mag_scale / sqrtf((float)N), fpc);
  DCS_CHECK_LAUNCH();
  p->ctx->launches++;
  return DCS_OK;
}

int launch_stft(dcs_stft* p, const float* d_audio, int64_t L, float2* d_X, float* d_mag, float* d_phase,
                float mag_scale, int64_t ldf, cudaStream_t st) {
  const int64_t T = dcs_num_frames(L, p->hop);
  DCS_REQUIRE(ldf >= p->N / 2 + 1, "ldf %lld < F %d", (long long)ldf, p->N / 2 + 1);
  DCS_REQUIRE(ldf - (p->N / 2 + 1) <= 16, "ldf %lld pads more than 16 columns", (long long)ldf);
  switch (p->N) {
    case 256: return launch_stft_n<256>(p, d_audio, L, d_X, d_mag, d_phase, mag_scale, ldf, T, st);
    case 512: return launch_stft_n<512>(p, d_audio, L, d_X, d_mag, d_phase, mag_scale, ldf, T, st);
    case 1024:
    case 2048: return launch_stft_reg(p, d_audio, L, d_X, d_mag, d_phase, mag_scale, ldf, T, st);
    case 4096: return launch_stft_n<4096>(p, d_audio, L, d_X, d_mag, d_phase, mag_scale, ldf, T, st);
  }
  DCS_REQUIRE(false, "unsupported frame size %d", p->N);
}

template <int N>
static int launch_istft_n(dcs_stft* p, const float2* d_S, const float* d_mag, const float* d_phase, float polar_scale,
                          int nsrc, int64_t T, int64_t ldf, int64_t src_stride, float* d_out, int64_t Lout,
                          int64_t out_stride, cudaStream_t st, const float* d_M = nullptr, int64_t m_stride = 0, int nx = 1) {
  // enough hops per CTA to amortise the N/hop-1 halo frames, small enough for many CTAs
  int hpc = 4 * (p->N / p->hop);
  if (hpc < 8) hpc = 8;
  while ((size_t)hpc * p->hop * sizeof(float) > 64 * 1024 && hpc > 1) hpc /= 2;
  const int64_t span = (int64_t)hpc * p->hop;
  const size_t dyn = (size_t)span * sizeof(float);
  if (d_M) {   // d_S: the mixture STFT of nx channels; nsrc masks
    dim3 grid((unsigned)(ceil_div64(Lout, span) * nsrc), (unsigned)nx);
    DCS_TRY(ensure_smem_attr(istft_masked_kernel<N>, 96 * 1024));
    istft_masked_kernel<N><<<grid, N / 8, dyn, st>>>(d_S, T, ldf, src_stride, d_M, m_stride, nsrc, nx, p->d_wsyn, p->d_w2,
                                                     p->d_tw, d_out, Lout, out_stride, p->hop, hpc);
    DCS_CHECK_LAUNCH();
    p->ctx->launches++;
    return DCS_OK;
  }
  dim3 grid((unsigned)ceil_div64(Lout, span), (unsigned)nsrc);
  DCS_TRY(ensure_smem_attr(istft_kernel<N>, 96 * 1024));
  istft_kernel<N><<<grid, N / 8, dyn, st>>>(d_S, d_mag, d_phase, polar_scale, T, ldf, src_stride, p->d_wsyn, p->d_w2,
                                            p->d_tw, d_out, Lout, out_stride, p->hop, hpc);
  DCS_CHECK_LAUNCH();
  p->ctx->launches++;
  return DCS_OK;
}

int launch_istft(dcs_stft* p, const float2* d_S, const float* d_mag, const float* d_phase, float polar_scale,
                 int nsrc, int64_t T, int64_t ldf, int64_t src_stride, float* d_out, int64_t Lout,
                 int64_t out_stride, cudaStream_t st, const float* d_M, int64_t m_stride, int nx) {
  DCS_REQUIRE(Lout <= (T - 1) * p->hop + p->N - p->N / 2, "num_out %lld exceeds the istft length", (long long)Lout);
  if (Lout <= 0 || nsrc <= 0 || nx <= 0) return DCS_OK;
  // the register path stages rows with 16-byte cp.async: aligned spectrum rows, and aligned mask rows of whole pieces
  const bool mask_rows_ok = !d_M || (ldf % 4 == 0 && m_stride % 4 == 0 && (uintptr_t)d_M % 16 == 0 && ldf >= p->N / 2 + 4);
  if (d_S && istft_reg_supported(p, d_out, out_stride) && ldf % 2 == 0 &&
      src_stride % 2 == 0 && ((uintptr_t)d_S % 16 == 0) && ldf >= (p->N / 2 + 2) / 2 * 2 && mask_rows_ok)
    return launch_istft_reg(p, d_S, nsrc, T, ldf, src_stride, d_out, Lout, out_stride, st, d_M, m_stride, nx);
#define DCS_ISTFT_CASE(NN) \
  case NN: return launch_istft_n<NN>(p, d_S, d_mag, d_phase, polar_scale, nsrc, T, ldf, src_stride, d_out, Lout, out_stride, st, d_M, m_stride, nx);
  switch (p->N) {
    DCS_ISTFT_CASE(256)
    DCS_ISTFT_CASE(512)
    DCS_ISTFT_CASE(1024)
    DCS_ISTFT_CASE(2048)
    DCS_ISTFT_CASE(4096)
  }
#undef DCS_ISTFT_CASE
  DCS_REQUIRE(false, "unsupported frame size %d", p->N);
}

int launch_pcm_decode(dcs_ctx* ctx, const int16_t* d_pcm, int64_t L, int channels, int downmix, float* d_audio,
                      cudaStream_t st) {
  if (L <= 0) return DCS_OK;
  pcm_decode_kernel<<<(unsigned)ceil_div64(L, 256), 256, 0, st>>>(d_pcm, L, channels, downmix, d_audio);
  DCS_CHECK_LAUNCH();
  ctx->launches++;
  return DCS_OK;
}

template <int FMT>
static void pcm_decode_channels_as(const void* d_in, int64_t L, int C, float* d_planes, cudaStream_t st) {
  pcm_decode_channels_kernel<FMT><<<(unsigned)ceil_div64(L, 256), 256, 0, st>>>(
      static_cast<const typename SampleFormat<FMT>::T*>(d_in), L, C, d_planes);
}

template <int FMT>
static void pcm_encode_channels_as(const float* d_stems, int64_t L, int nsrc, int C, int64_t stem_stride, void* d_out,
                                   cudaStream_t st) {
  dim3 grid((unsigned)ceil_div64(L, kPcmEncodeRows), (unsigned)nsrc);
  pcm_encode_channels_kernel<FMT><<<grid, kPcmEncodeRows, 0, st>>>(d_stems, L, C, stem_stride,
                                                                   static_cast<typename SampleFormat<FMT>::T*>(d_out));
}

int launch_pcm_decode_channels(dcs_ctx* ctx, int fmt, const void* d_in, int64_t L, int C, float* d_planes, cudaStream_t st) {
  if (L <= 0) return DCS_OK;
  DCS_REQUIRE(C >= 1 && C <= kPcmMaxChannels, "pcm_decode_channels: %d channels not in [1, %d]", C, kPcmMaxChannels);
  DCS_REQUIRE(sample_bytes(fmt) > 0 && (uintptr_t)d_in % sample_align(fmt) == 0,
              "pcm_decode_channels: format %d, or input not aligned to its samples", fmt);
  switch (fmt) {
    case DCS_SAMPLE_I16: pcm_decode_channels_as<DCS_SAMPLE_I16>(d_in, L, C, d_planes, st); break;
    case DCS_SAMPLE_I32: pcm_decode_channels_as<DCS_SAMPLE_I32>(d_in, L, C, d_planes, st); break;
    case DCS_SAMPLE_I24:
      pcm24_decode_channels_kernel<<<(unsigned)ceil_div64(L, kPcmEncodeRows), kPcmEncodeRows, 0, st>>>(
          static_cast<const uint8_t*>(d_in), L, C, d_planes);
      break;
    default: pcm_decode_channels_as<DCS_SAMPLE_F32>(d_in, L, C, d_planes, st); break;
  }
  DCS_CHECK_LAUNCH();
  ctx->launches++;
  return DCS_OK;
}

// the masked spectra of the stems-from-masks route, for the spectrum tap: S[s][t][f] = M_s[t][f] * X[t][f] componentwise
// (the lone rounded products the masked inverse STFT forms) for f < F, 0 in the pad columns
__global__ void masked_spectra_kernel(const float* __restrict__ M, const float2* __restrict__ X, int64_t plane, int64_t ldf, int F,
                                      int64_t n, float2* __restrict__ S) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t e = i % plane, f = e % ldf;
  if (f < F) {
    const float m = M[i];
    const float2 x = X[e];
    S[i] = make_float2(__fmul_rn(m, x.x), __fmul_rn(m, x.y));
  } else {
    S[i] = make_float2(0.f, 0.f);
  }
}

int launch_masked_spectra(dcs_ctx* ctx, const float* d_M, const float2* d_X, int nsrc, int64_t plane, int64_t ldf, int F,
                          float2* d_S, cudaStream_t st) {
  const int64_t n = (int64_t)nsrc * plane;
  if (n <= 0) return DCS_OK;
  masked_spectra_kernel<<<(unsigned)ceil_div64(n, 256), 256, 0, st>>>(d_M, d_X, plane, ldf, F, n, d_S);
  DCS_CHECK_LAUNCH();
  ctx->launches++;
  return DCS_OK;
}

int launch_downmix(dcs_ctx* ctx, const float* d_audio, int nx, int64_t audio_stride, int64_t L, float* d_mono, cudaStream_t st) {
  if (L <= 0) return DCS_OK;
  downmix_kernel<<<(unsigned)ceil_div64(L, 256), 256, 0, st>>>(d_audio, nx, audio_stride, L, d_mono);
  DCS_CHECK_LAUNCH();
  ctx->launches++;
  return DCS_OK;
}

int launch_pcm_encode_channels(dcs_ctx* ctx, int fmt, const float* d_stems, int64_t L, int nsrc, int C, int64_t stem_stride,
                               void* d_out, cudaStream_t st) {
  if (L <= 0) return DCS_OK;
  DCS_REQUIRE(C >= 1 && C <= kPcmMaxChannels, "pcm_encode_channels: %d channels not in [1, %d]", C, kPcmMaxChannels);
  DCS_REQUIRE(sample_bytes(fmt) > 0 && (uintptr_t)d_out % sample_align(fmt) == 0,
              "pcm_encode_channels: format %d, or output not aligned to its samples", fmt);
  switch (fmt) {
    case DCS_SAMPLE_I16: pcm_encode_channels_as<DCS_SAMPLE_I16>(d_stems, L, nsrc, C, stem_stride, d_out, st); break;
    case DCS_SAMPLE_I32: pcm_encode_channels_as<DCS_SAMPLE_I32>(d_stems, L, nsrc, C, stem_stride, d_out, st); break;
    case DCS_SAMPLE_I24:
      pcm24_encode_channels_kernel<<<dim3((unsigned)ceil_div64(L, kPcmEncodeRows), (unsigned)nsrc), kPcmEncodeRows, 0, st>>>(
          d_stems, L, C, stem_stride, static_cast<uint8_t*>(d_out));
      break;
    default: pcm_encode_channels_as<DCS_SAMPLE_F32>(d_stems, L, nsrc, C, stem_stride, d_out, st); break;
  }
  DCS_CHECK_LAUNCH();
  ctx->launches++;
  return DCS_OK;
}

int launch_pcm_encode(dcs_ctx* ctx, const float* d_stems, int64_t L, int nsrc, int64_t stem_stride, int16_t* d_out,
                      int64_t out_stride, cudaStream_t st) {
  if (L <= 0) return DCS_OK;
  dim3 grid((unsigned)ceil_div64(L, 256), (unsigned)nsrc);
  pcm_encode_kernel<<<grid, 256, 0, st>>>(d_stems, L, stem_stride, d_out, out_stride);
  DCS_CHECK_LAUNCH();
  ctx->launches++;
  return DCS_OK;
}

}  // namespace dcs
