// wiener.cu -- multichannel Wiener post-filter of stereo stems with EM re-estimation of each source's spatial
// covariance (Duong, Vincent & Gribonval 2010; the filter the reference's util.py:633-719 `mwf` set out to be).
//
// Planes: mixture channel c at X + c * x_plane, stem (source j, channel c) at S + (2 j + c) * src_stride, each
// complex[T][ldf]; bins f < F are filtered in place, pad bins are never touched.  Per iteration:
//   v_j(t,f) = (|y_jL|^2 + |y_jR|^2) / 2
//   R_j(f)   = sum_t y_j y_j^H / (eps s^2 + sum_t v_j)        eps = 2^-23, s = max(1, max|x| / 10)
//   C(t,f)   = sum_j v_j R_j + sqrt(eps) s^2 I
//   y_j      <- v_j R_j C^-1 x
// C is near rank one wherever one source dominates or the channels nearly agree (cond ~ 1e6 at full scale), so
// C, its adjugate and determinant and v R C^-1 x are fp64 in registers; the planes stay fp32 in HBM.
//
// One thread per bin walks a chunk of kWienerFrames frames; the grid is bin tiles x frame chunks.  The sums over
// t are per-chunk fp64 partials reduced in chunk order: no atomics, the same bits on every run.
//
// Sliding window (radius W >= 1): chunk c takes R_j(f; c) and s_c from the chunks max(0, c-W) .. min(n-1, c+W)
// instead of the whole clip.  Each chunk's window sum is formed directly from the partials, in ascending chunk order,
// so a chunk's R is the same bits in any segment that holds its window, and W >= n-1 gives the whole-clip bits.
//
// C channels (3 .. 8, wiener_ch_*): stem (j, c) at S + (j C + c) * src_stride, v_j = (1/C) sum_c |y_jc|^2, C x C
// covariances factored L D L^H in fp64; the same partials (C^2 per source and bin), reduces, chunks and windows.
#include "common.cuh"

namespace dcs {
namespace {

constexpr int kWienerBins = 128;     // threads per block: consecutive bins, coalesced float2 rows
constexpr int kWienerFrames = DCS_WIENER_CHUNK_FRAMES;   // frames per chunk: partials are 32 B per (source, bin) per 128 frames
constexpr int kReduceThreads = 256;
constexpr double kEps = 1.1920928955078125e-07;   // 2^-23 = FLT_EPSILON

struct WienerArgs {
  const float2* X; int64_t x_plane;
  float2* S; int64_t src_stride;
  int64_t T, ldf;
  int F, nchunks, ntiles;
  double* part;    // [nchunks][nsrc][4][F]: per-chunk sums of |yL|^2, |yR|^2, Re yL conj(yR), Im yL conj(yR)
  double* Q;       // [nsrc][4][F]: the same summed over all chunks (chunk order); windowed: [nchunks][nsrc][4][F]
  double* pmax;    // [nchunks][ntiles]: per-block max of |x|^2 over both channels
  double* scale;   // [1]: s; windowed: [nchunks]: s_c
  int64_t q_stride;   // doubles between the Q of consecutive chunks: 0 (one Q for the clip) or nsrc * 4 * F
  int s_stride;       // the same for the scale: 0 or 1
};

__device__ __forceinline__ void accumulate(double* q, float2 l, float2 r) {
  const double a = l.x, b = l.y, c = r.x, d = r.y;
  q[0] += fma(a, a, b * b);
  q[1] += fma(c, c, d * d);
  q[2] += fma(a, c, b * d);
  q[3] += fma(b, c, -(a * d));
}

template <int NSRC>
__device__ __forceinline__ void store_partials(const WienerArgs& a, const double (&acc)[NSRC][4], int f) {
  double* p = a.part + (int64_t)blockIdx.y * NSRC * 4 * a.F + f;
#pragma unroll
  for (int j = 0; j < NSRC; ++j)
#pragma unroll
    for (int q = 0; q < 4; ++q) p[(int64_t)(j * 4 + q) * a.F] = acc[j][q];
}

// the network's stems -> per-chunk partial sums, and the per-block max of |x|^2.  MASKED: the stems are formed here,
// y_jc = M_j * x_c per component (the product the masked inverse STFT forms), source j's float mask plane at
// M + j * m_stride, and stored to S
template <int NSRC, bool MASKED>
__global__ void __launch_bounds__(kWienerBins) wiener_init_kernel(const WienerArgs a, const float* __restrict__ M, int64_t m_stride) {
  const int f = blockIdx.x * kWienerBins + threadIdx.x;
  const int64_t t0 = (int64_t)blockIdx.y * kWienerFrames, t1 = min(a.T, t0 + kWienerFrames);
  double mx = 0.0;
  if (f < a.F) {
    double acc[NSRC][4];
#pragma unroll
    for (int j = 0; j < NSRC; ++j)
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[j][q] = 0.0;
    for (int64_t t = t0; t < t1; ++t) {
      const int64_t o = t * a.ldf + f;
      const float2 xl = a.X[o], xr = a.X[a.x_plane + o];
      mx = fmax(mx, fmax((double)xl.x * xl.x + (double)xl.y * xl.y, (double)xr.x * xr.x + (double)xr.y * xr.y));
#pragma unroll
      for (int j = 0; j < NSRC; ++j) {
        if constexpr (MASKED) {
          const float m = M[j * m_stride + o];
          const float2 l = make_float2(__fmul_rn(m, xl.x), __fmul_rn(m, xl.y)), r = make_float2(__fmul_rn(m, xr.x), __fmul_rn(m, xr.y));
          a.S[(2 * j) * a.src_stride + o] = l;
          a.S[(2 * j + 1) * a.src_stride + o] = r;
          accumulate(acc[j], l, r);
        } else {
          accumulate(acc[j], a.S[(2 * j) * a.src_stride + o], a.S[(2 * j + 1) * a.src_stride + o]);
        }
      }
    }
    store_partials<NSRC>(a, acc, f);
  }
  __shared__ double wmax[kWienerBins / 32];
#pragma unroll
  for (int k = 16; k > 0; k >>= 1) mx = fmax(mx, __shfl_down_sync(0xffffffffu, mx, k));
  if ((threadIdx.x & 31) == 0) wmax[threadIdx.x >> 5] = mx;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < kWienerBins / 32; ++w) mx = fmax(mx, wmax[w]);
    a.pmax[(int64_t)blockIdx.y * a.ntiles + blockIdx.x] = mx;
  }
}

// partials -> Q in chunk order, one thread per (source, quantity, bin); the extra last block: s from the maxima
__global__ void __launch_bounds__(kReduceThreads) wiener_reduce_kernel(const WienerArgs a, int64_t n) {
  if (blockIdx.x == gridDim.x - 1) {
    __shared__ double wmax[kReduceThreads / 32];
    double mx = 0.0;
    for (int64_t i = threadIdx.x; i < (int64_t)a.nchunks * a.ntiles; i += kReduceThreads) mx = fmax(mx, a.pmax[i]);
#pragma unroll
    for (int k = 16; k > 0; k >>= 1) mx = fmax(mx, __shfl_down_sync(0xffffffffu, mx, k));
    if ((threadIdx.x & 31) == 0) wmax[threadIdx.x >> 5] = mx;
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < kReduceThreads / 32; ++w) mx = fmax(mx, wmax[w]);
      *a.scale = fmax(1.0, sqrt(mx) / 10.0);
    }
    return;
  }
  const int64_t e = (int64_t)blockIdx.x * kReduceThreads + threadIdx.x;
  if (e >= n) return;
  double sum = 0.0;
#pragma unroll 8
  for (int c = 0; c < a.nchunks; ++c) sum += a.part[(int64_t)c * n + e];
  a.Q[e] = sum;
}

// partials -> the Q of chunk c = blockIdx.y over its window c-W .. c+W (clipped to the clip), summed directly in
// ascending chunk order, one thread per (source, quantity, bin); the extra last block of each row: s_c from the
// maxima of the window's chunks.  radius <= nchunks - 1 (the host clips it; a larger radius is the same window)
__global__ void __launch_bounds__(kReduceThreads) wiener_reduce_window_kernel(const WienerArgs a, int64_t n, int radius) {
  const int c = blockIdx.y;
  const int c0 = max(0, c - radius), c1 = min(a.nchunks - 1, c + radius);
  if (blockIdx.x == gridDim.x - 1) {
    __shared__ double wmax[kReduceThreads / 32];
    double mx = 0.0;
    for (int64_t i = (int64_t)c0 * a.ntiles + threadIdx.x; i < (int64_t)(c1 + 1) * a.ntiles; i += kReduceThreads)
      mx = fmax(mx, a.pmax[i]);
#pragma unroll
    for (int k = 16; k > 0; k >>= 1) mx = fmax(mx, __shfl_down_sync(0xffffffffu, mx, k));
    if ((threadIdx.x & 31) == 0) wmax[threadIdx.x >> 5] = mx;
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < kReduceThreads / 32; ++w) mx = fmax(mx, wmax[w]);
      a.scale[c] = fmax(1.0, sqrt(mx) / 10.0);
    }
    return;
  }
  const int64_t e = (int64_t)blockIdx.x * kReduceThreads + threadIdx.x;
  if (e >= n) return;
  double sum = 0.0;
#pragma unroll 8
  for (int k = c0; k <= c1; ++k) sum += a.part[(int64_t)k * n + e];
  a.Q[(int64_t)c * n + e] = sum;
}

// one EM iteration in place; STATS: also the next iteration's partial sums of the stems it stores.  Chunk
// blockIdx.y reads its Q and scale at q_stride / s_stride (0: the clip's)
template <int NSRC, bool STATS>
__global__ void __launch_bounds__(kWienerBins) wiener_em_kernel(const WienerArgs a) {
  const int f = blockIdx.x * kWienerBins + threadIdx.x;
  if (f >= a.F) return;
  const int64_t t0 = (int64_t)blockIdx.y * kWienerFrames, t1 = min(a.T, t0 + kWienerFrames);
  const double* Q = a.Q + (int64_t)blockIdx.y * a.q_stride;
  const double s = a.scale[(int64_t)blockIdx.y * a.s_stride];
  const double s2 = s * s, es2 = kEps * s2, ds2 = sqrt(kEps) * s2;
  double r[NSRC][4];   // R_j(f): [0][0], [1][1], Re [0][1], Im [0][1]
#pragma unroll
  for (int j = 0; j < NSRC; ++j) {
#pragma unroll
    for (int q = 0; q < 4; ++q) r[j][q] = Q[(int64_t)(j * 4 + q) * a.F + f];
    const double inv = 1.0 / (es2 + 0.5 * (r[j][0] + r[j][1]));
#pragma unroll
    for (int q = 0; q < 4; ++q) r[j][q] *= inv;
  }
  double acc[NSRC][4];
#pragma unroll
  for (int j = 0; j < NSRC; ++j)
#pragma unroll
    for (int q = 0; q < 4; ++q) acc[j][q] = 0.0;
  for (int64_t t = t0; t < t1; ++t) {
    const int64_t o = t * a.ldf + f;
    const float2 xl = a.X[o], xr = a.X[a.x_plane + o];
    double v[NSRC];
#pragma unroll
    for (int j = 0; j < NSRC; ++j) {
      const float2 l = a.S[(2 * j) * a.src_stride + o], rr = a.S[(2 * j + 1) * a.src_stride + o];
      v[j] = 0.5 * (((double)l.x * l.x + (double)l.y * l.y) + ((double)rr.x * rr.x + (double)rr.y * rr.y));
    }
    // C = sum_j v_j R_j + delta s^2 I: [[c11, c12], [conj(c12), c22]].  The fma trees of the two channels mirror
    // each other, so that equal channels (c11 = c22, Im c12 = 0) give bit-identical outputs
    double c11 = 0.0, c22 = 0.0, c12r = 0.0, c12i = 0.0;
#pragma unroll
    for (int j = 0; j < NSRC; ++j) {
      c11 = fma(v[j], r[j][0], c11);
      c22 = fma(v[j], r[j][1], c22);
      c12r = fma(v[j], r[j][2], c12r);
      c12i = fma(v[j], r[j][3], c12i);
    }
    c11 += ds2;
    c22 += ds2;
    const double idet = 1.0 / fma(c11, c22, -fma(c12r, c12r, c12i * c12i));
    // z = C^-1 x = adj(C) x / det
    const double x1r = xl.x, x1i = xl.y, x2r = xr.x, x2i = xr.y;
    const double z1r = fma(c22, x1r, -fma(c12r, x2r, -(c12i * x2i))) * idet;
    const double z1i = fma(c22, x1i, -fma(c12r, x2i, c12i * x2r)) * idet;
    const double z2r = fma(c11, x2r, -fma(c12r, x1r, c12i * x1i)) * idet;
    const double z2i = fma(c11, x2i, -fma(c12r, x1i, -(c12i * x1r))) * idet;
#pragma unroll
    for (int j = 0; j < NSRC; ++j) {
      // y_j = v_j R_j z
      const double r0 = r[j][0], r1 = r[j][1], r2 = r[j][2], r3 = r[j][3];
      const double ylr = v[j] * fma(r0, z1r, fma(r2, z2r, -(r3 * z2i))), yli = v[j] * fma(r0, z1i, fma(r2, z2i, r3 * z2r));
      const double yrr = v[j] * fma(r1, z2r, fma(r2, z1r, r3 * z1i)), yri = v[j] * fma(r1, z2i, fma(r2, z1i, -(r3 * z1r)));
      const float2 l = make_float2((float)ylr, (float)yli), rr = make_float2((float)yrr, (float)yri);
      a.S[(2 * j) * a.src_stride + o] = l;
      a.S[(2 * j + 1) * a.src_stride + o] = rr;
      if (STATS) accumulate(acc[j], l, rr);
    }
  }
  if (STATS) store_partials<NSRC>(a, acc, f);
}

// ---- C channels, 3 <= NCH <= 8.  The same filter with C x C algebra: R_j and the partial sums are NSRC * NCH^2 doubles
// per bin (up to 256 each), more than registers hold, so each thread keeps them in a private column of shared memory,
// laid out [entry][bin]: a warp's 32 lanes read 32 consecutive doubles.  One warp per block, so no barrier is needed.
// Entries of a Hermitian C x C matrix, packed in NCH^2 reals: the NCH diagonal entries, then Re and Im of [a][b] for
// a < b in row-major order -- at NCH = 2 the 4-entry order of the stereo kernels.
constexpr int kChBins = 32;

__host__ __device__ constexpr int pair_entry(int a, int b, int nch) { return nch + 2 * (a * nch - a * (a + 1) / 2 + (b - a - 1)); }

// q: a thread's column of NCH^2 partial sums (stride kChBins); adds y y^H of one frame
template <int NCH>
__device__ __forceinline__ void accumulate_ch(double* q, const float2 (&y)[NCH]) {
#pragma unroll
  for (int c = 0; c < NCH; ++c) q[c * kChBins] += fma((double)y[c].x, (double)y[c].x, (double)y[c].y * y[c].y);
#pragma unroll
  for (int p = 0; p < NCH; ++p)
#pragma unroll
    for (int b = p + 1; b < NCH; ++b) {
      const double ar = y[p].x, ai = y[p].y, br = y[b].x, bi = y[b].y;
      const int e = pair_entry(p, b, NCH);
      q[e * kChBins] += fma(ar, br, ai * bi);
      q[(e + 1) * kChBins] += fma(ai, br, -(ar * bi));
    }
}

template <int NCH, int NSRC>
__device__ __forceinline__ void store_partials_ch(const WienerArgs& a, const double* q, int f) {
  double* p = a.part + (int64_t)blockIdx.y * NSRC * NCH * NCH * a.F + f;
#pragma unroll 8
  for (int e = 0; e < NSRC * NCH * NCH; ++e) p[(int64_t)e * a.F] = q[e * kChBins];
}

// wiener_init_kernel with NCH channels: stem (j, c) at S + (j * NCH + c) * src_stride.  Dynamic shared memory: the
// partial sums, NSRC * NCH^2 x kChBins doubles
template <int NCH, int NSRC, bool MASKED>
__global__ void __launch_bounds__(kChBins) wiener_ch_init_kernel(const WienerArgs a, const float* __restrict__ M, int64_t m_stride) {
  extern __shared__ double sh_acc[];
  constexpr int NN = NCH * NCH;
  const int f = blockIdx.x * kChBins + threadIdx.x;
  const int64_t t0 = (int64_t)blockIdx.y * kWienerFrames, t1 = min(a.T, t0 + kWienerFrames);
  double mx = 0.0;
  if (f < a.F) {
    double* q = sh_acc + threadIdx.x;
#pragma unroll 8
    for (int e = 0; e < NSRC * NN; ++e) q[e * kChBins] = 0.0;
    for (int64_t t = t0; t < t1; ++t) {
      const int64_t o = t * a.ldf + f;
      float2 x[NCH];
#pragma unroll
      for (int c = 0; c < NCH; ++c) {
        x[c] = a.X[c * a.x_plane + o];
        mx = fmax(mx, (double)x[c].x * x[c].x + (double)x[c].y * x[c].y);
      }
#pragma unroll 1
      for (int j = 0; j < NSRC; ++j) {   // one source at a time: the plane addresses of all NSRC x NCH stems would not fit
        float2 y[NCH];
        float2* sj = a.S + j * NCH * a.src_stride + o;
        if constexpr (MASKED) {
          const float m = M[j * m_stride + o];
#pragma unroll
          for (int c = 0; c < NCH; ++c) {
            y[c] = make_float2(__fmul_rn(m, x[c].x), __fmul_rn(m, x[c].y));
            sj[c * a.src_stride] = y[c];
          }
        } else {
#pragma unroll
          for (int c = 0; c < NCH; ++c) y[c] = sj[c * a.src_stride];
        }
        accumulate_ch<NCH>(q + j * NN * kChBins, y);
      }
    }
    store_partials_ch<NCH, NSRC>(a, q, f);
  }
#pragma unroll
  for (int k = 16; k > 0; k >>= 1) mx = fmax(mx, __shfl_down_sync(0xffffffffu, mx, k));
  if (threadIdx.x == 0) a.pmax[(int64_t)blockIdx.y * a.ntiles + blockIdx.x] = mx;
}

// wiener_em_kernel with NCH channels.  Dynamic shared memory: R_j(f), NSRC * NCH^2 x kChBins doubles, then (STATS) the
// partial sums, as many.  C = sum_j v_j R_j + delta s^2 I is factored C = L D L^H (L unit lower, D real and positive:
// the delta term bounds D below), with no pivoting, in registers; z = C^-1 x by a forward and a backward substitution;
// y_j = v_j R_j z.  All in fp64, in a fixed order of operations
template <int NCH, int NSRC, bool STATS>
__global__ void __launch_bounds__(kChBins) wiener_ch_em_kernel(const WienerArgs a) {
  extern __shared__ double sh_r[];
  constexpr int NN = NCH * NCH, NP = NCH * (NCH - 1) / 2;
  const int f = blockIdx.x * kChBins + threadIdx.x;
  if (f >= a.F) return;
  const int64_t t0 = (int64_t)blockIdx.y * kWienerFrames, t1 = min(a.T, t0 + kWienerFrames);
  const double* Q = a.Q + (int64_t)blockIdx.y * a.q_stride;
  const double s = a.scale[(int64_t)blockIdx.y * a.s_stride];
  const double s2 = s * s, es2 = kEps * s2, ds2 = sqrt(kEps) * s2;
  double* r = sh_r + threadIdx.x;                 // R_j entry e at r[(j * NN + e) * kChBins]
  double* v = r + NSRC * NN * kChBins;            // v_j of the frame at v[j * kChBins]
  double* q = v + NSRC * kChBins;                 // STATS: the partial sums, laid out as R
#pragma unroll 1
  for (int j = 0; j < NSRC; ++j) {
    double tr = 0.0;
#pragma unroll
    for (int c = 0; c < NCH; ++c) tr += Q[(int64_t)(j * NN + c) * a.F + f];
    const double inv = 1.0 / (es2 + tr * (1.0 / NCH));
#pragma unroll 8
    for (int e = 0; e < NN; ++e) r[(j * NN + e) * kChBins] = Q[(int64_t)(j * NN + e) * a.F + f] * inv;
  }
  if (STATS) {
#pragma unroll 8
    for (int e = 0; e < NSRC * NN; ++e) q[e * kChBins] = 0.0;
  }
  for (int64_t t = t0; t < t1; ++t) {
    const int64_t o = t * a.ldf + f;
    // one source at a time throughout: the plane addresses of all NSRC x NCH stems would not fit in registers.  j0 is 0
    // but opaque to the compiler, so that at NSRC = 1 it neither unrolls these loops nor hoists R into registers
    int j0 = 0;
    asm volatile("" : "+r"(j0));
#pragma unroll 1
    for (int j = j0; j < NSRC; ++j) {
      const float2* sj = a.S + j * NCH * a.src_stride + o;
      double e2 = 0.0;
#pragma unroll
      for (int c = 0; c < NCH; ++c) {
        const float2 y = sj[c * a.src_stride];
        e2 += (double)y.x * y.x + (double)y.y * y.y;
      }
      v[j * kChBins] = e2 * (1.0 / NCH);
    }
    // C in the packed order: d[c] the diagonal, (cr, ci)[p] entry [a][b] of pair p, a < b
    double d[NCH], cr[NP], ci[NP];
#pragma unroll
    for (int c = 0; c < NCH; ++c) d[c] = 0.0;
#pragma unroll
    for (int p = 0; p < NP; ++p) cr[p] = ci[p] = 0.0;
#pragma unroll 1
    for (int j = j0; j < NSRC; ++j) {
      const double* rj = r + j * NN * kChBins;
      const double vj = v[j * kChBins];
#pragma unroll
      for (int c = 0; c < NCH; ++c) d[c] = fma(vj, rj[c * kChBins], d[c]);
#pragma unroll
      for (int p = 0; p < NP; ++p) {
        cr[p] = fma(vj, rj[(NCH + 2 * p) * kChBins], cr[p]);
        ci[p] = fma(vj, rj[(NCH + 2 * p + 1) * kChBins], ci[p]);
      }
    }
#pragma unroll
    for (int c = 0; c < NCH; ++c) d[c] += ds2;
    // L D L^H, row by row: L[i][k] = (C[i][k] - sum_{m<k} L[i][m] D[m] conj(L[k][m])) / D[k] and D[i] = C[i][i] -
    // sum_{m<i} |L[i][m]|^2 D[m].  C[i][k] = conj(C[k][i]); L[i][k] overwrites the slot of pair (k, i), d[i] becomes
    // 1 / D[i]
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      double ur[NCH], ui[NCH];   // ur + i ui [k] = L[i][k] D[k]
#pragma unroll
      for (int k = 0; k < i; ++k) {
        const int pk = (pair_entry(k, i, NCH) - NCH) / 2;
        double sr = cr[pk], si = -ci[pk];
#pragma unroll
        for (int m = 0; m < k; ++m) {   // -= u[m] conj(L[k][m])
          const int pm = (pair_entry(m, k, NCH) - NCH) / 2;
          sr = fma(-ur[m], cr[pm], fma(-ui[m], ci[pm], sr));
          si = fma(-ui[m], cr[pm], fma(ur[m], ci[pm], si));
        }
        ur[k] = sr;
        ui[k] = si;
        cr[pk] = sr * d[k];
        ci[pk] = si * d[k];
      }
      double di = d[i];
#pragma unroll
      for (int k = 0; k < i; ++k) {   // -= u[k] conj(L[i][k]), real
        const int pk = (pair_entry(k, i, NCH) - NCH) / 2;
        di = fma(-ur[k], cr[pk], fma(-ui[k], ci[pk], di));
      }
      d[i] = 1.0 / di;
    }
    // z = C^-1 x: w = L^-1 x, then z = L^-H (D^-1 w)
    double zr[NCH], zi[NCH];
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const float2 x = a.X[i * a.x_plane + o];
      double wr = x.x, wi = x.y;
#pragma unroll
      for (int k = 0; k < i; ++k) {   // -= L[i][k] w[k]
        const int pk = (pair_entry(k, i, NCH) - NCH) / 2;
        wr = fma(-cr[pk], zr[k], fma(ci[pk], zi[k], wr));
        wi = fma(-cr[pk], zi[k], fma(-ci[pk], zr[k], wi));
      }
      zr[i] = wr;
      zi[i] = wi;
    }
#pragma unroll
    for (int i = NCH - 1; i >= 0; --i) {
      double wr = zr[i] * d[i], wi = zi[i] * d[i];
#pragma unroll
      for (int k = i + 1; k < NCH; ++k) {   // -= conj(L[k][i]) z[k]
        const int pk = (pair_entry(i, k, NCH) - NCH) / 2;
        wr = fma(-cr[pk], zr[k], fma(-ci[pk], zi[k], wr));
        wi = fma(-cr[pk], zi[k], fma(ci[pk], zr[k], wi));
      }
      zr[i] = wr;
      zi[i] = wi;
    }
#pragma unroll 1
    for (int j = j0; j < NSRC; ++j) {
      // y_j = v_j R_j z: R_j[c][b] is the stored pair for c < b, its conjugate for c > b
      const double* rj = r + j * NN * kChBins;
      const double vj = v[j * kChBins];
      float2* sj = a.S + j * NCH * a.src_stride + o;
      float2 y[NCH];
#pragma unroll
      for (int c = 0; c < NCH; ++c) {
        const double rd = rj[c * kChBins];
        double yr = rd * zr[c], yi = rd * zi[c];
#pragma unroll
        for (int b = 0; b < NCH; ++b) {
          if (b == c) continue;
          const int e = b > c ? pair_entry(c, b, NCH) : pair_entry(b, c, NCH);
          const double pr = rj[e * kChBins], pi = b > c ? rj[(e + 1) * kChBins] : -rj[(e + 1) * kChBins];
          yr = fma(pr, zr[b], fma(-pi, zi[b], yr));
          yi = fma(pr, zi[b], fma(pi, zr[b], yi));
        }
        y[c] = make_float2((float)(vj * yr), (float)(vj * yi));
        sj[c * a.src_stride] = y[c];
      }
      if (STATS) accumulate_ch<NCH>(q + j * NN * kChBins, y);
    }
  }
  if (STATS) store_partials_ch<NCH, NSRC>(a, q, f);
}

// partials -> Q and scale: over the whole clip (radius 0) or over each chunk's window
void launch_reduce(const WienerArgs& a, int64_t n, int radius, cudaStream_t st) {
  const unsigned rgrid = (unsigned)ceil_div64(n, kReduceThreads) + 1;
  if (radius == 0)
    wiener_reduce_kernel<<<rgrid, kReduceThreads, 0, st>>>(a, n);
  else
    wiener_reduce_window_kernel<<<dim3(rgrid, (unsigned)a.nchunks), kReduceThreads, 0, st>>>(a, n, min(radius, a.nchunks - 1));
}

template <int NSRC, bool MASKED = false>
int launch_wiener_n(dcs_ctx* ctx, const WienerArgs& a, int iterations, int radius, cudaStream_t st, const float* M = nullptr,
                    int64_t m_stride = 0) {
  const dim3 grid((unsigned)a.ntiles, (unsigned)a.nchunks);
  const int64_t n = (int64_t)NSRC * 4 * a.F;
  {
    ProfScope ps(ctx, "wiener_init", st);
    wiener_init_kernel<NSRC, MASKED><<<grid, kWienerBins, 0, st>>>(a, M, m_stride);
    DCS_CHECK_LAUNCH();
    ctx->launches++;
    launch_reduce(a, n, radius, st);
    DCS_CHECK_LAUNCH();
    ctx->launches++;
  }
  for (int k = 1; k <= iterations; ++k) {
    ProfScope ps(ctx, "wiener_em", st);
    if (k < iterations) {
      wiener_em_kernel<NSRC, true><<<grid, kWienerBins, 0, st>>>(a);
      DCS_CHECK_LAUNCH();
      ctx->launches++;
      launch_reduce(a, n, radius, st);
    } else {
      wiener_em_kernel<NSRC, false><<<grid, kWienerBins, 0, st>>>(a);
    }
    DCS_CHECK_LAUNCH();
    ctx->launches++;
  }
  return DCS_OK;
}

// the C-channel kernels: the same launches, kChBins bins per block and NSRC * NCH^2 partial sums per bin
template <int NCH, int NSRC, bool MASKED = false>
int launch_wiener_ch_n(dcs_ctx* ctx, const WienerArgs& a, int iterations, int radius, cudaStream_t st, const float* M,
                       int64_t m_stride) {
  const dim3 grid((unsigned)a.ntiles, (unsigned)a.nchunks);
  const int64_t n = (int64_t)NSRC * NCH * NCH * a.F;
  // shared memory: one [entry][bin] array of NSRC * NCH^2 doubles for the partials (init), R (EM), R + v_j (EM, last
  // pass) or R + v_j + partials (EM)
  const size_t cols = (size_t)NSRC * NCH * NCH * kChBins * sizeof(double), vcols = (size_t)NSRC * kChBins * sizeof(double);
  auto init = wiener_ch_init_kernel<NCH, NSRC, MASKED>;
  auto em_stats = wiener_ch_em_kernel<NCH, NSRC, true>;
  auto em_last = wiener_ch_em_kernel<NCH, NSRC, false>;
  DCS_TRY(ensure_smem_attr(init, (int)cols));
  DCS_TRY(ensure_smem_attr(em_stats, (int)(2 * cols + vcols)));
  DCS_TRY(ensure_smem_attr(em_last, (int)(cols + vcols)));
  {
    ProfScope ps(ctx, "wiener_init", st);
    init<<<grid, kChBins, cols, st>>>(a, M, m_stride);
    DCS_CHECK_LAUNCH();
    ctx->launches++;
    launch_reduce(a, n, radius, st);
    DCS_CHECK_LAUNCH();
    ctx->launches++;
  }
  for (int k = 1; k <= iterations; ++k) {
    ProfScope ps(ctx, "wiener_em", st);
    if (k < iterations) {
      em_stats<<<grid, kChBins, 2 * cols + vcols, st>>>(a);
      DCS_CHECK_LAUNCH();
      ctx->launches++;
      launch_reduce(a, n, radius, st);
    } else {
      em_last<<<grid, kChBins, cols + vcols, st>>>(a);
    }
    DCS_CHECK_LAUNCH();
    ctx->launches++;
  }
  return DCS_OK;
}

template <int NCH>
int launch_wiener_ch_src(dcs_ctx* ctx, const WienerArgs& a, int nsrc, int iterations, int radius, cudaStream_t st, const float* M,
                         int64_t m_stride) {
  switch (nsrc * 2 + (M ? 1 : 0)) {
    case 2: return launch_wiener_ch_n<NCH, 1>(ctx, a, iterations, radius, st, M, m_stride);
    case 3: return launch_wiener_ch_n<NCH, 1, true>(ctx, a, iterations, radius, st, M, m_stride);
    case 4: return launch_wiener_ch_n<NCH, 2>(ctx, a, iterations, radius, st, M, m_stride);
    case 5: return launch_wiener_ch_n<NCH, 2, true>(ctx, a, iterations, radius, st, M, m_stride);
    case 6: return launch_wiener_ch_n<NCH, 3>(ctx, a, iterations, radius, st, M, m_stride);
    case 7: return launch_wiener_ch_n<NCH, 3, true>(ctx, a, iterations, radius, st, M, m_stride);
    case 8: return launch_wiener_ch_n<NCH, 4>(ctx, a, iterations, radius, st, M, m_stride);
    case 9: return launch_wiener_ch_n<NCH, 4, true>(ctx, a, iterations, radius, st, M, m_stride);
  }
  DCS_REQUIRE(false, "wiener: nsrc %d not in [1, 4]", nsrc);
}

struct WienerLayout {
  int nchunks, ntiles;
  int64_t part, Q, pmax, scale, total;   // offsets / size in doubles
};

// radius >= 1: one Q and one scale per chunk.  nch 2: the stereo kernels' tiles of kWienerBins bins, else kChBins
WienerLayout wiener_layout(int nsrc, int nch, int64_t T, int F, int radius) {
  WienerLayout l;
  l.nchunks = (int)ceil_div64(T, kWienerFrames);
  l.ntiles = (int)ceil_div64(F, nch == 2 ? kWienerBins : kChBins);
  const int64_t per = (int64_t)nsrc * nch * nch * F, nq = radius > 0 ? l.nchunks : 1;
  l.part = 0;
  l.Q = (int64_t)l.nchunks * per;
  l.pmax = l.Q + nq * per;
  l.scale = l.pmax + (int64_t)l.nchunks * l.ntiles;
  l.total = l.scale + nq;
  return l;
}

}  // namespace

int wiener_check(const char* fn, int nsrc, int64_t T, int64_t ldf, int F, int64_t x_plane, int64_t src_stride, int iterations,
                 int radius) {
  DCS_REQUIRE(iterations >= 0, "%s: iterations %d must be >= 0", fn, iterations);
  DCS_REQUIRE(radius >= 0, "%s: radius %d must be >= 0", fn, radius);
  DCS_REQUIRE(nsrc >= 1 && nsrc <= 4, "%s: nsrc %d not in [1, 4]", fn, nsrc);
  DCS_REQUIRE(T > 0 && ceil_div64(T, kWienerFrames) <= 65535, "%s: %lld frames out of range", fn, (long long)T);
  DCS_REQUIRE(F > 0 && ldf >= F, "%s: bins %d / row stride %lld", fn, F, (long long)ldf);
  DCS_REQUIRE(x_plane >= T * ldf && src_stride >= T * ldf, "%s: plane strides %lld / %lld below T * ldf = %lld", fn,
              (long long)x_plane, (long long)src_stride, (long long)(T * ldf));
  return DCS_OK;
}

size_t wiener_workspace_bytes(int nsrc, int nch, int64_t T, int F, int radius) {
  return (size_t)wiener_layout(nsrc, nch, T, F, radius).total * sizeof(double);
}

int launch_wiener(dcs_ctx* ctx, const float2* X, int64_t x_plane, float2* S, int64_t src_stride, int nsrc, int64_t T,
                  int64_t ldf, int F, int iterations, int radius, cudaStream_t st, const float* M, int64_t m_stride, int nch) {
  if (iterations <= 0) return DCS_OK;
  DCS_REQUIRE(nch >= 2 && nch <= 8, "wiener: %d channels not in [2, 8]", nch);
  const WienerLayout l = wiener_layout(nsrc, nch, T, F, radius);
  DCS_TRY(ctx->wiener.ensure((size_t)l.total * sizeof(double), st));
  double* w = ctx->wiener.as<double>();
  WienerArgs a;
  a.X = X; a.x_plane = x_plane; a.S = S; a.src_stride = src_stride; a.T = T; a.ldf = ldf;
  a.F = F; a.nchunks = l.nchunks; a.ntiles = l.ntiles;
  a.part = w + l.part; a.Q = w + l.Q; a.pmax = w + l.pmax; a.scale = w + l.scale;
  a.q_stride = radius > 0 ? (int64_t)nsrc * nch * nch * F : 0;
  a.s_stride = radius > 0 ? 1 : 0;
  switch (nch) {
    case 3: return launch_wiener_ch_src<3>(ctx, a, nsrc, iterations, radius, st, M, m_stride);
    case 4: return launch_wiener_ch_src<4>(ctx, a, nsrc, iterations, radius, st, M, m_stride);
    case 5: return launch_wiener_ch_src<5>(ctx, a, nsrc, iterations, radius, st, M, m_stride);
    case 6: return launch_wiener_ch_src<6>(ctx, a, nsrc, iterations, radius, st, M, m_stride);
    case 7: return launch_wiener_ch_src<7>(ctx, a, nsrc, iterations, radius, st, M, m_stride);
    case 8: return launch_wiener_ch_src<8>(ctx, a, nsrc, iterations, radius, st, M, m_stride);
  }
  switch (nsrc * 2 + (M ? 1 : 0)) {
    case 2: return launch_wiener_n<1>(ctx, a, iterations, radius, st);
    case 3: return launch_wiener_n<1, true>(ctx, a, iterations, radius, st, M, m_stride);
    case 4: return launch_wiener_n<2>(ctx, a, iterations, radius, st);
    case 5: return launch_wiener_n<2, true>(ctx, a, iterations, radius, st, M, m_stride);
    case 6: return launch_wiener_n<3>(ctx, a, iterations, radius, st);
    case 7: return launch_wiener_n<3, true>(ctx, a, iterations, radius, st, M, m_stride);
    case 8: return launch_wiener_n<4>(ctx, a, iterations, radius, st);
    case 9: return launch_wiener_n<4, true>(ctx, a, iterations, radius, st, M, m_stride);
  }
  DCS_REQUIRE(false, "wiener: nsrc %d not in [1, 4]", nsrc);
}

}  // namespace dcs
