// fft_reg.cuh -- register-resident FFT for the framed STFT / iSTFT: one group of T = N2/32 threads
// (a warp for N2 = 1024, a half warp for N2 = 512) transforms one frame with every point in
// registers (32 complex values per thread), Cooley-Tukey N2 = 32 x T:
//   1. thread b holds x[a*T + b], a < 32 (coalesced global loads) and runs a 32-point FFT over a
//   2. twiddle by w_N2^(b*ka), transpose through a per-group shared scratch (conflict-free,
//      padded rows), __syncwarp only -- no block-wide barrier anywhere
//   3. thread t runs the T-point FFTs over b for ka = t + T*q
// The 32- and 16-point kernels are fully unrolled decimation-in-frequency networks whose
// twiddles are compile-time constants; their bit-reversed output order is absorbed by static
// register renaming.
#pragma once
#include <cuda_runtime.h>
#include "fft.cuh"

namespace dcs {

// cos(2*pi*q/32), sin(2*pi*q/32), q = 0..15
__device__ __forceinline__ constexpr float cos32(int q) {
  constexpr float t[16] = {1.0f, 0.98078528040323043f, 0.92387953251128674f, 0.83146961230254524f, 0.70710678118654752f,
                           0.55557023301960218f, 0.38268343236508977f, 0.19509032201612825f, 0.0f, -0.19509032201612825f,
                           -0.38268343236508977f, -0.55557023301960218f, -0.70710678118654752f, -0.83146961230254524f,
                           -0.92387953251128674f, -0.98078528040323043f};
  return t[q];
}
__device__ __forceinline__ constexpr float sin32(int q) {
  constexpr float t[16] = {0.0f, 0.19509032201612825f, 0.38268343236508977f, 0.55557023301960218f, 0.70710678118654752f,
                           0.83146961230254524f, 0.92387953251128674f, 0.98078528040323043f, 1.0f, 0.98078528040323043f,
                           0.92387953251128674f, 0.83146961230254524f, 0.70710678118654752f, 0.55557023301960218f,
                           0.38268343236508977f, 0.19509032201612825f};
  return t[q];
}

__host__ __device__ constexpr int brev(int i, int bits) {
  int r = 0;
  for (int k = 0; k < bits; ++k) r |= ((i >> k) & 1) << (bits - 1 - k);
  return r;
}

// d * exp(-2*pi*i*q/32), q in [0,16), q known at compile time after unrolling
__device__ __forceinline__ float2 mul_w32(float2 d, int q) {
  if (q == 0) return d;
  if (q == 8) return make_float2(d.y, -d.x);
  if (q == 4) return make_float2(0.70710678118654752f * (d.x + d.y), 0.70710678118654752f * (d.y - d.x));
  if (q == 12) return make_float2(0.70710678118654752f * (d.y - d.x), -0.70710678118654752f * (d.x + d.y));
  const float c = cos32(q), s = sin32(q);  // w = c - i s
  return make_float2(fmaf(d.x, c, d.y * s), fmaf(d.y, c, -d.x * s));
}

// In-place DIF FFT of R = 32 or 16 points: on return v[i] = X[brev(i)].  One template level per
// butterfly stage (L = span of the stage), so that every loop has a compile-time trip count: with the
// stage as a loop variable the sm_90a compiler left the inner loop rolled and moved v[] to local memory.
template <int R, int L = R>
__device__ __forceinline__ void fft_dif(float2 (&v)[R]) {
  constexpr int half = L >> 1;
#pragma unroll
  for (int s = 0; s < R; s += L) {
#pragma unroll
    for (int j = 0; j < half; ++j) {
      const float2 a = v[s + j], b = v[s + j + half];
      v[s + j] = cadd(a, b);
      v[s + j + half] = mul_w32(csub(a, b), j * (32 / L));
    }
  }
  if constexpr (L > 2) fft_dif<R, L / 2>(v);
}

template <int T>
struct FftGroup {
  static constexpr int N2 = 32 * T;
  // tw2[ka*T + b] = tw[2*b*ka], tw[j] = exp(-2*pi*i*j/(2*N2)): 32*T = N2 entries (block-wide, then __syncthreads)
  __device__ static __forceinline__ void fill_tw2(float2* tw2, const float2* __restrict__ tw, int tid, int nthreads) {
    for (int i = tid; i < 32 * T; i += nthreads) {
      const int ka = i / T, b = i - ka * T;
      tw2[i] = __ldg(tw + 2 * b * ka);
    }
  }
  static constexpr int PITCH = T + 1;                 // float2 per scratch row
  static constexpr int SCRATCH = 32 * PITCH;          // float2 per group (>= N2)
  static constexpr int Q = 32 / T;                    // rows per thread in the second pass (1 or 2)
  static constexpr int TBITS = T == 32 ? 5 : 4;

  // in : v[a] = x[a*T + b]                          (b = lane within the group)
  // out: v[q*T + kb] = X[(b + T*q) + 32*kb]          (q < Q, kb < T)
  // tw[j] = exp(-2*pi*i*j/(2*N2)); `scr` = this group's scratch; all lanes of the warp call this.
  // TW_SHARED: `tw` is the shared-memory inter-stage table tw2[ka*T + b] = exp(-2*pi*i*b*ka/N2) (fill_tw2): lane b
  // reads consecutive 8-byte words for every ka -- conflict free.  (Indexing the plain table with 2*b*ka strides
  // the lanes by 4*ka banks: 8- to 16-way conflicts for ka = 4, 8, 16, ...)
  template <bool TW_SHARED = false>
  __device__ static __forceinline__ void forward(float2 (&v)[32], float2* scr, const float2* __restrict__ tw, int b) {
    fft_dif<32>(v);
#pragma unroll
    for (int ka = 0; ka < 32; ++ka) {
      float2 y = v[brev(ka, 5)];
      if (ka > 0) y = cmul(y, TW_SHARED ? tw[ka * T + b] : __ldg(tw + 2 * b * ka));
      scr[ka * PITCH + b] = y;
    }
    __syncwarp();
    if (T == 32) {
#pragma unroll
      for (int i = 0; i < 32; ++i) v[i] = scr[b * PITCH + i];
      fft_dif<32>(v);
      float2 u[32];
#pragma unroll
      for (int kb = 0; kb < 32; ++kb) u[kb] = v[brev(kb, 5)];
#pragma unroll
      for (int kb = 0; kb < 32; ++kb) v[kb] = u[kb];
    } else {
      float2 u0[16], u1[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        u0[i] = scr[b * PITCH + i];
        u1[i] = scr[(b + 16) * PITCH + i];
      }
      fft_dif<16>(u0);
      fft_dif<16>(u1);
#pragma unroll
      for (int kb = 0; kb < 16; ++kb) {
        v[kb] = u0[brev(kb, 4)];
        v[16 + kb] = u1[brev(kb, 4)];
      }
    }
    __syncwarp();  // scratch may be reused by the caller
  }

  // forward<true>() through half the scratch (HALF_SCRATCH float2: 16 rows of PITCH), the transpose in two rounds of
  // 16 rows, so that a CTA fits more groups next to its row rings.  Every lane sends 16 values and receives 16 a round,
  // which keeps 32 values live across the transpose as in forward().
  //   T = 16: round r moves rows ka = 16 r + ka'; the output is forward()'s.
  //   T = 32: lane i sends row ka' + 16 (hi(i) ^ r) in round r, hi(i) = bit 4 of i (two selects per float, no
  //   dynamic register index), and lane b receives its 32 second-pass inputs rotated by 16 when hi(b).  A rotation by
  //   N/2 of a DIF network's input negates its odd outputs exactly (the first stage's differences change sign, every
  //   later operation is odd), so on return v[kb] is forward()'s value times -1 for odd kb on lanes with hi(b) -- the
  //   same bits but for the sign of zero results.  The caller folds that sign into the constants it multiplies by.
  static constexpr int HALF_SCRATCH = 16 * PITCH;
  __device__ static __forceinline__ void forward_split(float2 (&v)[32], float2* scr, const float2* tw, int b) {
    fft_dif<32>(v);
    auto y = [&](int ka) { return ka > 0 ? cmul(v[brev(ka, 5)], tw[ka * T + b]) : v[0]; };
    if (T == 32) {
      const bool hi = (b & 16) != 0;
      float2 later[16];   // the value each lane sends in round 1
#pragma unroll
      for (int a = 0; a < 16; ++a) {
        const float2 lo = y(a), up = y(a + 16);
        scr[a * PITCH + b] = hi ? up : lo;
        later[a] = hi ? lo : up;
      }
      const float2* row = scr + (b & 15) * PITCH;
      __syncwarp();
#pragma unroll
      for (int i = 0; i < 16; ++i) v[i] = row[(hi ? 16 : 0) + i];
      __syncwarp();
#pragma unroll
      for (int a = 0; a < 16; ++a) scr[a * PITCH + b] = later[a];
      __syncwarp();
#pragma unroll
      for (int i = 0; i < 16; ++i) v[16 + i] = row[(hi ? 0 : 16) + i];
      fft_dif<32>(v);
      float2 u[32];
#pragma unroll
      for (int kb = 0; kb < 32; ++kb) u[kb] = v[brev(kb, 5)];
#pragma unroll
      for (int kb = 0; kb < 32; ++kb) v[kb] = u[kb];
    } else {
      float2 u0[16], u1[16];
#pragma unroll
      for (int a = 0; a < 16; ++a) scr[a * PITCH + b] = y(a);
      __syncwarp();
#pragma unroll
      for (int i = 0; i < 16; ++i) u0[i] = scr[b * PITCH + i];
      __syncwarp();
#pragma unroll
      for (int a = 0; a < 16; ++a) scr[a * PITCH + b] = y(16 + a);
      __syncwarp();
#pragma unroll
      for (int i = 0; i < 16; ++i) u1[i] = scr[b * PITCH + i];
      fft_dif<16>(u0);
      fft_dif<16>(u1);
#pragma unroll
      for (int kb = 0; kb < 16; ++kb) {
        v[kb] = u0[brev(kb, 4)];
        v[16 + kb] = u1[brev(kb, 4)];
      }
    }
    __syncwarp();  // scratch may be reused by the caller
  }
};

}  // namespace dcs
