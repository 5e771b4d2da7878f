// resample.cu -- polyphase rational resampling by up/down (dcs_resample, include/dcs.h): the filter of
// scipy.signal.resample_poly with zero padding,
//     y[n] = sum_j x[j] * h[n*down + half_len - j*up],   0 <= j < num_in,   0 <= n*down + half_len - j*up < ntaps,
// half_len = (ntaps - 1) / 2.  For n = P*up + r the sum runs over the Q = ceil(ntaps / up) taps h[ph_r + i*up] against
// x[P*down + c_r - i], with c_r = floor((r*down + half_len) / up), ph_r = (r*down + half_len) mod up: the taps depend
// only on the residue r, so the bank is stored as bank[i][r] (zero past ntaps) and outputs one period apart share it.
//
// Persistent CTAs load the bank (fp64, <= DCS_RESAMPLE_MAX_BANK_BYTES) into shared memory once.  A tile is tp
// consecutive periods (tp * up consecutive outputs) of one plane; its input span is staged as fp32 in shared memory,
// zeros outside [0, num_in) (nothing else of the plane is read).  A work item is (residue r, RS_V consecutive periods):
// each tap is loaded once for RS_V outputs, consecutive lanes take consecutive residues, so the tap loads are
// conflict-free and the sample loads nearly so.  The sum is accumulated in fp64 with fma in increasing i and rounded
// once to fp32: the same bits on every run.
//
// The C-channel batch at another rate fuses the sample conversions into the resampler (resample_decode_kernel,
// resample_encode_kernel, one instantiation per sample format): the same bank, the same work items and the same inner
// sum (polyphase_sum), so each value has the bits of resample_kernel on the fp32 planes the unfused route would have
// formed.
#include <algorithm>
#include <type_traits>
#include "common.cuh"

struct dcs_resampler {
  dcs_ctx* ctx;
  int up, down, ntaps, half_len, Q;
  int c0, cspan;          // c_0 and c_{up-1} - c_0
  int tp, span;           // periods per tile, input samples staged per tile
  size_t smem;            // bank + staged input
  double* d_bank;         // [Q][up]
};

namespace dcs {

constexpr int RS_THREADS = 512;
constexpr int RS_V = 4;                       // periods per work item
constexpr int RS_TILE_WORDS = 8192;           // staged input per tile (32 KB) when the period allows
constexpr int RS_SMEM_MAX = 227 * 1024;

struct ResampleArgs {
  const float* in; int64_t in_stride, num_in;
  float* out; int64_t out_stride, num_out;
  const double* bank;
  int up, down, Q, half_len, c0, tp, span;
  int64_t tiles_per_plane, ntiles;
};

// the RS_V outputs of residue r, one period apart, from the staged samples x(base + v*down - i): fma in increasing tap
// index i from the exactly widened fp32 sample, in fp64; the caller rounds each once to fp32
template <class Sample>
__device__ __forceinline__ void polyphase_sum(const double* __restrict__ bank, int up, int down, int Q, int r, int base,
                                              Sample x, double (&acc)[RS_V]) {
#pragma unroll
  for (int v = 0; v < RS_V; ++v) acc[v] = 0.0;
  for (int i = 0; i < Q; ++i) {
    const double hv = bank[i * up + r];
#pragma unroll
    for (int v = 0; v < RS_V; ++v) acc[v] = fma(hv, (double)x(base + v * down - i), acc[v]);
  }
}

__global__ void __launch_bounds__(RS_THREADS)
resample_kernel(const ResampleArgs a) {
  extern __shared__ __align__(16) unsigned char rs_smem[];
  double* bank = reinterpret_cast<double*>(rs_smem);
  float* xs = reinterpret_cast<float*>(bank + (size_t)a.Q * a.up);
  for (int k = threadIdx.x; k < a.Q * a.up; k += RS_THREADS) bank[k] = __ldg(a.bank + k);
  const int items = a.up * (a.tp / RS_V);
  for (int64_t tile = blockIdx.x; tile < a.ntiles; tile += gridDim.x) {
    const int64_t plane = tile / a.tiles_per_plane;
    const int64_t P0 = (tile % a.tiles_per_plane) * a.tp;
    const int64_t jlo = P0 * a.down + a.c0 - (a.Q - 1);          // input sample of xs[0]
    const float* __restrict__ x = a.in + plane * a.in_stride;
    __syncthreads();                                              // the previous tile's reads are done
    for (int k = threadIdx.x; k < a.span; k += RS_THREADS) {
      const int64_t j = jlo + k;
      xs[k] = (j >= 0 && j < a.num_in) ? __ldg(x + j) : 0.f;
    }
    __syncthreads();
    float* __restrict__ y = a.out + plane * a.out_stride;
    for (int w = threadIdx.x; w < items; w += RS_THREADS) {
      const int r = w % a.up, g = w / a.up;
      const int64_t n0 = (P0 + (int64_t)g * RS_V) * a.up + r;
      if (n0 >= a.num_out) continue;
      const int c = (int)(((int64_t)r * a.down + a.half_len) / a.up);
      // sample of (period P0 + g*V + v, tap i) at xs[base + v*down - i]
      const int base = g * RS_V * a.down + c - a.c0 + a.Q - 1;
      double acc[RS_V];
      polyphase_sum(bank, a.up, a.down, a.Q, r, base, [&](int k) { return xs[k]; }, acc);
#pragma unroll
      for (int v = 0; v < RS_V; ++v) {
        const int64_t n = n0 + (int64_t)v * a.up;
        if (n < a.num_out) y[n] = (float)acc[v];
      }
    }
  }
}

// The C-channel batch's conversions fused into the resampler.  Both take the bank and phase constants of a
// dcs_resampler, tiles of tp periods as resample_kernel does, and a plan per (resampler, C, format) that fits shared
// memory.
struct ResamplePcmArgs {
  const void* in; int64_t num_in;    // decode: samples [num_in][C]; encode: nsrc*C fp32 planes num_in apart
  void* out; int64_t num_out;        // decode: C + 1 fp32 planes num_out apart; encode: samples [nsrc][num_out][C]
  const double* bank;
  int up, down, Q, half_len, c0, tp, span;
  int C, cn, cs;                     // channels; channels per tile and staged values per sample (encode)
  int64_t tiles_t, ntiles;           // tiles along time, all tiles
};
// The windowed kernels' arguments (a type of its own: the plain kernels keep their parameter block).  The outputs are
// [out_first, out_first + num_out) of the whole signal's resampling, their periods counted from p_first =
// floor(out_first / up); input sample j of the whole signal is at in + (j - in_first) for j in [j_lo, j_hi), and zero
// elsewhere.
struct ResampleWindow { int64_t out_first, p_first, in_first, j_lo, j_hi; };
struct ResampleWinArgs : ResamplePcmArgs { ResampleWindow win; };
// the window of each argument type; the plain kernels' is the whole signal: periods from 0, input j at j for j in
// [0, num_in).  The bounds stay in the staging condition's own && (a bool helper changes the plain kernels' SASS)
__device__ __forceinline__ int64_t first_period(const ResamplePcmArgs&) { return 0; }
__device__ __forceinline__ int64_t first_period(const ResampleWinArgs& a) { return a.win.p_first; }
__device__ __forceinline__ int64_t first_out(const ResamplePcmArgs&) { return 0; }
__device__ __forceinline__ int64_t first_out(const ResampleWinArgs& a) { return a.win.out_first; }
__device__ __forceinline__ int64_t staged_lo(const ResamplePcmArgs&) { return 0; }
__device__ __forceinline__ int64_t staged_lo(const ResampleWinArgs& a) { return a.win.j_lo; }
__device__ __forceinline__ int64_t staged_hi(const ResamplePcmArgs& a) { return a.num_in; }
__device__ __forceinline__ int64_t staged_hi(const ResampleWinArgs& a) { return a.win.j_hi; }
__device__ __forceinline__ int64_t staged_at(const ResamplePcmArgs&, int64_t j) { return j; }
__device__ __forceinline__ int64_t staged_at(const ResampleWinArgs& a, int64_t j) { return j - a.win.in_first; }

// the tap value of a staged sample: int16 is converted per tap use, the 4-byte formats are staged already decoded
__device__ __forceinline__ float staged_tap(int16_t x) { return SampleFormat<DCS_SAMPLE_I16>::decode(x); }
__device__ __forceinline__ float staged_tap(float x) { return x; }

// [num_in][C] samples of format FMT at the clip's rate -> plane 1 + c: resample_kernel on the fp32 plane of the format's
// decode of channel c, and plane 0: (((y_0 + y_1) + y_2) + ...) * (1.0f / C) on those rounded values, downmix_kernel's
// expression.  A tile is tp periods of cn channels; its input span is staged channel by channel ([cn][span]).  A work
// item is (residue r, RS_V periods) for every channel of the tile in turn, so when the tile holds all C channels
// (cn = C) one thread forms the downmix of its outputs.
//  - int16: staged as int16 and converted per tap; cn = C always.
//  - int32 and float32: staged as their fp32 decode, one conversion per staged sample, so the inner sum is
//    resample_kernel's on the same values.  Where 4-byte staging leaves no room for all C channels, the channels are
//    split into equal groups of cn; plane 0 is then not written here but by one downmix_kernel launch on the planes.
// Args = ResampleWinArgs (kWin): a window of the whole recording's resampling; the same sums, tiles aligned to its
// periods.
template <int FMT, class Args = ResamplePcmArgs>
__global__ void __launch_bounds__(RS_THREADS)
resample_decode_kernel(const Args a) {
  constexpr bool kWin = std::is_same<Args, ResampleWinArgs>::value;
  using In = typename SampleFormat<FMT>::T;
  constexpr bool kWide = FMT != DCS_SAMPLE_I16;
  using Staged = typename std::conditional<kWide, float, int16_t>::type;
  extern __shared__ __align__(16) unsigned char rs_smem[];
  double* bank = reinterpret_cast<double*>(rs_smem);
  Staged* xs = reinterpret_cast<Staged*>(bank + (size_t)a.Q * a.up);
  const In* __restrict__ pcm = static_cast<const In*>(a.in);
  float* __restrict__ planes = static_cast<float*>(a.out);
  for (int k = threadIdx.x; k < a.Q * a.up; k += RS_THREADS) bank[k] = __ldg(a.bank + k);
  const int C = a.C, items = a.up * (a.tp / RS_V);
  const float inv = 1.0f / (float)C;
  for (int64_t tile = blockIdx.x; tile < a.ntiles; tile += gridDim.x) {
    const int64_t tt = kWide ? tile % a.tiles_t : tile;
    const int c_lo = kWide ? (int)(tile / a.tiles_t) * a.cn : 0;
    const int cn = kWide ? min(a.cn, C - c_lo) : C;
    const int64_t P0 = first_period(a) + tt * a.tp;
    const int64_t jlo = P0 * a.down + a.c0 - (a.Q - 1);
    __syncthreads();
    for (int k = threadIdx.x; k < a.span * cn; k += RS_THREADS) {    // consecutive threads read consecutive values
      const int jj = k / cn, c = k - jj * cn;
      const int64_t j = jlo + jj;
      if constexpr (kWide)
        xs[c * a.span + jj] = (j >= staged_lo(a) && j < staged_hi(a)) ? SampleFormat<FMT>::decode(pcm[staged_at(a, j) * C + c_lo + c]) : 0.f;
      else
        xs[c * a.span + jj] = (j >= staged_lo(a) && j < staged_hi(a)) ? pcm[staged_at(a, j) * C + c] : (int16_t)0;
    }
    __syncthreads();
    for (int w = threadIdx.x; w < items; w += RS_THREADS) {
      const int r = w % a.up, g = w / a.up;
      const int64_t n0 = (P0 + (int64_t)g * RS_V) * a.up + r - first_out(a);   // index in the output planes
      if (n0 >= a.num_out) continue;
      const int cr = (int)(((int64_t)r * a.down + a.half_len) / a.up);
      const int base = g * RS_V * a.down + cr - a.c0 + a.Q - 1;
      float mix[RS_V];
      for (int c = 0; c < cn; ++c) {
        const Staged* xc = xs + c * a.span;
        double acc[RS_V];
        polyphase_sum(bank, a.up, a.down, a.Q, r, base, [&](int k) { return staged_tap(xc[k]); }, acc);
        float* y = planes + (int64_t)(1 + c_lo + c) * a.num_out;
#pragma unroll
        for (int v = 0; v < RS_V; ++v) {
          const float yv = (float)acc[v];
          const int64_t n = n0 + (int64_t)v * a.up;
          if ((!kWin || n >= 0) && n < a.num_out) y[n] = yv;
          mix[v] = c == 0 ? yv : mix[v] + yv;
        }
      }
      if (cn == C) {
#pragma unroll
        for (int v = 0; v < RS_V; ++v) {
          const int64_t n = n0 + (int64_t)v * a.up;
          if ((!kWin || n >= 0) && n < a.num_out) planes[n] = mix[v] * inv;
        }
      }
    }
  }
}

// nsrc*C fp32 stem planes (source s, channel c at (s*C + c) * num_in) at 44.1 kHz -> [nsrc][num_out][C] samples of
// format FMT at the clip's rate: the format's encode of resample_kernel's fp32 value y (for int16 (int16_t)(int)(y *
// 32767.0f), the truncation of pcm_encode_channels_kernel).  A tile is tp periods of cn channels of one source (cn = C
// unless the bank leaves too little room); its span is staged interleaved, cs = cn | 1 values per sample so that the
// staging stores and the tap loads of neighbouring channels fall in different banks.  A work item is (channel, residue,
// RS_V periods) with the channel fastest, so neighbouring lanes write neighbouring values of the interleaved output.
// Args = ResampleWinArgs (kWin): a window of the resampling of stems placed at [in_first, in_first + num_in) of the 44.1 kHz signal (zeros
// elsewhere; j_lo = in_first, j_hi = in_first + num_in), the stem planes num_in apart.
template <int FMT, class Args = ResamplePcmArgs>
__global__ void __launch_bounds__(RS_THREADS)
resample_encode_kernel(const Args a) {
  constexpr bool kWin = std::is_same<Args, ResampleWinArgs>::value;
  using Out = typename SampleFormat<FMT>::T;
  extern __shared__ __align__(16) unsigned char rs_smem[];
  double* bank = reinterpret_cast<double*>(rs_smem);
  float* xs = reinterpret_cast<float*>(bank + (size_t)a.Q * a.up);
  const float* __restrict__ stems = static_cast<const float*>(a.in);
  Out* __restrict__ out = static_cast<Out*>(a.out);
  for (int k = threadIdx.x; k < a.Q * a.up; k += RS_THREADS) bank[k] = __ldg(a.bank + k);
  const int C = a.C, cs = a.cs, groups = (C + a.cn - 1) / a.cn;
  for (int64_t tile = blockIdx.x; tile < a.ntiles; tile += gridDim.x) {
    const int64_t tt = tile % a.tiles_t, sg = tile / a.tiles_t;
    const int s = (int)(sg / groups), c_lo = (int)(sg % groups) * a.cn;
    const int cn = min(a.cn, C - c_lo);
    const int64_t P0 = first_period(a) + tt * a.tp;
    const int64_t jlo = P0 * a.down + a.c0 - (a.Q - 1);
    const float* __restrict__ x = stems + ((int64_t)s * C + c_lo) * a.num_in;
    __syncthreads();
    for (int k = threadIdx.x; k < a.span * cn; k += RS_THREADS) {   // plane by plane: coalesced reads
      const int c = k / a.span, jj = k - c * a.span;
      const int64_t j = jlo + jj;
      xs[jj * cs + c] = (j >= staged_lo(a) && j < staged_hi(a)) ? __ldg(x + (int64_t)c * a.num_in + staged_at(a, j)) : 0.f;
    }
    __syncthreads();
    const int items = cn * a.up * (a.tp / RS_V);
    Out* __restrict__ o = out + (int64_t)s * a.num_out * C + c_lo;
    for (int w = threadIdx.x; w < items; w += RS_THREADS) {
      const int c = w % cn, rg = w / cn;
      const int r = rg % a.up, g = rg / a.up;
      const int64_t n0 = (P0 + (int64_t)g * RS_V) * a.up + r - first_out(a);
      if (n0 >= a.num_out) continue;
      const int cr = (int)(((int64_t)r * a.down + a.half_len) / a.up);
      const int base = g * RS_V * a.down + cr - a.c0 + a.Q - 1;
      double acc[RS_V];
      polyphase_sum(bank, a.up, a.down, a.Q, r, base, [&](int k) { return xs[k * cs + c]; }, acc);
#pragma unroll
      for (int v = 0; v < RS_V; ++v) {
        const int64_t n = n0 + (int64_t)v * a.up;
        if ((!kWin || n >= 0) && n < a.num_out) o[n * C + c] = SampleFormat<FMT>::encode((float)acc[v]);
      }
    }
  }
}

}  // namespace dcs

using namespace dcs;

static int64_t gcd64(int64_t a, int64_t b) {
  while (b) { const int64_t t = a % b; a = b; b = t; }
  return a;
}

namespace dcs {

// the tile of a fused kernel for C channels: periods per tile (a multiple of RS_V, no more work items than 4 rounds of
// the CTA, counting each channel's outputs for the encode), channels per tile and staged values per sample; false when
// even RS_V periods of one channel do not fit next to the bank.  The encode stages fp32 stems whatever the format.
// The int16 decode stages int16 and keeps all C channels in one tile (it forms the downmix); the 4-byte decodes stage
// fp32 and, like the encode, take the fewest equal channel groups that fit
struct PcmPlan { int tp, span, cn, cs; size_t smem; };

static bool pcm_plan(const dcs_resampler* r, int C, bool encode, int fmt, PcmPlan* pl) {
  const int64_t bank = (int64_t)r->Q * r->up * (int64_t)sizeof(double);
  const bool wide = encode || fmt != DCS_SAMPLE_I16;
  const int64_t bytes = wide ? (int64_t)sizeof(float) : (int64_t)sizeof(int16_t);
  for (int groups = 1; groups <= (wide ? C : 1); ++groups) {
    const int cn = (C + groups - 1) / groups;
    const int cs = encode ? (cn | 1) : cn;
    const int64_t per_round = (int64_t)r->up * (encode ? cn : 1);
    for (int64_t tp = std::max<int64_t>(1, 4 * RS_THREADS / per_round) * RS_V; tp >= RS_V; tp -= RS_V) {
      const int64_t span = (tp - 1) * r->down + r->cspan + r->Q;
      const int64_t smem = bank + span * cs * bytes;
      if (smem <= RS_SMEM_MAX) {
        pl->tp = (int)tp; pl->span = (int)span; pl->cn = cn; pl->cs = cs; pl->smem = (size_t)smem;
        return true;
      }
    }
  }
  return false;
}

template <class Kernel, class Args>
static int launch_pcm(const dcs_resampler* r, Kernel kernel, const char* scope, const PcmPlan& pl, Args a, cudaStream_t st) {
  dcs_ctx* ctx = r->ctx;
  a.bank = r->d_bank;
  a.up = r->up; a.down = r->down; a.Q = r->Q; a.half_len = r->half_len; a.c0 = r->c0;
  a.tp = pl.tp; a.span = pl.span; a.cn = pl.cn; a.cs = pl.cs;
  DCS_TRY(ensure_smem_attr(kernel, (int)pl.smem));
  int per_sm = 0;
  DCS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, RS_THREADS, pl.smem));
  const int64_t grid = std::min<int64_t>(a.ntiles, (int64_t)ctx->num_sms * std::max(per_sm, 1));
  ProfScope ps(ctx, scope, st);
  kernel<<<(unsigned)grid, RS_THREADS, pl.smem, st>>>(a);
  DCS_CHECK_LAUNCH();
  ctx->launches++;
  return DCS_OK;
}

int64_t resampler_length(const dcs_resampler* r, int64_t num_in) { return dcs_resampled_length(num_in, r->up, r->down); }
const dcs_ctx* resampler_ctx(const dcs_resampler* r) { return r->ctx; }
int resampler_up(const dcs_resampler* r) { return r->up; }
int resampler_down(const dcs_resampler* r) { return r->down; }
int resampler_ntaps(const dcs_resampler* r) { return r->ntaps; }

int check_resample_channels(const char* fn, const dcs_ctx* ctx, const dcs_resampler* to, const dcs_resampler* from, int C,
                            int in_fmt) {
  DCS_REQUIRE(to && from, "%s: NULL resampler", fn);
  DCS_REQUIRE(to->ctx == ctx && from->ctx == ctx, "%s: a resampler was made on another ctx", fn);
  DCS_REQUIRE(to->up == from->down && to->down == from->up,
              "%s: the resamplers %d/%d and %d/%d are not inverse (to_model up/down must be from_model down/up)", fn,
              to->up, to->down, from->up, from->down);
  PcmPlan pl;
  DCS_REQUIRE(pcm_plan(to, C, false, in_fmt, &pl), "%s: %d channels at %d/%d do not fit one tile in shared memory", fn, C,
              to->up, to->down);
  DCS_REQUIRE(pcm_plan(from, C, true, DCS_SAMPLE_F32, &pl), "%s: one channel at %d/%d does not fit one tile in shared memory",
              fn, from->up, from->down);
  return DCS_OK;
}

int resample_decode_groups(const dcs_resampler* r, int C, int fmt) {
  PcmPlan pl;
  return sample_bytes(fmt) > 0 && C >= 1 && pcm_plan(r, C, false, fmt, &pl) ? (C + pl.cn - 1) / pl.cn : 0;
}

// the decode / encode launches of a tile plan; a.tiles_t set, a.ntiles set here.  The decode of channel groups adds
// the downmix launch
template <class Args>
static int decode_launch(const dcs_resampler* r, int fmt, const PcmPlan& pl, Args a, cudaStream_t st) {
  const int groups = (a.C + pl.cn - 1) / pl.cn;
  a.ntiles = a.tiles_t * groups;
  switch (fmt) {
    case DCS_SAMPLE_I16: DCS_TRY(launch_pcm(r, resample_decode_kernel<DCS_SAMPLE_I16, Args>, "resample_decode", pl, a, st)); break;
    case DCS_SAMPLE_I32: DCS_TRY(launch_pcm(r, resample_decode_kernel<DCS_SAMPLE_I32, Args>, "resample_decode", pl, a, st)); break;
    case DCS_SAMPLE_I24: DCS_TRY(launch_pcm(r, resample_decode_kernel<DCS_SAMPLE_I24, Args>, "resample_decode", pl, a, st)); break;
    default: DCS_TRY(launch_pcm(r, resample_decode_kernel<DCS_SAMPLE_F32, Args>, "resample_decode", pl, a, st)); break;
  }
  if (groups == 1) return DCS_OK;
  float* planes = static_cast<float*>(a.out);
  ProfScope ps(r->ctx, "resample_decode_downmix", st);   // the channel groups' downmix: the same expression, the same bits
  return launch_downmix(r->ctx, planes + a.num_out, a.C, a.num_out, a.num_out, planes, st);
}

template <class Args>
static int encode_launch(const dcs_resampler* r, int fmt, const PcmPlan& pl, int nsrc, Args a, cudaStream_t st) {
  a.ntiles = a.tiles_t * ((a.C + pl.cn - 1) / pl.cn) * nsrc;
  switch (fmt) {
    case DCS_SAMPLE_I16: return launch_pcm(r, resample_encode_kernel<DCS_SAMPLE_I16, Args>, "resample_encode", pl, a, st);
    case DCS_SAMPLE_I32: return launch_pcm(r, resample_encode_kernel<DCS_SAMPLE_I32, Args>, "resample_encode", pl, a, st);
    case DCS_SAMPLE_I24: return launch_pcm(r, resample_encode_kernel<DCS_SAMPLE_I24, Args>, "resample_encode", pl, a, st);
    default: return launch_pcm(r, resample_encode_kernel<DCS_SAMPLE_F32, Args>, "resample_encode", pl, a, st);
  }
}

// the window's arguments: outputs [out_first, out_first + a->num_out), input j of the whole signal at in + (j - in_first)
// for j in [j_lo, j_hi)
static void set_window(const dcs_resampler* r, const PcmPlan& pl, int64_t out_first, int64_t in_first, int64_t j_lo,
                       int64_t j_hi, ResampleWinArgs* a) {
  a->win.out_first = out_first; a->win.p_first = out_first / r->up;
  a->win.in_first = in_first; a->win.j_lo = j_lo; a->win.j_hi = j_hi;
  a->tiles_t = ceil_div64((out_first + a->num_out - 1) / r->up - a->win.p_first + 1, pl.tp);
}

int launch_resample_decode(const dcs_resampler* r, int fmt, const void* d_in, int64_t L, int C, float* d_planes, int64_t Lout,
                           cudaStream_t st) {
  PcmPlan pl;
  DCS_REQUIRE(L >= 1 && Lout >= 1 && Lout <= resampler_length(r, L) && C >= 1 && C <= 16 && sample_bytes(fmt) > 0 &&
                  pcm_plan(r, C, false, fmt, &pl),
              "resample_decode: bad arguments");
  ResamplePcmArgs a{};
  a.in = d_in; a.num_in = L; a.out = d_planes; a.num_out = Lout; a.C = C;
  a.tiles_t = ceil_div64(ceil_div64(Lout, r->up), pl.tp);
  return decode_launch(r, fmt, pl, a, st);
}

int launch_resample_encode(const dcs_resampler* r, int fmt, const float* d_stems, int64_t Lin, int nsrc, int C, void* d_out,
                           int64_t L, cudaStream_t st) {
  PcmPlan pl;
  DCS_REQUIRE(Lin >= 1 && L >= 1 && L <= resampler_length(r, Lin) && nsrc >= 1 && C >= 1 && C <= 16 && sample_bytes(fmt) > 0 &&
                  pcm_plan(r, C, true, fmt, &pl),
              "resample_encode: bad arguments");
  ResamplePcmArgs a{};
  a.in = d_stems; a.num_in = Lin; a.out = d_out; a.num_out = L; a.C = C;
  a.tiles_t = ceil_div64(ceil_div64(L, r->up), pl.tp);
  return encode_launch(r, fmt, pl, nsrc, a, st);
}

int launch_resample_decode_range(const dcs_resampler* r, int fmt, const void* d_in, int64_t L, int64_t in_first,
                                 int64_t num_staged, int C, float* d_planes, int64_t out_first, int64_t Lout, cudaStream_t st) {
  PcmPlan pl;
  DCS_REQUIRE(L >= 1 && in_first >= 0 && num_staged >= 1 && in_first + num_staged <= L && out_first >= 0 && Lout >= 1 &&
                  out_first + Lout <= resampler_length(r, L) && C >= 1 && C <= 16 && sample_bytes(fmt) > 0 &&
                  pcm_plan(r, C, false, fmt, &pl),
              "resample_decode_range: bad arguments");
  ResampleWinArgs a{};
  a.in = d_in; a.num_in = L; a.out = d_planes; a.num_out = Lout; a.C = C;
  set_window(r, pl, out_first, in_first, in_first, in_first + num_staged, &a);
  return decode_launch(r, fmt, pl, a, st);
}

int launch_resample_encode_range(const dcs_resampler* r, int fmt, const float* d_stems, int64_t Lm, int64_t in_first,
                                 int64_t Lin, int nsrc, int C, void* d_out, int64_t out_first, int64_t L, cudaStream_t st) {
  PcmPlan pl;
  DCS_REQUIRE(Lm >= 1 && in_first >= 0 && Lin >= 1 && in_first + Lin <= Lm && out_first >= 0 && L >= 1 &&
                  out_first + L <= resampler_length(r, Lm) && nsrc >= 1 && C >= 1 && C <= 16 && sample_bytes(fmt) > 0 &&
                  pcm_plan(r, C, true, fmt, &pl),
              "resample_encode_range: bad arguments");
  ResampleWinArgs a{};
  a.in = d_stems; a.num_in = Lin; a.out = d_out; a.num_out = L; a.C = C;
  set_window(r, pl, out_first, in_first, in_first, in_first + Lin, &a);
  return encode_launch(r, fmt, pl, nsrc, a, st);
}

void resampler_support(const dcs_resampler* r, int64_t m_first, int64_t m_last, int64_t num_in, int64_t* lo, int64_t* hi) {
  *lo = std::max<int64_t>(0, support_lo(r->up, r->down, r->ntaps, m_first));
  *hi = std::min<int64_t>(num_in - 1, support_hi(r->up, r->down, r->ntaps, m_last));
}

}  // namespace dcs

extern "C" {

int64_t dcs_resampled_length(int64_t num_in, int up, int down) {
  if (num_in < 0 || up < 1 || down < 1) return -1;
  return (num_in * up + down - 1) / down;
}

int dcs_resampler_create(dcs_ctx* ctx, int up, int down, const double* h, int ntaps, dcs_resampler** out) {
  const char* fn = "dcs_resampler_create";
  DCS_REQUIRE(ctx && h && out, "%s: NULL argument", fn);
  DCS_REQUIRE(up >= 1 && down >= 1, "%s: up %d and down %d must be >= 1", fn, up, down);
  DCS_REQUIRE(gcd64(up, down) == 1, "%s: up %d and down %d are not coprime", fn, up, down);
  DCS_REQUIRE(ntaps >= 1 && ntaps % 2 == 1, "%s: ntaps %d must be odd and >= 1", fn, ntaps);
  const int64_t Q = ((int64_t)ntaps + up - 1) / up;
  const int64_t bank_bytes = Q * up * (int64_t)sizeof(double);
  DCS_REQUIRE(bank_bytes <= DCS_RESAMPLE_MAX_BANK_BYTES, "%s: the polyphase bank of %d/%d with %d taps is %lld bytes, over %d",
              fn, up, down, ntaps, (long long)bank_bytes, DCS_RESAMPLE_MAX_BANK_BYTES);
  const int half_len = (ntaps - 1) / 2;
  const int c0 = (int)(half_len / up);
  const int cspan = (int)(((int64_t)(up - 1) * down + half_len) / up) - c0;
  // periods per tile: as many as fit RS_TILE_WORDS staged samples, at least RS_V, a multiple of RS_V, and no more
  // work items than 4 rounds of the CTA
  int64_t tp = ((int64_t)RS_TILE_WORDS - cspan - Q) / down + 1;
  tp = std::min<int64_t>(tp, std::max<int64_t>(1, 4 * RS_THREADS / up) * RS_V);
  tp = std::max<int64_t>(RS_V, tp / RS_V * RS_V);
  const int64_t span = (tp - 1) * down + cspan + Q;
  const int64_t smem = bank_bytes + span * (int64_t)sizeof(float);
  DCS_REQUIRE(smem <= RS_SMEM_MAX, "%s: %d/%d with %d taps needs %lld bytes of shared memory per tile, over %d", fn, up,
              down, ntaps, (long long)smem, RS_SMEM_MAX);
  std::vector<double> bank((size_t)(Q * up), 0.0);
  for (int r = 0; r < up; ++r) {
    const int64_t ph = ((int64_t)r * down + half_len) % up;
    for (int64_t i = 0; i < Q && ph + i * up < ntaps; ++i) bank[(size_t)(i * up + r)] = h[ph + i * up];
  }
  DCS_CUDA(cudaSetDevice(ctx->device));
  dcs_resampler* p = new dcs_resampler();
  p->ctx = ctx; p->up = up; p->down = down; p->ntaps = ntaps; p->half_len = half_len; p->Q = (int)Q;
  p->c0 = c0; p->cspan = cspan; p->tp = (int)tp; p->span = (int)span; p->smem = (size_t)smem; p->d_bank = nullptr;
  cudaError_t e = cudaMalloc((void**)&p->d_bank, (size_t)bank_bytes);
  if (e == cudaSuccess) e = cudaMemcpy(p->d_bank, bank.data(), (size_t)bank_bytes, cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    set_error("%s: %s", fn, cudaGetErrorString(e));
    dcs_resampler_destroy(p);
    return e == cudaErrorMemoryAllocation ? DCS_ENOMEM : DCS_ECUDA;
  }
  *out = p;
  return DCS_OK;
}

int dcs_resampler_destroy(dcs_resampler* r) {
  if (!r) return DCS_OK;
  cudaFree(r->d_bank);
  delete r;
  return DCS_OK;
}

int dcs_resample(dcs_resampler* r, const float* d_in, int nplanes, int64_t in_stride, int64_t num_in, float* d_out,
                 int64_t out_stride, int64_t num_out, void* stream) {
  const char* fn = "dcs_resample";
  DCS_REQUIRE(r && d_in && d_out, "%s: NULL argument", fn);
  DCS_REQUIRE(nplanes >= 1, "%s: nplanes %d must be >= 1", fn, nplanes);
  DCS_REQUIRE(num_in >= 1, "%s: num_in %lld must be >= 1", fn, (long long)num_in);
  const int64_t most = dcs_resampled_length(num_in, r->up, r->down);
  DCS_REQUIRE(num_out >= 1 && num_out <= most, "%s: num_out %lld not in [1, %lld]", fn, (long long)num_out, (long long)most);
  DCS_REQUIRE(in_stride >= 0 && out_stride >= 0, "%s: negative stride", fn);
  DCS_REQUIRE(nplanes == 1 || (in_stride >= num_in && out_stride >= num_out),
              "%s: in_stride %lld < num_in %lld or out_stride %lld < num_out %lld", fn, (long long)in_stride,
              (long long)num_in, (long long)out_stride, (long long)num_out);
  DCS_REQUIRE((uintptr_t)d_in % sizeof(float) == 0 && (uintptr_t)d_out % sizeof(float) == 0, "%s: planes not 4-byte aligned",
              fn);
  cudaStream_t st = (cudaStream_t)stream;
  dcs_ctx* ctx = r->ctx;
  DCS_CUDA(cudaSetDevice(ctx->device));
  DCS_TRY(ensure_smem_attr(resample_kernel, (int)r->smem));
  ResampleArgs a;
  a.in = d_in; a.in_stride = in_stride; a.num_in = num_in;
  a.out = d_out; a.out_stride = out_stride; a.num_out = num_out;
  a.bank = r->d_bank;
  a.up = r->up; a.down = r->down; a.Q = r->Q; a.half_len = r->half_len; a.c0 = r->c0; a.tp = r->tp; a.span = r->span;
  a.tiles_per_plane = ceil_div64(ceil_div64(num_out, r->up), r->tp);
  a.ntiles = a.tiles_per_plane * nplanes;
  int per_sm = 0;
  DCS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, resample_kernel, RS_THREADS, r->smem));
  const int64_t grid = std::min<int64_t>(a.ntiles, (int64_t)ctx->num_sms * std::max(per_sm, 1));
  ProfScope ps(ctx, "resample", st);
  resample_kernel<<<(unsigned)grid, RS_THREADS, r->smem, st>>>(a);
  DCS_CHECK_LAUNCH();
  ctx->launches++;
  return DCS_OK;
}

}  // extern "C"
