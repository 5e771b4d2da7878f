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
#include <algorithm>
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
#pragma unroll
      for (int v = 0; v < RS_V; ++v) acc[v] = 0.0;
      for (int i = 0; i < a.Q; ++i) {
        const double hv = bank[i * a.up + r];
#pragma unroll
        for (int v = 0; v < RS_V; ++v) acc[v] = fma(hv, (double)xs[base + v * a.down - i], acc[v]);
      }
#pragma unroll
      for (int v = 0; v < RS_V; ++v) {
        const int64_t n = n0 + (int64_t)v * a.up;
        if (n < a.num_out) y[n] = (float)acc[v];
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
