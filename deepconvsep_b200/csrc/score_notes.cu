// score_notes.cu -- the normalised harmonic filters of the score-informed nets, rasterised on the device from the
// note table (the reference's `melody`, [ninst][nnotes][ncols]: first frame, last frame, MIDI number, then (lo, hi)
// bin pairs) instead of being built on the host as four dense planes (LargeDatasetMask2.filterSpec,
// dataset.py:839-862; deepconvsep_b200/score.py).
//
// The host compacts the rows that sound inside the frame window into a per-frame CSR of note records; one CTA per
// frame ORs the bin ranges of its notes into a shared-memory bitmap per instrument and writes
//     v_j = bit ? 1 : 1e-18f,   tot = ((v_0 + v_1) + v_2) + v_3,   out_j = v_j / tot   (times mag in channels mode)
// with IEEE division, i.e. filterSpec's float32 arithmetic bit for bit.
#include <math.h>
#include "common.cuh"

namespace dcs {

constexpr int SN_THREADS = 256;

// one frame per CTA; words = ceil(F / 32) bitmap words per instrument (dynamic shared memory)
__global__ void __launch_bounds__(SN_THREADS) score_notes_kernel(const int32_t* __restrict__ tab, NoteTable nt,
                                                                  const float* __restrict__ mag, float* __restrict__ out,
                                                                  int64_t ldf, int64_t plane) {
  extern __shared__ uint32_t bm[];   // [ninst][words]
  const int t = blockIdx.x;
  const int words = (nt.F + 31) >> 5;
  for (int i = threadIdx.x; i < nt.ninst * words; i += SN_THREADS) bm[i] = 0u;
  __syncthreads();
  const int32_t* frame_ptr = tab;
  const int32_t* entries = tab + nt.entries;
  const int32_t* recs = tab + nt.recs;       // (instrument, first range, range count) per sounding note
  const int32_t* ranges = tab + nt.ranges;   // (lo, hi) bin pairs, 0 <= lo < hi <= F
  const int e0 = frame_ptr[t], e1 = frame_ptr[t + 1];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int e = e0 + warp; e < e1; e += SN_THREADS / 32) {
    const int32_t* r = recs + 3 * entries[e];
    uint32_t* row = bm + r[0] * words;
    for (int k = lane; k < r[2]; k += 32) {
      const int lo = ranges[2 * (r[1] + k)], hi = ranges[2 * (r[1] + k) + 1];
      for (int w = lo >> 5; w <= (hi - 1) >> 5; ++w) {
        const int a = max(lo - (w << 5), 0), b = min(hi - (w << 5), 32);   // bits [a, b) of word w
        const uint32_t m = (b == 32 ? 0xffffffffu : ((1u << b) - 1u)) & ~((1u << a) - 1u);
        atomicOr(&row[w], m);
      }
    }
  }
  __syncthreads();
  const int64_t o = (int64_t)t * ldf;
  for (int b = threadIdx.x; b < ldf; b += SN_THREADS) {
    if (b >= nt.F) {   // pad columns
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (j < nt.ninst) out[j * plane + o + b] = 0.f;
      continue;
    }
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = j < nt.ninst && ((bm[j * words + (b >> 5)] >> (b & 31)) & 1u) ? 1.f : 1e-18f;
    float tot = v[0];   // numpy's sum over axis 0: one instrument after the other
#pragma unroll
    for (int j = 1; j < 4; ++j)
      if (j < nt.ninst) tot = tot + v[j];
    const float mg = mag ? mag[o + b] : 1.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (j >= nt.ninst) break;
      const float f = v[j] / tot;   // IEEE division (the build has no fast-math)
      out[j * plane + o + b] = mag ? f * mg : f;
    }
  }
}

// int(x) of Python on a float64 that is known to be finite: truncation toward zero
static inline double trunc_d(double x) { return x < 0 ? ceil(x) : floor(x); }

int notes_compact(const char* fn, const double* h_melody, int ninst, int nnotes, int ncols, int64_t start, int64_t T, int F,
                  std::vector<int32_t>* tab, NoteTable* nt) {
  DCS_REQUIRE(ninst >= 1 && ninst <= 4, "%s: ninst %d must be in [1, 4]", fn, ninst);
  DCS_REQUIRE(nnotes >= 0 && (nnotes == 0 || h_melody), "%s: bad note table (nnotes %d)", fn, nnotes);
  DCS_REQUIRE(ncols >= 3, "%s: ncols %d must be >= 3 (first frame, last frame, MIDI number, then bin pairs)", fn, ncols);
  DCS_REQUIRE(start >= 0 && T >= 1 && T < ((int64_t)1 << 30), "%s: frame window start %lld, T %lld out of range", fn,
              (long long)start, (long long)T);
  DCS_REQUIRE(F >= 1 && F <= 65536, "%s: F %d out of range [1, 65536]", fn, F);
  const int nh = (ncols - 3) / 2;
  const double stop = (double)(start + T), dstart = (double)start;
  // pass 1: validate every row whose MIDI number is > 0, whatever the window, and collect the sounding ones
  struct Row { int j; int64_t b, e; int off, cnt; };
  std::vector<Row> rows;
  std::vector<int32_t> rng;
  for (int j = 0; j < ninst; ++j)
    for (int p = 0; p < nnotes; ++p) {
      const double* r = h_melody + ((size_t)j * nnotes + p) * ncols;
      if (!(r[2] > 0)) continue;   // NaN ('?') fails this test, as in filterSpec
      DCS_REQUIRE(isfinite(r[0]) && isfinite(r[1]), "%s: instrument %d, note %d: non-finite frame (%g, %g)", fn, j, p, r[0], r[1]);
      const int off = (int)rng.size();
      for (int k = 0; k < nh; ++k) {
        const double ys = r[3 + 2 * k], ye = r[4 + 2 * k];
        DCS_REQUIRE(isfinite(ys) && isfinite(ye), "%s: instrument %d, note %d: non-finite bin range %d", fn, j, p, k);
        if (!(ye > 0)) continue;
        const double lo = trunc_d(ys), hi = trunc_d(ye);
        if (!(lo < hi)) continue;   // empty arange
        DCS_REQUIRE(lo >= 0 && hi <= F, "%s: instrument %d, note %d: bin range [%g, %g) outside [0, %d)", fn, j, p, lo, hi, F);
        rng.push_back((int32_t)lo);
        rng.push_back((int32_t)hi);
      }
      const double ov = fmax(0.0, fmin(r[1], stop) - fmax(r[0], dstart));
      const int64_t b = (int64_t)trunc_d(fmax(r[0], dstart)) - start, e = (int64_t)trunc_d(fmin(r[1], stop)) - start;
      const int cnt = (int)(rng.size() / 2) - off / 2;
      if (ov > 0 && e > b && cnt > 0) rows.push_back({j, b, e, off / 2, cnt});
      else rng.resize(off);
    }
  // pass 2: per-frame CSR of the sounding notes
  std::vector<int64_t> cnt(T + 1, 0);
  for (const Row& r : rows)
    for (int64_t t = r.b; t < r.e; ++t) cnt[t + 1]++;
  for (int64_t t = 0; t < T; ++t) cnt[t + 1] += cnt[t];
  const int64_t nnz = cnt[T], nrec = (int64_t)rows.size(), total = (T + 1) + nnz + 3 * nrec + (int64_t)rng.size();
  DCS_REQUIRE(total < ((int64_t)1 << 31), "%s: note table too large (%lld entries)", fn, (long long)total);
  nt->ninst = ninst; nt->F = F; nt->T = T;
  nt->entries = T + 1; nt->recs = nt->entries + nnz; nt->ranges = nt->recs + 3 * nrec; nt->size = total;
  tab->assign((size_t)total, 0);
  int32_t* d = tab->data();
  for (int64_t t = 0; t <= T; ++t) d[t] = (int32_t)cnt[t];
  std::vector<int64_t> fill(cnt.begin(), cnt.end() - 1);
  for (int64_t i = 0; i < nrec; ++i) {
    const Row& r = rows[i];
    for (int64_t t = r.b; t < r.e; ++t) d[nt->entries + fill[t]++] = (int32_t)i;
    d[nt->recs + 3 * i] = r.j; d[nt->recs + 3 * i + 1] = r.off; d[nt->recs + 3 * i + 2] = r.cnt;
  }
  if (!rng.empty()) memcpy(d + nt->ranges, rng.data(), rng.size() * sizeof(int32_t));
  return DCS_OK;
}

int notes_stage(dcs_ctx* ctx, const std::vector<int32_t>& tab, NoteTable* nt, cudaStream_t st) {
  const size_t bytes = tab.size() * sizeof(int32_t);
  if (!ctx->ev_notes) DCS_CUDA(cudaEventCreateWithFlags(&ctx->ev_notes, cudaEventDisableTiming));
  // the staging buffer is free again once the previous call's copy out of it has completed
  DCS_CUDA(cudaEventSynchronize(ctx->ev_notes));
  if (bytes > ctx->notes_host_cap) {
    if (ctx->notes_host) DCS_CUDA(cudaFreeHost(ctx->notes_host));
    ctx->notes_host = nullptr;
    ctx->notes_host_cap = 0;
    const size_t want = (bytes + (1u << 16) - 1) & ~((size_t)(1u << 16) - 1);
    DCS_CUDA(cudaMallocHost((void**)&ctx->notes_host, want));
    ctx->notes_host_cap = want;
  }
  DCS_TRY(ctx->net[NET_NOTES].ensure(bytes, st));
  memcpy(ctx->notes_host, tab.data(), bytes);
  DCS_CUDA(cudaMemcpyAsync(ctx->net[NET_NOTES].p, ctx->notes_host, bytes, cudaMemcpyHostToDevice, st));
  DCS_CUDA(cudaEventRecord(ctx->ev_notes, st));
  nt->d = ctx->net[NET_NOTES].as<int32_t>();
  return DCS_OK;
}

int launch_score_notes(dcs_ctx* ctx, const NoteTable& nt, const float* mag, float* out, int64_t ldf, int64_t plane,
                       cudaStream_t st) {
  const int smem = nt.ninst * ((nt.F + 31) / 32) * (int)sizeof(uint32_t);   // <= 32 KB (F <= 65536)
  score_notes_kernel<<<(unsigned)nt.T, SN_THREADS, smem, st>>>(nt.d, nt, mag, out, ldf, plane);
  DCS_CHECK_LAUNCH();
  ctx->launches++;
  return DCS_OK;
}

}  // namespace dcs
