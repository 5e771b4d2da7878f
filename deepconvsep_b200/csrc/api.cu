// api.cu -- C ABI of libdcs.so (include/dcs.h): context / workspace, STFT plans, model
// creation, and the host-side orchestration of the separation pipeline.
#include <stdarg.h>
#include <math.h>
#include <string.h>
#include <stdlib.h>
#include <map>
#include <mutex>
#include <utility>
#include <vector>
#include "common.cuh"

namespace dcs {

static thread_local char g_err[1024] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int DevBuf::ensure(size_t bytes, cudaStream_t stream, bool* grew) {
  if (grew) *grew = false;
  if (bytes <= cap) return DCS_OK;
  if (p) {
    DCS_CUDA(cudaStreamSynchronize(stream));
    DCS_CUDA(cudaFree(p));
    p = nullptr;
    cap = 0;
  }
  size_t want = (bytes + (1u << 20) - 1) & ~((size_t)(1u << 20) - 1);
  cudaError_t e = cudaMalloc(&p, want);
  if (e != cudaSuccess) {
    p = nullptr;
    set_error("cudaMalloc(%zu bytes) failed: %s", want, cudaGetErrorString(e));
    return DCS_ENOMEM;
  }
  cap = want;
  DCS_CUDA(cudaMemsetAsync(p, 0, want, stream));
  if (grew) *grew = true;
  return DCS_OK;
}

void DevBuf::release() {
  if (p) cudaFree(p);
  p = nullptr;
  cap = 0;
}

int ensure_smem_attr_impl(const void* kernel, int bytes) {
  int dev = 0;
  DCS_CUDA(cudaGetDevice(&dev));
  static std::mutex mu;
  static std::map<std::pair<const void*, int>, int> done;
  std::lock_guard<std::mutex> g(mu);
  const auto key = std::make_pair(kernel, dev);
  const auto it = done.find(key);
  if (it != done.end() && it->second >= bytes) return DCS_OK;
  DCS_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  done[key] = bytes;
  return DCS_OK;
}

int upload(const std::vector<float>& h, float** d, std::vector<void*>* owned) {
  DCS_CUDA(cudaMalloc((void**)d, h.size() * sizeof(float)));
  if (owned) owned->push_back(*d);
  DCS_CUDA(cudaMemcpy(*d, h.data(), h.size() * sizeof(float), cudaMemcpyHostToDevice));
  return DCS_OK;
}

bool shape_is(const int64_t* s, int nd, int want_nd, int64_t a, int64_t b, int64_t c, int64_t d) {
  return nd == want_nd && s[0] == a && s[1] == b && s[2] == c && s[3] == d;
}

int ensure_layout(dcs_ctx* ctx, NetSlot slot, size_t bytes, uint64_t sig, cudaStream_t st) {
  bool grew = false;
  DCS_TRY(ctx->net[slot].ensure(bytes, st, &grew));
  if (!grew && ctx->net_sig[slot] != sig) DCS_CUDA(cudaMemsetAsync(ctx->net[slot].p, 0, ctx->net[slot].cap, st));
  ctx->net_sig[slot] = sig;
  return DCS_OK;
}

}  // namespace dcs

using namespace dcs;

// every device buffer of a context's workspace
template <class Ctx, class F> static void for_each_buffer(Ctx* c, F f) {
  for (auto* b : {&c->audio, &c->X, &c->mag, &c->S, &c->stems, &c->pcm_in[0], &c->pcm_in[1], &c->pcm_out[0], &c->pcm_out[1], &c->wiener, &c->masks}) f(*b);
  for (auto& b : c->net) f(b);
}

extern "C" {

int dcs_version(void) { return DCS_VERSION; }
const char* dcs_last_error(void) { return g_err; }

int dcs_create(int device, dcs_ctx** out) {
  DCS_REQUIRE(out != nullptr, "dcs_create: out is NULL");
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    set_error("dcs_create: no usable CUDA device (%s); libdcs has no CPU fallback",
              e != cudaSuccess ? cudaGetErrorString(e) : "device count 0");
    return DCS_ECUDA;
  }
  DCS_REQUIRE(device >= 0 && device < n, "dcs_create: device %d out of range (%d devices)", device, n);
  DCS_CUDA(cudaSetDevice(device));
  cudaDeviceProp prop;
  DCS_CUDA(cudaGetDeviceProperties(&prop, device));
  DCS_REQUIRE(prop.major == 9 && prop.minor == 0, "dcs_create: device %d is sm_%d%d; this library is built for sm_90a only",
              device, prop.major, prop.minor);
  dcs_ctx* c = new dcs_ctx();
  c->device = device;
  c->num_sms = prop.multiProcessorCount;
  const char* dbg = getenv("DCS_DEBUG_SIMT_GEMM");
  c->debug_simt_gemm = dbg && dbg[0] == '1';
  *out = c;
  return DCS_OK;
}

int dcs_destroy(dcs_ctx* c) {
  if (!c) return DCS_OK;
  cudaSetDevice(c->device);
  for_each_buffer(c, [](DevBuf& b) { b.release(); });
  for (int i = 0; i < 2; ++i) {
    if (c->ev_in[i]) cudaEventDestroy(c->ev_in[i]);
    if (c->ev_dec[i]) cudaEventDestroy(c->ev_dec[i]);
    if (c->ev_enc[i]) cudaEventDestroy(c->ev_enc[i]);
    if (c->ev_out[i]) cudaEventDestroy(c->ev_out[i]);
  }
  if (c->ev_notes) {
    cudaEventSynchronize(c->ev_notes);   // the last copy out of the pinned staging has completed
    cudaEventDestroy(c->ev_notes);
  }
  if (c->notes_host) cudaFreeHost(c->notes_host);
  if (c->s_h2d) cudaStreamDestroy(c->s_h2d);
  if (c->s_d2h) cudaStreamDestroy(c->s_d2h);
  delete c;
  return DCS_OK;
}

int64_t dcs_workspace_bytes(const dcs_ctx* c) {
  int64_t s = 0;
  if (c) for_each_buffer(c, [&s](const DevBuf& b) { s += (int64_t)b.cap; });
  return s;
}
int64_t dcs_launch_count(const dcs_ctx* c) { return c ? c->launches : 0; }

int dcs_set_spectrum_tap(dcs_ctx* c, dcs_complex* d_S, int64_t capacity) {
  DCS_REQUIRE(c != nullptr && capacity >= 0, "dcs_set_spectrum_tap: bad argument");
  c->tap = (float2*)d_S;
  c->tap_cap = d_S ? capacity : 0;
  return DCS_OK;
}

int dcs_set_wiener(dcs_ctx* c, int iterations) {
  DCS_REQUIRE(c != nullptr, "dcs_set_wiener: NULL ctx");
  DCS_REQUIRE(iterations >= 0, "dcs_set_wiener: iterations %d must be >= 0", iterations);
  c->wiener_iters = iterations;
  return DCS_OK;
}

int dcs_set_wiener_radius(dcs_ctx* c, int radius) {
  DCS_REQUIRE(c != nullptr, "dcs_set_wiener_radius: NULL ctx");
  DCS_REQUIRE(radius >= 0, "dcs_set_wiener_radius: radius %d must be >= 0", radius);
  c->wiener_radius = radius;
  return DCS_OK;
}

int dcs_set_pool_tap(dcs_ctx* c, uint8_t* d_bits, int64_t capacity) {
  DCS_REQUIRE(c != nullptr && capacity >= 0, "dcs_set_pool_tap: bad argument");
  c->pool_tap = d_bits;
  c->pool_tap_cap = d_bits ? capacity : 0;
  return DCS_OK;
}

// the blended masked spectra the inverse STFT of this call consumed -> the caller's tap buffer
static int copy_tap(dcs_ctx* c, const float2* S, int64_t elems, cudaStream_t st) {
  if (!c->tap) return DCS_OK;
  DCS_REQUIRE(c->tap_cap >= elems, "spectrum tap holds %lld elements, this call produced %lld", (long long)c->tap_cap, (long long)elems);
  DCS_CUDA(cudaMemcpyAsync(c->tap, S, (size_t)elems * sizeof(float2), cudaMemcpyDeviceToDevice, st));
  return DCS_OK;
}

int dcs_profile(dcs_ctx* c, int enable) {
  DCS_REQUIRE(c != nullptr, "dcs_profile: NULL ctx");
  c->prof_on = enable != 0;
  return DCS_OK;
}

int dcs_profile_read(dcs_ctx* c, char* names_buf, int names_len, float* ms, int max_n) {
  DCS_REQUIRE(c && names_buf && ms && names_len > 0, "dcs_profile_read: bad argument");
  int n = 0;
  size_t pos = 0;
  names_buf[0] = 0;
  for (auto& r : c->prof) {
    float t = 0.f;
    if (n < max_n && cudaEventSynchronize(r.e1) == cudaSuccess && cudaEventElapsedTime(&t, r.e0, r.e1) == cudaSuccess) {
      const size_t len = strlen(r.name);
      if (pos + len + 2 < (size_t)names_len) {
        memcpy(names_buf + pos, r.name, len);
        pos += len;
        names_buf[pos++] = '\n';
        names_buf[pos] = 0;
        ms[n++] = t;
      }
    }
    cudaEventDestroy(r.e0);
    cudaEventDestroy(r.e1);
  }
  c->prof.clear();
  return n;
}

// ------------------------------------------------------------------------------------ STFT plan
int64_t dcs_num_frames(int64_t L, int hop) { return (L + hop - 1) / hop + 2; }
int64_t dcs_padded_bins(int N) { return ((int64_t)N / 2 + 1 + 7) / 8 * 8; }

int dcs_stft_plan(dcs_ctx* ctx, int N, int hop, const double* window, const double* syn_window, dcs_stft** out) {
  DCS_REQUIRE(ctx && window && out, "dcs_stft_plan: NULL argument");
  DCS_REQUIRE(N == 256 || N == 512 || N == 1024 || N == 2048 || N == 4096, "frame size %d not in {256..4096}", N);
  DCS_REQUIRE(hop > 0 && hop <= N && hop % 2 == 0, "hop %d must be even and in (0, %d]", hop, N);
  DCS_CUDA(cudaSetDevice(ctx->device));
  if (!syn_window) syn_window = window;
  std::vector<float> w(N), ws(N), w2(N), tw(2 * (size_t)N);
  for (int i = 0; i < N; ++i) {
    w[i] = (float)window[i];
    ws[i] = (float)syn_window[i];
    w2[i] = (float)(window[i] * syn_window[i]);
    const double a = -2.0 * M_PI * (double)i / (double)N;
    tw[2 * i] = (float)cos(a);
    tw[2 * i + 1] = (float)sin(a);
  }
  dcs_stft* p = new dcs_stft();
  p->ctx = ctx; p->N = N; p->hop = hop;
  p->d_win = p->d_wsyn = p->d_w2 = nullptr; p->d_tw = nullptr;
  int r = upload(w, &p->d_win);
  if (r == DCS_OK) r = upload(ws, &p->d_wsyn);
  if (r == DCS_OK) r = upload(w2, &p->d_w2);
  if (r == DCS_OK) r = upload(tw, (float**)&p->d_tw);
  if (r != DCS_OK) { dcs_stft_plan_destroy(p); return r; }
  *out = p;
  return DCS_OK;
}

int dcs_stft_plan_destroy(dcs_stft* p) {
  if (!p) return DCS_OK;
  cudaFree(p->d_win); cudaFree(p->d_wsyn); cudaFree(p->d_w2); cudaFree(p->d_tw);
  delete p;
  return DCS_OK;
}

int dcs_stft_forward(dcs_stft* p, const float* d_audio, int64_t L, dcs_complex* d_X, float* d_mag, float mag_scale,
                     int64_t ldf, void* stream) {
  DCS_REQUIRE(p && d_audio && L > 0, "dcs_stft_forward: bad argument");
  DCS_REQUIRE((uintptr_t)d_X % 8 == 0, "dcs_stft_forward: d_X not 8-byte aligned");
  DCS_CUDA(cudaSetDevice(p->ctx->device));
  return launch_stft(p, d_audio, L, (float2*)d_X, d_mag, nullptr, mag_scale, ldf, (cudaStream_t)stream);
}

int dcs_stft_forward_polar(dcs_stft* p, const float* d_audio, int64_t L, float* d_mag, float* d_phase, float mag_scale,
                           int64_t ldf, void* stream) {
  DCS_REQUIRE(p && d_audio && L > 0, "dcs_stft_forward_polar: bad argument");
  DCS_CUDA(cudaSetDevice(p->ctx->device));
  return launch_stft(p, d_audio, L, nullptr, d_mag, d_phase, mag_scale, ldf, (cudaStream_t)stream);
}

int dcs_istft(dcs_stft* p, const dcs_complex* d_S, int nsrc, int64_t T, int64_t ldf, int64_t src_stride, float* d_out,
              int64_t Lout, int64_t out_stride, void* stream) {
  DCS_REQUIRE(p && d_S && d_out && T > 0, "dcs_istft: bad argument");
  DCS_REQUIRE(ldf >= p->N / 2 + 1, "dcs_istft: ldf %lld < F %d", (long long)ldf, p->N / 2 + 1);
  DCS_REQUIRE(src_stride >= 0 && out_stride >= 0, "dcs_istft: negative stride");
  // sources must not share spectrum rows (reads past a row) nor output samples (CTAs of two sources race)
  DCS_REQUIRE(nsrc <= 1 || src_stride >= T * ldf, "dcs_istft: src_stride %lld < num_frames * ldf %lld",
              (long long)src_stride, (long long)(T * ldf));
  DCS_REQUIRE(nsrc <= 1 || out_stride >= Lout, "dcs_istft: out_stride %lld < num_out %lld", (long long)out_stride,
              (long long)Lout);
  DCS_REQUIRE((uintptr_t)d_S % 8 == 0, "dcs_istft: d_S not 8-byte aligned");
  DCS_CUDA(cudaSetDevice(p->ctx->device));
  return launch_istft(p, (const float2*)d_S, nullptr, nullptr, 1.f, nsrc, T, ldf, src_stride, d_out, Lout, out_stride,
                      (cudaStream_t)stream);
}

int dcs_istft_polar(dcs_stft* p, dcs_ctx* ctx, const float* d_mag, const float* d_phase, float mag_scale, int64_t T,
                    int64_t ldf, float* d_out, int64_t Lout, void* stream) {
  DCS_REQUIRE(p && d_mag && d_phase && d_out && T > 0, "dcs_istft_polar: bad argument");
  DCS_REQUIRE(ldf >= p->N / 2 + 1, "dcs_istft_polar: ldf %lld < F %d", (long long)ldf, p->N / 2 + 1);
  DCS_CUDA(cudaSetDevice(p->ctx->device));
  (void)ctx;
  return launch_istft(p, nullptr, d_mag, d_phase, mag_scale * sqrtf((float)p->N), 1, T, ldf, 0, d_out, Lout, Lout,
                      (cudaStream_t)stream);
}

// ------------------------------------------------------------------------------------ model
int64_t dcs_num_patches(int64_t T, int tc, int overlap, int patcher) {
  const int64_t step = tc - overlap;
  if (step <= 0) return 0;
  const int64_t lim = patcher == DCS_PATCHER_UTIL ? overlap : tc;
  if (T <= lim) return 0;
  return (T - lim - 1) / step + 1;
}

int dcs_model_nsources(const dcs_model* m) { return m ? m->nsrc : 0; }

int dcs_model_destroy(dcs_model* m) {
  if (!m) return DCS_OK;
  for (void* d : m->dev) cudaFree(d);
  delete m;
  return DCS_OK;
}

int dcs_model_create(dcs_ctx* ctx, int arch, int feat_size, int time_context, int nparams, const float* const* h_params,
                     const int64_t* shapes, const int* ndims, dcs_model** out) {
  DCS_REQUIRE(ctx && h_params && shapes && ndims && out, "dcs_model_create: NULL argument");
  // the 1x1 score net also runs on spectra of other widths through dcs_separate_spec_channels
  DCS_REQUIRE(feat_size >= 3 && (arch == DCS_ARCH_BACH10_SCORE_1X1 || ((feat_size - 1) & (feat_size - 2)) == 0),
              "feat_size %d is not 2^k+1", feat_size);
  DCS_REQUIRE(time_context >= 4 && time_context <= 64, "time_context %d out of range", time_context);
  DCS_CUDA(cudaSetDevice(ctx->device));
  dcs_model* m = new dcs_model();
  m->ctx = ctx; m->arch = arch; m->F = feat_size; m->tc = time_context;
  int r;
  switch (arch) {
    case DCS_ARCH_DSD:
    case DCS_ARCH_DSD_ILD: r = model_create_dsd(m, nparams, h_params, shapes, ndims); break;
    case DCS_ARCH_IKALA:
    case DCS_ARCH_IKALA_NOPOOL:
    case DCS_ARCH_BACH10:
    case DCS_ARCH_BACH10_SCORE: r = model_create_sconv(m, nparams, h_params, shapes, ndims); break;
    case DCS_ARCH_BACH10_SCORE_1X1: r = model_create_s1x1(m, nparams, h_params, shapes, ndims); break;
    default:
      set_error("dcs_model_create: architecture %d has no CUDA path yet", arch);
      r = DCS_EINVAL;
  }
  if (r != DCS_OK) { dcs_model_destroy(m); return r; }
  *out = m;
  return DCS_OK;
}

// ------------------------------------------------------------------------------------ pipeline
// the network stage of every entry point: the input planes (plane stride in_plane) and the mixture STFT
// (channel stride x_plane) -> masked spectra, nsrc x nch planes of stride src_stride.  M (masks mode): the blended
// masks instead, float planes ordered like the spectra, bins < F of each frame written; X and S are not used
static int run_network(dcs_ctx* ctx, const dcs_model* m, const float* in, int64_t in_plane, const float2* X, int64_t x_plane,
                       int64_t T, int64_t ldf, int overlap, int patcher, float2* S, int64_t src_stride, cudaStream_t st,
                       float* M = nullptr) {
  const bool dsd = m->arch == DCS_ARCH_DSD || m->arch == DCS_ARCH_DSD_ILD;
  NetCall n;
  n.P = dcs_num_patches(T, m->tc, overlap, patcher);
  if (n.P == 0) {  // clip shorter than one patch: nothing is predicted, every stem is silence (every mask 0)
    for (int s = 0; s < m->nsrc * m->nch; ++s) {
      if (M)
        DCS_CUDA(cudaMemset2DAsync(M + s * src_stride, (size_t)ldf * sizeof(float), 0, (size_t)m->F * sizeof(float), (size_t)T, st));
      else
        DCS_CUDA(cudaMemsetAsync(S + s * src_stride, 0, (size_t)T * ldf * sizeof(float2), st));
    }
    return DCS_OK;
  }
  n.in = in; n.in_plane = in_plane; n.X = X; n.x_plane = x_plane; n.S = S; n.src_stride = src_stride; n.M = M;
  n.T = T; n.ldf = ldf; n.overlap = overlap; n.step = m->tc - overlap;
  n.Tp = std::max<int64_t>(T, (n.P - 1) * n.step + m->tc);
  // the zero-padded slots are re-zeroed when the model changes; those of the 30-channel nets also when the overlap does
  n.sig = ((uint64_t)(m->arch + 1) << 48) ^ ((uint64_t)m->F << 24) ^ (uint64_t)(m->tc * 64 + (dsd ? 0 : overlap));
  if (dsd) return dsd_forward(ctx, m, n, st);
  return m->arch == DCS_ARCH_BACH10_SCORE_1X1 ? s1x1_forward(ctx, m, n, st) : sconv_forward(ctx, m, n, st);
}

static bool score_arch(int arch) { return arch == DCS_ARCH_BACH10_SCORE || arch == DCS_ARCH_BACH10_SCORE_1X1; }
// input planes of the score-informed nets
static int score_planes(const dcs_model* m) { return m->arch == DCS_ARCH_BACH10_SCORE_1X1 ? 4 : m->sc.nch; }

// arch: the architecture an entry point serves (DCS_ARCH_BACH10_SCORE: both score-informed nets), -1 for the
// single-channel nets
static int check_model(const char* fn, const dcs_ctx* ctx, const dcs_model* m, int arch, int overlap, int patcher) {
  DCS_REQUIRE(ctx && m, "%s: NULL argument", fn);
  const bool mono = m->arch != DCS_ARCH_DSD_ILD && !score_arch(m->arch);
  DCS_REQUIRE(arch < 0 ? mono : (arch == DCS_ARCH_BACH10_SCORE ? score_arch(m->arch) : m->arch == arch),
              "%s does not serve architecture %d: use %s", fn, m->arch,
              m->arch == DCS_ARCH_DSD_ILD ? "dcs_separate_audio_stereo"
              : score_arch(m->arch)       ? "dcs_separate_audio_score / dcs_separate_spec_channels"
                                          : "dcs_separate_audio / dcs_separate_spec");
  DCS_REQUIRE(overlap >= 0 && overlap < m->tc, "overlap %d must be in [0, time_context=%d)", overlap, m->tc);
  DCS_REQUIRE(patcher == DCS_PATCHER_STANDALONE || patcher == DCS_PATCHER_UTIL, "unknown patcher %d", patcher);
  return DCS_OK;
}

// the check every clip entry point makes before it queues anything: a clip of L samples (audio planes in_stride
// apart) into stems out_stride apart
static int check_clip(const char* fn, const dcs_ctx* ctx, const dcs_model* m, const dcs_stft* p, int arch, const void* in,
                      const void* out, int64_t L, int64_t in_stride, int64_t out_stride, int overlap, int patcher) {
  DCS_TRY(check_model(fn, ctx, m, arch, overlap, patcher));
  DCS_REQUIRE(p && in && out, "%s: NULL argument", fn);
  DCS_REQUIRE(p->N / 2 + 1 == m->F, "%s: frame size %d does not give the model's %d bins", fn, p->N, m->F);
  DCS_REQUIRE(L > 0 && in_stride >= L && out_stride >= L, "%s: bad length / stride", fn);
  return DCS_OK;
}

// the workspace of a clip of L samples: nch STFT planes, nsrc x nch masked spectra, the score-informed net's input
// channels; with `staged` also the device copies of host audio and stems.  The stereo net with the Wiener post-filter
// on: its partial sums and covariances.  masks (masks-output mode): the magnitude planes and the network's buffers only
// -- no mixture STFT, no spectra, no Wiener workspace
static int size_workspace(dcs_ctx* ctx, const dcs_model* m, const dcs_stft* p, int64_t L, bool staged, cudaStream_t st,
                          bool masks = false) {
  const int64_t plane = dcs_num_frames(L, p->hop) * dcs_padded_bins(p->N);
  if (!masks) DCS_TRY(ctx->X.ensure((size_t)m->nch * plane * sizeof(float2), st));
  DCS_TRY(ctx->mag.ensure((size_t)m->nch * plane * sizeof(float), st));
  if (!masks) DCS_TRY(ctx->S.ensure((size_t)m->nsrc * m->nch * plane * sizeof(float2), st));
  if (score_arch(m->arch)) DCS_TRY(ctx->net[NET_CHANS].ensure((size_t)score_planes(m) * plane * sizeof(float), st));
  if (!masks && ctx->wiener_iters > 0 && m->nch == 2)
    DCS_TRY(ctx->wiener.ensure(wiener_workspace_bytes(m->nsrc, 2, dcs_num_frames(L, p->hop), m->F, ctx->wiener_radius), st));
  if (staged) {
    DCS_TRY(ctx->audio.ensure((size_t)L * sizeof(float), st));
    DCS_TRY(ctx->stems.ensure((size_t)m->nsrc * L * sizeof(float), st));
  }
  return DCS_OK;
}

// the workspace of downmix_clip: the masks-output workspace, the downmix, the nsrc mask planes and ONE mixture STFT
// plane, whatever the channel count.  wx > 0 (the filter on, wx channels): wx STFT planes, nsrc x wx masked spectra
// and the filter's sums over covariance windows of `radius` chunks.  staged > 0 (the int16 batch of `staged` channels):
// staged + 1 audio planes (the downmix, then the channels) and nsrc x staged stem planes
static int size_downmix_workspace(dcs_ctx* ctx, const dcs_model* m, const dcs_stft* p, int64_t L, int wx, int radius, int staged,
                                  cudaStream_t st) {
  const int64_t plane = dcs_num_frames(L, p->hop) * dcs_padded_bins(p->N);
  DCS_TRY(size_workspace(ctx, m, p, L, false, st, true));
  DCS_TRY(ctx->audio.ensure((size_t)(staged + 1) * L * sizeof(float), st));
  DCS_TRY(ctx->masks.ensure((size_t)m->nsrc * plane * sizeof(float), st));
  DCS_TRY(ctx->X.ensure((size_t)(wx > 0 ? wx : 1) * plane * sizeof(float2), st));
  if (wx > 0) {
    DCS_TRY(ctx->S.ensure((size_t)m->nsrc * wx * plane * sizeof(float2), st));
    DCS_TRY(ctx->wiener.ensure(wiener_workspace_bytes(m->nsrc, wx, dcs_num_frames(L, p->hop), m->F, radius), st));
  }
  if (staged > 0) DCS_TRY(ctx->stems.ensure((size_t)m->nsrc * staged * L * sizeof(float), st));
  return DCS_OK;
}

// one clip, device to device: nch audio planes (audio_stride apart) -> nsrc x nch stem planes; d_filters: the
// score filters that form the score-informed net's input channels.  The stereo net's stems go through the Wiener
// post-filter between the network and the iSTFT when dcs_set_wiener is above 0, with the covariance window of
// dcs_set_wiener_radius.  masks (masks-output mode): d_stems receives the network's blended masks instead, float planes
// [T][ldf] stem_stride apart in the order of the stems; the STFT writes the magnitude only and there is no Wiener pass,
// spectrum tap or iSTFT
static int separate_clip(dcs_ctx* ctx, const dcs_model* m, dcs_stft* p, const float* d_audio, int64_t audio_stride, int64_t L,
                         const float* d_filters, const NoteTable* notes, float scale_factor, int overlap, int patcher,
                         float* d_stems, int64_t stem_stride, cudaStream_t st, bool masks = false) {
  DCS_TRY(size_workspace(ctx, m, p, L, false, st, masks));
  const int nch = m->nch;
  const int64_t T = dcs_num_frames(L, p->hop), ldf = dcs_padded_bins(p->N), plane = T * ldf;
  float2 *X = masks ? nullptr : ctx->X.as<float2>(), *S = masks ? nullptr : ctx->S.as<float2>();
  float* mag = ctx->mag.as<float>();
  {
    ProfScope ps(ctx, "stft_fwd", st);   // compute_transform: one STFT per channel (transform.py:105-119)
    for (int ch = 0; ch < nch; ++ch)
      DCS_TRY(launch_stft(p, d_audio + ch * audio_stride, L, masks ? nullptr : X + ch * plane, mag + ch * plane, nullptr,
                          scale_factor, ldf, st));
  }
  const float* in = mag;
  if (d_filters || notes) {
    float* chans = ctx->net[NET_CHANS].as<float>();
    ProfScope ps(ctx, "score_channels", st);
    if (notes)   // the filters rasterised from the note table, times mag: no filter plane in memory
      DCS_TRY(launch_score_notes(ctx, *notes, mag, chans, ldf, plane, st));
    else
      DCS_TRY(launch_channel_mul(ctx, mag, d_filters, chans, plane, score_planes(m), st));
    in = chans;
  }
  if (masks) return run_network(ctx, m, in, plane, nullptr, 0, T, ldf, overlap, patcher, nullptr, stem_stride, st, d_stems);
  if (m->arch == DCS_ARCH_DSD && nch == 1 && istft_reg_supported(p, d_stems, stem_stride)) {
    // the mono DSD100 / HHDS net: the network writes its masks (float planes, in the spectra's allocation) and the
    // register iSTFT forms M_s * X as it reads each row, X shared by the four sources -- the same products the mask
    // kernel's spectra mode stores, so the same stems, with no masked spectra in memory.  A spectrum tap gets them
    // from one elementwise pass
    float* M = reinterpret_cast<float*>(S);
    DCS_TRY(run_network(ctx, m, in, plane, X, plane, T, ldf, overlap, patcher, nullptr, plane, st, M));
    if (ctx->tap) {
      DCS_REQUIRE(ctx->tap_cap >= (int64_t)m->nsrc * plane, "spectrum tap holds %lld elements, this call produced %lld",
                  (long long)ctx->tap_cap, (long long)m->nsrc * plane);
      DCS_TRY(launch_masked_spectra(ctx, M, X, m->nsrc, plane, ldf, m->F, ctx->tap, st));
    }
    ProfScope ps(ctx, "istft_ola", st);
    return launch_istft(p, X, nullptr, nullptr, 1.f, m->nsrc, T, ldf, plane, d_stems, L, stem_stride, st, M, plane, 1);
  }
  DCS_TRY(run_network(ctx, m, in, plane, X, plane, T, ldf, overlap, patcher, S, plane, st));
  if (ctx->wiener_iters > 0 && nch == 2)
    DCS_TRY(launch_wiener(ctx, X, plane, S, plane, m->nsrc, T, ldf, m->F, ctx->wiener_iters, ctx->wiener_radius, st));
  DCS_TRY(copy_tap(ctx, S, (int64_t)m->nsrc * nch * plane, st));
  ProfScope ps(ctx, "istft_ola", st);
  return launch_istft(p, S, nullptr, nullptr, 1.f, m->nsrc * nch, T, ldf, plane, d_stems, L, stem_stride, st);
}

// channel by channel through ONE mixture STFT plane of the workspace: X-only STFT of channel c, then the masked inverse
// STFT of its nsrc stems, planes (s * nx + c)
static int apply_masks(dcs_ctx* ctx, dcs_stft* p, const float* d_audio, int nx, int64_t audio_stride, int64_t L,
                       const float* d_masks, int nsrc, int64_t m_stride, float* d_stems, int64_t stem_stride, cudaStream_t st) {
  const int64_t T = dcs_num_frames(L, p->hop), ldf = dcs_padded_bins(p->N), plane = T * ldf;
  DCS_TRY(ctx->X.ensure((size_t)plane * sizeof(float2), st));
  float2* X = ctx->X.as<float2>();
  for (int c = 0; c < nx; ++c) {
    {
      ProfScope ps(ctx, "stft_fwd", st);
      DCS_TRY(launch_stft(p, d_audio + c * audio_stride, L, X, nullptr, nullptr, 1.f, ldf, st));
    }
    ProfScope ps(ctx, "istft_masked", st);
    DCS_TRY(launch_istft(p, X, nullptr, nullptr, 1.f, nsrc, T, ldf, plane, d_stems + c * stem_stride, L, nx * stem_stride, st,
                         d_masks, m_stride, 1));
  }
  return DCS_OK;
}

// keep-channels without the Wiener post-filter forms no masked spectra: a spectrum tap is refused before anything is
// queued
static int check_keep_tap(const char* fn, const dcs_ctx* ctx) {
  DCS_REQUIRE(!ctx->tap || ctx->wiener_iters > 0,
              "%s: a spectrum tap is set (dcs_set_spectrum_tap), and without the Wiener post-filter this path forms no masked "
              "spectra to copy", fn);
  return DCS_OK;
}

// Stems of nx channels (audio_stride apart) from the masks of their downmix d_mono, single-channel nets: the network
// in masks mode into ctx->masks, then those masks applied to every channel inside the inverse STFT, planes (s * nx + c).
// d_mono NULL: the downmix is formed here, into ctx->audio.  iterations > 0 (nx in [2, 8]): the Wiener post-filter's
// first pass forms the masked spectra M_s * X_c of all nx channels in memory; `iterations` EM iterations over covariance
// windows of `radius` chunks filter them, and they are copied to the spectrum tap and inverted
static int downmix_clip(dcs_ctx* ctx, const dcs_model* m, dcs_stft* p, const float* d_mono, const float* d_audio, int nx,
                        int64_t audio_stride, int64_t L, int iterations, int radius, float scale_factor, int overlap,
                        int patcher, float* d_stems, int64_t stem_stride, cudaStream_t st) {
  const bool filter = iterations > 0;
  DCS_TRY(size_downmix_workspace(ctx, m, p, L, filter ? nx : 0, radius, 0, st));
  const int64_t T = dcs_num_frames(L, p->hop), ldf = dcs_padded_bins(p->N), plane = T * ldf;
  float* masks = ctx->masks.as<float>();
  if (!d_mono) {
    ProfScope ps(ctx, "downmix", st);
    DCS_TRY(launch_downmix(ctx, d_audio, nx, audio_stride, L, ctx->audio.as<float>(), st));
    d_mono = ctx->audio.as<float>();
  }
  DCS_TRY(separate_clip(ctx, m, p, d_mono, L, L, nullptr, nullptr, scale_factor, overlap, patcher, masks, plane, st, true));
  if (!filter) return apply_masks(ctx, p, d_audio, nx, audio_stride, L, masks, m->nsrc, plane, d_stems, stem_stride, st);
  float2 *X = ctx->X.as<float2>(), *S = ctx->S.as<float2>();
  {
    ProfScope ps(ctx, "stft_fwd", st);
    for (int c = 0; c < nx; ++c) DCS_TRY(launch_stft(p, d_audio + c * audio_stride, L, X + c * plane, nullptr, nullptr, 1.f, ldf, st));
  }
  DCS_TRY(launch_wiener(ctx, X, plane, S, plane, m->nsrc, T, ldf, m->F, iterations, radius, st, masks, plane, nx));
  DCS_TRY(copy_tap(ctx, S, (int64_t)m->nsrc * nx * plane, st));
  ProfScope ps(ctx, "istft_ola", st);
  return launch_istft(p, S, nullptr, nullptr, 1.f, m->nsrc * nx, T, ldf, plane, d_stems, L, stem_stride, st);
}

int dcs_separate_spec(dcs_ctx* ctx, dcs_model* m, const float* d_mag, const dcs_complex* d_X, int64_t T, int64_t ldf,
                      int overlap, int patcher, dcs_complex* d_S, int64_t src_stride, void* stream) {
  DCS_TRY(check_model("dcs_separate_spec", ctx, m, -1, overlap, patcher));
  DCS_REQUIRE(d_mag && d_X && d_S, "dcs_separate_spec: NULL argument");
  DCS_REQUIRE(T > 0 && ldf >= m->F && src_stride >= T * ldf, "dcs_separate_spec: bad shape");
  DCS_CUDA(cudaSetDevice(ctx->device));
  return run_network(ctx, m, d_mag, 0, (const float2*)d_X, 0, T, ldf, overlap, patcher, (float2*)d_S, src_stride,
                     (cudaStream_t)stream);
}

int dcs_separate_spec_channels(dcs_ctx* ctx, dcs_model* m, const float* d_in, int64_t in_plane, const dcs_complex* d_X,
                               int64_t T, int64_t ldf, int overlap, int patcher, dcs_complex* d_S, int64_t src_stride,
                               void* stream) {
  DCS_TRY(check_model("dcs_separate_spec_channels", ctx, m, DCS_ARCH_BACH10_SCORE, overlap, patcher));
  DCS_REQUIRE(d_in && d_X && d_S, "dcs_separate_spec_channels: NULL argument");
  DCS_REQUIRE(T > 0 && ldf >= m->F && src_stride >= T * ldf && in_plane >= T * ldf, "dcs_separate_spec_channels: bad shape");
  DCS_CUDA(cudaSetDevice(ctx->device));
  return run_network(ctx, m, d_in, in_plane, (const float2*)d_X, 0, T, ldf, overlap, patcher, (float2*)d_S, src_stride,
                     (cudaStream_t)stream);
}

int dcs_separate_audio_score(dcs_ctx* ctx, dcs_model* m, dcs_stft* p, const float* d_audio, int64_t L, const float* d_filters,
                             float scale_factor, int overlap, int patcher, float* d_stems, int64_t stem_stride, void* stream) {
  DCS_TRY(check_clip("dcs_separate_audio_score", ctx, m, p, DCS_ARCH_BACH10_SCORE, d_audio, d_stems, L, L, stem_stride,
                     overlap, patcher));
  DCS_REQUIRE(d_filters, "dcs_separate_audio_score: NULL filters");
  DCS_CUDA(cudaSetDevice(ctx->device));
  return separate_clip(ctx, m, p, d_audio, L, L, d_filters, nullptr, scale_factor, overlap, patcher, d_stems,
                       stem_stride, (cudaStream_t)stream);
}

int dcs_score_filters(dcs_ctx* ctx, const double* h_melody, int ninst, int nnotes, int ncols, int64_t start, int64_t T, int F,
                      const float* d_mag, int64_t ldf, float* d_out, int64_t plane, void* stream) {
  DCS_REQUIRE(ctx && d_out, "dcs_score_filters: NULL argument");
  std::vector<int32_t> tab;
  NoteTable nt;
  DCS_TRY(notes_compact("dcs_score_filters", h_melody, ninst, nnotes, ncols, start, T, F, &tab, &nt));
  DCS_REQUIRE(ldf >= F && ldf < ((int64_t)1 << 31) && plane >= T * ldf, "dcs_score_filters: bad shape (ldf %lld, plane %lld)",
              (long long)ldf, (long long)plane);
  cudaStream_t st = (cudaStream_t)stream;
  DCS_CUDA(cudaSetDevice(ctx->device));
  DCS_TRY(notes_stage(ctx, tab, &nt, st));
  ProfScope ps(ctx, "score_filters", st);
  return launch_score_notes(ctx, nt, d_mag, d_out, ldf, plane, st);
}

int dcs_separate_audio_notes(dcs_ctx* ctx, dcs_model* m, dcs_stft* p, const float* d_audio, int64_t L, const double* h_melody,
                             int nnotes, int ncols, int64_t frame0, float scale_factor, int overlap, int patcher, float* d_stems,
                             int64_t stem_stride, void* stream) {
  DCS_TRY(check_clip("dcs_separate_audio_notes", ctx, m, p, DCS_ARCH_BACH10_SCORE, d_audio, d_stems, L, L, stem_stride,
                     overlap, patcher));
  std::vector<int32_t> tab;
  NoteTable nt;
  DCS_TRY(notes_compact("dcs_separate_audio_notes", h_melody, score_planes(m), nnotes, ncols, frame0,
                        dcs_num_frames(L, p->hop), m->F, &tab, &nt));
  cudaStream_t st = (cudaStream_t)stream;
  DCS_CUDA(cudaSetDevice(ctx->device));
  DCS_TRY(notes_stage(ctx, tab, &nt, st));
  return separate_clip(ctx, m, p, d_audio, L, L, nullptr, &nt, scale_factor, overlap, patcher, d_stems, stem_stride,
                       st);
}

// one GEMM on view g with the host weight h_B[K][g.ldb]: uploaded for the FFMA kernel (engine 0) or transposed and
// split for the tensor cores (engine 1, with the epilogue epi); the stream is synchronised before the weight is freed
static int gemm_host_weight(const char* fn, dcs_ctx* ctx, int engine, int epi, GemmDesc g, const float* h_B, cudaStream_t st) {
  float* d_B = nullptr;
  TcWeight w;
  int r;
  if (engine == 1) {
    r = tc_weight_create(h_B, g.ldb, g.K, g.N, &w);
    if (r == DCS_OK) r = epi ? launch_gemm_tc_epi(ctx, g, w, epi, st) : launch_gemm_tc(ctx, g, w, st);
  } else {
    std::vector<float> hB((size_t)g.K * g.N);
    for (int k = 0; k < g.K; ++k) memcpy(&hB[(size_t)k * g.N], h_B + (size_t)k * g.ldb, (size_t)g.N * sizeof(float));
    r = upload(hB, &d_B);
    g.B = d_B; g.ldb = g.N;
    if (r == DCS_OK) r = launch_gemm(ctx, g, st);
  }
  cudaError_t e = cudaStreamSynchronize(st);
  tc_weight_destroy(&w);
  if (d_B) cudaFree(d_B);
  if (r == DCS_OK && e != cudaSuccess) {
    set_error("%s: %s", fn, cudaGetErrorString(e));
    return DCS_ECUDA;
  }
  return r;
}

int dcs_gemm_f32(dcs_ctx* ctx, int engine, const float* d_A, int64_t lda, const float* h_B, int64_t ldb,
                 const float* h_bias, float* d_C, int64_t ldc, int M, int N, int K, int relu, void* stream) {
  DCS_REQUIRE(ctx && d_A && h_B && d_C && M > 0 && N > 0 && K > 0, "dcs_gemm_f32: bad argument");
  DCS_REQUIRE(lda >= 1 && ldb >= N && ldc >= N, "dcs_gemm_f32: leading dimension too small");  // lda < K: overlapping rows
  DCS_CUDA(cudaSetDevice(ctx->device));
  float* d_bias = nullptr;
  if (h_bias) DCS_TRY(upload(std::vector<float>(h_bias, h_bias + N), &d_bias));
  const GemmDesc g = gemm_plain(d_A, lda, nullptr, ldb, d_bias, d_C, ldc, M, N, K, relu);
  const int r = gemm_host_weight("dcs_gemm_f32", ctx, engine, 0, g, h_B, (cudaStream_t)stream);
  if (d_bias) cudaFree(d_bias);
  return r;
}

static_assert(sizeof(dcs_gemm_view) == sizeof(GemmDesc) && offsetof(dcs_gemm_view, ldb) == offsetof(GemmDesc, ldb) &&
                  offsetof(dcs_gemm_view, kc_rows) == offsetof(GemmDesc, kc_rows) &&
                  offsetof(dcs_gemm_view, g_lim) == offsetof(GemmDesc, g_lim),
              "dcs_gemm_view must mirror GemmDesc");

int dcs_gemm_view_f32(dcs_ctx* ctx, int engine, int epi, const dcs_gemm_view* view, const float* h_B, void* stream) {
  DCS_REQUIRE(ctx && view && h_B && view->A && view->C, "dcs_gemm_view_f32: NULL argument");
  DCS_REQUIRE(engine == 0 || engine == 1, "dcs_gemm_view_f32: unknown engine %d", engine);
  DCS_REQUIRE(epi >= 0 && epi <= (EPI_POST | EPI_GATE) && (epi == 0 || engine == 1),
              "dcs_gemm_view_f32: epilogue %d needs engine 1", epi);
  GemmDesc g;
  memcpy(&g, view, sizeof g);
  DCS_REQUIRE(g.M > 0 && g.N > 0 && g.K > 0 && g.ldb >= g.N, "dcs_gemm_view_f32: bad shape");
  DCS_REQUIRE(g.m_inner > 0 && g.m_inner2 > 0 && g.k_seg > 0 && g.cm_inner > 0 && g.cm_inner2 > 0 && g.n_seg > 0 &&
                  (g.kc_rows == 0 || (g.kc_rows > 0 && g.kc_unit > 0 && g.kc_taps > 0)),
              "dcs_gemm_view_f32: bad view");
  DCS_CUDA(cudaSetDevice(ctx->device));
  return gemm_host_weight("dcs_gemm_view_f32", ctx, engine, epi, g, h_B, (cudaStream_t)stream);
}

static_assert(sizeof(dcs_dsd_mask_view) == sizeof(DsdMaskArgs) && offsetof(dcs_dsd_mask_view, ldw) == offsetof(DsdMaskArgs, ldw) &&
                  offsetof(dcs_dsd_mask_view, X) == offsetof(DsdMaskArgs, X) &&
                  offsetof(dcs_dsd_mask_view, src_stride) == offsetof(DsdMaskArgs, src_stride) &&
                  offsetof(dcs_dsd_mask_view, F) == offsetof(DsdMaskArgs, F) &&
                  offsetof(dcs_dsd_mask_view, ndec) == offsetof(DsdMaskArgs, ndec),
              "dcs_dsd_mask_view must mirror DsdMaskArgs");
static_assert(sizeof(dcs_dsd_convt2_view) == sizeof(DsdConvT2Args) && offsetof(dcs_dsd_convt2_view, G) == offsetof(DsdConvT2Args, G) &&
                  offsetof(dcs_dsd_convt2_view, ldg) == offsetof(DsdConvT2Args, ldg) &&
                  offsetof(dcs_dsd_convt2_view, tc) == offsetof(DsdConvT2Args, tc),
              "dcs_dsd_convt2_view must mirror DsdConvT2Args");
static_assert(sizeof(dcs_dsd_dense_view) == sizeof(DsdDenseArgs) && offsetof(dcs_dsd_dense_view, apad) == offsetof(DsdDenseArgs, apad) &&
                  offsetof(dcs_dsd_dense_view, nfc) == offsetof(DsdDenseArgs, nfc),
              "dcs_dsd_dense_view must mirror DsdDenseArgs");
static_assert(sizeof(dcs_sconv_mask_view) == sizeof(SconvMaskArgs) && offsetof(dcs_sconv_mask_view, G) == offsetof(SconvMaskArgs, G) &&
                  offsetof(dcs_sconv_mask_view, S) == offsetof(SconvMaskArgs, S) &&
                  offsetof(dcs_sconv_mask_view, src_stride) == offsetof(SconvMaskArgs, src_stride) &&
                  offsetof(dcs_sconv_mask_view, WP) == offsetof(SconvMaskArgs, WP) &&
                  offsetof(dcs_sconv_mask_view, t1) == offsetof(SconvMaskArgs, t1),
              "dcs_sconv_mask_view must mirror SconvMaskArgs");

// one mask launch, then the stream is synchronised
static int sync_after(const char* fn, int r, cudaStream_t st) {
  const cudaError_t e = cudaStreamSynchronize(st);
  if (r == DCS_OK && e != cudaSuccess) {
    set_error("%s: %s", fn, cudaGetErrorString(e));
    return DCS_ECUDA;
  }
  return r;
}

int dcs_dsd_mask_f32(dcs_ctx* ctx, int engine, const dcs_dsd_mask_view* view, void* stream) {
  DCS_REQUIRE(ctx && view && view->G && view->W1t && view->bout && view->X && view->S, "dcs_dsd_mask_f32: NULL argument");
  DCS_REQUIRE(engine == 0 || engine == 1, "dcs_dsd_mask_f32: unknown engine %d", engine);
  DsdMaskArgs a;
  memcpy(&a, view, sizeof a);
  const int64_t plane = (int64_t)a.T * a.ldf;
  DCS_REQUIRE(a.T > 0 && a.P > 0 && a.tc > a.overlap && a.overlap >= 0 && a.F >= 2 && a.ldf >= a.F && a.ldw >= a.F && a.ldg >= 50,
              "dcs_dsd_mask_f32: bad shape");
  DCS_REQUIRE(a.ndec == 3 || a.ndec == 4, "dcs_dsd_mask_f32: ndec %d not 3 or 4", a.ndec);
  DCS_REQUIRE(a.src_stride >= plane, "dcs_dsd_mask_f32: planes overlap");
  DCS_REQUIRE((uintptr_t)a.X % 8 == 0 && (uintptr_t)a.S % 8 == 0, "dcs_dsd_mask_f32: misaligned X or S");
  DCS_REQUIRE(engine == 0 || dsd_mask_tc_supported(a),
              "dcs_dsd_mask_f32: engine 1 takes at most 6 patches per frame, ldg >= 52 with ldg %% 4 == 0 and a 16-byte aligned G");
  DCS_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = (cudaStream_t)stream;
  return sync_after("dcs_dsd_mask_f32", engine == 1 ? launch_dsd_mask_tc(ctx, a, st) : launch_dsd_mask(ctx, a, st), st);
}

int dcs_dsd_convt2_f32(dcs_ctx* ctx, const dcs_dsd_convt2_view* view, const float* h_Wt2, void* stream) {
  DCS_REQUIRE(ctx && view && h_Wt2 && view->apad && view->G, "dcs_dsd_convt2_f32: NULL argument");
  DsdConvT2Args a;
  memcpy(&a, view, sizeof a);
  DCS_REQUIRE(a.npairs > 0 && a.tc >= 4 && a.tc <= 64 && a.ldg >= 50 && a.ldg % 2 == 0 && (int64_t)a.npairs * a.tc < ((int64_t)1 << 31),
              "dcs_dsd_convt2_f32: bad shape");
  DCS_REQUIRE((uintptr_t)a.apad % 16 == 0 && (uintptr_t)a.G % 8 == 0, "dcs_dsd_convt2_f32: apad must be 16-byte and G 8-byte aligned");
  DCS_REQUIRE(dsd_convT2_tc_supported(a), "dcs_dsd_convt2_f32: unsupported arguments");
  DCS_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = (cudaStream_t)stream;
  const int kh2 = a.tc / 2;
  TcWeight w;
  int r = tc_weight_create(h_Wt2, 50, kh2 * 52, 50, &w);
  if (r == DCS_OK) r = launch_dsd_convT2_tc(ctx, a, w, st);
  r = sync_after("dcs_dsd_convt2_f32", r, st);
  tc_weight_destroy(&w);
  return r;
}

int dcs_dsd_dense_f32(dcs_ctx* ctx, const dcs_dsd_dense_view* view, const float* h_W, int w_rows, int w_cols, void* stream) {
  DCS_REQUIRE(ctx && view && h_W && view->z && view->bias && view->apad, "dcs_dsd_dense_f32: NULL argument");
  DsdDenseArgs a;
  memcpy(&a, view, sizeof a);
  DCS_REQUIRE(a.P > 0 && a.tc >= 4 && a.tc <= 64 && (a.ndec == 3 || a.ndec == 4) && a.nfc > 0 && a.nfc % 32 == 0 && a.nfc <= 256,
              "dcs_dsd_dense_f32: bad shape");
  DCS_REQUIRE((uintptr_t)a.z % 4 == 0 && (uintptr_t)a.bias % 4 == 0 && (uintptr_t)a.apad % 8 == 0,
              "dcs_dsd_dense_f32: z and bias must be 4-byte and apad 8-byte aligned");
  const int N = a.ndec * (a.tc - a.tc / 2 + 1) * 52;
  DCS_REQUIRE(w_rows == a.nfc && w_cols == N, "dcs_dsd_dense_f32: weight is %dx%d, the layer wants %dx%d", w_rows, w_cols, a.nfc, N);
  DCS_REQUIRE(dsd_dense_tc_supported(a), "dcs_dsd_dense_f32: unsupported arguments");
  DCS_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = (cudaStream_t)stream;
  TcWeight w;
  int r = tc_weight_create(h_W, N, a.nfc, N, &w);
  if (r == DCS_OK) r = launch_dsd_dense_tc(ctx, a, w, st);
  r = sync_after("dcs_dsd_dense_f32", r, st);
  tc_weight_destroy(&w);
  return r;
}

int dcs_sconv_mask_f32(dcs_ctx* ctx, int engine, const dcs_sconv_mask_view* view, void* stream) {
  DCS_REQUIRE(ctx && view && view->G && view->W && view->bout && view->X && view->S, "dcs_sconv_mask_f32: NULL argument");
  DCS_REQUIRE(engine == 0 || engine == 1, "dcs_sconv_mask_f32: unknown engine %d", engine);
  SconvMaskArgs a;
  memcpy(&a, view, sizeof a);
  int KW, stride;
  switch (a.arch) {
    case DCS_ARCH_BACH10:
    case DCS_ARCH_BACH10_SCORE: KW = 30; stride = 4; break;
    case DCS_ARCH_BACH10_SCORE_1X1: KW = 5; stride = 2; break;
    case DCS_ARCH_IKALA:
    case DCS_ARCH_IKALA_NOPOOL: KW = 30; stride = 3; break;
    default: DCS_REQUIRE(false, "dcs_sconv_mask_f32: architecture %d has no strided conv1", a.arch);
  }
  const bool pooled = a.arch == DCS_ARCH_IKALA, chunked = a.arch == DCS_ARCH_BACH10_SCORE_1X1;
  const int step = a.tc - a.overlap;
  DCS_REQUIRE(a.T > 0 && a.P > 0 && step > 0 && a.overlap >= 0 && a.F >= KW && a.ldf >= a.F && a.src_stride >= (int64_t)a.T * a.ldf,
              "dcs_sconv_mask_f32: bad shape");
  DCS_REQUIRE(a.J == (a.F - KW) / stride + 1 && a.WP == (pooled ? a.J / 4 : a.J), "dcs_sconv_mask_f32: J %d / WP %d do not match F %d",
              a.J, a.WP, a.F);
  DCS_REQUIRE(pooled == (a.tie != nullptr), "dcs_sconv_mask_f32: tie bits go with the max-pool net only");
  DCS_REQUIRE(0 <= a.t0 && a.t0 < a.t1 && a.t1 <= a.T && a.p_base >= 0 && (chunked || (a.p_base == 0 && a.t0 == 0 && a.t1 == a.T)),
              "dcs_sconv_mask_f32: frames [%d, %d) from patch %d", a.t0, a.t1, a.p_base);
  // the first patch covering frame t0 must be in G
  DCS_REQUIRE(a.t0 - a.tc + 1 <= 0 || (a.t0 - a.tc + 1 + step - 1) / step >= a.p_base, "dcs_sconv_mask_f32: G starts after frame %d's patches",
              a.t0);
  DCS_REQUIRE(engine == 0 || ((uintptr_t)a.tie % 4 == 0 && sconv_mask_tc_supported(a)),
              "dcs_sconv_mask_f32: engine 1 needs a 16-byte aligned G and a 4-byte aligned tie");
  DCS_REQUIRE(engine == 1 || (a.tc + step - 1) / step <= 64, "dcs_sconv_mask_f32: engine 0 takes at most 64 patches per frame");
  DCS_REQUIRE((uintptr_t)a.W % 16 == 0 && (uintptr_t)a.X % 8 == 0 && (uintptr_t)a.S % 8 == 0, "dcs_sconv_mask_f32: misaligned W, X or S");
  DCS_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = (cudaStream_t)stream;
  return sync_after("dcs_sconv_mask_f32", engine == 1 ? launch_sconv_mask_tc(ctx, a, st) : launch_sconv_mask(ctx, a, st), st);
}

// ------------------------------------------------------------------------------------ int16 PCM conversions
// each one launch of the launcher the int16 batch entry points call, on the caller's buffers
int dcs_pcm16_decode(dcs_ctx* ctx, const dcs_resampler* r, int mode, const int16_t* d_pcm, int64_t L, int channels,
                     float* d_out, int64_t num_out, void* stream) {
  const char* fn = "dcs_pcm16_decode";
  DCS_REQUIRE(ctx && d_pcm && d_out, "%s: NULL argument", fn);
  DCS_REQUIRE(!r || resampler_ctx(r) == ctx, "%s: the resampler was made on another ctx", fn);
  DCS_REQUIRE(L >= 1, "%s: num_samples %lld must be >= 1", fn, (long long)L);
  DCS_REQUIRE((uintptr_t)d_pcm % 2 == 0 && (uintptr_t)d_out % 4 == 0, "%s: d_pcm not 2-byte or d_out not 4-byte aligned", fn);
  if (mode == DCS_PCM16_CHANNELS) {
    DCS_REQUIRE(channels >= 1 && channels <= 16, "%s: channels %d not in [1, 16]", fn, channels);
    const int64_t most = r ? resampler_length(r, L) : L;
    DCS_REQUIRE(num_out >= 1 && num_out <= most && (r || num_out == L), "%s: num_out %lld, want %s%lld", fn,
                (long long)num_out, r ? "1 .. " : "", (long long)most);
  } else {
    DCS_REQUIRE(mode >= 0 && mode <= 2, "%s: unknown mode %d", fn, mode);
    DCS_REQUIRE(!r, "%s: a resampler takes the C-channel mode only", fn);
    DCS_REQUIRE(channels >= 1 && channels <= 8, "%s: channels %d not in [1, 8]", fn, channels);
    DCS_REQUIRE(num_out == L, "%s: num_out %lld != num_samples %lld", fn, (long long)num_out, (long long)L);
  }
  DCS_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  if (r)
    rc = launch_resample_decode(r, DCS_SAMPLE_I16, d_pcm, L, channels, d_out, num_out, st);
  else if (mode == DCS_PCM16_CHANNELS)
    rc = launch_pcm_decode_channels(ctx, DCS_SAMPLE_I16, d_pcm, L, channels, d_out, st);
  else
    rc = launch_pcm_decode(ctx, d_pcm, L, channels, mode, d_out, st);
  return sync_after(fn, rc, st);
}

int dcs_pcm16_encode(dcs_ctx* ctx, const dcs_resampler* r, int mode, const float* d_stems, int64_t num_in, int nsrc,
                     int channels, int64_t stem_stride, int16_t* d_out, int64_t num_out, int64_t out_stride, void* stream) {
  const char* fn = "dcs_pcm16_encode";
  DCS_REQUIRE(ctx && d_stems && d_out, "%s: NULL argument", fn);
  DCS_REQUIRE(!r || resampler_ctx(r) == ctx, "%s: the resampler was made on another ctx", fn);
  DCS_REQUIRE(num_in >= 1 && nsrc >= 1, "%s: num_in %lld and nsrc %d must be >= 1", fn, (long long)num_in, nsrc);
  DCS_REQUIRE((uintptr_t)d_stems % 4 == 0 && (uintptr_t)d_out % 2 == 0, "%s: d_stems not 4-byte or d_out not 2-byte aligned",
              fn);
  if (mode == DCS_PCM16_CHANNELS) {
    DCS_REQUIRE(channels >= 1 && channels <= 16, "%s: channels %d not in [1, 16]", fn, channels);
    DCS_REQUIRE(r ? stem_stride == num_in : stem_stride >= num_in, "%s: stem_stride %lld, num_in %lld", fn,
                (long long)stem_stride, (long long)num_in);
    const int64_t most = r ? resampler_length(r, num_in) : num_in;
    DCS_REQUIRE(num_out >= 1 && num_out <= most && (r || num_out == num_in), "%s: num_out %lld, want %s%lld", fn,
                (long long)num_out, r ? "1 .. " : "", (long long)most);
    DCS_REQUIRE(out_stride == (int64_t)channels * num_out, "%s: out_stride %lld != channels * num_out", fn, (long long)out_stride);
  } else {
    DCS_REQUIRE(mode == DCS_PCM16_MONO, "%s: unknown mode %d", fn, mode);
    DCS_REQUIRE(!r, "%s: a resampler takes the C-channel mode only", fn);
    DCS_REQUIRE(channels == 1, "%s: the mono mode has one channel, not %d", fn, channels);
    DCS_REQUIRE(num_out == num_in && stem_stride >= num_in && out_stride >= num_out,
                "%s: num_out %lld, stem_stride %lld, out_stride %lld for num_in %lld", fn, (long long)num_out,
                (long long)stem_stride, (long long)out_stride, (long long)num_in);
  }
  DCS_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  if (r)
    rc = launch_resample_encode(r, DCS_SAMPLE_I16, d_stems, num_in, nsrc, channels, d_out, num_out, st);
  else if (mode == DCS_PCM16_CHANNELS)
    rc = launch_pcm_encode_channels(ctx, DCS_SAMPLE_I16, d_stems, num_in, nsrc, channels, stem_stride, d_out, st);
  else
    rc = launch_pcm_encode(ctx, d_stems, num_in, nsrc, stem_stride, d_out, out_stride, st);
  return sync_after(fn, rc, st);
}

// the C-channel conversions of every sample format, each one launch of the launcher dcs_separate_batch_channels_host
// calls (two for a decode whose channels take groups), on the caller's buffers
int dcs_channels_decode(dcs_ctx* ctx, const dcs_resampler* r, int format, const void* d_in, int64_t L, int channels,
                        float* d_out, int64_t num_out, void* stream) {
  const char* fn = "dcs_channels_decode";
  DCS_REQUIRE(ctx && d_in && d_out, "%s: NULL argument", fn);
  DCS_REQUIRE(!r || resampler_ctx(r) == ctx, "%s: the resampler was made on another ctx", fn);
  const int b = sample_bytes(format);
  DCS_REQUIRE(b > 0, "%s: unknown sample format %d", fn, format);
  DCS_REQUIRE(L >= 1, "%s: num_samples %lld must be >= 1", fn, (long long)L);
  DCS_REQUIRE((uintptr_t)d_in % sample_align(format) == 0 && (uintptr_t)d_out % 4 == 0,
              "%s: d_in not %d-byte or d_out not 4-byte aligned", fn, sample_align(format));
  DCS_REQUIRE(channels >= 1 && channels <= 16, "%s: channels %d not in [1, 16]", fn, channels);
  const int64_t most = r ? resampler_length(r, L) : L;
  DCS_REQUIRE(num_out >= 1 && num_out <= most && (r || num_out == L), "%s: num_out %lld, want %s%lld", fn, (long long)num_out,
              r ? "1 .. " : "", (long long)most);
  DCS_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = (cudaStream_t)stream;
  return sync_after(fn, r ? launch_resample_decode(r, format, d_in, L, channels, d_out, num_out, st)
                          : launch_pcm_decode_channels(ctx, format, d_in, L, channels, d_out, st), st);
}

int dcs_channels_encode(dcs_ctx* ctx, const dcs_resampler* r, int format, const float* d_stems, int64_t num_in, int nsrc,
                        int channels, int64_t stem_stride, void* d_out, int64_t num_out, int64_t out_stride, void* stream) {
  const char* fn = "dcs_channels_encode";
  DCS_REQUIRE(ctx && d_stems && d_out, "%s: NULL argument", fn);
  DCS_REQUIRE(!r || resampler_ctx(r) == ctx, "%s: the resampler was made on another ctx", fn);
  const int b = sample_bytes(format);
  DCS_REQUIRE(b > 0, "%s: unknown sample format %d", fn, format);
  DCS_REQUIRE(num_in >= 1 && nsrc >= 1, "%s: num_in %lld and nsrc %d must be >= 1", fn, (long long)num_in, nsrc);
  DCS_REQUIRE((uintptr_t)d_stems % 4 == 0 && (uintptr_t)d_out % sample_align(format) == 0,
              "%s: d_stems not 4-byte or d_out not %d-byte aligned", fn, sample_align(format));
  DCS_REQUIRE(channels >= 1 && channels <= 16, "%s: channels %d not in [1, 16]", fn, channels);
  DCS_REQUIRE(r ? stem_stride == num_in : stem_stride >= num_in, "%s: stem_stride %lld, num_in %lld", fn,
              (long long)stem_stride, (long long)num_in);
  const int64_t most = r ? resampler_length(r, num_in) : num_in;
  DCS_REQUIRE(num_out >= 1 && num_out <= most && (r || num_out == num_in), "%s: num_out %lld, want %s%lld", fn,
              (long long)num_out, r ? "1 .. " : "", (long long)most);
  DCS_REQUIRE(out_stride == (int64_t)channels * num_out, "%s: out_stride %lld != channels * num_out", fn, (long long)out_stride);
  DCS_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = (cudaStream_t)stream;
  return sync_after(fn, r ? launch_resample_encode(r, format, d_stems, num_in, nsrc, channels, d_out, num_out, st)
                          : launch_pcm_encode_channels(ctx, format, d_stems, num_in, nsrc, channels, stem_stride, d_out, st),
                    st);
}

int dcs_downmix_f32(dcs_ctx* ctx, const float* d_audio, int nx, int64_t audio_stride, int64_t L, float* d_mono, void* stream) {
  const char* fn = "dcs_downmix_f32";
  DCS_REQUIRE(ctx && d_audio && d_mono, "%s: NULL argument", fn);
  DCS_REQUIRE(nx >= 1 && nx <= 16, "%s: nx %d not in [1, 16]", fn, nx);
  DCS_REQUIRE(L >= 1 && audio_stride >= L, "%s: num_samples %lld, audio_stride %lld", fn, (long long)L, (long long)audio_stride);
  DCS_REQUIRE((uintptr_t)d_audio % 4 == 0 && (uintptr_t)d_mono % 4 == 0, "%s: planes not 4-byte aligned", fn);
  DCS_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = (cudaStream_t)stream;
  return sync_after(fn, launch_downmix(ctx, d_audio, nx, audio_stride, L, d_mono, st), st);
}

int dcs_separate_audio_stereo(dcs_ctx* ctx, dcs_model* m, dcs_stft* p, const float* d_audio, int64_t audio_stride, int64_t L,
                              float scale_factor, int overlap, int patcher, float* d_stems, int64_t stem_stride, void* stream) {
  DCS_TRY(check_clip("dcs_separate_audio_stereo", ctx, m, p, DCS_ARCH_DSD_ILD, d_audio, d_stems, L, audio_stride, stem_stride,
                     overlap, patcher));
  DCS_CUDA(cudaSetDevice(ctx->device));
  return separate_clip(ctx, m, p, d_audio, audio_stride, L, nullptr, nullptr, scale_factor, overlap, patcher, d_stems,
                       stem_stride, (cudaStream_t)stream);
}

int dcs_xcorr_lags(dcs_ctx* ctx, const float* const* h_a, const float* const* h_b, int npairs, int64_t num_samples, int flen,
                   double* h_out, void* stream) {
  DCS_REQUIRE(ctx && h_a && h_b && h_out, "dcs_xcorr_lags: NULL argument");
  DCS_CUDA(cudaSetDevice(ctx->device));
  return launch_xcorr_lags(ctx, h_a, h_b, npairs, num_samples, flen, h_out, (cudaStream_t)stream);
}

int dcs_separate_audio(dcs_ctx* ctx, dcs_model* m, dcs_stft* p, const float* d_audio, int64_t L, float scale_factor,
                       int overlap, int patcher, float* d_stems, int64_t stem_stride, void* stream) {
  DCS_TRY(check_clip("dcs_separate_audio", ctx, m, p, -1, d_audio, d_stems, L, L, stem_stride, overlap, patcher));
  DCS_CUDA(cudaSetDevice(ctx->device));
  return separate_clip(ctx, m, p, d_audio, L, L, nullptr, nullptr, scale_factor, overlap, patcher, d_stems,
                       stem_stride, (cudaStream_t)stream);
}

int dcs_separate_host(dcs_ctx* ctx, dcs_model* m, dcs_stft* p, const float* h_audio, int64_t L, float scale_factor,
                      int overlap, int patcher, float* h_stems, int64_t stem_stride, void* stream) {
  DCS_TRY(check_clip("dcs_separate_host", ctx, m, p, -1, h_audio, h_stems, L, L, stem_stride, overlap, patcher));
  cudaStream_t st = (cudaStream_t)stream;
  DCS_CUDA(cudaSetDevice(ctx->device));
  DCS_TRY(size_workspace(ctx, m, p, L, true, st));
  DCS_CUDA(cudaMemcpyAsync(ctx->audio.p, h_audio, (size_t)L * sizeof(float), cudaMemcpyHostToDevice, st));
  DCS_TRY(separate_clip(ctx, m, p, ctx->audio.as<float>(), L, L, nullptr, nullptr, scale_factor, overlap, patcher,
                        ctx->stems.as<float>(), L, st));
  DCS_CUDA(cudaMemcpy2DAsync(h_stems, (size_t)stem_stride * sizeof(float), ctx->stems.p, (size_t)L * sizeof(float),
                             (size_t)L * sizeof(float), m->nsrc, cudaMemcpyDeviceToHost, st));
  DCS_CUDA(cudaStreamSynchronize(st));
  return DCS_OK;
}

// one clip is a batch of one: the same checks, staging and kernels as every clip of dcs_separate_batch_pcm16_host
int dcs_separate_pcm16_host(dcs_ctx* ctx, dcs_model* m, dcs_stft* p, const int16_t* h_pcm, int64_t L, int channels,
                            int downmix, float scale_factor, int overlap, int patcher, int16_t* h_out,
                            int64_t out_stride, void* stream) {
  return dcs_separate_batch_pcm16_host(ctx, m, p, 1, &h_pcm, &L, channels, downmix, scale_factor, overlap, patcher, &h_out,
                                       &out_stride, stream);
}

// A clip of the pipeline is a PipeClip: a whole clip (seg NULL), or one segment of a long recording (nx > 0): its in
// range staged, its model range separated, its kept core encoded and copied into the recording's stems at out_start.
struct PipeClip {
  const void* in;            // staged samples: the clip, or the segment's in range
  int64_t n_in;              // their count
  void* out;                 // the stems' first kept sample (source 0)
  int64_t out_stride;        // samples (of nx channels) from one source's stems to the next
  const dcs_segment* seg;    // the segment, or NULL
  int64_t rec_len;           // the recording's samples (segments only)
};

// Multi-clip scheduler: the clips of a batch run through ONE context as a three-stage pipeline -- H2D of clip i+1
// (copy stream) | kernels of clip i (the caller's stream) | D2H of clip i-1 (second copy stream) -- with double-buffered
// int16 staging on the device and events for the hand-overs.  The reference's only multi-clip driver starts a Python
// process per file (examples/dsd100/separate_multiple.ipynb cell 3); per clip this is the wav contract of train_auto
// (separate_dsd.py:275-287,307-309), exactly dcs_separate_pcm16_host.  Host buffers should be pinned.
// the pipelined loop of the int16 and C-channel batch entry points; on any failure the caller drains the copy streams
// before it returns, because the copies in flight read and write the user's host buffers.  nx == 0: mono stems (int16
// in and out), the clip decoded into one plane (channel 0 or the downmix of `downmix`), int16 [nsrc][L] out.  nx > 0
// (C-channel stems, nx == channels): the clip, samples of in_fmt, is decoded into nx + 1 planes (the downmix, then the
// channels), separated as dcs_separate_audio_channels_wiener with `iterations` and `radius`, and the stems encoded in
// out_fmt as interleaved [L][nx] per source.  to / from (nx > 0, both or neither): the clip is at another rate; the
// decode resamples it to L' = resampler_length(to, L) samples, the clip is separated at L', and the encode resamples its
// stems back to L
static int batch_pipeline(dcs_ctx* ctx, dcs_model* m, dcs_stft* p, const dcs_resampler* to, const dcs_resampler* from,
                          int in_fmt, int out_fmt, int nclips, const PipeClip* clips, int channels, int downmix, int nx,
                          int iterations, int radius, float scale_factor, int overlap, int patcher, cudaStream_t st) {
  const size_t bi = (size_t)sample_bytes(in_fmt), bo = (size_t)sample_bytes(out_fmt);
  const size_t w = (size_t)(nx > 0 ? nx : 1) * bo;   // bytes per sample of a stem
  int pitch_attr = 0;
  DCS_CUDA(cudaDeviceGetAttribute(&pitch_attr, cudaDevAttrMaxPitch, ctx->device));
  const size_t max_pitch = (size_t)pitch_attr;
  float *audio = ctx->audio.as<float>(), *stems = ctx->stems.as<float>();
  // the copy streams start after whatever the caller queued on `st` (and after the memsets of fresh buffers)
  DCS_CUDA(cudaEventRecord(ctx->ev_dec[0], st));
  DCS_CUDA(cudaStreamWaitEvent(ctx->s_h2d, ctx->ev_dec[0], 0));
  DCS_CUDA(cudaStreamWaitEvent(ctx->s_d2h, ctx->ev_dec[0], 0));
  for (int i = 0; i < nclips; ++i) {
    const int b = i & 1;
    const PipeClip& cl = clips[i];
    const dcs_segment* sg = cl.seg;
    const int64_t L = cl.n_in;
    // H2D of clip i: its staging buffer is free once the decode of clip i-2 has read it
    if (i >= 2) DCS_CUDA(cudaStreamWaitEvent(ctx->s_h2d, ctx->ev_dec[b], 0));
    DCS_CUDA(cudaMemcpyAsync(ctx->pcm_in[b].p, cl.in, (size_t)L * channels * bi, cudaMemcpyHostToDevice, ctx->s_h2d));
    DCS_CUDA(cudaEventRecord(ctx->ev_in[b], ctx->s_h2d));
    // kernels of clip i
    DCS_CUDA(cudaStreamWaitEvent(st, ctx->ev_in[b], 0));
    // the clip's samples at the networks' rate (a segment: its model range) and the samples kept
    const int64_t Lm = sg ? sg->model_stop - sg->model_start : to ? resampler_length(to, L) : L;
    const int64_t K = sg ? sg->out_stop - sg->out_start : L;
    if (to) {
      if (sg)
        DCS_TRY(launch_resample_decode_range(to, in_fmt, ctx->pcm_in[b].p, cl.rec_len, sg->in_start, L, nx, audio,
                                             sg->model_start, Lm, st));
      else
        DCS_TRY(launch_resample_decode(to, in_fmt, ctx->pcm_in[b].p, L, nx, audio, Lm, st));
      DCS_CUDA(cudaEventRecord(ctx->ev_dec[b], st));
      ProfScope ps(ctx, "pcm16_separate", st);
      DCS_TRY(downmix_clip(ctx, m, p, audio, audio + Lm, nx, Lm, Lm, iterations, radius, scale_factor, overlap, patcher, stems,
                           Lm, st));
    } else if (nx > 0) {
      ProfScope ps(ctx, "pcm16_decode_separate", st);   // the clip's kernels up to its stem planes
      DCS_TRY(launch_pcm_decode_channels(ctx, in_fmt, ctx->pcm_in[b].p, L, nx, audio, st));
      DCS_CUDA(cudaEventRecord(ctx->ev_dec[b], st));
      DCS_TRY(downmix_clip(ctx, m, p, audio, audio + L, nx, L, L, iterations, radius, scale_factor, overlap, patcher, stems, L,
                           st));
    } else {
      DCS_TRY(launch_pcm_decode(ctx, ctx->pcm_in[b].as<int16_t>(), L, channels, downmix, audio, st));
      DCS_CUDA(cudaEventRecord(ctx->ev_dec[b], st));
      DCS_TRY(separate_clip(ctx, m, p, audio, L, L, nullptr, nullptr, scale_factor, overlap, patcher, stems, L,
                            st));
    }
    if (i >= 2) DCS_CUDA(cudaStreamWaitEvent(st, ctx->ev_out[b], 0));     // D2H of clip i-2 has drained the output staging
    if (from) {
      if (sg)
        DCS_TRY(launch_resample_encode_range(from, out_fmt, stems, resampler_length(to, cl.rec_len), sg->model_start, Lm,
                                             m->nsrc, nx, ctx->pcm_out[b].p, sg->out_start, K, st));
      else
        DCS_TRY(launch_resample_encode(from, out_fmt, stems, Lm, m->nsrc, nx, ctx->pcm_out[b].p, L, st));
    } else if (nx > 0) {
      ProfScope ps(ctx, "pcm16_encode", st);   // a segment: its kept core of the stem planes, Lm apart
      DCS_TRY(launch_pcm_encode_channels(ctx, out_fmt, stems + (sg ? sg->out_start - sg->model_start : 0), K, m->nsrc, nx, Lm,
                                         ctx->pcm_out[b].p, st));
    } else
      DCS_TRY(launch_pcm_encode(ctx, stems, L, m->nsrc, L, ctx->pcm_out[b].as<int16_t>(), L, st));
    DCS_CUDA(cudaEventRecord(ctx->ev_enc[b], st));
    // D2H of clip i
    DCS_CUDA(cudaStreamWaitEvent(ctx->s_d2h, ctx->ev_enc[b], 0));
    // one 2-D copy, rows = sources; a pitch over the device's limit (cudaDevAttrMaxPitch, 2^31 - 1 bytes: one source of a
    // long recording's stems can span more) takes one copy per source instead
    if (w * cl.out_stride <= max_pitch) {
      DCS_CUDA(cudaMemcpy2DAsync(cl.out, w * cl.out_stride, ctx->pcm_out[b].p, w * K, w * K, m->nsrc, cudaMemcpyDeviceToHost,
                                 ctx->s_d2h));
    } else {
      for (int s = 0; s < m->nsrc; ++s)
        DCS_CUDA(cudaMemcpyAsync((char*)cl.out + s * w * cl.out_stride, ctx->pcm_out[b].as<char>() + s * w * K, w * K,
                                 cudaMemcpyDeviceToHost, ctx->s_d2h));
    }
    DCS_CUDA(cudaEventRecord(ctx->ev_out[b], ctx->s_d2h));
  }
  return DCS_OK;
}

// the resources, sizing and drain around batch_pipeline: streams and events made once per ctx, every buffer sized before
// the pipeline starts (a grow-only buffer re-allocated mid-batch would synchronise the stream) from the longest staged
// input (Smax samples), the longest clip at the networks' rate (Swork) and the most samples kept of a clip (Kmax)
static int run_pipeline(dcs_ctx* ctx, dcs_model* m, dcs_stft* p, const dcs_resampler* to, const dcs_resampler* from, int in_fmt,
                        int out_fmt, const std::vector<PipeClip>& clips, int channels, int downmix, int nx, int iterations,
                        int radius, float scale_factor, int overlap, int patcher, int64_t Smax, int64_t Swork, int64_t Kmax,
                        cudaStream_t st) {
  const int nclips = (int)clips.size();
  DCS_CUDA(cudaSetDevice(ctx->device));
  // each resource on its own: a call that failed half-way through this block must not leave later calls with null handles
  if (!ctx->s_h2d) DCS_CUDA(cudaStreamCreateWithFlags(&ctx->s_h2d, cudaStreamNonBlocking));
  if (!ctx->s_d2h) DCS_CUDA(cudaStreamCreateWithFlags(&ctx->s_d2h, cudaStreamNonBlocking));
  for (int i = 0; i < 2; ++i) {
    if (!ctx->ev_in[i]) DCS_CUDA(cudaEventCreateWithFlags(&ctx->ev_in[i], cudaEventDisableTiming));
    if (!ctx->ev_dec[i]) DCS_CUDA(cudaEventCreateWithFlags(&ctx->ev_dec[i], cudaEventDisableTiming));
    if (!ctx->ev_enc[i]) DCS_CUDA(cudaEventCreateWithFlags(&ctx->ev_enc[i], cudaEventDisableTiming));
    if (!ctx->ev_out[i]) DCS_CUDA(cudaEventCreateWithFlags(&ctx->ev_out[i], cudaEventDisableTiming));
  }
  for (int b = 0; b < std::min(nclips, 2); ++b) {
    DCS_TRY(ctx->pcm_in[b].ensure((size_t)Smax * channels * sample_bytes(in_fmt), st));
    DCS_TRY(ctx->pcm_out[b].ensure((size_t)m->nsrc * (nx > 0 ? nx : 1) * Kmax * sample_bytes(out_fmt), st));
  }
  if (nx > 0)
    DCS_TRY(size_downmix_workspace(ctx, m, p, Swork, iterations > 0 ? nx : 0, radius, nx, st));
  else
    DCS_TRY(size_workspace(ctx, m, p, Smax, true, st));
  const int rc = batch_pipeline(ctx, m, p, to, from, in_fmt, out_fmt, nclips, clips.data(), channels, downmix, nx, iterations,
                                radius, scale_factor, overlap, patcher, st);
  // drain everything, success or not, before the host buffers go back to the caller
  const cudaError_t e0 = cudaStreamSynchronize(ctx->s_h2d), e1 = cudaStreamSynchronize(ctx->s_d2h), e2 = cudaStreamSynchronize(st);
  if (rc != DCS_OK) return rc;
  DCS_CUDA(e0);
  DCS_CUDA(e1);
  DCS_CUDA(e2);
  return DCS_OK;
}

// the checks, resources and drain of every batch entry point around batch_pipeline (formats, nx, iterations, radius,
// to, from as there; the entry point has checked the formats and the resampler pair).  check_model(Lmax): the entry
// point's own checks of the model, plan and options, run on the longest clip (its length at the networks' rate) after
// the per-clip checks and before anything is queued
extern "C++" {
template <class CheckModel>
static int batch_host(const char* fn, dcs_ctx* ctx, dcs_model* m, dcs_stft* p, const dcs_resampler* to,
                      const dcs_resampler* from, int in_fmt, int out_fmt, int nclips, const void* const* h_in,
                      const int64_t* num_samples, int channels, int downmix, int nx, int iterations, int radius,
                      float scale_factor, int overlap, int patcher, void* const* h_out, const int64_t* out_strides,
                      cudaStream_t st, CheckModel check_model) {
  DCS_REQUIRE(ctx && m && p && h_in && num_samples && h_out && out_strides && nclips >= 0, "%s: bad argument", fn);
  DCS_REQUIRE(nx > 0 || (channels >= 1 && channels <= 8 && downmix >= 0 && downmix <= 2), "bad channels/downmix");
  if (nclips == 0) return DCS_OK;
  int64_t Lmax = 0;
  for (int i = 0; i < nclips; ++i) {
    DCS_REQUIRE(h_in[i] && h_out[i] && num_samples[i] > 0 && out_strides[i] >= num_samples[i], "clip %d: bad buffer / length", i);
    Lmax = std::max(Lmax, num_samples[i]);
  }
  const int64_t Lwork = to ? resampler_length(to, Lmax) : Lmax;   // the longest clip at the networks' rate
  DCS_TRY(check_model(Lwork));
  std::vector<PipeClip> clips((size_t)nclips);
  for (int i = 0; i < nclips; ++i) clips[(size_t)i] = PipeClip{h_in[i], num_samples[i], h_out[i], out_strides[i], nullptr, 0};
  return run_pipeline(ctx, m, p, to, from, in_fmt, out_fmt, clips, channels, downmix, nx, iterations, radius, scale_factor,
                      overlap, patcher, Lmax, Lwork, Lmax, st);
}
}  // extern "C++"

int dcs_separate_batch_pcm16_host(dcs_ctx* ctx, dcs_model* m, dcs_stft* p, int nclips, const int16_t* const* h_pcm,
                                  const int64_t* num_samples, int channels, int downmix, float scale_factor, int overlap,
                                  int patcher, int16_t* const* h_out, const int64_t* out_strides, void* stream) {
  const char* fn = "dcs_separate_batch_pcm16_host";
  return batch_host(fn, ctx, m, p, nullptr, nullptr, DCS_SAMPLE_I16, DCS_SAMPLE_I16, nclips, (const void* const*)h_pcm,
                    num_samples, channels, downmix, 0, 0, 0, scale_factor, overlap, patcher, (void* const*)h_out, out_strides, (cudaStream_t)stream, [&](int64_t Lmax) {
                      return check_clip(fn, ctx, m, p, -1, h_pcm, h_out, Lmax, Lmax, Lmax, overlap, patcher);
                    });
}

// ------------------------------------------------------------------------------------ keep-channels (DSD100 net)
// the C = 2 batch with the filter settings of the ctx
int dcs_separate_batch_pcm16_keep_channels_host(dcs_ctx* ctx, dcs_model* m, dcs_stft* p, int nclips,
                                                const int16_t* const* h_pcm, const int64_t* num_samples, float scale_factor,
                                                int overlap, int patcher, int16_t* const* h_out, const int64_t* out_strides,
                                                void* stream) {
  const char* fn = "dcs_separate_batch_pcm16_keep_channels_host";
  return batch_host(fn, ctx, m, p, nullptr, nullptr, DCS_SAMPLE_I16, DCS_SAMPLE_I16, nclips, (const void* const*)h_pcm,
                    num_samples, 2, 1, 2, ctx ? ctx->wiener_iters : 0, ctx ? ctx->wiener_radius : 0, scale_factor, overlap,
                    patcher, (void* const*)h_out, out_strides, (cudaStream_t)stream,
                    [&](int64_t Lmax) {
                      DCS_TRY(check_clip(fn, ctx, m, p, DCS_ARCH_DSD, h_pcm, h_out, Lmax, Lmax, Lmax, overlap, patcher));
                      return check_keep_tap(fn, ctx);
                    });
}

int dcs_separate_audio_keep_channels(dcs_ctx* ctx, dcs_model* m, dcs_stft* p, const float* d_audio, int64_t audio_stride,
                                     int64_t L, float scale_factor, int overlap, int patcher, float* d_stems,
                                     int64_t stem_stride, void* stream) {
  const char* fn = "dcs_separate_audio_keep_channels";
  DCS_TRY(check_clip(fn, ctx, m, p, DCS_ARCH_DSD, d_audio, d_stems, L, audio_stride, stem_stride, overlap, patcher));
  DCS_TRY(check_keep_tap(fn, ctx));
  DCS_CUDA(cudaSetDevice(ctx->device));
  return downmix_clip(ctx, m, p, nullptr, d_audio, 2, audio_stride, L, ctx->wiener_iters, ctx->wiener_radius, scale_factor,
                      overlap, patcher, d_stems, stem_stride, (cudaStream_t)stream);
}

// ------------------------------------------------------------------------------------ masks output
// the checks of a masks entry point beyond check_clip's: the caller's planes hold T x ldf floats each
static int check_masks(const char* fn, const dcs_stft* p, int64_t L, const float* d_masks, int64_t m_stride) {
  const int64_t T = dcs_num_frames(L, p->hop), ldf = dcs_padded_bins(p->N);
  DCS_REQUIRE(m_stride >= T * ldf, "%s: m_stride %lld < num_frames * ldf %lld", fn, (long long)m_stride, (long long)(T * ldf));
  DCS_REQUIRE((uintptr_t)d_masks % sizeof(float) == 0, "%s: d_masks not 4-byte aligned", fn);
  return DCS_OK;
}

int dcs_separate_masks(dcs_ctx* ctx, dcs_model* m, dcs_stft* p, const float* d_audio, int64_t audio_stride, int64_t L,
                       float scale_factor, int overlap, int patcher, float* d_masks, int64_t m_stride, void* stream) {
  const int arch = m && m->arch == DCS_ARCH_DSD_ILD ? DCS_ARCH_DSD_ILD : -1;   // the single-channel nets or the stereo net
  DCS_TRY(check_clip("dcs_separate_masks", ctx, m, p, arch, d_audio, d_masks, L, audio_stride, L, overlap, patcher));
  DCS_TRY(check_masks("dcs_separate_masks", p, L, d_masks, m_stride));
  DCS_CUDA(cudaSetDevice(ctx->device));
  return separate_clip(ctx, m, p, d_audio, audio_stride, L, nullptr, nullptr, scale_factor, overlap, patcher, d_masks,
                       m_stride, (cudaStream_t)stream, true);
}

int dcs_separate_masks_score(dcs_ctx* ctx, dcs_model* m, dcs_stft* p, const float* d_audio, int64_t L, const float* d_filters,
                             float scale_factor, int overlap, int patcher, float* d_masks, int64_t m_stride, void* stream) {
  DCS_TRY(check_clip("dcs_separate_masks_score", ctx, m, p, DCS_ARCH_BACH10_SCORE, d_audio, d_masks, L, L, L, overlap, patcher));
  DCS_REQUIRE(d_filters, "dcs_separate_masks_score: NULL filters");
  DCS_TRY(check_masks("dcs_separate_masks_score", p, L, d_masks, m_stride));
  DCS_CUDA(cudaSetDevice(ctx->device));
  return separate_clip(ctx, m, p, d_audio, L, L, d_filters, nullptr, scale_factor, overlap, patcher, d_masks, m_stride,
                       (cudaStream_t)stream, true);
}

int dcs_separate_masks_notes(dcs_ctx* ctx, dcs_model* m, dcs_stft* p, const float* d_audio, int64_t L, const double* h_melody,
                             int nnotes, int ncols, int64_t frame0, float scale_factor, int overlap, int patcher, float* d_masks,
                             int64_t m_stride, void* stream) {
  DCS_TRY(check_clip("dcs_separate_masks_notes", ctx, m, p, DCS_ARCH_BACH10_SCORE, d_audio, d_masks, L, L, L, overlap, patcher));
  DCS_TRY(check_masks("dcs_separate_masks_notes", p, L, d_masks, m_stride));
  std::vector<int32_t> tab;
  NoteTable nt;
  DCS_TRY(notes_compact("dcs_separate_masks_notes", h_melody, score_planes(m), nnotes, ncols, frame0,
                        dcs_num_frames(L, p->hop), m->F, &tab, &nt));
  cudaStream_t st = (cudaStream_t)stream;
  DCS_CUDA(cudaSetDevice(ctx->device));
  DCS_TRY(notes_stage(ctx, tab, &nt, st));
  return separate_clip(ctx, m, p, d_audio, L, L, nullptr, &nt, scale_factor, overlap, patcher, d_masks, m_stride, st,
                       true);
}

// ------------------------------------------------------------------------------------ masks applied to C channels
// what dcs_istft_masked refuses; fn names the entry point
static int check_istft_masked(const char* fn, const dcs_stft* p, const void* d_X, int nx, int64_t x_plane, const void* d_M,
                              int nsrc, int64_t m_stride, int64_t T, int64_t ldf, const void* d_out, int64_t Lout,
                              int64_t out_stride) {
  DCS_REQUIRE(p && d_X && d_M && d_out, "%s: NULL argument", fn);
  DCS_REQUIRE(T > 0, "%s: num_frames %lld must be > 0", fn, (long long)T);
  DCS_REQUIRE(nx >= 1 && nx <= 16, "%s: nx %d not in [1, 16]", fn, nx);
  DCS_REQUIRE(nsrc >= 1, "%s: nsrc %d must be >= 1", fn, nsrc);
  DCS_REQUIRE(ldf >= p->N / 2 + 1, "%s: ldf %lld < F %d", fn, (long long)ldf, p->N / 2 + 1);
  DCS_REQUIRE(x_plane >= 0 && m_stride >= 0 && out_stride >= 0, "%s: negative stride", fn);
  DCS_REQUIRE(nx <= 1 || x_plane >= T * ldf, "%s: x_plane %lld < num_frames * ldf %lld", fn, (long long)x_plane, (long long)(T * ldf));
  DCS_REQUIRE(nsrc <= 1 || m_stride >= T * ldf, "%s: m_stride %lld < num_frames * ldf %lld", fn, (long long)m_stride,
              (long long)(T * ldf));
  DCS_REQUIRE(nsrc * nx <= 1 || out_stride >= Lout, "%s: out_stride %lld < num_out %lld", fn, (long long)out_stride, (long long)Lout);
  DCS_REQUIRE(Lout <= (T - 1) * p->hop + p->N - p->N / 2, "%s: num_out %lld exceeds the istft length", fn, (long long)Lout);
  DCS_REQUIRE((uintptr_t)d_X % 8 == 0, "%s: d_X not 8-byte aligned", fn);
  DCS_REQUIRE((uintptr_t)d_M % sizeof(float) == 0, "%s: d_M not 4-byte aligned", fn);
  return DCS_OK;
}

int dcs_istft_masked(dcs_stft* p, const dcs_complex* d_X, int nx, int64_t x_plane, const float* d_M, int nsrc, int64_t m_stride,
                     int64_t T, int64_t ldf, float* d_out, int64_t Lout, int64_t out_stride, void* stream) {
  DCS_TRY(check_istft_masked("dcs_istft_masked", p, d_X, nx, x_plane, d_M, nsrc, m_stride, T, ldf, d_out, Lout, out_stride));
  DCS_CUDA(cudaSetDevice(p->ctx->device));
  return launch_istft(p, (const float2*)d_X, nullptr, nullptr, 1.f, nsrc, T, ldf, x_plane, d_out, Lout, out_stride,
                      (cudaStream_t)stream, d_M, m_stride, nx);
}

// what dcs_apply_masks checks beyond the plan: nx channels of L samples, nsrc mask planes of the clip's T x ldf
static int check_apply_masks(const char* fn, const dcs_ctx* ctx, const dcs_stft* p, const float* d_audio, int nx,
                             int64_t audio_stride, int64_t L, const float* d_masks, int nsrc, int64_t m_stride,
                             const float* d_stems, int64_t stem_stride) {
  DCS_REQUIRE(ctx && p && d_audio && d_masks && d_stems, "%s: NULL argument", fn);
  DCS_REQUIRE(nx >= 1 && nx <= 16, "%s: nx %d not in [1, 16]", fn, nx);
  DCS_REQUIRE(nsrc >= 1, "%s: nsrc %d must be >= 1", fn, nsrc);
  DCS_REQUIRE(L > 0 && audio_stride >= L && stem_stride >= L, "%s: bad length / stride", fn);
  return check_masks(fn, p, L, d_masks, m_stride);
}

int dcs_apply_masks(dcs_ctx* ctx, dcs_stft* p, const float* d_audio, int nx, int64_t audio_stride, int64_t L,
                    const float* d_masks, int nsrc, int64_t m_stride, float* d_stems, int64_t stem_stride, void* stream) {
  DCS_TRY(check_apply_masks("dcs_apply_masks", ctx, p, d_audio, nx, audio_stride, L, d_masks, nsrc, m_stride, d_stems, stem_stride));
  DCS_CUDA(cudaSetDevice(ctx->device));
  return apply_masks(ctx, p, d_audio, nx, audio_stride, L, d_masks, nsrc, m_stride, d_stems, stem_stride, (cudaStream_t)stream);
}

// the checks of dcs_separate_audio_channels(_wiener): with iterations > 0 also those of the filter on the clip's spectra
static int check_channels(const char* fn, const dcs_ctx* ctx, const dcs_model* m, const dcs_stft* p, const void* d_audio, int nx,
                          int64_t audio_stride, int64_t L, int overlap, int patcher, const void* d_stems, int64_t stem_stride,
                          int iterations, int radius) {
  DCS_REQUIRE(!m || (m->arch != DCS_ARCH_DSD_ILD && !score_arch(m->arch)),
              "%s does not serve architecture %d: use dcs_separate_masks* + dcs_apply_masks", fn, m->arch);
  DCS_TRY(check_clip(fn, ctx, m, p, -1, d_audio, d_stems, L, audio_stride, stem_stride, overlap, patcher));
  DCS_REQUIRE(nx >= 1 && nx <= 16, "%s: nx %d not in [1, 16]", fn, nx);
  DCS_REQUIRE(iterations >= 0, "%s: iterations %d must be >= 0", fn, iterations);
  DCS_REQUIRE(radius >= 0, "%s: radius %d must be >= 0", fn, radius);
  if (iterations == 0) {
    DCS_REQUIRE(!ctx->tap, "%s: a spectrum tap is set (dcs_set_spectrum_tap), and this path forms no masked spectra to copy", fn);
    return DCS_OK;
  }
  DCS_REQUIRE(nx >= 2 && nx <= 8, "%s: the Wiener post-filter needs nx in [2, 8], got %d", fn, nx);
  const int64_t T = dcs_num_frames(L, p->hop), ldf = dcs_padded_bins(p->N);
  return wiener_check(fn, m->nsrc, T, ldf, m->F, T * ldf, T * ldf, iterations, radius);
}

int dcs_separate_audio_channels(dcs_ctx* ctx, dcs_model* m, dcs_stft* p, const float* d_audio, int nx, int64_t audio_stride,
                                int64_t L, float scale_factor, int overlap, int patcher, float* d_stems, int64_t stem_stride,
                                void* stream) {
  DCS_TRY(check_channels("dcs_separate_audio_channels", ctx, m, p, d_audio, nx, audio_stride, L, overlap, patcher, d_stems,
                         stem_stride, 0, 0));
  DCS_CUDA(cudaSetDevice(ctx->device));
  return downmix_clip(ctx, m, p, nullptr, d_audio, nx, audio_stride, L, 0, 0, scale_factor, overlap, patcher, d_stems,
                      stem_stride, (cudaStream_t)stream);
}

int dcs_separate_audio_channels_wiener(dcs_ctx* ctx, dcs_model* m, dcs_stft* p, const float* d_audio, int nx,
                                       int64_t audio_stride, int64_t L, float scale_factor, int overlap, int patcher,
                                       int iterations, int radius, float* d_stems, int64_t stem_stride, void* stream) {
  DCS_TRY(check_channels("dcs_separate_audio_channels_wiener", ctx, m, p, d_audio, nx, audio_stride, L, overlap, patcher,
                         d_stems, stem_stride, iterations, radius));
  DCS_CUDA(cudaSetDevice(ctx->device));
  return downmix_clip(ctx, m, p, nullptr, d_audio, nx, audio_stride, L, iterations, radius, scale_factor, overlap, patcher,
                      d_stems, stem_stride, (cudaStream_t)stream);
}

// the batch of C-channel clips, samples of in_fmt in and out_fmt out: per clip dcs_separate_audio_channels_wiener on
// the decoded planes, with the checks of that call on the longest clip.  resampled: the clips are at another rate,
// to / from the resampler pair (refused when NULL); else both are ignored
static int channels_batch(const char* fn, dcs_ctx* ctx, dcs_model* m, dcs_stft* p, bool resampled, const dcs_resampler* to,
                          const dcs_resampler* from, int in_fmt, int out_fmt, int nclips, const void* const* h_in,
                          const int64_t* num_samples, int channels, int iterations, int radius, float scale_factor,
                          int overlap, int patcher, void* const* h_out, const int64_t* out_strides, void* stream) {
  DCS_REQUIRE(sample_bytes(in_fmt) > 0 && sample_bytes(out_fmt) > 0, "%s: unknown sample format %d / %d", fn, in_fmt, out_fmt);
  if (resampled) {
    DCS_REQUIRE(ctx, "%s: NULL ctx", fn);
    DCS_REQUIRE(channels >= 1 && channels <= 16, "%s: channels %d not in [1, 16]", fn, channels);
    DCS_TRY(check_resample_channels(fn, ctx, to, from, channels, in_fmt));
  } else {
    to = from = nullptr;
  }
  DCS_REQUIRE(channels >= 1 && channels <= 16, "%s: channels %d not in [1, 16]", fn, channels);
  DCS_REQUIRE(iterations >= 0, "%s: iterations %d must be >= 0", fn, iterations);
  DCS_REQUIRE(radius >= 0, "%s: radius %d must be >= 0", fn, radius);
  DCS_REQUIRE(iterations == 0 || (channels >= 2 && channels <= 8), "%s: the Wiener post-filter needs channels in [2, 8], got %d",
              fn, channels);
  return batch_host(fn, ctx, m, p, to, from, in_fmt, out_fmt, nclips, h_in, num_samples, channels, 0, channels, iterations,
                    radius, scale_factor, overlap, patcher, h_out, out_strides, (cudaStream_t)stream, [&](int64_t Lmax) {
                      return check_channels(fn, ctx, m, p, h_in, channels, Lmax, Lmax, overlap, patcher, h_out, Lmax,
                                            iterations, radius);
                    });
}

int dcs_separate_batch_pcm16_channels_host(dcs_ctx* ctx, dcs_model* m, dcs_stft* p, int nclips, const int16_t* const* h_pcm,
                                           const int64_t* num_samples, int channels, int iterations, int radius,
                                           float scale_factor, int overlap, int patcher, int16_t* const* h_out,
                                           const int64_t* out_strides, void* stream) {
  return channels_batch("dcs_separate_batch_pcm16_channels_host", ctx, m, p, false, nullptr, nullptr, DCS_SAMPLE_I16,
                        DCS_SAMPLE_I16, nclips, (const void* const*)h_pcm, num_samples, channels, iterations, radius,
                        scale_factor, overlap, patcher, (void* const*)h_out, out_strides, stream);
}

int dcs_separate_batch_pcm16_channels_resampled_host(dcs_ctx* ctx, dcs_model* m, dcs_stft* p, const dcs_resampler* to_model,
                                                     const dcs_resampler* from_model, int nclips, const int16_t* const* h_pcm,
                                                     const int64_t* num_samples, int channels, int iterations, int radius,
                                                     float scale_factor, int overlap, int patcher, int16_t* const* h_out,
                                                     const int64_t* out_strides, void* stream) {
  return channels_batch("dcs_separate_batch_pcm16_channels_resampled_host", ctx, m, p, true, to_model, from_model,
                        DCS_SAMPLE_I16, DCS_SAMPLE_I16, nclips, (const void* const*)h_pcm, num_samples, channels, iterations,
                        radius, scale_factor, overlap, patcher, (void* const*)h_out, out_strides, stream);
}

int dcs_separate_batch_channels_host(dcs_ctx* ctx, dcs_model* m, dcs_stft* p, const dcs_resampler* to_model,
                                     const dcs_resampler* from_model, int in_format, int out_format, int nclips,
                                     const void* const* h_in, const int64_t* num_samples, int channels, int iterations,
                                     int radius, float scale_factor, int overlap, int patcher, void* const* h_out,
                                     const int64_t* out_strides, void* stream) {
  return channels_batch("dcs_separate_batch_channels_host", ctx, m, p, to_model || from_model, to_model, from_model,
                        in_format, out_format, nclips, h_in, num_samples, channels, iterations, radius, scale_factor, overlap,
                        patcher, h_out, out_strides, stream);
}

// ------------------------------------------------------------------------------------ long C-channel recordings
// The bounds of longclip.plan_segments (deepconvsep_b200/longclip.py documents their derivation) for the core [e0, e1)
// of a clip of Lm samples: the first frame frame0 (a multiple of step, of lcm(step, chunk) with the windowed Wiener
// filter) and the stop sample of the range whose separation is exact on the core.
static int64_t gcd_i64(int64_t a, int64_t b) { while (b) { const int64_t t = a % b; a = b; b = t; } return a; }

int64_t dcs_long_segments(int64_t num_samples, int64_t core_samples, int frame_size, int hop, int time_context, int overlap,
                          int wiener_reach, int to_up, int to_down, int to_ntaps, int from_ntaps, dcs_segment* out,
                          int64_t max_segments) {
  const int64_t L = num_samples, K = core_samples, N = frame_size, H = hop, tc = time_context, step = tc - overlap;
  if (L < 1 || K < 1 || N < 2 || H < 1 || overlap < 0 || step < 1 || wiener_reach < 0 || to_up < 1 || to_down < 1 ||
      to_ntaps < 1 || from_ntaps < 1 || max_segments < 0 || (max_segments > 0 && !out))
    return -1;
  const bool resampled = !(to_up == 1 && to_down == 1 && to_ntaps == 1 && from_ntaps == 1);
  const int64_t Lm = resampled ? dcs_resampled_length(L, to_up, to_down) : L;
  const int64_t CH = DCS_WIENER_CHUNK_FRAMES, R = wiener_reach;
  const int64_t q = ceil_div64(N / 2, H), s_v = ceil_div64(q, step) * step;
  const int64_t align = R ? step * CH / gcd_i64(step, CH) : step;
  const int64_t first_w = CH * (ceil_div64(s_v + overlap, CH) + R);   // longclip._wiener_first_frame(s_v + overlap, R)
  const int64_t nseg = ceil_div64(L, K);
  for (int64_t i = 0; i < nseg && i < max_segments; ++i) {
    dcs_segment& sg = out[i];
    sg.out_start = i * K;
    sg.out_stop = std::min(L, sg.out_start + K);
    // the core at 44.1 kHz: the samples the way back reads for it (from_model is to_down / to_up)
    int64_t e0 = sg.out_start, e1 = sg.out_stop;
    if (resampled) {
      e0 = std::max<int64_t>(0, support_lo(to_down, to_up, from_ntaps, sg.out_start));
      e1 = std::min<int64_t>(Lm, support_hi(to_down, to_up, from_ntaps, sg.out_stop - 1) + 1);
    }
    int64_t g0 = R ? floor_div64(floor_div64(e0 - N / 2, H) + 1 - first_w, align) * align
                   : floor_div64(floor_div64(e0 - N / 2, H) - s_v - overlap, step) * step;
    if (i == 0 || g0 <= 0) g0 = 0;   // the margin reaches the start: the true edge is the pipeline's own
    const int64_t s0 = g0 * H;
    int64_t s1 = Lm;
    if (i < nseg - 1) {
      int64_t G;
      if (R) {
        const int64_t b = floor_div64(e1 - 1 - s0 + N / 2, H);   // the last frame the last sample of the core reads
        G = CH * (floor_div64(b, CH) + R + 1) + q + tc - 2;
      } else {
        G = ceil_div64(e1 - s0 + N / 2, H) + q + tc - 1;
      }
      s1 = std::min(Lm, s0 + G * H);
    }
    sg.model_start = s0;
    sg.model_stop = s1;
    sg.in_start = s0;
    sg.in_stop = s1;
    if (resampled) {   // the recording's samples the decode of the model range reads
      sg.in_start = std::max<int64_t>(0, support_lo(to_up, to_down, to_ntaps, s0));
      sg.in_stop = std::min<int64_t>(L, support_hi(to_up, to_down, to_ntaps, s1 - 1) + 1);
    }
  }
  return nseg;
}

// the checks of the range entries beyond those of dcs_channels_decode / _encode: a window inside the whole signal's
// resampling, a staged range inside the signal that covers every input the window reads
static int check_range(const char* fn, const dcs_resampler* r, int64_t num_samples, int64_t in_first, int64_t num_staged,
                       int64_t out_first, int64_t num_out) {
  DCS_REQUIRE(num_samples >= 1, "%s: num_samples %lld must be >= 1", fn, (long long)num_samples);
  const int64_t most = resampler_length(r, num_samples);
  DCS_REQUIRE(out_first >= 0 && num_out >= 1 && out_first + num_out <= most, "%s: window [%lld, %lld) not inside [0, %lld)", fn,
              (long long)out_first, (long long)(out_first + num_out), (long long)most);
  DCS_REQUIRE(in_first >= 0 && num_staged >= 1 && in_first + num_staged <= num_samples,
              "%s: staged range [%lld, %lld) not inside [0, %lld)", fn, (long long)in_first, (long long)(in_first + num_staged),
              (long long)num_samples);
  int64_t lo, hi;
  resampler_support(r, out_first, out_first + num_out - 1, num_samples, &lo, &hi);
  DCS_REQUIRE(lo > hi || (in_first <= lo && in_first + num_staged > hi),
              "%s: the staged range [%lld, %lld) does not cover the window's inputs [%lld, %lld]", fn, (long long)in_first,
              (long long)(in_first + num_staged), (long long)lo, (long long)hi);
  return DCS_OK;
}

int dcs_channels_decode_range(dcs_ctx* ctx, const dcs_resampler* r, int format, const void* d_in, int64_t num_samples,
                              int64_t in_first, int64_t num_staged, int channels, float* d_out, int64_t out_first,
                              int64_t num_out, void* stream) {
  const char* fn = "dcs_channels_decode_range";
  DCS_REQUIRE(ctx && r && d_in && d_out, "%s: NULL argument", fn);
  DCS_REQUIRE(resampler_ctx(r) == ctx, "%s: the resampler was made on another ctx", fn);
  const int b = sample_bytes(format);
  DCS_REQUIRE(b > 0, "%s: unknown sample format %d", fn, format);
  DCS_REQUIRE((uintptr_t)d_in % sample_align(format) == 0 && (uintptr_t)d_out % 4 == 0,
              "%s: d_in not %d-byte or d_out not 4-byte aligned", fn, sample_align(format));
  DCS_REQUIRE(channels >= 1 && channels <= 16, "%s: channels %d not in [1, 16]", fn, channels);
  DCS_TRY(check_range(fn, r, num_samples, in_first, num_staged, out_first, num_out));
  DCS_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = (cudaStream_t)stream;
  return sync_after(fn, launch_resample_decode_range(r, format, d_in, num_samples, in_first, num_staged, channels, d_out,
                                                     out_first, num_out, st), st);
}

int dcs_channels_encode_range(dcs_ctx* ctx, const dcs_resampler* r, int format, const float* d_stems, int64_t num_samples,
                              int64_t in_first, int64_t num_in, int nsrc, int channels, void* d_out, int64_t out_first,
                              int64_t num_out, int64_t out_stride, void* stream) {
  const char* fn = "dcs_channels_encode_range";
  DCS_REQUIRE(ctx && r && d_stems && d_out, "%s: NULL argument", fn);
  DCS_REQUIRE(resampler_ctx(r) == ctx, "%s: the resampler was made on another ctx", fn);
  const int b = sample_bytes(format);
  DCS_REQUIRE(b > 0, "%s: unknown sample format %d", fn, format);
  DCS_REQUIRE(nsrc >= 1, "%s: nsrc %d must be >= 1", fn, nsrc);
  DCS_REQUIRE((uintptr_t)d_stems % 4 == 0 && (uintptr_t)d_out % sample_align(format) == 0,
              "%s: d_stems not 4-byte or d_out not %d-byte aligned", fn, sample_align(format));
  DCS_REQUIRE(channels >= 1 && channels <= 16, "%s: channels %d not in [1, 16]", fn, channels);
  DCS_TRY(check_range(fn, r, num_samples, in_first, num_in, out_first, num_out));
  DCS_REQUIRE(out_stride == (int64_t)channels * num_out, "%s: out_stride %lld != channels * num_out", fn, (long long)out_stride);
  DCS_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = (cudaStream_t)stream;
  return sync_after(fn, launch_resample_encode_range(r, format, d_stems, num_samples, in_first, num_in, nsrc, channels, d_out,
                                                     out_first, num_out, st), st);
}

int dcs_separate_long_channels_host(dcs_ctx* ctx, dcs_model* m, dcs_stft* p, const dcs_resampler* to_model,
                                    const dcs_resampler* from_model, int in_format, int out_format, const void* h_in,
                                    int64_t num_samples, int channels, int iterations, int radius, int64_t core_samples,
                                    float scale_factor, int overlap, int patcher, void* h_out, int64_t out_stride,
                                    void* stream) {
  const char* fn = "dcs_separate_long_channels_host";
  DCS_REQUIRE(sample_bytes(in_format) > 0 && sample_bytes(out_format) > 0, "%s: unknown sample format %d / %d", fn, in_format,
              out_format);
  DCS_REQUIRE(ctx, "%s: NULL ctx", fn);
  DCS_REQUIRE(channels >= 1 && channels <= 16, "%s: channels %d not in [1, 16]", fn, channels);
  const bool resampled = to_model || from_model;
  if (resampled) DCS_TRY(check_resample_channels(fn, ctx, to_model, from_model, channels, in_format));
  DCS_REQUIRE(iterations >= 0, "%s: iterations %d must be >= 0", fn, iterations);
  DCS_REQUIRE(radius >= 0, "%s: radius %d must be >= 0", fn, radius);
  DCS_REQUIRE(iterations == 0 || (channels >= 2 && channels <= 8), "%s: the Wiener post-filter needs channels in [2, 8], got %d",
              fn, channels);
  DCS_REQUIRE(h_in && h_out, "%s: NULL buffer", fn);
  DCS_REQUIRE(num_samples > 0 && core_samples >= 1 && out_stride >= num_samples,
              "%s: num_samples %lld, core_samples %lld, out_stride %lld", fn, (long long)num_samples, (long long)core_samples,
              (long long)out_stride);
  DCS_TRY(check_model(fn, ctx, m, -1, overlap, patcher));
  DCS_REQUIRE(p, "%s: NULL argument", fn);
  DCS_REQUIRE(!ctx->tap && !ctx->pool_tap,
              "%s: a spectrum or routing tap is set (dcs_set_spectrum_tap / dcs_set_pool_tap); a long recording's segments "
              "would overwrite it one after another", fn);
  const int64_t nseg = ceil_div64(num_samples, core_samples);
  DCS_REQUIRE(nseg <= (int64_t)1 << 24, "%s: %lld segments of %lld samples; take longer cores", fn, (long long)nseg,
              (long long)core_samples);
  DCS_REQUIRE(iterations == 0 || radius > 0 || nseg == 1,
              "%s: the Wiener post-filter with whole-clip covariances (radius 0) needs the whole recording in one segment, "
              "this one is cut into %lld: set radius >= 1 or core_samples >= num_samples", fn, (long long)nseg);
  std::vector<dcs_segment> segs((size_t)nseg);
  const int to_up = resampled ? resampler_up(to_model) : 1, to_down = resampled ? resampler_down(to_model) : 1;
  DCS_REQUIRE(dcs_long_segments(num_samples, core_samples, p->N, p->hop, m->tc, overlap, iterations * radius, to_up, to_down,
                                resampled ? resampler_ntaps(to_model) : 1, resampled ? resampler_ntaps(from_model) : 1,
                                segs.data(), nseg) == nseg,
              "%s: no segment plan for this geometry", fn);
  int64_t Smax = 0, Swork = 0, Kmax = 0;
  for (const dcs_segment& sg : segs) {
    Smax = std::max(Smax, sg.in_stop - sg.in_start);
    Swork = std::max(Swork, sg.model_stop - sg.model_start);
    Kmax = std::max(Kmax, sg.out_stop - sg.out_start);
  }
  DCS_TRY(check_channels(fn, ctx, m, p, h_in, channels, Swork, Swork, overlap, patcher, h_out, Swork, iterations, radius));
  const size_t bi = (size_t)sample_bytes(in_format) * channels, bo = (size_t)sample_bytes(out_format) * channels;
  std::vector<PipeClip> clips((size_t)nseg);
  for (int64_t i = 0; i < nseg; ++i) {
    const dcs_segment& sg = segs[(size_t)i];
    clips[(size_t)i] = PipeClip{(const char*)h_in + sg.in_start * bi, sg.in_stop - sg.in_start,
                                (char*)h_out + sg.out_start * bo, out_stride, &segs[(size_t)i], num_samples};
  }
  return run_pipeline(ctx, m, p, resampled ? to_model : nullptr, resampled ? from_model : nullptr, in_format, out_format, clips,
                      channels, 0, channels, iterations, radius, scale_factor, overlap, patcher, Smax, Swork, Kmax,
                      (cudaStream_t)stream);
}

// ------------------------------------------------------------------------------------ Wiener post-filter
static int wiener_stereo(const char* fn, dcs_ctx* ctx, const dcs_complex* d_X, int64_t x_plane, dcs_complex* d_S,
                         int64_t src_stride, int nsrc, int64_t T, int64_t ldf, int F, int iterations, int radius, void* stream) {
  DCS_REQUIRE(ctx && d_X && d_S, "%s: NULL argument", fn);
  DCS_REQUIRE((uintptr_t)d_X % sizeof(float2) == 0 && (uintptr_t)d_S % sizeof(float2) == 0, "%s: spectra not 8-byte aligned", fn);
  DCS_TRY(wiener_check(fn, nsrc, T, ldf, F, x_plane, src_stride, iterations, radius));
  DCS_CUDA(cudaSetDevice(ctx->device));
  return launch_wiener(ctx, (const float2*)d_X, x_plane, (float2*)d_S, src_stride, nsrc, T, ldf, F, iterations, radius,
                       (cudaStream_t)stream);
}

int dcs_wiener_stereo(dcs_ctx* ctx, const dcs_complex* d_X, int64_t x_plane, dcs_complex* d_S, int64_t src_stride, int nsrc,
                      int64_t T, int64_t ldf, int F, int iterations, void* stream) {
  return wiener_stereo("dcs_wiener_stereo", ctx, d_X, x_plane, d_S, src_stride, nsrc, T, ldf, F, iterations, 0, stream);
}

int dcs_wiener_stereo_windowed(dcs_ctx* ctx, const dcs_complex* d_X, int64_t x_plane, dcs_complex* d_S, int64_t src_stride,
                               int nsrc, int64_t T, int64_t ldf, int F, int iterations, int radius, void* stream) {
  return wiener_stereo("dcs_wiener_stereo_windowed", ctx, d_X, x_plane, d_S, src_stride, nsrc, T, ldf, F, iterations, radius,
                       stream);
}

int dcs_wiener_channels(dcs_ctx* ctx, const dcs_complex* d_X, int nx, int64_t x_plane, dcs_complex* d_S, int64_t src_stride,
                        int nsrc, int64_t T, int64_t ldf, int F, int iterations, int radius, void* stream) {
  const char* fn = "dcs_wiener_channels";
  DCS_REQUIRE(nx >= 2 && nx <= 8, "%s: nx %d not in [2, 8] (one channel has no spatial covariance)", fn, nx);
  DCS_REQUIRE(ctx && d_X && d_S, "%s: NULL argument", fn);
  DCS_REQUIRE((uintptr_t)d_X % sizeof(float2) == 0 && (uintptr_t)d_S % sizeof(float2) == 0, "%s: spectra not 8-byte aligned", fn);
  DCS_TRY(wiener_check(fn, nsrc, T, ldf, F, x_plane, src_stride, iterations, radius));
  DCS_CUDA(cudaSetDevice(ctx->device));
  return launch_wiener(ctx, (const float2*)d_X, x_plane, (float2*)d_S, src_stride, nsrc, T, ldf, F, iterations, radius,
                       (cudaStream_t)stream, nullptr, 0, nx);
}

}  // extern "C"
