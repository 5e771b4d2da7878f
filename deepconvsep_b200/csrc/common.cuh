// common.cuh -- shared helpers for libdcs (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>
#include <vector>
#include <string.h>
#include "../../include/dcs.h"

namespace dcs {

void set_error(const char* fmt, ...);

#define DCS_CUDA(expr)                                                                  \
  do {                                                                                  \
    cudaError_t _e = (expr);                                                            \
    if (_e != cudaSuccess) {                                                            \
      dcs::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return DCS_ECUDA;                                                                 \
    }                                                                                   \
  } while (0)

#define DCS_CHECK_LAUNCH()  DCS_CUDA(cudaGetLastError())

#define DCS_REQUIRE(cond, ...)                 \
  do {                                         \
    if (!(cond)) {                             \
      dcs::set_error(__VA_ARGS__);             \
      return DCS_EINVAL;                       \
    }                                          \
  } while (0)

#define DCS_TRY(expr)            \
  do {                           \
    int _r = (expr);             \
    if (_r != DCS_OK) return _r; \
  } while (0)

// cudaFuncAttributeMaxDynamicSharedMemorySize is a per-DEVICE property of a kernel: remembered per
// (kernel, current device), thread-safe (api.cu).  Call with the ctx's device current.
int ensure_smem_attr_impl(const void* kernel, int bytes);
template <typename K> inline int ensure_smem_attr(K kernel, int bytes) { return ensure_smem_attr_impl((const void*)kernel, bytes); }

__host__ __device__ inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }

// grow-only device buffer; newly allocated memory is zero-filled
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  int ensure(size_t bytes, cudaStream_t stream, bool* grew = nullptr);
  void release();
  template <typename T> T* as() const { return reinterpret_cast<T*>(p); }
};

// the context's scratch buffers beyond the clip buffers: the network's activations, the score-informed
// channel planes and the scratch of single launchers
enum NetSlot {
  NET_H1, NET_H2, NET_Z, NET_APAD, NET_G,   // both families: conv1, conv2, bottleneck, padded decoder, conv2^T
  NET_POOLED, NET_TIE,                      // max-pool net: pooled activations and tie bits
  NET_CHANS,                                // score-informed net: the 4 input channel planes
  NET_SPLITK,                               // split-K partial sums of the tensor-core GEMM
  NET_XC_PTRS, NET_XC_PARTIAL,              // dcs_xcorr_lags
  NET_XTAB, NET_AIMG,                       // DSD mask kernel's fade table and pre-split A operand image
  NET_ENC, NET_CODES, NET_DEC,              // 1x1 score net: encoder activations, ReLU gate codes, decoder chunk
  NET_NOTES,                                // compacted note table of the score-informed nets (score_notes.cu)
  NET_SLOTS
};

}  // namespace dcs

struct dcs_prof_rec {
  const char* name;
  cudaEvent_t e0, e1;
};

struct dcs_ctx {
  int device = 0;
  int num_sms = 132;
  int64_t launches = 0;
  bool prof_on = false;
  bool debug_simt_gemm = false;
  std::vector<dcs_prof_rec> prof;
  // workspace of one in-flight pipeline (api.cu walks every buffer for dcs_destroy / dcs_workspace_bytes)
  dcs::DevBuf audio, X, mag, S, stems;
  dcs::DevBuf masks;            // dcs_separate_audio_channels: the downmix's blended masks, nsrc float planes
  dcs::DevBuf net[dcs::NET_SLOTS];
  uint64_t net_sig[dcs::NET_SLOTS] = {0};   // layout signature of what each net[] buffer currently holds
  // multi-clip scheduler (dcs_separate_batch_pcm16_host, dcs_separate_batch_channels_host): copy streams,
  // double-buffered staging, hand-over events
  cudaStream_t s_h2d = nullptr, s_d2h = nullptr;
  cudaEvent_t ev_in[2] = {nullptr, nullptr}, ev_dec[2] = {nullptr, nullptr}, ev_enc[2] = {nullptr, nullptr}, ev_out[2] = {nullptr, nullptr};
  dcs::DevBuf pcm_in[2], pcm_out[2];
  float2* tap = nullptr;        // dcs_set_spectrum_tap: copy of the masked spectra the iSTFT consumed
  int64_t tap_cap = 0;
  uint8_t* pool_tap = nullptr;  // dcs_set_pool_tap: copy of the routing decisions of the forward pass
  int64_t pool_tap_cap = 0;
  int wiener_iters = 0;         // dcs_set_wiener: EM iterations of the stereo Wiener post-filter (0 = off)
  int wiener_radius = 0;        // dcs_set_wiener_radius: its covariance window in chunks to either side (0 = whole clip)
  dcs::DevBuf wiener;           // its partial sums, spatial covariances and mixture scale (wiener.cu)
  int32_t* notes_host = nullptr;      // pinned staging of the compacted note table (its device copy: net[NET_NOTES])
  size_t notes_host_cap = 0;
  cudaEvent_t ev_notes = nullptr;     // the copy out of notes_host; guards its reuse
};

struct dcs_stft {
  dcs_ctx* ctx;
  int N, hop;
  float* d_win;    // analysis window  float[N]
  float* d_wsyn;   // synthesis window float[N]
  float* d_w2;     // wsyn * win       float[N]
  float2* d_tw;    // exp(-2*pi*i*q/N), q < N
};

namespace dcs {
// records a pair of CUDA events around a pipeline stage when profiling is enabled on the ctx
struct ProfScope {
  dcs_ctx* c; cudaStream_t st; int idx;
  ProfScope(dcs_ctx* ctx, const char* name, cudaStream_t s) : c(ctx), st(s), idx(-1) {
    if (!c || !c->prof_on) return;
    dcs_prof_rec r; r.name = name;
    if (cudaEventCreate(&r.e0) != cudaSuccess || cudaEventCreate(&r.e1) != cudaSuccess) return;
    cudaEventRecord(r.e0, st);
    c->prof.push_back(r);
    idx = (int)c->prof.size() - 1;
  }
  ~ProfScope() { if (idx >= 0) cudaEventRecord(c->prof[idx].e1, st); }
};
}  // namespace dcs

namespace dcs {
// weight matrix prepared for the tensor-core path: K-major, zero padded, split for 3xTF32
struct TcWeight {
  float* hi = nullptr;   // [Np][Kp], K-major, zero padded
  float* lo = nullptr;   // = hi + Np*Kp (one allocation)
  int K = 0, N = 0, Kp = 0, Np = 0;
};
}  // namespace dcs

// ---- model (device-resident network)
struct dcs_dsd {     // DSD100 / hiphopss and the stereo / ILD net
  int C1, C2, kh2, h2, nfc, ndec;
  int C1p, C2p;   // channel pitch of the activation buffers (multiple of 4 floats)
  int64_t ldw;
  float *b1, *b2, *bfc, *bdec, *W1t, *bout;   // W1t is [nch][C1][ldw], bout [nch][4]
  // conv1, conv2, bottleneck, decoder dense and InverseLayer(conv2) weights for the tensor cores (K-major, 3xTF32 split)
  dcs::TcWeight tW1f, tW2c, tWfc, tWdec, tWt2;
};
struct dcs_sconv {   // strided-conv1 families: iKala (pool / no pool), Bach10
  int nch, sw1, J, pool, WP, kh2, kw2, h2, w2, HP, WPP, ndec, nfc, rule;   // nch: input planes of the network
  dcs::TcWeight tW[8];                 // 0 conv1, 1 conv2, 2 fc, 3 convT2, 4.. decoder dense layers
  float *b1, *b2, *bfc, *bdec[4], *bout, *Wsc;
};
struct dcs_s1x1 {    // score-informed build_ca_1x1: six strided ReLU convolutions, a 1x1 conv, gated transposed convs
  int W[7];             // W[0] = F, W[l] = width of conv l's output
  int C[7], CP[7];      // channels and channel pitch of each activation (C[0] = 4 input planes)
  dcs::TcWeight tF[7];  // forward: conv1..conv6 (index l), 1x1 conv (index 0; first 200 filters only)
  dcs::TcWeight tI[7];  // InverseLayer(conv l) for l = 2..6
  float *b[7], *c[7];   // bias before / after the ReLU (index 0: 1x1 conv)
  float *bout, *Wsc;    // final bias 0..3; K3s filter banks of conv1
};
struct dcs_model {
  dcs_ctx* ctx;
  int arch, F, tc, nsrc;
  int nch = 1;    // audio channels of a clip; the stems are nsrc x nch planes (2: stereo / ILD net)
  dcs_dsd dsd;
  dcs_sconv sc;
  dcs_s1x1 s1;
  std::vector<void*> dev;   // every device allocation of the model, tensor-core weights included
};
namespace dcs {
// owned: a list the allocation is recorded in (a model's, which dcs_model_destroy frees)
int upload(const std::vector<float>& h, float** d, std::vector<void*>* owned = nullptr);
int model_create_dsd(dcs_model* m, int nparams, const float* const* hp, const int64_t* shp, const int* nd);
int model_create_sconv(dcs_model* m, int nparams, const float* const* hp, const int64_t* shp, const int* nd);
int model_create_s1x1(dcs_model* m, int nparams, const float* const* hp, const int64_t* shp, const int* nd);
bool shape_is(const int64_t* s, int nd, int want_nd, int64_t a, int64_t b = 1, int64_t c = 1, int64_t d = 1);

// one call of the network stage (run_network, api.cu): the network's input planes [T][ldf] (plane c at
// in + c * in_plane), the mixture STFT (channel c at X + c * x_plane) -> the masked spectra, plane p at S + p * src_stride
struct NetCall {
  const float* in; int64_t in_plane;
  const float2* X; int64_t x_plane;
  float2* S; int64_t src_stride;
  float* M;         // masks mode (non-NULL): the blended masks, float plane p at M + p * src_stride; X and S unused
  int64_t T, ldf;
  int64_t P, Tp;    // patches (> 0) and the frames they span
  int overlap, step;
  uint64_t sig;     // layout signature of the zero-padded slots for this model and overlap
};
// the layer sequence of each family (dsd_model.cu, sconv_model.cu, score1x1.cu)
int dsd_forward(dcs_ctx* ctx, const dcs_model* m, const NetCall& n, cudaStream_t st);
int sconv_forward(dcs_ctx* ctx, const dcs_model* m, const NetCall& n, cudaStream_t st);
int s1x1_forward(dcs_ctx* ctx, const dcs_model* m, const NetCall& n, cudaStream_t st);
// (re)zero a workspace slot whenever what it holds changes layout: zero padding is relied upon
int ensure_layout(dcs_ctx* ctx, NetSlot slot, size_t bytes, uint64_t sig, cudaStream_t st);
}  // namespace dcs

// ---- kernel launchers (each returns a DCS_* code) ---------------------------------------------
namespace dcs {

int launch_stft(dcs_stft* plan, const float* d_audio, int64_t L, float2* d_X, float* d_mag,
                float* d_phase, float mag_scale, int64_t ldf, cudaStream_t st);
// d_M set (masked inverse, d_mag / d_phase NULL): d_S is the mixture STFT of nx channels (src_stride apart), d_M the
// float masks of nsrc sources [T][ldf] (m_stride apart); output plane s * nx + c = istft_norm(M_s * X_c)
int launch_istft(dcs_stft* plan, const float2* d_S, const float* d_mag, const float* d_phase,
                 float polar_scale, int nsrc, int64_t T, int64_t ldf, int64_t src_stride, float* d_out,
                 int64_t Lout, int64_t out_stride, cudaStream_t st, const float* d_M = nullptr, int64_t m_stride = 0,
                 int nx = 1);

// nsrc mask planes M (plane floats apart) times the one mixture STFT plane X -> nsrc complex planes S, bins >= F zeroed
int launch_masked_spectra(dcs_ctx* ctx, const float* d_M, const float2* d_X, int nsrc, int64_t plane, int64_t ldf, int F,
                          float2* d_S, cudaStream_t st);

int launch_stft_reg(dcs_stft* plan, const float* d_audio, int64_t L, float2* d_X, float* d_mag, float* d_phase,
                    float mag_scale, int64_t ldf, int64_t nframes, cudaStream_t st);
bool istft_reg_supported(const dcs_stft* plan, const float* d_out, int64_t out_stride);
int launch_istft_reg(dcs_stft* plan, const float2* d_S, int nsrc, int64_t nframes, int64_t ldf, int64_t src_stride,
                     float* d_out, int64_t Lout, int64_t out_stride, cudaStream_t st, const float* d_M = nullptr,
                     int64_t m_stride = 0, int nx = 1);

// generic strided-operand GEMM  C = act(A*B + bias)
struct GemmDesc {
  const float* A; const float* B; const float* bias; float* C;
  int M, N, K;
  int a_valid_rows;          // rows >= a_valid_rows of A read as zeros
  // A row offset = (m / m_inner) * a_so + ((m % m_inner) / m_inner2) * a_si + (m % m_inner2) * a_s2
  int m_inner; int64_t a_so, a_si;
  int m_inner2; int64_t a_s2;
  int k_seg; int64_t k_ss;           // A col offset  = (k / k_seg) * k_ss + (k % k_seg)
  int64_t ldb;                       // B[k][n] at B + k*ldb + n
  int cm_inner; int64_t c_so, c_si;  // C row offset (same three-level form)
  int cm_inner2; int64_t c_s2;
  int n_seg; int64_t n_ss, c_col0;   // C col offset  = c_col0 + (n / n_seg) * n_ss + (n % n_seg)
  int relu;
  // optional K clipping for transposed convolutions on a zero-padded operand: rows are grouped by
  // output position u = m / kc_rows; only taps q with kc_pad <= u + q < kc_pad + kc_n touch
  // non-zero input, so a tile skips the k-blocks outside [kc_unit*q_lo, kc_unit*(q_hi+1)).
  // kc_rows = 0 disables it.  (Pure optimisation: the skipped products are exact zeros.)
  int kc_rows, kc_unit, kc_pad, kc_n, kc_taps;
  // epilogue of the rectifier-gated 1x1 score net, read only by launch_gemm_tc_epi (compile-time options):
  //   EPI_POST: x = relu(x + bias) + bias2, and with `code` set the gate code 2*relu'(x + bias) in {0, 1, 2}
  //             (1 at exactly 0, Theano's 0.5*(x + |x|)) is stored at code[m * N + n]
  //   EPI_GATE: x *= 0.5 * gate[(m / g_inner) * g_so + ((m % g_inner) / g_inner2) * g_si + (m % g_inner2) * g_s2 + n];
  //             where (m % g_inner2) * g_s2 + n >= g_lim (outside the gated layer's width) nothing is stored
  const float* bias2; uint8_t* code;
  const uint8_t* gate; int g_inner, g_inner2; int64_t g_so, g_si, g_s2, g_lim;
};
enum { EPI_POST = DCS_GEMM_EPI_POST, EPI_GATE = DCS_GEMM_EPI_GATE };
// every C offset of the view is >= 0: the epilogues store without a lower bound check.  All layers build their views
// from non-negative strides; each launcher refuses a view that breaks this.
inline bool gemm_c_view_ok(const GemmDesc& d) {
  return d.c_so >= 0 && d.c_si >= 0 && d.c_s2 >= 0 && d.n_ss >= 0 && d.c_col0 >= 0;
}
// element offset of row m of C (without the column part)
__host__ __device__ __forceinline__ int64_t gemm_c_row_offset(const GemmDesc& d, int m) {
  return (int64_t)(m / d.cm_inner) * d.c_so + (int64_t)((m % d.cm_inner) / d.cm_inner2) * d.c_si +
         (int64_t)(m % d.cm_inner2) * d.c_s2 + d.c_col0;
}
GemmDesc gemm_plain(const float* A, int64_t lda, const float* B, int64_t ldb, const float* bias, float* C,
                    int64_t ldc, int M, int N, int K, int relu);
int launch_gemm(dcs_ctx* ctx, const GemmDesc& d, cudaStream_t st);

int tc_weight_create(const float* B_rowmajor, int64_t ldb, int K, int N, TcWeight* out, std::vector<void*>* owned = nullptr);
void tc_weight_destroy(TcWeight* w);
int launch_gemm_tc(dcs_ctx* ctx, const GemmDesc& d, const TcWeight& w, cudaStream_t st);
// the same GEMM with the gated epilogue `epi` (EPI_POST | EPI_GATE); never split over K
int launch_gemm_tc_epi(dcs_ctx* ctx, const GemmDesc& d, const TcWeight& w, int epi, cudaStream_t st);

struct DsdMaskArgs {
  const float* G;      // [P][ndec][tc][ldg]  decoder activations after the transposed conv2
  int ldg;
  const float* W1t;    // [50][ldw]  W1t[c][b] = conv1.W[c,0,0,F-1-b]
  int ldw;
  const float* bout;   // [4]
  const float2* X;     // [T][ldf]
  float2* S;           // [4][T][ldf]: source s at S + s * src_stride
  int64_t ldf, src_stride;
  int T, P, tc, overlap, F;
  int ndec;            // 3: DSD100 (4th output = decoder 2, all-zero bins get 1/4); 4: one decoder per source,
                       //    all-zero bins get 0 (stereo / ILD net, one launch per channel)
};
// every mask kernel takes a total of the rectified sources at or below this as "all sources zero" (the rule's 1/nsrc or
// 0): the reciprocal of a subnormal total overflows, and the masks would be inf * 0 = NaN.  dsd_tc.cu tests the same value.
constexpr float MASK_TOT_MIN = 1.2e-38f;
// Every mask launcher has a masks-output mode: with M set, the blended masks -- the fp32 values the other mode multiplies
// by X -- are stored instead, float plane of source s at M + s * src_stride (bins < F of each frame); X and S are not
// read or written.
int launch_dsd_mask(dcs_ctx* ctx, const DsdMaskArgs& a, cudaStream_t st, float* M = nullptr);
bool dsd_mask_tc_supported(const DsdMaskArgs& a);
int launch_dsd_mask_tc(dcs_ctx* ctx, const DsdMaskArgs& a, cudaStream_t st, float* M = nullptr);   // wgmma (dsd_tc.cu)
// InverseLayer(conv2) of the DSD nets: G[pair][u][c] = sum_{q, f} apad[pair][u + q][f] * Wt2[q][f][c] for the
// npairs = P * ndec (patch, decoder) pairs, u < tc; only the h2 interior rows [kh2 - 1, kh2 - 1 + h2) of apad are read
struct DsdConvT2Args {
  const float* apad;   // [npairs][h2 + 2 (kh2 - 1)][52], 16-byte aligned
  float* G;            // [npairs][tc][ldg]: columns 0..49 written, 8-byte aligned
  int ldg;
  int npairs, tc;
};
bool dsd_convT2_tc_supported(const DsdConvT2Args& a);
// w: the transposed conv2 weight as tc_weight_create lays it out (K = kh2 * 52, N = 50)
int launch_dsd_convT2_tc(dcs_ctx* ctx, const DsdConvT2Args& a, const TcWeight& w, cudaStream_t st);   // dsd_convT2_tc.cu
// the decoder dense layers of the DSD nets, N = ndec h2 52 columns, scattered into the interior rows of apad:
// apad[k][d][kh2 - 1 + i][c] = ReLU(z[k] . W[:, n] + bias[n]), n = (d h2 + i) 52 + c
struct DsdDenseArgs {
  const float* z;      // [P][nfc], 4-byte aligned
  const float* bias;   // [ndec h2 52]
  float* apad;         // [P][ndec][h2 + 2 (kh2 - 1)][52]: interior rows written, 8-byte aligned
  int P, tc, ndec, nfc;
};
bool dsd_dense_tc_supported(const DsdDenseArgs& a);
// w: the dense weight as tc_weight_create lays it out (K = nfc, N = ndec h2 52)
int launch_dsd_dense_tc(dcs_ctx* ctx, const DsdDenseArgs& a, const TcWeight& w, cudaStream_t st);   // dsd_dense_tc.cu
// strided-conv1 families (iKala / Bach10): K3s arguments
struct SconvMaskArgs {
  int arch;
  const float* G;       // [P*ndec][tc][WP or J][32] decoder activations after the transposed conv2
  const uint8_t* tie;   // [T'][WP][32] max-pool tie bits of the forward pass (pooled nets only)
  const float* W;       // float4 [ND][32]: W[dd][f][r] = conv1.W[f][0][0][KW-1-r-STRIDE*dd]
  const float* bout;    // [nsrc]
  const float2* X;      // [T][ldf]
  float2* S;            // [nsrc][T][ldf]
  int64_t ldf, src_stride;
  int T, P, tc, overlap, F, J, WP;
  // G holds patches p_base.. only; frames [t0, t1) are written (one decoder chunk; a whole clip: 0 and [0, T))
  int p_base, t0, t1;
};
int launch_pool4(dcs_ctx* ctx, const float* H1, float* Hp, uint8_t* tie, int64_t rows, int J, int WP, cudaStream_t st);
int launch_sconv_mask(dcs_ctx* ctx, const SconvMaskArgs& a, cudaStream_t st, float* M = nullptr);
bool sconv_mask_tc_supported(const SconvMaskArgs& a);
int launch_sconv_mask_tc(dcs_ctx* ctx, const SconvMaskArgs& a, cudaStream_t st, float* M = nullptr);   // wgmma (sconv_tc.cu)
int launch_channel_mul(dcs_ctx* ctx, const float* mag, const float* filt, float* out, int64_t plane, int nch, cudaStream_t st);

// the note table of the score-informed nets (score_notes.cu), compacted for the frame window [start, start + T):
// int32 words, frame_ptr[T + 1] at 0 (CSR of the notes sounding in each frame), note indices at `entries`,
// (instrument, first range, range count) per note at `recs`, (lo, hi) bin pairs at `ranges`
struct NoteTable {
  const int32_t* d;   // device copy
  int ninst, F;
  int64_t T, entries, recs, ranges, size;
};
// validates the whole table (DCS_EINVAL, nothing queued) and compacts it
int notes_compact(const char* fn, const double* h_melody, int ninst, int nnotes, int ncols, int64_t start, int64_t T, int F,
                  std::vector<int32_t>* tab, NoteTable* nt);
// pinned staging -> net[NET_NOTES] on `st`; sets nt->d
int notes_stage(dcs_ctx* ctx, const std::vector<int32_t>& tab, NoteTable* nt, cudaStream_t st);
// out + j * plane: filter j [T][ldf] (mag == NULL) or filter j * mag (mag [T][ldf]); pad columns F..ldf-1 = 0
int launch_score_notes(dcs_ctx* ctx, const NoteTable& nt, const float* mag, float* out, int64_t ldf, int64_t plane,
                       cudaStream_t st);

int launch_xcorr_lags(dcs_ctx* ctx, const float* const* h_a, const float* const* h_b, int npairs, int64_t L, int flen,
                      double* h_out, cudaStream_t st);
int launch_pcm_decode(dcs_ctx* ctx, const int16_t* d_pcm, int64_t L, int channels, int downmix, float* d_audio,
                      cudaStream_t st);
int launch_pcm_encode(dcs_ctx* ctx, const float* d_stems, int64_t L, int nsrc, int64_t stem_stride, int16_t* d_out,
                      int64_t out_stride, cudaStream_t st);

// The sample formats of the C-channel batch (DCS_SAMPLE_*, include/dcs.h): the stored type, the decode of a sample to
// the fp32 plane and the encode of an fp32 stem value, the rules written in dcs.h
template <int FMT> struct SampleFormat;
template <> struct SampleFormat<DCS_SAMPLE_I16> {
  using T = int16_t;
  static __device__ __forceinline__ float decode(T x) { return (float)x / 32767.0f; }
  static __device__ __forceinline__ T encode(float y) { return (int16_t)(int)(y * 32767.0f); }   // wraps modulo 2^16
};
template <> struct SampleFormat<DCS_SAMPLE_I32> {
  using T = int32_t;
  static __device__ __forceinline__ float decode(T x) { return (float)((double)x / 2147483647.0); }
  // truncates and saturates; cvt from f64 would give INT_MIN for NaN, so NaN is tested first
  static __device__ __forceinline__ T encode(float y) { return y == y ? __double2int_rz((double)y * 2147483647.0) : 0; }
};
template <> struct SampleFormat<DCS_SAMPLE_F32> {
  using T = float;
  static __device__ __forceinline__ float decode(T x) { return x; }
  static __device__ __forceinline__ T encode(float y) { return y; }
};
// packed 24-bit PCM: a 3-byte POD, so that pcm[j * C + c] is a sample's three byte loads or stores at any address
struct Pcm24 { uint8_t b[3]; };
template <> struct SampleFormat<DCS_SAMPLE_I24> {
  using T = Pcm24;
  // the int32 rule on v << 8: the bits the int32 route gives for scipy's read of the same WAV data chunk
  static __device__ __forceinline__ float decode(T x) {
    return SampleFormat<DCS_SAMPLE_I32>::decode((int32_t)(((uint32_t)x.b[0] << 8) | ((uint32_t)x.b[1] << 16) |
                                                          ((uint32_t)x.b[2] << 24)));
  }
  // the int32 encode's top 24 bits (its arithmetic shift right by 8): saturated to [-2^23, 2^23 - 1], NaN gives 0
  static __device__ __forceinline__ T encode(float y) {
    const uint32_t e = (uint32_t)SampleFormat<DCS_SAMPLE_I32>::encode(y);
    return T{{(uint8_t)(e >> 8), (uint8_t)(e >> 16), (uint8_t)(e >> 24)}};
  }
};
// bytes of one sample; 0 for an unknown format code
inline int sample_bytes(int fmt) {
  return fmt == DCS_SAMPLE_I16 ? 2 : (fmt == DCS_SAMPLE_I32 || fmt == DCS_SAMPLE_F32) ? 4 : fmt == DCS_SAMPLE_I24 ? 3 : 0;
}
// the alignment a device buffer of the format needs: its sample size, 1 byte for packed 24-bit
inline int sample_align(int fmt) { return fmt == DCS_SAMPLE_I24 ? 1 : sample_bytes(fmt); }

// C-channel stems, C in [1, 16], samples in format fmt: interleaved [L][C] -> C + 1 float planes L apart (the downmix
// of launch_downmix, then the C channels); nsrc x C stem planes (source, channel) -> [nsrc][L][C], source s at
// d_out + s * C * L samples
int launch_pcm_decode_channels(dcs_ctx* ctx, int fmt, const void* d_in, int64_t L, int C, float* d_planes, cudaStream_t st);
int launch_pcm_encode_channels(dcs_ctx* ctx, int fmt, const float* d_stems, int64_t L, int nsrc, int C, int64_t stem_stride,
                               void* d_out, cudaStream_t st);
// nx float planes -> (((a_0 + a_1) + a_2) + ...) * (1.0f / nx): the downmix of launch_pcm_decode_channels, a copy
// at nx = 1
int launch_downmix(dcs_ctx* ctx, const float* d_audio, int nx, int64_t audio_stride, int64_t L, float* d_mono, cudaStream_t st);

// the C-channel batch at another rate (resample.cu), C in [1, 16], on the resampler's ctx.  check_resample_channels:
// what the batch refuses of its resampler pair (NULL, another ctx, not inverse, no tile that fits for samples in
// in_fmt).  decode: [L][C] in fmt -> C + 1 float planes Lout apart at the resampler's output rate (the downmix, then the
// channels), each channel the bits of dcs_resample on the decoded plane; one launch, or two when the 4-byte staging
// splits the channels into groups (resample_decode_groups > 1: the downmix is then launch_downmix on the resampled
// planes).  encode: nsrc x C stem planes (source, channel) Lin apart -> [nsrc][L][C] in fmt at the output rate, the
// encode of dcs_resample's y trimmed to L
int64_t resampler_length(const dcs_resampler* r, int64_t num_in);
const dcs_ctx* resampler_ctx(const dcs_resampler* r);
int resampler_up(const dcs_resampler* r);
int resampler_down(const dcs_resampler* r);
int resampler_ntaps(const dcs_resampler* r);
int check_resample_channels(const char* fn, const dcs_ctx* ctx, const dcs_resampler* to, const dcs_resampler* from, int C,
                            int in_fmt);
int resample_decode_groups(const dcs_resampler* r, int C, int fmt);
int launch_resample_decode(const dcs_resampler* r, int fmt, const void* d_in, int64_t L, int C, float* d_planes, int64_t Lout,
                           cudaStream_t st);
int launch_resample_encode(const dcs_resampler* r, int fmt, const float* d_stems, int64_t Lin, int nsrc, int C, void* d_out,
                           int64_t L, cudaStream_t st);
// the same launches on a window of the whole signal: decode outputs [out_first, out_first + Lout) of the resampling of a
// recording of L samples staged as its samples [in_first, in_first + num_staged) (zeros elsewhere); encode outputs
// [out_first, out_first + L) of the resampling of a 44.1 kHz signal of Lm samples whose stems are given at
// [in_first, in_first + Lin) (zeros elsewhere), the stem planes Lin apart
int launch_resample_decode_range(const dcs_resampler* r, int fmt, const void* d_in, int64_t L, int64_t in_first,
                                 int64_t num_staged, int C, float* d_planes, int64_t out_first, int64_t Lout, cudaStream_t st);
int launch_resample_encode_range(const dcs_resampler* r, int fmt, const float* d_stems, int64_t Lm, int64_t in_first,
                                 int64_t Lin, int nsrc, int C, void* d_out, int64_t out_first, int64_t L, cudaStream_t st);
// the inputs output m of a resampler (up, down, ntaps) reads: lo(m) = ceil((m down + half - ntaps + 1) / up) through
// hi(m) = floor((m down + half) / up), half = (ntaps - 1) / 2, before clipping to the input
inline int64_t floor_div64(int64_t a, int64_t b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }
inline int64_t support_lo(int up, int down, int ntaps, int64_t m) {
  return -floor_div64(-(m * down + (ntaps - 1) / 2 - ntaps + 1), up);
}
inline int64_t support_hi(int up, int down, int ntaps, int64_t m) { return floor_div64(m * down + (ntaps - 1) / 2, up); }
// [lo, hi]: the inputs outputs m_first..m_last read, clipped to [0, num_in) (lo > hi: none)
void resampler_support(const dcs_resampler* r, int64_t m_first, int64_t m_last, int64_t num_in, int64_t* lo, int64_t* hi);

// multichannel Wiener post-filter (wiener.cu): nch (2..8) mixture channels, channel c at X + c * x_plane, stem (j, c) at
// S + (j * nch + c) * src_stride, bins f < F filtered in place by `iterations` EM iterations; radius: the covariance
// window in chunks of DCS_WIENER_CHUNK_FRAMES frames to either side (0 = the whole clip).  M set: the stems are not in S
// yet; the first pass forms stem (j, c) as M_j * X_c (float masks [T][ldf], m_stride apart), componentwise in fp32, and
// stores it to S.  nch 2 runs the 2 x 2 kernels, more channels the C x C ones
int wiener_check(const char* fn, int nsrc, int64_t T, int64_t ldf, int F, int64_t x_plane, int64_t src_stride, int iterations,
                 int radius);
size_t wiener_workspace_bytes(int nsrc, int nch, int64_t T, int F, int radius);
int launch_wiener(dcs_ctx* ctx, const float2* X, int64_t x_plane, float2* S, int64_t src_stride, int nsrc, int64_t T,
                  int64_t ldf, int F, int iterations, int radius, cudaStream_t st, const float* M = nullptr,
                  int64_t m_stride = 0, int nch = 2);

}  // namespace dcs
