/* dcs.h -- C ABI of libdcs.so, the H100 (sm_90a) separation hot path of DeepConvSep.
 *
 * The reference (MTG/DeepConvSep) is pure Python and has no FFI layer; the boundary it
 * exposes for this path is the Python surface `transform.transformFFT` and
 * `examples/<family>/separate_*.py`.  Each entry point below names the reference function(s) it
 * replaces (paths relative to the reference root).  INTEGRATION.md shows the ctypes stub a
 * maintainer would add to the reference.
 *
 * Conventions
 *  - every function returns 0 on success or a negative DCS_E* code; dcs_last_error() returns
 *    a thread-local message for the last failure on the calling thread;
 *  - `d_` pointers are device memory owned by the caller, `h_` pointers are host memory;
 *  - every launch is asynchronous on the given `stream` (a cudaStream_t passed as void*;
 *    NULL = the legacy default stream) unless the name ends in `_host`, which synchronises
 *    the stream before returning;
 *  - a dcs_ctx is bound to one device and owns the (grow-only) workspace of ONE in-flight
 *    pipeline: use one ctx per stream / host thread;
 *  - spectrogram row stride `ldf` is in elements and must be >= F = N/2+1; use
 *    dcs_padded_bins(N) for buffers handed to dcs_separate_spec.
 *  - there is NO CPU fallback: with no usable CUDA device dcs_create fails.
 */
#ifndef DCS_H_
#define DCS_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DCS_VERSION 101

/* frames per chunk of the Wiener post-filter's sums over time (dcs_wiener_stereo_windowed) */
#define DCS_WIENER_CHUNK_FRAMES 128

enum {
  DCS_OK = 0,
  DCS_EINVAL = -1,   /* bad argument / unsupported shape */
  DCS_ECUDA = -2,    /* CUDA runtime error (message has the cudaError string) */
  DCS_ENOMEM = -3,   /* device allocation failed */
  DCS_EMODEL = -4    /* parameter list does not match the architecture */
};

/* network families = the reference's build_ca() variants */
enum {
  DCS_ARCH_DSD = 0,          /* examples/dsd100/separate_dsd.py:172-236 (= hiphopss/separate_hhds.py) */
  DCS_ARCH_IKALA = 1,        /* examples/ikala/separate_ikala.py:172-192 (max-pool) */
  DCS_ARCH_IKALA_NOPOOL = 2, /* examples/ikala/trainCNN.py:66-110 */
  DCS_ARCH_BACH10 = 3,       /* examples/bach10/separate_bach10.py:172-229 */
  DCS_ARCH_BACH10_SCORE = 4, /* examples/bach10_scoreinformed/trainCNNrwc.py:134-193 (17 arrays); also the one-decoder
                                build_ca of trainCNNrwc_samp.py:195-235 (11 arrays) */
  DCS_ARCH_DSD_ILD = 5,      /* examples/dsd100_2ch_ILD/trainCNN_ILD_DSD100.py:66-113 (stereo in, nsrc x 2 out) */
  DCS_ARCH_BACH10_SCORE_1X1 = 6 /* examples/bach10_scoreinformed/trainCNNrwc.py:66-132 (--function build_ca_1x1, 22 arrays):
                                   six strided ReLU convolutions + a 1x1 conv, ReLU-gated InverseLayers.  Served by
                                   dcs_separate_audio_score and dcs_separate_spec_channels only.  feat_size (>= 253) and
                                   time_context (>= 19) are not in the weights; the trainer uses 2049 and 30.  feat_size
                                   need not be 2^k+1 for dcs_separate_spec_channels */
};

/* patch generators */
enum {
  DCS_PATCHER_STANDALONE = 0, /* separate_dsd.py:114-135  (while start+time_context < T, tail dropped) */
  DCS_PATCHER_UTIL = 1        /* util.py:220-248          (while start+overlap < T, zero padded) */
};

typedef struct dcs_ctx dcs_ctx;
typedef struct dcs_stft dcs_stft;
typedef struct dcs_model dcs_model;
typedef struct { float x, y; } dcs_complex; /* layout-compatible with CUDA float2 / numpy complex64 */

int dcs_version(void);
const char* dcs_last_error(void);

/* ---- context ---------------------------------------------------------------------------- */
int dcs_create(int device, dcs_ctx** out);
int dcs_destroy(dcs_ctx* ctx);
/* bytes of device workspace currently held by the ctx */
int64_t dcs_workspace_bytes(const dcs_ctx* ctx);
/* number of kernels this library has launched through `ctx` since creation */
int64_t dcs_launch_count(const dcs_ctx* ctx);

/* Inspection tap (used by the parity tests): while set, every dcs_separate_audio* / *_host call on this ctx
 * also copies the blended masked spectra its inverse STFT consumed -- complex[nplanes][T][ldf],
 * ldf = dcs_padded_bins(N), nplanes = nsrc (x 2 channels, ordered (source, channel), for the stereo net and for
 * dcs_separate_*keep_channels* with the Wiener post-filter on; without it those form no masked spectra and refuse the
 * tap, as dcs_separate_audio_channels does) -- to d_S (capacity in
 * elements; the call fails if it is too small).  d_S = NULL switches it off.  These are the tensors
 * `overlapadd_multi(...)/scale * exp(j*phase)` of separate_dsd.py:301-304. */
int dcs_set_spectrum_tap(dcs_ctx* ctx, dcs_complex* d_S, int64_t capacity);
/* Same for the discrete routing decisions of the forward pass, which the InverseLayers of the decoder follow.
 * The parity tests adopt the device's decisions where float64 flags them as ill-conditioned and require agreement
 * elsewhere.  capacity in bytes; NULL = off.
 *  - max-pool network (DCS_ARCH_IKALA): the tie bits of MaxPool2DLayer((1,4)) the un-pool (InverseLayer(pool),
 *    separate_ikala.py:183,188) routes by -- uint8[T][WP][32], bit r set: position 4*jp+r of the window equals its
 *    maximum, channel = last index (30 used), WP = ((F-30)/3+1)/4.
 *  - 1x1 score net (DCS_ARCH_BACH10_SCORE_1X1): one gate code 2*relu'(pre) in {0, 1, 2} (1: pre-activation exactly 0,
 *    where Theano's relu = 0.5*(x+|x|) has derivative 0.5) per encoder activation of conv1..conv6, the layers one after
 *    the other, each uint8[rows][W_l][C_l] with W_0 = feat_size, W_l = (W_{l-1}-5)/2+1, C = 30, 50, 70, 100, 200, 200;
 *    rows = Tp for conv1..conv4, Tp-9 for conv5, Tp-18 for conv6, where Tp = max(T, (P-1)*step + time_context) frames
 *    are the ones the P patches span (row r of patch k is frame k*step + r). */
int dcs_set_pool_tap(dcs_ctx* ctx, uint8_t* d_bits, int64_t capacity);

/* Multichannel Wiener post-filter of two-channel stems (see dcs_wiener_stereo): while iterations > 0, the entry points
 * that produce stereo stems -- dcs_separate_audio_keep_channels, dcs_separate_batch_pcm16_keep_channels_host and
 * dcs_separate_audio_stereo -- run that many EM iterations on the network's spectra before the inverse STFT (the
 * spectrum tap then holds the filtered spectra).  Single-channel entry points ignore the setting, and so does
 * dcs_separate_audio_channels: its filtered form, for 2 to 8 channels, is dcs_separate_audio_channels_wiener, which takes
 * the iterations as an argument.  Default 0 (off: the network's spectra, bit for bit); negative values are refused. */
int dcs_set_wiener(dcs_ctx* ctx, int iterations);
/* The covariance window of that filter on the same entry points (see dcs_wiener_stereo_windowed): 0 (the default) =
 * one R_j(f) and one scale for the whole clip, bit for bit the filter without this setting; radius >= 1 = per chunk
 * of DCS_WIENER_CHUNK_FRAMES frames, from the chunks within `radius` of it.  Negative values are refused. */
int dcs_set_wiener_radius(dcs_ctx* ctx, int radius);

/* per-stage device timing (CUDA events on the launching stream): enable, run, synchronise the
 * stream, then read.  dcs_profile_read writes up to max_n durations (ms) and the stage names
 * joined by '\n' into names_buf, clears the records and returns the number of records. */
int dcs_profile(dcs_ctx* ctx, int enable);
int dcs_profile_read(dcs_ctx* ctx, char* names_buf, int names_len, float* ms, int max_n);

/* ---- STFT / iSTFT: transform.py:277-396 (stft_norm / istft_norm), :224-274 ----------------- */
/* frame_size N in {256,512,1024,2048,4096}; hop even, hop <= N.
 * `window` = analysis window, `syn_window` = synthesis window (NULL: same), both host
 * double[N] (transformFFT passes window(frameSize) for both, transform.py:273). */
int dcs_stft_plan(dcs_ctx* ctx, int frame_size, int hop, const double* window,
                  const double* syn_window, dcs_stft** out);
int dcs_stft_plan_destroy(dcs_stft* plan);
/* T = ceil(L/hop) + 2            (transform.py:309) */
int64_t dcs_num_frames(int64_t num_samples, int hop);
/* F rounded up to a multiple of 8 */
int64_t dcs_padded_bins(int frame_size);

/* stft_norm (+ the |X|*scale/sqrt(N) of compute_file, transform.py:243-245, fused):
 * d_audio float[L] -> d_X complex[T][ldf] (may be NULL) and d_mag float[T][ldf] (may be NULL),
 * d_mag = mag_scale * |X| / sqrt(N).  Pad columns F..ldf-1 are written as zeros; F <= ldf <= F + 16.
 * d_X must be 8-byte aligned (DCS_EINVAL otherwise).  The imaginary parts of the DC and Nyquist bins are +0. */
int dcs_stft_forward(dcs_stft* plan, const float* d_audio, int64_t num_samples, dcs_complex* d_X,
                     float* d_mag, float mag_scale, int64_t ldf, void* stream);
/* same analysis, polar output: d_mag = mag_scale*|X|/sqrt(N), d_phase = angle(X)  (compute_file
 * with phase=True, transform.py:243-247) */
int dcs_stft_forward_polar(dcs_stft* plan, const float* d_audio, int64_t num_samples, float* d_mag,
                           float* d_phase, float mag_scale, int64_t ldf, void* stream);
/* istft_norm for nsrc spectrograms d_S complex[nsrc][T][ldf] (source stride src_stride elements)
 * -> d_out float[nsrc][out_stride], the first num_out samples of each (= data[:L],
 * separate_dsd.py:305-306; num_out <= (T-1)*hop + N - N/2).  Imaginary parts of the DC and
 * Nyquist bins are ignored like np.fft.irfft does: they are never read into the result, so they
 * may hold anything, NaN included; so may the pad columns F..ldf-1 and the gaps between sources.
 * Refused with DCS_EINVAL before anything is queued: ldf < N/2 + 1, a negative stride, d_S not
 * 8-byte aligned, and with nsrc > 1 src_stride < T*ldf or out_stride < num_out (sources that
 * share spectrum rows or output samples). */
int dcs_istft(dcs_stft* plan, const dcs_complex* d_S, int nsrc, int64_t num_frames, int64_t ldf,
              int64_t src_stride, float* d_out, int64_t num_out, int64_t out_stride, void* stream);
/* compute_inverse (transform.py:271-273): X = mag_scale*sqrt(N)*mag*exp(j*phase) -> istft_norm;
 * ldf < N/2 + 1 is DCS_EINVAL */
int dcs_istft_polar(dcs_stft* plan, dcs_ctx* ctx, const float* d_mag, const float* d_phase,
                    float mag_scale, int64_t num_frames, int64_t ldf, float* d_out, int64_t num_out,
                    void* stream);

/* ---- model: load_model + build_ca + set_all_param_values (separate_dsd.py:17-21,246-250) --- */
/* `h_params[i]` = the i-th array of the pickled `lasagne.layers.get_all_param_values(net)` list
 * (float32, C order), `shapes` = nparams x 4 int64 (unused dims = 1), `ndims[i]` = its rank.
 * Weights are re-laid-out for the kernels and uploaded once. */
int dcs_model_create(dcs_ctx* ctx, int arch, int feat_size, int time_context, int nparams,
                     const float* const* h_params, const int64_t* shapes, const int* ndims,
                     dcs_model** out);
int dcs_model_destroy(dcs_model* model);
int dcs_model_nsources(const dcs_model* model);
/* number of patches either patcher cuts from T frames */
int64_t dcs_num_patches(int64_t num_frames, int time_context, int overlap, int patcher);

/* ---- the separation graph on spectrograms ------------------------------------------------ */
/* generate_overlapadd -> predict_function2 (network + soft mask) -> overlapadd[_multi] ->
 * magnitude/scale * exp(j*phase), i.e. separate_dsd.py:292-304, with every per-patch tensor kept
 * on chip: d_mag float[T][ldf] (the scaled magnitude the network sees), d_X complex[T][ldf] (the
 * mixture STFT) -> d_S complex[nsrc][T][ldf] = blended mask_s * X (SURVEY.md App. A.1). */
int dcs_separate_spec(dcs_ctx* ctx, dcs_model* model, const float* d_mag, const dcs_complex* d_X,
                      int64_t num_frames, int64_t ldf, int overlap, int patcher, dcs_complex* d_S,
                      int64_t src_stride, void* stream);

/* Score-informed Bach10 (examples/bach10_scoreinformed/trainCNNrwc.py:357-416): the network sees 4
 * input channels in_ch = filter_ch * scaled magnitude, where filter_ch[T][F] are the normalised
 * harmonic masks derived from the scores on the host (LargeDatasetMask2.filterSpec,
 * dataset.py:839-879; deepconvsep_b200/score.py).  d_in: 4 planes [T][ldf], plane stride in_plane. */
int dcs_separate_spec_channels(dcs_ctx* ctx, dcs_model* model, const float* d_in, int64_t in_plane,
                               const dcs_complex* d_X, int64_t num_frames, int64_t ldf, int overlap,
                               int patcher, dcs_complex* d_S, int64_t src_stride, void* stream);
/* whole path on device buffers: d_filters float[4][T][ldf] (ldf = dcs_padded_bins(N), pad columns
 * arbitrary), d_audio float[L] -> d_stems float[4][stem_stride].  Like every separation entry point it checks
 * its arguments (overlap in [0, time_context) included) before anything is queued. */
int dcs_separate_audio_score(dcs_ctx* ctx, dcs_model* model, dcs_stft* plan, const float* d_audio,
                             int64_t num_samples, const float* d_filters, float scale_factor, int overlap,
                             int patcher, float* d_stems, int64_t stem_stride, void* stream);

/* Score filters from the note table, rasterised on the device (filterSpec(mag, melody, start, start + T),
 * dataset.py:839-862, bit for bit).  h_melody: the reference's `melody` as it is, HOST float64
 * [ninst][nnotes][ncols] (ninst 1..4, ncols >= 3): per row the first frame n0, the last frame n1 (exclusive), the
 * MIDI number, then (ncols-3)/2 (lo, hi) bin pairs.  A row sounds when its MIDI number is > 0 (NaN, the '?' note, is
 * not) and max(0, min(n1, stop) - max(n0, start)) > 0 in double; it covers frames int(max(n0, start)) - start ..
 * int(min(n1, stop)) - start (exclusive; int = C truncation) and the bins int(lo) .. int(hi) (exclusive) of every pair
 * with hi > 0.  Bins of sounding notes are 1, the others float(1e-18); filter_j = v_j / (((v_0 + v_1) + v_2) + v_3)
 * in fp32 with IEEE division.  Frame t of the output is frame start + t of the whole-clip filters.
 * Every row with a MIDI number > 0, whatever the window, is checked before anything is queued, and the call fails
 * with DCS_EINVAL where numpy would wrap or raise: a non-finite frame or bin, or a non-empty bin range reaching below
 * 0 or above F.
 * d_mag NULL (filters mode): d_out + j * plane = filter_j [T][ldf]; d_mag float[T][ldf] (channels mode): filter_j * mag.
 * Pad columns F..ldf-1 are written as 0.  The compacted table goes through a pinned staging buffer of the ctx (an
 * event guards its reuse) into a ctx workspace buffer; the stream is not synchronised. */
int dcs_score_filters(dcs_ctx* ctx, const double* h_melody, int ninst, int nnotes, int ncols, int64_t start,
                      int64_t num_frames, int F, const float* d_mag, int64_t ldf, float* d_out, int64_t plane,
                      void* stream);
/* dcs_separate_audio_score with the filter planes replaced by the note table (the model's 4 input planes = 4
 * instruments, h_melody [4][nnotes][ncols] as in dcs_score_filters): the filters are rasterised times the scaled
 * magnitude straight into the network's input channels, so no filter plane is read or written.  The clip's first STFT
 * frame is table frame frame0 (0 for a whole clip; a segment of a longer recording starting at sample frame0 * hop
 * passes frame0).  Same stems, spectrum tap and launch count as dcs_separate_audio_score on
 * filterSpec(..., frame0, frame0 + T); the table is validated with the other arguments before anything is queued. */
int dcs_separate_audio_notes(dcs_ctx* ctx, dcs_model* model, dcs_stft* plan, const float* d_audio,
                             int64_t num_samples, const double* h_melody, int nnotes, int ncols, int64_t frame0,
                             float scale_factor, int overlap, int patcher, float* d_stems, int64_t stem_stride,
                             void* stream);

/* ---- building block: the dense layer / im2col-free convolution GEMM ------------------------ */
/* d_C[M][ldc] = act(d_A[M][lda] * h_B[K][ldb] (+ h_bias[N])), fp32 in / fp32 out.  The weight is a
 * HOST array (it is transposed, padded and split for the tensor cores on the fly -- the models
 * do that once at load time).  engine 1: wgmma tf32 with the 3xTF32 split (the product
 * path); engine 0: exact-fp32 FFMA kernel (bring-up cross-check).  lasagne DenseLayer
 * (separate_dsd.py:206-221) is this with relu=1.  Synchronises the stream before returning. */
int dcs_gemm_f32(dcs_ctx* ctx, int engine, const float* d_A, int64_t lda, const float* h_B, int64_t ldb,
                 const float* h_bias, float* d_C, int64_t ldc, int M, int N, int K, int relu, void* stream);

/* Bring-up and test entry: the same GEMM on an arbitrary operand view -- the descriptor through which every layer of
 * every network reaches the kernels, field for field.  Its layout follows DCS_VERSION and may change with it.
 *   A row m      = (m / m_inner) * a_so + ((m % m_inner) / m_inner2) * a_si + (m % m_inner2) * a_s2; rows
 *                  >= a_valid_rows read as zeros
 *   A column k   = (k / k_seg) * k_ss + (k % k_seg)
 *   C row m      = the same three-level form with cm_inner, c_so, c_si, cm_inner2, c_s2; every stride and c_col0
 *                  must be >= 0
 *   C column n   = c_col0 + (n / n_seg) * n_ss + (n % n_seg)
 *   kc_*         K clipping of a transposed convolution on a zero-padded A (kc_rows = 0: off): rows are grouped by
 *                  u = m / kc_rows, and K block kc_unit * q (tap q) is skipped where kc_pad <= u + q < kc_pad + kc_n
 *                  fails.  The skipped products must be zeros of A.
 *   epi          0: C = act(A B + bias), relu selects the ReLU;  DCS_GEMM_EPI_POST: x = relu(AB + bias) + bias2 and,
 *                  with `code`, code[m * N + n] = 2 relu'(AB + bias) in {0, 1 (exactly 0), 2};  DCS_GEMM_EPI_GATE:
 *                  x *= 0.5 * gate[(m / g_inner) * g_so + ((m % g_inner) / g_inner2) * g_si + (m % g_inner2) * g_s2 + n],
 *                  and nothing is stored where (m % g_inner2) * g_s2 + n >= g_lim.
 * Pointers are device memory except `B`, which is ignored: the weight is the HOST array h_B[K][ldb], uploaded (engine 0,
 * the FFMA kernel) or transposed and split for the tensor cores (engine 1) on every call.  The epilogues need engine
 * 1 and a 16-byte aligned A view.  Synchronises the stream before returning. */
typedef struct {
  const float* A; const float* B; const float* bias; float* C;
  int M, N, K;
  int a_valid_rows;
  int m_inner; int64_t a_so, a_si;
  int m_inner2; int64_t a_s2;
  int k_seg; int64_t k_ss;
  int64_t ldb;
  int cm_inner; int64_t c_so, c_si;
  int cm_inner2; int64_t c_s2;
  int n_seg; int64_t n_ss, c_col0;
  int relu;
  int kc_rows, kc_unit, kc_pad, kc_n, kc_taps;
  const float* bias2; uint8_t* code;
  const uint8_t* gate; int g_inner, g_inner2; int64_t g_so, g_si, g_s2, g_lim;
} dcs_gemm_view;
enum { DCS_GEMM_EPI_POST = 1, DCS_GEMM_EPI_GATE = 2 };
int dcs_gemm_view_f32(dcs_ctx* ctx, int engine, int epi, const dcs_gemm_view* view, const float* h_B, void* stream);

/* Bring-up and test entries: the fused last stage of the networks -- InverseLayer(conv1) + output bias + ReLU + soft
 * ratio mask + sequential patch cross-fade + times the mixture STFT -- on one argument set, field for field the one
 * the layer sequence passes to the kernels.  Layouts follow DCS_VERSION and may change with it.  Every pointer is
 * device memory, weights included, in the kernels' own layouts.  engine 1: the wgmma kernel; engine 0: its FFMA twin.
 * Every argument is checked before anything is queued; a shape the chosen engine does not take is DCS_EINVAL with
 * nothing launched (there is no switch to the other engine).  Synchronises the stream before returning.
 *
 * DSD100 / hiphopss (ndec 3) and stereo / ILD (ndec 4, one call per input channel):
 *   G     [P][ndec][tc][ldg]  decoder activations after InverseLayer(conv2); columns 0..49 are the 50 conv1 filters
 *   W1t   [50][ldw]           W1t[c][b] = conv1.W[c, ch, 0, F-1-b] for bins b < F
 *   bout  [4]                 output biases (ndec 3: source 4 is decoder 2 with bias 4; all-zero bins get 1/4 each;
 *                             ndec 4: one decoder per source, all-zero bins get 0)
 *   X     complex [T][ldf];  S complex [4][T][ldf], source s at S + s * src_stride
 *   patch k covers frames [k*(tc-overlap), k*(tc-overlap) + tc); frames no patch covers get S = 0.
 *   engine 1 takes at most 6 patches per frame, ldg >= 52 with ldg % 4 == 0 and a 16-byte aligned G.
 *   Pad elements read: engine 1 multiplies G columns 50..51 by zero W1t rows, so they must be finite.  No other pad
 *   element (G columns >= 52, W1t columns >= F, X / S columns >= F) is read.
 */
typedef struct {
  const float* G; int ldg;
  const float* W1t; int ldw;
  const float* bout;
  const dcs_complex* X;
  dcs_complex* S;
  int64_t ldf, src_stride;
  int T, P, tc, overlap, F;
  int ndec;
} dcs_dsd_mask_view;
int dcs_dsd_mask_f32(dcs_ctx* ctx, int engine, const dcs_dsd_mask_view* view, void* stream);

/* Bring-up and test entry: InverseLayer(conv2) of the DSD nets on the tensor cores, on buffers laid out as the layer
 * sequence lays them out, for npairs = P * ndec (patch, decoder) pairs, time_context tc in 4..64, kh2 = tc / 2,
 * h2 = tc - kh2 + 1:
 *   apad  [npairs][h2 + 2 (kh2 - 1)][52]  decoder activations; only the h2 interior rows kh2 - 1 .. kh2 + h2 - 2 are
 *                                        read (channels 50..51 meet zero weights and must be finite); 16-byte aligned
 *   G     [npairs][tc][ldg]              G[i][u][c] = sum_{q < kh2, f < 52} apad[i][u + q][f] * h_Wt2[52 q + f][c];
 *                                        columns 0..49 are written, nothing else; ldg >= 50 even, 8-byte aligned
 *   h_Wt2 HOST [52 kh2][50]              transposed and split for the tensor cores on every call
 * Every argument is checked before anything is queued.  Synchronises the stream before returning. */
typedef struct {
  const float* apad;
  float* G; int ldg;
  int npairs, tc;
} dcs_dsd_convt2_view;
int dcs_dsd_convt2_f32(dcs_ctx* ctx, const dcs_dsd_convt2_view* view, const float* h_Wt2, void* stream);

/* Bring-up and test entry: the decoder dense layers of the DSD nets on the tensor cores, on buffers laid out as the
 * layer sequence lays them out, for P patches, ndec 3 or 4 decoders, time_context tc in 4..64, kh2 = tc / 2,
 * h2 = tc - kh2 + 1, bottleneck width nfc (a multiple of 32, at most 256), N = ndec * h2 * 52:
 *   z     [P][nfc]                            bottleneck activations; 4-byte aligned
 *   bias  [N]                                 device memory; 4-byte aligned
 *   apad  [P][ndec][h2 + 2 (kh2 - 1)][52]     apad[k][d][kh2 - 1 + i][c] = ReLU(z[k] . h_W[:, n] + bias[n]) with
 *                                            n = (d h2 + i) 52 + c; only these interior rows are written; 8-byte aligned
 *   h_W   HOST [w_rows][w_cols] = [nfc][N]    transposed and split for the tensor cores on every call
 * Every argument is checked before anything is queued.  Synchronises the stream before returning. */
typedef struct {
  const float* z;
  const float* bias;
  float* apad;
  int P, tc, ndec, nfc;
} dcs_dsd_dense_view;
int dcs_dsd_dense_f32(dcs_ctx* ctx, const dcs_dsd_dense_view* view, const float* h_W, int w_rows, int w_cols, void* stream);

/* The strided-conv1 networks (K3s): arch DCS_ARCH_BACH10, _BACH10_SCORE, _BACH10_SCORE_1X1, _IKALA, _IKALA_NOPOOL.
 * conv1 has KW taps at stride STRIDE over frequency (Bach10 nets 30 / 4, iKala 30 / 3, build_ca_1x1 5 / 2); J = (F-KW) /
 * STRIDE + 1 windows, WP = J / 4 pooled windows (DCS_ARCH_IKALA) or J; ND = ceil(KW / STRIDE).
 *   G     [P'][ndec][tc][WP][32] decoder activations, 30 channels of 32 (ndec: Bach10 4, iKala 2, score-informed 1);
 *         G holds patches p_base.. (P' = P - p_base)
 *   tie   [T][WP][32] (DCS_ARCH_IKALA only, else NULL): bit r of frame t, window jp, channel f set where position
 *         4*jp + r held the window maximum in the forward pass; InverseLayer(pool) routes the value to every set bit
 *   W     float4 [NW][ND][32]: W[o][dd][f][r] = conv1.W[f][o][0][KW-1-r-STRIDE*dd], one bank per source o for the
 *         score-informed nets (NW = 4), one bank otherwise (NW = 1)
 *   bout  [nsrc];  X complex [T][ldf];  S complex [nsrc][T][ldf], source s at S + s * src_stride
 *   frames [t0, t1) are written (build_ca_1x1 decodes in chunks; every other arch needs p_base = 0, t0 = 0, t1 = T);
 *   frames no patch covers get S = 0.  engine 1 needs a 16-byte aligned G and a 4-byte aligned tie.
 *   Pad elements read: both engines multiply the filter-bank entries whose tap index KW-1-r-STRIDE*dd is negative
 *   (r < STRIDE), and engine 1 multiplies G channels 30..31 by W channels 30..31: those weights must be zero and the
 *   activations finite.  No other pad element (components r >= STRIDE of W, X / S columns >= F) is read.
 */
typedef struct {
  int arch;
  const float* G;
  const uint8_t* tie;
  const float* W;
  const float* bout;
  const dcs_complex* X;
  dcs_complex* S;
  int64_t ldf, src_stride;
  int T, P, tc, overlap, F, J, WP;
  int p_base, t0, t1;
} dcs_sconv_mask_view;
int dcs_sconv_mask_f32(dcs_ctx* ctx, int engine, const dcs_sconv_mask_view* view, void* stream);

/* ---- stereo / ILD variant (examples/dsd100_2ch_ILD/trainCNN_ILD_DSD100.py:299-327) ------------ */
/* d_audio float[2][audio_stride] (left, right; first num_samples valid) ->
 * d_stems float[nsrc*2][stem_stride], plane (s*2 + j) = source s, channel j (`sep_audio[:, s, j]`).
 * One STFT per channel, both scaled magnitudes into the network, per-channel masks normalised over
 * the sources (:183-186), per-channel cross-fade, iSTFT with that channel's mixture phase. */
int dcs_separate_audio_stereo(dcs_ctx* ctx, dcs_model* model, dcs_stft* plan, const float* d_audio,
                              int64_t audio_stride, int64_t num_samples, float scale_factor, int overlap,
                              int patcher, float* d_stems, int64_t stem_stride, void* stream);

/* ---- evaluation: BSS-Eval 3.0 correlation lags (SURVEY.md 8(f) row 3) ------------------------ */
/* The O(num_samples) part of evaluation/bss_eval/bss_eval_sources.m: the inner products between
 * delayed copies of the true sources (:120-136) and between them and an estimate (:138-145), which
 * the reference takes from FFT cross-correlations and of which only lags |m| < flen (512) are used.
 * For each pair p of float device signals of num_samples samples:
 *     h_out[p][li] = sum_t a_p[t + li - (flen-1)] * b_p[t],   li = 0 .. 2*flen-2      (float64)
 * h_a / h_b: HOST arrays of npairs DEVICE pointers; h_out: HOST double[npairs][2*flen-1].
 * flen <= 512.  Deterministic (fixed summation order).  Synchronises the stream. */
int dcs_xcorr_lags(dcs_ctx* ctx, const float* const* h_a, const float* const* h_b, int npairs,
                   int64_t num_samples, int flen, double* h_out, void* stream);

/* ---- whole train_auto() on device buffers (separate_dsd.py:289-306) ----------------------- */
/* d_audio float[L] mono in [-1,1] -> d_stems float[nsrc][stem_stride] (first L samples valid) */
int dcs_separate_audio(dcs_ctx* ctx, dcs_model* model, dcs_stft* plan, const float* d_audio,
                       int64_t num_samples, float scale_factor, int overlap, int patcher,
                       float* d_stems, int64_t stem_stride, void* stream);
/* same with HOST buffers: H2D copy of the audio, pipeline, D2H copy of the stems, then
 * cudaStreamSynchronize.  Pinned host memory makes the copies asynchronous. */
int dcs_separate_host(dcs_ctx* ctx, dcs_model* model, dcs_stft* plan, const float* h_audio,
                      int64_t num_samples, float scale_factor, int overlap, int patcher,
                      float* h_stems, int64_t stem_stride, void* stream);
/* int16 PCM in / int16 PCM out, the wav-file contract of train_auto (separate_dsd.py:275-287,
 * 307-309): h_pcm int16[L][channels] interleaved; mono = (L+R)/2/32767 (downmix 1) or (L+R)/32767
 * (downmix 2, iKala separate_ikala.py:229) or channel 0 (channels == 1);
 * h_out int16[nsrc][out_stride] = (int16)(stem*32767) (C truncation, no clipping, as astype does).
 * The int16 encode of every entry point, exactly: v = stem * 32767.0f in fp32, truncated toward zero, then reduced
 * modulo 2^16 into [-32768, 32767] -- a stem past full scale wraps (1.5 gives -16386), as numpy's
 * (stem * maxn).astype('int16') does for |v| < 2^31.  NaN gives 0.  Beyond that the truncation saturates to int32
 * first: v >= 2^31 and +inf give -1, v < -2^31 and -inf give 0 (numpy's result there depends on the platform). */
int dcs_separate_pcm16_host(dcs_ctx* ctx, dcs_model* model, dcs_stft* plan, const int16_t* h_pcm,
                            int64_t num_samples, int channels, int downmix, float scale_factor,
                            int overlap, int patcher, int16_t* h_out, int64_t out_stride,
                            void* stream);

/* Multi-clip scheduler: `nclips` clips through one context as a pipeline -- H2D of clip i+1 | kernels of clip i | D2H of
 * clip i-1 -- on two internal copy streams and `stream`, with double-buffered int16 staging on the device.  Replaces the
 * reference's process-per-file loop (examples/dsd100/separate_multiple.ipynb cell 3); per clip the contract is that of
 * dcs_separate_pcm16_host.  h_pcm[i]: int16[num_samples[i]][channels] (pinned for real overlap), h_out[i]:
 * int16[nsrc][out_strides[i]].  Order the clips longest first if their lengths differ much (grow-only workspace).
 * Synchronises before returning -- also when it returns an error: every copy in flight has drained, so the host
 * buffers are the caller's again (outputs of clips after the failure are undefined).  Every argument is checked
 * before anything is queued: buffers and lengths of each clip (DCS_EINVAL names the offending clip), the plan's
 * N/2+1 against the model's bins, overlap in [0, time_context), the patcher, and a single-channel architecture. */
int dcs_separate_batch_pcm16_host(dcs_ctx* ctx, dcs_model* model, dcs_stft* plan, int nclips,
                                  const int16_t* const* h_pcm, const int64_t* num_samples, int channels, int downmix,
                                  float scale_factor, int overlap, int patcher, int16_t* const* h_out,
                                  const int64_t* out_strides, void* stream);

/* ---- keep-channels mode of the DSD100 / hiphopss network (DCS_ARCH_DSD only) ------------------------------ */
/* Stereo stems from the mono network: the network sees the downmix mono = (l + r) * 0.5f (fp32, the downmix 1 of
 * dcs_separate_pcm16_host), so its blended soft masks M_s are those of the mono call (separate_dsd.py:282-304); each
 * is applied to the STFT X_c of channel c and inverted with that channel's phase: plane (s*2 + c) = iSTFT(M_s * X_c).
 * With l == r every channel equals the mono call's stem; (stem_L + stem_R) / 2 equals it up to STFT rounding.
 * d_audio float[2][audio_stride] (left, right; first num_samples valid) -> d_stems float[nsrc*2][stem_stride], plane
 * (s*2 + c) = source s, channel c (the layout of dcs_separate_audio_stereo).  This is dcs_separate_audio_channels at
 * nx = 2, bit for bit, with the same workspace, and with the Wiener post-filter (dcs_set_wiener) in addition: its first
 * pass forms the masked spectra M_s * X_c (fp32, componentwise) in memory, filters them and inverts them.  Other
 * architectures are refused before anything is queued (the stereo / ILD net: dcs_separate_audio_stereo).  With the
 * filter on, the spectrum tap holds the nsrc*2 filtered planes ordered (source, channel); with it off, a spectrum tap is
 * refused before anything is queued. */
int dcs_separate_audio_keep_channels(dcs_ctx* ctx, dcs_model* model, dcs_stft* plan, const float* d_audio,
                                     int64_t audio_stride, int64_t num_samples, float scale_factor, int overlap,
                                     int patcher, float* d_stems, int64_t stem_stride, void* stream);
/* the same on int16 stereo clips through the multi-clip scheduler of dcs_separate_batch_pcm16_host:
 * h_pcm[i] int16[num_samples[i]][2] -> h_out[i] + s*2*out_strides[i] = source s as int16 [num_samples[i]][2]
 * interleaved (what util.writeAudioScipy writes for a 2-channel stem, util.py:56-58), (int16)(stem*32767) per
 * sample as in dcs_separate_pcm16_host.  Channels are decoded as pcm/32767 (fp32) and downmixed as above. */
int dcs_separate_batch_pcm16_keep_channels_host(dcs_ctx* ctx, dcs_model* model, dcs_stft* plan, int nclips,
                                                const int16_t* const* h_pcm, const int64_t* num_samples,
                                                float scale_factor, int overlap, int patcher, int16_t* const* h_out,
                                                const int64_t* out_strides, void* stream);

/* ---- masks output: the network's blended soft masks, from a pipeline that stops before the iSTFT ----------------- */
/* The soft masks M_s[t, f] every separation entry point computes and multiplies by the mixture STFT: the ratio masks of
 * each patch, cross-faded over the patches (overlapadd_multi, separate_dsd.py:139-169) -- the same fp32 values, bit for
 * bit, that the stems path multiplies by X, so  iSTFT(X * M_s)  (dcs_stft_forward, the product componentwise in fp32,
 * dcs_istft) is the stem of the matching dcs_separate_audio* call.  The masks of a downmix (l + r) * 0.5f applied to
 * each channel's STFT are the keep-channels mode.  Each entry point mirrors the stems call named beside it, with the same
 * checks, and writes d_masks float[nplanes][T][ldf], T = dcs_num_frames(num_samples, hop), ldf = dcs_padded_bins(N),
 * planes m_stride (>= T * ldf) apart: nplanes = nsrc, or nsrc x 2 ordered (source, channel) for the stereo / ILD net.
 * Only bins f < F of each frame are written: the pad columns F..ldf-1 and the gaps between planes keep their contents.
 *  - The forward STFT writes the magnitude only; there is no Wiener pass (dcs_set_wiener is ignored), no spectrum tap
 *    and no inverse STFT, and the workspace holds neither the mixture STFT nor the masked spectra.
 *  - The routing tap (dcs_set_pool_tap) is honoured as by the stems calls.
 *  - A clip shorter than one patch gives all-zero masks.
 *  - Refused with DCS_EINVAL before anything is queued: an architecture the entry point does not serve, a NULL pointer,
 *    a plan whose N/2+1 is not the model's F, m_stride < T * ldf, a misaligned d_masks, and what the mirrored stems call
 *    refuses (lengths, strides, overlap, patcher, the note table). */
/* dcs_separate_audio (single-channel nets: d_audio float[L], audio_stride >= L) and dcs_separate_audio_stereo (stereo /
 * ILD net: d_audio float[2][audio_stride]) */
int dcs_separate_masks(dcs_ctx* ctx, dcs_model* model, dcs_stft* plan, const float* d_audio, int64_t audio_stride,
                       int64_t num_samples, float scale_factor, int overlap, int patcher, float* d_masks,
                       int64_t m_stride, void* stream);
/* dcs_separate_audio_score: the score-informed nets with the filter planes d_filters float[4][T][ldf] */
int dcs_separate_masks_score(dcs_ctx* ctx, dcs_model* model, dcs_stft* plan, const float* d_audio,
                             int64_t num_samples, const float* d_filters, float scale_factor, int overlap,
                             int patcher, float* d_masks, int64_t m_stride, void* stream);
/* dcs_separate_audio_notes: the score-informed nets with the note table h_melody (HOST) from table frame frame0 */
int dcs_separate_masks_notes(dcs_ctx* ctx, dcs_model* model, dcs_stft* plan, const float* d_audio,
                             int64_t num_samples, const double* h_melody, int nnotes, int ncols, int64_t frame0,
                             float scale_factor, int overlap, int patcher, float* d_masks, int64_t m_stride,
                             void* stream);

/* ---- masks applied to any number of channels: stems for 5.1, microphone arrays, edited masks ------------------------ */
/* istft_norm(M_s * X_c): d_X complex[nx][T][ldf] (x_plane apart), d_M float[nsrc][T][ldf] (m_stride apart, same ldf)
 * -> d_out float[nsrc*nx][out_stride], plane (s*nx + c), the first num_out samples of each; the product is formed
 * componentwise in fp32 as a spectrum row is loaded -- make_float2(m * x.x, m * x.y), the expression of the mask kernels
 * -- so no masked spectrum is ever in memory and the samples are, bit for bit, those of dcs_istft on that product.  The
 * groups of the nsrc sources that walk the same frames of one channel are launched next to each other, so that their X
 * rows are shared through L2 rather than fetched nsrc times (an ordering, not a guarantee).
 * Never read into the result, so free to hold anything, NaN included: Im of the DC and Nyquist bins of d_X, the pad
 * columns F..ldf-1 of d_X and of d_M (dcs_separate_masks* leaves them unwritten), the gaps between planes.
 * Refused with DCS_EINVAL before anything is queued: a NULL pointer, num_frames <= 0, nx outside [1, 16], nsrc < 1,
 * ldf < N/2 + 1, a negative stride, x_plane < T*ldf with nx > 1, m_stride < T*ldf with nsrc > 1, out_stride < num_out
 * with more than one output plane, num_out > (T-1)*hop + N - N/2, d_X not 8-byte or d_M not 4-byte aligned. */
int dcs_istft_masked(dcs_stft* plan, const dcs_complex* d_X, int nx, int64_t x_plane, const float* d_M, int nsrc,
                     int64_t m_stride, int64_t num_frames, int64_t ldf, float* d_out, int64_t num_out,
                     int64_t out_stride, void* stream);
/* The caller's masks (from dcs_separate_masks*, edited or not) applied to nx audio channels: d_audio float[nx][audio_stride]
 * (first num_samples valid), d_masks float[nsrc][T][ldf] (T = dcs_num_frames(num_samples, hop), ldf = dcs_padded_bins(N),
 * m_stride >= T*ldf apart) -> d_stems float[nsrc*nx][stem_stride], plane (s*nx + c) = iSTFT(M_s * STFT(channel c)).
 * Per channel one X-only forward STFT into ONE workspace plane, then dcs_istft_masked for its nsrc planes: the workspace
 * does not depend on nx.  nsrc is the caller's (>= 1), with no link to a model.  Refused with DCS_EINVAL before anything
 * is queued: a NULL pointer, nx outside [1, 16], nsrc < 1, num_samples <= 0, audio_stride or stem_stride < num_samples,
 * m_stride < T*ldf, a misaligned d_masks. */
int dcs_apply_masks(dcs_ctx* ctx, dcs_stft* plan, const float* d_audio, int nx, int64_t audio_stride,
                    int64_t num_samples, const float* d_masks, int nsrc, int64_t m_stride, float* d_stems,
                    int64_t stem_stride, void* stream);
/* Stems for nx channels from a single-channel network (every architecture but the stereo / ILD and score-informed nets,
 * which are refused with a message naming dcs_separate_masks* + dcs_apply_masks): the network sees the downmix
 * (((a_0 + a_1) + a_2) + ...) * (1.0f / nx) in fp32 -- (l + r) * 0.5f at nx = 2, the channel itself at nx = 1 -- and its
 * blended masks, bit for bit those dcs_separate_masks returns for that downmix, go to every channel as in
 * dcs_apply_masks.  d_audio float[nx][audio_stride] -> d_stems float[nsrc*nx][stem_stride], plane (s*nx + c).  At nx = 1
 * the stems are those of dcs_separate_audio and at nx = 2 (DCS_ARCH_DSD) those of dcs_separate_audio_keep_channels,
 * bit for bit.  The workspace holds the downmix, its magnitude, nsrc float mask planes and one mixture STFT plane: no
 * masked spectra, and nothing that grows with nx.
 *  - dcs_set_wiener is ignored, as by the masks calls: the Wiener post-filter on these stems is
 *    dcs_separate_audio_channels_wiener, which takes its iterations and radius as arguments.
 *  - There are no masked spectra to copy: a spectrum tap set on the ctx is DCS_EINVAL before anything is queued.  The
 *    routing tap (dcs_set_pool_tap) is honoured as by the masks calls.
 *  - A clip shorter than one patch gives all-zero masks, so silent stems.
 *  - Refused with DCS_EINVAL before anything is queued: nx outside [1, 16] and what dcs_separate_audio refuses. */
int dcs_separate_audio_channels(dcs_ctx* ctx, dcs_model* model, dcs_stft* plan, const float* d_audio, int nx,
                                int64_t audio_stride, int64_t num_samples, float scale_factor, int overlap,
                                int patcher, float* d_stems, int64_t stem_stride, void* stream);

/* ---- multichannel Wiener filter with EM spatial covariances (Duong, Vincent & Gribonval 2010; util.py:633-719) -- */
/* In place on caller-owned spectra, the plane layout of the stereo entry points: mixture channel c at d_X + c*x_plane,
 * stem (source j, channel c) at d_S + (2j + c)*src_stride, each complex[T][ldf]; only bins f < F are read or written.
 * With s = max(1, max|x| / 10) over the clip and eps = 2^-23, each iteration computes
 *     v_j = (|y_jL|^2 + |y_jR|^2) / 2,   R_j(f) = sum_t y_j y_j^H / (eps s^2 + sum_t v_j),
 *     C = sum_j v_j R_j + sqrt(eps) s^2 I,   y_j <- v_j R_j C^-1 x
 * (2x2 algebra and the sums over t in fp64, fixed summation order: the same bits on every run).  Frames where every
 * y_j is 0 stay 0.  nsrc in [1, 4]; iterations 0 returns without queuing work.  Every argument is checked before
 * anything is queued.  The workspace grows to ~32 bytes per (source, bin) per 128 frames. */
int dcs_wiener_stereo(dcs_ctx* ctx, const dcs_complex* d_X, int64_t x_plane, dcs_complex* d_S, int64_t src_stride,
                      int nsrc, int64_t num_frames, int64_t ldf, int F, int iterations, void* stream);
/* The same with a sliding-window spatial covariance.  Chunk k is frames [128k, min(T, 128k + 128)) (128 =
 * DCS_WIENER_CHUNK_FRAMES), n chunks in all.  radius 0 is dcs_wiener_stereo, bit for bit.  radius W >= 1: chunk c's
 * window is chunks max(0, c-W) .. min(n-1, c+W), and for every frame of chunk c
 *     s_c = max(1, max|x| / 10) over the window's frames (both channels, bins < F),
 *     R_j(f; c) = sum_{t in window} y_j y_j^H / (eps s_c^2 + sum_{t in window} v_j),
 *     C = sum_j v_j R_j(f; c) + sqrt(eps) s_c^2 I,   y_j <- v_j R_j(f; c) C^-1 x.
 * Per-chunk sums run in frame order and each window adds them directly in ascending chunk order, so a chunk's filter
 * depends only on the frames within K*W chunks of it (K = iterations) and W >= n-1 gives the bits of radius 0.
 * Same launch count (2 * iterations + 1).  The workspace grows by one R and one scale per chunk (~32 bytes per
 * (source, bin) per chunk more).  A negative radius is refused with the other arguments before anything is queued. */
int dcs_wiener_stereo_windowed(dcs_ctx* ctx, const dcs_complex* d_X, int64_t x_plane, dcs_complex* d_S,
                               int64_t src_stride, int nsrc, int64_t num_frames, int64_t ldf, int F, int iterations,
                               int radius, void* stream);
/* The same filter on nx = 2 .. 8 channels: mixture channel c at d_X + c*x_plane, stem (source j, channel c) at
 * d_S + (j*nx + c)*src_stride (the stereo layout at nx = 2), in place, with the constants, chunks and windows of
 * dcs_wiener_stereo_windowed and C x C algebra:
 *     v_j = (1/nx) sum_c |y_jc|^2,   R_j(f) = sum_t y_j y_j^H / (eps s^2 + sum_t v_j),
 *     C = sum_j v_j R_j + sqrt(eps) s^2 I  (Hermitian, positive definite),   y_j <- v_j R_j C^-1 x,
 * s over every channel.  C is factored L D L^H without pivoting and solved by two triangular substitutions, in fp64, in
 * a fixed order of operations: the same bits on every run, W >= n-1 gives the bits of radius 0, and a chunk depends only
 * on the frames within K*W chunks of it.  nx = 2 runs the 2 x 2 kernels: the bytes of dcs_wiener_stereo_windowed.
 * Launch count 2 * iterations + 1.  The workspace (bytes) is
 *     8 * (n * P + q * P + n * ceil(F / b) + q),   P = nsrc * nx^2 * F,  q = (radius > 0 ? n : 1),  n = ceil(T / 128),
 * b = 128 at nx = 2 and 32 above: the per-chunk partial sums, the summed covariances, the per-block maxima and the scales.
 * Refused with DCS_EINVAL before anything is queued: nx outside [2, 8] (one channel has no spatial covariance) and what
 * dcs_wiener_stereo_windowed refuses. */
int dcs_wiener_channels(dcs_ctx* ctx, const dcs_complex* d_X, int nx, int64_t x_plane, dcs_complex* d_S,
                        int64_t src_stride, int nsrc, int64_t num_frames, int64_t ldf, int F, int iterations,
                        int radius, void* stream);
/* dcs_separate_audio_channels with the Wiener post-filter (dcs_wiener_channels) between the masks and the inverse STFT:
 * the filter's first pass forms the masked spectra M_s * X_c of every channel (fp32, componentwise, the product the
 * masked inverse STFT forms) in memory, `iterations` EM iterations over covariance windows of `radius` chunks filter
 * them, and the plain inverse STFT gives plane (s*nx + c).  The iterations and radius are arguments: dcs_set_wiener and
 * dcs_set_wiener_radius are not read.
 *  - iterations 0: the bits of dcs_separate_audio_channels, with its workspace and its refusal of a spectrum tap.
 *  - nx = 2, DCS_ARCH_DSD: the bits of dcs_separate_audio_keep_channels with the same iterations and radius set on the
 *    ctx.
 *  - iterations > 0: the spectrum tap holds the nsrc*nx filtered planes, ordered (source, channel).  The workspace adds
 *    to that of dcs_separate_audio_channels nx - 1 mixture STFT planes, nsrc*nx masked-spectrum planes (8 * T * ldf bytes
 *    each) and the filter's workspace of dcs_wiener_channels at F = N/2 + 1.
 *  - Refused with DCS_EINVAL before anything is queued: iterations or radius negative, nx outside [2, 8] with
 *    iterations > 0, and what dcs_separate_audio_channels refuses. */
int dcs_separate_audio_channels_wiener(dcs_ctx* ctx, dcs_model* model, dcs_stft* plan, const float* d_audio, int nx,
                                       int64_t audio_stride, int64_t num_samples, float scale_factor, int overlap,
                                       int patcher, int iterations, int radius, float* d_stems, int64_t stem_stride,
                                       void* stream);
/* C-channel int16 clips through the multi-clip scheduler of dcs_separate_batch_pcm16_host (5.1, 7.1, arrays of up to 16
 * channels): h_pcm[i] int16[num_samples[i]][channels] (pinned for real overlap) -> source s of clip i at
 * h_out[i] + s*channels*out_strides[i] as int16 [num_samples[i]][channels], interleaved (what scipy.io.wavfile.write
 * takes for a C-channel stem).  One launch decodes a clip into channels + 1 fp32 planes -- the downmix of
 * dcs_separate_audio_channels, then a_c = pcm/32767 per channel -- the clip is dcs_separate_audio_channels_wiener on
 * those planes with `iterations` and `radius` (dcs_set_wiener and dcs_set_wiener_radius are not read), and one launch
 * encodes its nsrc*channels stem planes as (int16)(int)(stem*32767) (C truncation, no clipping: wraps modulo 2^16 for
 * |stem*32767| < 2^31, NaN gives 0, saturating beyond, the encode of dcs_separate_pcm16_host).  Launches per clip: those of dcs_separate_audio_channels(_wiener) on the clip, plus one
 * (the decode forms the downmix in place of the downmix launch, and the encode is added).
 *  - channels = 1: the bytes of dcs_separate_batch_pcm16_host on the same clips (channels 1).
 *  - channels = 2, DCS_ARCH_DSD: the bytes of dcs_separate_batch_pcm16_keep_channels_host with the same iterations and
 *    radius set on the ctx.
 *  - any channels: per clip the bytes of (int16)(int)(stem*32767) on the stems of dcs_separate_audio_channels_wiener on
 *    the planes pcm/32767 (fp32).
 * With the filter on, the spectrum tap holds the last clip's nsrc*channels filtered planes; without it a tap is refused.
 * Workspace: every buffer is sized once from the longest clip, Lmax samples, before the pipeline starts.  With
 * B(x) = x rounded up to a multiple of 2^20 bytes and n = min(nclips, 2), a fresh ctx holds after the call
 *     W(Lmax) - B(4 Lmax) + B(4 (channels + 1) Lmax) + B(4 nsrc channels Lmax)
 *       + n B(2 channels Lmax) + n B(2 nsrc channels Lmax)
 * where W(Lmax) is what a fresh ctx holds after dcs_separate_audio_channels_wiener with the same iterations and radius
 * on one clip of Lmax samples: the fp32 staging of the audio planes replaces that call's downmix plane, and the stem
 * planes and the double-buffered int16 staging are added.
 * Synchronises before returning, also on an error (the copies in flight have drained).  Refused with DCS_EINVAL before
 * anything is queued: channels outside [1, 16], iterations or radius negative, iterations > 0 with channels outside
 * [2, 8], a NULL buffer, a non-positive length or out_strides[i] < num_samples[i] (the message names the clip), and what
 * dcs_separate_audio_channels_wiener refuses on the longest clip (the stereo / ILD and score-informed nets with a
 * message naming dcs_separate_masks*, a spectrum tap without the filter). */
int dcs_separate_batch_pcm16_channels_host(dcs_ctx* ctx, dcs_model* model, dcs_stft* plan, int nclips,
                                           const int16_t* const* h_pcm, const int64_t* num_samples, int channels,
                                           int iterations, int radius, float scale_factor, int overlap, int patcher,
                                           int16_t* const* h_out, const int64_t* out_strides, void* stream);

/* ---- polyphase resampling by up/down (scipy.signal.resample_poly, padtype='constant') -------------------------- */
/* The networks work on 44.1 kHz spectra; these take a recording at another rate to 44.1 kHz and its stems back.  The
 * reference has no counterpart: its scripts refuse such files (separate_dsd.py:313).
 * A resampler holds the polyphase bank of the caller's taps h[ntaps] (host double, already scaled by up, zero-phase about
 * half_len = (ntaps - 1)/2; scipy.signal.resample_poly designs firwin(2*10*max(up, down) + 1, 1/max(up, down),
 * window=('kaiser', 5.0)) * up).  The output is
 *     y[n] = sum_j x[j] * h[n*down + half_len - j*up],   0 <= j < num_in,   0 <= n*down + half_len - j*up < ntaps,
 * for n < num_out <= dcs_resampled_length(num_in, up, down): samples outside [0, num_in) are zeros.  The taps stay fp64 as
 * given, the fp32 input is widened exactly, the ceil(ntaps/up) products of an output are summed in fp64 in a fixed order
 * and rounded once to fp32: the same bits on every run.
 *  - Refused with DCS_EINVAL: up or down < 1 or not coprime, ntaps even or < 1, a bank (ceil(ntaps/up) * up doubles)
 *    over DCS_RESAMPLE_MAX_BANK_BYTES, a NULL argument.
 *  - The bank lives in the resampler (device memory of ctx's device) until dcs_resampler_destroy; the ctx's workspace
 *    does not change. */
#define DCS_RESAMPLE_MAX_BANK_BYTES (112 * 1024)
typedef struct dcs_resampler dcs_resampler;
int dcs_resampler_create(dcs_ctx* ctx, int up, int down, const double* h, int ntaps, dcs_resampler** out);
int dcs_resampler_destroy(dcs_resampler* resampler);
/* ceil(num_in * up / down); -1 for a negative num_in or up, down < 1 */
int64_t dcs_resampled_length(int64_t num_in, int up, int down);
/* nplanes planes: plane p of the input at d_in + p*in_stride (first num_in samples valid; nothing else is read), plane p
 * of the output at d_out + p*out_stride (num_out samples written).  A num_out shorter than the resampled length trims
 * the tail (the way back to a recording's own length).  One launch on `stream`.
 * Refused with DCS_EINVAL before anything is queued: a NULL pointer, nplanes < 1, num_in < 1, num_out < 1 or over
 * dcs_resampled_length, negative strides, strides shorter than the rows with nplanes > 1, planes not 4-byte aligned. */
int dcs_resample(dcs_resampler* resampler, const float* d_in, int nplanes, int64_t in_stride, int64_t num_in,
                 float* d_out, int64_t out_stride, int64_t num_out, void* stream);
/* dcs_separate_batch_pcm16_channels_host for clips at another rate (48 kHz film and broadcast material, 8 to 192 kHz):
 * to_model takes the clips' rate to the networks' 44.1 kHz and from_model brings the stems back, both made on ctx and
 * inverse (to_model up/down = from_model down/up).  Clip i of L = num_samples[i] samples is separated at
 * L' = dcs_resampled_length(L, to_model up, to_model down) samples and its stems come back at L, in the layout of
 * dcs_separate_batch_pcm16_channels_host.  One launch resamples and decodes a clip into channels + 1 fp32 planes of L'
 * samples -- channel c is the bits of dcs_resample(to_model) on the plane pcm_c/32767 (fp32), the downmix is
 * dcs_separate_audio_channels' on those planes -- the clip is dcs_separate_audio_channels_wiener on them with
 * `iterations` and `radius`, and one launch resamples and encodes its nsrc*channels stem planes as (int16)(int)(y*32767)
 * with y the fp32 value of dcs_resample(from_model, num_out = L) (C truncation, no clipping: the encode of
 * dcs_separate_pcm16_host, which wraps modulo 2^16 -- a full-scale clip's resampled stems may overshoot 1.0).  So per clip the bytes are
 * those of (int16)(int)(stem*32767) on the stems of: dcs_resample(to_model) of pcm/32767, then
 * dcs_separate_audio_channels_wiener, then dcs_resample(from_model) trimmed to L.  Launches per clip: those of
 * dcs_separate_audio_channels(_wiener) on a clip of L' samples, plus one -- one fewer than those three calls.
 * Workspace: every buffer is sized once before the pipeline starts, the fp32 planes from the longest clip at 44.1 kHz,
 * L'max samples, and the int16 staging from the longest clip, Lmax samples.  With B(x) and n as above, a fresh ctx holds
 * after the call
 *     W(L'max) - B(4 L'max) + B(4 (channels + 1) L'max) + B(4 nsrc channels L'max)
 *       + n B(2 channels Lmax) + n B(2 nsrc channels Lmax)
 * where W(L'max) is what a fresh ctx holds after dcs_separate_audio_channels_wiener with the same iterations and radius
 * on one clip of L'max samples; the resamplers' banks are their own, not the workspace.
 * Synchronises before returning, also on an error.  Refused with DCS_EINVAL before anything is queued: a NULL resampler,
 * a resampler made on another ctx, a pair that is not inverse, and what dcs_separate_batch_pcm16_channels_host refuses
 * (the model's checks on the longest clip at L'max). */
int dcs_separate_batch_pcm16_channels_resampled_host(dcs_ctx* ctx, dcs_model* model, dcs_stft* plan,
                                                     const dcs_resampler* to_model, const dcs_resampler* from_model,
                                                     int nclips, const int16_t* const* h_pcm, const int64_t* num_samples,
                                                     int channels, int iterations, int radius, float scale_factor,
                                                     int overlap, int patcher, int16_t* const* h_out,
                                                     const int64_t* out_strides, void* stream);

/* ---- bring-up and test entries: the int16 conversions of the int16 entry points -------------------------------- */
/* Each is one launch of the very kernel the int16 batch entry points run, on caller device buffers, on `stream`, which
 * is synchronised before returning.  resampler NULL: at the clip's rate; else the fused kernels of
 * dcs_separate_batch_pcm16_channels_resampled_host (C-channel mode only; made on ctx).  Every argument is checked before
 * anything is queued.
 * dcs_pcm16_decode: d_pcm int16 [num_samples][channels] interleaved ->
 *  - mode 0, 1, 2 (the `downmix` of dcs_separate_pcm16_host, channels 1..8): d_out float [num_samples], channel 0 /
 *    (l + r) * 0.5f / l + r of l = pcm_0 / 32767.0f, r = pcm_1 / 32767.0f (channel 0 whenever channels == 1);
 *    num_out = num_samples.
 *  - DCS_PCM16_CHANNELS (channels 1..16): d_out float [channels + 1][num_out], plane 0 the downmix
 *    (((a_0 + a_1) + a_2) + ...) * (1.0f / channels), plane 1 + c channel c: a_c = pcm_c / 32767.0f, num_out =
 *    num_samples; with a resampler, a_c = dcs_resample of pcm_c / 32767.0f and num_out in
 *    [1, dcs_resampled_length(num_samples)].
 * dcs_pcm16_encode: stem plane p of num_in samples at d_stems + p * stem_stride, the encode of dcs_separate_pcm16_host ->
 *  - DCS_PCM16_MONO (channels 1, nsrc planes): source s at d_out + s * out_stride, int16 [num_out], num_out = num_in,
 *    stem_stride and out_stride >= num_in.
 *  - DCS_PCM16_CHANNELS (channels 1..16, nsrc * channels planes ordered (source, channel), stem_stride >= num_in):
 *    source s at d_out + s * out_stride as int16 [num_out][channels], out_stride = channels * num_out; num_out = num_in;
 *    with a resampler the planes are the encode of dcs_resample(num_out) of each plane, stem_stride = num_in and
 *    num_out in [1, dcs_resampled_length(num_in)].
 *  d_out needs only 2-byte alignment; nothing outside the values listed is written.
 * dcs_downmix_f32: nx (1..16) float planes audio_stride (>= num_samples) apart -> d_mono float [num_samples], the
 *  downmix of DCS_PCM16_CHANNELS on float planes (the float route of dcs_separate_audio_channels). */
enum { DCS_PCM16_MONO = 0, DCS_PCM16_CHANNELS = 3 };
int dcs_pcm16_decode(dcs_ctx* ctx, const dcs_resampler* resampler, int mode, const int16_t* d_pcm, int64_t num_samples,
                     int channels, float* d_out, int64_t num_out, void* stream);
int dcs_pcm16_encode(dcs_ctx* ctx, const dcs_resampler* resampler, int mode, const float* d_stems, int64_t num_in, int nsrc,
                     int channels, int64_t stem_stride, int16_t* d_out, int64_t num_out, int64_t out_stride, void* stream);
int dcs_downmix_f32(dcs_ctx* ctx, const float* d_audio, int nx, int64_t audio_stride, int64_t num_samples, float* d_mono,
                    void* stream);

/* ---- C-channel clips in int16, int32 or float32 --------------------------------------------------------------- */
/* Sample formats of dcs_separate_batch_channels_host and of its conversions.  A sample decodes to the fp32 plane the
 * networks see, and an fp32 stem value y encodes back:
 *  - DCS_SAMPLE_I16 (2 bytes): decode pcm / 32767.0f; encode (int16)(int)(y * 32767.0f), the product in fp32, C
 *    truncation, wrapping modulo 2^16 (NaN gives 0, saturating to int32 first beyond +-2^31): the rule of
 *    dcs_separate_pcm16_host.
 *  - DCS_SAMPLE_I32 (4 bytes; 24-bit PCM as scipy.io.wavfile reads it, the sample in the top 24 bits): decode
 *    (float)((double)pcm / 2147483647.0), each step rounded to nearest (the bits of
 *    (a.astype(float) / iinfo(int32).max).astype(float32)); encode (double)y * 2147483647.0 in fp64, truncated toward
 *    zero and saturated to [-2^31, 2^31 - 1] (__double2int_rz), NaN gives 0 (tested first: the f64 conversion alone
 *    would give -2^31).  It saturates where int16 wraps: the wrap
 *    only reproduces the reference's astype('int16'), and numpy's own int32 result past 2^31 depends on the platform.
 *  - DCS_SAMPLE_F32 (4 bytes): decode the sample itself, bit for bit (no scaling); encode y itself, bit for bit (no
 *    clipping, NaN payloads kept).  Non-finite input gives undefined stems and is not checked, as on every float entry.
 *  - DCS_SAMPLE_I24 (3 bytes): packed signed 24-bit little-endian PCM, the samples of a WAV data chunk with a 3-byte
 *    container.  With v the sign-extended 24-bit value, decode the DCS_SAMPLE_I32 decode of v * 256 (the bits the int32
 *    route gives for scipy.io.wavfile's read of the same file); encode the DCS_SAMPLE_I32 encode of y shifted right by 8
 *    bits (arithmetic), its low 3 bytes stored little-endian: the top 24 bits of the int32 stem, saturated to
 *    [-2^23, 2^23 - 1], NaN gives 0, so the packed stems are the int32 stems shifted right by 8, byte for byte.  Buffers
 *    of this format need only 1-byte alignment.
 * The downmix is that of dcs_separate_audio_channels on the decoded planes in every format.  Code 3 is not a format. */
enum { DCS_SAMPLE_I16 = 0, DCS_SAMPLE_I32 = 1, DCS_SAMPLE_F32 = 2, DCS_SAMPLE_I24 = 4 };
/* C-channel clips (1 to 16 channels) in any sample format through the multi-clip scheduler: the clips in in_format, the
 * stems in out_format, chosen independently.  h_in[i]: [num_samples[i]][channels] samples of in_format (pinned for real
 * overlap) -> source s of clip i at h_out[i] + s*channels*out_strides[i] samples as [num_samples[i]][channels] of
 * out_format, interleaved: the layouts of dcs_separate_batch_pcm16_channels_host with each value 2, 3 or 4 bytes wide.
 * to_model and from_model are both NULL (clips at 44.1 kHz) or both set (clips at another rate, the pair of
 * dcs_separate_batch_pcm16_channels_resampled_host, with its checks).  Per clip the stems are, byte for byte,
 *     encode_out(dcs_separate_audio_channels_wiener(decode_in(clip), iterations, radius))
 * at 44.1 kHz, and at another rate encode_out of dcs_resample(from_model, num_out = L) of the stems of that call on
 * dcs_resample(to_model) of decode_in(clip), per channel.  With DCS_SAMPLE_I16 in and out these are the bytes of
 * dcs_separate_batch_pcm16_channels_host and dcs_separate_batch_pcm16_channels_resampled_host.
 * Launches per clip: those of dcs_separate_audio_channels(_wiener) on the clip at 44.1 kHz plus one, in every format.
 * At another rate, a 3- or 4-byte in_format stages each decode tile as fp32; where C channels then do not fit one tile next
 * to the bank (C >= 11 at some rates, 192 kHz at C = 16 among them) the decode runs on equal channel groups and one
 * more launch forms the downmix plane, with the same bits.
 * Workspace: as for dcs_separate_batch_pcm16_channels_host (resampled_host at another rate) with the staging terms
 *       n B(b_in channels Lmax) + n B(b_out nsrc channels Lmax)
 * where b_in and b_out are the formats' bytes per sample (2, 3 or 4).
 * Synchronises before returning, also on an error.  Refused with DCS_EINVAL before anything is queued: an unknown
 * format code, exactly one resampler NULL, and what the two int16 C-channel batch entries refuse. */
int dcs_separate_batch_channels_host(dcs_ctx* ctx, dcs_model* model, dcs_stft* plan, const dcs_resampler* to_model,
                                     const dcs_resampler* from_model, int in_format, int out_format, int nclips,
                                     const void* const* h_in, const int64_t* num_samples, int channels, int iterations,
                                     int radius, float scale_factor, int overlap, int patcher, void* const* h_out,
                                     const int64_t* out_strides, void* stream);
/* Bring-up and test entries: the conversions of dcs_separate_batch_channels_host, the C-channel layout of
 * dcs_pcm16_decode / dcs_pcm16_encode (DCS_PCM16_CHANNELS) in any format, with the same arguments and checks.  Each is
 * one launch of the kernel the batch runs (two for a resampled decode whose channels take groups), on caller device
 * buffers, on `stream`, which is synchronised before returning; every argument is checked before anything is queued.
 * 4-byte formats need 4-byte-aligned d_in / d_out; DCS_SAMPLE_I24 takes any address.
 * dcs_channels_decode: d_in [num_samples][channels] of `format` -> d_out float [channels + 1][num_out], plane 0 the
 *  downmix, plane 1 + c the decode of channel c; with a resampler, dcs_resample of it and num_out in
 *  [1, dcs_resampled_length(num_samples)].
 * dcs_channels_encode: nsrc * channels fp32 planes (source, channel) stem_stride apart -> source s at
 *  d_out + s * out_stride samples as [num_out][channels] of `format`, out_stride = channels * num_out; with a resampler
 *  the planes are the encode of dcs_resample(num_out) of each plane, stem_stride = num_in.  Nothing outside the values
 *  listed is written. */
int dcs_channels_decode(dcs_ctx* ctx, const dcs_resampler* resampler, int format, const void* d_in, int64_t num_samples,
                        int channels, float* d_out, int64_t num_out, void* stream);
int dcs_channels_encode(dcs_ctx* ctx, const dcs_resampler* resampler, int format, const float* d_stems, int64_t num_in,
                        int nsrc, int channels, int64_t stem_stride, void* d_out, int64_t num_out, int64_t out_stride,
                        void* stream);

/* ---- long C-channel recordings in bounded device memory ---------------------------------------------------------- */
/* One segment of a long recording: three sample ranges, half-open.
 *  - in:    [in_start, in_stop), the recording's samples staged on the device;
 *  - model: [model_start, model_stop), the range separated at 44.1 kHz (the in range itself at 44.1 kHz);
 *  - kept:  [out_start, out_stop), the core of the recording written to the output. */
typedef struct {
  int64_t in_start, in_stop;
  int64_t model_start, model_stop;
  int64_t out_start, out_stop;
} dcs_segment;
/* The segments of a recording of num_samples samples cut into cores of core_samples, written to out[0 ..
 * min(count, max_segments)); returns the count, ceil(num_samples / core_samples), or -1 for bad arguments.  Pure host
 * arithmetic (no ctx).  frame_size, hop, time_context, overlap: the separation's geometry; wiener_reach: iterations *
 * radius of the Wiener post-filter (0 without it).  The resampler pair is given as to_model's up, down and ntaps and
 * from_model's ntaps (from_model is down/up); up = down = ntaps = 1 for a recording at 44.1 kHz.  With half = (n - 1)/2,
 * output m of a resampler (u, d, n) reads inputs lo(m) = ceil((m d + half - n + 1) / u) .. hi(m) = floor((m d + half) /
 * u), clipped to the input.  Core i is [o0, o1) = [i K, min(L, (i + 1) K)); then
 *  1. its exact range at 44.1 kHz: [e0, e1) = [lo_from(o0), hi_from(o1 - 1) + 1) clipped to [0, L'),
 *     L' = dcs_resampled_length(L, to up, to down) (without resamplers [o0, o1) and L' = L);
 *  2. the model range: the two bounds of longclip.plan_segments for the core [e0, e1) of a clip of L' samples --
 *     model_start = frame0 * hop, frame0 the largest multiple of step = time_context - overlap (of lcm(step, 128) when
 *     wiener_reach > 0) whose margin makes the core exact, 0 for the first core or where the margin reaches the start;
 *     model_stop = model_start + G * hop with longclip's G, L' for the last core or where that overshoots;
 *  3. the in range: [lo_to(model_start), hi_to(model_stop - 1) + 1) clipped to [0, L).
 * The cores tile [0, L) once. */
int64_t dcs_long_segments(int64_t num_samples, int64_t core_samples, int frame_size, int hop, int time_context, int overlap,
                          int wiener_reach, int to_up, int to_down, int to_ntaps, int from_ntaps, dcs_segment* out,
                          int64_t max_segments);
/* One C-channel recording of any length (1 to 16 channels, any sample formats, 44.1 kHz or any rate of a resampler pair)
 * through the multi-clip scheduler of dcs_separate_batch_channels_host with a device workspace bounded by the segment
 * length: h_in [num_samples][channels] of in_format (pinned for real overlap) -> source s at h_out + s*channels*out_stride
 * samples as [num_samples][channels] of out_format, the layout of the batch.  The recording is cut by dcs_long_segments
 * (core_samples, the plan's geometry, wiener_reach = iterations * radius, the pair's up/down/ntaps) and each segment is a
 * clip of the pipeline: H2D of its in range straight from h_in, the decode (at another rate the windowed resampling
 * decode, whose planes are samples [model_start, model_stop) of the whole recording's), the separation of
 * dcs_separate_audio_channels_wiener on the model range, the encode of the kept core only (at another rate the windowed
 * encode of the stems placed at [model_start, model_stop)), and D2H of the core straight to h_out at out_start (one 2-D
 * copy, rows = sources).  Every output sample is written once; nothing is stitched on the host.
 * Byte contract, for each segment with X the recording:
 *  - 44.1 kHz: the kept samples are samples [out_start - in_start, out_stop - in_start) of dcs_separate_batch_channels_host
 *    on the single clip X[in_start:in_stop] with the same formats and options.
 *  - another rate: the kept samples are dcs_channels_encode_range(from_model, Y, window [out_start, out_stop)) with
 *    Y = dcs_separate_audio_channels_wiener on the channel planes of dcs_channels_decode_range(to_model, ...) over the model
 *    range; those planes are, bit for bit, samples [model_start, model_stop) of dcs_channels_decode(to_model) on the whole
 *    recording.
 *  - one segment (core_samples >= num_samples): the bytes of dcs_separate_batch_channels_host on the whole recording.
 *  - against the whole-recording call the stems differ only by the summation order of the network's GEMMs for another
 *    patch count (longclip.py).
 * Launches per segment: those of one clip of dcs_separate_batch_channels_host of the segment's length.
 * Workspace: every buffer is sized once, before the pipeline starts, from the longest model range S'max, the longest in
 * range Smax and the longest core Kmax: with B(x) and n = min(segments, 2) as for the batch, a fresh ctx holds
 *     W(S'max) - B(4 S'max) + B(4 (channels + 1) S'max) + B(4 nsrc channels S'max)
 *       + n B(b_in channels Smax) + n B(b_out nsrc channels Kmax)
 * Each model range is at most the core's exact range at 44.1 kHz plus longclip.margins and the rounding of its ends to the
 * frame grid (under (align + 1) * hop samples each, align = step, or lcm(step, 128) with the filter), so the workspace is
 * bounded by core_samples and the geometry, not by the recording's length; two recordings with the same core may still
 * differ by where their cores fall on that grid.
 * Synchronises before returning, also on an error.  Refused with DCS_EINVAL before anything is queued: what
 * dcs_separate_batch_channels_host refuses (the model's checks on the longest model range), core_samples < 1,
 * out_stride < num_samples, a NULL buffer, iterations > 0 with radius 0 over more than one segment (the message names the
 * radius), a spectrum tap or a routing tap set on the ctx (the segments would overwrite it one after another). */
int dcs_separate_long_channels_host(dcs_ctx* ctx, dcs_model* model, dcs_stft* plan, const dcs_resampler* to_model,
                                    const dcs_resampler* from_model, int in_format, int out_format, const void* h_in,
                                    int64_t num_samples, int channels, int iterations, int radius, int64_t core_samples,
                                    float scale_factor, int overlap, int patcher, void* h_out, int64_t out_stride,
                                    void* stream);
/* Bring-up and test entries: the windowed conversions of dcs_separate_long_channels_host at another rate, one launch of
 * the windowed kernels each (two for a decode whose channels take groups), on `stream`, which is synchronised before
 * returning; the resampler is required, and the checks of dcs_channels_decode / _encode apply.
 * dcs_channels_decode_range: outputs [out_first, out_first + num_out) of dcs_channels_decode(resampler) on a recording of
 *  num_samples samples, of which d_in holds samples [in_first, in_first + num_staged) as [num_staged][channels] (the
 *  recording is zero outside [0, num_samples)) -> d_out float [channels + 1][num_out].
 * dcs_channels_encode_range: outputs [out_first, out_first + num_out) of dcs_channels_encode(resampler) on stems of a
 *  44.1 kHz signal of num_samples samples, of which d_stems holds samples [in_first, in_first + num_in) (nsrc * channels
 *  planes num_in apart; zeros elsewhere) -> source s at d_out + s * out_stride as [num_out][channels], out_stride =
 *  channels * num_out.
 * Both also refuse a window outside [0, dcs_resampled_length(num_samples)), a staged range outside [0, num_samples), and
 * a staged range that does not cover every input the window reads (lo(out_first) .. hi(out_first + num_out - 1),
 * clipped). */
int dcs_channels_decode_range(dcs_ctx* ctx, const dcs_resampler* resampler, int format, const void* d_in,
                              int64_t num_samples, int64_t in_first, int64_t num_staged, int channels, float* d_out,
                              int64_t out_first, int64_t num_out, void* stream);
int dcs_channels_encode_range(dcs_ctx* ctx, const dcs_resampler* resampler, int format, const float* d_stems,
                              int64_t num_samples, int64_t in_first, int64_t num_in, int nsrc, int channels, void* d_out,
                              int64_t out_first, int64_t num_out, int64_t out_stride, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DCS_H_ */
