// score1x1.cu -- the score-informed Bach10 network build_ca_1x1 (examples/bach10_scoreinformed/trainCNNrwc.py:66-132,
// selected with --function build_ca_1x1, :629): weight re-layout and orchestration.  Every contraction is a strided-view
// GEMM on the tensor cores (gemm_tc.cu) with the gated epilogues (EPI_POST / EPI_GATE); the last stage is K3s (sconv_tc.cu).
//
// Encoder: six Lasagne Conv2DLayer(rectify) + BiasLayer, kernel (1,5) x4 then (10,5) x2, all stride (1,2), so each layer
// has a bias on each side of the ReLU:  h_l = relu(W_l * h_{l-1} + b_l) + c_l.  Then a 1x1 conv to 800 channels
// (rectify + BiasLayer) sliced into four 200-channel sources.  Decoder d: InverseLayer(conv6) ... InverseLayer(conv1);
// Lasagne's InverseLayer is the gradient of the layer's output -- AFTER its rectifier -- so
//     inv_l(g) = conv_l^T(g * relu'(pre_l)),   relu' in {0, 0.5 (pre == 0, Theano's 0.5*(x+|x|)), 1}.
// The concat of the four decoders has 16 channels; bias + ReLU, and only channels 0..3 -- all from decoder 1 -- feed the
// Bach10 mask (trainCNNrwc.py:357-416).  Decoders 2-4 and 1x1 filters 200..799 are dead at inference and never uploaded.
//
// Like the other nets, a patch is a view of the clip: the encoder value at patch row r is the whole-clip value at frame
// k*step + r, so conv1..conv6 run once per frame over the Tp frames the patches span, storing their gate codes
// 2*relu'(pre) (uint8, 0/1/2).  The decoder runs per patch, in chunks of S1_CHUNK patches:
//   D6  [Pc][h6+18][W6+4][200]   s6 = (relu(1x1 + b) + c) * gate6 (the 1x1 conv on each patch's rows), zero padded
//   Dl  [Pc][hl+2*pl][Wl+4][CPl] InverseLayer(conv l+1) of D(l+1), times gate_l of frame k*step + u   (l = 5..2)
//   G   [Pc][tc][W1][32]         InverseLayer(conv2) of D2, times gate1: the K3s operand
// (pl = 9 row padding for the (10,5) layers' inverses, 2 columns each side).  An InverseLayer of a stride-2, width-5
// conv is one GEMM per output pair: A row = 3 input columns x channels (per time tap), N = 2 output phases x channels.
// Columns outside the gated layer's width are never stored, so the padding stays zero.  A chunk recomputes the
// ceil(tc/step)-1 patches before it that share its first frames, and K3s writes only its frames.
#include <algorithm>
#include "common.cuh"

namespace dcs {

namespace {
constexpr int S1_CH[7] = {4, 30, 50, 70, 100, 200, 200};   // input planes, then conv1..conv6 filters
constexpr int S1_KH[7] = {0, 1, 1, 1, 1, 10, 10};          // kernel height of conv l
constexpr int S1_CHUNK = 128;                                // patches a decoder chunk writes
constexpr int64_t S1_SLACK = 2048;                           // floats after each buffer (padded K segments overrun)
constexpr int pitch4(int c) { return (c + 3) / 4 * 4; }
constexpr int round32(int k) { return (k + 31) / 32 * 32; }
// K segment of one time tap of a (10,5) layer, padded to the 32-wide GEMM stage so the operands load as float4: the
// extra floats are neighbouring activations times zero weight rows
int fwd_seg(int l) { return round32(5 * pitch4(S1_CH[l - 1])); }
int inv_seg(int l) { return S1_KH[l] == 1 ? 3 * pitch4(S1_CH[l]) : round32(3 * pitch4(S1_CH[l])); }
int fwd_k(int l) { return S1_KH[l] == 1 ? 5 * pitch4(S1_CH[l - 1]) : S1_KH[l] * fwd_seg(l); }
int inv_k(int l) { return S1_KH[l] * inv_seg(l); }
const char* const ENC_NAMES[7] = {"conv1x1_gemm", "enc_conv1_gemm", "enc_conv2_gemm", "enc_conv3_gemm",
                                  "enc_conv4_gemm", "enc_conv5_gemm", "enc_conv6_gemm"};
const char* const INV_NAMES[7] = {"", "", "dec_convT2_gemm", "dec_convT3_gemm", "dec_convT4_gemm", "dec_convT5_gemm",
                                  "dec_convT6_gemm"};
}  // namespace

// the four input planes [4][T][ldf] (plane stride in_plane) -> channel-interleaved X4[Tp][F][4], zero frames from T on
// (util patcher): conv1's A row (t, j) is then 5 bins x 4 channels = 20 contiguous floats at (t*F + 2j)*4
__global__ void interleave4_kernel(const float* __restrict__ in, int64_t in_plane, int64_t ldf, int64_t T, int64_t Tp, int F,
                                   float4* __restrict__ X4) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= Tp * F) return;
  const int64_t t = i / F, b = i - t * F;
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (t < T) {
    const float* p = in + t * ldf + b;
    v = make_float4(__ldg(p), __ldg(p + in_plane), __ldg(p + 2 * in_plane), __ldg(p + 3 * in_plane));
  }
  X4[i] = v;
}

int model_create_s1x1(dcs_model* m, int nparams, const float* const* hp, const int64_t* shp, const int* nd) {
  dcs_s1x1& s = m->s1;
  const int F = m->F, tc = m->tc;
  m->nsrc = 4;
  if (nparams != 22) { set_error("architecture %d (build_ca_1x1) needs 22 parameter arrays, got %d", m->arch, nparams); return DCS_EMODEL; }
  if (F < 253 || tc < 19) {
    set_error("build_ca_1x1 needs feat_size >= 253 and time_context >= 19 (conv6 must keep a column and a row), got %d / %d", F, tc);
    return DCS_EMODEL;
  }
  s.W[0] = F;
  for (int l = 0; l < 7; ++l) { s.C[l] = S1_CH[l]; s.CP[l] = pitch4(S1_CH[l]); }
  for (int l = 1; l <= 6; ++l) s.W[l] = (s.W[l - 1] - 5) / 2 + 1;
  bool ok = true;
  for (int l = 1; l <= 6 && ok; ++l) {
    const int i = 3 * (l - 1);
    ok = shape_is(shp + 4 * i, nd[i], 4, s.C[l], s.C[l - 1], S1_KH[l], 5) && shape_is(shp + 4 * (i + 1), nd[i + 1], 1, s.C[l]) &&
         shape_is(shp + 4 * (i + 2), nd[i + 2], 1, s.C[l]);
  }
  ok = ok && shape_is(shp + 4 * 18, nd[18], 4, 800, 200, 1, 1) && shape_is(shp + 4 * 19, nd[19], 1, 800) &&
       shape_is(shp + 4 * 20, nd[20], 1, 800) && shape_is(shp + 4 * 21, nd[21], 1, 16);
  if (!ok) { set_error("parameter shapes do not match build_ca_1x1 (conv1.W (30,4,1,5) ... 1x1 conv (800,200,1,1), bias (16,))"); return DCS_EMODEL; }

  for (int l = 1; l <= 6; ++l) {
    const float* W = hp[3 * (l - 1)];
    const int Ci = s.C[l - 1], Co = s.C[l], Pi = s.CP[l - 1], kh = S1_KH[l];
    // forward (flip_filters): K index (time tap p' = kh-1-p, column tap q' = 4-q, input channel)
    std::vector<float> B((size_t)fwd_k(l) * Co, 0.f);
    for (int f = 0; f < Co; ++f)
      for (int c = 0; c < Ci; ++c)
        for (int p = 0; p < kh; ++p)
          for (int q = 0; q < 5; ++q) {
            const float v = W[(((size_t)f * Ci + c) * kh + p) * 5 + q];
            const int qq = 4 - q, pp = kh - 1 - p;
            const size_t k = (size_t)pp * (kh == 1 ? 0 : fwd_seg(l)) + (size_t)qq * Pi + c;
            B[k * Co + f] = v;
          }
    DCS_TRY(tc_weight_create(B.data(), Co, fwd_k(l), Co, &s.tF[l], &m->dev));
    if (l >= 2) {   // InverseLayer(conv l): K index (time tap p, column dcol of the output pair, channel of conv l's output),
                    // N index (phase r, channel of conv l's input); column j = 2m + r takes tap q = 2*dcol - r
      const int Po = s.CP[l], seg = inv_seg(l), N = 2 * Ci;
      std::vector<float> Bi((size_t)inv_k(l) * N, 0.f);
      for (int ci = 0; ci < Co; ++ci)
        for (int co = 0; co < Ci; ++co)
          for (int p = 0; p < kh; ++p)
            for (int dcol = 0; dcol < 3; ++dcol)
              for (int r = 0; r < 2; ++r) {
                const int q = 2 * dcol - r;
                if (q < 0 || q > 4) continue;
                Bi[((size_t)p * seg + (size_t)dcol * Po + ci) * N + r * Ci + co] = W[(((size_t)ci * Ci + co) * kh + p) * 5 + q];
              }
      DCS_TRY(tc_weight_create(Bi.data(), N, inv_k(l), N, &s.tI[l], &m->dev));
    }
    std::vector<float> b(hp[3 * (l - 1) + 1], hp[3 * (l - 1) + 1] + Co), c(hp[3 * (l - 1) + 2], hp[3 * (l - 1) + 2] + Co);
    DCS_TRY(upload(b, &s.b[l], &m->dev));
    DCS_TRY(upload(c, &s.c[l], &m->dev));
  }
  {  // 1x1 conv, filters 0..199 (decoder 1's slice)
    std::vector<float> B((size_t)200 * 200);
    for (int f = 0; f < 200; ++f)
      for (int c = 0; c < 200; ++c) B[(size_t)c * 200 + f] = hp[18][(size_t)f * 200 + c];
    DCS_TRY(tc_weight_create(B.data(), 200, 200, 200, &s.tF[0], &m->dev));
    std::vector<float> b(hp[19], hp[19] + 200), c(hp[20], hp[20] + 200);
    DCS_TRY(upload(b, &s.b[0], &m->dev));
    DCS_TRY(upload(c, &s.c[0], &m->dev));
  }
  // K3s filter banks, one per input channel: w[ch][dd][f][r] = W1[f][ch][0][4 - r - 2*dd] (r < 2)
  std::vector<float> Wsc((size_t)4 * 3 * 32 * 4, 0.f), bout(hp[21], hp[21] + 4);
  for (int ch = 0; ch < 4; ++ch)
    for (int dd = 0; dd < 3; ++dd)
      for (int f = 0; f < 30; ++f)
        for (int r = 0; r < 2; ++r) {
          const int q = 4 - r - 2 * dd;
          if (q >= 0) Wsc[(((size_t)ch * 3 + dd) * 32 + f) * 4 + r] = hp[0][((size_t)f * 4 + ch) * 5 + q];
        }
  DCS_TRY(upload(Wsc, &s.Wsc, &m->dev));
  DCS_TRY(upload(bout, &s.bout, &m->dev));
  return DCS_OK;
}

int s1x1_forward(dcs_ctx* ctx, const dcs_model* m, const NetCall& n, cudaStream_t st) {
  const dcs_s1x1& s = m->s1;
  const int tc = m->tc, step = n.step;
  const int64_t T = n.T, P = n.P, Tp = n.Tp;
  const int* W = s.W;
  const int* C = s.C;
  const int* CP = s.CP;
  int64_t rows[7] = {0, Tp, Tp, Tp, Tp, Tp - 9, Tp - 18};
  DCS_REQUIRE(Tp * W[0] < ((int64_t)1 << 31), "clip too long for 32-bit row indices");

  // ---- encoder, once per frame: activations [rows][W_l][CP_l] and gate codes [rows][W_l][C_l], layer after layer
  int64_t eoff[7] = {0}, coff[7] = {0}, etot = Tp * W[0] * 4 + S1_SLACK, ctot = 0;   // X4 first
  for (int l = 1; l <= 6; ++l) {
    eoff[l] = etot; etot += rows[l] * W[l] * CP[l] + S1_SLACK;
    coff[l] = ctot; ctot += rows[l] * W[l] * C[l];
  }
  DCS_TRY(ensure_layout(ctx, NET_ENC, (size_t)etot * 4, n.sig, st));
  DCS_TRY(ensure_layout(ctx, NET_CODES, (size_t)ctot, n.sig, st));
  float* E = ctx->net[NET_ENC].as<float>();
  uint8_t* codes = ctx->net[NET_CODES].as<uint8_t>();
  {
    ProfScope ps(ctx, "enc_interleave", st);
    interleave4_kernel<<<(unsigned)ceil_div64(Tp * W[0], 256), 256, 0, st>>>(n.in, n.in_plane, n.ldf, T, Tp, W[0],
                                                                             reinterpret_cast<float4*>(E));
    DCS_CHECK_LAUNCH();
    ctx->launches++;
  }
  for (int l = 1; l <= 6; ++l) {
    ProfScope ps(ctx, ENC_NAMES[l], st);
    // rows (t, j): the 5 adjacent columns from 2j are contiguous -- one K segment, or one per time tap
    GemmDesc g = gemm_plain(l == 1 ? E : E + eoff[l - 1], 0, nullptr, C[l], s.b[l], E + eoff[l], CP[l], (int)(rows[l] * W[l]),
                            C[l], fwd_k(l), 0);
    g.m_inner = W[l]; g.a_so = (int64_t)W[l - 1] * CP[l - 1]; g.a_si = 2 * CP[l - 1];
    if (S1_KH[l] > 1) { g.k_seg = fwd_seg(l); g.k_ss = (int64_t)W[l - 1] * CP[l - 1]; }
    g.bias2 = s.c[l]; g.code = codes + coff[l];
    DCS_TRY(launch_gemm_tc_epi(ctx, g, s.tF[l], EPI_POST, st));
  }
  if (ctx->pool_tap) {   // inspection tap (parity tests): the gate codes of this call, dcs.h
    DCS_REQUIRE(ctx->pool_tap_cap >= ctot, "routing tap holds %lld bytes, this call produced %lld", (long long)ctx->pool_tap_cap, (long long)ctot);
    DCS_CUDA(cudaMemcpyAsync(ctx->pool_tap, codes, (size_t)ctot, cudaMemcpyDeviceToDevice, st));
  }

  // ---- decoder 1, per patch, in chunks
  const int halo = (tc - 1) / step;   // = ceil(tc/step) - 1 earlier patches share frames with a chunk's first patch
  const int64_t Pcap = std::min<int64_t>(P, S1_CHUNK + halo);
  int h[7], rp[7], HP[7], WPd[7], cpad[7];
  int64_t doff[7] = {0}, dtot = 0;
  for (int l = 1; l <= 6; ++l) {
    h[l] = l == 6 ? tc - 18 : (l == 5 ? tc - 9 : tc);
    rp[l] = l >= 2 ? S1_KH[l] - 1 : 0;
    cpad[l] = l >= 2 ? 2 : 0;
    HP[l] = h[l] + 2 * rp[l];
    WPd[l] = W[l] + 2 * cpad[l];
    doff[l] = dtot; dtot += Pcap * HP[l] * WPd[l] * CP[l] + S1_SLACK;
  }
  DCS_REQUIRE(Pcap * tc * ((W[1] + 1) / 2) < ((int64_t)1 << 31), "decoder chunk too large for 32-bit row indices");
  // the zero padding depends on the chunk capacity as well
  DCS_TRY(ensure_layout(ctx, NET_DEC, (size_t)dtot * 4, n.sig ^ ((uint64_t)Pcap << 16), st));
  float* D = ctx->net[NET_DEC].as<float>();
  for (int64_t p0 = 0; p0 < P; p0 += S1_CHUNK) {
    const int64_t p1 = std::min<int64_t>(P, p0 + S1_CHUNK), pb = std::max<int64_t>(0, p0 - halo), Pc = p1 - pb;
    {  // s6 = (relu(1x1 conv + b) + c) * gate6 on rows (k, u, j) of the patches, into D6's interior
      ProfScope ps(ctx, ENC_NAMES[0], st);
      const int h6 = h[6], W6 = W[6];
      GemmDesc g = gemm_plain(E + eoff[6] + pb * step * W6 * CP[6], 0, nullptr, 200, s.b[0], D + doff[6], 0, (int)(Pc * h6 * W6), 200,
                              200, 0);
      g.m_inner = h6 * W6; g.a_so = (int64_t)step * W6 * CP[6]; g.m_inner2 = W6; g.a_si = (int64_t)W6 * CP[6]; g.a_s2 = CP[6];
      g.cm_inner = h6 * W6; g.c_so = (int64_t)HP[6] * WPd[6] * CP[6]; g.cm_inner2 = W6; g.c_si = (int64_t)WPd[6] * CP[6]; g.c_s2 = CP[6];
      g.c_col0 = ((int64_t)rp[6] * WPd[6] + cpad[6]) * CP[6];
      g.bias2 = s.c[0];
      g.gate = codes + coff[6] + pb * step * W6 * C[6];
      g.g_inner = h6 * W6; g.g_so = (int64_t)step * W6 * C[6]; g.g_inner2 = W6; g.g_si = (int64_t)W6 * C[6]; g.g_s2 = C[6];
      g.g_lim = INT64_MAX;
      DCS_TRY(launch_gemm_tc_epi(ctx, g, s.tF[0], EPI_POST | EPI_GATE, st));
    }
    for (int l = 6; l >= 2; --l) {   // InverseLayer(conv l): D_l -> D_{l-1} (G for l = 2), rows (u, k, output pair)
      ProfScope ps(ctx, INV_NAMES[l], st);
      const int kh = S1_KH[l], Pi = CP[l], Co = C[l - 1], Po = CP[l - 1], M2 = (W[l - 1] + 1) / 2;
      const int64_t rowsU = Pc * M2;
      GemmDesc g = gemm_plain(D + doff[l], 0, nullptr, 2 * Co, nullptr, D + doff[l - 1], 0, (int)(h[l - 1] * rowsU), 2 * Co, inv_k(l), 0);
      g.m_inner = (int)rowsU; g.a_so = (int64_t)WPd[l] * Pi; g.m_inner2 = M2; g.a_si = (int64_t)HP[l] * WPd[l] * Pi; g.a_s2 = Pi;
      g.k_seg = inv_seg(l); g.k_ss = (int64_t)WPd[l] * Pi;
      g.cm_inner = (int)rowsU; g.c_so = (int64_t)WPd[l - 1] * Po; g.cm_inner2 = M2; g.c_si = (int64_t)HP[l - 1] * WPd[l - 1] * Po;
      g.c_s2 = 2 * Po; g.c_col0 = ((int64_t)rp[l - 1] * WPd[l - 1] + cpad[l - 1]) * Po;
      g.n_seg = Co; g.n_ss = Po;
      g.gate = codes + coff[l - 1] + pb * step * W[l - 1] * Co;
      g.g_inner = (int)rowsU; g.g_so = (int64_t)W[l - 1] * Co; g.g_inner2 = M2; g.g_si = (int64_t)step * W[l - 1] * Co; g.g_s2 = 2 * Co;
      g.g_lim = (int64_t)W[l - 1] * Co;
      if (kh > 1) { g.kc_rows = (int)rowsU; g.kc_unit = inv_seg(l); g.kc_pad = kh - 1; g.kc_n = h[l]; g.kc_taps = kh; }
      DCS_TRY(launch_gemm_tc_epi(ctx, g, s.tI[l], EPI_GATE, st));
    }
    // InverseLayer(conv1) over the four filter banks + bias + ReLU + Bach10 mask + cross-fade + phase: this chunk's frames
    SconvMaskArgs a;
    a.arch = m->arch; a.G = D + doff[1]; a.tie = nullptr; a.W = s.Wsc; a.bout = s.bout; a.X = n.X; a.S = n.S;
    a.ldf = n.ldf; a.src_stride = n.src_stride; a.T = (int)T; a.P = (int)P; a.tc = tc; a.overlap = n.overlap; a.F = m->F;
    a.J = W[1]; a.WP = W[1];
    a.p_base = (int)pb; a.t0 = (int)(p0 * step); a.t1 = p1 == P ? (int)T : (int)(p1 * step);
    ProfScope ps(ctx, "dec_convT1_mask_xfade", st);
    if (!ctx->debug_simt_gemm) {   // the product path
      DCS_REQUIRE(sconv_mask_tc_supported(a), "s1x1_forward: tensor-core mask kernel does not take this shape");
      DCS_TRY(launch_sconv_mask_tc(ctx, a, st, n.M));
    } else {
      DCS_TRY(launch_sconv_mask(ctx, a, st, n.M));   // FFMA twin: cross-check (DCS_DEBUG_SIMT_GEMM=1)
    }
  }
  return DCS_OK;
}

}  // namespace dcs
