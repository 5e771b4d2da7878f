// sconv_model.cu -- the strided-conv1 networks on the GPU: iKala (max-pool and no-pool variants,
// examples/ikala/separate_ikala.py:172-192, examples/ikala/trainCNN.py:66-110) and Bach10
// (examples/bach10/separate_bach10.py:172-229).  Weight re-layout + orchestration; every dense
// contraction is a strided-view GEMM on the tensor cores (gemm_tc.cu), exactly like the DSD100
// path: conv1 and conv2 run ONCE PER FRAME (conv1 has kernel height 1; conv2's time taps make
// each patch a strided window of the per-frame result), channels are padded 30 -> 32 so that
// every convolution tap is one aligned 32-float K segment.
//
// Activation layouts (f' = channel, fastest):
//   H1  [Tp][J][32]            conv1 + biases                 J = (F-30)/sw1 + 1
//   Hp  [Tp][WP][32], tie      max-pool (1,4) (iKala)         WP = J/4
//   H2  [Tp-kh2+1][w2][32]     conv2 + biases                 w2 = WP-kw2+1
//   z   [P][256]               bottleneck (ReLU)
//   apad[P][ndec][HP][WPP][32] decoder dense (ReLU), zero padded by kh2-1 rows / kw2-1 columns
//   G   [P*ndec][tc][WP][32]   InverseLayer(conv2) (full correlation, taps clipped per row group)
// then K3s (sconv.cu): un-pool + InverseLayer(conv1) + mask + cross-fade + phase.
#include "common.cuh"

namespace dcs {

int model_create_sconv(dcs_model* m, int nparams, const float* const* hp, const int64_t* shp, const int* nd) {
  dcs_sconv& c = m->sc;
  const int F = m->F, tc = m->tc, C = 30, CP = 32, KW = 30;
  c.nch = 1;
  c.nfc = 256;
  int ndec_params = 0;   // decoders present in the parameter list (>= the ones inference needs)
  if (m->arch == DCS_ARCH_BACH10) {
    c.sw1 = 4; c.pool = 0; c.kh2 = (2 * tc) / 3; c.kw2 = 1; c.ndec = 4; c.rule = 1; m->nsrc = 4;
  } else if (m->arch == DCS_ARCH_BACH10_SCORE) {
    // 4 input channels; every InverseLayer(., conv1) returns 4 channels, the concat has 16 and only
    // channels 0..3 -- all from decoder 1 -- are used: decoders 2-4 are dead at inference
    // (trainCNNrwc.py:189,248-251; SURVEY.md 0.8)
    // The one-decoder variant (the default build_ca of trainCNNrwc_samp.py:195-235, 11 arrays) is decoder 1 alone
    c.nch = 4; c.sw1 = 4; c.pool = 0; c.kh2 = (2 * tc) / 3; c.kw2 = 1; c.ndec = 1; ndec_params = nparams == 11 ? 1 : 4; c.rule = 1; m->nsrc = 4;
  } else {
    c.sw1 = 3; c.pool = m->arch == DCS_ARCH_IKALA ? 4 : 0; c.kh2 = 10; c.kw2 = 20; c.ndec = 2; c.rule = 0; m->nsrc = 2;
  }
  DCS_REQUIRE(F >= KW, "feat_size %d smaller than the conv1 kernel", F);
  c.J = (F - KW) / c.sw1 + 1;
  c.WP = c.pool ? c.J / c.pool : c.J;
  c.h2 = tc - c.kh2 + 1;
  c.w2 = c.WP - c.kw2 + 1;
  if (c.w2 < 1 || c.h2 < 1) { set_error("feat_size %d / time_context %d too small for this architecture", F, tc); return DCS_EMODEL; }
  c.HP = c.h2 + 2 * (c.kh2 - 1);
  c.WPP = c.w2 + 2 * (c.kw2 - 1);
  const int h2 = c.h2, w2 = c.w2, kh2 = c.kh2, kw2 = c.kw2, ndec = c.ndec;
  const int64_t flat = (int64_t)C * h2 * w2, flatp = (int64_t)h2 * w2 * CP;
  if (!ndec_params) ndec_params = ndec;
  const int want = 8 + 2 * ndec_params + 1, nout = ndec_params * c.nch == 16 ? 16 : m->nsrc;
  if (nparams != want) {
    set_error(m->arch == DCS_ARCH_BACH10_SCORE ? "architecture %d needs %d (or 11) parameter arrays, got %d" : "architecture %d needs %d parameter arrays, got %d",
              m->arch, want, nparams);
    return DCS_EMODEL;
  }
  bool ok = shape_is(shp + 0, nd[0], 4, C, c.nch, 1, KW) && shape_is(shp + 4, nd[1], 1, C) && shape_is(shp + 8, nd[2], 1, C) &&
            shape_is(shp + 12, nd[3], 4, C, C, kh2, kw2) && shape_is(shp + 16, nd[4], 1, C) && shape_is(shp + 20, nd[5], 1, C) &&
            shape_is(shp + 24, nd[6], 2, flat, c.nfc) && shape_is(shp + 28, nd[7], 1, c.nfc) &&
            shape_is(shp + 4 * (want - 1), nd[want - 1], 1, nout);
  for (int d = 0; d < ndec_params && ok; ++d)
    ok = shape_is(shp + 4 * (8 + 2 * d), nd[8 + 2 * d], 2, c.nfc, flat) && shape_is(shp + 4 * (9 + 2 * d), nd[9 + 2 * d], 1, flat);
  if (!ok) { set_error("parameter shapes do not match architecture %d with feat_size=%d time_context=%d", m->arch, F, tc); return DCS_EMODEL; }

  const float *W1 = hp[0], *W2 = hp[3], *Wfc = hp[6];
  // conv1 forward: B1[ch*KW + q'][f] = W1[f][ch][0][KW-1-q']
  const int nch = c.nch;
  std::vector<float> B1((size_t)nch * KW * C), b1(CP, 0.f), b2(CP, 0.f);
  for (int f = 0; f < C; ++f)
    for (int ch = 0; ch < nch; ++ch)
      for (int q = 0; q < KW; ++q) B1[((size_t)ch * KW + q) * C + f] = W1[((size_t)f * nch + ch) * KW + (KW - 1 - q)];
  for (int f = 0; f < C; ++f) { b1[f] = hp[1][f] + hp[2][f]; b2[f] = hp[4][f] + hp[5][f]; }
  // conv2 forward / transposed: K index ((p'*kw2 + q')*32 + channel)
  const size_t K2 = (size_t)kh2 * kw2 * CP;
  std::vector<float> B2(K2 * C, 0.f), Bt2(K2 * C, 0.f);
  for (int fo = 0; fo < C; ++fo)
    for (int ci = 0; ci < C; ++ci)
      for (int p = 0; p < kh2; ++p)
        for (int q = 0; q < kw2; ++q) {
          const float v = W2[(((size_t)fo * C + ci) * kh2 + p) * kw2 + q];
          B2[(((size_t)(kh2 - 1 - p) * kw2 + (kw2 - 1 - q)) * CP + ci) * C + fo] = v;  // out channel fo <- in ci
          Bt2[(((size_t)p * kw2 + q) * CP + fo) * C + ci] = v;                        // InverseLayer: in fo -> out ci
        }
  DCS_TRY(tc_weight_create(B1.data(), C, nch * KW, C, &c.tW[0], &m->dev));
  DCS_TRY(tc_weight_create(B2.data(), C, (int)K2, C, &c.tW[1], &m->dev));
  DCS_TRY(tc_weight_create(Bt2.data(), C, (int)K2, C, &c.tW[3], &m->dev));
  {  // bottleneck: rows permuted from Lasagne's (f', i, v) flattening to (i, v, f' padded to 32)
    std::vector<float> Bfc((size_t)flatp * c.nfc, 0.f);
    for (int f = 0; f < C; ++f)
      for (int i = 0; i < h2; ++i)
        for (int v = 0; v < w2; ++v)
          memcpy(&Bfc[(((size_t)i * w2 + v) * CP + f) * c.nfc], &Wfc[(((size_t)f * h2 + i) * w2 + v) * c.nfc],
                 c.nfc * sizeof(float));
    DCS_TRY(tc_weight_create(Bfc.data(), c.nfc, (int)flatp, c.nfc, &c.tW[2], &m->dev));
  }
  for (int d = 0; d < ndec; ++d) {  // decoder dense layers: columns permuted the same way
    const float* Wd = hp[8 + 2 * d];
    const float* bd = hp[9 + 2 * d];
    std::vector<float> Bd((size_t)c.nfc * flatp, 0.f), bb((size_t)flatp, 0.f);
    for (int f = 0; f < C; ++f)
      for (int i = 0; i < h2; ++i)
        for (int v = 0; v < w2; ++v) {
          const size_t col = ((size_t)i * w2 + v) * CP + f, src = ((size_t)f * h2 + i) * w2 + v;
          bb[col] = bd[src];
          for (int o = 0; o < c.nfc; ++o) Bd[(size_t)o * flatp + col] = Wd[(size_t)o * flat + src];
        }
    DCS_TRY(tc_weight_create(Bd.data(), flatp, c.nfc, (int)flatp, &c.tW[4 + d], &m->dev));
    DCS_TRY(upload(bb, &c.bdec[d], &m->dev));
  }
  // K3s filter banks (one per conv1 input channel): w[ch][dd][f][r] = W1[f][ch][KW-1-r-sw1*dd]
  const int ND = (KW + c.sw1 - 1) / c.sw1;
  std::vector<float> Wsc((size_t)nch * ND * 32 * 4, 0.f);
  for (int ch = 0; ch < nch; ++ch)
    for (int dd = 0; dd < ND; ++dd)
      for (int f = 0; f < C; ++f)
        for (int r = 0; r < c.sw1; ++r) {
          const int q = KW - 1 - r - c.sw1 * dd;
          if (q >= 0) Wsc[(((size_t)ch * ND + dd) * 32 + f) * 4 + r] = W1[((size_t)f * nch + ch) * KW + q];
        }
  std::vector<float> bfc(hp[7], hp[7] + c.nfc), bout(hp[want - 1], hp[want - 1] + m->nsrc);
  struct { const std::vector<float>* h; float** d; } ups[] = {{&b1, &c.b1}, {&b2, &c.b2}, {&bfc, &c.bfc}, {&bout, &c.bout}, {&Wsc, &c.Wsc}};
  for (auto& u : ups) DCS_TRY(upload(*u.h, u.d, &m->dev));
  return DCS_OK;
}

int sconv_forward(dcs_ctx* ctx, const dcs_model* m, const NetCall& n, cudaStream_t st) {
  const dcs_sconv& c = m->sc;
  const int tc = m->tc, step = n.step, CP = 32, C = 30;
  const int J = c.J, WP = c.WP, kh2 = c.kh2, kw2 = c.kw2, h2 = c.h2, w2 = c.w2, HP = c.HP, WPP = c.WPP, ndec = c.ndec;
  const int64_t T = n.T, ldf = n.ldf, P = n.P, Tp = n.Tp;
  const int64_t U = Tp - kh2 + 1;  // conv2 output rows
  DCS_REQUIRE(P * ndec * tc * WP < ((int64_t)1 << 31) && Tp * J < ((int64_t)1 << 31), "clip too long for 32-bit row indices");
  const int64_t flatp = (int64_t)h2 * w2 * CP;
  DCS_TRY(ensure_layout(ctx, NET_H1, (size_t)Tp * J * CP * 4, n.sig, st));
  DCS_TRY(ensure_layout(ctx, NET_H2, (size_t)U * w2 * CP * 4, n.sig, st));
  DCS_TRY(ensure_layout(ctx, NET_Z, (size_t)P * c.nfc * 4, n.sig, st));
  DCS_TRY(ensure_layout(ctx, NET_APAD, ((size_t)P * ndec * HP * WPP + kw2 + 1) * CP * 4, n.sig, st));
  DCS_TRY(ensure_layout(ctx, NET_G, (size_t)P * ndec * tc * WP * CP * 4, n.sig, st));
  float *H1 = ctx->net[NET_H1].as<float>(), *H2 = ctx->net[NET_H2].as<float>(), *z = ctx->net[NET_Z].as<float>();
  float *ap = ctx->net[NET_APAD].as<float>(), *G = ctx->net[NET_G].as<float>();
  float* Hp = H1;
  uint8_t* tie = nullptr;
  if (c.pool) {
    DCS_TRY(ensure_layout(ctx, NET_POOLED, (size_t)Tp * WP * CP * 4, n.sig, st));
    DCS_TRY(ensure_layout(ctx, NET_TIE, (size_t)Tp * WP * CP, n.sig, st));
    Hp = ctx->net[NET_POOLED].as<float>();
    tie = ctx->net[NET_TIE].as<uint8_t>();
  }

  {  // conv1 + biases: rows (t, j) are 30-sample windows of the magnitude frame, stride sw1
    ProfScope ps(ctx, "enc_conv1_gemm", st);
    GemmDesc g = gemm_plain(n.in, 0, nullptr, C, c.b1, H1, CP, (int)(Tp * J), C, 30 * c.nch, 0);
    g.m_inner = J; g.a_so = ldf; g.a_si = c.sw1;
    g.k_seg = 30; g.k_ss = n.in_plane;      // one 30-tap segment per input channel
    g.a_valid_rows = (int)(T * J);
    DCS_TRY(launch_gemm_tc(ctx, g, c.tW[0], st));
  }
  if (c.pool) {
    ProfScope ps(ctx, "enc_maxpool", st);
    DCS_TRY(launch_pool4(ctx, H1, Hp, tie, Tp, J, WP, st));
    if (ctx->pool_tap) {   // inspection tap (parity tests): the discrete un-pool routing decisions of this call
      const int64_t n = T * WP * CP;
      DCS_REQUIRE(ctx->pool_tap_cap >= n, "pool tap holds %lld bytes, this call produced %lld", (long long)ctx->pool_tap_cap, (long long)n);
      DCS_CUDA(cudaMemcpyAsync(ctx->pool_tap, tie, (size_t)n, cudaMemcpyDeviceToDevice, st));
    }
  }
  {  // conv2 + biases, once per (frame offset u, position v): K = kh2 time taps x (kw2 x 32) contiguous
    ProfScope ps(ctx, "enc_conv2_gemm", st);
    GemmDesc g = gemm_plain(Hp, 0, nullptr, C, c.b2, H2, CP, (int)(U * w2), C, kh2 * kw2 * CP, 0);
    g.m_inner = w2; g.a_so = (int64_t)WP * CP; g.a_si = CP;
    g.k_seg = kw2 * CP; g.k_ss = (int64_t)WP * CP;
    DCS_TRY(launch_gemm_tc(ctx, g, c.tW[1], st));
  }
  {  // bottleneck: patch k = h2 consecutive rows of H2 starting at k*step
    ProfScope ps(ctx, "bottleneck_gemm", st);
    GemmDesc g = gemm_plain(H2, (int64_t)step * w2 * CP, nullptr, c.nfc, c.bfc, z, c.nfc, (int)P, c.nfc, (int)flatp, 1);
    DCS_TRY(launch_gemm_tc(ctx, g, c.tW[2], st));
  }
  {  // decoder dense layers, scattered into the zero-padded buffer
    ProfScope ps(ctx, "dec_dense_gemm", st);
    for (int d = 0; d < ndec; ++d) {
      GemmDesc g = gemm_plain(z, c.nfc, nullptr, flatp, c.bdec[d], ap + (int64_t)d * HP * WPP * CP,
                              (int64_t)ndec * HP * WPP * CP, (int)P, (int)flatp, c.nfc, 1);
      g.n_seg = w2 * CP; g.n_ss = (int64_t)WPP * CP; g.c_col0 = ((int64_t)(kh2 - 1) * WPP + (kw2 - 1)) * CP;
      DCS_TRY(launch_gemm_tc(ctx, g, c.tW[4 + d], st));
    }
  }
  {  // InverseLayer(conv2): rows (u, kd, jp) u-major so tiles can skip the all-zero time taps
    ProfScope ps(ctx, "dec_convT2_gemm", st);
    const int64_t KD = P * ndec;
    GemmDesc g = gemm_plain(ap, 0, nullptr, C, nullptr, G, CP, (int)(KD * tc * WP), C, kh2 * kw2 * CP, 0);
    g.m_inner = (int)(KD * WP); g.a_so = (int64_t)WPP * CP;
    g.m_inner2 = WP; g.a_si = (int64_t)HP * WPP * CP; g.a_s2 = CP;
    g.k_seg = kw2 * CP; g.k_ss = (int64_t)WPP * CP;
    g.cm_inner = (int)(KD * WP); g.c_so = (int64_t)WP * CP;
    g.cm_inner2 = WP; g.c_si = (int64_t)tc * WP * CP; g.c_s2 = CP;
    g.kc_rows = (int)(KD * WP); g.kc_unit = kw2 * CP; g.kc_pad = kh2 - 1; g.kc_n = h2; g.kc_taps = kh2;
    DCS_TRY(launch_gemm_tc(ctx, g, c.tW[3], st));
  }
  SconvMaskArgs a;
  a.arch = m->arch; a.G = G; a.tie = tie; a.W = c.Wsc; a.bout = c.bout; a.X = n.X; a.S = n.S;
  a.ldf = ldf; a.src_stride = n.src_stride; a.T = (int)T; a.P = (int)P; a.tc = tc; a.overlap = n.overlap; a.F = m->F;
  a.J = J; a.WP = WP;
  a.p_base = 0; a.t0 = 0; a.t1 = (int)T;
  ProfScope ps(ctx, "dec_convT1_mask_xfade", st);
  if (!ctx->debug_simt_gemm) {
    DCS_REQUIRE(sconv_mask_tc_supported(a), "sconv_forward: tensor-core mask kernel does not take this shape");
    return launch_sconv_mask_tc(ctx, a, st, n.M);
  }
  return launch_sconv_mask(ctx, a, st, n.M);    // FFMA twin: cross-check (DCS_DEBUG_SIMT_GEMM=1)
}

}  // namespace dcs
