// dsd_model.cu -- the DSD100 / hiphopss network and its stereo / ILD variant on the GPU: weight re-layout +
// orchestration.  Every layer runs on the tensor cores: conv1, conv2 and the bottleneck as strided-view GEMMs
// (gemm_tc.cu), once per frame; the decoder dense layers (dsd_dense_tc.cu) and InverseLayer(conv2)
// (dsd_convT2_tc.cu) on their own kernels; then K3 (dsd_tc.cu, or dsd.cu): InverseLayer(conv1) + mask +
// cross-fade + phase.
#include "common.cuh"

namespace dcs {

int model_create_dsd(dcs_model* m, int nparams, const float* const* hp, const int64_t* shp, const int* nd) {
  dcs_dsd& ds = m->dsd;
  const int F = m->F, tc = m->tc;
  // DSD100 / hiphopss: 1 input channel, 128-wide bottleneck, 3 decoders feeding 4 outputs
  // (separate_dsd.py:196-231); stereo / ILD: 2 input channels, 256-wide bottleneck, one decoder per
  // source, 4 x 2 outputs ordered (source, channel) (trainCNN_ILD_DSD100.py:88-108)
  const bool ild = m->arch == DCS_ARCH_DSD_ILD;
  const int nch = ild ? 2 : 1, ndec = ild ? 4 : 3, nfc = ild ? 256 : 128, nout = 4 * nch;
  const int C1 = 50, C2 = 50, kh2 = tc / 2, h2 = tc - kh2 + 1, flat = C2 * h2;
  ds.C1 = C1; ds.C2 = C2; ds.kh2 = kh2; ds.h2 = h2; ds.nfc = nfc; ds.ndec = ndec; m->nsrc = 4; m->nch = nch;
  const int want = 8 + 2 * ndec + 1;
  if (nparams != want) { set_error("this DSD model needs %d parameter arrays, got %d (SURVEY.md App. A.4)", want, nparams); return DCS_EMODEL; }
  bool ok = shape_is(shp + 0, nd[0], 4, C1, nch, 1, F) && shape_is(shp + 4, nd[1], 1, C1) &&
            shape_is(shp + 8, nd[2], 1, C1) && shape_is(shp + 12, nd[3], 4, C2, C1, kh2, 1) &&
            shape_is(shp + 16, nd[4], 1, C2) && shape_is(shp + 20, nd[5], 1, C2) &&
            shape_is(shp + 24, nd[6], 2, flat, nfc) && shape_is(shp + 28, nd[7], 1, nfc) &&
            shape_is(shp + 4 * (want - 1), nd[want - 1], 1, nout);
  for (int d = 0; d < ndec; ++d)
    ok = ok && shape_is(shp + 4 * (8 + 2 * d), nd[8 + 2 * d], 2, nfc, flat) && shape_is(shp + 4 * (9 + 2 * d), nd[9 + 2 * d], 1, flat);
  if (!ok) { set_error("DSD parameter shapes do not match feat_size=%d time_context=%d", F, tc); return DCS_EMODEL; }
  const int64_t ldf = dcs_padded_bins(2 * (F - 1));
  ds.ldw = ldf;
  const float *W1 = hp[0], *W2 = hp[3], *Wfc = hp[6];
  // channel pitch of the activation buffers: 52 floats, so that every row and every time step starts
  // on a 16-byte boundary (what the TMA-fed GEMM needs); the K index of each weight follows the
  // same pitch with zero rows at the two pad channels
  const int C1p = (C1 + 3) / 4 * 4, C2p = (C2 + 3) / 4 * 4, flatp = C2p * h2;
  ds.C1p = C1p; ds.C2p = C2p;
  // W1f: conv1 as a GEMM weight, K index = ch * F + bin; W1t: its transpose per input channel for K3
  std::vector<float> W1f((size_t)nch * ldf * C1, 0.f), W1t((size_t)nch * C1 * ldf, 0.f), b1(C1), W2c((size_t)kh2 * C1p * C2, 0.f),
      Wt2((size_t)kh2 * C2p * C1, 0.f), b2(C2), Wfcp((size_t)flatp * nfc, 0.f), Wdec((size_t)nfc * ndec * flatp, 0.f),
      bdec((size_t)ndec * flatp, 0.f);
  for (int f = 0; f < C1; ++f)
    for (int ch = 0; ch < nch; ++ch)
      for (int b = 0; b < F; ++b) {
        const float v = W1[((size_t)f * nch + ch) * F + (F - 1 - b)];  // flip_filters
        W1f[((size_t)ch * F + b) * C1 + f] = v;
        W1t[((size_t)ch * C1 + f) * ldf + b] = v;
      }
  for (int f = 0; f < C1; ++f) b1[f] = hp[1][f] + hp[2][f];
  for (int f = 0; f < C2; ++f) b2[f] = hp[4][f] + hp[5][f];
  for (int f = 0; f < C2; ++f)
    for (int c = 0; c < C1; ++c)
      for (int q = 0; q < kh2; ++q) {
        const float v = W2[((size_t)f * C1 + c) * kh2 + q];
        W2c[((size_t)(kh2 - 1 - q) * C1p + c) * C2 + f] = v;  // conv2 forward, tap p' = kh2-1-q
        Wt2[((size_t)q * C2p + f) * C1 + c] = v;              // InverseLayer(conv2)
      }
  for (int f = 0; f < C2; ++f)
    for (int i = 0; i < h2; ++i)
      memcpy(&Wfcp[((size_t)i * C2p + f) * nfc], &Wfc[((size_t)f * h2 + i) * nfc], nfc * sizeof(float));
  for (int d = 0; d < ndec; ++d) {
    const float* Wd = hp[8 + 2 * d];
    const float* bd = hp[9 + 2 * d];
    for (int f = 0; f < C2; ++f)
      for (int i = 0; i < h2; ++i) {
        const size_t col = (size_t)d * flatp + (size_t)i * C2p + f;
        bdec[col] = bd[f * h2 + i];
        for (int o = 0; o < nfc; ++o) Wdec[(size_t)o * ndec * flatp + col] = Wd[(size_t)o * flat + f * h2 + i];
      }
  }
  // output bias per channel: bout[ch][s] = b[(s, ch)] (one K3 launch per channel)
  std::vector<float> bout((size_t)nch * 4), bfc(hp[7], hp[7] + nfc);
  for (int ch = 0; ch < nch; ++ch)
    for (int sidx = 0; sidx < 4; ++sidx) bout[(size_t)ch * 4 + sidx] = hp[want - 1][sidx * nch + ch];
  struct { const std::vector<float>* h; float** d; } ups[] = {
      {&b1, &ds.b1}, {&b2, &ds.b2}, {&bfc, &ds.bfc}, {&bdec, &ds.bdec}, {&W1t, &ds.W1t}, {&bout, &ds.bout}};
  for (auto& u : ups) DCS_TRY(upload(*u.h, u.d, &m->dev));
  DCS_TRY(tc_weight_create(W1f.data(), C1, nch * F, C1, &ds.tW1f, &m->dev));
  DCS_TRY(tc_weight_create(W2c.data(), C2, kh2 * C1p, C2, &ds.tW2c, &m->dev));
  DCS_TRY(tc_weight_create(Wfcp.data(), nfc, flatp, nfc, &ds.tWfc, &m->dev));
  DCS_TRY(tc_weight_create(Wdec.data(), ndec * flatp, nfc, ndec * flatp, &ds.tWdec, &m->dev));
  DCS_TRY(tc_weight_create(Wt2.data(), C1, kh2 * C2p, C1, &ds.tWt2, &m->dev));
  return DCS_OK;
}

// the DSD layer sequence: n.in holds nch magnitude planes (nch = 1: the DSD100 net); masked spectra plane
// (s * nch + ch) at (s * nch + ch) * n.src_stride
int dsd_forward(dcs_ctx* ctx, const dcs_model* m, const NetCall& n, cudaStream_t st) {
  const dcs_dsd& ds = m->dsd;
  const int tc = m->tc, step = n.step, C1 = ds.C1, C2 = ds.C2, kh2 = ds.kh2, h2 = ds.h2, nfc = ds.nfc;
  const int C1p = ds.C1p, C2p = ds.C2p;   // channel pitch of H1 / H2 / the padded decoder activations
  const int nch = m->nch, ndec = ds.ndec;
  const int64_t T = n.T, ldf = n.ldf, P = n.P, Tp = n.Tp;
  DCS_REQUIRE(P * ndec * tc < (int64_t)1 << 31, "clip too long (%lld patches)", (long long)P);
  const int HP = h2 + 2 * (kh2 - 1), ldg = (C1 + 3) / 4 * 4;
  // zero on (re)allocation or layout change; afterwards only the interior (rows and the C of the
  // Cp channels) is ever written, so the zero padding persists
  DCS_TRY(ensure_layout(ctx, NET_H1, (size_t)Tp * C1p * 4, n.sig, st));
  DCS_TRY(ensure_layout(ctx, NET_H2, (size_t)(Tp - kh2 + 1) * C2p * 4, n.sig, st));
  DCS_TRY(ensure_layout(ctx, NET_Z, (size_t)P * nfc * 4, n.sig, st));
  DCS_TRY(ensure_layout(ctx, NET_APAD, (size_t)P * ndec * HP * C2p * 4, n.sig, st));
  // G: the transposed conv2 output, patch-major [P][ndec][tc][ldg]
  DCS_TRY(ensure_layout(ctx, NET_G, (size_t)P * ndec * tc * ldg * 4, n.sig, st));
  float *H1 = ctx->net[NET_H1].as<float>(), *H2 = ctx->net[NET_H2].as<float>(), *z = ctx->net[NET_Z].as<float>();
  float *ap = ctx->net[NET_APAD].as<float>(), *G = ctx->net[NET_G].as<float>();

  // conv1 + both biases, once per frame (kernel height 1): H1[Tp][C1] = mag[T][nch x F] * W1f
  GemmDesc g1 = gemm_plain(n.in, ldf, nullptr, C1, ds.b1, H1, C1p, (int)Tp, C1, nch * m->F, 0);
  if (nch > 1) { g1.k_seg = m->F; g1.k_ss = n.in_plane; }   // one K segment per input channel plane
  g1.a_valid_rows = (int)T;  // util patcher: frames beyond T are zero input
  { ProfScope ps(ctx, "enc_conv1_gemm", st); DCS_TRY(launch_gemm_tc(ctx, g1, ds.tW1f, st)); }
  // conv2 + both biases, once per frame offset: rows overlap in H1 (stride C1p, length kh2*C1p)
  GemmDesc g2 = gemm_plain(H1, C1p, nullptr, C2, ds.b2, H2, C2p, (int)(Tp - kh2 + 1), C2, kh2 * C1p, 0);
  { ProfScope ps(ctx, "enc_conv2_gemm", st); DCS_TRY(launch_gemm_tc(ctx, g2, ds.tW2c, st)); }
  // bottleneck: patch k reads H2 rows k*step .. k*step+h2-1 (contiguous h2*C2p floats)
  GemmDesc g3 = gemm_plain(H2, (int64_t)step * C2p, nullptr, nfc, ds.bfc, z, nfc, (int)P, nfc, h2 * C2p, 1);
  { ProfScope ps(ctx, "bottleneck_gemm", st); DCS_TRY(launch_gemm_tc(ctx, g3, ds.tWfc, st)); }
  // the decoder dense layers side by side, scattered into the interior rows of the zero-padded buffer: the
  // tensor-core kernel keeps a slab of the weight in shared memory over many patches (dsd_dense_tc.cu)
  {
    ProfScope ps(ctx, "dec_dense_gemm", st);
    DsdDenseArgs a4;
    a4.z = z; a4.bias = ds.bdec; a4.apad = ap; a4.P = (int)P; a4.tc = tc; a4.ndec = ndec; a4.nfc = nfc;
    DCS_TRY(launch_dsd_dense_tc(ctx, a4, ds.tWdec, st));
  }
  // InverseLayer(conv2): full correlation on the padded activations, rows (k, d, u).  The tensor-core
  // kernel reads each (patch, decoder) pair's interior rows once into shared memory (dsd_convT2_tc.cu).
  {
    ProfScope ps(ctx, "dec_convT2_gemm", st);
    DsdConvT2Args a5;
    a5.apad = ap; a5.G = G; a5.ldg = ldg; a5.npairs = (int)(P * ndec); a5.tc = tc;
    DCS_TRY(launch_dsd_convT2_tc(ctx, a5, ds.tWt2, st));
  }
  // InverseLayer(conv1) + bias + ReLU + mask + cross-fade + phase; the stereo net: once per channel
  // with that channel's conv1 weights, output biases and mixture STFT (trainCNN_ILD_DSD100.py:183-186)
  ProfScope ps(ctx, "dec_convT1_mask_xfade", st);
  // else the FFMA kernel: > 6 patches per frame, cross-check
  const bool tc_path = !ctx->debug_simt_gemm && (tc + step - 1) / step <= 6;
  for (int ch = 0; ch < nch; ++ch) {
    DsdMaskArgs a;
    a.G = G; a.ldg = ldg; a.W1t = ds.W1t + (int64_t)ch * C1 * ds.ldw; a.ldw = (int)ds.ldw; a.bout = ds.bout + 4 * ch;
    a.ldf = ldf; a.T = (int)T; a.P = (int)P; a.tc = tc; a.overlap = n.overlap; a.F = m->F;
    a.ndec = ndec;
    a.src_stride = nch * n.src_stride;
    float* M = nullptr;   // masks mode: plane (s * nch + ch), the layout of the spectra
    if (n.M) {
      a.X = nullptr; a.S = nullptr; M = n.M + ch * n.src_stride;
    } else {
      a.X = n.X + ch * n.x_plane; a.S = n.S + ch * n.src_stride;
    }
    if (tc_path) {
      DCS_REQUIRE(dsd_mask_tc_supported(a), "dsd_forward: tensor-core mask kernel does not take this shape");
      DCS_TRY(launch_dsd_mask_tc(ctx, a, st, M));
    } else {
      DCS_TRY(launch_dsd_mask(ctx, a, st, M));
    }
  }
  return DCS_OK;
}

}  // namespace dcs
