"""The fused last stage of every network -- InverseLayer(conv1) + output bias + ReLU + soft ratio mask + sequential patch
cross-fade + times the mixture STFT -- on both engines against a float64 reference, element by element, through
dcs_dsd_mask_f32 (dsd_tc.cu / dsd.cu) and dcs_sconv_mask_f32 (sconv_tc.cu / sconv.cu).

Reference.  Float64 from the fp32 operands, out of the oracle's pieces: oracle.nets.conv2d_inverse on the Lasagne
conv1.W (stride STRIDE for the strided nets), after the un-pool routed by the case's tie bits (every set bit receives
the value); oracle.nets.soft_masks with the family's rule (DSD100: source 4 = decoder 2 with bias 4, all-zero bins 1/4;
iKala: 1/2; ILD and the Bach10 nets: 0); the cross-fade weights of oracle.patch.crossfade_weights, the closed form of
overlapadd_multi (test_fade_weights_match_overlapadd_multi pins one to the other); the product with X.  The kernel
layouts are made from the Lasagne weights by w1t_layout / bank_layout; test_layouts_reproduce_conv2d_inverse evaluates
the kernels' index formulas on them against conv2d_inverse.

Per-element bound, with u = 2^-24.  Per frame t, covering slot j (patch k_lo(t) + j, frame-in-patch p), bin b and
source s: y = the transposed-conv1 value, S_y = sum |G W| of its terms (float64), pre = y + bout_s.
  e_y = c_e S_y, where c_e follows each engine's accumulation plan:
    - FFMA: fp32 FMA chains over the K = 50 (DSD) or 30 ND (K3s) terms: c = (K + 4) u.
    - dsd_tc.cu, 3xTF32: every product a b = (ah + al)(bh + bl) is formed as ah bh + ah bl + al bh from TF32 operands
      (the lo parts truncated again), off by < 3 * 2^-20 = 48u relative.  All 21 k8 products of one value go into ONE
      truncating accumulator, the 14 correction steps first: a step adds up to 9 terms (8 products and the
      accumulator) with truncation after alignment, < 2u per term of the step's sum of magnitudes, 18u.  The
      accumulator entering main step j holds < 2^-9 S + sum_{i<j} S_i, so the 7 main steps cost
      18u sum_j (2^-9 S + sum_{i<=j} S_i) <= 18u (7 + 0.014) S, and the corrections 14 * 18u * 2^-9 S < 0.5u S:
      c = 48u + 126.3u + 0.5u < 176u, taken as 192u.
    - sconv_tc.cu, 3xTF32: per filter bank 12 k8 products (K = 32 channels) in one truncating accumulator, corrections
      first: 48u + 18u (4 + 0.008) + 0.1u < 121u of that value's S; then an fp32 sum over the ND taps, (ND - 1) u of
      sum |Z| <= S_y: c = (128 + ND) u.
  e_p = e_y + u |pre| (the fp32 bias addition; ReLU is 1-Lipschitz), E = sum_s e_p + 3u tot (tot = sum_s relu(pre)
  and its fp32 summation).
  A slot is well-conditioned if tot > 2E (the mask's denominator cannot reach 0), or if every pre_s < -e_y,s: then
  the kernel's pre is negative too, tot is exactly 0 and the mask is exactly the rule's all-zero value ("settled").
  Its mask error is (e_p,s + m_s E) / (tot - E) (0 if settled), plus 8u for the reciprocal or division, the two
  products and the fused add of the epilogue.
A frame's mask error is the omega-weighted sum over its n slots plus (8 + 4n) u for the fp32 fade weights (up and
down each carry 2u relative; omega_j is a product of up to n of them) and the two roundings of each step of the
recurrence.  The bound on S is that error times |X|, plus 2u |m| |X| for the final product.
A frame and bin with an ill-conditioned slot of non-zero weight (the mask's discontinuity, where any fp32 evaluation
may land on either side) is held to admissibility only: the value is finite; |S_s| <= (1 + tol) |X|; DSD / iKala rule
|sum_s S_s - w X| <= tol |X| (w = sum of the frame's weights), 0-rule sum_s |S_s| <= (1 + tol) |X|; tol = 1e-6 + 8n u,
the fade's own rounding over n slots.  Every case requires at least 99 % of its (frame, bin) pairs to be
well-conditioned, so none passes vacuously.
Plain TF32 (hi products only: the kernel without its corrections) errs by ~2^-10 per product, 50x the tensor-core c_e on
sign-coherent terms; the 'coherent' cases (non-negative G and W, biases the size of y, different per source) make
such a bias visible in the masks.  test_bound_has_teeth shows the bound accepting an emulation of each engine's plan
and rejecting plain TF32 and six index mutations.

Exact parts: frames no patch covers are 0; 0-rule bins whose every slot is settled are 0; a one-slot frame whose
sources are all settled is exactly 1/4 X (DSD100) or 1/2 X (iKala).

Every case fills S with a NaN-payload sentinel and every input element the kernels never read with NaN (X pad columns
and plane gaps, W1t columns >= F, filter-bank components r >= STRIDE, G columns >= 52 (DSD), G rows of patches >= P,
and in chunked cases everything before the G pointer), fails if a sentinel changes or a stored value is not finite,
runs twice per engine and requires the same bits, and with DCS_TEST_RECORDS set records its worst error / bound ratio
(tests/parity.py).  The elements the kernels multiply against zero weights (DSD G columns 50..51, K3s G channels
30..31) hold finite garbage."""
import ctypes
import os
import sys
import zlib

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from parity import record  # noqa: E402
from oracle import nets, patch  # noqa: E402

U = 2.0 ** -24
SLACK = 64                           # NaN / sentinel elements before and after every buffer
S_SENTINEL = np.uint32(0x7FC5A5A5)   # quiet NaN with a payload no kernel produces
ARCH_IDS = {"dsd": 0, "ikala": 1, "ikala_nopool": 2, "bach10": 3, "bach10_score": 4, "dsd_ild": 5, "bach10_score_1x1": 6}
# K3s families: conv1 taps KW at STRIDE, sources, decoders, filter banks, max-pool width, all-zero rule
K3S = {"bach10": (30, 4, 4, 4, 1, 0, "bach10"), "bach10_score": (30, 4, 4, 1, 4, 0, "bach10"),
       "bach10_score_1x1": (5, 2, 4, 1, 4, 0, "bach10"), "ikala": (30, 3, 2, 2, 1, 4, "dsd"),
       "ikala_nopool": (30, 3, 2, 2, 1, 0, "dsd")}
OUT_TC = {"bach10": 121, "bach10_score": 121, "bach10_score_1x1": 126, "ikala": 119, "ikala_nopool": 119}   # 128 - (ND-1)


def _rng(name):
    return np.random.default_rng(zlib.crc32(name.encode()))


def _ldf(F):
    return (F + 7) // 8 * 8


def c_ffma(K):
    return U * (K + 4)


C_TC_DSD = 192 * U


def c_tc_k3s(nd):
    return U * (128 + nd)


# ---------------------------------------------------------------------------------------------- kernel layouts
def w1t_layout(W, ch, ldw):
    """Lasagne conv1.W [50, nch, 1, F] -> W1t [50][ldw]: W1t[c][b] = W[c, ch, 0, F-1-b]; columns >= F are NaN"""
    F = W.shape[3]
    out = np.full((W.shape[0], ldw), np.nan, np.float32)
    out[:, :F] = W[:, ch, 0, ::-1]
    return out


def bank_layout(W, stride):
    """Lasagne conv1.W [30, nw, 1, KW] -> float4 banks [nw][ND][32][4]: [o][dd][f][r] = W[f, o, 0, KW-1-r-stride*dd];
    0 where that tap index is negative or f >= 30, NaN in the components r >= stride (never read)"""
    nf, nw, _, KW = W.shape
    nd = -(-KW // stride)
    out = np.zeros((nw, nd, 32, 4), np.float32)
    for dd in range(nd):
        for r in range(4):
            q = KW - 1 - r - stride * dd
            if r >= stride:
                out[:, dd, :, r] = np.nan
            elif q >= 0:
                out[:, dd, :nf, r] = W[:, :, 0, q].T
    return out


def k3s_kernel_y(gu, bank, stride, F, arith="f64"):
    """the kernels' index formula  Y[o][STRIDE*m + r] = sum_{dd, f < 32} Gu[m - dd][f] * bank[o][dd][f][r]  on
    gu [B, J, 32] (one decoder): [B, nw, F].  arith: 'f64', or the tensor-core plan 'tc' (3xTF32, fp32 tap sum),
    'tf32' (hi products only), 'ffma' (one fp32 FMA chain over dd, f)"""
    B, J, _ = gu.shape
    nw, nd = bank.shape[:2]
    mtot = -(-F // stride)
    w = np.nan_to_num(bank[..., :stride].astype(np.float64))       # [nw, nd, 32, stride]
    pos = np.zeros((B, mtot + nd, 32))
    pos[:, nd - 1:nd - 1 + min(J, mtot + 1)] = gu[:, :min(J, mtot + 1)]   # row m + nd - 1 - dd holds position m - dd
    y = np.zeros((B, nw, mtot, stride), np.float64 if arith == "f64" else np.float32)
    for dd in range(nd):
        g = pos[:, nd - 1 - dd:nd - 1 - dd + mtot]                  # [B, mtot, 32]
        if arith == "f64":
            y += np.einsum("bmf,ofr->bomr", g, w[:, dd])
        elif arith == "ffma":
            for f in range(32):
                y = (y.astype(np.float64) + g[:, None, :, f, None] * w[None, :, dd, f, None, :]).astype(np.float32)
        else:
            z = _tf32_dot(g.astype(np.float32), w[:, dd].astype(np.float32), arith == "tc")   # [B, nw, mtot, stride]
            y = (y.astype(np.float64) + z).astype(np.float32)
    return y.reshape(B, nw, mtot * stride)[..., :F]


def _trunc_tf32(x):
    return (np.ascontiguousarray(x, dtype=np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def _tf32_dot(g, w, corr):
    """sum over the 32-wide channel axis as the tensor cores do it: per k8 step the exact product sum of TF32 operands
    rounded into an fp32 accumulator; with `corr` the ah*bl and al*bh steps first.  g [B, M, K], w [O, K, R] ->
    [B, O, M, R]"""
    gh, wh = _trunc_tf32(g), _trunc_tf32(w)
    gl, wl = _trunc_tf32(g - gh), _trunc_tf32(w - wh)
    f = lambda x: x.astype(np.float64)
    acc = np.zeros((g.shape[0], w.shape[0], g.shape[1], w.shape[2]), np.float32)
    passes = [(gh, wl), (gl, wh), (gh, wh)] if corr else [(gh, wh)]
    for a, b in passes:
        for k0 in range(0, g.shape[2], 8):
            ks = slice(k0, k0 + 8)
            acc = (f(acc) + np.einsum("bmk,okr->bomr", f(a[..., ks]), f(b[:, ks]))).astype(np.float32)
    return acc


def dsd_kernel_y(g, w1t, F, arith="f64"):
    """Y[b] = sum_c G[c] W1t[c][b] for g [B, 52] (columns 50, 51 against zero rows), W1t [50][ldw]: [B, F]"""
    w = np.zeros((52, F), np.float32)
    w[:50] = w1t[:, :F]
    g = g[:, :52].astype(np.float32)
    if arith == "f64":
        return g.astype(np.float64) @ w.astype(np.float64)
    if arith == "ffma":
        y = np.zeros((g.shape[0], F), np.float32)
        for c in range(50):
            y = (y.astype(np.float64) + g[:, c:c + 1].astype(np.float64) * w[c].astype(np.float64)).astype(np.float32)
        return y
    return _tf32_dot(g[:, None, :], w[None, :, :], arith == "tc")[:, 0, 0, :]


# ---------------------------------------------------------------------------------------------- float64 reference
def covering(frames, P, tc, ov):
    """k_lo and the number of patches covering each frame, as the kernels compute them"""
    step = tc - ov
    t = np.asarray(frames, np.int64)
    k_hi = np.minimum(t // step, P - 1)
    k_lo = np.where(t - tc + 1 > 0, -(-(t - tc + 1) // step), 0)
    return k_lo, np.maximum(k_hi - k_lo + 1, 0)


def fade_weights(frames, P, tc, ov):
    """omega [frames, slots]: weight of patch k_lo + j in frame t (oracle.patch.crossfade_weights)"""
    k_lo, n = covering(frames, P, tc, ov)
    om = np.zeros((len(frames), max(1, int(n.max()))))
    for i, t in enumerate(frames):
        for k, w in patch.crossfade_weights(int(t), P, tc, ov):
            om[i, k - k_lo[i]] = w
    return om


def _take(G, k, p):
    """G[k, :, p] for host arrays and device tensors"""
    if isinstance(G, np.ndarray):
        return G[k, :, p]
    import torch
    kk, pp = torch.from_numpy(k).to(G.device), torch.from_numpy(p).to(G.device)
    return G[kk, :, pp].cpu().numpy()


def dsd_slot_y(case, ch, g):
    """g [B, ndec, ldg] -> y, S_y [B, 4, F] (sources) through conv2d_inverse on the Lasagne weights"""
    W = case["W"].astype(np.float64)
    B, F = g.shape[0], W.shape[3]
    ys, Ss = [], []
    for d in range(case["ndec"]):
        gi = g[:, d, :50].astype(np.float64)[:, :, None, None]
        ys.append(nets.conv2d_inverse(gi, W, (B, W.shape[1], 1, F))[:, ch, 0])
        Ss.append(nets.conv2d_inverse(np.abs(gi), np.abs(W), (B, W.shape[1], 1, F))[:, ch, 0])
    dec = (0, 1, 2, 1) if case["ndec"] == 3 else (0, 1, 2, 3)
    return np.stack([ys[d] for d in dec], 1), np.stack([Ss[d] for d in dec], 1)


def unpool(g, tie):
    """InverseLayer(pool): g [B, ndec, WP, 32] pooled, tie [B, WP, 32] -> [B, ndec, 4 WP, 32]; every position whose
    tie bit is set receives the window's value"""
    bits = ((tie[:, None, :, :, None] >> np.arange(4, dtype=np.uint8)) & 1).astype(np.float64)   # [B, 1, WP, 32, 4]
    u = g[..., None] * bits
    return u.transpose(0, 1, 2, 4, 3).reshape(g.shape[0], g.shape[1], 4 * g.shape[2], 32)


def k3s_slot_y(case, g, tie):
    """g [B, ndec, WP, 32] -> y, S_y [B, nsrc, F] through the un-pool and conv2d_inverse (stride STRIDE)"""
    KW, stride, nsrc, ndec, nw, pool, _ = K3S[case["arch"]]
    W = case["W"].astype(np.float64)
    B, F, J = g.shape[0], case["F"], case["J"]
    g = g.astype(np.float64)
    if pool:
        g = unpool(g, tie)
    gu = np.zeros((B, ndec, J, 30))
    n = min(J, g.shape[2])
    gu[:, :, :n] = g[:, :, :n, :30]
    ys, Ss = [], []
    for d in range(ndec):
        x = gu[:, d].transpose(0, 2, 1)[:, :, None, :]
        ys.append(nets.conv2d_inverse(x, W, (B, nw, 1, F), (1, stride))[:, :, 0])
        Ss.append(nets.conv2d_inverse(np.abs(x), np.abs(W), (B, nw, 1, F), (1, stride))[:, :, 0])
    if nw == 1:
        return np.concatenate(ys, 1), np.concatenate(Ss, 1)
    return ys[0], Ss[0]


def slot_masks(pre, Sy, c_e, rule, nsrc):
    """masks of one slot [B, nsrc, F] and their error bound; ok = well-conditioned, settled = every pre < -e_y"""
    e_y = c_e * Sy
    p = np.maximum(pre, 0.0)
    tot = p.sum(1)
    m = nets.soft_masks(p, rule, nsrc)
    e_p = e_y + U * np.abs(pre)
    E = e_p.sum(1) + 3 * U * tot
    settled = (pre < -e_y).all(1)
    well = tot > 2 * E
    err = (e_p + m * E[:, None]) / np.where(well, tot - E, 1.0)[:, None] + 8 * U
    err = np.where(settled[:, None], 0.0, err)
    return m, err, well | settled, settled


def reference_masks(case, frames, mask_set=0, y_fn=None):
    """the cross-faded masks of `frames` and their bounds: M, errM [B, nsrc, F], ill [B, F] (an ill-conditioned slot of
    non-zero weight), settled_all [B, F], n [B] (covering slots), w [B] (sum of the weights).  y_fn(k, p, frames) ->
    (y, S_y) overrides the float64 transposed conv (the emulations of test_bound_has_teeth)."""
    T, P, tc, ov, F = case["T"], case["P"], case["tc"], case["ov"], case["F"]
    frames = np.asarray(frames, np.int64)
    k_lo, n = covering(frames, P, tc, ov)
    om = fade_weights(frames, P, tc, ov)
    step = tc - ov
    if case["kind"] == "dsd":
        nsrc, rule = 4, ("dsd" if case["ndec"] == 3 else "bach10")
        bout = case["bout"][mask_set].astype(np.float64)
        c_e = C_TC_DSD if case["engine"] == "tc" else c_ffma(50)
    else:
        KW, stride, nsrc, _, _, _, rule = K3S[case["arch"]]
        nd = -(-KW // stride)
        bout = case["bout"].astype(np.float64)
        c_e = c_tc_k3s(nd) if case["engine"] == "tc" else c_ffma(30 * nd)
    B = len(frames)
    M = np.zeros((B, nsrc, F))
    errM = np.zeros((B, nsrc, F))
    ill = np.zeros((B, F), bool)
    settled_all = np.repeat((n > 0)[:, None], F, 1)
    for j in range(om.shape[1]):
        v = np.nonzero(j < n)[0]
        if v.size == 0:
            continue
        k = k_lo[v] + j
        p = frames[v] - k * step
        if y_fn is not None:
            y, Sy = y_fn(k, p, frames[v])
        elif case["kind"] == "dsd":
            y, Sy = dsd_slot_y(case, mask_set, _take(case["G"], k, p).astype(np.float64))
        else:
            tie = case["tie"][frames[v]] if case["tie"] is not None else None
            y, Sy = k3s_slot_y(case, _take(case["G"], k - case["p_base"], p), tie)
        pre = y + bout[None, :, None]
        m, err, ok, settled = slot_masks(pre, Sy, c_e, rule, nsrc)
        w = om[v, j][:, None, None]
        M[v] += w * m
        errM[v] += w * err
        ill[v] |= (om[v, j][:, None] > 0) & ~ok
        settled_all[v] &= settled
    errM += ((8 + 4 * n) * U)[:, None, None]
    return dict(M=M, errM=errM, ill=ill, settled_all=settled_all, n=n, w=om.sum(1), rule=rule, nsrc=nsrc)


def evaluate(ref, S, X):
    """S complex [nsrc, B, F] (one channel's planes) against the reference masks times X [B, F].  Returns the worst
    error / bound over the well-conditioned elements and the list of failed admissibility / exactness checks."""
    M = ref["M"].transpose(1, 0, 2)
    errM = ref["errM"].transpose(1, 0, 2)
    X = X.astype(np.complex128)
    aX = np.abs(X)
    S = S.astype(np.complex128)
    fails = []
    if not np.isfinite(S).all():
        return np.inf, ["%d values not finite" % int((~np.isfinite(S)).sum())]
    ill = ref["ill"][None]
    bnd = errM * aX + 2 * U * M * aX
    err = np.abs(S - M * X)
    ratio = np.where(ill, 0.0, np.where(err > 0, err / np.maximum(bnd, 1e-300), 0.0))
    worst = float(ratio.max())
    tol = (1e-6 + 8 * U * ref["n"])[None, :, None]
    if ill.any():
        bad = (np.abs(S) > (1 + tol) * aX) & ill
        if ref["rule"] == "dsd":
            bad |= (np.abs(S.sum(0) - ref["w"][:, None] * X) > tol[0] * aX)[None] & ill
        else:
            bad |= (np.abs(S).sum(0) > (1 + tol[0]) * aX)[None] & ill
        if bad.any():
            fails.append("%d inadmissible values at the mask discontinuity" % int(bad.sum()))
    uncovered = ref["n"] == 0
    if (S[:, uncovered] != 0).any():
        fails.append("frames no patch covers are not 0")
    if ref["rule"] == "bach10":
        if (S[:, ref["settled_all"]] != 0).any():
            fails.append("settled all-zero bins are not exactly 0")
    else:
        one = ref["settled_all"] & (ref["n"] == 1)[:, None]
        want = (np.complex64(1.0 / ref["nsrc"]) * X.astype(np.complex64)).astype(np.complex128)
        if (S[:, one] != want[None][:, one]).any():
            fails.append("one-slot all-zero bins are not exactly X / nsrc")
    return worst, fails


def well_fraction(ref):
    cov = ref["n"] > 0
    return 1.0 - float(ref["ill"][cov].mean()) if cov.any() else 1.0


# ---------------------------------------------------------------------------------------------- cases
def dsd_case(name, F, T, tc, ov, patcher="util", ndec=3, ldg=52, coherent=False, zero_slots=()):
    """a DSD-family argument set: Lasagne conv1.W [50, nch, 1, F], G [P, ndec, tc, ldg], bout [nch][4], X planes"""
    rng = _rng(name)
    nch = 2 if ndec == 4 else 1
    P = patch.num_patches(T, tc, ov, patcher)
    a = np.sqrt(6.0 / (51 * F))
    W = rng.uniform(-a, a, (50, nch, 1, F)).astype(np.float32)
    G = rng.standard_normal((P, ndec, tc, ldg), dtype=np.float32)
    sig = np.sqrt(50 / 3.0) * a
    bout = (rng.standard_normal((nch, 4)) * 0.7 * sig).astype(np.float32)
    if coherent:   # non-negative terms, biases of the size of y and different per source: relative errors of y show
        W, G = np.abs(W), np.abs(G)
        bout = np.tile(-np.array([0.2, 0.5, 0.8, 0.35]) * 50 * 0.8 * a / 2, (nch, 1)).astype(np.float32)
    G[..., 50:] = rng.uniform(-1e3, 1e3, G[..., 50:].shape)        # read by engine 1 against zero weight rows
    for k, p in zero_slots:                                          # subnormal totals: y = 0, pre = (1e-40, -1, -1, -1)
        G[k, :, p] = 0.0
    if zero_slots:
        bout[:] = np.float32([1e-40, -1, -1, -1])
    X = (rng.standard_normal((nch, T, F)) + 1j * rng.standard_normal((nch, T, F))).astype(np.complex64)
    return dict(kind="dsd", name=name, F=F, T=T, tc=tc, ov=ov, P=P, ndec=ndec, nch=nch, ldg=ldg, ldf=_ldf(F),
                W=W, G=G, bout=bout, X=X, p_base=0, t0=0, t1=T)


def k3s_case(name, arch, F, T, tc, ov, patcher="util", chunk=None, coherent=False, zero_slots=(), bias_mean=0.0):
    """a K3s argument set; chunk = (p_base, p0, p1): G holds patches p_base .. p1 - 1, frames [p0 step, p1 step) (or T);
    bias_mean (in units of the spread of y) makes all-zero slots rarer"""
    rng = _rng(name)
    KW, stride, nsrc, ndec, nw, pool, _ = K3S[arch]
    P = patch.num_patches(T, tc, ov, patcher)
    J = (F - KW) // stride + 1
    WP = J // 4 if pool else J
    step = tc - ov
    p_base, t0, t1, p_end = 0, 0, T, P
    if chunk:
        p_base, p0, p1 = chunk
        t0, t1, p_end = p0 * step, (T if p1 == P else p1 * step), p1
    a = np.sqrt(6.0 / ((30 + nw) * KW))
    W = rng.uniform(-a, a, (30, nw, 1, KW)).astype(np.float32)
    G = rng.standard_normal((p_end - p_base, ndec, tc, WP, 32), dtype=np.float32)
    sig = np.sqrt(30 * -(-KW // stride) / 3.0) * a
    bout = ((rng.standard_normal(nsrc) * 0.7 + bias_mean) * sig).astype(np.float32)
    if coherent:
        W, G = np.abs(W), np.abs(G)
        bout = (-np.array([0.2, 0.5, 0.8, 0.35])[:nsrc] * 30 * -(-KW // stride) * 0.8 * a / 2).astype(np.float32)
    G[..., 30:] = rng.uniform(-1e3, 1e3, G[..., 30:].shape)          # read by engine 1 against zero weight channels
    for k, p in zero_slots:
        G[k - p_base, :, p] = 0.0
    if zero_slots:
        bout[:] = np.float32([1e-40, -1, -1, -1][:nsrc])
    tie = rng.integers(1, 16, (T, WP, 32)).astype(np.uint8) if pool else None   # single, double, ..., all-four ties
    X = (rng.standard_normal((T, F)) + 1j * rng.standard_normal((T, F))).astype(np.complex64)
    return dict(kind="k3s", name=name, arch=arch, F=F, T=T, tc=tc, ov=ov, P=P, J=J, WP=WP, ldf=_ldf(F), W=W, G=G,
                bout=bout, X=X, tie=tie, p_base=p_base, t0=t0, t1=t1, nch=1)


SLOT_GEOMS = [(30, 0), (10, 5), (12, 8), (4, 3), (30, 24), (30, 25)]   # 1 .. 6 patches per frame
DSD_CASES = {
    "dsd_F513": lambda n: dsd_case(n, 513, 300, 30, 25),
    "dsd_F1025": lambda n: dsd_case(n, 1025, 300, 30, 25, "standalone"),
    "dsd_F1025_T1000": lambda n: dsd_case(n, 1025, 1000, 30, 25),          # 1125 items: CTA ranges cross tiles
    "dsd_F2049_T37": lambda n: dsd_case(n, 2049, 37, 30, 25),              # 85 items, a last group of 5 frames
    "dsd_F129": lambda n: dsd_case(n, 129, 120, 30, 25, "standalone"),     # the second tile holds only the Nyquist bin
    "dsd_overlap1": lambda n: dsd_case(n, 129, 120, 10, 1),
    "dsd_slots7": lambda n: dsd_case(n, 129, 150, 31, 26),                 # engine 0 only
    "dsd_slots16": lambda n: dsd_case(n, 129, 200, 64, 60),                # engine 0 only
    "dsd_ldg56": lambda n: dsd_case(n, 257, 100, 30, 25, ldg=56),
    "dsd_ild": lambda n: dsd_case(n, 513, 150, 30, 25, ndec=4),
    "dsd_ild_standalone": lambda n: dsd_case(n, 129, 97, 20, 15, "standalone", ndec=4),
    "dsd_coherent": lambda n: dsd_case(n, 257, 60, 30, 25, coherent=True),
    # defect: subnormal totals, in a one-slot frame, a zero-weight first frame of a later patch and a faded frame
    "dsd_subnormal": lambda n: dsd_case(n, 129, 400, 30, 25, zero_slots=((0, 2), (1, 0), (3, 2))),
    "dsd_ild_subnormal": lambda n: dsd_case(n, 129, 400, 30, 25, ndec=4, zero_slots=((0, 2), (1, 0), (3, 2))),
}
DSD_CASES.update({"dsd_slots%d" % (i + 1): (lambda g: lambda n: dsd_case(n, 129, 120, g[0], g[1]))(g)
                  for i, g in enumerate(SLOT_GEOMS)})
K3S_CASES = {
    "bach10_F2049": lambda n: k3s_case(n, "bach10", 2049, 40, 30, 25),     # 5 tiles of 121, bins past the last window
    "bach10_F129": lambda n: k3s_case(n, "bach10", 129, 120, 30, 25, "standalone"),
    "bach10_F257": lambda n: k3s_case(n, "bach10", 257, 120, 30, 25),
    "bach10_F129_T500": lambda n: k3s_case(n, "bach10", 129, 500, 30, 25),   # many CTAs per tile in time
    "bach10_slots30": lambda n: k3s_case(n, "bach10", 129, 100, 30, 29, bias_mean=0.5),   # 30 chances per bin of a kink
    "bach10_score": lambda n: k3s_case(n, "bach10_score", 1025, 60, 30, 25),
    "ikala_F513": lambda n: k3s_case(n, "ikala", 513, 120, 30, 25),          # positions 160..161 no window covers
    "ikala_nopool_F513": lambda n: k3s_case(n, "ikala_nopool", 513, 120, 30, 25, "standalone"),
    "ikala_nopool_F1025": lambda n: k3s_case(n, "ikala_nopool", 1025, 60, 30, 25),
    "s1x1_F253_tc19": lambda n: k3s_case(n, "bach10_score_1x1", 253, 120, 19, 14),
    "s1x1_chunk_interior": lambda n: k3s_case(n, "bach10_score_1x1", 2049, 1373, 30, 25, chunk=(123, 128, 256)),
    "s1x1_chunk_last": lambda n: k3s_case(n, "bach10_score_1x1", 2049, 1373, 30, 25, chunk=(251, 256, 270)),
    "bach10_coherent": lambda n: k3s_case(n, "bach10", 513, 50, 30, 25, coherent=True),
    # bins past the last window have y = 0 too, so bias 1e-40 makes them subnormal in every frame: few such bins
    "bach10_subnormal": lambda n: k3s_case(n, "bach10", 1025, 400, 30, 25, zero_slots=((1, 0), (3, 2))),
    "ikala_subnormal": lambda n: k3s_case(n, "ikala", 1025, 400, 30, 25, zero_slots=((1, 0), (3, 2))),
}


def make_case(name, engine):
    c = (DSD_CASES.get(name) or K3S_CASES[name])(name)
    c["engine"] = engine
    return c


def refused(case, engine):
    """why engine takes no such view (the C entry must return DCS_EINVAL), or None"""
    if case["kind"] == "dsd" and engine == "tc":
        step = case["tc"] - case["ov"]
        if -(-case["tc"] // step) > 6:
            return "more than 6 patches per frame"
    return None


# ---------------------------------------------------------------------------------------------- CPU tests
@pytest.mark.parametrize("F", [129, 257])
def test_layouts_reproduce_conv2d_inverse(F):
    """the kernels' index formulas evaluated on w1t_layout / bank_layout give oracle.nets.conv2d_inverse"""
    rng = np.random.default_rng(F)
    f32 = lambda *shape: rng.standard_normal(shape).astype(np.float32).astype(np.float64)
    W = f32(50, 2, 1, F)
    g = f32(3, 52)
    want = nets.conv2d_inverse(g[:, :50, None, None], W, (3, 2, 1, F))[:, :, 0]
    for ch in range(2):
        np.testing.assert_allclose(dsd_kernel_y(g, w1t_layout(W, ch, _ldf(F)), F), want[:, ch], rtol=1e-12, atol=1e-12)
    for arch in K3S:
        KW, stride, nsrc, ndec, nw, pool, _ = K3S[arch]
        J = (F - KW) // stride + 1
        W = f32(30, nw, 1, KW)
        gu = f32(3, J, 32)
        want = nets.conv2d_inverse(gu[:, :, :30].transpose(0, 2, 1)[:, :, None, :], W, (3, nw, 1, F), (1, stride))[:, :, 0]
        bank = bank_layout(W, stride)
        assert np.isnan(bank[..., stride:]).all() and (bank[:, :, 30:, :stride] == 0).all()
        np.testing.assert_allclose(k3s_kernel_y(gu, bank, stride, F), want, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("tc,ov,P", [(30, 25, 9), (10, 1, 6), (12, 8, 7), (30, 0, 3), (4, 3, 12)])
def test_fade_weights_match_overlapadd_multi(tc, ov, P):
    """sum_j omega_j m_{k_lo + j}[p_j] equals overlapadd_multi on the per-patch masks (one frame row per patch row)"""
    rng = np.random.default_rng(tc * 100 + ov)
    F = 3
    m = rng.random((P, 2, tc, F))
    fb = m.transpose(1, 0, 2, 3)[None, :, :, None]                    # [1 batch, nsrc, P, 1, tc, F]
    want = patch.overlapadd_multi(fb, None, P, overlap=ov)
    step = tc - ov
    frames = np.arange((P - 1) * step + tc)
    k_lo, n = covering(frames, P, tc, ov)
    om = fade_weights(frames, P, tc, ov)
    got = np.zeros((2, len(frames), F))
    for j in range(om.shape[1]):
        v = np.nonzero(j < n)[0]
        k = k_lo[v] + j
        got[:, v] += om[v, j][None, :, None] * m[k, :, frames[v] - k * step].transpose(1, 0, 2)
    np.testing.assert_allclose(got, want[:, :len(frames)], rtol=0, atol=1e-15)


def _emulate(case, arith, mut=None):
    """the device arithmetic on the case's kernel-layout operands: the plan `arith` for y, fp32 epilogue, fp32 fade
    weights and recurrence, fp32 product with X.  `mut` injects one index error.  Returns S complex64 [nsrc, T, F]."""
    T, P, tc, ov, F = case["T"], case["P"], case["tc"], case["ov"], case["F"]
    step = tc - ov
    frames = np.arange(T)
    k_lo, n = covering(frames, P, tc, ov)
    f32 = np.float32
    inv = f32(1.0) / f32(ov - 1) if ov > 1 else f32(0.0)
    if case["kind"] == "dsd":
        nsrc, zero_val = 4, f32(0.25)
        w1t = w1t_layout(case["W"], 0, _ldf(F))
        if mut == "nyquist":
            w1t[:, F - 1] = w1t[:, F - 2]
        dec = (0, 1, 2, 2) if mut == "dec3" else (0, 1, 2, 1)
        bout = case["bout"][0]
    else:
        KW, stride, nsrc, ndec, nw, pool, rule = K3S[case["arch"]]
        zero_val = f32(1.0 / nsrc) if rule == "dsd" else f32(0.0)
        bank = bank_layout(case["W"], stride)
        bout = case["bout"]
    macc = np.zeros((T, nsrc, F), f32)
    for j in range(int(n.max())):
        v = np.nonzero(j < n)[0]
        k = k_lo[v] + j
        p = frames[v] - k * step
        if mut == "p_off" and j == 1:
            p = np.minimum(p + 1, tc - 1)
        if case["kind"] == "dsd":
            g = case["G"][k, :, p]
            ys = [dsd_kernel_y(g[:, d], w1t, F, arith).astype(f32) for d in range(3)]
            y = np.stack([ys[d] for d in dec], 1)
        else:
            g = case["G"][k - case["p_base"], :, p].astype(np.float64)
            if pool:
                tie = case["tie"][frames[v]]
                if mut == "unpool_first":
                    tie = tie & (-tie.astype(np.int16)).astype(np.uint8)     # lowest set bit only
                g = unpool(g, tie)
            J = case["J"]
            gu = np.zeros((len(v), ndec, J, 32))
            gu[:, :, :min(J, g.shape[2])] = g[:, :, :J]
            if nw == 1:
                y = np.concatenate([k3s_kernel_y(gu[:, d], bank, stride, F, arith) for d in range(ndec)], 1)
            else:
                y = k3s_kernel_y(gu[:, 0], bank, stride, F, arith)
            if mut == "tap_seam":   # the last tap of the first position of tile 1 (a halo row of the staged tile) dropped
                m = OUT_TC[case["arch"]]
                nd = bank.shape[1]
                ex = np.zeros((len(v), y.shape[1], F))
                one = np.zeros_like(gu)
                one[:, :, m - (nd - 1)] = gu[:, :, m - (nd - 1)]
                cut = np.zeros_like(bank)
                cut[:, nd - 1] = bank[:, nd - 1]
                ex = np.concatenate([k3s_kernel_y(one[:, d], cut, stride, F) for d in range(ndec)], 1) if nw == 1 else \
                    k3s_kernel_y(one[:, 0], cut, stride, F)
                sl = slice(stride * m, stride * m + stride)
                y[:, :, sl] = (y[:, :, sl].astype(np.float64) - ex[:, :, sl]).astype(f32)
            y = y.astype(f32)
        pre = (y + bout[None, :, None].astype(f32)).astype(f32)
        pv = np.maximum(pre, f32(0))
        tot = pv.sum(1, dtype=f32)
        if j == 0:
            up, down = np.ones(len(v), f32), np.zeros(len(v), f32)
        else:
            pp = (p + 1) if mut == "fade" else p
            up = (pp.astype(f32) * inv).astype(f32)
            down = ((ov - 1 - p).astype(f32) * inv).astype(f32)
        pos = tot > f32(1.2e-38)
        with np.errstate(divide="ignore", invalid="ignore"):
            r = np.where(pos, (up[:, None] / np.where(pos, tot, f32(1))).astype(f32), f32(0))
        q = np.where(pos, f32(0), (up[:, None] * zero_val).astype(f32))
        mk = (pv * r[:, None] + q[:, None]).astype(f32)
        macc[v] = (down[:, None, None] * macc[v] + mk).astype(f32)
    X = case["X"][0] if case["kind"] == "dsd" else case["X"]
    return (macc.transpose(1, 0, 2) * X[None]).astype(np.complex64)


def _teeth_ratio(case, arith, mut=None):
    S = _emulate(case, arith, mut)
    ref = reference_masks(case, np.arange(case["T"]))
    worst, fails = evaluate(ref, S, case["X"][0] if case["kind"] == "dsd" else case["X"])
    return worst, fails, well_fraction(ref)


def _teeth_case(kind, engine):
    if kind == "dsd":
        c = dsd_case("teeth_dsd", 257, 40, 12, 8, coherent=True)
    elif kind == "bach10":
        c = k3s_case("teeth_bach10", "bach10", 513, 24, 12, 8, coherent=True)
    else:
        c = k3s_case("teeth_ikala", "ikala", 513, 24, 12, 8, coherent=True)
    c["engine"] = engine
    return c


@pytest.mark.parametrize("kind", ["dsd", "bach10", "ikala"])
def test_bound_accepts_each_engines_plan(kind):
    for engine, arith in (("tc", "tc"), ("ffma", "ffma")):
        worst, fails, well = _teeth_ratio(_teeth_case(kind, engine), arith)
        assert worst <= 1.0 and not fails and well >= 0.99, (kind, engine, worst, fails, well)


@pytest.mark.parametrize("kind,mut", [("dsd", "tf32"), ("bach10", "tf32"), ("dsd", "p_off"), ("bach10", "p_off"),
                                      ("dsd", "fade"), ("bach10", "fade"), ("dsd", "nyquist"), ("dsd", "dec3"),
                                      ("bach10", "tap_seam"), ("ikala", "tap_seam"), ("ikala", "unpool_first")])
def test_bound_has_teeth(kind, mut):
    """plain TF32 on the sign-coherent case, and each index mutation of the tensor-core plan, fails the bound (ratio
    above 1) or an admissibility / exactness check"""
    case = _teeth_case(kind, "tc")
    worst, fails, _ = _teeth_ratio(case, "tf32" if mut == "tf32" else "tc", None if mut == "tf32" else mut)
    assert worst > 1.0 or fails, (kind, mut, worst)


# ---------------------------------------------------------------------------------------------- GPU harness
@pytest.fixture(scope="module")
def ctx():
    pytest.importorskip("torch")
    from deepconvsep_b200.engine import Context
    return Context(0)


def _padded(a, fill=np.nan):
    """flat float32 buffer with SLACK `fill` elements on both sides"""
    a = np.ascontiguousarray(a, np.float32).ravel()
    pad = np.full(SLACK, fill, np.float32)
    return np.concatenate([pad, a, pad])


def _planes(X, ldf, stride):
    """complex [nplanes, T, F] -> float32 interleaved [nplanes][stride][2] with NaN pad columns and plane gaps"""
    npl, T, F = X.shape
    out = np.full((npl, stride, 2), np.nan, np.float32)
    body = np.full((npl, T, ldf, 2), np.nan, np.float32)
    body[:, :, :F, 0], body[:, :, :F, 1] = X.real, X.imag
    out[:, :T * ldf] = body.reshape(npl, T * ldf, 2)
    return out


class Buffers:
    """device copies of a case's operands in the kernels' layouts, NaN wherever the kernels never read"""

    def __init__(self, case):
        import torch
        self.torch = torch
        T, F, ldf = case["T"], case["F"], case["ldf"]
        self.plane = T * ldf
        self.xp = self.plane + 24          # complex elements between mixture planes (a NaN gap)
        self.sp = self.plane + 40          # between output planes (a sentinel gap)
        dev = lambda a: torch.from_numpy(a).cuda()
        if case["kind"] == "dsd":
            G = np.concatenate([case["G"], np.zeros((2,) + case["G"].shape[1:], np.float32)])
            G[:, :, :, 52:] = np.nan
            G[case["P"]:] = np.nan                                   # patches >= P
            self.G = dev(_padded(G))
            self.W1t = dev(_padded(np.stack([w1t_layout(case["W"], ch, ldf) for ch in range(case["nch"])])))
            self.bout = dev(_padded(case["bout"]))
            self.tie = None
            self.nplanes = 4 * case["nch"]
            Xp = case["X"]
        else:
            KW, stride, nsrc, ndec, nw, pool, _ = K3S[case["arch"]]
            G = case["G"]
            lead = G[:1] * np.nan if case["p_base"] > 0 else G[:0]    # a NaN patch before the G pointer
            G = np.concatenate([lead, G, np.full((2,) + G.shape[1:], np.nan, np.float32)])
            self.g_off = SLACK + lead.size
            self.G = dev(np.concatenate([np.full(SLACK, np.nan, np.float32), G.ravel(), np.full(SLACK, np.nan, np.float32)]))
            self.W = dev(_padded(bank_layout(case["W"], stride)))
            self.bout = dev(_padded(case["bout"]))
            self.tie = dev(np.ascontiguousarray(case["tie"]).ravel()) if pool else None
            self.nplanes = nsrc
            Xp = case["X"][None]
        self.X = dev(_padded(_planes(Xp, ldf, self.xp)))
        self.S_init = np.full(2 * (self.nplanes * self.sp + 2 * SLACK), S_SENTINEL, np.uint32)

    def fresh_S(self):
        return self.torch.from_numpy(self.S_init.view(np.float32).copy()).cuda()


def _ptr(t, floats=SLACK):
    return t.data_ptr() + 4 * floats


def dsd_views(case, b, S, engine):
    """the argument sets dsd_forward builds: mono, ILD (one call per channel, planes (s, ch))"""
    from deepconvsep_b200 import _lib
    T, F, ldf = case["T"], case["F"], case["ldf"]
    calls = []
    for ch in range(case["nch"]):
        v = _lib.DsdMaskView()
        v.G, v.ldg = _ptr(b.G), case["ldg"]
        v.W1t, v.ldw = _ptr(b.W1t) + 4 * ch * 50 * ldf, ldf
        v.bout = _ptr(b.bout) + 16 * ch
        v.X = _ptr(b.X) + 8 * ch * b.xp
        v.S = _ptr(S, 2 * SLACK) + 8 * ch * b.sp
        v.ldf, v.T, v.P, v.tc, v.overlap, v.F, v.ndec = ldf, T, case["P"], case["tc"], case["ov"], F, case["ndec"]
        v.src_stride = b.sp * case["nch"]
        calls.append(v)
    return calls


def sconv_view(case, b, S):
    from deepconvsep_b200 import _lib
    v = _lib.SconvMaskView()
    v.arch = ARCH_IDS[case["arch"]]
    v.G = b.G.data_ptr() + 4 * b.g_off
    v.tie = b.tie.data_ptr() if b.tie is not None else None
    v.W, v.bout = _ptr(b.W), _ptr(b.bout)
    v.X, v.S = _ptr(b.X), _ptr(S, 2 * SLACK)
    v.ldf, v.src_stride = case["ldf"], b.sp
    v.T, v.P, v.tc, v.overlap, v.F, v.J, v.WP = case["T"], case["P"], case["tc"], case["ov"], case["F"], case["J"], case["WP"]
    v.p_base, v.t0, v.t1 = case["p_base"], case["t0"], case["t1"]
    return v


def _call(ctx, case, engine, v):
    fn = ctx.lib.dcs_dsd_mask_f32 if case["kind"] == "dsd" else ctx.lib.dcs_sconv_mask_f32
    return fn(ctx.handle, engine, ctypes.byref(v), None)


def _run(ctx, case, b, engine):
    from deepconvsep_b200 import _lib
    S = b.fresh_S()
    views = dsd_views(case, b, S, engine) if case["kind"] == "dsd" else [sconv_view(case, b, S)]
    for v in views:
        _lib.check(_call(ctx, case, engine, v))
    return S.cpu().numpy().view(np.uint32)


def _plane_map(case):
    """output plane -> (source, mask set, mixture plane)"""
    if case["kind"] == "k3s":
        return [(s, 0, 0) for s in range(K3S[case["arch"]][2])]
    return [(s, c, c) for s in range(4) for c in range(case["nch"])]


ENGINES = {"tc": 1, "ffma": 0}


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ["tc", "ffma"])
@pytest.mark.parametrize("name", list(DSD_CASES) + list(K3S_CASES))
def test_mask_view_matches_float64(ctx, name, engine):
    case = make_case(name, engine)
    b = Buffers(case)
    why = refused(case, engine)
    if why:
        S = b.fresh_S()
        n0 = ctx.launch_count()
        for v in dsd_views(case, b, S, ENGINES[engine]):
            assert _call(ctx, case, ENGINES[engine], v) == -1, why
        assert ctx.launch_count() == n0
        assert np.array_equal(S.cpu().numpy().view(np.uint32), b.S_init)
        return
    Sb = _run(ctx, case, b, ENGINES[engine])
    assert np.array_equal(Sb, _run(ctx, case, b, ENGINES[engine])), "two runs gave different bits"

    T, F, ldf = case["T"], case["F"], case["ldf"]
    t0, t1 = case["t0"], case["t1"]
    body = Sb[2 * SLACK:2 * SLACK + 2 * b.nplanes * b.sp].reshape(b.nplanes, b.sp, 2)
    written = np.zeros((b.nplanes, b.sp), bool)
    w = written[:, :T * ldf].reshape(b.nplanes, T, ldf)
    w[:, t0:t1, :F] = True
    assert (Sb[:2 * SLACK] == S_SENTINEL).all() and (Sb[2 * SLACK + 2 * b.nplanes * b.sp:] == S_SENTINEL).all()
    assert (body[~written] == S_SENTINEL).all(), "%d S elements outside the written frames and bins changed" % \
        int((body[~written] != S_SENTINEL).any(-1).sum())
    vals = body[:, :T * ldf].reshape(b.nplanes, T, ldf, 2).view(np.float32)[:, t0:t1, :F]
    assert np.isfinite(vals).all(), "%d stored values are not finite" % int((~np.isfinite(vals)).sum())
    S = vals[..., 0] + 1j * vals[..., 1].astype(np.float64)

    frames = np.arange(t0, t1)
    pm = _plane_map(case)
    worst, fails, wf = 0.0, [], 1.0
    Xall = case["X"] if case["kind"] == "dsd" else case["X"][None]
    for mset in sorted(set(m for _, m, _ in pm)):
        ref = reference_masks(case, frames, mset)
        wf = min(wf, well_fraction(ref))
        for xpl in sorted(set(x for _, m, x in pm if m == mset)):
            idx = [i for i, (s, m, x) in enumerate(pm) if m == mset and x == xpl]
            wo, fa = evaluate(ref, S[idx], Xall[xpl][t0:t1])
            worst = max(worst, wo)
            fails += fa
    record("mask_view:" + name, engine=engine, F=F, T=T, tc=case["tc"], overlap=case["ov"],
           well_conditioned=wf, worst_error_over_bound=worst)
    assert not fails, (name, engine, fails)
    assert wf >= 0.99, (name, engine, wf)
    assert worst <= 1.0, (name, engine, worst)


@pytest.mark.gpu
def test_dsd_ffma_clip_longer_than_grid_y(ctx):
    """dsd.cu on 1,048,577 frames (more than 65535 CTAs of 16 frames), 7 patches per frame: the first and last 64
    frames against the float64 reference, and the sentinels past the last frame"""
    import torch
    from deepconvsep_b200 import _lib
    T, F, tc, ov = 1048577, 129, 7, 6
    ldf, ldg = _ldf(F), 52
    P = patch.num_patches(T, tc, ov, "util")
    gen = torch.Generator(device="cuda").manual_seed(7)
    G = torch.randn((P, 3, tc, ldg), generator=gen, device="cuda")
    G[..., 50:] = float("nan")
    rng = _rng("dsd_long")
    a = np.sqrt(6.0 / (51 * F))
    W = rng.uniform(-a, a, (50, 1, 1, F)).astype(np.float32)
    bout = (rng.standard_normal((1, 4)) * 0.7 * np.sqrt(50 / 3.0) * a).astype(np.float32)
    X = torch.randn((T, ldf, 2), generator=gen, device="cuda")
    X[:, F:] = float("nan")
    plane = T * ldf
    S = torch.full((2 * (4 * plane + SLACK),), int(S_SENTINEL), dtype=torch.int32, device="cuda")
    W1t = torch.from_numpy(w1t_layout(W, 0, ldf)).cuda()
    bo = torch.from_numpy(bout[0]).cuda()
    v = _lib.DsdMaskView()
    v.G, v.ldg, v.W1t, v.ldw, v.bout = G.data_ptr(), ldg, W1t.data_ptr(), ldf, bo.data_ptr()
    v.X, v.S, v.ldf, v.src_stride = X.data_ptr(), S.data_ptr(), ldf, plane
    v.T, v.P, v.tc, v.overlap, v.F, v.ndec = T, P, tc, ov, F, 3
    assert ctx.lib.dcs_dsd_mask_f32(ctx.handle, 1, ctypes.byref(v), None) == -1    # 7 patches per frame
    _lib.check(ctx.lib.dcs_dsd_mask_f32(ctx.handle, 0, ctypes.byref(v), None))
    case = dict(kind="dsd", T=T, P=P, tc=tc, ov=ov, F=F, ndec=3, W=W, G=G, bout=bout, engine="ffma")
    frames = np.concatenate([np.arange(64), np.arange(T - 64, T)])
    ref = reference_masks(case, frames)
    Sv = S.view(torch.float32)[:2 * 4 * plane].view(4, T, ldf, 2)
    fr = torch.from_numpy(frames).cuda()
    got = Sv[:, fr].cpu().numpy()
    assert (got[:, :, F:].view(np.uint32) == S_SENTINEL).all()
    got = got[:, :, :F]
    assert np.isfinite(got).all()
    Xh = X[fr].cpu().numpy()[:, :F]
    worst, fails = evaluate(ref, got[..., 0] + 1j * got[..., 1].astype(np.float64), Xh[..., 0] + 1j * Xh[..., 1].astype(np.float64))
    assert (S[2 * 4 * plane:].cpu().numpy().view(np.uint32) == S_SENTINEL).all()
    record("mask_view:dsd_long", engine="ffma", F=F, T=T, tc=tc, overlap=ov, worst_error_over_bound=worst)
    assert not fails and worst <= 1.0 and well_fraction(ref) >= 0.99, (worst, fails)


@pytest.mark.gpu
def test_mask_views_refuse_what_the_engine_does_not_take(ctx):
    """each refusal returns DCS_EINVAL with nothing launched and S untouched"""
    case = make_case("dsd_F513", "tc")
    b = Buffers(case)
    S = b.fresh_S()
    n0 = ctx.launch_count()

    def bad(engine, **kw):
        v = dsd_views(case, b, S, 1)[0]
        for k, x in kw.items():
            setattr(v, k, x)
        assert ctx.lib.dcs_dsd_mask_f32(ctx.handle, engine, ctypes.byref(v), None) == -1, (engine, kw)

    bad(1, ndec=5)
    bad(1, ldg=50)
    bad(1, ldg=54)
    bad(1, G=_ptr(b.G) + 4)                  # G not 16-byte aligned
    bad(2)
    bad(1, src_stride=b.plane - 1)           # overlapping output planes
    kc = make_case("bach10_F129", "tc")
    kb = Buffers(kc)
    S2 = kb.fresh_S()

    def bad_k3s(engine, **kw):
        v = sconv_view(kc, kb, S2)
        for k, x in kw.items():
            setattr(v, k, x)
        assert ctx.lib.dcs_sconv_mask_f32(ctx.handle, engine, ctypes.byref(v), None) == -1, (engine, kw)

    bad_k3s(1, arch=ARCH_IDS["dsd"])
    bad_k3s(0, J=kc["J"] + 1)
    bad_k3s(1, t0=1)                         # only build_ca_1x1 decodes in chunks
    bad_k3s(1, tie=_ptr(kb.G))               # tie bits without the max-pool net
    bad_k3s(1, G=_ptr(kb.G) + 4)
    bad_k3s(2)
    assert ctx.launch_count() == n0
    assert np.array_equal(S.cpu().numpy().view(np.uint32), b.S_init)
    assert np.array_equal(S2.cpu().numpy().view(np.uint32), kb.S_init)
