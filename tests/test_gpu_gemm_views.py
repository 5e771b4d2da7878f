"""Every operand view and epilogue of the GEMM (csrc/common.cuh GemmDesc) on both engines against a float64 reference,
element by element, through dcs_gemm_view_f32.

The views are built the way the layers build them (dsd_model.cu dsd_forward, sconv_model.cu sconv_forward, score1x1.cu
s1x1_forward), at their real shapes, plus the edges of the kernels' control logic.  Every case
  - requires |C - C64| <= bound (below) for every stored element;
  - fills every C element outside the view with a NaN-payload sentinel and every A element outside the view with NaN,
    and fails if a sentinel changes or a stored value is not finite; the gate-code array gets the same treatment;
  - runs twice per engine and requires the same bits;
  - with DCS_TEST_RECORDS set, records its largest |error| / bound (tests/parity.py).

Per-element bound.  With u = 2^-24, S = sum_k |A_mk B_kn| (float64 over the fp32 operands), pre = AB + bias and
post = act(pre) (+ bias2), both in float64, and g = 0.5 * gate (EPI_GATE) or 1:
    |C - C64| <= g * (c(K) * S + u * (|pre| + |post|)).
The u terms are the fp32 roundings of the bias, ReLU-bias2 and final additions (ReLU is 1-Lipschitz; the gate scale
is a power of two or 0, exact).  c(K) follows each engine's accumulation plan:
  - FFMA (gemm.cu): one fp32 FMA chain of K terms, each FMA rounds once to nearest: c = (K + 4) u (gamma_K, rounded up).
  - tensor cores (gemm_tc.cu), 3xTF32: a = ah + al with ah = a truncated to TF32 (|al| < 2^-10 |a|); the tensor core
    reads al truncated to TF32 again (error < 2^-20 |a|) and the dropped al*bl is < 2^-20 |ab|, so every product is
    off by < 3 * 2^-20 = 48u relative.  Each k8 wgmma step adds up to 9 terms with truncation after alignment (< 2u
    per term of the step's sum of magnitudes, 18u), four steps per 32-wide stage: 72u of the stage's S.  The stages
    are summed in an fp32 register with round to nearest: K/32 roundings, u each.  The two correction terms (< 2^-9 of
    S) share one truncating accumulator over the whole K: (K/4) * 18u * 2^-9 < 0.01 K u.  Split K adds at most
    K/256 fixed-order fp32 additions.  Total < (120 + 0.045 K) u, taken as c = (128 + K/16) u.
Plain TF32 (hi*hi only: what the kernel computes without its correction term) errs by up to 2^-9 per product; on
sign-coherent products that is a bias of ~2^-10.5 S at any K, far above c(K) for K < 10^5, so every case has weight
columns that are all non-negative against non-negative activations.  test_bound_rejects_tf32_accepts_3xtf32 shows
both on an emulation of the two plans.

Exact parts: EPI_POST gate codes equal the float64 codes wherever |pre| exceeds its bound (everywhere in the
small-integer cases, whose products and sums are exact under 3xTF32, so pre == 0 and code 1 are reached); columns at
or past g_lim are never stored (their C elements keep the sentinel); a K-clipped tile whose tap range is empty gives
exactly the bias."""
import os
import sys
import zlib

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from parity import record  # noqa: E402

U = 2.0 ** -24
EPI_POST, EPI_GATE = 1, 2
SLACK = 64                         # sentinel elements before and after every buffer
C_SENTINEL = np.uint32(0x7FC5A5A5)  # quiet NaN with a payload no kernel produces
CODE_SENTINEL = np.uint8(0xA5)

FIELDS = ("M", "N", "K", "a_valid_rows", "m_inner", "a_so", "a_si", "m_inner2", "a_s2", "k_seg", "k_ss", "ldb",
          "cm_inner", "c_so", "c_si", "cm_inner2", "c_s2", "n_seg", "n_ss", "c_col0", "relu",
          "kc_rows", "kc_unit", "kc_pad", "kc_n", "kc_taps", "g_inner", "g_inner2", "g_so", "g_si", "g_s2", "g_lim")


def plain(A_ld, ldc, M, N, K, relu=0):
    """gemm_plain (gemm.cu): dense rows lda apart, one K segment, C rows ldc apart"""
    return dict(M=M, N=N, K=K, a_valid_rows=M, m_inner=1, a_so=A_ld, a_si=0, m_inner2=1, a_s2=0, k_seg=K, k_ss=0,
                ldb=N, cm_inner=1, c_so=ldc, c_si=0, cm_inner2=1, c_s2=0, n_seg=N, n_ss=0, c_col0=0, relu=relu,
                kc_rows=0, kc_unit=0, kc_pad=0, kc_n=0, kc_taps=0,
                g_inner=1, g_inner2=1, g_so=0, g_si=0, g_s2=0, g_lim=2 ** 63 - 1)


# ---------------------------------------------------------------------------------------------- float64 reference
def three_level(m, inner, so, si, inner2, s2):
    return (m // inner) * so + ((m % inner) // inner2) * si + (m % inner2) * s2


def a_rows(v):
    m = np.arange(v["M"], dtype=np.int64)
    return three_level(m, v["m_inner"], v["a_so"], v["a_si"], v["m_inner2"], v["a_s2"])


def a_cols(v):
    k = np.arange(v["K"], dtype=np.int64)
    return (k // v["k_seg"]) * v["k_ss"] + k % v["k_seg"]


def c_index(v):
    """[M, N] offsets of C from the view's C pointer"""
    m = np.arange(v["M"], dtype=np.int64)
    n = np.arange(v["N"], dtype=np.int64)
    rows = three_level(m, v["cm_inner"], v["c_so"], v["c_si"], v["cm_inner2"], v["c_s2"]) + v["c_col0"]
    return rows[:, None] + ((n // v["n_seg"]) * v["n_ss"] + n % v["n_seg"])[None, :]


def gate_index(v):
    """[M, N] gate offsets and the [M, N] mask of columns inside g_lim"""
    m = np.arange(v["M"], dtype=np.int64)
    n = np.arange(v["N"], dtype=np.int64)
    rows = (m // v["g_inner"]) * v["g_so"] + ((m % v["g_inner"]) // v["g_inner2"]) * v["g_si"]
    gcol = (m % v["g_inner2"]) * v["g_s2"]
    col = gcol[:, None] + n[None, :]
    return rows[:, None] + col, col < v["g_lim"]


def k_chunks(v):
    step = int(max(8, min(v["K"], (1 << 23) // v["M"])))
    return [np.arange(k0, min(v["K"], k0 + step)) for k0 in range(0, v["K"], step)]


def a_addressed(v, size):
    """mask of the A elements the view reads (rows below a_valid_rows)"""
    rows, cols = a_rows(v)[: v["a_valid_rows"]], a_cols(v)
    mask = np.zeros(size, dtype=bool)
    for ks in k_chunks(v):
        mask[(rows[:, None] + cols[ks][None, :]).ravel()] = True
    return mask


def reference(v, A, B, bias=None, bias2=None, gate=None, epi=0):
    """The view in float64, as the common.cuh comments define it.  A: the flat buffer (offset 0 = the view's A
    pointer).  Returns out (what is stored), S = sum |a b|, pre, the gate scale g, the codes (EPI_POST) and the mask of
    stored elements."""
    M, N = v["M"], v["N"]
    rows, cols = a_rows(v), a_cols(v)
    valid = np.arange(M) < v["a_valid_rows"]
    acc = np.zeros((M, N))
    S = np.zeros((M, N))
    B64 = B.astype(np.float64)
    for ks in k_chunks(v):
        blk = A[rows[:, None] + cols[ks][None, :]].astype(np.float64)
        blk[~valid] = 0.0
        acc += blk @ B64[ks]
        S += np.abs(blk) @ np.abs(B64[ks])
    code = None
    g = np.ones((M, N))
    stored = np.ones((M, N), dtype=bool)
    if epi & EPI_POST:
        pre = acc + bias.astype(np.float64)
        code = np.where(pre > 0, 2, np.where(pre == 0, 1, 0)).astype(np.uint8)
        post = np.maximum(pre, 0.0) + bias2.astype(np.float64)
    elif epi:
        pre = post = acc                      # EPI_GATE alone: no bias, no ReLU
    else:
        pre = acc + (0.0 if bias is None else bias.astype(np.float64))
        post = np.maximum(pre, 0.0) if v["relu"] else pre
    if epi & EPI_GATE:
        gi, stored = gate_index(v)
        g = 0.5 * gate[gi].astype(np.float64)
    return dict(out=post * g, S=S, pre=pre, post=post, g=g, code=code, stored=stored)


def c_tc(K):
    return U * (128 + K / 16.0)


def c_ffma(K):
    return U * (K + 4)


def bound(ref, c):
    return ref["g"] * (c * ref["S"] + U * (np.abs(ref["pre"]) + np.abs(ref["post"])))


# ---------------------------------------------------------------------------------------------- CPU: the reference
def _loop_reference(v, A, B, bias, bias2, gate, epi):
    """the same view with explicit loops over m, n, k and Python integers, straight from the common.cuh formulas"""
    M, N, K = v["M"], v["N"], v["K"]
    out = np.full((M, N), np.nan)
    code = np.zeros((M, N), dtype=np.uint8)
    for m in range(M):
        arow = (m // v["m_inner"]) * v["a_so"] + ((m % v["m_inner"]) // v["m_inner2"]) * v["a_si"] + (m % v["m_inner2"]) * v["a_s2"]
        for n in range(N):
            x = 0.0
            for k in range(K):
                a = float(A[arow + (k // v["k_seg"]) * v["k_ss"] + k % v["k_seg"]]) if m < v["a_valid_rows"] else 0.0
                x += a * float(B[k, n])
            if epi & EPI_POST:
                pre = x + float(bias[n])
                code[m, n] = 2 if pre > 0 else (1 if pre == 0 else 0)
                x = max(pre, 0.0) + float(bias2[n])
            elif not epi:
                x += float(bias[n]) if bias is not None else 0.0
                if v["relu"]:
                    x = max(x, 0.0)
            if epi & EPI_GATE:
                gcol = (m % v["g_inner2"]) * v["g_s2"]
                if gcol + n >= v["g_lim"]:
                    continue
                grow = (m // v["g_inner"]) * v["g_so"] + ((m % v["g_inner"]) // v["g_inner2"]) * v["g_si"]
                x *= 0.5 * float(gate[grow + gcol + n])
            out[m, n] = x
    return out, code


@pytest.mark.parametrize("epi", [0, EPI_POST, EPI_GATE, EPI_POST | EPI_GATE])
def test_view_reference_matches_explicit_loops(epi):
    rng = np.random.default_rng(11 + epi)
    v = plain(0, 0, M=13, N=7, K=10, relu=1)
    v.update(a_valid_rows=11, m_inner=6, a_so=37, m_inner2=3, a_si=11, a_s2=4, k_seg=4, k_ss=9,
             cm_inner=6, c_so=121, cm_inner2=3, c_si=40, c_s2=13, n_seg=3, n_ss=5, c_col0=2,
             g_inner=6, g_so=50, g_inner2=3, g_si=9, g_s2=7, g_lim=17)
    A = rng.standard_normal(400)
    B = rng.standard_normal((10, 7))
    bias, bias2 = rng.standard_normal(7), rng.standard_normal(7)
    bias[2] = -(A[0:4] @ B[0:4, 2] + A[9:13] @ B[4:8, 2] + A[18:20] @ B[8:10, 2])   # pre of (0, 2) is ~0
    gate = rng.integers(0, 3, 200).astype(np.uint8)
    ref = reference(v, A, B, bias, bias2, gate, epi)
    out, code = _loop_reference(v, A, B, bias, bias2, gate, epi)
    assert np.array_equal(np.isnan(out), ~ref["stored"])
    if epi & EPI_GATE:
        assert 0 < ref["stored"].sum() < ref["stored"].size
    np.testing.assert_allclose(ref["out"][ref["stored"]], out[ref["stored"]], rtol=1e-12, atol=1e-12)
    if epi & EPI_POST:
        near = np.abs(ref["pre"]) < 1e-12
        assert np.array_equal(ref["code"][~near], code[~near])
    # every stored element has its own C offset
    ci = c_index(v)[ref["stored"]]
    assert len(np.unique(ci)) == ci.size


def _trunc_tf32(x):
    return (np.ascontiguousarray(x, dtype=np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def _emulate_tc(A, B, corr):
    """the tensor-core plan on fp32 operands: per 32-wide stage a fresh hi*hi sum (rounded to fp32) added to an fp32
    running sum; with `corr` the ah*bl + al*bh terms (al, bl truncated to TF32 again) in one fp32 accumulator"""
    Ah, Bh = _trunc_tf32(A), _trunc_tf32(B)
    Al, Bl = _trunc_tf32(A - Ah), _trunc_tf32(B - Bh)
    f64 = lambda x: x.astype(np.float64)
    s = np.zeros((A.shape[0], B.shape[1]), dtype=np.float32)
    c = np.zeros_like(s)
    for k0 in range(0, A.shape[1], 32):
        ks = slice(k0, k0 + 32)
        s = (s + (f64(Ah[:, ks]) @ f64(Bh[ks])).astype(np.float32)).astype(np.float32)
        if corr:
            for j in range(k0, min(A.shape[1], k0 + 32), 8):
                kj = slice(j, j + 8)
                c = (c + (f64(Ah[:, kj]) @ f64(Bl[kj]) + f64(Al[:, kj]) @ f64(Bh[kj])).astype(np.float32)).astype(np.float32)
    return (s + c).astype(np.float32)


def _emulate_ffma(A, B):
    acc = np.zeros((A.shape[0], B.shape[1]), dtype=np.float32)
    for k in range(A.shape[1]):   # fma: exact product, one rounding (the float64 sum is exact to well below fp32)
        acc = (acc.astype(np.float64) + A[:, k:k + 1].astype(np.float64) * B[k:k + 1].astype(np.float64)).astype(np.float32)
    return acc


@pytest.mark.parametrize("K,signed", [(32, True), (200, True), (1040, True), (5120, False), (10240, False)])
def test_bound_rejects_tf32_accepts_3xtf32(K, signed):
    """The bound is tight enough to matter: plain TF32 fails it at every K the layers use, while the 3xTF32 plan (and
    the FFMA chain against its own c(K)) pass.  Signed operands at moderate K; at 5120 / 10240 (build_ca_1x1 conv5 /
    conv6) non-negative activations against non-negative weight columns, the sign-coherent case every GPU case has."""
    rng = np.random.default_rng(K)
    A = rng.standard_normal((48, K)).astype(np.float32)
    B = (rng.standard_normal((K, 16)) / np.sqrt(K)).astype(np.float32)
    if not signed:
        A, B = np.abs(A), np.abs(B)
    v = plain(K, 16, 48, 16, K)
    ref = reference(v, A.ravel(), B)
    for got, c, ok in ((_emulate_tc(A, B, True), c_tc(K), True), (_emulate_tc(A, B, False), c_tc(K), False)):
        ratio = np.abs(got - ref["out"]) / bound(ref, c)
        assert (ratio.max() <= 1.0) == ok, (K, ok, ratio.max())
    if K <= 1040:
        ratio = np.abs(_emulate_ffma(A, B) - ref["out"]) / bound(ref, c_ffma(K))
        assert ratio.max() <= 1.0


# ---------------------------------------------------------------------------------------------- the cases
def _weights(rng, K, N, coherent=4):
    """weights ~ 1/sqrt(K), the first `coherent` columns non-negative (sign-coherent against non-negative activations)"""
    B = (rng.standard_normal((K, N)) / np.sqrt(K)).astype(np.float32)
    B[:, :coherent] = np.abs(B[:, :coherent])
    return B


def _padded(rng, shape, interior):
    """non-negative activations inside `interior` (a tuple of slices), zero padding elsewhere"""
    x = np.zeros(shape, dtype=np.float32)
    x[interior] = np.abs(rng.standard_normal(x[interior].shape)).astype(np.float32)
    return x.ravel()


def _rng(name):
    return np.random.default_rng(zlib.crc32(name.encode()))


def _case(name, v, fill, B, bias=None, bias2=None, gate=None, epi=0, exact=False):
    return dict(name=name, v=v, fill=fill, B=B, bias=bias, bias2=bias2, gate=gate, epi=epi, exact=exact)


def _bias(rng, n, s=0.1):
    return (rng.standard_normal(n) * s).astype(np.float32)


def dsd_layer(name):
    """the DSD100 net at N = 2048 (F = 1025, ldf 1032), time_context 30, overlap 25, util patcher, on a 180 s clip at
    hop 512 (T = 15506, P = 3097, Tp = 15510), as dsd_model.cu dsd_forward builds each view"""
    rng = _rng(name)
    T, P, Tp, F, ldf, step = 15506, 3097, 15510, 1025, 1032, 5
    C1 = C2 = 50
    C1p = C2p = 52
    kh2, h2, nfc, ndec = 15, 16, 128, 3
    HP, ldg = h2 + 2 * (kh2 - 1), 52
    if name == "dsd_conv1":          # a_valid_rows = T inside a tile (T % 128 = 18), K tail of 1 past a float4
        v = plain(ldf, C1p, Tp, C1, F)
        v["a_valid_rows"] = T
        fill = np.abs(rng.standard_normal(T * ldf)).astype(np.float32)
        return _case(name, v, fill, _weights(rng, F, C1), _bias(rng, C1))
    if name == "dsd_conv2":          # overlapping rows: stride C1p, length kh2 * C1p
        v = plain(C1p, C2p, Tp - kh2 + 1, C2, kh2 * C1p)
        fill = _padded(rng, (Tp, C1p), (slice(None), slice(0, C1)))
        return _case(name, v, fill, _weights(rng, kh2 * C1p, C2), _bias(rng, C2))
    if name == "dsd_bottleneck":     # 25 x 2 tiles, 26 k-blocks: split over 2 slices
        v = plain(step * C2p, nfc, P, nfc, h2 * C2p, relu=1)
        fill = _padded(rng, (Tp - kh2 + 1, C2p), (slice(None), slice(0, C2)))
        return _case(name, v, fill, _weights(rng, h2 * C2p, nfc), _bias(rng, nfc))
    if name == "dsd_dec_dense":      # scatter into the zero-padded apad: n_seg / n_ss / c_col0
        v = plain(nfc, ndec * HP * C2p, P, ndec * h2 * C2p, nfc, relu=1)
        v.update(n_seg=h2 * C2p, n_ss=HP * C2p, c_col0=(kh2 - 1) * C2p)
        fill = np.abs(rng.standard_normal(P * nfc)).astype(np.float32)
        return _case(name, v, fill, _weights(rng, nfc, ndec * h2 * C2p), _bias(rng, ndec * h2 * C2p))
    if name == "dsd_convT2":         # rows (u, k, d), K clipping: 9291 rows per output position u
        KD = P * ndec
        v = plain(0, ldg, KD * 30, C1, kh2 * C2p)
        v.update(m_inner=KD, a_so=C2p, a_si=HP * C2p, cm_inner=KD, c_so=ldg, c_si=30 * ldg,
                 kc_rows=KD, kc_unit=C2p, kc_pad=kh2 - 1, kc_n=h2, kc_taps=kh2)
        fill = _padded(rng, (KD, HP, C2p), (slice(None), slice(kh2 - 1, kh2 - 1 + h2), slice(0, C2)))
        return _case(name, v, fill, _weights(rng, kh2 * C2p, C1))
    raise KeyError(name)


def sconv_layer(name):
    rng = _rng(name)
    if name == "sconv_conv1":
        # the 17-array score-informed Bach10 net, F = 2049 (N = 4096, ldf 2056), 10 s at hop 512: T = 863, Tp = 865,
        # J = 505 windows of 30 bins at stride 4 per frame, one 30-tap K segment per input plane -> A vector width 1
        T, Tp, F, ldf, J, nch = 863, 865, 2049, 2056, 505, 4
        v = plain(0, 32, Tp * J, 30, 30 * nch)
        v.update(m_inner=J, a_so=ldf, a_si=4, k_seg=30, k_ss=T * ldf, a_valid_rows=T * J)
        fill = _padded(rng, (nch, T, ldf), (slice(None), slice(None), slice(0, F)))
        return _case(name, v, fill, _weights(rng, 30 * nch, 30), _bias(rng, 30))
    if name == "sconv_convT2":
        # iKala (max-pool net, F = 513): three-level rows (u, kd, jp), kh2 = 10 time taps clipped, kw2 = 20 column
        # taps as K segments, 8 patches x 2 decoders
        tc, WP, kh2, kw2, h2, w2, CP = 30, 40, 10, 20, 21, 21, 32
        HP, WPP, KD = h2 + 2 * (kh2 - 1), w2 + 2 * (kw2 - 1), 16
        v = plain(0, CP, KD * tc * WP, 30, kh2 * kw2 * CP)
        v.update(m_inner=KD * WP, a_so=WPP * CP, m_inner2=WP, a_si=HP * WPP * CP, a_s2=CP, k_seg=kw2 * CP, k_ss=WPP * CP,
                 cm_inner=KD * WP, c_so=WP * CP, cm_inner2=WP, c_si=tc * WP * CP, c_s2=CP,
                 kc_rows=KD * WP, kc_unit=kw2 * CP, kc_pad=kh2 - 1, kc_n=h2, kc_taps=kh2)
        fill = _padded(rng, (KD, HP, WPP, CP), (slice(None), slice(kh2 - 1, kh2 - 1 + h2), slice(kw2 - 1, kw2 - 1 + w2), slice(0, 30)))
        return _case(name, v, fill, _weights(rng, kh2 * kw2 * CP, 30))
    raise KeyError(name)


# build_ca_1x1 at feat_size 2049, time_context 30, step 5 (score1x1.cu)
S1_W = [2049, 1023, 510, 253, 125, 61, 29]
S1_C = [4, 30, 50, 70, 100, 200, 200]
S1_CP = [4, 32, 52, 72, 100, 200, 200]
S1_KH = [0, 1, 1, 1, 1, 10, 10]
S1_H = [0, 30, 30, 30, 30, 21, 12]


def _r32(k):
    return (k + 31) // 32 * 32


def _fwd_seg(l):
    return _r32(5 * S1_CP[l - 1])


def _fwd_k(l):
    return 5 * S1_CP[l - 1] if S1_KH[l] == 1 else S1_KH[l] * _fwd_seg(l)


def _inv_seg(l):
    return 3 * S1_CP[l] if S1_KH[l] == 1 else _r32(3 * S1_CP[l])


def s1x1_layer(name):
    if not name.startswith("s1x1_"):
        raise KeyError(name)
    rng = _rng(name)
    W, C, CP, KH, h = S1_W, S1_C, S1_CP, S1_KH, S1_H
    step = 5
    if name.startswith("s1x1_conv"):       # conv l, EPI_POST with gate codes, on 64 frames (conv5 / conv6: 55 / 46 rows)
        l = int(name[-1])
        rows = {5: 55, 6: 46}.get(l, 64)
        rows_in = 55 if l == 6 else 64
        K = _fwd_k(l)
        v = plain(0, CP[l], rows * W[l], C[l], K)
        v.update(m_inner=W[l], a_so=W[l - 1] * CP[l - 1], a_si=2 * CP[l - 1])
        if KH[l] > 1:
            v.update(k_seg=_fwd_seg(l), k_ss=W[l - 1] * CP[l - 1])
        fill = _padded(rng, (rows_in, W[l - 1], CP[l - 1]), (slice(None), slice(None), slice(0, C[l - 1])))
        return _case(name, v, fill, _weights(rng, K, C[l]), _bias(rng, C[l]), _bias(rng, C[l]), epi=EPI_POST)
    Pc = 10 if name != "s1x1_invT2" else 4
    rp = [0, 0, 0, 0, 0, 9, 9]
    cpad = [0, 0, 2, 2, 2, 2, 2]
    HP = [h[l] + 2 * rp[l] for l in range(7)]
    WPd = [W[l] + 2 * cpad[l] for l in range(7)]
    if name == "s1x1_1x1":                # EPI_POST | EPI_GATE on rows (k, u, j) of 10 patches, into D6's interior
        h6, W6 = h[6], W[6]
        rows6 = (Pc - 1) * step + h6
        v = plain(0, 0, Pc * h6 * W6, 200, 200)
        v.update(m_inner=h6 * W6, a_so=step * W6 * CP[6], m_inner2=W6, a_si=W6 * CP[6], a_s2=CP[6],
                 cm_inner=h6 * W6, c_so=HP[6] * WPd[6] * CP[6], cm_inner2=W6, c_si=WPd[6] * CP[6], c_s2=CP[6],
                 c_col0=(rp[6] * WPd[6] + cpad[6]) * CP[6],
                 g_inner=h6 * W6, g_so=step * W6 * C[6], g_inner2=W6, g_si=W6 * C[6], g_s2=C[6], g_lim=2 ** 63 - 1)
        fill = np.abs(rng.standard_normal(rows6 * W6 * CP[6])).astype(np.float32)
        gate = rng.integers(0, 3, rows6 * W6 * C[6] + 4096).astype(np.uint8)
        return _case(name, v, fill, _weights(rng, 200, 200), _bias(rng, 200), _bias(rng, 200), gate, EPI_POST | EPI_GATE)
    # InverseLayer(conv l), EPI_GATE: l = 6 with K clipping (K = 6080) and W5 = 61 odd (g_lim drops the last phase);
    # l = 2 into the K3s operand G, W1 = 1023
    l = int(name[-1])
    Pi, Co, Po, M2 = CP[l], C[l - 1], CP[l - 1], (W[l - 1] + 1) // 2
    rowsU = Pc * M2
    v = plain(0, 0, h[l - 1] * rowsU, 2 * Co, KH[l] * _inv_seg(l))
    v.update(m_inner=rowsU, a_so=WPd[l] * Pi, m_inner2=M2, a_si=HP[l] * WPd[l] * Pi, a_s2=Pi,
             k_seg=_inv_seg(l), k_ss=WPd[l] * Pi,
             cm_inner=rowsU, c_so=WPd[l - 1] * Po, cm_inner2=M2, c_si=HP[l - 1] * WPd[l - 1] * Po, c_s2=2 * Po,
             c_col0=(rp[l - 1] * WPd[l - 1] + cpad[l - 1]) * Po, n_seg=Co, n_ss=Po,
             g_inner=rowsU, g_so=W[l - 1] * Co, g_inner2=M2, g_si=step * W[l - 1] * Co, g_s2=2 * Co, g_lim=W[l - 1] * Co)
    if KH[l] > 1:
        v.update(kc_rows=rowsU, kc_unit=_inv_seg(l), kc_pad=KH[l] - 1, kc_n=h[l], kc_taps=KH[l])
    fill = _padded(rng, (Pc, HP[l], WPd[l], Pi), (slice(None), slice(rp[l], rp[l] + h[l]), slice(cpad[l], cpad[l] + W[l]), slice(0, C[l])))
    rows_g = (Pc - 1) * step + h[l - 1]
    gate = rng.integers(0, 3, rows_g * W[l - 1] * Co + 4 * Co * M2).astype(np.uint8)
    return _case(name, v, fill, _weights(rng, v["K"], 2 * Co), gate=gate, epi=EPI_GATE)


def edge_case(name):
    rng = _rng(name)
    kind, _, arg = name.partition(":")
    if kind in ("kclip_span", "kclip_empty"):
        # transposed conv on a zero-padded operand, tap width 52 (blocks straddle taps), rows (u, kd)
        if kind == "kclip_span":     # 40 rows per u: a 128-row tile spans 4 output positions
            taps, pad, n, KD, unit = 5, 4, 6, 40, 52
        else:                        # 64 rows per u, 6 padding rows before 5 data rows: the first and last tiles'
            taps, pad, n, KD, unit = 4, 6, 5, 64, 52   # tap ranges are empty
        HP = n + 2 * pad
        Uo = HP - taps + 1
        v = plain(0, 0, KD * Uo, 24, taps * unit, relu=1)
        v.update(m_inner=KD, a_so=unit, a_si=HP * unit, cm_inner=KD, c_so=28, c_si=Uo * 28,
                 kc_rows=KD, kc_unit=unit, kc_pad=pad, kc_n=n, kc_taps=taps)
        fill = _padded(rng, (KD, HP, unit), (slice(None), slice(pad, pad + n), slice(0, 50)))
        return _case(name, v, fill, _weights(rng, taps * unit, 24), _bias(rng, 24))
    if kind == "splitk":             # one tile, 37 / 33 k-blocks over 4 slices of 10 / 9: the last one ragged; C
        K = int(arg)                 # scattered (three-level rows, n segments), rows past a_valid_rows
        v = plain(K + 4, 0, 100, 40, K)
        v.update(a_valid_rows=90, cm_inner=25, c_so=60, c_si=240, n_seg=8, n_ss=10, c_col0=3)
        fill = np.abs(rng.standard_normal(100 * (K + 4))).astype(np.float32)
        return _case(name, v, fill, _weights(rng, K, 40), _bias(rng, 40))
    if kind == "ktail":              # K = 64 + r with rows 68 / 70 / 69 apart: vector widths 4 / 2 / 1
        r, lda = (int(x) for x in arg.split("/"))
        K = 64 + r
        v = plain(lda, 40, 300, 37, K)
        fill = rng.standard_normal(300 * lda).astype(np.float32)
        return _case(name, v, fill, _weights(rng, K, 37, 0), _bias(rng, 37))
    if kind == "ktail_seg":          # three 32-wide K segments 40 apart, the last one cut short by r
        r = int(arg)
        v = plain(200, 64, 300, 64, 64 + r)
        v.update(k_seg=32, k_ss=40)
        fill = rng.standard_normal(300 * 200).astype(np.float32)
        return _case(name, v, fill, _weights(rng, 64 + r, 64, 0), _bias(rng, 64))
    if kind == "n":                  # BN = 32 / 64 switch and partial column tiles
        N = int(arg)
        v = plain(96, N + 3, 300, N, 96)
        fill = rng.standard_normal(300 * 96).astype(np.float32)
        return _case(name, v, fill, _weights(rng, 96, N, 0), _bias(rng, N))
    if kind == "m":
        M = int(arg)
        v = plain(72, 52, M, 50, 70)
        fill = rng.standard_normal(M * 72).astype(np.float32)
        return _case(name, v, fill, _weights(rng, 70, 50, 0), _bias(rng, 50))
    if kind == "msplit":             # > 65535 row tiles of 128: the FFMA launcher splits M in two halves
        M = 65535 * 128 + 257
        v = plain(4, 3, M, 2, 3)
        v["a_valid_rows"] = int(arg)
        fill = rng.standard_normal(M * 4).astype(np.float32)
        return _case(name, v, fill, _weights(rng, 3, 2, 0), _bias(rng, 2))
    if kind == "int":                # small integers: exact under 3xTF32, pre-activations exactly 0 reach code 1
        epi = int(arg)
        v = plain(40, 80, 200, 72, 40)
        v.update(g_inner=200, g_inner2=1, g_so=0, g_si=72, g_s2=0, g_lim=67)
        fill = rng.integers(-1, 2, 200 * 40).astype(np.float32)
        B = rng.integers(-1, 2, (40, 72)).astype(np.float32)
        gate = rng.integers(0, 3, 200 * 72).astype(np.uint8)
        return _case(name, v, fill, B, rng.integers(-2, 3, 72).astype(np.float32),
                     rng.integers(-1, 2, 72).astype(np.float32), gate, epi, exact=True)
    raise KeyError(name)


LAYERS = (["dsd_conv1", "dsd_conv2", "dsd_bottleneck", "dsd_dec_dense", "dsd_convT2", "sconv_conv1", "sconv_convT2"] +
          ["s1x1_conv%d" % l for l in range(1, 7)] + ["s1x1_1x1", "s1x1_invT6", "s1x1_invT2"])
EDGES = (["kclip_span", "kclip_empty", "splitk:1179", "splitk:1040"] +
         ["ktail:%d/%d" % (r, lda) for r in (1, 2, 3) for lda in (68, 70, 69)] + ["ktail_seg:%d" % r for r in (1, 2, 3)] +
         ["n:%d" % n for n in (1, 31, 32, 33, 64, 65)] + ["m:1", "m:129", "m:257"] +
         ["msplit:%d" % (65535 * 128 - 300), "msplit:1000"] + ["int:%d" % EPI_POST, "int:%d" % (EPI_POST | EPI_GATE)])


def make_case(name):
    for f in (dsd_layer, sconv_layer, s1x1_layer, edge_case):
        try:
            return f(name)
        except KeyError:
            continue
    raise KeyError(name)


# ---------------------------------------------------------------------------------------------- GPU harness
@pytest.fixture(scope="module")
def ctx():
    pytest.importorskip("torch")
    from deepconvsep_b200.engine import Context
    return Context(0)


def _span(idx):
    return int(idx.max()) + 1


def _run(ctx, engine, case, A_dev, C_init, code_len, gate_dev, bias_dev, bias2_dev):
    """one call on fresh C / code buffers; returns (C buffer, code buffer) as host arrays"""
    import torch
    from deepconvsep_b200 import _lib
    v = case["v"]
    C_dev = torch.from_numpy(C_init.view(np.float32)).cuda()
    code_dev = torch.full((code_len + 2 * SLACK,), int(CODE_SENTINEL), dtype=torch.uint8, device="cuda")
    gv = _lib.GemmView(**{f: v[f] for f in FIELDS})
    gv.A = A_dev.data_ptr() + 4 * SLACK
    gv.C = C_dev.data_ptr() + 4 * SLACK
    gv.bias = bias_dev.data_ptr() if bias_dev is not None else None
    gv.bias2 = bias2_dev.data_ptr() if bias2_dev is not None else None
    gv.code = code_dev.data_ptr() + SLACK if case["epi"] & EPI_POST else None
    gv.gate = gate_dev.data_ptr() if gate_dev is not None else None
    B = np.ascontiguousarray(case["B"], dtype=np.float32)
    gv.ldb = B.shape[1]
    _lib.check(ctx.lib.dcs_gemm_view_f32(ctx.handle, engine, case["epi"], _ctypes_ref(gv), B.ctypes.data, None))
    return C_dev.cpu().numpy().view(np.uint32), code_dev.cpu().numpy()


def _ctypes_ref(x):
    import ctypes
    return ctypes.byref(x)


_REF_CACHE = {}


def _prepared(name):
    """the case, its A buffer (NaN outside the view), the float64 reference and the C offsets, computed once"""
    if name in _REF_CACHE:
        return _REF_CACHE[name]
    _REF_CACHE.clear()
    case = make_case(name)
    v = case["v"]
    a_size = int(a_rows(v).max() + a_cols(v).max()) + 1       # every row m < M, valid or not, lies inside
    fill = case["fill"]
    if fill.size < a_size:   # padded K segments read past the layer's buffer into the zeroed slack after it (S1_SLACK)
        fill = np.concatenate([fill, np.zeros(a_size - fill.size, np.float32)])
    A = np.where(a_addressed(v, fill.size), fill, np.float32(np.nan)).astype(np.float32)
    A = np.concatenate([np.full(SLACK, np.nan, np.float32), A, np.full(SLACK, np.nan, np.float32)])
    ref = reference(v, A[SLACK:], case["B"], case["bias"], case["bias2"], case["gate"], case["epi"])
    if case["gate"] is not None:   # every (m, n), stored or not, reads inside the gate array
        assert gate_index(v)[0].max() < case["gate"].size
    ci = c_index(v)
    written = ci[ref["stored"]]
    assert len(np.unique(written)) == written.size, "the case's view writes one C element twice"
    c_size = _span(ci) + 2 * SLACK                               # covers every (m, n), stored or not
    _REF_CACHE[name] = (case, A, ref, ci, c_size)
    return _REF_CACHE[name]


ENGINES = {"tc": 1, "ffma": 0}


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ["tc", "ffma"])
@pytest.mark.parametrize("name", LAYERS + EDGES)
def test_gemm_view_matches_float64(ctx, name, engine):
    import torch
    case, A, ref, ci, c_size = _prepared(name)
    v, epi = case["v"], case["epi"]
    if epi and engine == "ffma":
        pytest.skip("the gated epilogues exist on the tensor-core engine only")
    if engine == "ffma" and v["M"] > 65535 * 128 and v["m_inner"] != 1:
        pytest.skip("the FFMA launcher splits only dense rows")
    dev = lambda x: None if x is None else torch.from_numpy(np.ascontiguousarray(x)).cuda()
    A_dev = dev(A)
    C_init = np.full(c_size, C_SENTINEL, dtype=np.uint32)
    code_len = v["M"] * v["N"]
    outs = [_run(ctx, ENGINES[engine], case, A_dev, C_init, code_len, dev(case["gate"]), dev(case["bias"]),
                 dev(case["bias2"])) for _ in range(2)]
    (Cb, codes), (Cb2, codes2) = outs
    assert np.array_equal(Cb, Cb2) and np.array_equal(codes, codes2), "two runs gave different bits"

    stored = ref["stored"]
    written = np.zeros(c_size, dtype=bool)
    written[SLACK + ci[stored]] = True
    assert np.array_equal(Cb[~written], C_init[~written]), \
        "%d C elements outside the view changed" % int((Cb[~written] != C_init[~written]).sum())
    got = Cb.view(np.float32)[SLACK + ci].astype(np.float64)
    assert np.isfinite(got[stored]).all(), "%d stored values are not finite" % int((~np.isfinite(got[stored])).sum())

    err = np.abs(got - ref["out"])[stored]
    bnd = bound(ref, c_tc(v["K"]) if engine == "tc" else c_ffma(v["K"]))[stored]
    ratio = np.where(err > 0, err / np.maximum(bnd, 1e-300), 0.0)
    worst = float(ratio.max())
    record("gemm_view:" + name, engine=engine, K=v["K"], M=v["M"], N=v["N"], worst_error_over_bound=worst)
    assert worst <= 1.0, (name, engine, worst, np.unravel_index(int(np.argmax(ratio)), ratio.shape))
    zero_rows = ref["S"][stored] == 0        # rows of an empty tap range, rows past a_valid_rows: exactly act(bias)
    assert np.array_equal(got[stored][zero_rows], ref["out"][stored][zero_rows])
    if case["exact"]:
        assert np.array_equal(got[stored], ref["out"][stored])

    if epi & EPI_POST:
        assert (codes[:SLACK] == CODE_SENTINEL).all() and (codes[SLACK + code_len:] == CODE_SENTINEL).all()
        dev_codes = codes[SLACK:SLACK + code_len].reshape(v["M"], v["N"])
        pre_bound = c_tc(v["K"]) * ref["S"] + U * np.abs(ref["pre"])
        sure = np.abs(ref["pre"]) > pre_bound     # the sign of pre is settled by the bound
        if case["exact"]:
            sure[:] = True
            assert (ref["code"] == 1).sum() > 0
        assert np.array_equal(dev_codes[sure], ref["code"][sure])
    if name == "kclip_empty":
        assert zero_rows.sum() >= 128 * v["N"]


@pytest.mark.gpu
@pytest.mark.parametrize("engine", [1, 0])
@pytest.mark.parametrize("field,value", [("c_col0", -1), ("c_so", -52), ("n_ss", -1)])
def test_negative_c_offsets_are_refused(ctx, engine, field, value):
    """A view whose C offsets could go below the C pointer is refused by both launchers before anything runs (every
    layer builds its views from non-negative strides, so neither epilogue checks the lower bound)."""
    import torch
    from deepconvsep_b200 import _lib
    v = plain(16, 52, 40, 50, 16)
    v.update(n_seg=25, n_ss=26)
    v[field] = value
    A = torch.ones(40 * 16, device="cuda")
    C = torch.full((64 * 52,), 7.0, device="cuda")
    gv = _lib.GemmView(**{f: v[f] for f in FIELDS})
    gv.A, gv.C = A.data_ptr(), C.data_ptr() + 4 * 64
    B = np.ones((16, 50), dtype=np.float32)
    n0 = ctx.launch_count()
    rc = ctx.lib.dcs_gemm_view_f32(ctx.handle, engine, 0, _ctypes_ref(gv), B.ctypes.data, None)
    assert rc == -1 and b"negative C" in ctx.lib.dcs_last_error()
    assert ctx.launch_count() == n0 and (C == 7.0).all()


@pytest.mark.gpu
def test_epilogues_need_the_tensor_core_engine(ctx):
    import torch
    A = torch.ones(64 * 64, device="cuda")
    C = torch.zeros(64 * 64, device="cuda")
    from deepconvsep_b200 import _lib
    gv = _lib.GemmView(**{f: plain(64, 64, 64, 64, 64)[f] for f in FIELDS})
    gv.A, gv.C, gv.bias, gv.bias2 = A.data_ptr(), C.data_ptr(), A.data_ptr(), A.data_ptr()
    B = np.ones((64, 64), dtype=np.float32)
    for engine, epi in ((0, EPI_POST), (0, EPI_GATE), (2, 0), (1, 4)):
        assert ctx.lib.dcs_gemm_view_f32(ctx.handle, engine, epi, _ctypes_ref(gv), B.ctypes.data, None) == -1
