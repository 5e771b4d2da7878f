"""InverseLayer(conv2) of the DSD nets on its own tensor-core kernel (dsd_convT2_tc.cu, through dcs_dsd_convt2_f32),
against the generic tensor-core GEMM on the same overlapping view of apad (dcs_gemm_view_f32, engine 1) and against
float64.

Every case
  - requires G to equal the GEMM's G as values (the kernel keeps the GEMM's accumulation plan: the same 32-wide stages
    at the same absolute K offsets, and the stages either kernel adds or skips are exact zeros);
  - requires |G - G64| <= the per-element bound of tests/test_gpu_gemm_views.py (3xTF32 plan, c(K) = (128 + K/16) u);
  - fills every padding row of apad with NaN (the GEMM reference runs on a zero-padded copy of the same buffer), so a
    read of one would show;
  - fills G columns 50..51 and the elements around G with a NaN-payload sentinel, which must stay;
  - runs twice and requires the same bits.
Pair counts: 1, Q - 1, Q, Q + 1 (Q pairs per block), one giving more items than SMs, the 180 s clip's P * ndec (3096
patches), and one where a CTA's range starts on a block's last u block."""
import ctypes
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_gemm_views import FIELDS, SLACK, C_SENTINEL, U, bound, c_tc, plain  # noqa: E402

pytestmark = pytest.mark.gpu

CP, NF = 52, 50
P_180S = 3096   # patches of a 180 s clip at time_context 30, overlap 25 (15506 frames)


def geometry(tc):
    kh2 = tc // 2
    h2 = tc - kh2 + 1
    u = 4 if h2 <= 16 else 8          # output positions per item (dsd_convT2_tc.cu launch_dsd_convT2_tc)
    return kh2, h2, h2 + 2 * (kh2 - 1), 128 // u, -(-tc // u)


def _ranges(items, nsm):
    grid = min(nsm, items)
    return [items * b // grid for b in range(grid)]


def pair_counts(tc, nsm):
    kh2, h2, hp, q, nub = geometry(tc)
    more = q * -(-(nsm + 1) // nub)               # ceil(npairs / Q) * nub > SM count
    last_ub = None
    for n in range(more, more + 64 * q):         # some CTA's range starts on u block nub - 1
        items = -(-n // q) * nub
        if any(i0 % nub == nub - 1 for i0 in _ranges(items, nsm)):
            last_ub = n
            break
    assert last_ub is not None
    return {"one": 1, "q_minus_1": q - 1, "q": q, "q_plus_1": q + 1, "sm_plus_1": more, "last_ub": last_ub}


@pytest.fixture(scope="module")
def ctx():
    pytest.importorskip("torch")
    from deepconvsep_b200.engine import Context
    return Context(0)


@pytest.fixture(scope="module")
def nsm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _inputs(tc, npairs, seed):
    """apad with NaN padding rows (and the NaN-free copy the GEMM reads), the host weight [52 kh2][50]"""
    kh2, h2, hp, _, _ = geometry(tc)
    rng = np.random.default_rng(seed)
    ap = np.full((npairs, hp, CP), np.nan, dtype=np.float32)
    inner = rng.random((npairs, h2, CP), dtype=np.float32)       # post-ReLU activations: non-negative
    inner[:, :, NF:] = 0.0                                       # pad channels, zero as the dense layer leaves them
    ap[:, kh2 - 1:kh2 - 1 + h2] = inner
    W = rng.standard_normal((kh2 * CP, NF)).astype(np.float32)
    W[:, :8] = np.abs(W[:, :8])                                  # sign-coherent columns: plain TF32 fails the bound
    W.reshape(kh2, CP, NF)[:, NF:] = 0.0                         # pad channels of the transposed conv2 weight
    return ap, np.nan_to_num(ap, nan=0.0), W


def _flat_with_slack(a, fill):
    buf = np.full(a.size + 2 * SLACK, fill, dtype=a.dtype)
    buf[SLACK:SLACK + a.size] = a.ravel()
    return buf


def _g_init(npairs, tc, ldg):
    return np.full(npairs * tc * ldg + 2 * SLACK, C_SENTINEL, dtype=np.uint32)


def _run_convT2(ctx, ap_dev, tc, npairs, ldg, W):
    import torch
    from deepconvsep_b200 import _lib
    G_dev = torch.from_numpy(_g_init(npairs, tc, ldg).view(np.float32)).cuda()
    v = _lib.DsdConvT2View(apad=ap_dev.data_ptr() + 4 * SLACK, G=G_dev.data_ptr() + 4 * SLACK, ldg=ldg, npairs=npairs, tc=tc)
    _lib.check(ctx.lib.dcs_dsd_convt2_f32(ctx.handle, ctypes.byref(v), W.ctypes.data, None))
    return G_dev.cpu().numpy().view(np.uint32)


def _run_gemm(ctx, ap_dev, tc, npairs, ldg, W):
    """the layer as dsd_forward built it before: the generic GEMM on the u-major overlapping view of apad"""
    import torch
    from deepconvsep_b200 import _lib
    kh2, h2, hp, _, _ = geometry(tc)
    v = plain(0, ldg, npairs * tc, NF, kh2 * CP)
    v.update(m_inner=npairs, a_so=CP, a_si=hp * CP, cm_inner=npairs, c_so=ldg, c_si=tc * ldg,
             kc_rows=npairs, kc_unit=CP, kc_pad=kh2 - 1, kc_n=h2, kc_taps=kh2, ldb=NF)
    G_dev = torch.from_numpy(_g_init(npairs, tc, ldg).view(np.float32)).cuda()
    gv = _lib.GemmView(**{f: v[f] for f in FIELDS})
    gv.A = ap_dev.data_ptr() + 4 * SLACK
    gv.C = G_dev.data_ptr() + 4 * SLACK
    _lib.check(ctx.lib.dcs_gemm_view_f32(ctx.handle, 1, 0, ctypes.byref(gv), W.ctypes.data, None))
    return G_dev.cpu().numpy().view(np.uint32)


def _float64(ap0, W, tc):
    """G64 and S = sum |a w| per element, on the GPU in float64"""
    import torch
    kh2 = tc // 2
    a = torch.from_numpy(ap0).cuda().double()
    w = torch.from_numpy(W).cuda().double().reshape(kh2, CP, NF)
    out = torch.zeros(a.shape[0], tc, NF, dtype=torch.float64, device="cuda")
    S = torch.zeros_like(out)
    for q in range(kh2):
        blk = a[:, q:q + tc, :]
        out += blk @ w[q]
        S += blk.abs() @ w[q].abs()
    return out.cpu().numpy(), S.cpu().numpy()


TCS = (4, 5, 30, 31, 64)
COUNTS = ("one", "q_minus_1", "q", "q_plus_1", "sm_plus_1", "last_ub", "clip_180s")
# the kernel sees P * ndec pairs, whatever ndec is: both decoder counts at the clip's pair count
CASES = [(c, 3) for c in COUNTS] + [("clip_180s", 4)]


@pytest.mark.parametrize("count,ndec", CASES)
@pytest.mark.parametrize("tc", TCS)
def test_convT2_matches_gemm_and_float64(ctx, nsm, tc, count, ndec):
    import torch
    npairs = P_180S * ndec if count == "clip_180s" else pair_counts(tc, nsm)[count]
    ldg = 52
    kh2 = tc // 2
    ap, ap0, W = _inputs(tc, npairs, seed=1000 * tc + 10 * ndec + COUNTS.index(count))
    ap_dev = torch.from_numpy(_flat_with_slack(ap, np.float32(np.nan))).cuda()
    ap0_dev = torch.from_numpy(_flat_with_slack(ap0, np.float32(0.0))).cuda()

    got = _run_convT2(ctx, ap_dev, tc, npairs, ldg, W)
    again = _run_convT2(ctx, ap_dev, tc, npairs, ldg, W)
    assert np.array_equal(got, again), "two runs differ in bits"
    ref = _run_gemm(ctx, ap0_dev, tc, npairs, ldg, W)

    # sentinels: around G and in columns 50..51 of every row
    assert (got[:SLACK] == C_SENTINEL).all() and (got[-SLACK:] == C_SENTINEL).all()
    G = got[SLACK:-SLACK].reshape(npairs, tc, ldg)
    assert (G[:, :, NF:] == C_SENTINEL).all(), "columns 50..51 were written"
    Gf = G[:, :, :NF].view(np.float32)
    assert np.isfinite(Gf).all(), "a padding row of apad was read, or a column was not stored"

    Gg = ref[SLACK:-SLACK].reshape(npairs, tc, ldg)[:, :, :NF].view(np.float32)
    diff = Gf != Gg
    assert not diff.any(), "G differs from the GEMM path at %d elements, first %s" % (diff.sum(), np.argwhere(diff)[0])

    G64, S = _float64(ap0, W, tc)
    bnd = bound(dict(g=1.0, S=S, pre=G64, post=G64), c_tc(kh2 * CP))
    err = np.abs(Gf.astype(np.float64) - G64)
    assert (err <= bnd).all(), "worst |error| / bound %.3g" % float((err / bnd).max())


def test_pair_count_cases_reach_their_edges(nsm):
    """the generated counts hit what they are named for"""
    for tc in TCS:
        kh2, h2, hp, q, nub = geometry(tc)
        c = pair_counts(tc, nsm)
        assert -(-c["sm_plus_1"] // q) * nub > nsm
        items = -(-c["last_ub"] // q) * nub
        assert any(i0 % nub == nub - 1 for i0 in _ranges(items, nsm))


def test_refusals_queue_no_work(ctx):
    import torch
    from deepconvsep_b200 import _lib
    tc, npairs, ldg = 30, 40, 52
    ap, _, W = _inputs(tc, npairs, seed=7)
    ap_dev = torch.from_numpy(_flat_with_slack(ap, np.float32(np.nan))).cuda()
    G_dev = torch.from_numpy(_g_init(npairs, tc, ldg + 2).view(np.float32)).cuda()
    good = dict(apad=ap_dev.data_ptr() + 4 * SLACK, G=G_dev.data_ptr() + 4 * SLACK, ldg=ldg, npairs=npairs, tc=tc)
    bad = [dict(apad=None), dict(G=None), dict(npairs=0), dict(npairs=-1), dict(tc=3), dict(tc=65), dict(ldg=49),
           dict(ldg=53), dict(apad=good["apad"] + 4), dict(G=good["G"] + 4), dict(npairs=(1 << 31) // tc + 1)]
    before = G_dev.cpu().numpy().view(np.uint32).copy()
    n0 = ctx.lib.dcs_launch_count(ctx.handle)
    for kw in bad:
        v = _lib.DsdConvT2View(**dict(good, **kw))
        assert ctx.lib.dcs_dsd_convt2_f32(ctx.handle, ctypes.byref(v), W.ctypes.data, None) == -1, kw
    v = _lib.DsdConvT2View(**good)
    assert ctx.lib.dcs_dsd_convt2_f32(ctx.handle, ctypes.byref(v), None, None) == -1
    assert ctx.lib.dcs_dsd_convt2_f32(None, ctypes.byref(v), W.ctypes.data, None) == -1
    torch.cuda.synchronize()
    assert ctx.lib.dcs_launch_count(ctx.handle) == n0
    assert np.array_equal(G_dev.cpu().numpy().view(np.uint32), before)
    # and the good view runs
    _lib.check(ctx.lib.dcs_dsd_convt2_f32(ctx.handle, ctypes.byref(v), W.ctypes.data, None))
    assert ctx.lib.dcs_launch_count(ctx.handle) == n0 + 1
