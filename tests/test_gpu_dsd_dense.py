"""The decoder dense layers of the DSD nets on their own tensor-core kernel (dsd_dense_tc.cu, through dcs_dsd_dense_f32),
against the generic tensor-core GEMM on the same scattered view of apad (dcs_gemm_view_f32, engine 1) and against
float64.

Every case
  - requires apad to equal the GEMM's apad bit for bit (the kernel keeps the GEMM's accumulation plan: the same 32-wide
    stages, the same correction accumulator, the same epilogue order);
  - requires |apad - ReLU(z W + b)_64| <= the per-element bound of tests/test_gpu_gemm_views.py (3xTF32 plan,
    c(K) = (128 + K/16) u);
  - fills every padding row of apad and the elements around it with a NaN-payload sentinel, which must stay, and the
    elements around z with NaN;
  - runs twice and requires the same bits.
Patch counts: 1, one 64-row block per CTA minus one / exact / plus one (the CTAs of a slab split the patches into equal
contiguous ranges), the SM count + 1, and the 180 s clip's 3096."""
import ctypes
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_gemm_views import FIELDS, SLACK, C_SENTINEL, bound, c_tc, plain  # noqa: E402

pytestmark = pytest.mark.gpu

CP, NF = 52, 50
P_180S = 3096   # patches of a 180 s clip at time_context 30, overlap 25 (15506 frames)
SLAB = 96       # GEMM columns per CTA (dsd_dense_tc.cu DN_NS)
ROWS = 64       # rows per block


def geometry(tc, ndec):
    kh2 = tc // 2
    h2 = tc - kh2 + 1
    nfc = 128 if ndec == 3 else 256     # DSD100 / HHDS and the stereo / ILD net
    return kh2, h2, h2 + 2 * (kh2 - 1), nfc, ndec * h2 * CP


def ctas_per_slab(n, nsm, P):
    """dsd_dense_tc.cu launch_dsd_dense_tc"""
    return max(1, min(nsm // -(-n // SLAB), P))


def patch_counts(tc, ndec, nsm):
    n = geometry(tc, ndec)[4]
    c = ctas_per_slab(n, nsm, 1 << 30)
    return {"one": 1, "block_minus_1": ROWS * c - 1, "block": ROWS * c, "block_plus_1": ROWS * c + 1,
            "sm_plus_1": nsm + 1, "clip_180s": P_180S}


@pytest.fixture(scope="module")
def ctx():
    pytest.importorskip("torch")
    from deepconvsep_b200.engine import Context
    return Context(0)


@pytest.fixture(scope="module")
def nsm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _inputs(tc, ndec, P, seed):
    """z (post-ReLU: non-negative), the host weight [nfc][N] and bias [N], zero at the pad channels as the model has them"""
    _, h2, _, nfc, n = geometry(tc, ndec)
    rng = np.random.default_rng(seed)
    z = rng.random((P, nfc), dtype=np.float32)
    W = (rng.standard_normal((nfc, n)) / np.sqrt(nfc)).astype(np.float32)
    W[:, :8] = np.abs(W[:, :8])                       # sign-coherent columns: plain TF32 fails the bound
    b = (0.1 * rng.standard_normal(n)).astype(np.float32)
    W.reshape(nfc, ndec * h2, CP)[:, :, NF:] = 0.0
    b.reshape(ndec * h2, CP)[:, NF:] = 0.0
    return z, W, b


def _with_slack(a, fill):
    buf = np.full(a.size + 2 * SLACK, fill, dtype=a.dtype)
    buf[SLACK:SLACK + a.size] = a.ravel()
    return buf


def _apad_init(tc, ndec, P):
    hp = geometry(tc, ndec)[2]
    return np.full(P * ndec * hp * CP + 2 * SLACK, C_SENTINEL, dtype=np.uint32)


def _view(z_dev, b_dev, apad_dev, shape, **kw):
    """the view of a (P, tc, ndec) case; kw overrides fields"""
    from deepconvsep_b200 import _lib
    P, tc, ndec = shape
    args = dict(z=z_dev.data_ptr() + 4 * SLACK, bias=b_dev.data_ptr(), apad=apad_dev.data_ptr() + 4 * SLACK,
                P=P, tc=tc, ndec=ndec, nfc=geometry(tc, ndec)[3])
    args.update(kw)
    return _lib.DsdDenseView(**args)


def _run_dense(ctx, z_dev, b_dev, tc, ndec, P, W):
    import torch
    from deepconvsep_b200 import _lib
    apad_dev = torch.from_numpy(_apad_init(tc, ndec, P).view(np.float32)).cuda()
    v = _view(z_dev, b_dev, apad_dev, (P, tc, ndec))
    _lib.check(ctx.lib.dcs_dsd_dense_f32(ctx.handle, ctypes.byref(v), W.ctypes.data, W.shape[0], W.shape[1], None))
    return apad_dev.cpu().numpy().view(np.uint32)


def _run_gemm(ctx, z_dev, b_dev, tc, ndec, P, W):
    """the layer as dsd_forward built it before: the generic GEMM, columns scattered by n_seg / n_ss / c_col0"""
    import torch
    from deepconvsep_b200 import _lib
    kh2, h2, hp, nfc, n = geometry(tc, ndec)
    v = plain(nfc, ndec * hp * CP, P, n, nfc, relu=1)
    v.update(n_seg=h2 * CP, n_ss=hp * CP, c_col0=(kh2 - 1) * CP)
    apad_dev = torch.from_numpy(_apad_init(tc, ndec, P).view(np.float32)).cuda()
    gv = _lib.GemmView(**{f: v[f] for f in FIELDS})
    gv.A = z_dev.data_ptr() + 4 * SLACK
    gv.C = apad_dev.data_ptr() + 4 * SLACK
    gv.bias = b_dev.data_ptr()
    _lib.check(ctx.lib.dcs_gemm_view_f32(ctx.handle, 1, 0, ctypes.byref(gv), W.ctypes.data, None))
    return apad_dev.cpu().numpy().view(np.uint32)


def _float64(z, W, b):
    """pre = z W + b, post = ReLU(pre) and S = |z| |W|, on the GPU in float64"""
    import torch
    zd, Wd = torch.from_numpy(z).cuda().double(), torch.from_numpy(W).cuda().double()
    pre = zd @ Wd + torch.from_numpy(b).cuda().double()
    S = zd.abs() @ Wd.abs()
    return pre.cpu().numpy(), torch.relu(pre).cpu().numpy(), S.cpu().numpy()


TCS = (4, 5, 30, 31, 64)
COUNTS = ("one", "block_minus_1", "block", "block_plus_1", "sm_plus_1", "clip_180s")


@pytest.mark.parametrize("count", COUNTS)
@pytest.mark.parametrize("ndec", (3, 4))
@pytest.mark.parametrize("tc", TCS)
def test_dense_matches_gemm_and_float64(ctx, nsm, tc, ndec, count):
    import torch
    P = patch_counts(tc, ndec, nsm)[count]
    kh2, h2, hp, nfc, n = geometry(tc, ndec)
    z, W, b = _inputs(tc, ndec, P, seed=1000 * tc + 10 * ndec + COUNTS.index(count))
    z_dev = torch.from_numpy(_with_slack(z, np.float32(np.nan))).cuda()
    b_dev = torch.from_numpy(b).cuda()

    got = _run_dense(ctx, z_dev, b_dev, tc, ndec, P, W)
    again = _run_dense(ctx, z_dev, b_dev, tc, ndec, P, W)
    assert np.array_equal(got, again), "two runs differ in bits"
    ref = _run_gemm(ctx, z_dev, b_dev, tc, ndec, P, W)

    # sentinels: around apad and in every padding row
    assert (got[:SLACK] == C_SENTINEL).all() and (got[-SLACK:] == C_SENTINEL).all()
    ap = got[SLACK:-SLACK].reshape(P, ndec, hp, CP)
    interior = np.zeros(hp, dtype=bool)
    interior[kh2 - 1:kh2 - 1 + h2] = True
    assert (ap[:, :, ~interior] == C_SENTINEL).all(), "a padding row of apad was written"
    inner = ap[:, :, interior].view(np.float32).reshape(P, n)
    assert np.isfinite(inner).all(), "an interior element was not stored"

    diff = got != ref
    assert not diff.any(), "apad differs from the GEMM path at %d elements, first %s" % (
        diff.sum(), np.argwhere(diff)[0])

    pre, post, S = _float64(z, W, b)
    bnd = bound(dict(g=1.0, S=S, pre=pre, post=post), c_tc(nfc))
    err = np.abs(inner.astype(np.float64) - post)
    assert (err <= bnd).all(), "worst |error| / bound %.3g" % float((err / bnd).max())


def test_patch_count_cases_reach_their_edges(nsm):
    """the block cases give every CTA of a slab one 64-row block, one row fewer for some, one more for one"""
    for tc in TCS:
        for ndec in (3, 4):
            n = geometry(tc, ndec)[4]
            c = patch_counts(tc, ndec, nsm)
            for name, lo, hi in (("block_minus_1", ROWS - 1, ROWS), ("block", ROWS, ROWS), ("block_plus_1", ROWS, ROWS + 1)):
                P = c[name]
                cps = ctas_per_slab(n, nsm, P)
                sizes = [P * (i + 1) // cps - P * i // cps for i in range(cps)]
                assert lo <= min(sizes) and max(sizes) <= hi and (lo if name == "block_minus_1" else hi) in sizes, \
                    (tc, ndec, name, sizes)


def test_refusals_queue_no_work(ctx):
    import torch
    from deepconvsep_b200 import _lib
    tc, ndec, P = 30, 3, 40
    nfc, n = geometry(tc, ndec)[3:]
    z, W, b = _inputs(tc, ndec, P, seed=7)
    z_dev = torch.from_numpy(_with_slack(z, np.float32(np.nan))).cuda()
    b_dev = torch.from_numpy(b).cuda()
    apad_dev = torch.from_numpy(_apad_init(tc, ndec, P).view(np.float32)).cuda()
    good = _view(z_dev, b_dev, apad_dev, (P, tc, ndec))
    bad = [dict(z=None), dict(bias=None), dict(apad=None), dict(P=0), dict(P=-1), dict(tc=3), dict(tc=65),
           dict(ndec=2), dict(ndec=5), dict(nfc=0), dict(nfc=100), dict(nfc=288),
           dict(apad=good.apad + 4), dict(z=good.z + 2), dict(bias=good.bias + 2)]
    before = apad_dev.cpu().numpy().view(np.uint32).copy()
    n0 = ctx.lib.dcs_launch_count(ctx.handle)
    for kw in bad:
        v = _view(z_dev, b_dev, apad_dev, (P, tc, ndec), **kw)
        assert ctx.lib.dcs_dsd_dense_f32(ctx.handle, ctypes.byref(v), W.ctypes.data, nfc, n, None) == -1, kw
    for rows, cols in ((nfc + 1, n), (nfc, n - CP), (nfc, n + 1), (128, 3 * 17 * CP)):
        assert ctx.lib.dcs_dsd_dense_f32(ctx.handle, ctypes.byref(good), W.ctypes.data, rows, cols, None) == -1
    assert ctx.lib.dcs_dsd_dense_f32(ctx.handle, ctypes.byref(good), None, nfc, n, None) == -1
    assert ctx.lib.dcs_dsd_dense_f32(None, ctypes.byref(good), W.ctypes.data, nfc, n, None) == -1
    torch.cuda.synchronize()
    assert ctx.lib.dcs_launch_count(ctx.handle) == n0
    assert np.array_equal(apad_dev.cpu().numpy().view(np.uint32), before)
    # and the good view runs
    _lib.check(ctx.lib.dcs_dsd_dense_f32(ctx.handle, ctypes.byref(good), W.ctypes.data, nfc, n, None))
    assert ctx.lib.dcs_launch_count(ctx.handle) == n0 + 1
