"""Edges of the warp-specialised schedule of the wgmma mask + cross-fade kernel (dsd_tc.cu) against the float64
reference of test_gpu_mask_views.py, element by element, with its per-element bound (192u for the tensor-core bins).

The kernel runs persistent CTAs over contiguous ranges of (tile, group) items; a producer warpgroup fills two B
stages and two consumer warpgroups alternate on the tensor cores, half an item apart.  When F = 128 m + 1 the tiles
cover bins [0, F - 1) and the producer computes the Nyquist bin from the fp32 rows it loads.  The cases, sized from the
device's SM count S, put the schedule at its edges:

- S + 1 items: one CTA runs two items, the others one;
- 2 S and 3 S items: every CTA runs an even or an odd number of items, so the last item ends on either consumer;
- a CTA range that starts on the last item of a tile: the consumers reload A after their first item;
- F = 129: one full tile and the Nyquist bin is all there is;
- F = 513 and F = 2049 with the DSD100 net (3 decoders) and the stereo net (4).

Every case runs twice with identical bits, leaves the NaN sentinels around and between the output planes untouched,
and reports the worst error / bound ratio at the Nyquist bin apart from the bins below it."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from parity import record  # noqa: E402
from test_gpu_mask_views import (S_SENTINEL, SLACK, Buffers, _plane_map, _run, dsd_case, evaluate,  # noqa: E402
                                 reference_masks, well_fraction)

pytestmark = pytest.mark.gpu
BINS, FRAMES = 128, {3: 8, 4: 4}


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _tile_last_start(F, ndec, sms, t_min):
    """the smallest T >= t_min at which some CTA's range starts on the last item of a tile"""
    tiles = (F - 1) // BINS
    for T in range(t_min, t_min + 64 * FRAMES[ndec]):
        groups = -(-T // FRAMES[ndec])
        items = tiles * groups
        ctas = min(sms, items)
        starts = [i * items // ctas for i in range(1, ctas)]
        if any(s % groups == groups - 1 for s in starts):
            return T
    raise AssertionError("no such T")


# name -> (F, T(S), ndec)
CASES = {
    "items_sms_plus_1": lambda S: (129, 8 * S + 3, 3),
    "items_2sms_even": lambda S: (129, 16 * S, 3),
    "items_3sms_odd": lambda S: (129, 24 * S, 3),
    "ild_items_3sms_odd": lambda S: (129, 12 * S, 4),
    "range_starts_on_tile_last": lambda S: (257, _tile_last_start(257, 3, S, 4 * S), 3),
    "F129": lambda S: (129, 300, 3),
    "F513": lambda S: (513, 200, 3),
    "F513_ild": lambda S: (513, 150, 4),
    "F2049": lambda S: (2049, 150, 3),
    "F2049_ild": lambda S: (2049, 101, 4),
}


@pytest.fixture(scope="module")
def ctx():
    pytest.importorskip("torch")
    from deepconvsep_b200.engine import Context
    return Context(0)


def _bins(ref, sl):
    """the reference restricted to the bins `sl`"""
    out = dict(ref)
    for k in ("M", "errM"):
        out[k] = ref[k][:, :, sl]
    for k in ("ill", "settled_all"):
        out[k] = ref[k][:, sl]
    return out


@pytest.mark.parametrize("name", list(CASES))
def test_mask_pipeline_edges_match_float64(ctx, name):
    F, T, ndec = CASES[name](_sms())
    case = dsd_case("pipeline_" + name, F, T, 30, 25, ndec=ndec)
    case["engine"] = "tc"
    b = Buffers(case)
    Sb = _run(ctx, case, b, 1)
    assert np.array_equal(Sb, _run(ctx, case, b, 1)), "two runs gave different bits"

    ldf = case["ldf"]
    body = Sb[2 * SLACK:2 * SLACK + 2 * b.nplanes * b.sp].reshape(b.nplanes, b.sp, 2)
    written = np.zeros((b.nplanes, b.sp), bool)
    written[:, :T * ldf].reshape(b.nplanes, T, ldf)[:, :, :F] = True
    assert (Sb[:2 * SLACK] == S_SENTINEL).all() and (Sb[2 * SLACK + 2 * b.nplanes * b.sp:] == S_SENTINEL).all()
    assert (body[~written] == S_SENTINEL).all(), "%d S elements outside the written frames and bins changed" % \
        int((body[~written] != S_SENTINEL).any(-1).sum())
    vals = body[:, :T * ldf].reshape(b.nplanes, T, ldf, 2).view(np.float32)[:, :, :F]
    assert np.isfinite(vals).all(), "%d stored values are not finite" % int((~np.isfinite(vals)).sum())
    S = vals[..., 0] + 1j * vals[..., 1].astype(np.float64)

    pm = _plane_map(case)
    worst = {"below": 0.0, "nyquist": 0.0}
    fails, wf = [], 1.0
    for mset in sorted(set(m for _, m, _ in pm)):
        ref = reference_masks(case, np.arange(T), mset)
        wf = min(wf, well_fraction(ref))
        for xpl in sorted(set(x for _, m, x in pm if m == mset)):
            idx = [i for i, (s, m, x) in enumerate(pm) if m == mset and x == xpl]
            for part, sl in (("below", slice(0, F - 1)), ("nyquist", slice(F - 1, F))):
                wo, fa = evaluate(_bins(ref, sl), S[idx][:, :, sl], case["X"][xpl][:, sl])
                worst[part] = max(worst[part], wo)
                fails += ["%s: %s" % (part, f) for f in fa]
    record("mask_pipeline:" + name, F=F, T=T, ndec=ndec, well_conditioned=wf,
           worst_error_over_bound=max(worst.values()), worst_below_nyquist=worst["below"],
           worst_at_nyquist=worst["nyquist"])
    assert not fails, (name, fails)
    assert wf >= 0.99, (name, wf)
    assert worst["below"] <= 1.0 and worst["nyquist"] <= 1.0, (name, worst)
