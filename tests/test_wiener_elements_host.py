"""The element-wise bound of tests/wiener_elements_oracle.py, on the CPU:

- the float64 emulation of the device's plan (chunk-ordered sums, adjugate / L D L^H without pivoting, one fp32 rounding
  per component) stays under the bound against em_step on every case the GPU element tests run, same generator and
  seeds;
- every mutant of that plan exceeds the bound on at least one element of the mutant cases; whether the per-plane
  relative L2 <= 1e-5 bar of the end-to-end Wiener tests would have accepted it is recorded next to that verdict;
- the generated cases carry the features they promise."""
import numpy as np
import pytest

import wiener_elements_oracle as we
from parity import record

L2_BAR = 1e-5
# nx = 2 and 8 at radius 1 (the windows differ: chunk 0's has s = 1), nx = 3 with one source, nx = 5 at radius 0
MUTANT_CASES = [(2, 4, 300, 129, 1), (3, 1, 300, 129, 1), (5, 3, 300, 129, 0), (8, 4, 300, 129, 1)]


@pytest.fixture(scope="module")
def references():
    cache = {}

    def get(c):
        if c not in cache:
            X, Y = we.make_case(c)
            cache[c] = (X, Y) + we.reference(X, Y, c[4])
        return cache[c]
    return get


@pytest.mark.parametrize("c", we.CASES, ids=we.case_id)
def test_the_device_plan_is_within_the_bound(c, references):
    X, Y, ref, slack = references(c)
    got = we.emulate(X, Y, c[4])
    res = we.check(got, ref, slack, c[4])
    record("wiener_elements_emulation_" + we.case_id(c), ratio=res["ratio"], fp64_fraction=res["fp64_fraction"])
    assert res["ok"], res
    assert not np.array_equal(got, Y.astype(np.complex64))                  # it filtered


@pytest.mark.parametrize("mutant", we.MUTANTS)
def test_each_mutant_is_rejected(mutant, references):
    rejected, l2 = [], []
    with np.errstate(all="ignore"):
        for c in MUTANT_CASES:
            X, Y, ref, slack = references(c)
            got = we.emulate(X, Y, c[4], mutant)
            res = we.check(got, ref, slack, c[4])
            if not res["ok"]:
                rejected.append(we.case_id(c))
            l2.append(max(we.plane_l2(got, ref)))
    l2_accepts = [we.case_id(c) for c, e in zip(MUTANT_CASES, l2) if e <= L2_BAR]
    record("wiener_elements_mutant_" + mutant, rejected_by_bound=rejected, max_plane_l2=l2, accepted_by_l2_bar=l2_accepts)
    print("%s: the bound rejects it on %d of %d cases, the per-plane L2 <= 1e-5 bar accepts it on %d (worst plane L2 per "
          "case %s)" % (mutant, len(rejected), len(MUTANT_CASES), len(l2_accepts), ", ".join("%.1e" % e for e in l2)))
    assert rejected, mutant


def test_cases_have_their_features():
    nx, nsrc, T, F, radius = c = (4, 3, 300, 129, 1)
    X, Y = we.make_case(c)
    f = np.arange(F)
    tiny = np.abs(Y[(Y != 0)])
    assert tiny.min() < 2.0 ** -126 and np.abs(X).max() > 9e3                # fp32 subnormals up to ~1e4
    assert not Y[0][..., f % 8 == 1].any() and Y[1][..., f % 8 == 1].any()   # a source silent over whole bins
    assert not X[..., f % 8 == 2].any() and Y[..., f % 8 == 2].any()         # x = 0, the stems not
    assert np.array_equal(X[:, :, f % 8 == 3], np.repeat(X[:1, :, f % 8 == 3], nx, axis=0))   # equal channels
    assert not Y[nsrc - 1, :, 128:256].any() and Y[nsrc - 1, :, :128].any()  # a source silent for a whole chunk
    assert not Y[:, :, 17].any() and not Y[:, :, 267].any() and Y[:, :, T - 1].any()   # all-stem-zero frames
    loud = np.abs(Y[0][..., f % 8 == 4]).mean() / np.abs(Y[1][..., f % 8 == 4]).mean()
    assert loud > 300                                                       # one source 60 dB up
    s = we.wco._scales(X, radius)
    assert s[0] == 1.0 and s[1] > 1.0 and s[2] > 1.0                        # a window with s = 1 next to s > 1
    assert np.array_equal(X.astype(np.complex64).astype(np.complex128), X)  # fp32 values
    assert np.array_equal(Y.astype(np.complex64).astype(np.complex128), Y)
