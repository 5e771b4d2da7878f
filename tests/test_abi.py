"""CPU-side checks of the boundary: the C-ABI library loads and exports every symbol that
include/dcs.h declares; the pure host helpers agree with the oracle.  No compute calls."""
import os
import re
import pickle
import numpy as np
import pytest

from deepconvsep_b200 import _lib, models
from oracle import dsp, patch, nets

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build():
    from deepconvsep_b200 import build
    build.build()


def test_library_exports_every_declared_symbol():
    _build()
    hdr = open(os.path.join(ROOT, "include", "dcs.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = sorted(set(re.findall(r"\b(dcs_[a-z0-9_]+)\s*\(", hdr)))
    assert len(declared) >= 20
    lib = _lib.load()
    for name in declared:
        assert hasattr(lib, name), "libdcs.so does not export %s" % name
    assert sorted(declared) == _lib.exported_symbols()
    assert lib.dcs_version() == 101


def test_no_cpu_fallback():
    """Without a CUDA device the product path must fail loudly."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from deepconvsep_b200.engine import Context
    with pytest.raises(_lib.DcsError):
        Context(0)


def test_frame_and_patch_counts_match_oracle():
    _build()
    lib = _lib.load()
    for L in (1, 511, 512, 513, 5000, 7938000):
        for hop in (256, 512):
            assert lib.dcs_num_frames(L, hop) == dsp.num_frames(L, hop)
    for T in range(1, 200):
        for tc, ov in ((30, 25), (30, 20), (30, 0), (20, 15)):
            assert lib.dcs_num_patches(T, tc, ov, 0) == patch.num_patches(T, tc, ov, "standalone")
            assert lib.dcs_num_patches(T, tc, ov, 1) == patch.num_patches(T, tc, ov, "util")
    assert lib.dcs_num_patches(15506, 30, 25, 0) == 3096      # SURVEY.md section 8
    assert lib.dcs_num_patches(15506, 30, 25, 1) == 3097
    assert lib.dcs_padded_bins(1024) == 520 and lib.dcs_padded_bins(2048) == 1032


def test_product_package_does_not_import_oracle():
    pkg = os.path.join(ROOT, "deepconvsep_b200")
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dp, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, re.M), f
                assert "from oracle" not in src and "import oracle" not in src, f


def test_load_model_roundtrip_and_arch_inference(tmp_path):
    for arch, F in (("dsd", 513), ("dsd", 1025), ("ikala", 513), ("bach10", 129)):
        params = nets.make_synthetic_params(arch, F, seed=3)
        fn = str(tmp_path / (arch + ".pkl"))
        models.save_model(fn, params)
        back = models.load_model(fn)
        assert len(back) == len(params)
        for a, b in zip(params, back):
            np.testing.assert_array_equal(a, b)
        got = models.infer_arch(back, feat_size=F if arch != "dsd" else None)
        assert got == (arch, F, 30)
        if F in (513, 1025, 2049):
            assert got[:2] == nets.infer_arch(back)[:2]
    # a Python-2 style pickle (protocol 2, str payloads) loads through the latin1 path
    fn = str(tmp_path / "p2.pkl")
    with open(fn, "wb") as f:
        pickle.dump([np.arange(4, dtype=np.float32)], f, protocol=2)
    assert models.load_model(fn)[0].tolist() == [0, 1, 2, 3]


@pytest.mark.parametrize("arch", ["dsd", "dsd_ild"])
@pytest.mark.parametrize("tc", [4, 17, 31, 64])
def test_models_infer_arch_recovers_time_context(arch, tc):
    """the DSD nets' time_context from the conv2 / fc.W shapes, odd values and both ends of the accepted 4..64"""
    params = [np.zeros(s, dtype=np.float32) for s in nets.param_shapes(arch, 513, tc)]
    assert models.infer_arch(params) == (arch, 513, tc)
    assert nets.infer_arch(params) == (arch, 513, tc)
