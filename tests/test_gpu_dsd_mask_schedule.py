"""Edges of the persistent schedule of the wgmma mask + cross-fade kernel (dsd_tc.cu), checked against its
exact-fp32 FFMA twin (dsd.cu, selected by DCS_DEBUG_SIMT_GEMM=1, read when a context is created; every other layer
stays on the tensor cores):

- DSD100 at N=2048 on a 0.5 s clip: fewer (tile, group) work items than SMs, and a last group of 8 frames that is
  only partly inside the clip;
- the stereo / ILD net at N=2048: the 4-decoder register mapping together with the tile that holds only the
  Nyquist bin (F = 1025)."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from oracle import nets, pipeline  # noqa: E402
from parity import TOL  # noqa: E402


def rel(a, b):
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


@pytest.mark.parametrize("arch,N,seconds", [("dsd", 2048, 0.5), ("dsd_ild", 2048, 3.0)])
def test_mask_schedule_edges_match_ffma_twin(monkeypatch, arch, N, seconds):
    from deepconvsep_b200.engine import Separator
    F = N // 2 + 1
    params = nets.make_synthetic_params(arch, F, seed=2)
    if arch == "dsd":
        audio, _ = pipeline.synth_mixture(seconds, 1001)
    else:
        rng = np.random.default_rng(5)
        mono, _ = pipeline.synth_mixture(seconds, 1002)
        audio = np.stack([mono, 0.6 * mono + 0.05 * rng.standard_normal(mono.size)], axis=1).astype(np.float32)
    outs = []
    for simt in ("0", "1"):
        monkeypatch.setenv("DCS_DEBUG_SIMT_GEMM", simt)
        sep = Separator(params, frame_size=N, hop=512, window="hanning", overlap=25, device=0)
        got, _ = sep.separate_tapped(audio)
        outs.append(np.asarray(got, dtype=np.float64))
    tc, ffma = outs
    assert np.isfinite(tc).all() and tc.shape == ffma.shape
    stems = tc if arch == "dsd" else tc.reshape(tc.shape[0], -1).T    # (source, channel) planes of the stereo net
    ref = ffma if arch == "dsd" else ffma.reshape(ffma.shape[0], -1).T
    for s in range(stems.shape[0]):
        assert np.linalg.norm(ref[s]) > 0
        assert rel(stems[s], ref[s]) <= TOL, (s, rel(stems[s], ref[s]))
