"""Host tests of the masks output: the float64 blended masks of tests/masks_oracle.py against the separation oracles
(oracle.pipeline, score1x1_oracle) -- masks times the network's mixture must give their blended masked magnitudes mm
to 1e-12 of the mixture for every family -- their range, and the argument rules of Separator.separate_masks that are
decided before anything reaches the library."""
from types import SimpleNamespace

import numpy as np
import pytest

from oracle import dsp, nets, pipeline
import masks_oracle as mo
import score1x1_oracle as s1


def score_filters(T, F, seed=4):
    rng = np.random.default_rng(seed)
    raw = np.full((4, T, F), 1e-18, dtype=np.float32)
    for j in range(4):
        for _ in range(6 + T // 40):
            t0, b0 = rng.integers(0, max(1, T - 40)), rng.integers(1, F - 24)
            raw[j, t0:t0 + 40, b0:b0 + F // 8] = 1.0
    return (raw / raw.sum(axis=0)).astype(np.float32)


def check(masks, mix, mm_pipe, mm):
    """masks * mix == the pipeline's mm to 1e-12 of the mixture where it is non-zero; masks in [0, 1]"""
    T = masks.shape[-2]
    mm_pipe = np.asarray(mm_pipe)[..., :T, :]
    assert mm_pipe.shape == masks.shape == mm.shape
    assert np.all(np.isfinite(masks)) and masks.min() >= 0 and masks.max() <= 1 + 1e-12
    pos = np.broadcast_to(mix > 0, masks.shape)
    d = np.abs(masks * mix - mm_pipe)
    assert pos.sum() > 0.5 * pos.size
    assert np.all(d[pos] <= 1e-12 * np.broadcast_to(mix, masks.shape)[pos]), float(d[pos].max())
    assert np.all(np.abs(mm - mm_pipe) <= 1e-12 * np.abs(mm_pipe).max())
    assert masks.std() > 0.01      # the masks vary: the comparison exercises something


@pytest.mark.parametrize("arch,F,N,win,patcher,overlap", [
    ("dsd", 513, 1024, np.hanning, "standalone", 25), ("dsd", 513, 1024, np.hanning, "util", 25),
    ("ikala", 513, 1024, np.hanning, "standalone", 20), ("ikala_nopool", 513, 1024, np.hanning, "util", 20),
    ("bach10", 129, 256, dsp.blackmanharris, "standalone", 25)])
def test_single_channel_nets(arch, F, N, win, patcher, overlap):
    params = nets.make_synthetic_params(arch, F, seed=3)
    mix, _ = pipeline.synth_mixture(1.0, 17 + F)
    mix[8000:20000] = 0.0                         # a silent segment: |X| = 0 there
    hop = N // 2
    masks, mag, mm, kmap = mo.separate_masks(mix, params, arch, frameSize=N, hopSize=hop, window=win, overlap=overlap,
                                             patcher=patcher)
    _, mag_p, _, mm_p = pipeline.separate(mix, params, arch, frameSize=N, hopSize=hop, window=win, overlap=overlap,
                                          patcher=patcher, return_spec=True)
    assert np.array_equal(mag, mag_p)
    check(masks, mag, mm_p, mm)
    assert kmap.shape == mag.shape
    silent = mag.max(axis=1) == 0
    assert silent.sum() >= 10
    # where |X| = 0 the masks are still defined: the all-zero rule gives 1/nsrc for the DSD and iKala nets
    covered = masks.sum(axis=0) > 0
    if arch != "bach10":
        assert np.allclose(masks[:, silent & covered.any(axis=1)].sum(axis=0), 1.0)


def test_score_informed_build_ca():
    F, N = 129, 256
    params = nets.make_synthetic_params("bach10_score", F, seed=8)
    mix, _ = pipeline.synth_mixture(1.0, 5)
    T = dsp.num_frames(mix.size, N // 2)
    filters = score_filters(T, F)
    masks, chsum, mm, _ = mo.separate_score_masks(mix, filters, params, frameSize=N, hopSize=N // 2)
    mm_p = pipeline.separate_score(mix, filters, params, frameSize=N, hopSize=N // 2, return_spec=True)[3]
    check(masks, chsum, mm_p, mm)


def test_score_informed_build_ca_1x1():
    N = 512
    params = s1.make_synthetic_params_1x1(seed=7)
    mix, _ = pipeline.synth_mixture(1.0, 91)
    T = dsp.num_frames(mix.size, N // 2)
    filters = score_filters(T, N // 2 + 1)
    masks, chsum, mm, _ = mo.separate_score_1x1_masks(mix, filters, params, frameSize=N, hopSize=N // 2)
    mm_p = s1.separate_score_1x1(mix, filters, params, frameSize=N, hopSize=N // 2, return_spec=True)[3]
    check(masks, chsum, mm_p, mm)


def test_stereo_ild_net():
    F, N = 513, 1024
    params = nets.make_synthetic_params("dsd_ild", F, seed=5)
    a, _ = pipeline.synth_mixture(1.0, 3)
    b, _ = pipeline.synth_mixture(1.0, 4)
    audio = np.stack([a, 0.5 * a + 0.5 * b], axis=1)
    masks, mag, mms, kmaps = mo.separate_stereo_masks(audio, params, frameSize=N, hopSize=512)
    _, mag_p, _, mms_p = pipeline.separate_stereo(audio, params, frameSize=N, hopSize=512, return_spec=True)
    assert masks.shape == (4, 2) + mag.shape[1:] and kmaps.shape == mag.shape
    assert np.array_equal(mag, mag_p)
    check(masks, mag[None], np.stack(mms_p, axis=1), mms)


def test_clip_shorter_than_one_patch_gives_zero_masks():
    params = nets.make_synthetic_params("dsd", 513, seed=1)
    mix, _ = pipeline.synth_mixture(0.2, 2)      # 20 frames < time_context
    masks, mag, mm, _ = mo.separate_masks(mix, params, "dsd")
    assert masks.shape == (4,) + mag.shape and not masks.any() and not mm.any()


@pytest.mark.parametrize("arch,kw,msg", [
    ("dsd", {"melody": np.zeros((4, 1, 3))}, "separate_notes needs a score-informed network"),
    ("dsd_ild", {"filters": np.zeros((4, 1, 3))}, "separate_score needs a score-informed network"),
    ("bach10_score", {}, "needs either the score filters or the note table"),
    ("bach10_score_1x1", {"filters": np.zeros((4, 1, 3)), "melody": np.zeros((4, 1, 3))}, "needs either"),
    ("bach10_score", {"melody": np.zeros((4, 1, 3)), "frame0": -1}, "frame0 -1 must be >= 0")])
def test_separate_masks_refuses_wrong_family_inputs(arch, kw, msg):
    pytest.importorskip("torch")
    from deepconvsep_b200.engine import Separator
    stand_in = SimpleNamespace(model=SimpleNamespace(arch=arch))
    with pytest.raises(ValueError, match=msg):
        Separator.separate_masks(stand_in, np.zeros(1000, dtype=np.float32), **kw)
