"""GPU parity off the reference geometry: every network family at other time contexts, overlaps and (frame size,
hop) pairs, against the float64 oracle.

The library accepts time_context 4..64 and any overlap in [0, time_context); the layer shapes (conv2 taps, h2, the
K of conv2 / bottleneck / transposed conv2, the K clipping of the transposed conv2, the decoder scatter and the G
layout) all follow from time_context, and the number of patches covering a frame, ceil(tc / (tc - overlap)), picks
the DSD mask kernel: 1..6 on the tensor cores (dsd_tc.cu), 7 or more on the FFMA kernel (dsd.cu).  Each case names
the branch it exists for.  Comparison rule as everywhere (tests/parity.py): 1e-4 relative L2 per stem, the bins the
oracle flags on the soft mask's discontinuity taken out bin by bin; the max-pool net's routing via its tie bits."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from oracle import dsp, nets, pipeline  # noqa: E402
from parity import strict_check  # noqa: E402
from channels_oracle import separate_channels  # noqa: E402


def slots(tc, overlap):
    """patches covering one frame: what selects the DSD mask kernel"""
    return -(-tc // (tc - overlap))


def assert_energy(want, mix):
    """the synthetic weights must exercise every stem (no constant or vanishing mask)"""
    for s in range(want.shape[0]):
        assert np.linalg.norm(want[s]) > 0.02 * np.linalg.norm(mix), (s, np.linalg.norm(want[s]), np.linalg.norm(mix))


def stereo_clip(seconds, seed):
    """two different channels (float32-representable, as the device sees them)"""
    mix, _ = pipeline.synth_mixture(seconds, seed)
    other, _ = pipeline.synth_mixture(seconds, seed + 1)
    a = np.stack([0.7 * mix + 0.3 * other, 0.4 * mix + 0.6 * np.roll(other, 11)], axis=1)
    return a.astype(np.float32).astype(np.float64)


def score_filters(T, F, seed=4):
    """synthetic score filters with the structure filterSpec produces: 1 on note bins, 1e-18 elsewhere, normalised"""
    rng = np.random.default_rng(seed)
    raw = np.full((4, T, F), 1e-18, dtype=np.float32)
    for j in range(4):
        for _ in range(6):
            t0, b0 = rng.integers(0, T - 40), rng.integers(1, F - 12)
            raw[j, t0:t0 + 40, b0:b0 + 8] = 1.0
    return (raw / raw.sum(axis=0)).astype(np.float32)


# ------------------------------------------------------------------------------------------------ DSD100 net (mono)
# (N, hop, time_context, overlap, patcher, clip samples, id naming the branch)
DSD_CASES = [
    (1024, 512, 30, 0, "util", 66150, "ov0_1slot_no_crossfade"),
    (1024, 512, 30, 1, "standalone", 66150, "ov1_zero_weight_fade_frame"),
    (1024, 512, 30, 22, "standalone", 66150, "4slots_wgmma_standalone"),
    (1024, 512, 30, 22, "util", 66150, "4slots_wgmma_util"),
    (1024, 512, 30, 24, "standalone", 66150, "5slots_wgmma_standalone"),
    (1024, 512, 30, 24, "util", 66150, "5slots_wgmma_util"),
    (1024, 512, 30, 26, "standalone", 66150, "8slots_ffma"),
    (1024, 512, 30, 29, "standalone", 44100, "30slots_ffma_chunk_loop"),
    (1024, 512, 31, 25, "util", 66150, "odd_tc31_6slots_wgmma"),
    (1024, 512, 31, 26, "util", 66150, "odd_tc31_7slots_ffma_switch"),
    (1024, 512, 4, 2, "standalone", 44100, "min_tc4_2slots_standalone"),
    (1024, 512, 4, 2, "util", 44100, "min_tc4_2slots_util"),
    (1024, 512, 4, 3, "standalone", 44100, "min_tc4_4slots_standalone"),
    (1024, 512, 4, 3, "util", 44100, "min_tc4_4slots_util"),
    (1024, 512, 64, 53, "standalone", 110250, "max_tc64_6slots_wgmma"),
    (1024, 512, 64, 54, "standalone", 110250, "max_tc64_7slots_ffma"),
    (1024, 512, 64, 54, "standalone", 32000, "max_tc64_T65_one_patch"),
    (2048, 256, 17, 13, "util", 52920, "istft_reg32x4_odd_tc17_5slots"),
    (2048, 1024, 20, 10, "standalone", 88200, "smem_istft_complex_N2048_H1024"),
    (4096, 1024, 30, 25, "standalone", 66150, "F2049_17_mask_tiles"),
]


@pytest.mark.parametrize("N,hop,tc,overlap,patcher,L", [c[:6] for c in DSD_CASES], ids=[c[6] for c in DSD_CASES])
def test_dsd_geometry(N, hop, tc, overlap, patcher, L):
    from deepconvsep_b200.engine import Separator
    F = N // 2 + 1
    seed = 7 * tc + overlap + N
    params = nets.make_synthetic_params("dsd", F, tc=tc, seed=seed)
    mix, _ = pipeline.synth_mixture(L / 44100.0, 100 + seed)
    assert mix.size == L
    sep = Separator(params, frame_size=N, hop=hop, window="hanning", time_context=tc, overlap=overlap, patcher=patcher)
    assert sep.model.tc == tc
    want, mag, ph, mm = pipeline.separate(mix, params, "dsd", frameSize=N, hopSize=hop, window=np.hanning, time_context=tc,
                                          overlap=overlap, patcher=patcher, count_kinks=True, return_spec=True)
    kmap = pipeline.separate.last_kink_map
    got, S = sep.separate_tapped(mix)
    assert got.shape == want.shape and got.dtype == np.float32
    assert_energy(want, mix)
    T = dsp.num_frames(L, hop)
    if L == 32000:                   # T = 65 at time_context 64: exactly one patch, the last frame gets no mask
        assert T == 65 and sep.num_patches(T) == 1 and np.all(S[:, 64] == 0)
    assert sep.num_patches(T) >= 1
    strict_check("geom_dsd_N%d_H%d_tc%d_ov%d_%s_L%d" % (N, hop, tc, overlap, patcher, L), got, S, want, mag, ph, mm, kmap,
                 N, hop, np.hanning, 0.3, extra={"slots": slots(tc, overlap)})


# ------------------------------------------------------------------------------------------------ stereo / ILD net
ILD_CASES = [(31, 25, "odd_tc31_6slots_wgmma"), (16, 12, "tc16_4slots_wgmma"), (30, 27, "10slots_ffma_4decoders")]


@pytest.mark.parametrize("tc,overlap", [c[:2] for c in ILD_CASES], ids=[c[2] for c in ILD_CASES])
def test_ild_geometry(tc, overlap):
    from deepconvsep_b200.engine import Separator
    N, hop, F = 1024, 512, 513
    params = nets.make_synthetic_params("dsd_ild", F, tc=tc, seed=40 + tc + overlap)
    sep = Separator(params, frame_size=N, hop=hop, window="hanning", time_context=tc, overlap=overlap, patcher="util")
    assert sep.model.arch == "dsd_ild" and sep.model.tc == tc
    audio = stereo_clip(1.5, 600 + tc)
    want, mag, phs, mms = pipeline.separate_stereo(audio, params, frameSize=N, hopSize=hop, time_context=tc, overlap=overlap,
                                                   count_kinks=True, return_spec=True)
    kmap = pipeline.separate_stereo.last_kink_map
    got, S = sep.separate_tapped(audio)
    assert got.shape == want.shape == (audio.shape[0], 4, 2) and got.dtype == np.float32
    for j in range(2):
        assert_energy(np.ascontiguousarray(want[:, :, j].T), audio[:, j])
        strict_check("geom_ild_tc%d_ov%d_ch%d" % (tc, overlap, j), np.ascontiguousarray(got[:, :, j].T), S[j::2],
                     np.ascontiguousarray(want[:, :, j].T), mag[j], phs[j], mms[j], kmap[j], N, hop, np.hanning, 0.3,
                     extra={"slots": slots(tc, overlap)})


def test_keep_channels_tc23_5slots_nx2_wgmma():
    """keep-channels mode (the downmix's masks from the tensor-core mask kernel, applied to both channels) at
    time_context 23, overlap 18: 5 patches per frame"""
    from deepconvsep_b200.engine import Separator
    N, hop, F, tc, overlap = 1024, 512, 513, 23, 18
    params = nets.make_synthetic_params("dsd", F, tc=tc, seed=123)
    sep = Separator(params, frame_size=N, hop=hop, window="hanning", time_context=tc, overlap=overlap)
    audio = stereo_clip(1.5, 321)
    want, mags, phs, mms, _, kmap = separate_channels(audio, params, frameSize=N, hopSize=hop, time_context=tc,
                                                      overlap=overlap)
    got, S = sep.separate_tapped(audio, keep_channels=True)
    assert got.shape == want.shape == (audio.shape[0], 4, 2) and got.dtype == np.float32
    for c in range(2):
        assert_energy(np.ascontiguousarray(want[:, :, c].T), audio[:, c])
        strict_check("geom_keep_tc%d_ov%d_ch%d" % (tc, overlap, c), np.ascontiguousarray(got[:, :, c].T), S[c::2],
                     np.ascontiguousarray(want[:, :, c].T), mags[c], phs[c], mms[c], kmap, N, hop, np.hanning, 0.3,
                     extra={"slots": slots(tc, overlap)})


# ------------------------------------------------------------------------------------------------ 30-channel nets
# (arch, F, N, hop, window, tc, overlap, patcher, seconds, silence, weight seed, id)
SCONV_CASES = [
    ("bach10", 257, 512, 256, "blackmanharris", 24, 20, "util", 1.5, None, 92, "bach10_tc24_kh2_16"),
    ("bach10", 257, 512, 256, "blackmanharris", 31, 28, "standalone", 1.5, None, 121, "bach10_tc31_kh2_20_11slots"),
    ("bach10", 257, 512, 256, "blackmanharris", 30, 0, "util", 1.5, None, 90, "bach10_ov0_1slot"),
    ("bach10", 257, 512, 256, "blackmanharris", 30, 1, "standalone", 1.5, None, 91, "bach10_ov1_zero_weight_fade_frame"),
    ("ikala", 513, 1024, 512, "hanning", 16, 12, "standalone", 2.0, (20000, 40000), 60, "ikala_pool_tc16_h2_7"),
    ("ikala", 513, 1024, 512, "hanning", 40, 39, "standalone", 2.0, (20000, 40000), 160, "ikala_pool_tc40_40slots"),
    ("ikala_nopool", 513, 1024, 512, "hanning", 12, 0, "util", 1.5, None, 36, "ikala_nopool_tc12_h2_3_1slot"),
]


@pytest.mark.parametrize("arch,F,N,hop,win,tc,overlap,patcher,seconds,silence,seed", [c[:11] for c in SCONV_CASES],
                         ids=[c[11] for c in SCONV_CASES])
def test_sconv_geometry(arch, F, N, hop, win, tc, overlap, patcher, seconds, silence, seed):
    """the 30-channel nets: models.infer_arch assumes time_context 30 for them, so it is passed explicitly"""
    from deepconvsep_b200.engine import Separator
    win_fn = dsp.blackmanharris if win == "blackmanharris" else np.hanning
    params = nets.make_synthetic_params(arch, F, tc=tc, seed=seed)
    mix, _ = pipeline.synth_mixture(seconds, 70 + F + tc)
    if silence:
        mix[silence[0]:silence[1]] = 0.0      # exact zeros: constant conv1 output -> max-pool ties everywhere
    sep = Separator(params, arch=arch, frame_size=N, hop=hop, window=win, time_context=tc, overlap=overlap, patcher=patcher,
                    feat_size=F)
    assert sep.model.tc == tc
    kw = dict(frameSize=N, hopSize=hop, window=win_fn, time_context=tc, overlap=overlap, patcher=patcher, count_kinks=True,
              return_spec=True)
    extra = {"slots": slots(tc, overlap)}
    if arch == "ikala":
        got, S, bits = sep.separate_tapped(mix, pool=True)
        want, mag, ph, mm = pipeline.separate(mix, params, arch, pool_bits=bits, **kw)
        st = pipeline.separate.last_pool_stats
        assert st["disagree_well_conditioned"] == 0 and st["inadmissible"] == 0, st
        assert st["ambiguous"] <= 0.01 * st["windows"], st
        extra.update(pool_windows=st["windows"], pool_windows_ill_conditioned=st["ambiguous"])
    else:
        got, S = sep.separate_tapped(mix)
        want, mag, ph, mm = pipeline.separate(mix, params, arch, **kw)
    kmap = pipeline.separate.last_kink_map
    assert got.shape == want.shape
    assert_energy(want, mix)
    strict_check("geom_%s_tc%d_ov%d_%s" % (arch, tc, overlap, patcher), got, S, want, mag, ph, mm, kmap, N, hop, win_fn, 0.3,
                 extra=extra)


def test_score_informed_tc21_kh2_14():
    """the 4-channel score-conditioned net at time_context 21 (conv2 taps int(2 * 21 / 3) = 14), overlap 17"""
    from deepconvsep_b200.engine import Separator
    F, N, hop, tc, overlap = 129, 256, 128, 21, 17
    params = nets.make_synthetic_params("bach10_score", F, tc=tc, seed=21)
    assert params[3].shape == (30, 30, 14, 1)
    mix, _ = pipeline.synth_mixture(1.0, 92)
    filters = score_filters(dsp.num_frames(mix.size, hop), F)
    want, mag, ph, mm = pipeline.separate_score(mix, filters, params, frameSize=N, hopSize=hop, window=dsp.blackmanharris,
                                                scale_factor=0.2, time_context=tc, overlap=overlap, count_kinks=True,
                                                return_spec=True)
    kmap = pipeline.separate_score.last_kink_map
    sep = Separator(params, arch="bach10_score", frame_size=N, hop=hop, window="blackmanharris", time_context=tc,
                    overlap=overlap, patcher="util", scale_factor=0.2, feat_size=F)
    got, S = sep.separate_tapped(mix, filters)
    assert got.shape == want.shape == (4, mix.size)
    assert_energy(want, mix)
    strict_check("geom_bach10_score_tc%d_ov%d" % (tc, overlap), got, S, want, mag, ph, mm, kmap, N, hop, dsp.blackmanharris,
                 0.2, extra={"slots": slots(tc, overlap)})
