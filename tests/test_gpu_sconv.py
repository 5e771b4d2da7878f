"""GPU parity of the strided-conv1 networks -- Bach10 (examples/bach10/separate_bach10.py) and iKala
(examples/ikala/separate_ikala.py, pooled; ikala/trainCNN.py, un-pooled) -- against the float64 oracle.
Same comparison rule as tests/test_gpu_dsd.py (tests/parity.py): plain 1e-4 relative L2 per stem, the
few bins the oracle flags on the mask discontinuity taken out bin by bin, no whole-stem allowance."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from oracle import dsp, nets, pipeline  # noqa: E402
from parity import strict_check, TOL  # noqa: E402


def rel(a, b):
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def run_case(arch, F, N, hop, win_name, win_fn, overlap, seconds, patcher="standalone", seed=5, silence=None):
    from deepconvsep_b200.engine import Separator
    params = nets.make_synthetic_params(arch, F, seed=seed)
    mix, _ = pipeline.synth_mixture(seconds, 70 + F)
    if silence:
        mix[silence[0]:silence[1]] = 0.0      # exact zeros: constant conv1 output -> max-pool ties everywhere
    sep = Separator(params, arch=arch, frame_size=N, hop=hop, window=win_name, overlap=overlap, patcher=patcher,
                    feat_size=F)
    extra = None
    if arch == "ikala":
        # the un-pool routing (argmax of each max-pool window) is a discrete decision of the reference's graph:
        # where float64 flags a window as ill-conditioned the oracle adopts the device's choice (checked to be
        # among the near-maximal positions), everywhere else the device must agree (oracle.nets.maxpool_w_inverse)
        got, S, bits = sep.separate_tapped(mix, pool=True)
        want, mag, ph, mm = pipeline.separate(mix, params, arch, frameSize=N, hopSize=hop, window=win_fn, overlap=overlap,
                                              patcher=patcher, count_kinks=True, return_spec=True, pool_bits=bits)
        st = pipeline.separate.last_pool_stats
        assert st["disagree_well_conditioned"] == 0 and st["inadmissible"] == 0, st
        assert st["ambiguous"] <= 0.01 * st["windows"], st
        extra = {"pool_windows": st["windows"], "pool_windows_ill_conditioned": st["ambiguous"]}
    else:
        got, S = sep.separate_tapped(mix)
        want, mag, ph, mm = pipeline.separate(mix, params, arch, frameSize=N, hopSize=hop, window=win_fn, overlap=overlap,
                                              patcher=patcher, count_kinks=True, return_spec=True)
    kmap = pipeline.separate.last_kink_map
    assert got.shape == want.shape
    assert min(np.linalg.norm(w) for w in want) > 0.02 * np.linalg.norm(mix)
    strict_check("%s_N%d_%gs_%s%s" % (arch, N, seconds, patcher, "_silence" if silence else ""), got, S, want, mag, ph, mm,
                 kmap, N, hop, win_fn, 0.3, extra=extra)
    return sep


@pytest.mark.parametrize("F,N,hop,seconds,patcher", [(129, 256, 128, 1.0, "standalone"), (257, 512, 256, 1.5, "util"),
                                                     (129, 256, 128, 0.4, "util")])
def test_bach10_small(F, N, hop, seconds, patcher):
    run_case("bach10", F, N, hop, "blackmanharris", dsp.blackmanharris, 25, seconds, patcher)


def test_ikala_pooled_with_silence():
    sep = run_case("ikala", 513, 1024, 512, "hanning", np.hanning, 20, 3.0, silence=(20000, 40000))
    assert sep.nsrc == 2 and sep.sources == ["voice", "music"]


def test_ikala_nopool():
    run_case("ikala_nopool", 513, 1024, 512, "hanning", np.hanning, 20, 1.2, seed=9)


def test_bach10_full_size():
    """The real configuration: N=4096, F=2049, 214 M parameters (856 MB), one second of audio."""
    run_case("bach10", 2049, 4096, 512, "blackmanharris", dsp.blackmanharris, 25, 1.0, seed=2)


def test_models_share_a_context_safely():
    """DSD100 and Bach10 alternating on ONE ctx, at two time contexts and three overlaps of the DSD100 net and two
    overlaps of Bach10: the zero-padded workspaces are re-zeroed when the layout changes (the layout signature leaves
    the overlap out for the DSD nets), so every call gives the bits of its first round."""
    from deepconvsep_b200.engine import Context, Model, Stft
    from deepconvsep_b200 import _lib
    import ctypes as C
    ctx = Context(0)
    lib = ctx.lib
    mix, _ = pipeline.synth_mixture(1.0, 3)
    outs = {}
    for rnd in range(2):
        for arch, F, N, hop, win, tc, ov in (("dsd", 257, 512, 256, np.hanning, 30, 25),
                                             ("dsd", 257, 512, 256, np.hanning, 30, 0),
                                             ("dsd", 257, 512, 256, np.hanning, 31, 26),
                                             ("bach10", 257, 512, 256, dsp.blackmanharris, 30, 25),
                                             ("bach10", 257, 512, 256, dsp.blackmanharris, 30, 28)):
            params = nets.make_synthetic_params(arch, F, tc=tc, seed=4)
            model = Model(ctx, params, arch=arch, feat_size=F, time_context=tc)
            st = Stft(ctx, N, hop, win(N))
            a = np.ascontiguousarray(mix, dtype=np.float32)
            out = np.empty((4, a.size), dtype=np.float32)
            _lib.check(lib.dcs_separate_host(ctx.handle, model.handle, st.handle, a.ctypes.data, a.size, C.c_float(0.3), ov, 0,
                                             out.ctypes.data, a.size, None))
            if rnd == 0:
                outs[arch, tc, ov] = out
                want = pipeline.separate(mix, params, arch, frameSize=N, hopSize=hop, window=win, time_context=tc, overlap=ov)
                assert max(rel(out[s].astype(np.float64), want[s]) for s in range(4)) < 5e-4, (arch, tc, ov)
            else:
                assert np.array_equal(out, outs[arch, tc, ov]), (arch, tc, ov)


def test_score_informed_bach10():
    """4-channel score-conditioned network (trainCNNrwc.py:134-263): only decoder 1 is live, the four
    sources are the four input-channel filter banks of the tied conv1; util patcher, scale 0.2."""
    from deepconvsep_b200.engine import Separator
    F, N, hop = 129, 256, 128
    params = nets.make_synthetic_params("bach10_score", F, seed=8)
    assert len(params) == 17 and params[0].shape == (30, 4, 1, 30) and params[-1].shape == (16,)
    mix, _ = pipeline.synth_mixture(1.0, 91)
    T = dsp.num_frames(mix.size, hop)
    rng = np.random.default_rng(4)
    # synthetic "score" filters with the structure filterSpec produces: 1 on note bins, 1e-18 elsewhere, normalised
    raw = np.full((4, T, F), 1e-18, dtype=np.float32)
    for j in range(4):
        for _ in range(6):
            t0, b0 = rng.integers(0, T - 40), rng.integers(1, F - 12)
            raw[j, t0:t0 + 40, b0:b0 + 8] = 1.0
    filters = (raw / raw.sum(axis=0)).astype(np.float32)
    want, mag, ph, mm = pipeline.separate_score(mix, filters, params, frameSize=N, hopSize=hop, window=dsp.blackmanharris,
                                                scale_factor=0.2, overlap=25, count_kinks=True, return_spec=True)
    kmap = pipeline.separate_score.last_kink_map
    sep = Separator(params, arch="bach10_score", frame_size=N, hop=hop, window="blackmanharris", overlap=25,
                    patcher="util", scale_factor=0.2, feat_size=F)
    got, S = sep.separate_tapped(mix, filters)
    assert got.shape == want.shape == (4, mix.size)
    assert min(np.linalg.norm(w) for w in want) > 0.02 * np.linalg.norm(mix)
    strict_check("bach10_score_N%d_1s" % N, got, S, want, mag, ph, mm, kmap, N, hop, dsp.blackmanharris, 0.2)
    with pytest.raises(Exception):
        sep.separate(mix)          # the single-channel entry point must refuse this architecture


def test_separate_spec_channels_matches_audio_score():
    """dcs_separate_spec_channels on the four channel planes (score filter x scaled magnitude) and the mixture STFT of a
    clip gives the masked spectra dcs_separate_audio_score records for the same clip, bit for bit."""
    from deepconvsep_b200.engine import Separator, _ptr
    from deepconvsep_b200._lib import check
    F, N, hop = 129, 256, 128
    params = nets.make_synthetic_params("bach10_score", F, seed=8)
    mix, _ = pipeline.synth_mixture(1.0, 91)
    T = dsp.num_frames(mix.size, hop)
    rng = np.random.default_rng(4)
    raw = np.full((4, T, F), 1e-18, dtype=np.float32)
    for j in range(4):
        for _ in range(6):
            t0, b0 = rng.integers(0, T - 40), rng.integers(1, F - 12)
            raw[j, t0:t0 + 40, b0:b0 + 8] = 1.0
    filters = (raw / raw.sum(axis=0)).astype(np.float32)
    sep = Separator(params, arch="bach10_score", frame_size=N, hop=hop, window="blackmanharris", overlap=25,
                    patcher="util", scale_factor=0.2, feat_size=F)
    _, tapped = sep.separate_tapped(mix, filters)
    dev, ldf = sep.stft.dev, sep.stft.ldf
    X, mag = sep.stft.forward(torch.as_tensor(mix.astype(np.float32), device=dev), mag_scale=0.2)
    fd = torch.zeros((4, T, ldf), dtype=torch.float32, device=dev)
    fd[:, :, :F] = torch.as_tensor(filters, device=dev)
    chans = (fd * mag).contiguous()
    S = torch.empty((4, T, ldf), dtype=torch.complex64, device=dev)
    check(sep.lib.dcs_separate_spec_channels(sep.ctx.handle, sep.model.handle, _ptr(chans), T * ldf, _ptr(X), T, ldf,
                                             sep.overlap, sep.patcher, _ptr(S), T * ldf, None))
    torch.cuda.synchronize(dev)
    got = S[:, :, :F].cpu().numpy()
    assert np.abs(tapped).max() > 0 and np.array_equal(got, tapped)


@pytest.mark.parametrize("arch,F,N,hop,win,overlap,seconds", [("bach10", 257, 512, 256, "blackmanharris", 25, 1.5),
                                                              ("bach10_score", 129, 256, 128, "blackmanharris", 25, 1.0),
                                                              ("ikala", 513, 1024, 512, "hanning", 20, 3.0),
                                                              ("ikala_nopool", 513, 1024, 512, "hanning", 20, 3.0)])
def test_tensor_core_mask_matches_ffma_twin(monkeypatch, arch, F, N, hop, win, overlap, seconds):
    """the wgmma K3s kernel (sconv_tc.cu) against its exact-fp32 FFMA twin (sconv.cu, selected by
    DCS_DEBUG_SIMT_GEMM=1, read when a context is created): same stems within the parity bar"""
    from deepconvsep_b200.engine import Separator
    params = nets.make_synthetic_params(arch, F, seed=5)
    mix, _ = pipeline.synth_mixture(seconds, 70 + F)
    filters = None
    patcher = "standalone"
    if arch == "bach10_score":
        T = dsp.num_frames(mix.size, hop)
        rng = np.random.default_rng(4)
        raw = np.full((4, T, F), 1e-18, dtype=np.float32)
        for j in range(4):
            for _ in range(6):
                t0, b0 = rng.integers(0, T - 40), rng.integers(1, F - 12)
                raw[j, t0:t0 + 40, b0:b0 + 8] = 1.0
        filters = (raw / raw.sum(axis=0)).astype(np.float32)
        patcher = "util"
    outs = []
    for simt in ("0", "1"):
        monkeypatch.setenv("DCS_DEBUG_SIMT_GEMM", simt)
        sep = Separator(params, arch=arch, frame_size=N, hop=hop, window=win, overlap=overlap, patcher=patcher,
                        scale_factor=0.2 if filters is not None else 0.3, feat_size=F)
        got, _ = sep.separate_tapped(mix, filters) if filters is not None else sep.separate_tapped(mix)
        outs.append(np.asarray(got, dtype=np.float64))
    tc, ffma = outs
    assert np.isfinite(tc).all() and tc.shape == ffma.shape
    for s in range(tc.shape[0]):
        assert np.linalg.norm(ffma[s]) > 0
        assert rel(tc[s], ffma[s]) <= TOL, (s, rel(tc[s], ffma[s]))
