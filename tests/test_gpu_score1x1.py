"""GPU parity of the score-informed build_ca_1x1 network (examples/bach10_scoreinformed/trainCNNrwc.py:66-132) against
the float64 oracle (tests/score1x1_oracle.py) under the strict rule of tests/parity.py: 1e-4 relative L2 per stem, the bins
the oracle flags on the mask discontinuity taken out bin by bin.  The ReLU gate codes of the encoder are discrete
decisions of the graph: the oracle adopts the device's (routing tap) only where near_gate flags the pre-activation,
and the device must agree everywhere else."""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from oracle import dsp, nets, pipeline  # noqa: E402
import score1x1_oracle as s1  # noqa: E402
from parity import strict_check, record, TOL  # noqa: E402

ARCH = "bach10_score_1x1"


def score_filters(T, F, seed=4):
    """synthetic filters with filterSpec's structure: 1 on note bins, 1e-18 elsewhere, normalised over the sources"""
    rng = np.random.default_rng(seed)
    raw = np.full((4, T, F), 1e-18, dtype=np.float32)
    for j in range(4):
        for _ in range(6 + T // 40):
            t0, b0 = rng.integers(0, max(1, T - 40)), rng.integers(1, F - 24)
            raw[j, t0:t0 + 40, b0:b0 + 20] = 1.0
    return (raw / raw.sum(axis=0)).astype(np.float32)


def separator(params, N, hop, overlap, tc, patcher="util"):
    from deepconvsep_b200.engine import Separator
    return Separator(params, arch=ARCH, frame_size=N, hop=hop, window="blackmanharris", overlap=overlap, patcher=patcher,
                     scale_factor=0.2, feat_size=N // 2 + 1, time_context=tc)


def profile_names(sep):
    buf = C.create_string_buffer(1 << 16)
    ms = np.zeros(4096, dtype=np.float32)
    n = sep.lib.dcs_profile_read(sep.ctx.handle, buf, len(buf), ms.ctypes.data, ms.size)
    return buf.value.decode().split("\n")[:n]


def run_case(name, N, hop, overlap, tc, seconds, patcher="util", seed=7, silence=None, zero_bias=False, sep=None,
             params=None, mix_seed=91):
    F = N // 2 + 1
    if params is None:
        params = s1.make_synthetic_params_1x1(seed=seed)
        if zero_bias:
            for l in range(6):
                params[3 * l + 1][:] = 0
                params[3 * l + 2][:] = 0
    mix, _ = pipeline.synth_mixture(seconds, mix_seed)
    if silence:
        mix[silence[0]:silence[1]] = 0.0
    T = dsp.num_frames(mix.size, hop)
    filters = score_filters(T, F)
    sep = sep or separator(params, N, hop, overlap, tc, patcher)
    got, S, codes = sep.separate_tapped(mix, filters, pool=True)
    want, mag, ph, mm = s1.separate_score_1x1(mix, filters, params, frameSize=N, hopSize=hop, scale_factor=0.2,
                                              time_context=tc, overlap=overlap, gate_codes_dev=codes, return_spec=True,
                                              patcher=patcher)
    st = s1.separate_score_1x1.last_gate_stats
    kmap = s1.separate_score_1x1.last_kink_map
    assert st["disagree_unflagged"] == 0, st
    assert st["flagged"] <= 1e-3 * st["positions"], st
    assert got.shape == want.shape == (4, mix.size)
    assert min(np.linalg.norm(w) for w in want) > 0.01 * np.linalg.norm(mix)
    errs = strict_check(name, got, S, want, mag, ph, mm, kmap, N, hop, dsp.blackmanharris, 0.2,
                        extra={"gate_positions": st["positions"], "gate_flagged": st["flagged"],
                               "gate_flagged_fraction": st["flagged"] / st["positions"], "gate_half": st["half"]})
    return sep, got, st, errs


@pytest.mark.parametrize("N,hop,overlap,tc,patcher", [
    (512, 256, 25, 30, "util"), (512, 256, 0, 19, "standalone"), (512, 256, 28, 31, "util"),
    (1024, 512, 25, 30, "standalone"), (1024, 512, 0, 31, "util"), (1024, 256, 28, 30, "standalone"),
    (512, 256, 18, 19, "util")])
def test_score1x1_parity(N, hop, overlap, tc, patcher):
    run_case("score1x1_N%d_h%d_ov%d_tc%d_%s" % (N, hop, overlap, tc, patcher), N, hop, overlap, tc, 1.5, patcher)


def test_score1x1_silence_with_zero_biases():
    """exact zeros in, zero biases: every encoder pre-activation of the silent frames is exactly 0, where Theano's
    rectifier has derivative 0.5 (gate code 1); the device must produce that code there"""
    _, _, st, _ = run_case("score1x1_silence_zero_bias", 512, 256, 25, 30, 1.5, silence=(15000, 45000), zero_bias=True)
    assert st["half"] > 10000, st


def test_score1x1_full_size_3s():
    """the trainer's geometry: N = 4096, hop 512, F = 2049, tc 30"""
    run_case("score1x1_N4096_3s", 4096, 512, 25, 30, 3.0, seed=2)


@pytest.mark.parametrize("extra", [0, 1])
def test_score1x1_decoder_chunks(extra):
    """3 x 128 patches (exactly 3 chunks) and one more (a 4th chunk of one patch, whose halo reaches back into the 3rd):
    each chunk writes only its own frames, the profile shows one K3s record per chunk"""
    N, hop, overlap, tc = 512, 256, 25, 30
    P = 384 + extra
    T = overlap + 1 + (P - 1) * (tc - overlap)          # util patcher: P = (T - overlap - 1) // step + 1
    seconds = (T - 2) * hop / 44100.0
    params = s1.make_synthetic_params_1x1(seed=9)
    sep = separator(params, N, hop, overlap, tc)
    assert sep.num_patches(dsp.num_frames(int(round(seconds * 44100)), hop)) == P
    _lib_check = sep.lib.dcs_profile(sep.ctx.handle, 1)
    assert _lib_check == 0
    run_case("score1x1_chunks_P%d" % P, N, hop, overlap, tc, seconds, sep=sep, params=params, mix_seed=5)
    torch.cuda.synchronize()
    names = profile_names(sep)
    sep.lib.dcs_profile(sep.ctx.handle, 0)
    nchunks = names.count("dec_convT1_mask_xfade")
    assert nchunks == 3 + extra, names
    record("score1x1_chunks_P%d_profile" % P, patches=P, chunks=nchunks)


def test_score1x1_spec_channels_odd_width():
    """F = 300 (not an STFT size) through dcs_separate_spec_channels: columns uncovered by the next layer's windows in
    five of the six layers; the blended masks against the oracle's (device gate codes adopted where flagged), flagged
    bins excluded"""
    from deepconvsep_b200.engine import Model, Context, _ptr
    from deepconvsep_b200._lib import check
    from deepconvsep_b200.models import gate_code_layout
    F, tc, overlap, T = 300, 30, 25, 260
    params = s1.make_synthetic_params_1x1(seed=21)
    rng = np.random.default_rng(3)
    mag = (0.2 * rng.random((T, F)) ** 4).astype(np.float32)
    filt = score_filters(T, F, seed=6)
    chans = (filt * mag[None]).astype(np.float32)
    X = (rng.standard_normal((T, F)) + 1j * rng.standard_normal((T, F))).astype(np.complex64)
    ctx = Context(0)
    model = Model(ctx, params, arch=ARCH, feat_size=F, time_context=tc)
    ldf = 304
    dev = torch.device("cuda", 0)
    cd = torch.zeros((4, T, ldf), dtype=torch.float32, device=dev)
    cd[:, :, :F] = torch.as_tensor(chans, device=dev)
    Xd = torch.zeros((T, ldf), dtype=torch.complex64, device=dev)
    Xd[:, :F] = torch.as_tensor(X, device=dev)
    S = torch.zeros((4, T, ldf), dtype=torch.complex64, device=dev)
    P = int(ctx.lib.dcs_num_patches(T, tc, overlap, 1))
    layout = gate_code_layout(F, tc, max(T, (P - 1) * (tc - overlap) + tc))
    bits = torch.zeros(sum(r * w * c for r, w, c in layout), dtype=torch.uint8, device=dev)
    check(ctx.lib.dcs_set_pool_tap(ctx.handle, _ptr(bits), bits.numel()))
    check(ctx.lib.dcs_separate_spec_channels(ctx.handle, model.handle, _ptr(cd), T * ldf, _ptr(Xd), T, ldf, overlap, 1,
                                             _ptr(S), T * ldf, None))
    torch.cuda.synchronize()
    check(ctx.lib.dcs_set_pool_tap(ctx.handle, None, 0))
    flat, codes = bits.cpu().numpy(), []
    for r, w, c in layout:
        codes.append(flat[:r * w * c].reshape(r, w, c))
        flat = flat[r * w * c:]
    Sd = S[:, :, :F].cpu().numpy().astype(np.complex128)
    batches, nchunks = s1.patches(chans.astype(np.float64), tc, overlap, 32)
    out = []
    kmap = np.zeros((nchunks * (tc - overlap) + tc, F), dtype=bool)
    stats = {}
    for bi, b in enumerate(batches):
        pre = s1.predict_1x1(params, b, return_pre=True, gate_stats=stats,
                             gate_dev=s1.device_gates(codes, bi, b.shape[0], nchunks, tc - overlap, tc))
        out.append([nets.soft_masks(nets.relu(pre), "bach10", 4)[:, i:i + 1] for i in range(4)])
        nb = max(0, min(nchunks - bi * 32, 32))
        flag = nets.near_kink(pre[:nb], "bach10", 4)
        for i in np.nonzero(flag.reshape(nb, -1).any(axis=1))[0]:
            k0 = (bi * 32 + int(i)) * (tc - overlap)
            kmap[k0:k0 + tc] |= flag[i]
    from oracle import patch
    masks = patch.overlapadd_multi(np.array(out), batches, nchunks, overlap=overlap)[:, :T]
    keep = ~kmap[:T]
    assert stats["disagree_unflagged"] == 0 and stats["flagged"] <= 1e-3 * stats["positions"], stats
    for s in range(4):
        want = masks[s] * X
        err = np.linalg.norm((Sd[s] - want)[keep]) / np.linalg.norm(want)
        assert err <= TOL, (s, err)
    record("score1x1_spec_channels_F300", rel_l2_spectrum=[float(np.linalg.norm((Sd[s] - masks[s] * X)[keep]) /
                                                                 np.linalg.norm(masks[s] * X)) for s in range(4)],
           flagged_bins=int(kmap[:T].sum()))


def test_score1x1_deterministic_and_shares_a_context():
    """twice on one context, and alternating with the 17-array score net on the same context: the same bytes each time"""
    from deepconvsep_b200.engine import Context, Model, Stft
    N, hop, F = 512, 256, 257
    ctx = Context(0)
    mix, _ = pipeline.synth_mixture(1.0, 3)
    a = torch.as_tensor(mix.astype(np.float32), device="cuda:0")
    T = dsp.num_frames(mix.size, hop)
    st = Stft(ctx, N, hop, "blackmanharris")
    fd = torch.zeros((4, T, st.ldf), dtype=torch.float32, device="cuda:0")
    fd[:, :, :F] = torch.as_tensor(score_filters(T, F), device="cuda:0")
    models = [Model(ctx, s1.make_synthetic_params_1x1(seed=4), arch=ARCH, feat_size=F, time_context=30),
              Model(ctx, nets.make_synthetic_params("bach10_score", F, seed=4), arch="bach10_score", feat_size=F)]
    outs = {}
    for rnd in range(2):
        for i, m in enumerate(models):
            for ov in (25, 0):
                out = torch.empty((4, mix.size), dtype=torch.float32, device="cuda:0")
                rc = ctx.lib.dcs_separate_audio_score(ctx.handle, m.handle, st.handle, _p(a), mix.size, _p(fd), C.c_float(0.2),
                                                      ov, 1, _p(out), mix.size, None)
                assert rc == 0
                torch.cuda.synchronize()
                o = out.cpu().numpy()
                if rnd == 0:
                    outs[i, ov] = o
                    assert np.abs(o).max() > 0
                else:
                    assert np.array_equal(o, outs[i, ov]), (i, ov)


def _p(t):
    return C.c_void_p(t.data_ptr())


def test_score1x1_refused_entry_points_queue_nothing():
    """every single-channel, stereo and batch entry point refuses the 1x1 net before queuing work and names the two
    entry points that serve it"""
    from deepconvsep_b200.engine import Context, Model, Stft
    N, hop, F = 512, 256, 257
    ctx = Context(0)
    lib = ctx.lib
    m = Model(ctx, s1.make_synthetic_params_1x1(seed=4), arch=ARCH, feat_size=F, time_context=30)
    st = Stft(ctx, N, hop, "blackmanharris")
    L = 20000
    a = torch.zeros((2, L), dtype=torch.float32, device="cuda:0")
    out = torch.zeros((8, L), dtype=torch.float32, device="cuda:0")
    h = np.zeros(L, dtype=np.float32)
    ho = np.zeros((4, L), dtype=np.float32)
    pcm = np.zeros(L, dtype=np.int16)
    pout = np.zeros((4, L), dtype=np.int16)
    Ls = np.array([L], dtype=np.int64)
    pins = (C.c_void_p * 1)(pcm.ctypes.data)
    pouts = (C.c_void_p * 1)(pout.ctypes.data)
    T = dsp.num_frames(L, hop)
    mag = torch.zeros((T, st.ldf), dtype=torch.float32, device="cuda:0")
    X = torch.zeros((T, st.ldf), dtype=torch.complex64, device="cuda:0")
    S = torch.zeros((4, T, st.ldf), dtype=torch.complex64, device="cuda:0")
    before = lib.dcs_launch_count(ctx.handle)
    calls = [
        lambda: lib.dcs_separate_audio(ctx.handle, m.handle, st.handle, _p(a), L, C.c_float(0.2), 25, 1, _p(out), L, None),
        lambda: lib.dcs_separate_host(ctx.handle, m.handle, st.handle, h.ctypes.data, L, C.c_float(0.2), 25, 1, ho.ctypes.data, L, None),
        lambda: lib.dcs_separate_spec(ctx.handle, m.handle, _p(mag), _p(X), T, st.ldf, 25, 1, _p(S), T * st.ldf, None),
        lambda: lib.dcs_separate_audio_stereo(ctx.handle, m.handle, st.handle, _p(a), L, L, C.c_float(0.2), 25, 1, _p(out), L, None),
        lambda: lib.dcs_separate_audio_keep_channels(ctx.handle, m.handle, st.handle, _p(a), L, L, C.c_float(0.2), 25, 1, _p(out), L, None),
        lambda: lib.dcs_separate_pcm16_host(ctx.handle, m.handle, st.handle, pcm.ctypes.data, L, 1, 0, C.c_float(0.2), 25, 1,
                                            pout.ctypes.data, L, None),
        lambda: lib.dcs_separate_batch_pcm16_host(ctx.handle, m.handle, st.handle, 1, pins, Ls.ctypes.data, 1, 0, C.c_float(0.2),
                                                  25, 1, pouts, Ls.ctypes.data, None),
    ]
    for f in calls:
        assert f() != 0
        msg = lib.dcs_last_error().decode()
        assert "dcs_separate_audio_score" in msg and "dcs_separate_spec_channels" in msg, msg
    assert lib.dcs_launch_count(ctx.handle) == before


def test_one_decoder_score_net_matches_decoder_one_of_the_17_array_net():
    """the default build_ca of trainCNNrwc_samp.py:195-235 (11 arrays) is decoder 1 of the 17-array net: same bits"""
    from deepconvsep_b200.engine import Separator
    F, N, hop = 129, 256, 128
    p17 = nets.make_synthetic_params("bach10_score", F, seed=8)
    p11 = p17[:10] + [np.ascontiguousarray(p17[16][:4])]
    mix, _ = pipeline.synth_mixture(1.0, 91)
    T = dsp.num_frames(mix.size, hop)
    filters = score_filters(T, F)
    outs = []
    for p in (p17, p11):
        sep = Separator(p, frame_size=N, hop=hop, window="blackmanharris", overlap=25, patcher="util", scale_factor=0.2,
                        feat_size=F)
        assert sep.model.arch == "bach10_score"
        outs.append(sep.separate_score(mix, filters))
    assert np.abs(outs[0]).max() > 0 and np.array_equal(outs[0], outs[1])


def test_score1x1_tensor_core_mask_matches_ffma_twin(monkeypatch):
    """K3s on the tensor cores (the product path) against its FFMA twin (DCS_DEBUG_SIMT_GEMM=1)"""
    params = s1.make_synthetic_params_1x1(seed=5)
    mix, _ = pipeline.synth_mixture(1.0, 77)
    T = dsp.num_frames(mix.size, 256)
    filters = score_filters(T, 257)
    outs = []
    for simt in ("0", "1"):
        monkeypatch.setenv("DCS_DEBUG_SIMT_GEMM", simt)
        sep = separator(params, 512, 256, 25, 30)
        outs.append(np.asarray(sep.separate_score(mix, filters), dtype=np.float64))
    for s in range(4):
        assert np.linalg.norm(outs[1][s]) > 0
        assert np.linalg.norm(outs[0][s] - outs[1][s]) / np.linalg.norm(outs[1][s]) <= TOL
