"""GPU parity of the DSD100 separation path (through the C ABI) against the float64 oracle.

Tolerance (BASELINE.json north_star): per-stem relative L2 on the float waveform <= 1e-4;
SDR delta vs the synthetic ground-truth stems <= 0.01 dB."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from oracle import dsp, nets, pipeline, patch, bsseval  # noqa: E402
from parity import strict_check, TOL  # noqa: E402

# Comparison rule (tests/parity.py): plain 1e-4 per stem, NO whole-stem allowance.  The handful of
# time-frequency bins the ORACLE flags as sitting on the soft mask's discontinuity
# (oracle.nets.near_kink) are taken out bin by bin: there the oracle spectrum adopts the device's
# (admissible) value before the comparison; everything else is held to the bar.


def run_strict(name, sep, params, mix, N, hop, overlap, patcher="standalone", window=np.hanning):
    want, mag, ph, mm = pipeline.separate(mix, params, "dsd", frameSize=N, hopSize=hop, window=window, overlap=overlap,
                                          patcher=patcher, count_kinks=True, return_spec=True)
    kmap = pipeline.separate.last_kink_map
    got, S = sep.separate_tapped(mix)
    assert got.shape == want.shape and got.dtype == np.float32
    strict_check(name, got, S, want, mag, ph, mm, kmap, N, hop, window, 0.3)
    return got, want


def rel(a, b):
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def sdr(ref, est):
    return 10 * np.log10(np.sum(ref ** 2) / max(np.sum((ref - est) ** 2), 1e-30))


def check_bss_eval(got, want, stems):
    """the reference's own metric (evaluation/bss_eval/bss_eval_sources.m, restated in oracle.bsseval):
    SDR / SIR / SAR of the GPU stems and of the oracle stems against the true sources differ by
    <= 0.01 dB and pick the same source ordering"""
    g = bsseval.bss_eval_sources(got.astype(np.float64), stems)
    w = bsseval.bss_eval_sources(want, stems)
    assert list(g[3]) == list(w[3])
    for name, a, b in zip(("SDR", "SIR", "SAR"), g[:3], w[:3]):
        assert np.max(np.abs(a - b)) <= 0.01, (name, a, b)


def make_sep(N, seed=0, overlap=25, patcher="standalone", window="hanning", hop=512):
    from deepconvsep_b200.engine import Separator
    F = N // 2 + 1
    params = nets.make_synthetic_params("dsd", F, seed=seed)
    return params, Separator(params, frame_size=N, hop=hop, window=window, overlap=overlap, patcher=patcher)


@pytest.mark.parametrize("N,seconds,overlap,patcher", [
    (1024, 4.0, 25, "standalone"), (2048, 3.0, 25, "standalone"), (1024, 2.5, 25, "util"),
    (1024, 2.0, 20, "standalone"), (1024, 1.3, 10, "util"), (512, 1.0, 25, "standalone")])
def test_separate_matches_oracle(N, seconds, overlap, patcher):
    hop = min(512, N // 2)
    params, sep = make_sep(N, seed=N + overlap, overlap=overlap, patcher=patcher, hop=hop)
    mix, stems = pipeline.synth_mixture(seconds, 1000 + N)
    got, want = run_strict("dsd_N%d_%gs_ov%d_%s" % (N, seconds, overlap, patcher), sep, params, mix, N, hop, overlap, patcher)
    # the synthetic weights must exercise every source (no constant masks)
    assert min(np.linalg.norm(want[s]) for s in range(4)) > 0.02 * np.linalg.norm(mix)
    for s in range(4):
        assert abs(sdr(stems[s], got[s]) - sdr(stems[s], want[s])) <= 0.01
    if (N, seconds) == (1024, 4.0):
        check_bss_eval(got, want, stems)
    # the device-buffer entry point gives the same bits as the host-buffer one
    d = sep.separate_device(torch.tensor(mix, dtype=torch.float32, device="cuda"))
    assert np.array_equal(d.cpu().numpy(), got)


def test_spec_level_matches_oracle():
    """dcs_separate_spec: blended masked spectra vs overlapadd_multi(predict(...)) of the oracle."""
    N, F = 1024, 513
    params, sep = make_sep(N, seed=7)
    mix, _ = pipeline.synth_mixture(3.0, 77)
    _, mag, ph, mm = pipeline.separate(mix, params, "dsd", frameSize=N, overlap=25, return_spec=True)
    X = dsp.stft_norm(mix, window=np.hanning(N), hopsize=512.0, nfft=float(N))
    T = X.shape[0]
    ldf = sep.stft.ldf
    magd = torch.zeros((T, ldf), dtype=torch.float32, device="cuda")
    Xd = torch.zeros((T, ldf), dtype=torch.complex64, device="cuda")
    magd[:, :F] = torch.tensor(mag, device="cuda")
    Xd[:, :F] = torch.tensor(X.astype(np.complex64), device="cuda")
    S = sep.separate_spec(magd, Xd).cpu().numpy()[:, :, :F].astype(np.complex128)
    want = (mm[:, :T] / 0.3) * np.sqrt(N) * np.exp(1j * ph)[None]
    for s in range(4):
        assert rel(S[s], want[s]) <= TOL, (s, rel(S[s], want[s]))
    # mask level, bin by bin.  The reference's mask is discontinuous where the rectified
    # outputs of all sources vanish (1/4 each vs p/sum(p)): a bin whose float64 sum(p) is
    # within fp32 noise of that kink cannot be reproduced by ANY fp32 evaluation.  Flag those
    # with the oracle and require tight agreement everywhere else.
    b, n = patch.generate_overlapadd(mag, F, 30, 25, 32)
    pred = np.concatenate([nets.predict(params, bb, "dsd") for bb in b])[:n]   # [P,4,30,F]
    near_kink = np.zeros((T, F), bool)
    for k in range(n):
        tot = pred[k].sum(axis=0)
        near_kink[k * 5:k * 5 + 30] |= (tot < 1e-6) & (np.abs(pred[k]).max(axis=0) < 1e-6) & ~((tot == 0) & (pred[k].max(axis=0) == 0)) | ((tot > 0) & (tot < 1e-7))
    Xn = np.abs(X)
    ok = (Xn > 1e-3 * Xn.mean()) & ~near_kink
    mg = np.abs(S) / np.maximum(Xn, 1e-30)
    mw = np.abs(want) / np.maximum(Xn, 1e-30)
    dm = np.abs(mg - mw)[:, ok]
    assert near_kink.mean() < 1e-3
    assert dm.max() < 2e-4, dm.max()
    assert np.sqrt((dm ** 2).mean()) < 2e-6
    # frames past the last patch are exactly zero (stand-alone patcher drops the tail)
    P = patch.num_patches(T, 30, 25)
    assert sep.num_patches(T) == P
    assert np.all(S[:, (P - 1) * 5 + 30:] == 0)


@pytest.mark.parametrize("L", [1, 100, 14336, 14848, 15361])
def test_short_and_edge_lengths(L):
    """T <= time_context gives no patch (all-zero stems); T = 31, 32 give exactly one."""
    N = 1024
    params, sep = make_sep(N, seed=3)
    rng = np.random.default_rng(L)
    x = rng.standard_normal(L) * 0.1
    got = sep.separate(x)
    T = dsp.num_frames(L, 512)
    if patch.num_patches(T, 30, 25) == 0:
        assert np.all(got == 0)
    else:
        want = pipeline.separate(x, params, "dsd", frameSize=N, overlap=25)
        for s in range(4):
            assert rel(got[s].astype(np.float64), want[s]) <= TOL


def test_medium_clip_parity():
    """20 s clip, both BASELINE frame sizes."""
    for N in (1024, 2048):
        params, sep = make_sep(N, seed=42)
        mix, stems = pipeline.synth_mixture(20.0, 4242 + N)
        got, want = run_strict("dsd_N%d_20s" % N, sep, params, mix, N, 512, 25)
        for s in range(4):
            assert abs(sdr(stems[s], got[s]) - sdr(stems[s], want[s])) <= 0.01
        check_bss_eval(got, want, stems)


def test_pcm16_wav_contract():
    """int16 stereo in -> (L+R)/2 downmix -> int16 stems out, as train_auto reads/writes wavs."""
    N = 1024
    params, sep = make_sep(N, seed=11)
    mix, _ = pipeline.synth_mixture(2.0, 5)
    rng = np.random.default_rng(0)
    left = np.round(mix * 32767 * 0.9).astype(np.int16)
    right = np.round((mix * 0.7 + 0.01 * rng.standard_normal(mix.size)) * 32767).astype(np.int16)
    pcm = np.stack([left, right], axis=1)
    mono = pipeline.decode_wav_array(pcm, "dsd")
    want = pipeline.separate(mono, params, "dsd", frameSize=N, overlap=25)
    want16 = (want * 32767).astype("int16")
    got16 = sep.separate_pcm16(pcm)
    assert got16.shape == want16.shape and got16.dtype == np.int16
    d = got16.astype(np.int32) - want16.astype(np.int32)
    assert np.abs(d).max() <= 1                      # truncation flips at most one LSB
    assert np.mean(d != 0) < 0.02


def test_full_size_properties():
    """BASELINE size (180 s, N=2048): masks sum to one, so the four stems add up to the
    reconstructed mixture wherever a patch covers the frame; the tail is zero; repeatable."""
    N = 2048
    params, sep = make_sep(N, seed=0)
    g = torch.Generator(device="cuda").manual_seed(9)
    x = (torch.rand(7938000, generator=g, device="cuda") - 0.5) * 0.4
    y = sep.separate_device(x)
    torch.cuda.synchronize()
    assert y.shape == (4, 7938000) and bool(torch.isfinite(y).all())
    T = dsp.num_frames(7938000, 512)
    P = patch.num_patches(T, 30, 25)
    covered = ((P - 1) * 5 + 30 - 4) * 512 - N          # samples whose every frame has a mask
    tot = y.sum(0)[:covered]
    err = (torch.linalg.vector_norm(tot - x[:covered]) / torch.linalg.vector_norm(x[:covered])).item()
    assert err < 1e-5, err
    y2 = sep.separate_device(x)
    assert torch.equal(y, y2)                             # deterministic (no atomics)


@pytest.mark.parametrize("arch,N,seconds", [("dsd", 1024, 1.5), ("dsd", 2048, 6.0), ("dsd_ild", 1024, 3.0)])
def test_tensor_core_mask_matches_ffma_twin(monkeypatch, arch, N, seconds):
    """the wgmma mask + cross-fade kernel (dsd_tc.cu) against its exact-fp32 FFMA twin (dsd.cu, selected by
    DCS_DEBUG_SIMT_GEMM=1, read when a context is created; every other layer stays on the tensor cores): same stems
    within the parity bar"""
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
