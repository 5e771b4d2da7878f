"""Keep-channels mode of the DSD100 / hiphopss network on the GPU (dcs_separate_audio_keep_channels,
dcs_separate_batch_pcm16_keep_channels_host): the soft masks of the downmix (l + r) * 0.5f applied to the STFT of each
channel inside the masked inverse STFT (the C-channel path at C = 2); the masks come from the wgmma mask kernel
(dsd_tc.cu) in masks mode, or from its FFMA twin (dsd.cu).

- equal channels: each output channel is byte-identical to the mono call;
- parity per (source, channel) against the float64 oracle (tests/channels_oracle.py at C = 2) under tests/parity.strict_check,
  the downmix's ill-conditioned bins taken out bin by bin;
- one mask for both channels: S_c / X_c agrees across the channels and with the mono call;
- the tensor-core kernel against the FFMA twin at the schedule edge of test_gpu_dsd_mask_schedule.py;
- the int16 batch path against one-clip calls and the float path;
- refusals before anything is queued, a spectrum tap without the Wiener post-filter included."""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from oracle import nets, pipeline  # noqa: E402
from parity import strict_check, TOL  # noqa: E402
from channels_oracle import separate_channels  # noqa: E402


def rel(a, b):
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def stereo_clip(seconds, seed):
    """two different channels (float32-representable, as the device sees them)"""
    mix, _ = pipeline.synth_mixture(seconds, seed)
    other, _ = pipeline.synth_mixture(seconds, seed + 1)
    a = np.stack([0.7 * mix + 0.3 * other, 0.4 * mix + 0.6 * np.roll(other, 11)], axis=1)
    return a.astype(np.float32).astype(np.float64)


def separator(N, seed, overlap=25, patcher="standalone", hop=None):
    from deepconvsep_b200.engine import Separator
    params = nets.make_synthetic_params("dsd", N // 2 + 1, seed=seed)
    hop = hop or min(512, N // 2)
    return params, Separator(params, frame_size=N, hop=hop, window="hanning", overlap=overlap, patcher=patcher)


@pytest.mark.parametrize("N", [1024, 2048])
def test_equal_channels_match_the_mono_call_bytes(N):
    params, sep = separator(N, 40 + N)
    x, _ = pipeline.synth_mixture(2.0, 7 + N)
    x = x.astype(np.float32)
    mono = sep.separate(x)
    keep = sep.separate_keep_channels(np.stack([x, x], axis=1))
    assert keep.shape == (x.size, 4, 2) and keep.dtype == np.float32
    for c in range(2):
        assert np.array_equal(keep[:, :, c].T, mono), c
    # device planes: (source, channel) order, the same bits
    d = sep.separate_keep_channels(torch.tensor(np.stack([x, x]), device="cuda"))
    assert np.array_equal(d.cpu().numpy().reshape(4, 2, -1).transpose(2, 0, 1), keep)
    # int16: a stereo clip with equal channels, against the mono int16 call (downmix 1)
    pcm = np.round(x * 32767).astype(np.int16)
    pcm2 = np.stack([pcm, pcm], axis=1)
    want = sep.separate_pcm16(pcm2)
    got = sep.separate_pcm16(pcm2, keep_channels=True)
    assert got.shape == (4, x.size, 2) and got.dtype == np.int16
    for c in range(2):
        assert np.array_equal(got[:, :, c], want), c


def run_strict(name, sep, params, audio, N, hop, overlap=25, patcher="standalone"):
    want, mags, phs, mms, _, kmap = separate_channels(audio, params, frameSize=N, hopSize=hop, overlap=overlap,
                                                      patcher=patcher)
    got, S = sep.separate_tapped(audio, keep_channels=True)     # got [L, 4, 2]; S planes (source, channel)
    assert got.shape == want.shape == (audio.shape[0], 4, 2) and got.dtype == np.float32
    for c in range(2):
        strict_check("%s_ch%d" % (name, c), np.ascontiguousarray(got[:, :, c].T), S[c::2], np.ascontiguousarray(want[:, :, c].T),
                     mags[c], phs[c], mms[c], kmap, N, hop, np.hanning, 0.3)
    for i in range(4):
        for c in range(2):
            # every (source, channel) must carry energy, or the comparison exercises nothing
            assert np.linalg.norm(want[:, i, c]) > 1e-3 * np.linalg.norm(audio[:, c]), (i, c)
    return got, want


@pytest.mark.parametrize("N,seconds", [(512, 1.2), (1024, 3.0), (2048, 2.5)])
@pytest.mark.parametrize("patcher", ["standalone", "util"])
def test_keep_channels_matches_oracle(N, seconds, patcher):
    params, sep = separator(N, N + 3, patcher=patcher)
    hop = sep.hop
    run_strict("keep_N%d_%gs_%s" % (N, seconds, patcher), sep, params, stereo_clip(seconds, 500 + N), N, hop, patcher=patcher)


def test_keep_channels_medium_clip_strict():
    """15 s clip"""
    params, sep = separator(1024, 91)
    run_strict("keep_N1024_15s", sep, params, stereo_clip(15.0, 4322), 1024, 512)


def test_keep_channels_anti_phase_segment():
    """L = -R over 1 s: the downmix is silent there, the channels are not"""
    params, sep = separator(1024, 92)
    audio = stereo_clip(3.0, 77)
    audio[44100:88200, 1] = -audio[44100:88200, 0]
    got, want = run_strict("keep_N1024_antiphase", sep, params, audio, 1024, 512)
    assert np.isfinite(got).all()
    seg = slice(50000, 80000)
    assert np.linalg.norm(got[seg, :, 0]) > 0 and np.linalg.norm(got[seg, :, 1]) > 0


def test_keep_channels_many_patches_per_frame_ffma_twin():
    """overlap 27: 10 patches per frame, the FFMA mask kernel runs once per channel"""
    params, sep = separator(1024, 93, overlap=27)
    run_strict("keep_N1024_ov27", sep, params, stereo_clip(2.0, 88), 1024, 512, overlap=27)


def test_one_mask_for_both_channels():
    """S_c / X_c from the tap and the device STFTs: the same real mask for L, R and the mono call"""
    N = 1024
    params, sep = separator(N, 94)
    audio = stereo_clip(3.0, 99).astype(np.float32)
    F = sep.model.F
    _, S = sep.separate_tapped(audio, keep_channels=True)
    mono = (audio[:, 0] + audio[:, 1]) * np.float32(0.5)
    _, Sm = sep.separate_tapped(mono)
    X = [sep.stft.forward(torch.tensor(np.ascontiguousarray(a), device="cuda"), want_mag=False)[0][:, :F].cpu().numpy()
         for a in (audio[:, 0], audio[:, 1], mono)]
    floor = 1e-3 * max(float(np.abs(x).max()) for x in X)
    ok = (np.abs(X[0]) > floor) & (np.abs(X[1]) > floor) & (np.abs(X[2]) > floor)
    assert ok.sum() > 1000
    ulp = 2.0 ** -24
    for s in range(4):
        r = [S[2 * s + c][ok].astype(np.complex128) / X[c][ok].astype(np.complex128) for c in range(2)]
        rm = Sm[s][ok].astype(np.complex128) / X[2][ok].astype(np.complex128)
        scale = np.maximum(np.abs(rm.real), 1e-30)
        assert np.all(np.abs(r[0].real - r[1].real) <= 8 * ulp * scale), s
        assert np.all(np.abs(r[0].real - rm.real) <= 8 * ulp * scale), s
        for rr in r + [rm]:
            assert np.all(np.abs(rr.imag) <= 8 * ulp * scale), s


def test_tensor_core_kernel_matches_ffma_twin(monkeypatch):
    """the schedule edge of test_gpu_dsd_mask_schedule.py: 0.5 s at N = 2048"""
    from deepconvsep_b200.engine import Separator
    N = 2048
    params = nets.make_synthetic_params("dsd", N // 2 + 1, seed=2)
    audio = stereo_clip(0.5, 1003)
    outs = []
    for simt in ("0", "1"):
        monkeypatch.setenv("DCS_DEBUG_SIMT_GEMM", simt)
        sep = Separator(params, frame_size=N, hop=512, window="hanning", overlap=25, device=0)
        got, _ = sep.separate_tapped(audio, keep_channels=True)
        outs.append(np.asarray(got, dtype=np.float64))
    tc, ffma = outs
    assert np.isfinite(tc).all() and tc.shape == ffma.shape
    for s in range(4):
        for c in range(2):
            assert np.linalg.norm(ffma[:, s, c]) > 0
            assert rel(tc[:, s, c], ffma[:, s, c]) <= TOL, (s, c, rel(tc[:, s, c], ffma[:, s, c]))


def test_int16_batch_matches_one_clip_calls_and_the_float_path():
    params, sep = separator(1024, 95)
    clips = []
    for k, seconds in enumerate((3.0, 1.7, 2.4)):
        a = stereo_clip(seconds, 700 + k)
        clips.append(np.round(a * 0.8 * 32767).astype(np.int16))
    got = sep.separate_pcm16_batch(clips, keep_channels=True)
    for pcm, g in zip(clips, got):
        L = pcm.shape[0]
        assert g.shape == (4, L, 2) and g.dtype == np.int16
        assert np.array_equal(g, sep.separate_pcm16(pcm, keep_channels=True))
        planes = torch.tensor(np.ascontiguousarray(pcm.T.astype(np.float32) / np.float32(32767)), device="cuda")
        stems = sep.separate_keep_channels(planes).cpu().numpy()                 # [8, L], (source, channel)
        want = (stems * np.float32(32767)).astype(np.int16).reshape(4, 2, L).transpose(0, 2, 1)
        assert np.array_equal(g, want)
        assert np.abs(g.astype(np.int64)).sum() > 0


def test_refusals_queue_nothing():
    from deepconvsep_b200 import _lib
    from deepconvsep_b200.engine import Model, _ptr
    params, sep = separator(1024, 96)
    ctx, lib = sep.ctx, sep.lib
    audio = stereo_clip(1.0, 5)
    ref = sep.separate_keep_channels(audio)
    pcm = np.round(audio * 32767).astype(np.int16)
    ref16 = sep.separate_pcm16(pcm, keep_channels=True)
    others = {a: Model(ctx, nets.make_synthetic_params(a, F, seed=3), arch=a, feat_size=F)
              for a, F in (("ikala", 513), ("bach10", 129), ("bach10_score", 129), ("dsd_ild", 513))}
    L = audio.shape[0]
    x = torch.tensor(np.ascontiguousarray(audio.T.astype(np.float32)), device="cuda")
    stems = torch.empty((8, L), dtype=torch.float32, device="cuda")
    Ls = np.array([L], dtype=np.int64)
    out16 = np.empty((4, L, 2), dtype=np.int16)
    pin = (C.c_void_p * 1)(pcm.ctypes.data)
    pout = (C.c_void_p * 1)(out16.ctypes.data)

    def audio_call(model, stride=L, overlap=25):
        return lib.dcs_separate_audio_keep_channels(ctx.handle, model.handle, sep.stft.handle, _ptr(x), stride, L,
                                                    C.c_float(0.3), overlap, 0, _ptr(stems), L, None)

    def batch_call(model, overlap=25):
        return lib.dcs_separate_batch_pcm16_keep_channels_host(ctx.handle, model.handle, sep.stft.handle, 1, pin,
                                                               Ls.ctypes.data, C.c_float(0.3), overlap, 0, pout,
                                                               Ls.ctypes.data, None)
    refused = {}
    for a, m in others.items():
        refused["audio, " + a] = (lambda m=m: audio_call(m), None)
        refused["batch, " + a] = (lambda m=m: batch_call(m), None)
    refused["audio, stride < length"] = (lambda: audio_call(sep.model, stride=L - 1), None)
    refused["audio, overlap = time_context"] = (lambda: audio_call(sep.model, overlap=sep.model.tc), None)
    refused["batch, overlap = time_context"] = (lambda: batch_call(sep.model, overlap=sep.model.tc), None)
    tap = torch.zeros((8, sep.stft.num_frames(L), sep.stft.ldf), dtype=torch.complex64, device="cuda")

    def tapped(call):
        _lib.check(lib.dcs_set_spectrum_tap(ctx.handle, _ptr(tap), tap.numel()))
        try:
            return call()
        finally:
            _lib.check(lib.dcs_set_spectrum_tap(ctx.handle, None, 0))
    refused["audio, spectrum tap without Wiener"] = (lambda: tapped(lambda: audio_call(sep.model)), "spectrum tap")
    refused["batch, spectrum tap without Wiener"] = (lambda: tapped(lambda: batch_call(sep.model)), "spectrum tap")
    for name, (call, msg) in refused.items():
        torch.cuda.synchronize()
        n0 = ctx.launch_count()
        with pytest.raises(_lib.DcsError) as e:
            _lib.check(call())
        assert ctx.launch_count() == n0, name
        if name == "audio, dsd_ild":
            assert "dcs_separate_audio_stereo" in str(e.value)
        if msg:
            assert msg in str(e.value), name
    with pytest.raises(ValueError):
        sep.separate_keep_channels(audio[:, 0])
    assert np.array_equal(sep.separate_keep_channels(audio), ref)
    assert np.array_equal(sep.separate_pcm16(pcm, keep_channels=True), ref16)
