"""The multichannel Wiener post-filter on the GPU (csrc/wiener.cu: dcs_wiener_stereo, dcs_set_wiener) against the
float64 restatement in oracle/wiener.py:

- off (0 iterations, or a context the setting never touched): the stereo entry points give the same bytes as before;
- spectrum level: seeded synthetic spectra, K = 1, 2, 3, per-plane relative L2 <= 1e-5; pad bins and all-zero frames
  untouched;
- end to end: keep-channels on a 180 s clip at N = 2048 and the stereo / ILD net on 15 s, the oracle fed the network's
  spectra of the same call with the filter off and the float64 STFT of the input: spectra <= 1e-5, stems <= 1e-4;
- equal channels: bit-identical channels and the closed form;
- determinism, the int16 batch path, refusals before anything is queued."""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from oracle import dsp, nets, pipeline  # noqa: E402
from oracle import wiener as W  # noqa: E402
from parity import record  # noqa: E402

SPEC_BAR, STEM_BAR = 1e-5, 1e-4


def rel(a, b):
    return float(np.linalg.norm(np.asarray(a, np.complex128) - b) / max(np.linalg.norm(b), 1e-30))


def stereo_clip(seconds, seed):
    """two different channels (float32-representable, as the device sees them) -- test_gpu_keep_channels.py's clip"""
    mix, _ = pipeline.synth_mixture(seconds, seed)
    other, _ = pipeline.synth_mixture(seconds, seed + 1)
    a = np.stack([0.7 * mix + 0.3 * other, 0.4 * mix + 0.6 * np.roll(other, 11)], axis=1)
    return a.astype(np.float32).astype(np.float64)


def separator(arch, N, seed, patcher="standalone"):
    from deepconvsep_b200.engine import Separator
    params = nets.make_synthetic_params(arch, N // 2 + 1, seed=seed)
    return Separator(params, frame_size=N, hop=min(512, N // 2), window="hanning", overlap=25, patcher=patcher)


def synthetic(T, F, ldf, seed, silent=()):
    """X [2, T, ldf] and soft-mask stems [8, T, ldf] (complex64), pad bins of X zero, of S a sentinel; frames in
    `silent` have every stem zero"""
    rng = np.random.default_rng(seed)
    pans = np.array([0.1, 0.35, 0.65, 0.9])
    src = (rng.standard_normal((4, T, F)) + 1j * rng.standard_normal((4, T, F))) \
        * rng.uniform(0.01, 1.0, (4, 1, F)) * rng.gamma(0.3, 1.0, (4, T, F))
    img = np.stack([np.cos(pans * np.pi / 2), np.sin(pans * np.pi / 2)], axis=1)[:, :, None, None] * src[:, None] * 40.0
    X = np.zeros((2, T, ldf), np.complex64)
    X[:, :, :F] = img.sum(axis=0)
    mag = np.abs(img).sum(axis=1) * rng.uniform(1.0, 1.8, (4, T, F))
    S = np.full((4, 2, T, ldf), 7 - 3j, np.complex64)
    S[:, :, :, :F] = (mag / mag.sum(axis=0))[:, None] * X[None, :, :, :F]
    S[:, :, list(silent), :F] = 0
    return X, S.reshape(8, T, ldf)


@pytest.mark.parametrize("K", [1, 2, 3])
def test_spectra_match_the_oracle(K):
    from deepconvsep_b200.engine import Context, wiener_stereo
    T, F, ldf = 2000, 1025, 1032
    X, S = synthetic(T, F, ldf, seed=K, silent=range(1960, 2000))
    ctx = Context(0)
    Xd, Sd = torch.tensor(X, device="cuda"), torch.tensor(S, device="cuda")
    n0 = ctx.launch_count()
    wiener_stereo(ctx, Xd, Sd, K, num_bins=F)
    torch.cuda.synchronize()
    assert ctx.launch_count() - n0 == 2 * K + 1            # init + reduce, then EM (+ reduce but for the last)
    got = Sd.cpu().numpy()
    want = W.wiener(X[:, :, :F], S.reshape(4, 2, T, ldf)[:, :, :, :F], K).reshape(8, T, F)
    errs = [rel(got[p, :, :F], want[p]) for p in range(8)]
    record("wiener_spectra_K%d" % K, max_rel=max(errs), per_plane=errs)
    assert max(errs) <= SPEC_BAR, errs
    assert np.array_equal(got[:, :, F:], S[:, :, F:])                         # pad bins untouched
    assert not got[:, 1960:, :F].any()                                      # all-zero frames stay zero
    assert all(np.linalg.norm(got[p] - S[p]) > 1e-3 * np.linalg.norm(S[p, :, :F]) for p in range(8))   # it did filter
    # the same bits on a second run
    Sd2 = torch.tensor(S, device="cuda")
    wiener_stereo(ctx, Xd, Sd2, K, num_bins=F)
    assert torch.equal(Sd2, torch.tensor(got, device="cuda"))


def test_off_is_byte_identical_to_a_fresh_context():
    """wiener=0 after a filtered call, on every stereo entry point, against a context that never saw the setting"""
    from deepconvsep_b200.engine import _ptr
    audio = stereo_clip(3.0, 31)
    L = audio.shape[0]
    x = torch.tensor(np.ascontiguousarray(audio.T.astype(np.float32)), device="cuda")
    pcm = np.round(audio * 0.8 * 32767).astype(np.int16)
    for arch, N in (("dsd", 1024), ("dsd_ild", 1024)):
        fresh, sep = separator(arch, N, 5), separator(arch, N, 5)
        fn = "dcs_separate_audio_keep_channels" if arch == "dsd" else "dcs_separate_audio_stereo"
        want = torch.empty((8, L), dtype=torch.float32, device="cuda")
        assert getattr(fresh.lib, fn)(fresh.ctx.handle, fresh.model.handle, fresh.stft.handle, _ptr(x), L, L, C.c_float(0.3),
                                      25, fresh.patcher, _ptr(want), L, None) == 0
        call = sep.separate_keep_channels if arch == "dsd" else sep.separate_stereo
        filtered = call(x, wiener=2).clone()
        assert not torch.equal(filtered, want)
        assert torch.equal(call(x, wiener=0), want)
        assert torch.equal(call(x), want)
        if arch == "dsd":
            ref16 = fresh.separate_pcm16(pcm, keep_channels=True)
            sep.separate_pcm16(pcm, keep_channels=True, wiener=2)
            assert np.array_equal(sep.separate_pcm16(pcm, keep_channels=True), ref16)


def _end_to_end(name, sep, audio, K):
    N, hop = sep.frame_size, sep.hop
    L = audio.shape[0]
    F = N // 2 + 1
    stems0, S0 = sep.separate_tapped(audio, keep_channels=sep.model.arch == "dsd")             # the network's spectra
    stems, S = sep.separate_tapped(audio, keep_channels=sep.model.arch == "dsd", wiener=K)
    T = S0.shape[1]
    win = np.hanning(N)
    X = np.stack([dsp.stft_norm(audio[:, c], win, hop, N) for c in range(2)])                  # float64 STFT of the input
    assert X.shape == (2, T, F)
    want = W.wiener(X, S0.reshape(4, 2, T, F), K)
    del S0
    spec_errs, stem_errs = [], []
    for j in range(4):
        for c in range(2):
            spec_errs.append(rel(S[2 * j + c], want[j, c]))
            y = dsp.istft_norm(want[j, c], win, hopsize=hop, nfft=N)[:L]
            g = stems[:, j, c].astype(np.float64)
            stem_errs.append(float(np.linalg.norm(g - y) / np.linalg.norm(y)))
            assert np.linalg.norm(y) > 1e-3 * np.linalg.norm(audio[:, c]), (j, c)   # every image carries energy
            assert rel(stems[:, j, c], stems0[:, j, c]) > 1e-3, (j, c)               # and the filter moved it
    record(name, K=K, max_spec_rel=max(spec_errs), max_stem_rel=max(stem_errs), spec=spec_errs, stems=stem_errs)
    assert max(spec_errs) <= SPEC_BAR, spec_errs
    assert max(stem_errs) <= STEM_BAR, stem_errs
    return stems


def test_keep_channels_180s_n2048_matches_the_oracle():
    sep = separator("dsd", 2048, 2049)
    audio = stereo_clip(180.0, 600)
    stems = _end_to_end("wiener_keep_N2048_180s", sep, audio, 2)
    again = sep.separate_keep_channels(audio, wiener=2)
    assert np.array_equal(again, stems)                                     # the same bits on every run


def test_stereo_net_15s_matches_the_oracle():
    sep = separator("dsd_ild", 1024, 77, patcher="util")
    _end_to_end("wiener_ild_N1024_15s", sep, stereo_clip(15.0, 4321), 2)


def test_equal_channels_are_identical_and_give_the_closed_form():
    """l == r: both channels the same bits, and per iteration y_j = x rho_j v_j / (sum_k rho_k v_k + delta s^2 / 2)"""
    sep = separator("dsd", 1024, 41)
    x = stereo_clip(4.0, 17)[:, 0]
    audio = np.stack([x, x], axis=1)
    stems0, S0 = sep.separate_tapped(audio, keep_channels=True)
    stems, S = sep.separate_tapped(audio, keep_channels=True, wiener=2)
    for j in range(4):
        assert np.array_equal(stems[:, j, 0], stems[:, j, 1]), j
        assert np.array_equal(S[2 * j], S[2 * j + 1]), j
    N, F = 1024, 513
    X = dsp.stft_norm(x, np.hanning(N), 512, N)
    s = max(1.0, np.abs(X).max() / 10.0)
    y = S0[0::2].astype(np.complex128)
    for _ in range(2):
        v = np.abs(y) ** 2
        A = v.sum(axis=1, keepdims=True)
        rho = A / (W.EPS * s * s + A)
        y = X[None] * rho * v / ((rho * v).sum(axis=0) + W.DELTA * s * s / 2)
    errs = [rel(S[2 * j], y[j]) for j in range(4)]
    record("wiener_equal_channels_closed_form", errs=errs)
    assert max(errs) <= SPEC_BAR, errs


def test_int16_batch_matches_one_clip_calls_and_the_float_path():
    sep = separator("dsd", 1024, 95)
    clips = [np.round(stereo_clip(sec, 800 + k) * 0.8 * 32767).astype(np.int16) for k, sec in enumerate((3.0, 1.7, 2.4))]
    got = sep.separate_pcm16_batch(clips, keep_channels=True, wiener=2)
    for pcm, g in zip(clips, got):
        L = pcm.shape[0]
        assert g.shape == (4, L, 2) and g.dtype == np.int16
        assert np.array_equal(g, sep.separate_pcm16(pcm, keep_channels=True, wiener=2))
        planes = torch.tensor(np.ascontiguousarray(pcm.T.astype(np.float32) / np.float32(32767)), device="cuda")
        stems = sep.separate_keep_channels(planes, wiener=2).cpu().numpy()
        want = (stems * np.float32(32767)).astype(np.int16).reshape(4, 2, L).transpose(0, 2, 1)
        assert np.array_equal(g, want)
        assert not np.array_equal(g, sep.separate_pcm16(pcm, keep_channels=True))


def test_refusals_queue_nothing():
    from deepconvsep_b200 import _lib
    from deepconvsep_b200.engine import Context, _ptr
    ctx = Context(0)
    lib = ctx.lib
    T, ldf, F = 300, 520, 513
    X = torch.zeros((2, T, ldf), dtype=torch.complex64, device="cuda")
    S = torch.zeros((10, T, ldf), dtype=torch.complex64, device="cuda")

    def call(x=X, x_plane=T * ldf, s=S, src_stride=T * ldf, nsrc=4, t=T, ld=ldf, f=F, k=1):
        return lib.dcs_wiener_stereo(ctx.handle, _ptr(x), x_plane, _ptr(s), src_stride, nsrc, t, ld, f, k, None)
    refused = {
        "negative iterations": lambda: call(k=-1),
        "nsrc > 4": lambda: call(nsrc=5),
        "nsrc 0": lambda: call(nsrc=0),
        "x plane stride < T * ldf": lambda: call(x_plane=T * ldf - 1),
        "source stride < T * ldf": lambda: call(src_stride=T * ldf - 8),
        "T = 0": lambda: call(t=0),
        "F > ldf": lambda: call(f=ldf + 1),
        "NULL spectra": lambda: call(x=None),
        "set_wiener negative": lambda: lib.dcs_set_wiener(ctx.handle, -1),
    }
    torch.cuda.synchronize()
    n0 = ctx.launch_count()
    for name, fn in refused.items():
        with pytest.raises(_lib.DcsError):
            _lib.check(fn())
        assert ctx.launch_count() == n0, name
    assert call(k=0) == 0 and ctx.launch_count() == n0                      # 0 iterations: nothing to do
    # single-channel paths take no Wiener setting
    sep = separator("dsd", 1024, 7)
    mono = stereo_clip(1.0, 3)[:, 0]
    pcm = np.round(mono * 32767).astype(np.int16)
    n0 = sep.ctx.launch_count()
    with pytest.raises(ValueError):
        sep.separate_pcm16(pcm, wiener=1)
    with pytest.raises(ValueError):
        sep.separate_pcm16_batch([pcm], wiener=1)
    with pytest.raises(ValueError):
        sep.separate_tapped(mono, wiener=1)
    assert sep.ctx.launch_count() == n0
    # and the setting is ignored by the single-channel entry points of the library
    ref = sep.separate(mono)
    sep.ctx.set_wiener(3)
    assert np.array_equal(sep.separate(mono), ref)
    sep.ctx.set_wiener(0)
