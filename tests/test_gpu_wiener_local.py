"""The sliding-window Wiener post-filter on the GPU (csrc/wiener.cu: dcs_wiener_stereo_windowed, dcs_set_wiener_radius)
against the float64 restatement in tests/wiener_local_oracle.py:

- spectrum level: seeded spectra with T off the chunk grid and silent frames, K = 1, 2, 3 and W = 1, 3: per-plane
  relative L2 <= 1e-5, pad bins untouched, 2K + 1 launches, the same bits on a second run;
- a radius covering the clip gives the bytes of dcs_wiener_stereo;
- end to end: keep-channels on 180 s at N = 2048 (K = 2, W = 2) and the stereo / ILD net on 15 s, the oracle fed the
  network's spectra of the same call: spectra <= 1e-5, stems <= 1e-4;
- the int16 batch path equals one-clip calls; refusals queue nothing."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from oracle import dsp  # noqa: E402
from parity import record  # noqa: E402
import wiener_local_oracle as WL  # noqa: E402
from test_gpu_wiener import SPEC_BAR, STEM_BAR, rel, separator, stereo_clip, synthetic  # noqa: E402


def _run(ctx, X, S, K, W, F):
    from deepconvsep_b200.engine import wiener_stereo
    Sd = torch.tensor(S, device="cuda")
    wiener_stereo(ctx, torch.tensor(X, device="cuda"), Sd, K, num_bins=F, radius=W)
    torch.cuda.synchronize()
    return Sd.cpu().numpy()


@pytest.mark.parametrize("W", [1, 3])
@pytest.mark.parametrize("K", [1, 2, 3])
def test_spectra_match_the_oracle(K, W):
    from deepconvsep_b200.engine import Context
    T, F, ldf = 1900, 1025, 1032                          # 15 chunks, the last one of 108 frames
    X, S = synthetic(T, F, ldf, seed=10 * K + W, silent=list(range(700, 740)) + list(range(1880, 1900)))
    X[:, 384:512] *= 8.0                                  # a loud chunk: the window scales s_c differ
    S[:, 384:512] *= 8.0
    ctx = Context(0)
    n0 = ctx.launch_count()
    got = _run(ctx, X, S, K, W, F)
    assert ctx.launch_count() - n0 == 2 * K + 1            # init + reduce, then EM (+ reduce but for the last)
    want = WL.wiener_windowed(X[:, :, :F], S.reshape(4, 2, T, ldf)[:, :, :, :F], K, W).reshape(8, T, F)
    errs = [rel(got[p, :, :F], want[p]) for p in range(8)]
    record("wiener_local_spectra_K%d_W%d" % (K, W), max_rel=max(errs), per_plane=errs)
    assert max(errs) <= SPEC_BAR, errs
    assert np.array_equal(got[:, :, F:], S[:, :, F:])                         # pad bins untouched
    assert not got[:, 700:740, :F].any() and not got[:, 1880:, :F].any()     # all-zero frames stay zero
    whole = _run(ctx, X, S, K, 0, F)
    assert rel(got[:, :, :F], whole[:, :, :F]) > 1e-4                          # the windows matter
    assert np.array_equal(_run(ctx, X, S, K, W, F), got)                      # the same bits on a second run


@pytest.mark.parametrize("T", [1900, 128, 129])
def test_a_window_over_the_clip_is_byte_identical_to_the_whole_clip_filter(T):
    from deepconvsep_b200.engine import Context
    F, ldf = 513, 520
    X, S = synthetic(T, F, ldf, seed=T)
    n = -(-T // WL.CHUNK)
    ctx = Context(0)
    for K in (1, 2):
        whole = _run(ctx, X, S, K, 0, F)
        for W in (n - 1, n, 1000):
            if W >= 1:
                assert np.array_equal(_run(ctx, X, S, K, W, F).view(np.uint32), whole.view(np.uint32)), (K, W)


def _end_to_end(name, sep, audio, K, W):
    N, hop = sep.frame_size, sep.hop
    L = audio.shape[0]
    F = N // 2 + 1
    keep = sep.model.arch == "dsd"
    stems0, S0 = sep.separate_tapped(audio, keep_channels=keep)                                 # the network's spectra
    stems, S = sep.separate_tapped(audio, keep_channels=keep, wiener=K, wiener_radius=W)
    T = S0.shape[1]
    win = np.hanning(N)
    X = np.stack([dsp.stft_norm(audio[:, c], win, hop, N) for c in range(2)])
    want = WL.wiener_windowed(X, S0.reshape(4, 2, T, F), K, W)
    del S0
    spec_errs, stem_errs = [], []
    for j in range(4):
        for c in range(2):
            spec_errs.append(rel(S[2 * j + c], want[j, c]))
            y = dsp.istft_norm(want[j, c], win, hopsize=hop, nfft=N)[:L]
            stem_errs.append(float(np.linalg.norm(stems[:, j, c].astype(np.float64) - y) / np.linalg.norm(y)))
            assert rel(stems[:, j, c], stems0[:, j, c]) > 1e-3, (j, c)               # the filter moved it
    record(name, K=K, W=W, max_spec_rel=max(spec_errs), max_stem_rel=max(stem_errs), spec=spec_errs, stems=stem_errs)
    assert max(spec_errs) <= SPEC_BAR, spec_errs
    assert max(stem_errs) <= STEM_BAR, stem_errs
    return stems


def test_keep_channels_180s_n2048_matches_the_oracle():
    sep = separator("dsd", 2048, 2049)
    audio = stereo_clip(180.0, 600)
    stems = _end_to_end("wiener_local_keep_N2048_180s", sep, audio, 2, 2)
    assert np.array_equal(sep.separate_keep_channels(audio, wiener=2, wiener_radius=2), stems)
    assert not np.array_equal(sep.separate_keep_channels(audio, wiener=2), stems)


def test_stereo_net_15s_matches_the_oracle():
    sep = separator("dsd_ild", 1024, 77, patcher="util")
    _end_to_end("wiener_local_ild_N1024_15s", sep, stereo_clip(15.0, 4321), 2, 1)


def test_int16_batch_matches_one_clip_calls():
    sep = separator("dsd", 1024, 95)
    clips = [np.round(stereo_clip(sec, 900 + k) * 0.8 * 32767).astype(np.int16) for k, sec in enumerate((9.0, 4.1, 6.4))]
    got = sep.separate_pcm16_batch(clips, keep_channels=True, wiener=2, wiener_radius=1)
    for pcm, g in zip(clips, got):
        L = pcm.shape[0]
        assert g.shape == (4, L, 2) and g.dtype == np.int16
        assert np.array_equal(g, sep.separate_pcm16(pcm, keep_channels=True, wiener=2, wiener_radius=1))
        planes = torch.tensor(np.ascontiguousarray(pcm.T.astype(np.float32) / np.float32(32767)), device="cuda")
        stems = sep.separate_keep_channels(planes, wiener=2, wiener_radius=1).cpu().numpy()
        want = (stems * np.float32(32767)).astype(np.int16).reshape(4, 2, L).transpose(0, 2, 1)
        assert np.array_equal(g, want)
        assert not np.array_equal(g, sep.separate_pcm16(pcm, keep_channels=True, wiener=2))


def test_refusals_queue_nothing():
    from deepconvsep_b200 import _lib
    from deepconvsep_b200.engine import Context, _ptr
    ctx = Context(0)
    lib = ctx.lib
    T, ldf, F = 300, 520, 513
    X = torch.zeros((2, T, ldf), dtype=torch.complex64, device="cuda")
    S = torch.zeros((10, T, ldf), dtype=torch.complex64, device="cuda")

    def call(x=X, x_plane=T * ldf, s=S, src_stride=T * ldf, nsrc=4, t=T, ld=ldf, f=F, k=1, w=1):
        return lib.dcs_wiener_stereo_windowed(ctx.handle, _ptr(x), x_plane, _ptr(s), src_stride, nsrc, t, ld, f, k, w, None)
    refused = {
        "negative radius": lambda: call(w=-1),
        "negative iterations": lambda: call(k=-1),
        "nsrc > 4": lambda: call(nsrc=5),
        "source stride < T * ldf": lambda: call(src_stride=T * ldf - 8),
        "T = 0": lambda: call(t=0),
        "F > ldf": lambda: call(f=ldf + 1),
        "NULL spectra": lambda: call(s=None),
        "set_wiener_radius negative": lambda: lib.dcs_set_wiener_radius(ctx.handle, -1),
    }
    torch.cuda.synchronize()
    n0 = ctx.launch_count()
    for name, fn in refused.items():
        with pytest.raises(_lib.DcsError):
            _lib.check(fn())
        assert ctx.launch_count() == n0, name
    assert call(k=0) == 0 and ctx.launch_count() == n0                      # 0 iterations: nothing to do
    sep = separator("dsd", 1024, 7)
    audio = stereo_clip(1.0, 3)
    pcm = np.round(audio * 32767).astype(np.int16)
    n0 = sep.ctx.launch_count()
    for bad in (dict(wiener=0, wiener_radius=1), dict(wiener=1, wiener_radius=-1)):
        with pytest.raises(ValueError, match="--wiener-radius"):
            sep.separate_keep_channels(audio, **bad)
        with pytest.raises(ValueError, match="--wiener-radius"):
            sep.separate_pcm16(pcm, keep_channels=True, **bad)
        with pytest.raises(ValueError, match="--wiener-radius"):
            sep.separate_tapped(audio, keep_channels=True, **bad)
    with pytest.raises(ValueError):
        sep.separate_pcm16(pcm[:, 0], wiener_radius=1)
    assert sep.ctx.launch_count() == n0
