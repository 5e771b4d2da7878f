"""Stereo stems of one ~120 s recording cut into 3 segments over 2 contexts (deepconvsep_b200.longclip) with the
sliding-window Wiener post-filter (K = 2, W = 2), keep-channels on the DSD100 network and the stereo / ILD network:

- against the float64 oracle (network, sliding-window filter, iSTFT) at the north-star 1e-4 per stem; the oracle's
  Wiener input follows tests/parity.py: the network's spectra in float64, with the device's values adopted at the bins
  the oracle flags on the soft mask's discontinuity, and only there;
- against the whole-clip device call with the same radius.  The two runs differ in the last float32 bits of the
  network (the GEMMs' K split depends on the patch count), and a bin on the soft mask's discontinuity may take the
  other branch in either run; through the covariance windows such a bin moves its whole window at that frequency by a
  little, so over all samples the bar is the north-star one, and on the samples no flagged frame reaches through the
  inverse STFT it is 1e-5;
- one context run sequentially gives the threaded result bit for bit."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from oracle import dsp, pipeline  # noqa: E402
from parity import record, TOL  # noqa: E402
import channels_oracle as co  # noqa: E402
import wiener_local_oracle as WL  # noqa: E402
from test_gpu_wiener import separator, stereo_clip  # noqa: E402

K, W = 2, 2


def oracle_spectra(sep, audio):
    """the network's spectra in float64 [4, 2, T, F] and the flagged bins [2, T, F]"""
    N, H = sep.frame_size, sep.hop
    if sep.model.arch == "dsd":
        _, _, phs, mms, _, kmap = co.separate_channels(audio, sep._params, frameSize=N, hopSize=H, overlap=sep.overlap)
        kmaps = np.stack([kmap, kmap])
    else:
        _, _, phs, mms = pipeline.separate_stereo(audio, sep._params, frameSize=N, hopSize=H, overlap=sep.overlap,
                                                  count_kinks=True, return_spec=True)
        kmaps = pipeline.separate_stereo.last_kink_map
    T = phs[0].shape[0]
    S = np.stack([[mms[c][j, :T] / 0.3 * np.sqrt(N) * np.exp(1j * phs[c]) for c in range(2)] for j in range(4)])
    return S, kmaps


@pytest.mark.parametrize("arch,seed", [("dsd", 1201), ("dsd_ild", 1301)])
def test_stitched_stereo_stems_match_the_oracle_and_the_whole_clip(arch, seed):
    from deepconvsep_b200 import longclip
    from oracle import nets
    N = 1024
    seps = [separator(arch, N, seed, patcher="util" if arch == "dsd_ild" else "standalone") for _ in range(2)]
    for s in seps:
        s._params = nets.make_synthetic_params(arch, N // 2 + 1, seed=seed)
    sep = seps[0]
    keep = arch == "dsd"
    audio = stereo_clip(120.0, seed)
    L = audio.shape[0]
    segs = longclip.plan_segments(L, 3, N, sep.hop, sep.model.tc, sep.overlap, wiener_reach=K * W)
    assert len(segs) == 3
    got = longclip.separate_long(seps, audio, parts=3, keep_channels=keep, wiener=K, wiener_radius=W)
    assert got.shape == (L, 4, 2)
    seq = longclip.separate_long(seps[1], audio, parts=3, keep_channels=keep, wiener=K, wiener_radius=W)
    assert np.array_equal(seq, got)                                       # one context, sequential: the same bits

    whole, _ = sep.separate_tapped(audio, keep_channels=keep, wiener=K, wiener_radius=W)
    _, S_dev = sep.separate_tapped(audio, keep_channels=keep)                   # the device's network spectra
    S_or, kmaps = oracle_spectra(sep, audio)
    T, F = S_or.shape[2], S_or.shape[3]
    nflag = int(kmaps.sum())
    assert nflag <= 1e-4 * kmaps.size + 8
    for j in range(4):
        for c in range(2):
            S_or[j, c][kmaps[c]] = S_dev[2 * j + c][kmaps[c]]
    del S_dev
    win = np.hanning(N)
    X = np.stack([dsp.stft_norm(audio[:, c], win, sep.hop, N) for c in range(2)])
    Y = WL.wiener_windowed(X, S_or, K, W)
    del S_or
    away = np.ones(L, dtype=bool)                         # samples no flagged frame reaches through the iSTFT
    for f in np.nonzero(kmaps.any(axis=(0, 2)))[0]:
        away[max(0, (f - 1) * sep.hop - N // 2):(f + 1) * sep.hop + N // 2] = False
    errs, whole_errs, away_errs = [], [], []
    for j in range(4):
        for c in range(2):
            y = dsp.istft_norm(Y[j, c], win, hopsize=sep.hop, nfft=N)[:L]
            g = got[:, j, c].astype(np.float64)
            errs.append(float(np.linalg.norm(g - y) / np.linalg.norm(y)))
            w = whole[:, j, c].astype(np.float64)
            whole_errs.append(float(np.linalg.norm(g - w) / np.linalg.norm(w)))
            away_errs.append(float(np.linalg.norm((g - w)[away]) / np.linalg.norm(w[away])))
    record("longclip_stereo_%s_120s_K%d_W%d" % (arch, K, W), flagged_bins=nflag, rel_l2=errs, rel_l2_vs_whole=whole_errs,
           rel_l2_vs_whole_away_from_flagged=away_errs, away_fraction=float(away.mean()), segments=[tuple(s) for s in segs])
    assert max(errs) <= TOL, errs
    assert max(whole_errs) <= TOL, whole_errs
    assert max(away_errs) <= 1e-5, away_errs
