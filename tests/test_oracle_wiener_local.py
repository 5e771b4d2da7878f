"""The float64 sliding-window Wiener filter (tests/wiener_local_oracle.py) without a GPU: a window covering the clip is
the whole-clip filter, it agrees with a literal chunk-by-chunk restatement, and a chunk's output depends on exactly the
frames within K * W chunks of it."""
import numpy as np
import pytest

from oracle import wiener as W
import wiener_local_oracle as WL
from test_oracle_wiener import spectra


def rel(a, b):
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def literal(X, Y, iterations, radius):
    """chunk by chunk: the whole-clip formulas of oracle/wiener.py applied to the window's frames, and the result kept
    for the chunk's own frames"""
    X = np.asarray(X, np.complex128)
    Y = np.array(Y, np.complex128)
    T = X.shape[1]
    n = -(-T // WL.CHUNK)
    frames = [slice(c * WL.CHUNK, min(T, (c + 1) * WL.CHUNK)) for c in range(n)]
    for _ in range(iterations):
        out = np.empty_like(Y)
        for c in range(n):
            win = list(WL.window(c, n, radius))
            span = slice(frames[win[0]].start, frames[win[-1]].stop)
            s = W.mixture_scale(X[:, span])
            _, R = W.spatial_covariances(Y[:, :, span], s)
            Yc = Y[:, :, frames[c]]
            v = 0.5 * (np.abs(Yc[:, 0]) ** 2 + np.abs(Yc[:, 1]) ** 2)
            c00, c11, c01, det = W.mixture_covariance(v, R, s)
            Xc = X[:, frames[c]]
            z0 = (c11 * Xc[0] - c01 * Xc[1]) / det
            z1 = (c00 * Xc[1] - c01.conj() * Xc[0]) / det
            r00, r11, r01 = R
            for j in range(Y.shape[0]):
                out[j, 0, frames[c]] = v[j] * (r00[j][None] * z0 + r01[j][None] * z1)
                out[j, 1, frames[c]] = v[j] * (r01[j].conj()[None] * z0 + r11[j][None] * z1)
        Y = out
    return Y


@pytest.mark.parametrize("T,radius", [(700, 5), (700, 6), (700, 40), (128, 1), (257, 2)])
def test_a_window_over_the_whole_clip_is_the_whole_clip_filter(T, radius):
    """W >= n - 1: every chunk's window is the clip (numpy's pairwise sums differ from the chunked ones in order)"""
    assert radius >= -(-T // WL.CHUNK) - 1
    X, Y, _ = spectra(T, 9, seed=T + radius)
    Y[:, :, 300:330] = 0
    for K in (1, 2):
        got, want = WL.wiener_windowed(X, Y, K, radius), W.wiener(X, Y, K)
        assert rel(got, want) <= 1e-13, (K, rel(got, want))
        assert not got[:, :, 300:330].any()


@pytest.mark.parametrize("K,radius", [(1, 1), (2, 1), (3, 2)])
def test_matches_a_literal_per_chunk_restatement(K, radius):
    X, Y, _ = spectra(1000, 7, seed=10 * K + radius)
    X[:, 256:384] *= 40.0                             # one loud chunk: the scales s_c differ between windows
    got = WL.wiener_windowed(X, Y, K, radius)
    want = literal(X, Y, K, radius)
    assert rel(got, want) <= 1e-12
    assert rel(got, W.wiener(X, Y, K)) > 1e-3          # and the windows matter


def test_zero_radius_is_the_whole_clip_filter():
    X, Y, _ = spectra(300, 5, seed=2)
    assert np.array_equal(WL.wiener_windowed(X, Y, 2, 0), W.wiener(X, Y, 2))


@pytest.mark.parametrize("K,radius", [(1, 1), (2, 1), (1, 3), (2, 2)])
def test_a_chunk_depends_on_exactly_its_k_w_neighbourhood(K, radius):
    """changing one frame (mixture and stems) outside chunk c's K * W chunks leaves chunk c's output bits unchanged;
    changing one just inside changes them"""
    n, c = 14, 7
    X, Y, _ = spectra(n * WL.CHUNK - 50, 6, seed=K + 7 * radius)
    base = WL.wiener_windowed(X, Y, K, radius)
    own = slice(c * WL.CHUNK, (c + 1) * WL.CHUNK)
    reach = K * radius
    first_out, last_out = (c - reach) * WL.CHUNK - 1, (c + reach + 1) * WL.CHUNK
    first_in, last_in = first_out + 1, last_out - 1
    for t, inside in ((first_out, False), (last_out, False), (first_in, True), (last_in, True)):
        X2, Y2 = X.copy(), Y.copy()
        X2[:, t] *= 3.0
        Y2[:, :, t] *= 1.7 - 0.4j
        got = WL.wiener_windowed(X2, Y2, K, radius)
        same = np.array_equal(got[:, :, own], base[:, :, own])
        assert same != inside, (t, inside)
