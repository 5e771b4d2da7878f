"""The float64 multichannel Wiener filter (oracle/wiener.py) without a GPU: against an independent per-bin loop that
solves each 2x2 system with np.linalg.solve, the equal-channel closed form, the identity sum_j y_j + delta s^2 C^-1 x = x,
K = 0, and the image SDR gain on panned sources that the filter exists for."""
import numpy as np
import pytest

from oracle import bsseval, dsp
from oracle import wiener as W


def spectra(T, F, nsrc=4, seed=0, scale=30.0, pans=(0.1, 0.35, 0.65, 0.9)):
    """sparse-ish sources panned (constant power) across the stereo field, X their sum, soft-mask initial stems from
    magnitudes perturbed by up to +80 %"""
    rng = np.random.default_rng(seed)
    src = (rng.standard_normal((nsrc, T, F)) + 1j * rng.standard_normal((nsrc, T, F))) \
        * rng.uniform(0.01, 1.0, (nsrc, 1, F)) * rng.gamma(0.3, 1.0, (nsrc, T, F))
    g = np.array([[np.cos(p * np.pi / 2), np.sin(p * np.pi / 2)] for p in pans[:nsrc]])
    img = g[:, :, None, None] * src[:, None]
    X = img.sum(axis=0) * scale
    mag = np.abs(img).sum(axis=1) * rng.uniform(1.0, 1.8, (nsrc, T, F))
    Y = (mag / np.maximum(mag.sum(axis=0), 1e-300))[:, None] * X[None]
    return X, Y, img * scale


def per_bin_loop(X, Y, iterations):
    """the same equations, one (t, f) at a time, with a 2x2 solve instead of the adjugate"""
    X = np.asarray(X, np.complex128)
    Y = np.array(Y, np.complex128)
    nsrc, _, T, F = Y.shape
    s = max(1.0, np.abs(X).max() / 10.0)
    for _ in range(iterations):
        R = np.zeros((nsrc, F, 2, 2), np.complex128)
        v = np.zeros((nsrc, T, F))
        for j in range(nsrc):
            for f in range(F):
                acc, vs = np.zeros((2, 2), np.complex128), 0.0
                for t in range(T):
                    y = Y[j, :, t, f]
                    v[j, t, f] = 0.5 * np.vdot(y, y).real
                    acc += np.outer(y, y.conj())
                    vs += v[j, t, f]
                R[j, f] = acc / (W.EPS * s * s + vs)
        out = np.empty_like(Y)
        for t in range(T):
            for f in range(F):
                C = sum(v[j, t, f] * R[j, f] for j in range(nsrc)) + W.DELTA * s * s * np.eye(2)
                z = np.linalg.solve(C, X[:, t, f])
                for j in range(nsrc):
                    out[j, :, t, f] = v[j, t, f] * (R[j, f] @ z)
        Y = out
    return Y


def rel(a, b):
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


@pytest.mark.parametrize("K", [1, 2, 3])
def test_matches_a_per_bin_solve(K):
    X, Y, _ = spectra(24, 9, seed=K)
    got = W.wiener(X, Y, K)
    want = per_bin_loop(X, Y, K)
    for j in range(4):
        for c in range(2):
            assert rel(got[j, c], want[j, c]) < 1e-10, (j, c)


def test_zero_iterations_return_the_input():
    X, Y, _ = spectra(10, 7)
    assert np.array_equal(W.wiener(X, Y, 0), Y)


def test_sources_and_residual_add_up_to_the_mixture():
    X, Y, _ = spectra(40, 33, seed=3)
    s = W.mixture_scale(X)
    for _ in range(2):
        Yn = W.em_step(X, Y, s)
        total = Yn.sum(axis=0) + W.residual(X, Y, s)
        assert np.abs(total - X).max() <= 1e-9 * np.abs(X).max()
        Y = Yn


def test_equal_channels_give_the_closed_form():
    """l == r: y_jc = x_c rho_j v_j / (sum_k rho_k v_k + delta s^2 / 2), rho_j = A_j / (eps s^2 + A_j), A_j = sum_t v_j"""
    X, Y, _ = spectra(50, 17, seed=4)
    X = np.stack([X[0], X[0]])
    Y = np.stack([Y[:, 0], Y[:, 0]], axis=1)
    s = W.mixture_scale(X)
    v = np.abs(Y[:, 0]) ** 2
    A = v.sum(axis=1, keepdims=True)
    rho = A / (W.EPS * s * s + A)
    want = X[0] * rho * v / ((rho * v).sum(axis=0) + W.DELTA * s * s / 2)
    got = W.wiener(X, Y, 1)
    for j in range(4):
        assert rel(got[j, 1], got[j, 0]) < 1e-14
        assert rel(got[j, 0], want[j]) < 1e-11


def test_silent_frames_stay_silent_and_are_finite():
    X, Y, _ = spectra(30, 11, seed=5)
    Y[:, :, 20:] = 0
    got = W.wiener(X, Y, 3)
    assert np.isfinite(got).all() and not got[:, :, 20:].any()


def test_one_iteration_raises_the_image_sdr_of_panned_sources():
    """4 sources at 0.1 / 0.35 / 0.65 / 0.9 of the stereo field, soft masks from magnitudes perturbed by up to +80 %:
    one mask per source cannot give each source its own stereo image, the spatial covariances can"""
    N, hop, L = 512, 256, 12000
    rng = np.random.default_rng(11)
    win = np.hanning(N)
    src = []
    for j in range(4):                   # gated noise with its own spectral tilt and gating
        x = np.convolve(rng.standard_normal(L), rng.standard_normal(8 + 6 * j) / (1 + j), mode="same")
        src.append(x * (rng.uniform(size=L // 1000 + 1).repeat(1000)[:L] > 0.3))
    pans = (0.1, 0.35, 0.65, 0.9)
    img = np.array([[np.cos(p * np.pi / 2) * s, np.sin(p * np.pi / 2) * s] for p, s in zip(pans, src)]) * 0.2
    mix = img.sum(axis=0)
    X = np.stack([dsp.stft_norm(mix[c], win, hop, N) for c in range(2)])
    S = np.array([[dsp.stft_norm(img[j, c], win, hop, N) for c in range(2)] for j in range(4)])
    mag = np.abs(S).sum(axis=1) * rng.uniform(1.0, 1.8, (4,) + X.shape[1:])
    Y = (mag / np.maximum(mag.sum(axis=0), 1e-300))[:, None] * X[None]

    def sdr(Ys):
        est = np.array([[dsp.istft_norm(Ys[j, c], win, hopsize=hop, nfft=N)[:L] for c in range(2)] for j in range(4)])
        return float(np.mean(bsseval.bss_eval_images(est, img, flen=64)[0]))
    before, after = sdr(Y), sdr(W.wiener(X, Y, 1))
    assert after > before + 1.0, (before, after)
