"""Float64 sliding-window Wiener filter (TEST INFRASTRUCTURE: built on oracle/wiener.py).

The estimator of dcs_wiener_stereo_windowed (include/dcs.h): chunk k is frames [128k, min(T, 128k + 128)), n chunks;
radius W >= 1 gives chunk c the window of chunks max(0, c-W) .. min(n-1, c+W), and every frame of chunk c uses

    s_c       = max(1, max |x| over the window's frames / 10)
    R_j(f; c) = sum_{t in window} y_j y_j^H / (eps s_c^2 + sum_{t in window} v_j)
    C(t, f)   = sum_j v_j R_j(f; c) + delta s_c^2 I,   y_j <- v_j R_j(f; c) C^-1 x

with eps, delta and v_j as in oracle.wiener.  The sums over time are per-chunk sums added over the window in ascending
chunk order, so a chunk's result is a function of its window alone, computed by the same operations wherever the
window sits (a segment of a longer clip holding the window gives the same bits).  radius 0 is oracle.wiener.wiener."""
import numpy as np

from oracle import wiener as W

CHUNK = 128


def chunk_of_frames(T):
    return np.arange(T) // CHUNK


def window(c, n, radius):
    """the chunks of chunk c's window"""
    return range(max(0, c - radius), min(n - 1, c + radius) + 1)


def _per_chunk(a, T):
    """a [..., T, F] -> the sums over each chunk's frames [..., n, F] (frame order within a chunk)"""
    n = -(-T // CHUNK)
    pad = np.zeros(a.shape[:-2] + (n * CHUNK - T, a.shape[-1]), dtype=a.dtype)
    b = np.concatenate([a, pad], axis=-2).reshape(a.shape[:-2] + (n, CHUNK, a.shape[-1]))
    return b.sum(axis=-2)


def _window_sums(P, radius):
    """P [..., n, F] per-chunk sums -> [..., n, F]: for each chunk the direct sum over its window, ascending"""
    n = P.shape[-2]
    out = np.zeros_like(P)
    for c in range(n):
        acc = np.zeros_like(P[..., 0, :])
        for k in window(c, n, radius):
            acc = acc + P[..., k, :]
        out[..., c, :] = acc
    return out


def chunk_scales(X, radius):
    """X [2, T, F] -> s_c per chunk [n]"""
    T = X.shape[1]
    n = -(-T // CHUNK)
    pmax = np.array([np.abs(X[:, c * CHUNK:(c + 1) * CHUNK]).max() for c in range(n)])
    return np.array([max(1.0, float(max(pmax[k] for k in window(c, n, radius))) / 10.0) for c in range(n)])


def em_step_windowed(X, Y, s_chunk, radius):
    """one iteration with the windowed covariances; s_chunk [n] from chunk_scales"""
    nsrc, _, T, F = Y.shape
    idx = chunk_of_frames(T)
    v = 0.5 * (np.abs(Y[:, 0]) ** 2 + np.abs(Y[:, 1]) ** 2)
    P00 = _window_sums(_per_chunk(np.abs(Y[:, 0]) ** 2, T), radius)
    P11 = _window_sums(_per_chunk(np.abs(Y[:, 1]) ** 2, T), radius)
    P01 = _window_sums(_per_chunk(Y[:, 0] * Y[:, 1].conj(), T), radius)
    s2 = (s_chunk * s_chunk)[:, None]                                  # [n, 1]
    den = W.EPS * s2 + 0.5 * (P00 + P11)                               # [nsrc, n, F]
    r00, r11, r01 = (P00 / den)[:, idx], (P11 / den)[:, idx], (P01 / den)[:, idx]    # per frame [nsrc, T, F]
    d = (W.DELTA * s2)[idx]                                            # [T, 1]
    c00 = (v * r00).sum(axis=0) + d
    c11 = (v * r11).sum(axis=0) + d
    c01 = (v * r01).sum(axis=0)
    det = c00 * c11 - np.abs(c01) ** 2
    z0 = (c11 * X[0] - c01 * X[1]) / det
    z1 = (c00 * X[1] - c01.conj() * X[0]) / det
    out = np.empty_like(Y)
    for j in range(nsrc):
        out[j, 0] = v[j] * (r00[j] * z0 + r01[j] * z1)
        out[j, 1] = v[j] * (r01[j].conj() * z0 + r11[j] * z1)
    return out


def wiener_windowed(X, Y, iterations, radius):
    """X [2, T, F], Y [nsrc, 2, T, F] -> the stems after `iterations` EM iterations with covariance windows of
    `radius` chunks, complex128 (radius 0: oracle.wiener.wiener)"""
    if radius == 0:
        return W.wiener(X, Y, iterations)
    X = np.asarray(X, dtype=np.complex128)
    Y = np.array(Y, dtype=np.complex128)
    if X.ndim != 3 or X.shape[0] != 2 or Y.ndim != 4 or Y.shape[1:] != X.shape:
        raise ValueError("X must be [2, T, F] and Y [nsrc, 2, T, F], got %r and %r" % (X.shape, Y.shape))
    s = chunk_scales(X, radius)
    for _ in range(int(iterations)):
        Y = em_step_windowed(X, Y, s, radius)
    return Y
