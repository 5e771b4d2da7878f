"""Float64 C-channel Wiener filter (TEST INFRASTRUCTURE: the estimator of dcs_wiener_channels, include/dcs.h).

X complex [C, T, F] (the mixture's channels), Y complex [nsrc, C, T, F] (the stems, (source, channel)).  Per iteration,
with eps, delta and the chunks of oracle.wiener / wiener_local_oracle:

    v_j(t,f) = (1/C) sum_c |y_jc|^2
    R_j(f)   = sum_t y_j y_j^H / (eps s^2 + sum_t v_j)        (radius W >= 1: sums and s over chunk c's window)
    C(t,f)   = sum_j v_j R_j + delta s^2 I
    y_j      <- v_j R_j C^-1 x

solved batched over [t, f] with numpy's LU solve, one chunk of frames at a time (so a 180 s clip fits in memory).  At
C = 2 this is oracle.wiener.wiener (radius 0) and wiener_local_oracle.wiener_windowed (radius >= 1)."""
import numpy as np

from oracle import wiener as W
from wiener_local_oracle import CHUNK, window

EPS, DELTA = W.EPS, W.DELTA


def _chunk_sums(Y):
    """Y [nsrc, C, T, F] -> P [n, nsrc, C, C, F]: sum over each chunk's frames of y_j y_j^H"""
    T = Y.shape[2]
    n = -(-T // CHUNK)
    return np.stack([np.einsum("jatf,jbtf->jabf", Y[:, :, k * CHUNK:(k + 1) * CHUNK],
                               Y[:, :, k * CHUNK:(k + 1) * CHUNK].conj()) for k in range(n)])


def _scales(X, radius):
    """s per chunk [n] (radius 0: the clip's s in every chunk)"""
    T = X.shape[1]
    n = -(-T // CHUNK)
    if radius == 0:
        return np.full(n, W.mixture_scale(X))
    pmax = np.array([np.abs(X[:, k * CHUNK:(k + 1) * CHUNK]).max() for k in range(n)])
    return np.array([max(1.0, float(max(pmax[k] for k in window(c, n, radius))) / 10.0) for c in range(n)])


def _covariances(Y, s, radius):
    """R_j per chunk [n, nsrc, C, C, F] from the chunk sums over each chunk's window (radius 0: the whole clip)"""
    P = _chunk_sums(Y)
    n, C = P.shape[0], Y.shape[1]
    if radius == 0:
        win = np.broadcast_to(P.sum(axis=0), P.shape)
    else:
        win = np.stack([sum(P[k] for k in window(c, n, radius)) for c in range(n)])
    tr = np.einsum("njaaf->njf", win).real / C
    den = EPS * (s * s)[:, None, None] + tr                            # [n, nsrc, F]
    return win / den[:, :, None, None, :]


def _solve(X, Y, s, R, d_only=False):
    """per chunk: z = C^-1 x and y_j = v_j R_j z (d_only: delta s^2 z, the residual)"""
    nsrc, C, T, F = Y.shape
    out = np.empty((C, T, F) if d_only else Y.shape, dtype=np.complex128)
    eye = np.eye(C)
    for k in range(R.shape[0]):
        sl = slice(k * CHUNK, min(T, (k + 1) * CHUNK))
        v = (np.abs(Y[:, :, sl]) ** 2).sum(axis=1) / C                  # [nsrc, t, F]
        d = DELTA * s[k] * s[k]
        Cm = np.einsum("jtf,jabf->tfab", v, R[k]) + d * eye             # [t, F, C, C]
        x = np.moveaxis(X[:, sl], 0, -1)[..., None]                     # [t, F, C, 1]
        z = np.linalg.solve(Cm, x)[..., 0]                              # [t, F, C]
        if d_only:
            out[:, sl] = np.moveaxis(d * z, -1, 0)
        else:
            out[:, :, sl] = v[:, None] * np.einsum("jabf,tfb->jatf", R[k], z)
    return out


def em_step(X, Y, s, radius=0):
    """one iteration; s per chunk from _scales"""
    return _solve(X, Y, s, _covariances(Y, s, radius))


def residual(X, Y_prev, radius=0):
    """delta s^2 C^-1 x [C, T, F] for the C built from Y_prev: sum_j em_step(X, Y_prev)[j] + residual = x"""
    X = np.asarray(X, dtype=np.complex128)
    Y = np.asarray(Y_prev, dtype=np.complex128)
    s = _scales(X, radius)
    return _solve(X, Y, s, _covariances(Y, s, radius), d_only=True)


def wiener(X, Y, iterations, radius=0):
    """X [C, T, F], Y [nsrc, C, T, F] -> the stems after `iterations` EM iterations, complex128"""
    X = np.asarray(X, dtype=np.complex128)
    Y = np.array(Y, dtype=np.complex128)
    if X.ndim != 3 or Y.ndim != 4 or Y.shape[1:] != X.shape:
        raise ValueError("X must be [C, T, F] and Y [nsrc, C, T, F], got %r and %r" % (X.shape, Y.shape))
    s = _scales(X, radius)
    for _ in range(int(iterations)):
        Y = em_step(X, Y, s, radius)
    return Y


def equal_channels(a, b, C, iterations):
    """The closed form with every channel equal to a [T, F] and the stems of every channel b [nsrc, T, F] (radius 0):
    R_j = rho_j J, rho_j = sum_t |b_j|^2 / (eps s^2 + sum_t |b_j|^2), and each channel's output is
    v_j rho_j C a / (C sum_k v_k rho_k + delta s^2).  Returns the stems [nsrc, T, F] (the same on every channel)."""
    a = np.asarray(a, dtype=np.complex128)
    y = np.array(b, dtype=np.complex128)
    s = max(1.0, float(np.abs(a).max()) / 10.0)
    for _ in range(int(iterations)):
        v = np.abs(y) ** 2
        A = v.sum(axis=1, keepdims=True)
        rho = A / (EPS * s * s + A)
        y = v * rho * C * a[None] / (C * (v * rho).sum(axis=0) + DELTA * s * s)
    return y
