"""Multichannel Wiener filter with EM re-estimation of each source's spatial covariance, float64.

The reference set out to write this filter in `util.mwf` (util.py:633-719) and left it unfinished: the loop stops at a
`pdb.set_trace()` (:718) and its R update (:719) divides by the wrong shape.  The commented MATLAB block at
util.py:647-682 is the EM of Duong, Vincent & Gribonval (2010).  This is the form libdcs implements
(csrc/wiener.cu, dcs_wiener_stereo), with norbert's mixture scaling written as scaled constants:

    eps = 2^-23, delta = sqrt(eps), s = max(1, max_{t,f,c} |x| / 10)
    v_j(t,f) = (|y_jL|^2 + |y_jR|^2) / 2
    R_j(f)   = sum_t y_j y_j^H / (eps s^2 + sum_t v_j)
    C(t,f)   = sum_j v_j R_j + delta s^2 I
    y_j      <- v_j R_j C^-1 x

Shapes: X complex [2, T, F] (the mixture's channels), Y complex [nsrc, 2, T, F] (the stems, (source, channel)).
The 2x2 algebra is written out by components, so a 180 s clip fits in memory."""
import numpy as np

EPS = 2.0 ** -23
DELTA = np.sqrt(EPS)


def mixture_scale(X):
    return max(1.0, float(np.abs(np.asarray(X)).max()) / 10.0)


def spatial_covariances(Y, s):
    """Y [nsrc, 2, T, F] -> v [nsrc, T, F] and R_j(f) as (R00, R11, R01) each [nsrc, F] (R10 = conj(R01))"""
    v = 0.5 * (np.abs(Y[:, 0]) ** 2 + np.abs(Y[:, 1]) ** 2)
    den = EPS * s * s + v.sum(axis=1)
    r00 = (np.abs(Y[:, 0]) ** 2).sum(axis=1) / den
    r11 = (np.abs(Y[:, 1]) ** 2).sum(axis=1) / den
    r01 = (Y[:, 0] * Y[:, 1].conj()).sum(axis=1) / den
    return v, (r00, r11, r01)


def mixture_covariance(v, R, s):
    """C = sum_j v_j R_j + delta s^2 I as (C00, C11, C01) each [T, F], and det C"""
    r00, r11, r01 = R
    d = DELTA * s * s
    c00 = np.einsum("jtf,jf->tf", v, r00) + d
    c11 = np.einsum("jtf,jf->tf", v, r11) + d
    c01 = np.einsum("jtf,jf->tf", v, r01)
    return c00, c11, c01, c00 * c11 - np.abs(c01) ** 2


def em_step(X, Y, s):
    """one iteration: the stems y_j -> v_j R_j C^-1 x"""
    v, R = spatial_covariances(Y, s)
    r00, r11, r01 = R
    c00, c11, c01, det = mixture_covariance(v, R, s)
    z0 = (c11 * X[0] - c01 * X[1]) / det
    z1 = (c00 * X[1] - c01.conj() * X[0]) / det
    out = np.empty_like(Y)
    for j in range(Y.shape[0]):
        out[j, 0] = v[j] * (r00[j] * z0 + r01[j] * z1)
        out[j, 1] = v[j] * (r01[j].conj() * z0 + r11[j] * z1)
    return out


def wiener(X, Y, iterations):
    """X [2, T, F], Y [nsrc, 2, T, F] -> the stems after `iterations` EM iterations, complex128 (0: Y itself)"""
    X = np.asarray(X, dtype=np.complex128)
    Y = np.array(Y, dtype=np.complex128)
    if X.ndim != 3 or X.shape[0] != 2 or Y.ndim != 4 or Y.shape[1:] != X.shape:
        raise ValueError("X must be [2, T, F] and Y [nsrc, 2, T, F], got %r and %r" % (X.shape, Y.shape))
    s = mixture_scale(X)
    for _ in range(int(iterations)):
        Y = em_step(X, Y, s)
    return Y


def residual(X, Y_prev, s):
    """delta s^2 C^-1 x for the C built from Y_prev: the part of x no source takes, so that
    sum_j em_step(X, Y_prev, s)[j] + residual(X, Y_prev, s) = x"""
    X = np.asarray(X, dtype=np.complex128)
    v, R = spatial_covariances(np.asarray(Y_prev, dtype=np.complex128), s)
    c00, c11, c01, det = mixture_covariance(v, R, s)
    d = DELTA * s * s
    return np.stack([d * (c11 * X[0] - c01 * X[1]) / det, d * (c00 * X[1] - c01.conj() * X[0]) / det])
