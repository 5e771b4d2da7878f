"""Element-wise bound for one EM iteration of the Wiener post-filter (TEST INFRASTRUCTURE: csrc/wiener.cu against
wiener_channels_oracle.em_step, one iteration at a time, every output component on its own).

One iteration maps the fp32 stems Y [nsrc, nx, T, F] and the fp32 mixture X [nx, T, F] to new fp32 stems.  The device
reads the stems it stored in the previous iteration and nothing else (the scale comes from X again), so checking each
iteration against the float64 step fed the device's own previous stems compares element by element however many
iterations run.

The bound.  Let y be the exact step (em_step: complex128), y^ the device's fp64 value before its store, and
dev = fl32(y^) rounded once per real and imaginary component.  Round to nearest gives |dev - y^| <= 2^-24 |y^| in the
normal range and <= 2^-150 below it, so per component

    |dev - y| <= 2^-24 |y| + 2^-149 + (1 + 2^-24) |y^ - y|.

The fp64 error |y^ - y|, to first order in u = 2^-53, for source j and channel c, with n_w the frames of the
covariance window (T at radius 0) and R, z, C of that frame's chunk:

(a) sums: Q = sum_t y y^H is per-chunk partials added in chunk order, one rounding per frame and per chunk, so
    |dQ_ab| <= n_w u sum_t |y_a| |y_b| <= n_w u sqrt(Q_aa Q_bb) (Cauchy-Schwarz); den = eps s^2 + tr Q / nx adds
    (nx + 3) u relatively, hence |dR_ab| <= (2 n_w + nx + 4) u sqrt(R_aa R_bb) and ||dR_j||_F <= (2 n_w + nx + 4) u tr R_j.
    The bound on an off-diagonal entry is sqrt(R_aa R_bb), not |R_ab|: the exact R_ab may cancel to 0.
(b) C = sum_j v_j R_j + delta s^2 I, v_j from nx + 1 operations, nsrc fmas per entry: with sum_j v_j tr R_j <= tr C <=
    nx ||C||_2, ||dC||_2 <= nx (2 n_w + 2 nx + nsrc + 6) u ||C||_2.
(c) solve: the 2 x 2 adjugate, and L D L^H of a Hermitian positive definite matrix without pivoting (D >= delta s^2 > 0),
    are backward stable, (C + E) z^ = x with ||E||_2 <= 3 nx (nx + 1) u ||C||_2 in complex arithmetic; with (b),
    ||z^ - z||_2 <= kappa_2(C) (||dC||_2 + ||E||_2) / ||C||_2 ||z||_2.
(d) y_jc = v_j (R_j z)_c: a row of a positive semidefinite matrix has ||R_j[c, :]||_2 <= sqrt(R_j,cc tr R_j), so the
    errors of z, of R_j and of the nx + 2 operations of the product are all at most
    v_j sqrt(R_j,cc tr R_j) ||z||_2 times their factor.  The error of z is bounded in norm only: a component of z much
    smaller than ||z|| can carry an error of size kappa u ||z||, which is why the envelope is not (|R_j| |z|)_c.

For nx >= 2 and nsrc <= 4 the factors of (a) to (d) add up to at most 14 (nx n_w + nx^2).  The reference's own float64
evaluation (the same sums, LU with partial pivoting, also backward stable) errs by as much again, so c = 32 and

    |dev - ref| <= 2^-24 |ref| + 2^-149 + 32 * 2^-53 * (nx n_w + nx^2) * kappa_2(C(t,f)) * v_j sqrt(R_j,cc tr R_j) ||z||_2

per real and per imaginary component, kappa_2 computed here in float64.  The fp64 term matters where C is nearly
singular or the component is small next to the frame's other stems; `check` reports the fraction of components where
it exceeds the fp32 term.

This module also holds the case generator of the element tests, a float64 emulation of the device's plan (per-chunk
partials in frame order, window sums in ascending chunk order, the adjugate at nx = 2 and L D L^H without pivoting
above, round to fp32 per component), and the mutants of that plan the bound must reject."""
import numpy as np

import wiener_channels_oracle as wco
from wiener_local_oracle import CHUNK, window

EPS, DELTA = wco.EPS, wco.DELTA
U32, U64, TINY = 2.0 ** -24, 2.0 ** -53, 2.0 ** -149
C_BOUND = 32.0

MUTANTS = ("fp32_algebra", "s_for_s2", "prev_chunk_R_first_frame", "clip_scale", "drop_last_frame", "pair_conjugate",
           "v_from_channel0")


# ---------------------------------------------------------------------------------------------- cases
def nchunks(T):
    return -(-T // CHUNK)


# (nx, nsrc, T, F, radius): every nx in 2..8 x nsrc in 1..4 at radius 0 and 1 on 300 frames (chunks of 128, 128 and
# 44) and 129 bins, one radius covering the clip, then the shape edges: T around one chunk, F around the C-channel
# kernels' tiles of 32 bins and the stereo kernels' tiles of 128
MATRIX = [(nx, nsrc, 300, 129, radius) for nx in range(2, 9) for nsrc in range(1, 5) for radius in (0, 1)] \
    + [(5, 3, 300, 129, 2)]
EDGES = [(nx, nsrc, T, F, 1) for T in (1, 127, 128, 129) for nx, nsrc, F in ((2, 3, 129), (6, 2, 33))] \
    + [(nx, nsrc, 300, F, radius) for F in (1, 31, 32, 33) for nx, nsrc, radius in ((3, 4, 1), (8, 1, 0))] \
    + [(2, nsrc, 300, F, radius) for F in (127, 128, 129) for nsrc, radius in ((2, 0), (4, 1))]
CASES = MATRIX + EDGES


def case_id(c):
    return "nx%d-nsrc%d-T%d-F%d-W%d" % c


def make_case(c):
    """the spectra of one entry of CASES, seeded by the entry"""
    nx, nsrc, T, F, radius = c
    return case(nx, nsrc, T, F, seed=[nx, nsrc, T, F, radius])


def case(nx, nsrc, T, F, seed):
    """X [nx, T, F] and stems Y [nsrc, nx, T, F], complex128 holding fp32 values: nsrc sources with their own gain and
    delay per channel (complex off-diagonal covariances) and soft-mask stems, with these features by bin class f % 8
    (where F reaches them) and by frame:
      1: source 0 silent in the bin;           2: x = 0, the stems not;           3: every channel equal (rank-one C);
      4: source 0 60 dB above the rest;        5-7: gains from fp32 subnormals up to the loud end (~1e4);
      frames t % 50 == 17 (not the last frame): every stem 0;  chunk 1 (n >= 2): the last source silent;
      n >= 3: chunks 0 .. n-2 quiet (max |x| = 5: a radius-1 window with s = 1), chunk n-1 at max |x| = 1e4."""
    rng = np.random.default_rng(seed)
    n = nchunks(T)
    f = np.arange(F)
    src = (rng.standard_normal((nsrc, T, F)) + 1j * rng.standard_normal((nsrc, T, F))) \
        * rng.uniform(0.2, 1.0, (nsrc, 1, F)) * rng.gamma(0.3, 1.0, (nsrc, T, F))
    gain = rng.uniform(0.1, 1.0, (nsrc, nx, 1, 1))
    delay = rng.uniform(0.0, 40.0, (nsrc, nx, 1, 1))
    img = gain * np.exp(-1j * np.pi * f * delay / max(F - 1, 1)) * src[:, None]          # [nsrc, nx, T, F]
    cls = f % 8
    img[0][..., cls == 1] = 0
    img[..., cls == 3] = img[:, :1][..., cls == 3]
    img[0][..., cls == 4] *= 1e3
    ramp = np.array([1e-44, 1e-41, 1e-38, 1e-30, 1e-20, 1e-10, 1e-3, 1e2])
    ramp_bins = np.nonzero(cls >= 5)[0]
    img[..., ramp_bins] *= ramp[(ramp_bins // 8 + cls[ramp_bins]) % ramp.size]
    if n >= 2:
        img[nsrc - 1, :, CHUNK:2 * CHUNK] = 0
    X = img.sum(axis=0)
    mag = np.abs(img).sum(axis=1) * rng.uniform(1.0, 1.8, (nsrc, T, F))
    tot = mag.sum(axis=0)
    mask = np.divide(mag, tot, out=np.zeros_like(mag), where=tot > 0)
    loud = slice(CHUNK * (n - 1), T) if n >= 3 else slice(0, T)
    scale = np.ones(T)
    scale[loud] = 1e4 / max(np.abs(X[:, loud]).max(), 1e-300)
    if n >= 3:
        scale[:loud.start] = 5.0 / max(np.abs(X[:, :loud.start]).max(), 1e-300)
    X = X * scale[None, :, None]
    Y = mask[:, None] * X[None]
    X[..., cls == 2] = 0
    silent = [t for t in range(T) if t % 50 == 17 and t != T - 1]
    Y[:, :, silent] = 0
    return X.astype(np.complex64).astype(np.complex128), Y.astype(np.complex64).astype(np.complex128)


# ---------------------------------------------------------------------------------------------- the reference and the bound
def window_frames(T, radius):
    """n_w per frame [T]: the frames of the covariance window of each frame's chunk"""
    n = nchunks(T)
    if radius == 0:
        return np.full(T, T)
    lens = np.array([min(T, (k + 1) * CHUNK) - k * CHUNK for k in range(n)])
    per_chunk = np.array([lens[list(window(c, n, radius))].sum() for c in range(n)])
    return per_chunk[np.arange(T) // CHUNK]


def reference(X, Y, radius):
    """(em_step(X, Y) complex128 [nsrc, nx, T, F], slack [nsrc, nx, T, F] = kappa_2(C) v_j sqrt(R_j,cc tr R_j) ||z||_2)"""
    X = np.asarray(X, np.complex128)
    Y = np.asarray(Y, np.complex128)
    nsrc, nx, T, F = Y.shape
    s = wco._scales(X, radius)
    R = wco._covariances(Y, s, radius)                                  # [n, nsrc, nx, nx, F]
    ref = wco.em_step(X, Y, s, radius)
    slack = np.empty(Y.shape)
    eye = np.eye(nx)
    for k in range(R.shape[0]):
        sl = slice(k * CHUNK, min(T, (k + 1) * CHUNK))
        v = (np.abs(Y[:, :, sl]) ** 2).sum(axis=1) / nx                 # [nsrc, t, F]
        Cm = np.einsum("jtf,jabf->tfab", v, R[k]) + DELTA * s[k] * s[k] * eye
        z = np.linalg.solve(Cm, np.moveaxis(X[:, sl], 0, -1)[..., None])[..., 0]
        kappa = np.linalg.cond(Cm)                                      # [t, F]
        diag = np.einsum("jaaf->jaf", R[k]).real                        # [nsrc, nx, F]
        env = np.sqrt(diag * diag.sum(axis=1, keepdims=True))           # sqrt(R_cc tr R)
        slack[:, :, sl] = (kappa * np.linalg.norm(z, axis=-1))[None, None] * v[:, None] * env[:, :, None]
    return ref, slack


def fp64_term(slack, nx, T, radius):
    nw = window_frames(T, radius)[:, None]
    return C_BOUND * U64 * (nx * nw + nx * nx) * slack


def check(dev, ref, slack, radius):
    """dev (fp32 values) against ref under the bound, per real and imaginary component -> dict: ratio (worst
    err / bound), where (its index and component), fp64_fraction (components whose fp64 term exceeds 2^-24 |ref| +
    2^-149), ok (every component within; NaN is not)"""
    nsrc, nx, T, F = ref.shape
    d64 = fp64_term(slack, nx, T, radius)
    dev = np.asarray(dev).astype(np.complex128)
    worst, where, frac, ok = 0.0, None, 0.0, True
    for part, name in ((np.real, "re"), (np.imag, "im")):
        r = part(ref)
        f32 = U32 * np.abs(r) + TINY
        err = np.abs(part(dev) - r)
        ratio = err / (f32 + d64)
        ok = ok and bool(np.all(ratio <= 1.0))
        frac += float(np.count_nonzero(d64 > f32)) / (2 * r.size)
        i = int(np.nanargmax(ratio)) if np.isfinite(ratio).any() else 0
        if not np.all(np.isfinite(ratio)):
            worst, where = float("inf"), (np.unravel_index(int(np.argmin(np.isfinite(ratio))), r.shape), name)
        elif ratio.flat[i] > worst:
            worst, where = float(ratio.flat[i]), (tuple(int(a) for a in np.unravel_index(i, r.shape)), name)
    return dict(ratio=worst, where=where, fp64_fraction=frac, ok=ok)


def plane_l2(dev, ref):
    """the per-plane relative L2 of the end-to-end tests, [nsrc * nx]"""
    nsrc, nx = ref.shape[:2]
    d = np.asarray(dev, np.complex128).reshape(nsrc * nx, -1)
    r = ref.reshape(nsrc * nx, -1)
    return [float(np.linalg.norm(d[p] - r[p]) / max(np.linalg.norm(r[p]), 1e-30)) for p in range(nsrc * nx)]


# ---------------------------------------------------------------------------------------------- the device's plan
def _solve(Cm, x):
    """z = C^-1 x over [..., nx, nx] / [..., nx] as the kernels do: the adjugate at nx = 2, else L D L^H without
    pivoting, row by row, then the forward and backward substitutions"""
    nx = Cm.shape[-1]
    if nx == 2:
        c11, c22, c12 = Cm[..., 0, 0].real, Cm[..., 1, 1].real, Cm[..., 0, 1]
        det = c11 * c22 - (c12.real * c12.real + c12.imag * c12.imag)
        return np.stack([(c22 * x[..., 0] - c12 * x[..., 1]) / det, (c11 * x[..., 1] - c12.conj() * x[..., 0]) / det], -1)
    L = np.zeros_like(Cm)
    D = np.zeros(Cm.shape[:-1], dtype=Cm.real.dtype)
    for i in range(nx):
        for k in range(i):
            acc = Cm[..., i, k].copy()
            for m in range(k):
                acc -= L[..., i, m] * D[..., m] * L[..., k, m].conj()
            L[..., i, k] = acc / D[..., k]
        di = Cm[..., i, i].real.copy()
        for k in range(i):
            di -= (L[..., i, k] * L[..., i, k].conj()).real * D[..., k]
        D[..., i] = di
    w = np.zeros_like(x)
    for i in range(nx):
        acc = x[..., i].copy()
        for k in range(i):
            acc -= L[..., i, k] * w[..., k]
        w[..., i] = acc
    z = np.zeros_like(x)
    for i in range(nx - 1, -1, -1):
        acc = w[..., i] / D[..., i]
        for k in range(i + 1, nx):
            acc -= L[..., k, i].conj() * z[..., k]
        z[..., i] = acc
    return z


def emulate(X, Y, radius, mutant=None):
    """one iteration by the device's plan in float64, rounded to fp32 per component -> complex64 [nsrc, nx, T, F];
    mutant: one of MUTANTS, the plan with that defect"""
    X = np.asarray(X, np.complex128)
    Y = np.asarray(Y, np.complex128)
    nsrc, nx, T, F = Y.shape
    n = nchunks(T)
    # per-chunk partials, frames in order
    P = np.zeros((n, nsrc, nx, nx, F), np.complex128)
    last = T - 1 if mutant == "drop_last_frame" and T % CHUNK else T
    for t in range(last):
        P[t // CHUNK] += np.einsum("jaf,jbf->jabf", Y[:, :, t], Y[:, :, t].conj())
    if mutant == "pair_conjugate" and nx >= 3:
        P[:, :, 1, 2], P[:, :, 2, 1] = P[:, :, 1, 2].conj(), P[:, :, 2, 1].conj()
    pmax = np.array([(X[:, k * CHUNK:(k + 1) * CHUNK].real ** 2 + X[:, k * CHUNK:(k + 1) * CHUNK].imag ** 2).max()
                     for k in range(n)])
    Q = np.zeros_like(P)
    s = np.empty(n)
    for c in range(n):
        win = range(n) if radius == 0 else window(c, n, radius)
        for k in win:
            Q[c] = Q[c] + P[k]
        s[c] = max(1.0, np.sqrt(max(pmax[k] for k in win)) / 10.0)
    if mutant == "clip_scale":
        s[:] = max(1.0, np.sqrt(pmax.max()) / 10.0)
    s2 = s if mutant == "s_for_s2" else s * s
    tr = np.einsum("njaaf->njf", Q).real / nx
    R = Q / (EPS * s2[:, None, None] + tr)[:, :, None, None, :]
    out = np.empty(Y.shape, np.complex64)
    eye = np.eye(nx)
    for t0 in range(0, T, CHUNK):
        c = t0 // CHUNK
        for sl, cr in ((slice(t0, t0 + 1), c - 1), (slice(t0 + 1, min(T, t0 + CHUNK)), c)) \
                if mutant == "prev_chunk_R_first_frame" and c >= 1 else ((slice(t0, min(T, t0 + CHUNK)), c),):
            if sl.start >= sl.stop:
                continue
            y = Y[:, :, sl]
            v = (np.abs(y[:, :1]) ** 2).sum(axis=1) if mutant == "v_from_channel0" else (np.abs(y) ** 2).sum(axis=1) / nx
            Rk, x = R[cr], np.moveaxis(X[:, sl], 0, -1)
            if mutant == "fp32_algebra":
                v, Rk, x = v.astype(np.float32), Rk.astype(np.complex64), x.astype(np.complex64)
                eye32 = np.float32(DELTA * s2[cr]) * np.eye(nx, dtype=np.float32)
                Cm = np.einsum("jtf,jabf->tfab", v, Rk) + eye32
            else:
                Cm = np.einsum("jtf,jabf->tfab", v, Rk) + DELTA * s2[cr] * eye
            z = _solve(Cm, x)
            out[:, :, sl] = (v[:, None] * np.einsum("jabf,tfb->jatf", Rk, z)).astype(np.complex64)
    return out
