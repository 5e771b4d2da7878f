"""Float64 reference and per-element error bounds for the framed STFT (K1: stft.cu, stft_reg.cu) and the inverse STFT
with overlap-add (K4: istft_kernel, istft_reg_kernel), shared by tests/test_stft_views_host.py (CPU) and
tests/test_gpu_stft_views.py (GPU).  Test infrastructure only.

Reference.  A vectorised restatement of oracle.dsp.stft_norm / istft_norm (transform.py:277-396): all frames at once
through np.fft.rfft / irfft, overlap-add by hop offsets.  The forward takes the float32 audio converted exactly to
float64 and the float64 windows.  The inverse takes the float32 spectra and drops the imaginary parts of DC and Nyquist
(irfft's rule).  The polar forms are compute_file(phase=True) and compute_inverse.

Forward bound, per element.  u = 2^-24.  For frame n, A_n = sum_i |w_i x_i| over its windowed samples.  Every value
inside a radix-2/4 FFT is a partial DFT with unit-modulus twiddles of a disjoint block of the packed input
z_m = v_2m + i v_2m+1, so it is at most the block's sum of |z|, and the values that feed one output bin partition the
input.  A pass that rounds each of its values to within eta u of that sum therefore moves every output by at most
eta u A_n.  Per pass (complex moduli, fused multiply-adds):
  - a product by a rounded twiddle: u for the table entry plus 2 sqrt(2) u for the fused complex product, 3.83u;
  - a radix-4 pass of fft.cuh: twiddles then two levels of complex additions, 5.83u (2u for the first pass, which has
    no twiddles); a radix-2 pass of fft.cuh or a DIF stage of fft_reg.cuh's 32- and 16-point networks, 4.83u;
  - fft_reg.cuh (N/2 = 32 x T): five DIF stages, the inter-stage twiddle (3.83u) and log2 T DIF stages.
The real split step X_k = (Z_k + conj Z_{N/2-k})/2 + tw_k (Z_k - conj Z_{N/2-k})/(2i) doubles the FFT's error and adds
8u A_n of its own (two halvings-and-additions, a twiddle product, a last addition); the window is rounded to float32
and multiplied, 2u |w x| per sample, 2u A_n.  So
  c_F(N) = 2 + 2 eta_FFT(N) + 8:   stft.cu 47 / 49 / 70 (N = 256 / 512 / 4096), stft_reg.cu 105 / 114 (1024 / 2048),
and |X^ - X| <= g c_F(N) u A_n with the safety factor g = 2 (second-order terms, and no claim that the accounting above
is tight to the last u).  Magnitude: |m^ - m| <= (scale / sqrt N) bound_X + 6u m (scale / sqrtf(N) and the sum of
squares, square root and product are rounded).  Phase: where |X| > 8 bound_X, the wrapped difference is at most
bound_X / (|X| - bound_X) + 8u (atan2f is good to 2 ulp, 8u at pi); elsewhere it only has to be finite and in
[-pi, pi] (float32(pi) included).  A_n is per frame, so a quiet frame is held to its own scale.

Inverse bound, per output sample.  q = i + N/2 (padded coordinate), frames n covering q, s the synthesis window, z_n the
float64 irfft of frame n, R = ceil(N / H).  The merge step real_pre_conj rounds each packed bin to within 6u of
|X_k| + |X_{N/2-k}|, whose sum over k is N B_n with B_n = (|Re S_0| + 2 sum_{0<k<N/2} |S_k| + |Re S_{N/2}|) / N, and the
complex FFT of N/2 points then divides by N/2:
  E_n = c_I(N) u B_n,  c_I(N) = 2 (eta_FFT(N) + 6)   (+ 9 for the polar entry: sqrtf(N), mag_scale * sqrtf(N), the
        product with mag, sincosf and the two products of the polar form; B_n then takes |S_0| and |S_{N/2}| whole).
  num_err = sum_n |s| (E_n + 2u |z_n|) + R u sum_n |s z_n|   (s rounded and multiplied; at most R frames accumulated)
  c(q) = sum_n w s carries (R + 1) u sum_n |w s| (each w s rounded to float32, then summed)
  bound = g [num_err / |c| + |y| c_err / |c| + 2u |y|]   (2u: the division, or istft_reg's reciprocal and product)
Where c(q) = 0 in float64, c := 1 (transform.py:392, and both kernels).  The bound grows by itself where the window
tails make a sample ill-conditioned (the last N/2 samples, hop = N with a vanishing window).

Second tier.  The element bound is a worst case and is loose for white noise: a systematic error of a few u per value
(a twiddle table good to 16 bits) passes it.  So each case also compares its error with that of a float32 FFT on the
same frames: scipy.fft.rfft / irfft on float32 input (single-precision pocketfft) plus a float32 overlap-add.  Both
errors are taken element by element relative to the element's bound (so quiet frames and ill-conditioned samples weigh
like the rest), and the ratio of their root-mean-squares is held to a bar (tests/test_gpu_stft_views.py)."""
import math

import numpy as np

U = 2.0 ** -24
G = 2.0                    # safety factor of every element bound
SLACK = 64                 # fence elements before and after every buffer in the GPU tests
ETA_TW = 2.0 * math.sqrt(2.0) + 1.0
ETA2 = ETA_TW + 1.0
ETA4 = ETA_TW + 2.0
ETA4_FIRST = 2.0
ETA_PRE = 6.0
POLAR_EXTRA = 9.0
REG_SIZES = (1024, 2048)
# second tier: the kernels' bound-relative RMS error over that of scipy's float32 FFT may be at most 2x the worst ratio
# measured on an H100 80GB HBM3 (700 W): 1.26 (stft_reg.cu; stft.cu 1.14, istft_reg_kernel 1.09, istft_kernel 1.05,
# polar inverse 1.07)
RMS_BAR = 2.52


def _log2(n):
    k = int(round(math.log2(n)))
    assert 1 << k == n
    return k


def eta_fft(N, reg):
    """rounding of the N/2-point complex FFT, in u times the L1 norm of its input"""
    n2 = N // 2
    if reg:
        return 5 * ETA2 + ETA_TW + _log2(n2 // 32) * ETA2
    m = _log2(n2)
    return ETA4_FIRST + (m // 2 - 1) * ETA4 + (m % 2) * ETA2


def forward_reg(N):
    """stft_reg.cu takes N = 1024 and 2048, stft.cu every other size"""
    return N in REG_SIZES


def c_forward(N):
    return 2.0 + 2.0 * eta_fft(N, forward_reg(N)) + 8.0


def c_inverse(N, reg, polar=False):
    return 2.0 * (eta_fft(N, reg) + ETA_PRE) + (POLAR_EXTRA if polar else 0.0)


# ---------------------------------------------------------------------------------------------- float64 reference
def num_frames(L, H):
    return -(-L // H) + 2


def _padded_audio(x, N, H):
    L = x.size
    T = num_frames(L, H)
    xp = np.zeros((T - 1) * H + N)
    xp[N // 2:N // 2 + L] = np.asarray(x, np.float64)
    return xp, T


def frame_view(x, N, H):
    """[T, N] read-only view of stft_norm's frames of x (zeros before and after, float64)"""
    xp, T = _padded_audio(x, N, H)
    return np.lib.stride_tricks.sliding_window_view(xp, N)[::H][:T]


CHUNK = 4096


def stft_ref(x, w, N, H):
    """stft_norm in float64 on the float32 audio x and the float64 window w -> X [T, F] complex128, A [T]"""
    fr = frame_view(x, N, H)
    T = fr.shape[0]
    X = np.empty((T, N // 2 + 1), np.complex128)
    A = np.empty(T)
    for a in range(0, T, CHUNK):
        v = fr[a:a + CHUNK] * w
        X[a:a + CHUNK] = np.fft.rfft(v, axis=1)
        A[a:a + CHUNK] = np.abs(v).sum(axis=1)
    return X, A


def ola(frames, H):
    """overlap-add of [T, N] frames at hop H -> length (T - 1) H + N (float64)"""
    T, N = frames.shape
    R = -(-N // H)
    fp = np.zeros((T, R * H), frames.dtype)
    fp[:, :N] = frames
    fp = fp.reshape(T, R, H)
    out = np.zeros((T - 1 + R, H), frames.dtype)
    for j in range(R):
        out[j:j + T] += fp[:, j]
    return out.ravel()[:(T - 1) * H + N]


def ola_const(v, T, H):
    """overlap-add of the same frame v at T hops"""
    N = v.size
    R = -(-N // H)
    vp = np.zeros(R * H, v.dtype)
    vp[:N] = v
    vp = vp.reshape(R, H)
    out = np.zeros((T - 1 + R, H), v.dtype)
    for j in range(R):
        out[j:j + T] += vp[j]
    return out.ravel()[:(T - 1) * H + N]


def drop_dc_nyquist_imag(S):
    S = np.array(S, np.complex128)
    S[..., 0] = S[..., 0].real
    S[..., -1] = S[..., -1].real
    return S


def istft_ref(S, s, w, H, N, cI=None, polar=False):
    """istft_norm(S, window=s, analysisWindow=w) in float64 -> y (length (T-1) H + N/2), and with cI the element bound.
    S [T, F] complex (float32 values); Im of DC and Nyquist are dropped as irfft does."""
    S = np.asarray(S)
    T = S.shape[0]
    Sr = drop_dc_nyquist_imag(S)
    R = -(-N // H)
    num = np.zeros((T - 1) * H + N)
    aerr = np.zeros_like(num) if cI is not None else None
    for a in range(0, T, CHUNK):
        z = np.fft.irfft(Sr[a:a + CHUNK], N, axis=1)
        part = ola(z * s, H)
        num[a * H:a * H + part.size] += part
        if cI is not None:
            Sa = np.abs(S[a:a + CHUNK]) if polar else np.abs(Sr[a:a + CHUNK])
            B = (Sa[:, 0] + 2.0 * Sa[:, 1:-1].sum(axis=1) + Sa[:, -1]) / N
            fe = cI * U * B[:, None] * np.abs(s)[None, :] + (2.0 + R) * U * np.abs(z * s)
            pe = ola(fe, H)
            aerr[a * H:a * H + pe.size] += pe
    c = ola_const(w * s, T, H)
    cabs = ola_const(np.abs(w * s), T, H)
    num, c, cabs = num[N // 2:], c[N // 2:], cabs[N // 2:]
    zero = c == 0
    c = np.where(zero, 1.0, c)
    y = num / c
    if cI is None:
        return y
    aerr = aerr[N // 2:]
    cerr = np.where(zero, 0.0, (R + 1) * U * cabs)
    bound = G * (aerr / np.abs(c) + np.abs(y) * cerr / np.abs(c) + 2.0 * U * np.abs(y))
    return y, bound


def polar_spectrum(mag, phase, mag_scale, N):
    """compute_inverse's X = mag_scale sqrt(N) mag exp(j phase) in float64 from float32 mag / phase"""
    return float(mag_scale) * math.sqrt(N) * np.asarray(mag, np.float64) * np.exp(1j * np.asarray(phase, np.float64))


# ---------------------------------------------------------------------------------------------- element checks
def forward_bounds(A, N):
    return G * c_forward(N) * U * A


def check_forward(Xg, mag, phase, X, A, N, scale):
    """Xg complex [T, F] (or None), mag / phase float32 [T, F] (or None) against X (float64) and A.
    -> (worst error / bound, list of failures)"""
    bx = forward_bounds(A, N)[:, None] * np.ones((1, X.shape[1]))
    fails, worst = [], 0.0
    absX = np.abs(X)

    def ratio(err, b, tag):
        nonlocal worst
        r = np.where(b > 0, err / np.where(b > 0, b, 1.0), np.where(err > 0, np.inf, 0.0))
        m = float(r.max()) if r.size else 0.0
        worst = max(worst, m)
        if m > 1.0:
            t, k = np.unravel_index(int(np.argmax(r)), r.shape)
            fails.append((tag, int(t), int(k), m))
    if Xg is not None:
        ratio(np.abs(Xg.astype(np.complex128) - X), bx, "X")
    if mag is not None:
        ms = float(scale) / math.sqrt(N)
        m = ms * absX
        ratio(np.abs(mag.astype(np.float64) - m), ms * bx + 6.0 * U * m, "mag")
    if phase is not None:
        p = phase.astype(np.float64)
        if not (np.all(np.isfinite(p)) and np.all(np.abs(p) <= float(np.float32(np.pi)))):
            fails.append(("phase range",))
        well = absX > 8.0 * bx
        d = np.angle(np.exp(1j * (p - np.angle(X))))
        lim = bx / np.maximum(absX - bx, 1e-300) + 8.0 * U
        ratio(np.where(well, np.abs(d), 0.0), np.where(well, lim, 1.0), "phase")
    return worst, fails


def ratio(err, bound):
    """err / bound element by element: 0 where both are 0, inf where only the bound is"""
    err, bound = np.asarray(err, np.float64), np.asarray(bound, np.float64)
    pos = bound > 0
    return np.where(pos, err / np.where(pos, bound, 1.0), np.where(err > 0, np.inf, 0.0))


def norm_rms(err, bound):
    """root-mean-square of err / bound over the elements with a positive bound"""
    ok = bound > 0
    e = err[ok] / bound[ok]
    return float(np.sqrt(np.mean(e * e))) if e.size else 0.0


def rms_ratio(err_kernel, err_base, bound):
    """the second-tier figure: RMS of the kernel's bound-relative error over that of the float32 baseline"""
    b = norm_rms(err_base, bound)
    k = norm_rms(err_kernel, bound)
    if b == 0.0:
        return 0.0 if k == 0.0 else math.inf
    return k / b


# ---------------------------------------------------------------------------------------------- float32 baselines
def stft_f32(x, w, N, H, fft=None):
    """float32 frames fl(fl(w) x), then a float32 real FFT: scipy.fft.rfft (single-precision pocketfft) or `fft`
    (a function of float32 frames [M, N] -> complex64 [M, F])"""
    import scipy.fft
    x32 = np.asarray(x, np.float32)
    fr = frame_view(x32, N, H)
    w32 = np.asarray(w, np.float64).astype(np.float32)
    out = np.empty((fr.shape[0], N // 2 + 1), np.complex64)
    for a in range(0, fr.shape[0], CHUNK):
        v = fr[a:a + CHUNK].astype(np.float32) * w32
        out[a:a + CHUNK] = scipy.fft.rfft(v, axis=1) if fft is None else fft(v)
    return out


def istft_f32(S, s, w, H, N, ifft=None):
    """float32 inverse: irfft per frame (scipy.fft.irfft on complex64, or `ifft`), times fl(s), float32 overlap-add,
    divided by the float32 sum of fl(w s) (0 -> 1)"""
    import scipy.fft
    S = np.asarray(S, np.complex64).copy()
    S[:, 0] = S[:, 0].real
    S[:, -1] = S[:, -1].real
    s32 = np.asarray(s, np.float64).astype(np.float32)
    T = S.shape[0]
    num = np.zeros((T - 1) * H + N, np.float32)
    for a in range(0, T, CHUNK):
        z = scipy.fft.irfft(S[a:a + CHUNK], N, axis=1) if ifft is None else ifft(S[a:a + CHUNK])
        z = z.astype(np.float32) * s32
        part = ola(z, H)
        num[a * H:a * H + part.size] += part
    c = ola_const((np.asarray(w, np.float64) * s).astype(np.float32), T, H)
    num, c = num[N // 2:], c[N // 2:]
    c = np.where(c == 0, np.float32(1), c)
    return (num / c).astype(np.float32)


def twiddles(n, bits=None):
    """exp(-2 pi i k / n), k < n/2, as complex64: correctly rounded, or with both parts rounded to `bits`-bit fixed
    point (a table good to only that many bits)"""
    a = np.exp(-2j * np.pi * np.arange(n // 2) / n)
    if bits is not None:
        q = 2.0 ** (bits - 1)
        a = np.round(a.real * q) / q + 1j * (np.round(a.imag * q) / q)
    return a.astype(np.complex64)


def _bitrev(n):
    k = _log2(n)
    i = np.arange(n)
    r = np.zeros(n, np.int64)
    for b in range(k):
        r |= ((i >> b) & 1) << (k - 1 - b)
    return r


def fft_radix2_f32(a, tw):
    """plain iterative radix-2 DIT FFT in complex64 arithmetic, vectorised over the rows of a [M, n]"""
    M, n = a.shape
    a = np.ascontiguousarray(np.asarray(a, np.complex64)[:, _bitrev(n)])
    m = 1
    while m < n:
        wj = tw[::n // (2 * m)][:m]
        b = a.reshape(M, n // (2 * m), 2, m)
        t = b[:, :, 1, :] * wj
        u = b[:, :, 0, :]
        a = np.stack([u + t, u - t], axis=2).reshape(M, n)
        m *= 2
    return a


def radix2_rfft(N, bits=None):
    tw = twiddles(N, bits)
    return lambda v: fft_radix2_f32(v.astype(np.complex64), tw)[:, :N // 2 + 1]


def radix2_irfft(N, bits=None):
    """irfft through the forward radix-2 FFT: x = Re FFT(conj Y) / N for the Hermitian extension Y"""
    tw = twiddles(N, bits)

    def f(S):
        S = np.asarray(S, np.complex64)
        Y = np.empty((S.shape[0], N), np.complex64)
        Y[:, :N // 2 + 1] = S
        Y[:, N // 2 + 1:] = np.conj(S[:, 1:N // 2][:, ::-1])
        return (fft_radix2_f32(np.conj(Y), tw).real / np.float32(N)).astype(np.float32)
    return f


# ---------------------------------------------------------------------------------------------- case shapes
FPC = {256: 8, 512: 8, 1024: 32, 2048: 16, 4096: 8}     # frames per CTA of the forward kernels
SIGNALS = ("white", "quiet", "tone_bin", "tone_between", "dc", "nyquist", "int16", "zeros")
SIZES = (256, 512, 1024, 2048, 4096)
SCALE = float(np.float32(0.3))


def hops(N):
    return sorted({2, 6, N // 4, N // 2, N - 2, N})


def padded_bins(N):
    return (N // 2 + 1 + 7) // 8 * 8


def ldfs(N):
    F = N // 2 + 1
    return (F, F + 1, padded_bins(N), F + 16)


def _cap(N, H, L, budget=1 << 22):
    """largest L <= the given one whose frames hold at most `budget` samples"""
    return max(1, min(L, (budget // N - 2) * H))


def forward_cases(N, H):
    """(L, signal, ldf, audio offset in floats) of the forward cases at (N, H).  Over the hops of one N the frame
    counts T take every residue modulo the frames per CTA (for the <16> kernel that includes a last warp with one live
    group); each hop adds L = 1, L < N, a clip where one frame starts at sample 0 and one ends at sample L (the edges of
    stft_reg's interior fast path) and a longer clip."""
    hs = hops(N)
    hi = hs.index(H)
    fpc = FPC[N]
    Ls = []
    for r in range(fpc):
        if r % len(hs) != hi:
            continue
        T = fpc * (1 + (r // len(hs)) % 3) + r
        if T < 3:
            T += fpc
        lo = (T - 3) * H
        Ls.append(lo + 1 + (r * 7919) % H)
    Ls += [1, N // 2 + 1, N - 1]
    if (N // 2) % H == 0:
        Ls.append(N + 3 * H)            # frame N/(2H) starts at sample 0, frame N/(2H) + 3 ends at sample L
    else:
        Ls.append(5 * H + N // 2)       # frame 5 ends at sample L
    Ls.append(_cap(N, H, 40 * N + 3 * H // 2 + 1))
    out = []
    for i, L in enumerate(Ls):
        sig = SIGNALS[(i + hi) % len(SIGNALS)]
        out.append(dict(L=int(L), signal=sig, ldf=ldfs(N)[(i + hi) % 4], off=(i + N // 256) % 2))
    return out


def signal(kind, L, N, rng):
    """float32 test audio"""
    t = np.arange(L, dtype=np.float64)
    if kind == "white":
        x = rng.standard_normal(L) * 0.1
    elif kind == "quiet":           # a loud segment next to a quiet one: quiet frames are held to their own scale
        x = rng.standard_normal(L) * 0.5
        x[L // 3:] *= 2e-5
    elif kind == "tone_bin":
        k = max(1, N // 16 + 3)
        x = 0.7 * np.cos(2 * np.pi * k * t / N + 0.3)
    elif kind == "tone_between":
        x = 0.7 * np.sin(2 * np.pi * (N / 5.0 + 0.37) * t / N) + 0.01 * rng.standard_normal(L)
    elif kind == "dc":
        x = 0.25 + 0.01 * rng.standard_normal(L)
    elif kind == "nyquist":
        x = np.where(np.arange(L) % 2 == 0, 1.0, -1.0)
    elif kind == "int16":
        x = np.clip(np.round(rng.standard_normal(L) * 12000), -32767, 32767) / 32767.0
    elif kind == "zeros":
        x = np.zeros(L)
    else:
        raise ValueError(kind)
    return x.astype(np.float32)


def window(name, N):
    from deepconvsep_b200.engine import get_window
    return get_window(name, N)


def reg_inverse(N, H):
    """the (N, hop) pairs istft_reg_kernel serves (when the pointers, strides and ldf allow it)"""
    return N in REG_SIZES and H in (256, 512)


def target_groups(N, sms):
    """istft_reg_kernel's one full wave of groups (launch_istft_reg_t)"""
    return sms * 8 * (32 // (N // 64))


def reg_hpg(N, H, nsrc, num_out, sms):
    num_hops = -(-num_out // H)
    return int(min(64, max(12, -(-(nsrc * num_hops) // target_groups(N, sms)))))


def num_outs(T, H, N):
    """num_out values of an inverse case: 1, 2, H - 1, H, H + 1, max - 1, max, and a partial last group"""
    mx = (T - 1) * H + N // 2
    vals = {1, 2, H - 1, H, H + 1, mx - 1, mx, 12 * H * 2 + 5 * H + H // 2 + 1}
    return sorted(v for v in vals if 1 <= v <= mx)


def inverse_cases(sms=132):
    """inverse cases: dicts with N, H, syn (synthesis window), nsrc, T, force (what moves the register kernel's pairs
    onto the shared-memory kernel, or None), polar, scale, outs (num_out values), and seam (hops per group the register
    kernel is expected to take at num_out = max, where large frames are planted, or None)"""
    cases = []

    def add(N, H, T, nsrc=1, syn="hanning", force=None, polar=False, outs=None, seam=None, name=None):
        cases.append(dict(N=N, H=H, T=int(T), nsrc=nsrc, syn=syn, force=force, polar=polar,
                          scale=float(np.float32(0.7)) if polar else 1.0,
                          outs=outs if outs is not None else num_outs(int(T), H, N), seam=seam,
                          name=name or "N%d_H%d_T%d_s%d_%s_%s%s" % (N, H, T, nsrc, syn, force, "_polar" if polar else "")))
    # the register kernel at its four pairs: hops per group 12 (several seams), in between, 64
    for N, H in ((2048, 512), (2048, 256), (1024, 512), (1024, 256)):
        C0, R = (N // 2) // H, N // H
        for nsrc, syn in ((1, "hanning"), (3, "sinebell"), (9, "blackmanharris")):
            T = 12 * 5 + 7 + 3 - C0 + (nsrc % 3)
            add(N, H, T, nsrc, syn, seam=12)
        for force in ("odd_ldf", "odd_stride", "out_off", "s_off8"):
            add(N, H, 40 + R, 3 if force != "odd_ldf" else 1, "sinebell" if force == "odd_stride" else "hanning", force)
        add(N, H, 3 * R + 1, 1, "hanning", polar=True)
    tg = target_groups(2048, sms)
    # 180 s at 2048/512, one source: hpg = ceil(15504 / groups) (15 on 132 SMs)
    L180 = 180 * 44100
    T180 = num_frames(L180, 512)
    add(2048, 512, T180, 1, "hanning", outs=[L180, (T180 - 1) * 512 + 1024], seam=reg_hpg(2048, 512, 1, L180, sms),
        name="N2048_H512_180s")
    # hops per group 64: nine sources of ceil(63.1 groups * 8 / 9) hops
    nh = -(-(63 * tg + tg // 8) // 9)
    T64 = nh - 1                        # num_out = max covers T + 1 hops
    mx = (T64 - 1) * 512 + 1024
    add(2048, 512, T64, 9, "sinebell", outs=[mx - 1, mx], seam=reg_hpg(2048, 512, 9, mx, sms), name="N2048_H512_hpg64")
    # hops per group in between at 1024/256: three sources
    nh = -(-(30 * target_groups(1024, sms)) // 3)
    Tm = nh - 1
    mx = (Tm - 1) * 256 + 512
    add(1024, 256, Tm, 3, "hanning", outs=[mx], seam=reg_hpg(1024, 256, 3, mx, sms), name="N1024_H256_hpg_mid")
    # the shared-memory kernel everywhere else
    for N in SIZES:
        for H in hops(N):
            if reg_inverse(N, H):
                continue
            T = min(3 * (N // H) + 5, (1 << 21) // N)
            nsrc = (1, 3, 9)[hops(N).index(H) % 3]
            syn = ("hanning", "sinebell", "blackmanharris")[(hops(N).index(H) + N // 256) % 3]
            add(N, H, T, nsrc, syn)
        H = N // 4
        add(N, H, 2 * (N // H) + 3, 1, "hanning" if N != 4096 else "blackmanharris", polar=True)
    return cases


def inverse_layout(case):
    """ldf, source stride, out stride, S offset (complex elements), out offset (floats) and whether istft_reg_kernel is
    expected"""
    N, H, T, force = case["N"], case["H"], case["T"], case["force"]
    F = N // 2 + 1
    ldf = F if force == "odd_ldf" else {1: padded_bins(N), 3: F + 1}.get(case["nsrc"], padded_bins(N) + 8)
    src_stride = T * ldf + 24
    mx = max(case["outs"])
    out_stride = mx + mx % 2 + 6 + (1 if force == "odd_stride" else 0)
    s_off = 1 if force == "s_off8" else 0
    o_off = 1 if force == "out_off" else 0
    reg = reg_inverse(N, H) and force is None and not case["polar"]
    return ldf, src_stride, out_stride, s_off, o_off, reg


def inverse_spectra(case, rng):
    """complex64 [nsrc, T, F] spectra (polar: mag, phase float32 [T, F]) with large frames on either side of every
    expected group seam, so that a lost or doubled halo frame lands far outside the bound"""
    N, H, T, nsrc = case["N"], case["H"], case["T"], case["nsrc"]
    F = N // 2 + 1
    if case["polar"]:
        mag = np.abs(rng.standard_normal((T, F))).astype(np.float32) * np.float32(0.05)
        ph = rng.uniform(-np.pi, np.pi, (T, F)).astype(np.float32)
        return mag, ph
    Z = np.empty((nsrc, T, F), np.complex64)
    Z.real = rng.standard_normal((nsrc, T, F), dtype=np.float32)
    Z.imag = rng.standard_normal((nsrc, T, F), dtype=np.float32)
    if case["seam"]:
        hpg, C0, R = case["seam"], (N // 2) // H, N // H
        mx = max(case["outs"])
        nh = -(-mx // H)
        h0 = np.arange(hpg, nh, hpg)
        for d in (-R + 1, -1, 0):
            n = h0 + C0 + d
            n = n[(n >= 0) & (n < T)]
            Z[:, n] *= np.float32(1e3)
    return Z
