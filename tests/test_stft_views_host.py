"""CPU checks of tests/stft_views_oracle.py, the float64 reference and element bounds that tests/test_gpu_stft_views.py
holds the STFT / iSTFT kernels to:
  - the vectorised reference equals oracle.dsp (stft_norm, istft_norm, compute_file, compute_inverse) and the golden
    vectors made by the reference project's own functions;
  - the bounds accept a float32 FFT (scipy's single-precision pocketfft, float32 overlap-add) at every shape the GPU
    suite runs;
  - they reject each of nine index / arithmetic mutations by at least 10x;
  - the second-tier bar accepts a plain float32 radix-2 FFT with a correctly rounded twiddle table and rejects the same
    FFT with its table rounded to 16 bits."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import stft_views_oracle as so  # noqa: E402
from oracle import dsp  # noqa: E402

U = so.U


def _maxrel(a, b):
    return float(np.abs(np.asarray(a) - b).max() / max(np.abs(b).max(), 1e-300))


@pytest.mark.parametrize("N,H,wname,sname,L", [(256, 64, "hanning", "hanning", 3001), (512, 384, "sinebell", "hanning", 777),
                                               (1024, 512, "hanning", "sinebell", 20000),
                                               (2048, 1536, "blackmanharris", "hanning", 9000),
                                               (4096, 4096, "hanning", "blackmanharris", 5000), (2048, 2, "hanning", "hanning", 301),
                                               (256, 254, "hanning", "sinebell", 1)])
def test_reference_matches_oracle_dsp(N, H, wname, sname, L):
    rng = np.random.default_rng(N + H + L)
    x = (rng.standard_normal(L) * 0.1).astype(np.float32)
    w, s = so.window(wname, N), so.window(sname, N)
    X, A = so.stft_ref(x, w, N, H)
    Xr = dsp.stft_norm(x.astype(np.float64), w, hopsize=float(H), nfft=float(N))
    assert X.shape == Xr.shape and _maxrel(X, Xr) <= 1e-15
    Ar = np.array([np.abs(w * f).sum() for f in so.frame_view(x, N, H)])
    assert np.array_equal(A, Ar)
    S = (rng.standard_normal(X.shape) + 1j * rng.standard_normal(X.shape)).astype(np.complex64)
    y = so.istft_ref(S, s, w, H, N)
    yr = dsp.istft_norm(S.astype(np.complex128), window=s, analysisWindow=w, hopsize=float(H), nfft=float(N))
    assert y.shape == yr.shape and _maxrel(y, yr) <= 1e-15
    # polar forms: compute_file(phase=True) / compute_inverse
    mag, ph = dsp.compute_file(x.astype(np.float64), phase=True, frameSize=N, hopSize=H, window=w)
    assert _maxrel(np.abs(X) / np.sqrt(N), mag) <= 1e-15 and np.array_equal(np.angle(X), ph)
    m32, p32 = (mag * 0.5).astype(np.float32), ph.astype(np.float32)
    yp = so.istft_ref(so.polar_spectrum(m32, p32, 1.0, N), w, w, H, N)
    ypr = dsp.compute_inverse(m32.astype(np.float64), p32.astype(np.float64), frameSize=N, hopSize=H, window=w)
    assert _maxrel(yp, ypr) <= 1e-15


def test_reference_matches_golden(golden):
    g = golden
    for ci in range(int(g["n_stft"])):
        N, H = (int(v) for v in g["stft%d_NH" % ci])
        x, w = g["stft%d_x" % ci], g["stft%d_w" % ci]
        X, _ = so.stft_ref(x, w, N, H)
        assert _maxrel(X, g["stft%d_X" % ci]) <= 1e-15, ci
        for spec, want in ((g["stft%d_X" % ci], g["stft%d_y" % ci]), (g["stft%d_Z" % ci], g["stft%d_y2" % ci])):
            y = so.istft_ref(spec, w, w, H, N)
            assert y.shape == want.shape and _maxrel(y, want) <= 1e-15, ci


# ---------------------------------------------------------------------------------------------- bounds vs float32
def forward_emulation_ratio(N, H, case):
    x = so.signal(case["signal"], case["L"], N, np.random.default_rng(case["L"] + N))
    w = so.window("hanning", N)
    X, A = so.stft_ref(x, w, N, H)
    worst, fails = so.check_forward(so.stft_f32(x, w, N, H), None, None, X, A, N, so.SCALE)
    return worst, fails


@pytest.mark.parametrize("N", so.SIZES)
def test_bounds_accept_float32_fft_forward(N):
    """scipy's float32 rfft on fl(fl(w) x), at every forward case shape of the GPU suite (all signals)"""
    worst = 0.0
    for H in so.hops(N):
        for case in so.forward_cases(N, H):
            r, fails = forward_emulation_ratio(N, H, case)
            assert not fails, (N, H, case, fails)
            worst = max(worst, r)
    print("forward N=%d: worst error / bound of the float32 FFT %.4f" % (N, worst))
    assert worst <= 1.0


def inverse_emulation(case, S=None):
    N, H = case["N"], case["H"]
    rng = np.random.default_rng(case["T"] + N + H)
    spec = so.inverse_spectra(case, rng) if S is None else S
    w, s = so.window("hanning", N), so.window(case["syn"], N)
    reg = so.inverse_layout(case)[5]
    cI = so.c_inverse(N, reg, case["polar"])
    if case["polar"]:
        Sp = so.polar_spectrum(spec[0], spec[1], case["scale"], N)
        return [(Sp.astype(np.complex64), so.istft_ref(Sp, s, w, H, N, cI, polar=True))], w, s
    return [(spec[k], so.istft_ref(spec[k], s, w, H, N, cI)) for k in range(spec.shape[0])], w, s


def test_bounds_accept_float32_fft_inverse():
    """scipy's float32 irfft, float32 overlap-add and normaliser, at every inverse case shape of the GPU suite"""
    worst = 0.0
    for case in so.inverse_cases():
        N, H = case["N"], case["H"]
        srcs, w, s = inverse_emulation(case)
        for S, (y, b) in srcs:
            e = np.abs(so.istft_f32(S, s, w, H, N).astype(np.float64) - y)
            r = float(so.ratio(e, b).max())
            assert r <= 1.0, (case["name"], r, int(np.argmax(so.ratio(e, b))))
            worst = max(worst, r)
    print("inverse: worst error / bound of the float32 FFT %.4f" % worst)


# ---------------------------------------------------------------------------------------------- teeth
def _fwd_setup(N=1024, H=256, L=20000, kind="white"):
    x = so.signal(kind, L, N, np.random.default_rng(11))
    w = so.window("hanning", N)
    X, A = so.stft_ref(x, w, N, H)
    return x, w, X, A


def _fwd_ratio(Xm, X, A, N):
    return so.check_forward(Xm, None, None, X, A, N, so.SCALE)[0]


def _inv_case(N=1024, H=256, syn="sinebell", seam=None, T=70):
    return dict(N=N, H=H, T=T, nsrc=1, syn=syn, force=None, polar=False, scale=1.0, outs=[(T - 1) * H + N // 2],
                seam=seam, name="teeth")


def _inv_ratio(ym, y, b):
    return float(so.ratio(np.abs(ym - y), b).max())


def _mut_forward(mut):
    N, H = 1024, 256
    x, w, X, A = _fwd_setup(N, H)
    if mut == "window_shift":
        Xm = so.stft_f32(x, np.roll(w, 1), N, H)
    elif mut == "window_bf16":
        b = w.astype(np.float32).view(np.uint32)
        wb = ((b + np.uint32(0x8000)) & np.uint32(0xFFFF0000)).view(np.float32).astype(np.float64)
        Xm = so.stft_f32(x, wb, N, H)
    elif mut == "frame_hop_late":
        Xm = so.stft_f32(x, w, N, H)
        Xm[40] = Xm[41]
    elif mut == "nyquist_plus":
        Xm = so.stft_f32(x, w, N, H)
        Xm[:, -1] = Xm[:, 0].real        # Re Z0 + Im Z0 = sum of all windowed samples = X_0
    return _fwd_ratio(Xm, X, A, N)


def packed_irfft(S, N, keep_imag=False):
    """the kernels' inverse in float64: merge to N/2 packed bins (real_pre_conj), complex inverse FFT, unpack; with
    keep_imag the imaginary parts of DC and Nyquist are not dropped"""
    S = np.array(S, np.complex128)
    if not keep_imag:
        S = so.drop_dc_nyquist_imag(S)
    n2 = N // 2
    k = np.arange(n2)
    xk, xn = S[:, :n2], np.conj(S[:, n2 - k])
    e, d = (xk + xn) / 2, (xk - xn) / 2
    Z = e + 1j * d * np.exp(2j * np.pi * k / N)
    z = np.fft.ifft(Z, axis=1)
    out = np.empty((S.shape[0], N))
    out[:, 0::2], out[:, 1::2] = z.real, z.imag
    return out


def _mut_inverse(mut):
    if mut == "halo_dropped":
        N, H = 2048, 512
        case = _inv_case(N, H, "hanning", seam=12, T=70)
    else:
        N, H = 1024, 256
        case = _inv_case(N, H)
    C0, R = (N // 2) // H, N // H
    rng = np.random.default_rng(5)
    S = so.inverse_spectra(case, rng)[0]
    w, s = so.window("hanning", N), so.window(case["syn"], N)
    y, b = so.istft_ref(S, s, w, H, N, so.c_inverse(N, True))
    yf = so.istft_f32(S, s, w, H, N).astype(np.float64)
    T = case["T"]
    c = so.ola_const(w * s, T, H)[N // 2:]
    c = np.where(c == 0, 1.0, c)
    if mut == "normaliser_ww":
        cm = so.ola_const(w * w, T, H)[N // 2:]
        ym = yf * c / np.where(cm == 0, 1.0, cm)
    elif mut == "interior_at_start":
        ym = yf.copy()
        q = np.arange(ym.size) + N // 2
        first = q < (R - 1) * H
        ci = sum(np.roll(w * s, -r * H)[:H] for r in range(R))       # every hop sees R frames
        ym[first] = yf[first] * c[first] / ci[q[first] % H]
    elif mut == "halo_dropped":
        h0 = 12
        n = h0 + C0 - R + 1
        z = np.fft.irfft(so.drop_dc_nyquist_imag(S[n:n + 1]), N, axis=1)[0] * s
        ym = yf.copy()
        i = np.arange(h0 * H, (h0 + 1) * H)          # output hop h0 <-> frame samples i + N/2 - n H
        ym[i] -= z[i + N // 2 - n * H] / c[i]
    elif mut in ("dc_imag_kept", "nyquist_imag_kept"):
        S2 = S.copy()
        col = 0 if mut == "dc_imag_kept" else -1
        S2[:, col] = S2[:, col].real + 1j * rng.standard_normal(T).astype(np.float32)
        zk = packed_irfft(S2, N, keep_imag=True) * s
        ym = so.ola(zk, H)[N // 2:] / c
        assert np.abs(packed_irfft(S2, N) - np.fft.irfft(so.drop_dc_nyquist_imag(S2), N, axis=1)).max() < 1e-12
    return _inv_ratio(ym, y, b)


MUTATIONS = ["window_shift", "window_bf16", "frame_hop_late", "nyquist_plus", "halo_dropped", "normaliser_ww",
             "interior_at_start", "dc_imag_kept", "nyquist_imag_kept"]


@pytest.mark.parametrize("mut", MUTATIONS)
def test_bound_has_teeth(mut):
    """each mutation, applied to the float32 emulation, exceeds the element bound by >= 10x somewhere"""
    r = _mut_forward(mut) if mut in ("window_shift", "window_bf16", "frame_hop_late", "nyquist_plus") else _mut_inverse(mut)
    print("%s: worst error / bound %.3g" % (mut, r))
    assert r >= 10.0, (mut, r)


# ---------------------------------------------------------------------------------------------- second tier
def _tier_forward(N, H, bits):
    x, w, X, A = _fwd_setup(N, H, L=30000)
    b = so.forward_bounds(A, N)[:, None] * np.ones((1, X.shape[1]))
    e_base = np.abs(so.stft_f32(x, w, N, H).astype(np.complex128) - X)
    e_r2 = np.abs(so.stft_f32(x, w, N, H, fft=so.radix2_rfft(N, bits)).astype(np.complex128) - X)
    return so.rms_ratio(e_r2, e_base, b)


def _tier_inverse(N, H, bits):
    case = _inv_case(N, H, "hanning", T=200)
    S = so.inverse_spectra(case, np.random.default_rng(3))[0]
    w = s = so.window("hanning", N)
    y, b = so.istft_ref(S, s, w, H, N, so.c_inverse(N, False))
    e_base = np.abs(so.istft_f32(S, s, w, H, N).astype(np.float64) - y)
    e_r2 = np.abs(so.istft_f32(S, s, w, H, N, ifft=so.radix2_irfft(N, bits)).astype(np.float64) - y)
    return so.rms_ratio(e_r2, e_base, b)


@pytest.mark.parametrize("N,H", [(256, 64), (1024, 256), (2048, 512), (4096, 1024)])
def test_second_tier_bar_catches_a_coarse_twiddle_table(N, H):
    """a plain float32 radix-2 FFT passes the RMS bar with a correctly rounded twiddle table and fails it with the
    table rounded to 16 bits, forward and inverse (both pass the element bound's worst case or not: the bar is what
    catches them)"""
    good = (_tier_forward(N, H, None), _tier_inverse(N, H, None))
    coarse = (_tier_forward(N, H, 16), _tier_inverse(N, H, 16))
    print("N=%d radix-2 RMS ratio: exact table %.3f / %.3f, 16-bit table %.3f / %.3f" % ((N,) + good + coarse))
    assert max(good) <= so.RMS_BAR, good
    assert min(coarse) > so.RMS_BAR, coarse
