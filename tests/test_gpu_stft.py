"""GPU parity: framed STFT / iSTFT kernels (through the C ABI) vs the oracle and the golden
vectors produced by the reference's own functions.  fp32 kernels vs float64 reference:
tolerance 2e-6 relative L2 on spectra, 5e-6 on reconstructed audio (stated per assert)."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from oracle import dsp  # noqa: E402
from parity import record  # noqa: E402


def rel(a, b):
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


@pytest.fixture(scope="module")
def ctx():
    from deepconvsep_b200.engine import Context
    return Context(0)


def _plan(ctx, N, H, w):
    from deepconvsep_b200.engine import Stft
    return Stft(ctx, N, H, w)


def test_golden_stft_istft(ctx, golden):
    g = golden
    for ci in range(int(g["n_stft"])):
        N, H = (int(v) for v in g["stft%d_NH" % ci])
        x, w, Xr = g["stft%d_x" % ci], g["stft%d_w" % ci], g["stft%d_X" % ci]
        st = _plan(ctx, N, H, w)
        xd = torch.tensor(x, dtype=torch.float32, device="cuda")
        X, mag = st.forward(xd, mag_scale=0.3)
        torch.cuda.synchronize()
        T, F = Xr.shape
        assert X.shape == (T, st.ldf)
        Xg = X.cpu().numpy()[:, :F].astype(np.complex128)
        assert rel(Xg, Xr) < 2e-6, (ci, rel(Xg, Xr))
        assert np.all(X.cpu().numpy()[:, F:] == 0) and np.all(mag.cpu().numpy()[:, F:] == 0)
        mref = 0.3 * (np.abs(Xr) / np.sqrt(N))
        assert rel(mag.cpu().numpy()[:, :F].astype(np.float64), mref) < 2e-6
        # inverse of the reference spectrum vs the reference's istft
        Z = g["stft%d_Z" % ci]
        for spec, want in ((Xr, g["stft%d_y" % ci]), (Z, g["stft%d_y2" % ci])):
            S = torch.zeros((1, T, st.ldf), dtype=torch.complex64, device="cuda")
            S[0, :, :F] = torch.tensor(spec.astype(np.complex64), device="cuda")
            y = st.inverse(S).cpu().numpy()[0].astype(np.float64)
            assert y.shape == want.shape
            # the last N/2 samples divide by sum(w^2) -> 0 (only the vanishing tail of the last
            # frame covers them): ill-conditioned in any precision and cut by data[:L] in the
            # pipeline.  Strict on the samples the pipeline keeps, loose on the full length.
            keep = x.size
            assert rel(y[:keep], want[:keep]) < 5e-6, (ci, rel(y[:keep], want[:keep]))
            assert rel(y, want) < 1e-4, (ci, rel(y, want))
        # GPU round trip reconstructs the signal
        y = st.inverse(X.unsqueeze(0), num_out=x.size).cpu().numpy()[0]
        assert rel(y.astype(np.float64), x) < 5e-6


def hamming(n):
    """for hop = N: every sample sees one frame, so sum(w^2) must stay away from 0 at the frame edges (a Hann window's
    vanishing edges make those samples ill-conditioned in any finite precision)"""
    return np.hamming(n)


@pytest.mark.parametrize("N,H,wname", [(1024, 512, "hanning"), (2048, 512, "hanning"), (4096, 512, "blackmanharris"),
                                       (1024, 256, "hanning"), (512, 256, "sinebell"), (256, 128, "hanning"),
                                       (256, 64, "hanning"), (512, 384, "hanning"), (1024, 128, "hanning"),
                                       (1024, 1024, "hamming"), (2048, 256, "sinebell"), (2048, 1536, "hanning"),
                                       (4096, 1024, "blackmanharris")])
def test_polar_compute_file_and_inverse(ctx, N, H, wname):
    """transformFFT.compute_file(phase=True) / compute_inverse semantics; hops that do not divide N, hop = N."""
    from deepconvsep_b200.engine import get_window
    rng = np.random.default_rng(N + H)
    x = rng.standard_normal(7777) * 0.1
    w = get_window(hamming if wname == "hamming" else wname, N)
    st = _plan(ctx, N, H, w)
    mag_r, ph_r = dsp.compute_file(x, phase=True, frameSize=N, hopSize=H, window=w)
    xd = torch.tensor(x, dtype=torch.float32, device="cuda")
    mag, ph = st.forward_polar(xd)
    F = N // 2 + 1
    mg, pg = mag.cpu().numpy()[:, :F].astype(np.float64), ph.cpu().numpy()[:, :F].astype(np.float64)
    assert rel(mg, mag_r) < 2e-6
    # phases compare as unit phasors weighted by magnitude (angle is ill-conditioned at |X| ~ 0)
    assert rel(mg * np.exp(1j * pg), mag_r * np.exp(1j * ph_r)) < 3e-6
    y_r = dsp.compute_inverse(mag_r * 0.5, ph_r, frameSize=N, hopSize=H, window=w)
    mt = torch.zeros((mag.shape[0], st.ldf), dtype=torch.float32, device="cuda")
    pt = torch.zeros_like(mt)
    mt[:, :F] = torch.tensor(mag_r * 0.5, dtype=torch.float32, device="cuda")
    pt[:, :F] = torch.tensor(ph_r, dtype=torch.float32, device="cuda")
    y = st.inverse_polar(mt, pt).cpu().numpy().astype(np.float64)
    assert y.shape == y_r.shape
    assert rel(y[:x.size], y_r[:x.size]) < 5e-6
    assert rel(y, y_r) < 1e-4          # includes the ill-conditioned tail (sum(w^2) -> 0)


def _normaliser(w, N, H, T):
    """istft_norm's sum of window * analysis window per output sample (transform.py:384-392), leading N/2 dropped"""
    c = np.zeros(H * (T - 1) + N)
    for n in range(T):
        c[n * H:n * H + N] += w * w
    return c[N // 2:]


SENTINEL = np.float32(-12345.5)


@pytest.mark.parametrize("N,H,wname", [(256, 64, "hanning"), (512, 384, "hanning"), (1024, 128, "hanning"),
                                       (1024, 1024, "hamming"), (2048, 256, "hanning"), (2048, 1536, "hanning"),
                                       (4096, 1024, "blackmanharris"), (1024, 256, "hanning"), (1024, 512, "hanning"),
                                       (2048, 512, "hanning")])
def test_complex_stft_and_istft_dispatch(ctx, N, H, wname):
    """dcs_stft_forward / dcs_istft on complex spectra vs stft_norm / istft_norm, at clip lengths around one hop and one
    frame.  The forward STFT gives the same bits from an audio pointer one float off 8-byte alignment (the interior fast
    path and the bounds-checked path form the same products).  The inverse reads 3 sources src_stride = T * ldf + 24
    apart whose pad columns and stride gaps hold NaN (never read), and writes them with an even out_stride (the register
    kernel for N = 1024 / 2048 with hop 256 / 512), an odd one and an unaligned output pointer (both force the
    shared-memory kernel); the gaps between the output rows keep a sentinel."""
    from deepconvsep_b200.engine import get_window, _ptr, _stream_ptr
    from deepconvsep_b200._lib import check
    w = get_window(hamming if wname == "hamming" else wname, N)
    st = _plan(ctx, N, H, w)
    F, ldf, nsrc = N // 2 + 1, st.ldf, 3
    rng = np.random.default_rng(7 * N + H)
    worst = dict(forward=0.0, inverse_well_conditioned=0.0, inverse_all=0.0)
    for L in (1, H - 1, N // 2 + 1, N + 3, 10 * H + 1):
        T = dsp.num_frames(L, H)
        # ---- forward, aligned and one float off
        x = (rng.standard_normal(L) * 0.1).astype(np.float32)
        xa = torch.zeros(L + 1, dtype=torch.float32, device="cuda")
        xu = torch.zeros(L + 1, dtype=torch.float32, device="cuda")
        xa[:L] = torch.from_numpy(x).cuda()
        xu[1:] = torch.from_numpy(x).cuda()
        Xa, ma = st.forward(xa[:L], mag_scale=0.3)
        Xu, mu = st.forward(xu[1:], mag_scale=0.3)
        torch.cuda.synchronize()
        assert torch.equal(torch.view_as_real(Xa), torch.view_as_real(Xu)) and torch.equal(ma, mu), L
        Xr = dsp.stft_norm(x.astype(np.float64), window=w, hopsize=float(H), nfft=float(N))
        Xg, mg = Xa.cpu().numpy(), ma.cpu().numpy()
        assert Xg.shape == (T, ldf) == Xr.shape[:1] + (ldf,)
        ex, em = rel(Xg[:, :F].astype(np.complex128), Xr), rel(mg[:, :F].astype(np.float64), 0.3 * np.abs(Xr) / np.sqrt(N))
        worst["forward"] = max(worst["forward"], ex, em)
        assert ex < 2e-6 and em < 2e-6, (L, ex, em)
        assert np.all(Xg[:, F:] == 0) and np.all(mg[:, F:] == 0)

        # ---- inverse of 3 random spectra, NaN in every element outside the [T, F] planes
        src_stride = T * ldf + 24
        Z = (rng.standard_normal((nsrc, T, F)) + 1j * rng.standard_normal((nsrc, T, F))).astype(np.complex64)
        S = torch.full((nsrc * src_stride,), complex(float("nan"), float("nan")), dtype=torch.complex64, device="cuda")
        for s in range(nsrc):
            S[s * src_stride:s * src_stride + T * ldf].view(T, ldf)[:, :F] = torch.from_numpy(Z[s]).cuda()
        want = [dsp.istft_norm(Z[s].astype(np.complex128), window=w, analysisWindow=w, hopsize=float(H), nfft=float(N))
                for s in range(nsrc)]
        Lmax = (T - 1) * H + N // 2
        assert want[0].size == Lmax
        c = _normaliser(w, N, H, T)
        for Lout in (L, Lmax):                 # odd num_out (every L here is odd), and the maximum
            good = c[:Lout] >= 1e-3 * c.max()      # away from the vanishing window tails at the ends
            assert good.mean() > 0.5
            even = Lout + Lout % 2 + 4
            for stride, off in ((even, 0), (even + 1, 0), (even, 1)):
                out = torch.full((nsrc * stride + 2,), float(SENTINEL), dtype=torch.float32, device="cuda")
                check(ctx.lib.dcs_istft(st.handle, _ptr(S), nsrc, T, ldf, src_stride, out.data_ptr() + 4 * off, Lout, stride,
                                        _stream_ptr(None, ctx.device)))
                torch.cuda.synchronize()
                o = out.cpu().numpy()
                written = np.zeros(o.size, bool)
                for s in range(nsrc):
                    a = off + s * stride
                    written[a:a + Lout] = True
                    y = o[a:a + Lout].astype(np.float64)
                    ref = want[s][:Lout]
                    tag = (L, Lout, stride, off, s)
                    assert np.isfinite(y).all(), tag
                    eg, ea = rel(y[good], ref[good]), rel(y, ref)
                    worst["inverse_well_conditioned"] = max(worst["inverse_well_conditioned"], eg)
                    worst["inverse_all"] = max(worst["inverse_all"], ea)
                    assert eg < 5e-6 and ea < 1e-4, (tag, eg, ea)
                assert np.all(o[~written].view(np.int32) == SENTINEL.view(np.int32)), (L, Lout, stride, off)
    record("stft_complex_N%d_H%d_%s" % (N, H, wname), **worst)


def test_large_roundtrip_property(ctx):
    """Full-size (180 s @ 44.1 kHz) size-independent property: istft(stft(x)) == x."""
    st = _plan(ctx, 2048, 512, np.hanning)
    g = torch.Generator(device="cuda").manual_seed(5)
    x = (torch.rand(7938000, generator=g, device="cuda") - 0.5) * 0.4
    X, _ = st.forward(x, want_mag=False)
    assert X.shape[0] == 15506
    y = st.inverse(X.unsqueeze(0), num_out=x.numel())[0]
    err = (torch.linalg.vector_norm(y - x) / torch.linalg.vector_norm(x)).item()
    assert err < 5e-6, err
    # linearity of the analysis: stft(a*x) == a*stft(x) bit-exactly for a power of two
    X2, _ = st.forward(x * 0.5, want_mag=False)
    assert torch.equal(torch.view_as_real(X2), torch.view_as_real(X) * 0.5)
