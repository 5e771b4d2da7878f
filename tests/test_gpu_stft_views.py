"""The forward STFT (K1: stft.cu at N = 256 / 512 / 4096, stft_reg.cu at 1024 / 2048) and the inverse STFT with
overlap-add (K4: istft_reg_kernel at N = 1024 / 2048 with hop 256 / 512, istft_kernel everywhere else and for the polar
entry) against a float64 reference, element by element, through dcs_stft_forward, dcs_stft_forward_polar, dcs_istft
and dcs_istft_polar.

The reference and the bounds are tests/stft_views_oracle.py (its docstring derives them; tests/test_stft_views_host.py
pins the reference to oracle.dsp and the golden vectors and shows the bounds reject index and arithmetic mutations).

Forward cases: every N, hops 2, 6, N/4, N/2, N - 2 and N; clip lengths whose frame counts take every residue modulo the
frames per CTA (8 for stft.cu, 32 / 16 for stft_reg.cu's <16> / <32>), L = 1, L < N, a frame starting at sample 0 and
one ending at sample L, a longer clip and a 180 s clip at 2048/512; ldf = F, F + 1, dcs_padded_bins and F + 16; the audio
pointer 8-byte aligned and one float off; white noise, a loud segment next to a 2e-5 one, tones on and between bins, a DC
offset, the +-1 Nyquist sequence, int16-quantised audio and all zeros (exact zeros out).  Every case runs X only, mag
only, X + mag and the polar mag + phase, and what is written must be the same bits in every combination.

Inverse cases: istft_reg_kernel at its four (N, hop) pairs with 1, 3 and 9 sources, hops per group 12 (several seams in
the clip), in between and 64 (the source and hop counts are chosen from the device's SM count), and one frame of large
magnitude on each side of every seam; istft_kernel at every other (N, hop), and at the register kernel's pairs when an
odd ldf, an odd out_stride, an output pointer one float off or a spectrum pointer 8- but not 16-byte aligned moves them
there; num_out in {1, 2, H - 1, H, H + 1, max - 1, max} and one that leaves the last group partial; hann analysis with
hann, sinebell or Blackman-Harris synthesis; the polar entry with mag_scale 0.7.

Fences and exact parts.  The SLACK elements before and after the audio hold NaN, and so do every spectrum element the
kernels must not use: pad columns, source-stride gaps and the imaginary parts of DC and Nyquist.  Outputs are pre-filled
with a NaN-payload sentinel; the SLACK elements around every output and the inverse's output-stride gaps must keep their
bits.  Stored values must be finite, pad columns exact zeros, X at DC and Nyquist must have an imaginary part of exactly
+0, and the phase there must be exactly 0 or float32(pi).  Each case runs twice and must give the same bits.

Second tier: each case's bound-relative RMS error over that of scipy's float32 FFT on the same frames
(stft_views_oracle.rms_ratio) must stay within RMS_BAR, set to 2x the worst ratio measured on an H100 (see
stft_views_oracle.RMS_BAR); cases with fewer than 2048 compared elements are recorded, not held to it.  With
DCS_TEST_RECORDS set every test records its worst error / bound and RMS ratio per kernel (tests/parity.py)."""
import os
import sys
import zlib

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import stft_views_oracle as so  # noqa: E402
from parity import record  # noqa: E402

SLACK = so.SLACK
SENT = np.uint32(0x7FC5A5A5)      # quiet NaN with a payload no kernel produces
PI32 = np.float32(np.pi)
MIN_TIER = 2048


@pytest.fixture(scope="module")
def ctx():
    from deepconvsep_b200.engine import Context
    return Context(0)


_PLANS = {}


def _plan(ctx, N, H, syn="hanning"):
    from deepconvsep_b200.engine import Stft
    key = (id(ctx), N, H, syn)
    if key not in _PLANS:
        _PLANS[key] = Stft(ctx, N, H, "hanning", syn_window=None if syn == "hanning" else syn)
    return _PLANS[key]


def _stream(ctx):
    from deepconvsep_b200.engine import _stream_ptr
    return _stream_ptr(None, ctx.device)


def _sentinels(n):
    return torch.from_numpy(np.full(n, SENT, np.uint32).view(np.float32)).cuda()


def _bits(t):
    return t.cpu().numpy().view(np.uint32)


class Stats:
    def __init__(self):
        self.worst = 0.0
        self.rms = 0.0
        self.cases = 0

    def add(self, worst, rms):
        self.worst = max(self.worst, worst)
        self.rms = max(self.rms, rms)
        self.cases += 1


def _tier(e_kernel, e_base, bound):
    ok = (bound > 0) & (e_base > 0)
    return so.rms_ratio(e_kernel, e_base, bound), int(ok.sum())


# ---------------------------------------------------------------------------------------------- forward
COMBOS = ("X", "mag", "Xmag", "polar")


def _forward_run(ctx, st, aptr, L, T, ldf, combo):
    n = T * ldf
    Xb = _sentinels(2 * (n + 2 * SLACK))
    mb = _sentinels(n + 2 * SLACK)
    pb = _sentinels(n + 2 * SLACK)
    Xp = Xb.data_ptr() + 8 * SLACK if combo in ("X", "Xmag") else None
    mp = mb.data_ptr() + 4 * SLACK
    pp = pb.data_ptr() + 4 * SLACK
    if combo == "polar":
        r = ctx.lib.dcs_stft_forward_polar(st.handle, aptr, L, mp, pp, so.SCALE, ldf, _stream(ctx))
    else:
        r = ctx.lib.dcs_stft_forward(st.handle, aptr, L, Xp, mp if combo != "X" else None, so.SCALE, ldf, _stream(ctx))
    assert r == 0, (combo, r)
    torch.cuda.synchronize()
    return _bits(Xb), _bits(mb), _bits(pb)


def _check_fenced(buf, body_len, written, tag):
    """buf uint32 with SLACK * k fences; written: whether the body was an output of this call"""
    k = (buf.size - body_len) // 2
    if not written:
        assert (buf == SENT).all(), ("buffer not passed was written", tag)
        return None
    assert (buf[:k] == SENT).all() and (buf[k + body_len:] == SENT).all(), ("fence overwritten", tag)
    return buf[k:k + body_len]


def forward_case(ctx, N, H, case, stats):
    L, ldf, off, kind = case["L"], case["ldf"], case["off"], case["signal"]
    F = N // 2 + 1
    st = _plan(ctx, N, H)
    w = st.window
    x = so.signal(kind, L, N, np.random.default_rng(zlib.crc32(("%d/%d/%d/%s" % (N, H, L, kind)).encode())))
    a = np.full(L + 2 * SLACK + 1, np.nan, np.float32)
    a[SLACK + off:SLACK + off + L] = x
    ad = torch.from_numpy(a).cuda()
    aptr = ad.data_ptr() + 4 * (SLACK + off)
    T = so.num_frames(L, H)
    n = T * ldf
    tag = (N, H, L, kind, ldf, off)
    got = {}
    for combo in COMBOS:
        r1 = _forward_run(ctx, st, aptr, L, T, ldf, combo)
        r2 = _forward_run(ctx, st, aptr, L, T, ldf, combo)
        assert all(np.array_equal(p, q) for p, q in zip(r1, r2)), ("two runs gave different bits",) + tag + (combo,)
        Xb = _check_fenced(r1[0], 2 * n, combo in ("X", "Xmag"), tag + (combo, "X"))
        mb = _check_fenced(r1[1], n, combo != "X", tag + (combo, "mag"))
        pb = _check_fenced(r1[2], n, combo == "polar", tag + (combo, "phase"))
        got[combo] = (Xb, mb, pb)
    # the same bits in every combination
    assert np.array_equal(got["X"][0], got["Xmag"][0]), tag
    assert np.array_equal(got["mag"][1], got["Xmag"][1]) and np.array_equal(got["mag"][1], got["polar"][1]), tag
    Xbits = got["X"][0].reshape(T, ldf, 2)
    mbits = got["mag"][1].reshape(T, ldf)
    pbits = got["polar"][2].reshape(T, ldf)
    # exact parts: pad columns +0, Im of DC and Nyquist +0, finite values, phase at DC / Nyquist 0 or float32(pi)
    assert (Xbits[:, F:] == 0).all() and (mbits[:, F:] == 0).all() and (pbits[:, F:] == 0).all(), ("pad columns",) + tag
    assert (Xbits[:, 0, 1] == 0).all() and (Xbits[:, F - 1, 1] == 0).all(), ("Im of DC / Nyquist is not +0",) + tag
    Xv = Xbits[:, :F].view(np.float32)
    mv, pv = mbits[:, :F].view(np.float32), pbits[:, :F].view(np.float32)
    assert np.isfinite(Xv).all() and np.isfinite(mv).all() and np.isfinite(pv).all(), ("not finite",) + tag
    for col in (0, F - 1):
        assert np.isin(pv[:, col], (np.float32(0), PI32)).all(), ("phase of a real bin",) + tag
    Xg = Xv[..., 0].astype(np.float64) + 1j * Xv[..., 1].astype(np.float64)
    Xr, A = so.stft_ref(x, w, N, H)
    if kind == "zeros":
        assert (Xv == 0).all() and (mv == 0).all(), ("zeros in, zeros out",) + tag
    worst, fails = so.check_forward(Xg, mv, pv, Xr, A, N, so.SCALE)
    assert not fails, tag + tuple(fails[:4])
    b = so.forward_bounds(A, N)[:, None] * np.ones((1, F))
    ratio, cnt = _tier(np.abs(Xg - Xr), np.abs(so.stft_f32(x, w, N, H).astype(np.complex128) - Xr), b)
    held = cnt >= MIN_TIER
    stats.add(worst, ratio if held else 0.0)
    if held:
        assert ratio <= so.RMS_BAR, ("RMS ratio over the float32 FFT",) + tag + (ratio,)


def _fwd_path(N):
    return "stft_reg.cu" if so.forward_reg(N) else "stft.cu"


@pytest.mark.parametrize("N,H", [(N, H) for N in so.SIZES for H in so.hops(N)])
def test_forward_matches_float64(ctx, N, H):
    stats = Stats()
    for case in so.forward_cases(N, H):
        forward_case(ctx, N, H, case, stats)
    record("stft_view:forward_N%d_H%d" % (N, H), path=_fwd_path(N), cases=stats.cases,
           worst_error_over_bound=stats.worst, worst_rms_ratio=stats.rms)


def test_forward_180s(ctx):
    """a 180 s clip at 2048/512 (15,506 frames), the DSD100 configuration"""
    stats = Stats()
    forward_case(ctx, 2048, 512, dict(L=180 * 44100, signal="white", ldf=so.padded_bins(2048), off=0), stats)
    record("stft_view:forward_180s", path="stft_reg.cu", worst_error_over_bound=stats.worst, worst_rms_ratio=stats.rms)


# ---------------------------------------------------------------------------------------------- inverse
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _inv_path(case, reg):
    return "polar" if case["polar"] else ("istft_reg_kernel" if reg else "istft_kernel")


def inverse_case(ctx, case):
    N, H, T, nsrc = case["N"], case["H"], case["T"], case["nsrc"]
    F = N // 2 + 1
    ldf, src_stride, out_stride, s_off, o_off, reg = so.inverse_layout(case)
    st = _plan(ctx, N, H, case["syn"])
    w, s = st.window, so.window(case["syn"], N)
    spec = so.inverse_spectra(case, np.random.default_rng(zlib.crc32(case["name"].encode())))
    cI = so.c_inverse(N, reg, case["polar"])
    if case["polar"]:
        mag, ph = spec
        Sref = [so.polar_spectrum(mag, ph, case["scale"], N)]
        bufs = []
        for v in (mag, ph):
            b = np.full(T * ldf + 2 * SLACK, np.nan, np.float32)
            b[SLACK:SLACK + T * ldf].reshape(T, ldf)[:, :F] = v
            bufs.append(torch.from_numpy(b).cuda())
        nsrc = 1
    else:
        Sref = list(spec)
        b = np.full((2 * SLACK + s_off + nsrc * src_stride, 2), np.nan, np.float32)
        for k in range(nsrc):
            rows = b[SLACK + s_off + k * src_stride:SLACK + s_off + k * src_stride + T * ldf].reshape(T, ldf, 2)
            rows[:, :F, 0], rows[:, :F, 1] = spec[k].real, spec[k].imag
            rows[:, 0, 1] = np.nan                   # never read: irfft drops Im of DC and Nyquist
            rows[:, F - 1, 1] = np.nan
        Sd = torch.from_numpy(b).cuda()
        sptr = Sd.data_ptr() + 8 * (SLACK + s_off)
    refs = [so.istft_ref(Sk, s, w, H, N, cI, polar=case["polar"]) for Sk in Sref]
    mx = (T - 1) * H + N // 2
    stats_rms, worst = 0.0, 0.0
    for num_out in case["outs"]:
        stride = num_out if case["polar"] else out_stride
        tag = (case["name"], num_out)

        def run():
            ob = _sentinels(2 * SLACK + o_off + nsrc * stride)
            optr = ob.data_ptr() + 4 * (SLACK + o_off)
            if case["polar"]:
                r = ctx.lib.dcs_istft_polar(st.handle, ctx.handle, bufs[0].data_ptr() + 4 * SLACK,
                                            bufs[1].data_ptr() + 4 * SLACK, case["scale"], T, ldf, optr, num_out,
                                            _stream(ctx))
            else:
                r = ctx.lib.dcs_istft(st.handle, sptr, nsrc, T, ldf, src_stride, optr, num_out, stride, _stream(ctx))
            assert r == 0, tag
            torch.cuda.synchronize()
            return _bits(ob)
        o1 = run()
        assert np.array_equal(o1, run()), ("two runs gave different bits",) + tag
        written = np.zeros(o1.size, bool)
        for k in range(nsrc):
            a0 = SLACK + o_off + k * stride
            written[a0:a0 + num_out] = True
        assert (o1[~written] == SENT).all(), ("%d fence / gap elements changed" % int((o1[~written] != SENT).sum()),) + tag
        for k in range(nsrc):
            a0 = SLACK + o_off + k * stride
            yg = o1[a0:a0 + num_out].view(np.float32)
            assert np.isfinite(yg).all(), ("not finite", k) + tag
            y, bd = refs[k]
            e = np.abs(yg.astype(np.float64) - y[:num_out])
            r = so.ratio(e, bd[:num_out])
            worst = max(worst, float(r.max()))
            assert r.max() <= 1.0, ("error over bound", k, float(r.max()), int(np.argmax(r))) + tag
            if num_out == mx:
                Sk = Sref[k].astype(np.complex64) if case["polar"] else Sref[k]
                eb = np.abs(so.istft_f32(Sk, s, w, H, N).astype(np.float64) - y)
                ratio, cnt = _tier(e, eb, bd)
                if cnt >= MIN_TIER:
                    stats_rms = max(stats_rms, ratio)
                    assert ratio <= so.RMS_BAR, ("RMS ratio over the float32 FFT", k, ratio) + tag
    record("stft_view:inverse_" + case["name"], path=_inv_path(case, reg), nsrc=nsrc, hpg=case["seam"],
           worst_error_over_bound=worst, worst_rms_ratio=stats_rms)


_INV = {c["name"]: c for c in so.inverse_cases()}


@pytest.mark.parametrize("name", list(_INV))
def test_inverse_matches_float64(ctx, name):
    inverse_case(ctx, {c["name"]: c for c in so.inverse_cases(_sms())}[name])


# ---------------------------------------------------------------------------------------------- refusals
def test_refusals_queue_nothing(ctx):
    """each bad call returns DCS_EINVAL with nothing launched and every buffer untouched"""
    N, H = 1024, 256
    st = _plan(ctx, N, H)
    F, ldf, T, L = N // 2 + 1, so.padded_bins(N), 12, 9 * H
    S = _sentinels(2 * (2 * T * ldf + 2 * SLACK))
    out = _sentinels(2 * L + 2 * SLACK)
    X = _sentinels(2 * (T * ldf + 2 * SLACK))
    audio = torch.zeros(L, dtype=torch.float32, device="cuda")
    sp, op = S.data_ptr() + 8 * SLACK, out.data_ptr() + 4 * SLACK
    n0 = ctx.launch_count()
    lib, h, stream = ctx.lib, st.handle, _stream(ctx)
    bad = [
        lib.dcs_istft(h, sp, 1, T, F - 1, T * ldf, op, L, L, stream),             # ldf < N/2 + 1
        lib.dcs_istft(h, sp, 2, T, ldf, T * ldf - 1, op, L, L, stream),           # sources share spectrum rows
        lib.dcs_istft(h, sp, 2, T, ldf, T * ldf, op, L, L - 1, stream),           # sources share output samples
        lib.dcs_istft(h, sp, 1, T, ldf, -1, op, L, L, stream),                    # negative strides
        lib.dcs_istft(h, sp, 1, T, ldf, T * ldf, op, L, -1, stream),
        lib.dcs_istft(h, sp + 4, 1, T, ldf, T * ldf, op, L, L, stream),           # d_S not 8-byte aligned
        lib.dcs_istft_polar(h, ctx.handle, op, op, 1.0, T, F - 1, op, L, stream),  # ldf < N/2 + 1
        lib.dcs_stft_forward(h, audio.data_ptr(), L, X.data_ptr() + 8 * SLACK + 4, None, 1.0, ldf, stream),  # d_X
    ]
    torch.cuda.synchronize()
    assert bad == [-1] * len(bad), bad
    assert ctx.launch_count() == n0
    for b in (S, out, X):
        assert (_bits(b) == SENT).all()
