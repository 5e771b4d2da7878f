"""The int16 conversion kernels element by element against the exact host reference of tests/pcm16_oracle.py, through
the test entries dcs_pcm16_decode / dcs_pcm16_encode / dcs_downmix_f32 (one launch of the kernel the int16 batch entry
points run, on fenced caller buffers).  Every output is compared bit for bit, every case runs twice with the same bits,
and the values around every output (NaN payloads for fp32, 0x5A5A for int16) stay unchanged.

- decode (pcm_decode_kernel): channels 1..8 x downmix 0..2; (pcm_decode_channels_kernel) C 1..16; every int16 value in
  every channel position, L in {1, 255, 256, 257, 4099} and a 180 s clip; (downmix_kernel) nx 1..16 float planes with
  NaN gaps, subnormals and sums that overflow;
- encode (pcm_encode_kernel): nsrc 1..4, out_stride > L; (pcm_encode_channels_kernel) C 1..16, nsrc 1..4, every
  destination shift 0..7 (the output's byte offset modulo 16, over 2), L around the 256-row tile; the stem values of
  pcm16_oracle.stem_values (k / 32767, neighbours of every integer boundary, past full scale up to +-65537, +-0,
  subnormals, NaN, +-inf, +-3e9) and NaN in the gaps between stem planes;
- fused (resample_decode_pcm16_kernel, resample_encode_pcm16_kernel): every rate of the resampler's table in both
  directions, C 1..16 at 48 kHz and {1, 2, 5, 16} elsewhere, lengths of 1, 7, half the filter and one tile +-1; full-range
  random int16 and +-32767 square waves whose resampled planes overshoot 1.0.  Channel planes are the bits of
  dcs_resample on pcm / 32767 and meet the float64 bound of tests/test_gpu_resample.py; the downmix is the reference's
  on them; the encode is the reference's of dcs_resample's fp32 output;
- end to end at full scale: a clip reaching -32768 and 32767 through every int16 batch entry point equals the
  reference encode of the float route, bit for bit, with stems that wrap."""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import pcm16_oracle as po  # noqa: E402
import resample_oracle as ro  # noqa: E402
from parity import record  # noqa: E402

NAN_IN = np.uint32(0x7fc0beef)      # fp32 the kernels must not read
NAN_OUT = np.uint32(0x7fc0dead)     # fp32 the kernels must not write
PAD = 64                            # fence values on either side of an output (a multiple of 8)


@pytest.fixture(scope="module")
def ctx():
    from deepconvsep_b200.engine import Context
    return Context(0)


@pytest.fixture(scope="module")
def resamplers(ctx):
    from deepconvsep_b200.engine import Resampler
    made = {}

    def get(rate_in, rate_out):
        if (rate_in, rate_out) not in made:
            made[rate_in, rate_out] = Resampler(ctx, rate_in, rate_out)
        return made[rate_in, rate_out]
    return get


def _lib():
    from deepconvsep_b200 import _lib
    return _lib


def _fenced_f32(n):
    return torch.from_numpy(np.full(2 * PAD + n, NAN_OUT, dtype=np.uint32).view(np.int32)).cuda()


def _f32_planes(a, gap):
    """float32 [P, L] -> (device buffer, pointer of plane 0, stride): NaN payloads before, between and after the planes"""
    P, L = a.shape
    stride = L + gap
    buf = np.full(PAD + P * stride + PAD, NAN_IN, dtype=np.uint32)
    buf[PAD:PAD + P * stride].reshape(P, stride)[:, :L] = np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)
    d = torch.from_numpy(buf.view(np.int32)).cuda()
    return d, d.data_ptr() + 4 * PAD, stride


def _pcm_in(pcm):
    """int16 [L, C] -> (device buffer, pointer): 0x5A5A before and after"""
    buf = np.full(2 * PAD + pcm.size, po.SENTINEL, dtype=np.int16)
    buf[PAD:PAD + pcm.size] = pcm.ravel()
    d = torch.from_numpy(buf).cuda()
    return d, d.data_ptr() + 2 * PAD


def decode(ctx, pcm, mode, rs=None, num_out=None):
    """-> (uint32 bits [P, num_out], fences intact)"""
    lib = _lib()
    L, nch = pcm.shape
    n = L if num_out is None else num_out
    P = nch + 1 if mode == lib.PCM16_CHANNELS else 1
    din, pin = _pcm_in(pcm)
    out = _fenced_f32(P * n)
    lib.check(ctx.lib.dcs_pcm16_decode(ctx.handle, rs.handle if rs else None, mode, pin, L, nch,
                                       out.data_ptr() + 4 * PAD, n, None))
    raw = out.cpu().numpy().view(np.uint32)
    fenced = bool(np.all(raw[:PAD] == NAN_OUT) and np.all(raw[PAD + P * n:] == NAN_OUT))
    return raw[PAD:PAD + P * n].reshape(P, n).copy(), fenced


def encode(ctx, stems, nsrc, mode, shift, rs=None, num_out=None, gap=0, out_gap=0):
    """stem planes float32 [nsrc * C, num_in] -> (int16 [nsrc, num_out * C], fences intact); the output starts `shift`
    values past a 16-byte boundary, sources out_gap values apart beyond their own (mono mode)"""
    lib = _lib()
    P, Lin = stems.shape
    nch = P // nsrc
    n = Lin if num_out is None else num_out
    din, pst, stride = _f32_planes(stems, gap)
    ostride = nch * n + out_gap
    total = nsrc * ostride
    out = torch.from_numpy(np.full(2 * PAD + total + 8, po.SENTINEL, dtype=np.int16)).cuda()
    assert out.data_ptr() % 16 == 0
    lib.check(ctx.lib.dcs_pcm16_encode(ctx.handle, rs.handle if rs else None, mode, pst, Lin, nsrc, nch, stride,
                                       out.data_ptr() + 2 * (PAD + shift), n, ostride, None))
    raw = out.cpu().numpy()[shift:]
    body = raw[PAD:PAD + total].reshape(nsrc, ostride)
    fences = np.concatenate([raw[:PAD], raw[PAD + total:PAD + total + PAD], body[:, nch * n:].ravel()])
    return body[:, :nch * n].copy(), bool(np.all(fences == po.SENTINEL))


def _cuda_planes(a):
    """float32 [P, L] -> cuda tensor with rows one after the other (numpy may keep any stride on a length-1 axis)"""
    t = torch.empty(a.shape, dtype=torch.float32, device="cuda")
    t.copy_(torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)))
    return t


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _twice(fn):
    a, fa = fn()
    b, fb = fn()
    assert fa and fb, "a fence changed"
    assert a.tobytes() == b.tobytes(), "two runs differ"
    return a


def _random_pcm(rng, L, nch):
    pcm = rng.integers(-32768, 32768, (L, nch)).astype(np.int16)
    pcm[rng.integers(0, L, max(1, L // 64)), :] = -32768
    pcm[rng.integers(0, L, max(1, L // 64)), :] = 32767
    return pcm


LENGTHS = (1, 255, 256, 257, 4099)


# ---------------------------------------------------------------------------------------------- 1. decode
@pytest.mark.parametrize("channels", range(1, 9))
def test_decode_mono_modes(ctx, channels):
    rng = np.random.default_rng(channels)
    clips = [po.all_int16(channels)] + [_random_pcm(rng, L, channels) for L in LENGTHS]
    for mode in (0, 1, 2):
        for pcm in clips:
            got = _twice(lambda: decode(ctx, pcm, mode))
            want = _bits(po.decode_mono(pcm, mode))[None]
            assert got.tobytes() == want.tobytes(), (channels, mode, pcm.shape, int(np.sum(got != want)))


@pytest.mark.parametrize("nch", range(1, 17))
def test_decode_channels(ctx, nch):
    rng = np.random.default_rng(100 + nch)
    for pcm in [po.all_int16(nch)] + [_random_pcm(rng, L, nch) for L in LENGTHS]:
        got = _twice(lambda: decode(ctx, pcm, _lib().PCM16_CHANNELS))
        want = _bits(po.decode_channels(pcm))
        assert got.tobytes() == want.tobytes(), (nch, pcm.shape, np.argwhere(got != want)[:4].tolist())


def test_decode_180_s(ctx):
    rng = np.random.default_rng(180)
    pcm = _random_pcm(rng, 180 * 44100, 2)
    got = _twice(lambda: decode(ctx, pcm, _lib().PCM16_CHANNELS))
    assert got.tobytes() == _bits(po.decode_channels(pcm)).tobytes()
    for mode in (1, 2):
        got = _twice(lambda: decode(ctx, pcm, mode))
        assert got.tobytes() == _bits(po.decode_mono(pcm, mode))[None].tobytes(), mode


@pytest.mark.parametrize("nx", range(1, 17))
def test_downmix_float_planes(ctx, nx):
    rng = np.random.default_rng(200 + nx)
    edges = np.float32([1e-45, -1e-45, 3e-45, 1.2e-38, 3e38, -3e38, 1.7e38, 0.0, -0.0, 1.0])
    for L in (1, 255, 257, 4099):
        a = rng.uniform(-1.0, 1.0, (nx, L)).astype(np.float32)
        a[:, rng.integers(0, L, max(1, L // 8))] = rng.choice(edges, (nx, 1))
        if L > 3:
            a[:, :3] = edges[[0, 4, 6]][None, :].repeat(nx, 0)
        din, pin, stride = _f32_planes(a, 3 + nx)

        def run():
            out = _fenced_f32(L)
            _lib().check(ctx.lib.dcs_downmix_f32(ctx.handle, pin, nx, stride, L, out.data_ptr() + 4 * PAD, None))
            raw = out.cpu().numpy().view(np.uint32)
            return raw[PAD:PAD + L].copy(), bool(np.all(raw[:PAD] == NAN_OUT) and np.all(raw[PAD + L:] == NAN_OUT))
        got = _twice(run)
        want = _bits(po.downmix(a))
        assert got.tobytes() == want.tobytes(), (nx, L, np.argwhere(got != want)[:4].tolist())


# ---------------------------------------------------------------------------------------------- 2. encode
VALUES = po.stem_values()


def _stems(rng, P, L):
    return rng.choice(VALUES, (P, L)).astype(np.float32)


def _all_values(rng, P):
    """[P, L] stem planes holding every value of VALUES at least once"""
    L = -(-VALUES.size // P)
    return np.resize(rng.permutation(VALUES), (P, L)).astype(np.float32)


@pytest.mark.parametrize("nsrc", range(1, 5))
def test_encode_mono(ctx, nsrc):
    rng = np.random.default_rng(300 + nsrc)
    cases = [_all_values(rng, nsrc)] + [_stems(rng, nsrc, L) for L in LENGTHS]
    for k, stems in enumerate(cases):
        shift, gap, out_gap = k % 8, (k * 5) % 11, (k * 3) % 7 + (nsrc > 1)
        got = _twice(lambda: encode(ctx, stems, nsrc, _lib().PCM16_MONO, shift, gap=gap, out_gap=out_gap))
        want = po.encode(stems)
        assert got.tobytes() == want.tobytes(), (nsrc, stems.shape, np.argwhere(got != want)[:4].tolist())


ENC_LENGTHS = (1, 7, 255, 256, 257, 513)


@pytest.mark.parametrize("nch", range(1, 17))
def test_encode_channels(ctx, nch):
    """every shift 0..7 at every length, nsrc 1..4 in turn; then every stem value"""
    rng = np.random.default_rng(400 + nch)
    k = 0
    for shift in range(8):
        for L in ENC_LENGTHS:
            nsrc = 1 + k % 4
            k += 1
            stems = _stems(rng, nsrc * nch, L)
            got = _twice(lambda: encode(ctx, stems, nsrc, _lib().PCM16_CHANNELS, shift, gap=1 + k % 9))
            want = po.interleave(stems, nsrc).reshape(nsrc, -1)
            assert got.tobytes() == want.tobytes(), (nch, nsrc, L, shift, np.argwhere(got != want)[:4].tolist())
    for nsrc in (1, 4):
        stems = _all_values(rng, nsrc * nch)
        got = _twice(lambda: encode(ctx, stems, nsrc, _lib().PCM16_CHANNELS, (nch + nsrc) % 8, gap=5))
        assert got.tobytes() == po.interleave(stems, nsrc).reshape(nsrc, -1).tobytes(), (nch, nsrc)


# ---------------------------------------------------------------------------------------------- 3. fused with the resampler
def _rate_cases():
    for rate in ro.TABLE_RATES:
        for direction in ("in", "back"):
            yield rate, direction


def _channel_set(rate):
    return range(1, 17) if rate == 48000 else (1, 2, 5, 16)


def _bound(x64, up, down, h):
    Q = -(-h.size // up)
    y = ro.direct(x64, up, down, h)
    return y, 2.0 ** -24 * np.abs(y) + 2 * Q * 2.0 ** -53 * ro.direct(np.abs(x64), up, down, np.abs(h))


def _square(L, nch, period):
    t = np.arange(L)[:, None] + 3 * np.arange(nch)[None, :]
    return np.where((t // period) % 2 == 0, 32767, -32767).astype(np.int16)


@pytest.mark.parametrize("rate,direction", list(_rate_cases()))
def test_fused_decode(ctx, resamplers, rate, direction):
    rate_in, rate_out = (rate, ro.MODEL_RATE) if direction == "in" else (ro.MODEL_RATE, rate)
    rs = resamplers(rate_in, rate_out)
    up, down, h = rs.up, rs.down, rs.taps
    rng = np.random.default_rng(rate + (direction == "back"))
    worst, overshoot = 0.0, 0
    for nch in _channel_set(rate):
        for k, (Lin, Lout) in enumerate(po.fused_lengths(up, down, nch, False)):
            pcm = _random_pcm(rng, Lin, nch) if k % 2 == 0 else _square(Lin, nch, 5 + k)
            got = _twice(lambda: decode(ctx, pcm, _lib().PCM16_CHANNELS, rs, Lout))
            a = np.ascontiguousarray(po.decode(pcm).T)
            planes = rs.resample(_cuda_planes(a), num_out=Lout).cpu().numpy()
            want = np.concatenate([po.downmix(planes)[None], planes])
            assert got.tobytes() == _bits(want).tobytes(), (rate, direction, nch, Lin, Lout,
                                                             np.argwhere(got != _bits(want))[:4].tolist())
            y, bound = _bound(a.astype(np.float64), up, down, h)
            err = np.abs(got[1:].view(np.float32).astype(np.float64) - y[:, :Lout])
            assert np.all(err <= bound[:, :Lout]), (rate, direction, nch, Lin)
            worst = max(worst, float(np.max(err / np.maximum(bound[:, :Lout], 1e-300))))
            overshoot += int(np.sum(np.abs(planes) > 1.0))
    assert overshoot > 0
    record("pcm16_fused_decode_%d_%s" % (rate, direction), kind="pcm16", worst_error_over_bound=worst,
           overshoot=overshoot)


@pytest.mark.parametrize("rate,direction", list(_rate_cases()))
def test_fused_encode(ctx, resamplers, rate, direction):
    rate_in, rate_out = (ro.MODEL_RATE, rate) if direction == "back" else (rate, ro.MODEL_RATE)
    rs = resamplers(rate_in, rate_out)
    up, down, h = rs.up, rs.down, rs.taps
    rng = np.random.default_rng(2 * rate + (direction == "back"))
    worst, wrapped = 0.0, 0
    for nch in _channel_set(rate):
        for k, (Lin, Lout) in enumerate(po.fused_lengths(up, down, nch, True)):
            nsrc = 1 + (k + nch) % 4
            pcm = _random_pcm(rng, Lin, nsrc * nch) if k % 2 == 0 else _square(Lin, nsrc * nch, 4 + k)
            stems = np.ascontiguousarray(po.decode(pcm).T)
            shift = (k + nch) % 8
            got = _twice(lambda: encode(ctx, stems, nsrc, _lib().PCM16_CHANNELS, shift, rs, Lout))
            y32 = rs.resample(_cuda_planes(stems), num_out=Lout).cpu().numpy()
            want = po.interleave(y32, nsrc).reshape(nsrc, -1)
            assert got.tobytes() == want.tobytes(), (rate, direction, nch, nsrc, Lin, Lout,
                                                     np.argwhere(got != want)[:4].tolist())
            y, bound = _bound(stems.astype(np.float64), up, down, h)
            err = np.abs(y32.astype(np.float64) - y[:, :Lout])
            assert np.all(err <= bound[:, :Lout]), (rate, direction, nch, Lin)
            worst = max(worst, float(np.max(err / np.maximum(bound[:, :Lout], 1e-300))))
            wrapped += int(np.sum(np.abs(y32) * 32767 >= 32768))
    assert wrapped > 0
    record("pcm16_fused_encode_%d_%s" % (rate, direction), kind="pcm16", worst_error_over_bound=worst, wrapped=wrapped)


def test_refusals_queue_nothing(ctx, resamplers):
    lib, L = _lib(), 1000
    rs = resamplers(48000, 44100)
    from deepconvsep_b200.engine import Context, Resampler
    foreign = Resampler(Context(0), 48000, 44100)
    pcm = torch.zeros(L * 17, dtype=torch.int16, device="cuda")
    f = torch.zeros(17 * 4 * L + 64, dtype=torch.float32, device="cuda")
    o = torch.zeros(17 * 4 * L + 64, dtype=torch.int16, device="cuda")
    p, fp, op = pcm.data_ptr(), f.data_ptr(), o.data_ptr()
    n = rs.length(L)
    CH, MONO = lib.PCM16_CHANNELS, lib.PCM16_MONO
    bad_decode = [(None, 1, None, L, 2, fp, L), (None, 1, p, L, 2, None, L),
                  (None, 4, p, L, 2, fp, L), (None, -1, p, L, 2, fp, L), (None, 1, p, 0, 2, fp, 0),
                  (None, 1, p, L, 9, fp, L), (None, 1, p, L, 0, fp, L), (None, 1, p, L, 2, fp, L - 1),
                  (None, CH, p, L, 17, fp, L), (None, CH, p, L, 0, fp, L), (None, CH, p, L, 2, fp, L + 1),
                  (rs.handle, 1, p, L, 2, fp, n), (rs.handle, CH, p, L, 2, fp, n + 1), (rs.handle, CH, p, L, 2, fp, 0),
                  (foreign.handle, CH, p, L, 2, fp, n), (None, CH, p + 1, L, 2, fp, L), (None, CH, p, L, 2, fp + 2, L)]
    bad_encode = [(None, MONO, fp, L, 1, 2, L, op, L, L), (None, MONO, fp, L, 2, 1, L - 1, op, L, L),
                  (None, MONO, fp, L, 2, 1, L, op, L, L - 1), (None, MONO, fp, L, 1, 1, L, op, L - 1, L),
                  (None, 1, fp, L, 1, 1, L, op, L, L), (None, MONO, fp, 0, 1, 1, L, op, 0, L),
                  (None, MONO, fp, L, 0, 1, L, op, L, L), (None, CH, fp, L, 1, 17, L, op, L, 17 * L),
                  (None, CH, fp, L, 2, 3, L, op, L, 3 * L + 1), (None, CH, fp, L, 2, 3, L - 1, op, L, 3 * L),
                  (None, CH, fp, L, 2, 3, L, op, L + 1, 3 * L + 3), (None, CH, fp, L, 2, 3, L, op + 1, L, 3 * L),
                  (None, CH, fp + 2, L, 2, 3, L, op, L, 3 * L), (rs.handle, MONO, fp, L, 1, 1, L, op, n, n),
                  (rs.handle, CH, fp, L, 1, 2, L + 1, op, n, 2 * n), (rs.handle, CH, fp, L, 1, 2, L, op, n + 1, 2 * n + 2),
                  (foreign.handle, CH, fp, L, 1, 2, L, op, n, 2 * n), (None, CH, None, L, 1, 2, L, op, L, 2 * L),
                  (None, CH, fp, L, 1, 2, L, None, L, 2 * L)]
    torch.cuda.synchronize()
    n0 = ctx.launch_count()
    for args in bad_decode:
        assert ctx.lib.dcs_pcm16_decode(ctx.handle, *args, None) == -1, args
    for args in bad_encode:
        assert ctx.lib.dcs_pcm16_encode(ctx.handle, *args, None) == -1, args
    for args in [(fp, 0, L, L, fp), (fp, 17, L, L, fp), (fp, 2, L - 1, L, fp), (fp, 1, 0, 0, fp), (None, 1, L, L, fp),
                 (fp + 2, 1, L, L, fp)]:
        assert ctx.lib.dcs_downmix_f32(ctx.handle, *args, None) == -1, args
    assert ctx.lib.dcs_pcm16_decode(None, None, 1, p, L, 2, fp, L, None) == -1
    torch.cuda.synchronize()
    assert ctx.launch_count() == n0 and not f.any() and not o.any()
    # and the ctx still works
    lib.check(ctx.lib.dcs_pcm16_decode(ctx.handle, rs.handle, CH, p, L, 2, fp, n, None))
    assert ctx.launch_count() == n0 + 1


# ---------------------------------------------------------------------------------------------- 4. end to end at full scale
def _separator(arch, N=1024, overlap=25, seed=11):
    from deepconvsep_b200.engine import Separator
    from oracle import nets
    F = N // 2 + 1
    return Separator(nets.make_synthetic_params(arch, F, seed=seed), arch=arch, frame_size=N, hop=512, window="hanning",
                     overlap=overlap, feat_size=F)


def _channels_float_route(sep, pcm, **kw):
    x = torch.from_numpy(np.ascontiguousarray(po.decode(pcm).T)).cuda()
    stems = sep.separate_channels(x, **kw).cpu().numpy()
    return stems, po.interleave(stems, sep.nsrc)


def test_full_scale_clip_through_every_int16_entry_point():
    """The mono modes and the C-channel batches with the iKala net, whose synthetic stems overshoot a full-scale
    mixture (the decode does not depend on the net); the keep-channels batch with the DSD100 net, the one it serves."""
    pcm2 = po.full_scale_clip(2 * 44100 + 77, 2, 7)
    pcm6 = po.full_scale_clip(2 * 44100 + 91, 6, 8)
    pcm48 = po.full_scale_clip(2 * 48000 + 13, 6, 9)
    for p in (pcm2, pcm6, pcm48):
        assert p.min() == -32768 and p.max() == 32767
    dsd, ikala = _separator("dsd"), _separator("ikala", overlap=20)
    wrapped = {}
    for mode in (1, 2):
        got = ikala.separate_pcm16_batch([pcm2], downmix=mode)[0]
        stems = ikala.separate(po.decode_mono(pcm2, mode))
        assert got.tobytes() == po.encode(stems).tobytes(), (mode, int(np.sum(got != po.encode(stems))))
        wrapped["mono downmix %d" % mode] = int(np.sum(np.abs(stems) * 32767 >= 32768))
    got = ikala.separate_pcm16_channels_batch([pcm6])[0]
    stems, want = _channels_float_route(ikala, pcm6)
    assert got.tobytes() == want.tobytes(), int(np.sum(got != want))
    wrapped["C = 6"] = int(np.sum(np.abs(stems) * 32767 >= 32768))
    got = ikala.separate_pcm16_channels_batch([pcm48], sample_rate=48000)[0]
    stems, want = _channels_float_route(ikala, pcm48, sample_rate=48000)
    assert got.tobytes() == want.tobytes(), int(np.sum(got != want))
    wrapped["C = 6 at 48 kHz"] = int(np.sum(np.abs(stems) * 32767 >= 32768))
    got = dsd.separate_pcm16_batch([pcm2], keep_channels=True)[0]
    stems, want = _channels_float_route(dsd, pcm2)
    assert got.tobytes() == want.tobytes(), int(np.sum(got != want))
    wrapped["keep-channels"] = int(np.sum(np.abs(stems) * 32767 >= 32768))
    record("pcm16_full_scale", kind="pcm16", **{k.replace(" ", "_"): v for k, v in wrapped.items()})
    assert all(v > 0 for v in wrapped.values()), wrapped
