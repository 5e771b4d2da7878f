"""int16, int32 and float32 C-channel clips through the multi-clip scheduler (dcs_separate_batch_channels_host,
Separator.separate_channels_batch), and their conversion kernels element by element (dcs_channels_decode /
dcs_channels_encode), against the rules of include/dcs.h restated in tests/channels_formats_oracle.py.

- kernels, every format: the plain decode (pcm_decode_channels_kernel) and encode (pcm_encode_channels_kernel) against
  the numpy rules, the fused ones (resample_decode_kernel, resample_encode_kernel) against the rules applied to
  dcs_resample's fp32 output; C 1..16, lengths around the tiles, every destination offset modulo 16 bytes, NaN payloads
  between the stem planes, sentinels around every output, every case twice; the channel-group decode and its launch;
- pipeline, byte for byte against encode_out(separate_channels(decode_in(clip))): all 9 (in, out) pairs at 44.1 and
  48 kHz; each input format at C in {1, 2, 6, 16}, 44.1 kHz and every rate class, with clips of 1, 7, fewer than the
  filter's taps and tile-boundary +-1 samples; 192 kHz at C = 16, whose decode takes channel groups; I16 / I16 against
  separate_pcm16_channels_batch; the Wiener post-filter at C in {2, 6, 8}; batches against one-clip calls with pinned and
  pageable buffers; the workspace formula; refusals with nothing queued.
Inputs cover the full range: int32 at -2^31 and 2^31 - 1 and 24-bit values in the top bytes, float32 past +-1."""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import channels_formats_oracle as fo  # noqa: E402
import resample_oracle as ro  # noqa: E402
from oracle import nets, pipeline  # noqa: E402

FORMATS = (fo.I16, fo.I32, fo.F32)
NAN_IN = np.uint32(0x7fc0beef)      # fp32 the kernels must not read
NAN_OUT = np.uint32(0x7fc0dead)     # fp32 the kernels must not write
PAD = 64                            # fence bytes / 4 on either side of an output
# the bits around every input and output: int16 / int32 sentinels, and a NaN payload for float32
SENT = {fo.I16: (np.uint16, 0x5A5A), fo.I32: (np.uint32, 0x5A5A5A5A), fo.F32: (np.uint32, 0x7fc05a5a)}
MB = 1 << 20
RATES = [8000, 22050, 32000, 48000, 64000, 96000, 192000]


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


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _twice(fn):
    a, fa = fn()
    b, fb = fn()
    assert fa and fb, "a fence changed"
    assert a.tobytes() == b.tobytes(), "two runs differ"
    return a


def _cuda_planes(a):
    t = torch.empty(a.shape, dtype=torch.float32, device="cuda")
    t.copy_(torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)))
    return t


def _fenced(fmt, n):
    """device buffer of PAD * 4 bytes + n samples of fmt + PAD * 4 bytes, all sentinel; (tensor, pointer of sample 0)"""
    b = np.dtype(fo.DTYPES[fmt]).itemsize
    ut, bits = SENT[fmt]
    buf = np.full(2 * PAD * 4 // b + n + 16 // b, bits, dtype=ut)
    d = torch.from_numpy(buf.view(np.uint8).copy()).cuda()
    assert d.data_ptr() % 16 == 0
    return d, d.data_ptr() + 4 * PAD


def decode(ctx, pcm, fmt, rs=None, num_out=None):
    """[L, C] of fmt -> (uint32 bits [C + 1, num_out], fences intact); the input has sentinels before and after"""
    L, nch = pcm.shape
    n = L if num_out is None else num_out
    din, pin = _fenced(fmt, pcm.size)
    host = din.cpu().numpy()
    host[4 * PAD:4 * PAD + pcm.nbytes] = np.ascontiguousarray(pcm).view(np.uint8).ravel()
    din.copy_(torch.from_numpy(host))
    out = torch.from_numpy(np.full(2 * PAD + (nch + 1) * n, NAN_OUT, dtype=np.uint32).view(np.int32)).cuda()
    _lib().check(ctx.lib.dcs_channels_decode(ctx.handle, rs.handle if rs else None, fmt, pin, L, nch,
                                             out.data_ptr() + 4 * PAD, n, None))
    raw = out.cpu().numpy().view(np.uint32)
    fenced = bool(np.all(raw[:PAD] == NAN_OUT) and np.all(raw[PAD + (nch + 1) * n:] == NAN_OUT))
    return raw[PAD:PAD + (nch + 1) * n].reshape(nch + 1, n).copy(), fenced


def encode(ctx, stems, nsrc, fmt, shift, rs=None, num_out=None, gap=0):
    """stem planes float32 [nsrc * C, num_in], NaN payloads in the gaps -> ([nsrc, num_out * C] of fmt, fences intact);
    the output starts shift values past a 16-byte boundary"""
    P, Lin = stems.shape
    nch = P // nsrc
    n = Lin if num_out is None else num_out
    stride = Lin + gap
    sbuf = np.full(PAD + P * stride + PAD, NAN_IN, dtype=np.uint32)
    sbuf[PAD:PAD + P * stride].reshape(P, stride)[:, :Lin] = _bits(stems)
    ds = torch.from_numpy(sbuf.view(np.int32)).cuda()
    total = nsrc * nch * n
    b = np.dtype(fo.DTYPES[fmt]).itemsize
    dout, pout = _fenced(fmt, total + shift)
    _lib().check(ctx.lib.dcs_channels_encode(ctx.handle, rs.handle if rs else None, fmt, ds.data_ptr() + 4 * PAD, Lin, nsrc,
                                             nch, stride, pout + b * shift, n, nch * n, None))
    raw = dout.cpu().numpy().view(fo.DTYPES[fmt])
    k0 = 4 * PAD // b + shift
    ut, bits = SENT[fmt]
    fences = np.concatenate([raw.view(ut)[:k0], raw.view(ut)[k0 + total:]])
    return raw[k0:k0 + total].reshape(nsrc, nch * n).copy(), bool(np.all(fences == bits))


def _stems(rng, fmt, P, L):
    return rng.choice(fo.stem_values(fmt), (P, L)).astype(np.float32)


# ---------------------------------------------------------------------------------------------- 1. plain kernels
LENGTHS = (1, 255, 256, 257, 4099)


@pytest.mark.parametrize("fmt", FORMATS, ids=["i16", "i32", "f32"])
def test_plain_decode(ctx, fmt):
    rng = np.random.default_rng(10 + fmt)
    for nch in range(1, 17):
        clips = [fo.random_clip(rng, L, nch, fmt) for L in LENGTHS]
        if fmt == fo.I32:
            v = fo.int32_values()
            clips.append(np.resize(rng.permutation(v), (-(-v.size // nch), nch)).astype(np.int32))
        if fmt == fo.F32:
            clips[0] = np.resize(fo.stem_values(fo.F32)[np.isfinite(fo.stem_values(fo.F32))], (997, nch))
        for pcm in clips:
            got = _twice(lambda: decode(ctx, pcm, fmt))
            want = _bits(fo.decode_channels(pcm, fmt))
            assert got.tobytes() == want.tobytes(), (fmt, nch, pcm.shape, np.argwhere(got != want)[:4].tolist())


@pytest.mark.parametrize("fmt", FORMATS, ids=["i16", "i32", "f32"])
def test_plain_encode_every_shift(ctx, fmt):
    """every destination offset modulo 16 bytes at lengths around the 256-row tile, nsrc 1..4; then every stem value"""
    rng = np.random.default_rng(20 + fmt)
    shifts = range(16 // np.dtype(fo.DTYPES[fmt]).itemsize)
    k = 0
    for nch in range(1, 17):
        for shift in shifts:
            for L in (1, 7, 255, 256, 257, 513):
                nsrc = 1 + k % 4
                k += 1
                stems = _stems(rng, fmt, nsrc * nch, L)
                got = _twice(lambda: encode(ctx, stems, nsrc, fmt, shift, gap=1 + k % 9))
                want = fo.interleave(stems, nsrc, fmt).reshape(nsrc, -1)
                assert fo.same_bits(got, want), (fmt, nch, nsrc, L, shift, np.argwhere(got != want)[:4].tolist())
        vals = fo.stem_values(fmt)
        stems = np.resize(rng.permutation(vals), (2 * nch, -(-vals.size // (2 * nch)))).astype(np.float32)
        got = _twice(lambda: encode(ctx, stems, 2, fmt, nch % len(shifts), gap=5))
        assert fo.same_bits(got, fo.interleave(stems, 2, fmt).reshape(2, -1)), (fmt, nch)


# ---------------------------------------------------------------------------------------------- 2. fused kernels
def _channel_set(rate):
    return range(1, 17) if rate in (48000, 192000) else (1, 2, 5, 16)


@pytest.mark.parametrize("fmt", FORMATS, ids=["i16", "i32", "f32"])
@pytest.mark.parametrize("rate", ro.TABLE_RATES)
def test_fused_decode(ctx, resamplers, rate, fmt):
    rs = resamplers(rate, ro.MODEL_RATE)
    rng = np.random.default_rng(rate + fmt)
    for nch in _channel_set(rate):
        groups = fo.pcm_plan(rs.up, rs.down, nch, False, fmt)[2]
        for k, (Lin, Lout) in enumerate(fo.fused_lengths(rs.up, rs.down, nch, False, fmt)):
            pcm = fo.random_clip(rng, Lin, nch, fmt)
            n0 = ctx.launch_count()
            got = _twice(lambda: decode(ctx, pcm, fmt, rs, Lout))
            assert ctx.launch_count() - n0 == 2 * (1 + (groups > 1)), (rate, nch, groups)
            planes = rs.resample(_cuda_planes(fo.decode(pcm, fmt).T), num_out=Lout).cpu().numpy()
            want = _bits(np.concatenate([fo.po.downmix(planes)[None], planes]))
            assert got.tobytes() == want.tobytes(), (rate, fmt, nch, Lin, Lout, np.argwhere(got != want)[:4].tolist())


@pytest.mark.parametrize("fmt", FORMATS, ids=["i16", "i32", "f32"])
@pytest.mark.parametrize("rate", ro.TABLE_RATES)
def test_fused_encode(ctx, resamplers, rate, fmt):
    rs = resamplers(ro.MODEL_RATE, rate)
    rng = np.random.default_rng(3 * rate + fmt)
    nv = 16 // np.dtype(fo.DTYPES[fmt]).itemsize
    for nch in _channel_set(rate):
        for k, (Lin, Lout) in enumerate(fo.fused_lengths(rs.up, rs.down, nch, True, fmt)):
            nsrc = 1 + (k + nch) % 4
            stems = fo.decode(fo.random_clip(rng, Lin, nsrc * nch, fo.F32 if fmt == fo.F32 else fo.I32),
                              fo.F32 if fmt == fo.F32 else fo.I32).T.copy()
            stems *= np.float32(1.2)                                   # resampled values past full scale
            got = _twice(lambda: encode(ctx, stems, nsrc, fmt, (k + nch) % nv, rs, Lout))
            y32 = rs.resample(_cuda_planes(stems), num_out=Lout).cpu().numpy()
            want = fo.interleave(y32, nsrc, fmt).reshape(nsrc, -1)
            assert fo.same_bits(got, want), (rate, fmt, nch, nsrc, Lin, Lout, np.argwhere(got != want)[:4].tolist())


def test_group_decode_launches(ctx, resamplers):
    """the (rate, C) pairs whose 4-byte decode takes channel groups launch one downmix more, and no others"""
    for rate in RATES + [176400, 88200, 11025]:
        rs = resamplers(rate, ro.MODEL_RATE)
        pcm = np.zeros((rate // 50, 16), dtype=np.int32)
        for nch in range(1, 17):
            for fmt in FORMATS:
                g = fo.decode_groups(rate, nch, fmt)
                n0 = ctx.launch_count()
                decode(ctx, np.ascontiguousarray(pcm[:, :nch]).astype(fo.DTYPES[fmt]), fmt, rs, rs.length(pcm.shape[0]))
                assert ctx.launch_count() - n0 == 1 + (g > 1), (rate, nch, fmt, g)
    assert fo.decode_groups(192000, 16, fo.I32) > 1 and fo.decode_groups(192000, 16, fo.I16) == 1


# ---------------------------------------------------------------------------------------------- 3. pipeline
def separator(arch="dsd", N=1024, seed=5, overlap=25, patcher="standalone"):
    from deepconvsep_b200.engine import Separator
    F = N // 2 + 1
    return Separator(nets.make_synthetic_params(arch, F, seed=seed), arch=arch, frame_size=N, hop=512, window="hanning",
                     overlap=overlap, patcher=patcher, feat_size=F)


def audio_clip(L, nch, seed, fmt):
    """[L, nch] of fmt: two sources at different gains and delays per channel, at full scale: int16 and int32 (24-bit
    values in the top bytes) reach both ends, float32 peaks at 1.25"""
    n = max(L, 4410) + 64
    a, _ = pipeline.synth_mixture(n / 44100.0, seed)
    b, _ = pipeline.synth_mixture(n / 44100.0, seed + 1)
    rng = np.random.default_rng(seed)
    cols = []
    for c in range(nch):
        g, h = rng.uniform(-1.0, 1.0, 2)
        cols.append(g * np.roll(a, int(rng.integers(0, 60))) + h * np.roll(b, int(rng.integers(0, 60))))
    x = np.stack(cols, axis=1)[:L]
    x = 1.25 * x / max(np.abs(x).max(), 1e-9)
    if fmt == fo.F32:
        return x.astype(np.float32)
    if fmt == fo.I16:
        return np.clip(np.round(x * 32767), -32768, 32767).astype(np.int16)
    v = np.clip(np.round(x * 2 ** 23), -2 ** 23, 2 ** 23 - 1).astype(np.int64) * 256
    v[x >= 1.0] = 2 ** 31 - 1                     # a 32-bit file at both ends
    v[x <= -1.0] = -2 ** 31
    return v.astype(np.int32)


def float_route(sep, clip, fin, fout, rate=44100, wiener=0, wiener_radius=0):
    """encode_out(separate_channels(decode_in(clip), wiener, wiener_radius, rate)) -> [nsrc, L, C] of fout"""
    x = _cuda_planes(fo.decode(clip, fin).T)
    stems = sep.separate_channels(x, wiener=wiener, wiener_radius=wiener_radius, sample_rate=rate).cpu().numpy()
    L, nch = clip.shape
    return fo.interleave(stems.reshape(sep.nsrc * nch, L), sep.nsrc, fout)


def edge_lengths(rate, nch, fmt):
    """1, 7, fewer than the filter's taps, and +-1 around the first tile boundary of the decode (at 44.1 kHz) and of
    the encode (at the rate)"""
    Ls = {1, 7}
    if rate == 44100:
        return sorted(Ls | {255, 256, 257})
    up, down = ro.ratio(rate, 44100)
    ntaps = 20 * max(up, down) + 1
    out_tile = fo.pcm_plan(up, down, nch, False, fmt)[0] * up
    first = -(-out_tile * down // up)
    enc_tile = fo.pcm_plan(down, up, nch, True, fmt)[0] * down
    Ls |= {ntaps // 2, first - 1, first, first + 1, enc_tile - 1, enc_tile, enc_tile + 1}
    return sorted(L for L in Ls if L >= 1)


@pytest.mark.parametrize("rate", [44100, 48000])
def test_every_format_pair(rate):
    sep = separator("dsd", 1024, seed=40)
    nch = 6
    for fin in FORMATS:
        clips = [audio_clip(int(0.9 * rate) + 11 * fin, nch, 500 + fin, fin), audio_clip(3001, nch, 510 + fin, fin)]
        if fin == fo.I32:
            clips[0][:2] = [[-2 ** 31] * nch, [2 ** 31 - 1] * nch]
        for fout in FORMATS:
            got = sep.separate_channels_batch(clips, out_dtype=fo.DTYPES[fout], sample_rate=rate)
            for g, c in zip(got, clips):
                want = float_route(sep, c, fin, fout, rate)
                assert fo.same_bits(g, want), (rate, fin, fout, c.shape, int(np.sum(g != want)))
            assert np.abs(got[0].astype(np.float64)).sum() > 0


@pytest.mark.parametrize("fmt", FORMATS, ids=["i16", "i32", "f32"])
@pytest.mark.parametrize("rate", [44100] + RATES)
def test_each_format_at_every_rate(rate, fmt):
    sep = separator("dsd", 1024, seed=41 + rate % 13)
    for k, nch in enumerate((1, 2, 6, 16)):
        lengths = [int(0.6 * rate) + 13 * k] + edge_lengths(rate, nch, fmt)
        clips = [audio_clip(L, nch, 600 + 7 * k + i + rate % 1009, fmt) for i, L in enumerate(lengths)]
        got = sep.separate_channels_batch(clips, sample_rate=rate)
        for g, c in zip(got, clips):
            want = float_route(sep, c, fmt, fmt, rate)
            assert g.shape == (sep.nsrc, c.shape[0], nch) and g.dtype == fo.DTYPES[fmt]
            assert fo.same_bits(g, want), (rate, fmt, nch, c.shape[0], int(np.sum(g != want)))
        assert np.abs(got[0].astype(np.float64)).sum() > 0, nch


def test_channel_groups_at_192k():
    """192 kHz at C = 16: the 4-byte decode takes channel groups and one more launch per clip than int16"""
    sep = separator("dsd", 1024, seed=43)
    rate, nch = 192000, 16
    assert fo.decode_groups(rate, nch, fo.I32) > 1
    clips = {f: [audio_clip(int(0.5 * rate), nch, 700, f), audio_clip(int(0.3 * rate) + 5, nch, 701, f)] for f in FORMATS}
    sep.separate_channels_batch(clips[fo.I16], sample_rate=rate)                 # resamplers made
    counts = {}
    for f in FORMATS:
        n0 = sep.ctx.launch_count()
        got = sep.separate_channels_batch(clips[f], sample_rate=rate)
        counts[f] = sep.ctx.launch_count() - n0
        for g, c in zip(got, clips[f]):
            assert fo.same_bits(g, float_route(sep, c, f, f, rate)), f
    assert counts[fo.I32] == counts[fo.F32] == counts[fo.I16] + 2, counts


@pytest.mark.parametrize("rate", [44100, 96000])
def test_i16_is_the_pcm16_batch(rate):
    sep = separator("dsd", 2048, seed=44)
    clips = [audio_clip(int(s * rate), 6, 710 + k, fo.I16) for k, s in enumerate((1.3, 0.7))]
    a = sep.separate_pcm16_channels_batch(clips, wiener=1, sample_rate=rate)
    n0 = sep.ctx.launch_count()
    b = sep.separate_channels_batch(clips, wiener=1, sample_rate=rate)
    n1 = sep.ctx.launch_count()
    sep.separate_pcm16_channels_batch(clips, wiener=1, sample_rate=rate)
    assert sep.ctx.launch_count() - n1 == n1 - n0
    for x, y in zip(a, b):
        assert np.abs(x.astype(np.int64)).sum() > 0 and fo.same_bits(x, y)


@pytest.mark.parametrize("nch", [2, 6, 8])
def test_wiener(nch):
    sep = separator("dsd", 1024, seed=45)
    for fin, fout, rate in ((fo.I32, fo.I32, 44100), (fo.F32, fo.F32, 48000), (fo.I32, fo.F32, 48000)):
        pcm = audio_clip(3 * rate, nch, 720 + nch, fin)
        plain = sep.separate_channels_batch([pcm], out_dtype=fo.DTYPES[fout], sample_rate=rate)[0]
        for wiener, radius in ((1, 0), (2, 2)):
            got = sep.separate_channels_batch([pcm], out_dtype=fo.DTYPES[fout], wiener=wiener, wiener_radius=radius,
                                              sample_rate=rate)[0]
            want = float_route(sep, pcm, fin, fout, rate, wiener, radius)
            assert fo.same_bits(got, want), (nch, fin, fout, wiener, radius, int(np.sum(got != want)))
            assert not fo.same_bits(got, plain)


@pytest.mark.parametrize("pinned", [True, False])
def test_batch_is_one_clip_calls(pinned):
    sep = separator("dsd", 2048, seed=46)
    nch = 6
    for fin, fout, rate in ((fo.I32, fo.F32, 48000), (fo.F32, fo.I32, 44100)):
        clips = [audio_clip(int(s * rate), nch, 730 + k, fin) for k, s in enumerate((2.0, 3.5, 1.2, 2.7))]
        if pinned:
            pin = [torch.empty(c.shape, dtype=getattr(torch, str(c.dtype)), pin_memory=True).numpy() for c in clips]
            for p_, c in zip(pin, clips):
                p_[...] = c
            clips = pin
            outs = [torch.empty((sep.nsrc, c.shape[0], nch), dtype=getattr(torch, np.dtype(fo.DTYPES[fout]).name),
                                pin_memory=True).numpy() for c in clips]
        else:
            outs = None
        got = sep.separate_channels_batch(clips, outs=outs, out_dtype=fo.DTYPES[fout], sample_rate=rate)
        if outs is not None:
            assert all(g is o for g, o in zip(got, outs))
        for g, c in zip(got, clips):
            one = sep.separate_channels_batch([np.array(c)], out_dtype=fo.DTYPES[fout], sample_rate=rate)[0]
            assert np.abs(one.astype(np.float64)).sum() > 0 and fo.same_bits(g, one)
        assert fo.same_bits(got[1], float_route(sep, np.array(clips[1]), fin, fout, rate))


def rounded(nbytes):
    return (nbytes + MB - 1) // MB * MB


@pytest.mark.parametrize("rate,nch,wiener,fin,fout", [(44100, 6, 0, fo.I32, fo.I32), (48000, 8, 2, fo.F32, fo.I16),
                                                      (96000, 3, 0, fo.I16, fo.F32)])
def test_workspace_formula(rate, nch, wiener, fin, fout):
    clips = [audio_clip(int(s * rate), nch, 740 + k, fin) for k, s in enumerate((1.7, 3.3, 2.1))]
    Lmax = max(c.shape[0] for c in clips)
    batch = separator("dsd", 2048, seed=47)
    batch.separate_channels_batch(clips, out_dtype=fo.DTYPES[fout], wiener=wiener, wiener_radius=2 if wiener else 0,
                                  sample_rate=rate)
    Lm = batch.resampler(rate, 44100).length(Lmax) if rate != 44100 else Lmax
    single = separator("dsd", 2048, seed=47)
    single.separate_channels(torch.zeros((nch, Lm), dtype=torch.float32, device="cuda"), wiener=wiener,
                             wiener_radius=2 if wiener else 0)
    nsrc, n = batch.nsrc, 2
    bi, bo = (np.dtype(fo.DTYPES[f]).itemsize for f in (fin, fout))
    want = (single.ctx.workspace_bytes() - rounded(4 * Lm) + rounded(4 * (nch + 1) * Lm) + rounded(4 * nsrc * nch * Lm)
            + n * rounded(bi * nch * Lmax) + n * rounded(bo * nsrc * nch * Lmax))
    assert batch.ctx.workspace_bytes() == want, (batch.ctx.workspace_bytes(), want)


def test_refusals_queue_nothing():
    from deepconvsep_b200 import _lib
    sep = separator("dsd", 1024, seed=48)
    ctx, lib = sep.ctx, sep.lib
    rate, nch = 48000, 3
    clips = [audio_clip(48000, nch, 750, fo.I32), audio_clip(33600, nch, 751, fo.I32)]
    to, back = sep.resampler(rate, 44100), sep.resampler(44100, rate)
    to96 = sep.resampler(96000, 44100)
    Ls = np.array([c.shape[0] for c in clips], dtype=np.int64)
    outs = [np.empty((4, c.shape[0], 17), dtype=np.int32) for c in clips]
    sep.separate_channels_batch(clips, sample_rate=rate)
    ws = ctx.workspace_bytes()

    def call(pair=(to, back), fin=1, fout=1, channels=nch, iterations=0, lens=None):
        lens = Ls if lens is None else lens
        h = [None if r is None else r.handle for r in pair]
        return lib.dcs_separate_batch_channels_host(
            ctx.handle, sep.model.handle, sep.stft.handle, h[0], h[1], fin, fout, 2,
            (C.c_void_p * 2)(*[c.ctypes.data for c in clips]), lens.ctypes.data, channels, iterations, 0, C.c_float(0.3),
            25, 0, (C.c_void_p * 2)(*[o.ctypes.data for o in outs]), lens.ctypes.data, None)

    zero = Ls.copy()
    zero[1] = 0
    refused = {
        "in format 3": (lambda: call(fin=3), "unknown sample format"),
        "out format -1": (lambda: call(fout=-1), "unknown sample format"),
        "NULL to_model": (lambda: call(pair=(None, back)), "NULL resampler"),
        "NULL from_model": (lambda: call(pair=(to, None)), "NULL resampler"),
        "not inverse": (lambda: call(pair=(to96, back)), "not inverse"),
        "channels 17": (lambda: call(channels=17), "channels 17"),
        "filter on 9 channels": (lambda: call(channels=9, iterations=1), "Wiener"),
        "clip 1 length 0": (lambda: call(lens=zero), "clip 1"),
        "clip 1 length 0 at 44.1 kHz": (lambda: call(pair=(None, None), lens=zero), "clip 1"),
    }
    for name, (fn, msg) in refused.items():
        torch.cuda.synchronize()
        n0 = ctx.launch_count()
        with pytest.raises(_lib.DcsError) as e:
            _lib.check(fn())
        assert ctx.launch_count() == n0 and ctx.workspace_bytes() == ws, name
        assert msg in str(e.value), (name, str(e.value))
    # the conversion entries
    L = 1000
    d = torch.zeros(17 * 4 * L + 64, dtype=torch.float32, device="cuda")
    p = d.data_ptr()
    n = to.length(L)
    bad = [lambda: lib.dcs_channels_decode(ctx.handle, None, 3, p, L, 2, p, L, None),
           lambda: lib.dcs_channels_decode(ctx.handle, None, 1, p + 2, L, 2, p, L, None),
           lambda: lib.dcs_channels_decode(ctx.handle, None, 2, p, L, 17, p, L, None),
           lambda: lib.dcs_channels_decode(ctx.handle, to.handle, 1, p, L, 2, p, n + 1, None),
           lambda: lib.dcs_channels_encode(ctx.handle, None, 1, p, L, 1, 2, L, p + 2, L, 2 * L, None),
           lambda: lib.dcs_channels_encode(ctx.handle, None, 5, p, L, 1, 2, L, p, L, 2 * L, None),
           lambda: lib.dcs_channels_encode(ctx.handle, back.handle, 2, p, L, 1, 2, L, p, back.length(L) + 1, 0, None),
           lambda: lib.dcs_channels_encode(ctx.handle, None, 2, p, L, 1, 2, L, p, L, 2 * L + 1, None)]
    torch.cuda.synchronize()
    n0 = ctx.launch_count()
    for k, fn in enumerate(bad):
        assert fn() == -1, k
    assert ctx.launch_count() == n0 and not d.any()
    got = sep.separate_channels_batch(clips, sample_rate=rate)
    for g, c in zip(got, clips):
        assert fo.same_bits(g, float_route(sep, c, fo.I32, fo.I32, rate))
