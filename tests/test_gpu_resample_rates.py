"""The resampler and its fused sample conversions at the rates of tests/rate_classes.py: every extreme of the plain and
fused geometry over the whole rate policy, the channel-group encode (C = 14, 15, 16, the uneven 8 + 7 split), the
banks of up = 682, the tiles at exactly 227 KB of shared memory, near-unity and everyday ratios, the table rates and a
seeded sample -- not only the 12 table rates the other GPU files run.

- plain dcs_resample against the float64 direct sum of tests/resample_oracle.py on the widened fp32 input, under
  |y_dev - y| <= 2^-24 |y| + 2 ceil(K/up) 2^-53 sum|h x|: 1 and 3 planes with gaps, lengths 1, 7, fewer than the taps,
  one plain tile of outputs +-1 and about 1 s, both directions; a shorter num_out is the head of the whole output;
- fused decode (resample_decode_kernel) in I16, I24, I32 and F32, C in {1, 2, 6, 16}, every C where the rate's plan
  changes its channel groups and every C whose tile takes all 227 KB, at fused_lengths: bit for bit the format's
  decode, dcs_resample's fp32 output per channel and downmix_kernel's expression for plane 0, with one more launch
  where the channels are grouped;
- fused encode (resample_encode_kernel) in the four formats, C in {1, 6, 14, 15, 16}, nsrc 2 and 4, every destination
  offset modulo 16 bytes: bit for bit the format's encode of dcs_resample's fp32 output of each stem plane;
- windowed entries (dcs_channels_decode_range / _encode_range): windows starting on a period boundary and one sample
  either side and one ending at the last output, at C = 6 and 16, equal to the slice of the whole-signal kernel;
- pipeline, byte for byte against encode_out(separate_channels(decode_in(clip))): 8025 Hz at C = 16 (the encode
  splits), 57288 Hz (the largest bank, with I24 in and out), 46550 Hz at C = 16 (the int16 decode tile at the
  limit), 44000 Hz (441/440); and the long path over two segments at 8025 Hz with C = 16.
Every kernel case runs twice for the same bits, with NaN or sentinel bytes wherever the kernel must not read or
write."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import channels_formats_oracle as fo  # noqa: E402
import pcm24_oracle as p24  # noqa: E402
import rate_classes as rc  # noqa: E402
import resample_oracle as ro  # noqa: E402
from parity import record  # noqa: E402
from test_gpu_channels_formats import _cuda_planes, audio_clip, float_route, separator  # noqa: E402
from test_gpu_long_channels import _same_values, _support, check  # noqa: E402
from test_gpu_long_channels import decode_range, decode_whole, encode_range, encode_whole  # noqa: E402
from test_gpu_pcm24 import _twice, _v3_bytes, audio24, decode, encode  # noqa: E402
from test_gpu_pcm24 import float_route as float_route24  # noqa: E402
from test_gpu_resample import _run  # noqa: E402

I24 = p24.I24
FORMATS = (fo.I16, I24, fo.I32, fo.F32)
NAMES = {fo.I16: "i16", I24: "i24", fo.I32: "i32", fo.F32: "f32"}
BYTES = {fo.I16: 2, I24: 3, fo.I32: 4, fo.F32: 4}
RATES = sorted(rc.SELECTION)


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


def _staging(fmt):
    return "i16" if fmt == fo.I16 else "4byte"


def _clip(rng, L, nch, fmt):
    return p24.random_clip(rng, L, nch) if fmt == I24 else fo.random_clip(rng, L, nch, fmt)


def _decoded(pcm, fmt):
    return p24.decode(pcm) if fmt == I24 else fo.decode(pcm, fmt)


def _encoded_bytes(y32, nsrc, fmt):
    """stem planes float32 [nsrc * C, L] -> the bytes of [nsrc, L, C] of fmt, one row per source"""
    if fmt == I24:
        return _v3_bytes(p24.interleave(y32, nsrc).reshape(nsrc, -1))
    return np.ascontiguousarray(fo.interleave(y32, nsrc, fmt)).view(np.uint8).reshape(nsrc, -1)


# ---------------------------------------------------------------------------------------------- a. plain kernel
@pytest.mark.parametrize("direction", ["in", "back"])
@pytest.mark.parametrize("rate", RATES)
def test_plain_against_float64(ctx, resamplers, rate, direction):
    rate_in, rate_out = (rate, ro.MODEL_RATE) if direction == "in" else (ro.MODEL_RATE, rate)
    rs = resamplers(rate_in, rate_out)
    up, down = rs.up, rs.down
    h = ro.taps(up, down)
    Q = -(-h.size // up)
    tile = rc.plain_geometry(up, down)["tp"] * up
    rng = np.random.default_rng(rate * 2 + (direction == "back"))
    cases = [(L, ro.length(L, up, down)) for L in (1, 7, h.size // 2, rate_in)]
    cases += [(-(-m * down // up), m) for m in (tile - 1, tile, tile + 1)]          # one plain tile of outputs +-1
    worst = 0.0
    for P in (1, 3):
        for L, n in cases:
            x = rng.uniform(-1.0, 1.0, (P, L)).astype(np.float32)
            got, fenced = _run(rs, x, n)
            assert fenced, (rate, direction, P, L, n)
            y = ro.direct(x.astype(np.float64), up, down, h, num_out=n)
            bound = 2.0 ** -24 * np.abs(y) + 2 * Q * 2.0 ** -53 * ro.direct(np.abs(x.astype(np.float64)), up, down,
                                                                             np.abs(h), num_out=n)
            err = np.abs(got.astype(np.float64) - y)
            assert np.all(np.isfinite(got)) and np.all(err <= bound), (rate, direction, P, L, n,
                                                                       float(np.max(err - bound)))
            worst = max(worst, float(np.max(err / np.maximum(bound, 1e-300))))
            again, fenced = _run(rs, x, n, gap_in=3, gap_out=5)
            assert fenced and again.tobytes() == got.tobytes(), (rate, direction, P, L, n)
            if n > 3:                                                     # a shorter num_out is the head
                head, fenced = _run(rs, x, n - 3, gap_in=1, gap_out=2)
                assert fenced and head.tobytes() == got[:, :n - 3].tobytes(), (rate, direction, P, L, n)
    record("resample_rates_%d_%s" % (rate, direction), kind="resample_rates", up=up, down=down, taps_per_phase=Q,
           worst_error_over_bound=worst)


# ---------------------------------------------------------------------------------------------- b. fused decode
@pytest.mark.parametrize("fmt", FORMATS, ids=[NAMES[f] for f in FORMATS])
@pytest.mark.parametrize("rate", RATES)
def test_fused_decode(ctx, resamplers, rate, fmt):
    rs = resamplers(rate, ro.MODEL_RATE)
    staging = _staging(fmt)
    rng = np.random.default_rng(5 * rate + fmt)
    k = 0
    at_limit = {C for C in rc.CHANNELS
                if rc.fused_geometry(rs.up, rs.down, C, "decode", staging)["smem"] == rc.RS_SMEM_MAX}
    for nch in sorted({1, 2, 6, 16} | set(rc.group_changes(rate, "decode", staging)) | at_limit):
        groups = rc.fused_geometry(rs.up, rs.down, nch, "decode", staging)["groups"]
        for Lin, Lout in fo.fused_lengths(rs.up, rs.down, nch, False, fo.I16 if fmt == fo.I16 else fo.I32):
            pcm = _clip(rng, Lin, nch, fmt)
            off = BYTES[fmt] * (k % (16 // BYTES[fmt])) if fmt != I24 else k % 16
            k += 1
            n0 = ctx.launch_count()
            got = _twice(lambda: decode(ctx, pcm, fmt, off, rs, Lout))
            assert ctx.launch_count() - n0 == 2 * (1 + (groups > 1)), (rate, fmt, nch, groups)
            planes = rs.resample(_cuda_planes(_decoded(pcm, fmt).T), num_out=Lout).cpu().numpy()
            want = np.ascontiguousarray(np.concatenate([fo.po.downmix(planes)[None], planes])).view(np.uint32)
            assert got.tobytes() == want.tobytes(), (rate, fmt, nch, Lin, Lout, np.argwhere(got != want)[:4].tolist())
    record("resample_rates_decode_%d_%s" % (rate, NAMES[fmt]), kind="resample_rates_fused", cases=k, mismatches=0)


# ---------------------------------------------------------------------------------------------- c. fused encode
ENCODE_CHANNELS = (1, 6, 14, 15, 16)


@pytest.mark.parametrize("fmt", FORMATS, ids=[NAMES[f] for f in FORMATS])
@pytest.mark.parametrize("rate", RATES)
def test_fused_encode(ctx, resamplers, rate, fmt):
    rs = resamplers(ro.MODEL_RATE, rate)
    rng = np.random.default_rng(7 * rate + fmt)
    offsets = range(0, 16, 1 if fmt == I24 else BYTES[fmt])
    seen = set()
    k = 0
    for nch in ENCODE_CHANNELS:
        for Lin, Lout in fo.fused_lengths(rs.up, rs.down, nch, True, fo.I32):
            for nsrc in (2, 4):
                off = offsets[k % len(offsets)]
                seen.add(off)
                k += 1
                src_fmt = fo.F32 if fmt == fo.F32 else fo.I32
                stems = fo.decode(fo.random_clip(rng, Lin, nsrc * nch, src_fmt), src_fmt).T.copy()
                stems *= np.float32(1.2)                                            # resampled values past full scale
                got = _twice(lambda: encode(ctx, stems, nsrc, fmt, off, rs, Lout))
                y32 = rs.resample(_cuda_planes(stems), num_out=Lout).cpu().numpy()
                want = _encoded_bytes(y32, nsrc, fmt)
                assert np.array_equal(got, want), (rate, fmt, nch, nsrc, Lin, Lout, off,
                                                   np.argwhere(got != want)[:4].tolist())
    assert seen == set(offsets), (rate, fmt)
    record("resample_rates_encode_%d_%s" % (rate, NAMES[fmt]), kind="resample_rates_fused", cases=k, mismatches=0,
           groups_at_16=rc.fused_geometry(rs.up, rs.down, 16, "encode", "4byte")["groups"])


# ---------------------------------------------------------------------------------------------- d. windowed entries
def _period_windows(n, up):
    """(first, count): starting on a period boundary and one sample either side, and one ending at the last output"""
    p = max(1, (n // 2) // up) * up
    w = {(p, min(n - p, 2 * up + 3)), (p - 1, min(n - p + 1, up + 2)), (p + 1, min(n - p - 1, 3)),
         (max(0, n - up - 5), n - max(0, n - up - 5))}
    return sorted((f, c) for f, c in w if 0 <= f < n and c >= 1)


@pytest.mark.parametrize("rate", RATES)
def test_windows_are_slices_of_the_whole(ctx, resamplers, rate):
    to, back = resamplers(rate, ro.MODEL_RATE), resamplers(ro.MODEL_RATE, rate)
    rng = np.random.default_rng(11 * rate)
    fmt = (fo.I16, fo.I32, fo.F32)[RATES.index(rate) % 3]
    for nch in (6, 16):
        pcm = fo.random_clip(rng, int(0.2 * rate) + 13, nch, fmt)
        L = pcm.shape[0]
        whole = decode_whole(ctx, to, pcm, fmt)
        n = whole.shape[1]
        for o0, cnt in _period_windows(n, to.up):
            i0, i1 = _support(to.up, to.down, o0, o0 + cnt - 1, L)
            got = decode_range(ctx, to, pcm, fmt, i0, i1 + 1, o0, cnt)
            assert _same_values(got, whole[:, o0:o0 + cnt]), (rate, fmt, nch, o0, cnt)
        nsrc = 2
        Lm = ro.length(L, back.down, back.up)
        stems = (rng.standard_normal((nsrc * nch, Lm)) * 0.6).astype(np.float32)
        ewhole = encode_whole(ctx, back, stems, nsrc, fmt, L)
        for o0, cnt in _period_windows(L, back.up):
            i0, i1 = _support(back.up, back.down, o0, o0 + cnt - 1, Lm)
            got = encode_range(ctx, back, np.ascontiguousarray(stems[:, i0:i1 + 1]), nsrc, fmt, Lm, i0, o0, cnt)
            assert _same_values(got, ewhole[:, o0:o0 + cnt]), (rate, fmt, nch, o0, cnt)


# ---------------------------------------------------------------------------------------------- e. pipeline
PIPELINE = [(8025, 16, fo.I32), (57288, 6, fo.F32), (46550, 16, fo.I16), (44000, 2, fo.I32)]


def test_pipeline_rates_cover_their_edges():
    assert rc.fused_geometry(*rc.pair(8025, "back"), 16, "encode", "4byte")["groups"] == 2
    assert rc.plain_geometry(*rc.pair(57288, "back"))["bank"] == 114576
    assert rc.fused_geometry(*rc.pair(46550, "in"), 16, "decode", "i16")["smem"] == rc.RS_SMEM_MAX
    assert rc.pair(44000, "in") == (441, 440)


@pytest.mark.parametrize("rate,nch,fmt", PIPELINE)
def test_pipeline(rate, nch, fmt):
    sep = separator("dsd", 1024, seed=90 + rate % 7)
    clips = [audio_clip(int(0.7 * rate) + 3, nch, 900 + rate % 101, fmt), audio_clip(4001, nch, 901 + rate % 101, fmt)]
    got = sep.separate_channels_batch(clips, sample_rate=rate)
    for g, c in zip(got, clips):
        want = float_route(sep, c, fmt, fmt, rate)
        assert g.shape == (sep.nsrc, c.shape[0], nch) and fo.same_bits(g, want), (rate, nch, fmt, c.shape)
    assert np.abs(got[0].astype(np.float64)).sum() > 0
    if rate == 57288:                                       # packed 24-bit in and out
        c24 = [audio24(int(0.6 * rate), nch, 910), audio24(3001, nch, 911)]
        g24 = sep.separate_channels_batch(c24, out_dtype=p24.PCM24, sample_rate=rate)
        for g, c in zip(g24, c24):
            assert g.dtype == p24.PCM24 and fo.same_bits(g, float_route24(sep, c, I24, I24, rate)), c.shape


def test_long_two_segments_at_8025_c16():
    sep = separator("dsd", 1024, seed=95)
    rate, nch = 8025, 16
    rec = audio_clip(int(3.1 * rate), nch, 920, fo.I16)
    _, segs = check(sep, rec, fo.I16, fo.I32, rate, int(1.6 * rate), min_segments=2)
    assert len(segs) == 2 and any(s.model_start > 0 for s in segs)
