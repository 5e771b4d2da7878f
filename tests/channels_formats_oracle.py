"""Exact host reference of the sample formats of dcs_separate_batch_channels_host (include/dcs.h):

- DCS_SAMPLE_I16: the int16 rules of tests/pcm16_oracle.py (pcm / 32767 in fp32; y * 32767 in fp32, truncated, wrapping);
- DCS_SAMPLE_I32: decode (float)((double)pcm / 2147483647.0), both steps rounded to nearest -- the bits of
  (a.astype(float) / iinfo(int32).max).astype(float32); encode (double)y * 2147483647.0 in fp64, truncated toward zero,
  saturated to [-2^31, 2^31 - 1], NaN -> 0;
- DCS_SAMPLE_F32: the sample itself and the stem itself, bit for bit;
- the downmix of the decoded planes and the interleave [nsrc][L][C] in any format;
- the tile plan of the fused resampling kernels per format (resample.cu pcm_plan), in closed form: the 4-byte decodes
  stage fp32 and take the fewest equal channel groups that fit, the int16 decode keeps all C channels in one tile, the
  encode stages fp32 stems in every format;
- the case values of the 4-byte formats: int32 at both ends and 24-bit values in the top bytes, float32 past +-1 with
  NaN payloads, and stem values at and past full scale of int32."""
import numpy as np

import pcm16_oracle as po

I16, I32, F32 = 0, 1, 2                       # DCS_SAMPLE_*
DTYPES = {I16: np.int16, I32: np.int32, F32: np.float32}
NAMES = {I16: "i16", I32: "i32", F32: "f32"}
I32_MAX = 2147483647.0


def decode(a, fmt):
    """samples [...] of fmt -> float32 [...]"""
    a = np.asarray(a)
    assert a.dtype == DTYPES[fmt]
    if fmt == I16:
        return po.decode(a)
    if fmt == I32:
        return (a.astype(np.float64) / I32_MAX).astype(np.float32)
    return a.copy()


def encode(y, fmt):
    """float32 [...] -> samples [...] of fmt"""
    y = np.asarray(y, dtype=np.float32)
    if fmt == I16:
        return po.encode(y)
    if fmt == I32:
        with np.errstate(invalid="ignore", over="ignore"):
            t = np.trunc(y.astype(np.float64) * I32_MAX)
        t = np.where(np.isnan(t), 0.0, np.clip(t, -2.0 ** 31, 2.0 ** 31 - 1))
        return t.astype(np.int64).astype(np.int32)
    return y.copy()


def decode_channels(pcm, fmt):
    """[L, C] of fmt -> float32 [C + 1, L]: the downmix, then each channel"""
    a = np.ascontiguousarray(decode(pcm, fmt).T)
    return np.concatenate([po.downmix(a)[None], a])


def interleave(stems, nsrc, fmt):
    """stem planes float32 [nsrc * C, L] ordered (source, channel) -> [nsrc, L, C] of fmt"""
    return po.interleave(stems, nsrc, enc=lambda y: encode(y, fmt))


def same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


# ---------------------------------------------------------------------------------------------- fused kernels' tiles
RS_THREADS, RS_V, RS_SMEM_MAX = po.RS_THREADS, po.RS_V, po.RS_SMEM_MAX


def resampler_geometry(up, down):
    """(Q, cspan, bank bytes) of the resampler of resample_taps(up, down)"""
    ntaps = 20 * max(up, down) + 1
    Q = -(-ntaps // up)
    half = (ntaps - 1) // 2
    return Q, ((up - 1) * down + half) // up - half // up, Q * up * 8


def pcm_plan(up, down, C, encode_side, fmt):
    """resample.cu pcm_plan -> (periods per tile, channels per tile, channel groups); None when nothing fits"""
    Q, cspan, bank = resampler_geometry(up, down)
    wide = encode_side or fmt != I16
    for groups in range(1, (C if wide else 1) + 1):
        cn = -(-C // groups)
        cs = (cn | 1) if encode_side else cn
        start = max(1, 4 * RS_THREADS // (up * (cn if encode_side else 1))) * RS_V
        room = (RS_SMEM_MAX - bank) // (cs * (4 if wide else 2))       # staged samples that fit
        tp = min(start, ((room - cspan - Q) // down + 1) // RS_V * RS_V) if room >= cspan + Q else 0
        if tp >= RS_V:
            return tp, cn, -(-C // cn)
    return None


def decode_groups(rate, C, fmt):
    """channel groups of the fused decode of a clip at `rate` with C channels (1: one launch, the downmix in it)"""
    from resample_oracle import ratio, MODEL_RATE
    up, down = ratio(rate, MODEL_RATE)
    return pcm_plan(up, down, C, False, fmt)[2]


def fused_lengths(up, down, C, encode_side, fmt):
    """(num_in, num_out) pairs: 1, 7 and ntaps // 2 input samples at full output length, and outputs of one tile
    +-1 of the plan for fmt"""
    ntaps = 20 * max(up, down) + 1
    tile = pcm_plan(up, down, C, encode_side, fmt)[0] * up
    pairs = {(n, -(-n * up // down)) for n in (1, 7, ntaps // 2)}
    for m in (tile - 1, tile, tile + 1):
        pairs.add((-(-m * down // up), m))
    return sorted(pairs)


# ---------------------------------------------------------------------------------------------- case values
NAN_PAYLOADS = np.frombuffer(np.array([0x7fc0beef, 0xffc00001, 0x7f800001, 0xff812345], dtype=np.uint32).tobytes(),
                             np.float32)


def int32_values():
    """int32 samples at and near both ends, 24-bit values in the top bytes (every multiple of 256 near the ends and a
    spread between), small values"""
    ends = np.array([-2 ** 31, -2 ** 31 + 1, -2 ** 31 + 255, -2 ** 31 + 256, 2 ** 31 - 1, 2 ** 31 - 2, 2 ** 31 - 256,
                     2 ** 31 - 257, 0, 1, -1, 255, -256, 0x7fffff00, -0x7fffff00], dtype=np.int64)
    top24 = np.concatenate([np.arange(-2 ** 23, -2 ** 23 + 300), np.arange(2 ** 23 - 300, 2 ** 23),
                            np.arange(-2 ** 23, 2 ** 23, 4099)]) * 256
    return np.concatenate([ends, top24]).astype(np.int32)


def random_clip(rng, L, C, fmt):
    """[L, C] of fmt over the whole range: int32 24-bit values in the top bytes with rows at both ends, float32 past
    +-1 with rows at +-3; int16 as tests/test_gpu_pcm16_kernels.py draws it"""
    if fmt == I16:
        a = rng.integers(-32768, 32768, (L, C)).astype(np.int16)
        a[rng.integers(0, L, max(1, L // 64)), :] = -32768
        a[rng.integers(0, L, max(1, L // 64)), :] = 32767
        return a
    if fmt == I32:
        a = (rng.integers(-2 ** 23, 2 ** 23, (L, C)) * 256).astype(np.int32)
        a[rng.integers(0, L, max(1, L // 64)), :] = -2 ** 31
        a[rng.integers(0, L, max(1, L // 64)), :] = 2 ** 31 - 1
        return a
    a = rng.uniform(-1.5, 1.5, (L, C)).astype(np.float32)
    a[rng.integers(0, L, max(1, L // 64)), :] = 3.0
    a[rng.integers(0, L, max(1, L // 64)), :] = -3.0
    return a


def i32_stem_values():
    """float32 stem values for the int32 encode: k / 2^23 over [-2, 2]; the fp32 neighbours (4 steps) of +-2^31 /
    (2^31 - 1) and of +-1; +-0, subnormals, NaN, +-inf, +-3e9"""
    out = [np.arange(-2 ** 24, 2 ** 24 + 1, 97, dtype=np.float64).astype(np.float32) / np.float32(2 ** 23)]
    for v in (2.0 ** 31 / I32_MAX, -2.0 ** 31 / I32_MAX, 1.0, -1.0, 0.5, -0.5):
        base = np.float32(v)
        up_, dn = base, base
        near = [base]
        for _ in range(4):
            up_ = np.nextafter(up_, np.float32(np.inf))
            dn = np.nextafter(dn, np.float32(-np.inf))
            near += [up_, dn]
        out.append(np.array(near, dtype=np.float32))
    out.append(np.array([0.0, -0.0, 1e-45, -1e-45, 1.2e-38, -1.2e-38, np.nan, np.inf, -np.inf, 3e9, -3e9, 1.5, -1.5,
                         1e-9, -1e-9], dtype=np.float32))
    out.append(NAN_PAYLOADS)
    return np.concatenate(out).astype(np.float32)


def stem_values(fmt):
    """the encode cases of fmt: pcm16_oracle.stem_values for int16, i32_stem_values for int32, and for float32 both
    with NaN payloads"""
    if fmt == I16:
        return po.stem_values()
    if fmt == I32:
        return i32_stem_values()
    return np.concatenate([po.stem_values(), i32_stem_values(), NAN_PAYLOADS])
