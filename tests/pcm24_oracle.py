"""Exact host reference of DCS_SAMPLE_I24 (include/dcs.h): packed signed 24-bit little-endian PCM, 3 bytes per sample,
the samples of a WAV data chunk with a 3-byte container, as numpy arrays of dtype V3 (engine.PCM24).

- decode: v the sign-extended 24-bit value, the DCS_SAMPLE_I32 decode of v << 8 (channels_formats_oracle);
- encode: the DCS_SAMPLE_I32 encode shifted right by 8 bits (arithmetic), the low 3 bytes stored little-endian;
- the downmix and the interleave [nsrc][L][C] of the other formats with these rules;
- the case values: every byte pattern at random, both ends, and stem values on and around the 24-bit grid."""
import numpy as np

import channels_formats_oracle as fo

I24 = 4                                   # DCS_SAMPLE_I24; 3 is not a format
PCM24 = np.dtype("V3")


def unpack(a):
    """V3 [...] -> int32 [...], the sign-extended 24-bit values"""
    a = np.ascontiguousarray(a)
    assert a.dtype == PCM24
    b = a.view(np.uint8).reshape(a.shape + (3,)).astype(np.int32)
    v = b[..., 0] | (b[..., 1] << 8) | (b[..., 2] << 16)
    return np.where(v >= 1 << 23, v - (1 << 24), v).astype(np.int32)


def pack(v):
    """int [...] in [-2^23, 2^23) -> V3 [...]"""
    v = np.asarray(v, dtype=np.int64)
    assert v.size == 0 or (v.min() >= -2 ** 23 and v.max() < 2 ** 23)
    u = (v & 0xFFFFFF).astype(np.uint32)
    b = np.stack([u & 0xFF, (u >> 8) & 0xFF, u >> 16], axis=-1).astype(np.uint8)
    return np.ascontiguousarray(b).view(PCM24).reshape(v.shape)


def to_i32(a):
    """V3 -> the int32 samples carrying the same values in their top 24 bits (scipy.io.wavfile's read of the file)"""
    return (unpack(a).astype(np.int64) << 8).astype(np.int32)


def decode(a):
    return fo.decode(to_i32(a), fo.I32)


def encode(y):
    return pack(fo.encode(y, fo.I32) >> 8)


def decode_channels(pcm):
    """[L, C] V3 -> float32 [C + 1, L]: the downmix, then each channel"""
    return fo.decode_channels(to_i32(pcm), fo.I32)


def interleave(stems, nsrc):
    """stem planes float32 [nsrc * C, L] ordered (source, channel) -> [nsrc, L, C] V3"""
    return pack(fo.interleave(stems, nsrc, fo.I32) >> 8)


def random_clip(rng, L, C):
    """[L, C] V3 of random bytes (every 24-bit value equally likely), with rows at both ends"""
    a = rng.integers(-2 ** 23, 2 ** 23, (L, C))
    a[rng.integers(0, L, max(1, L // 64)), :] = -2 ** 23
    a[rng.integers(0, L, max(1, L // 64)), :] = 2 ** 23 - 1
    return pack(a)


def values24():
    """24-bit samples at and near both ends, a spread between, and small values"""
    return np.concatenate([np.arange(-2 ** 23, -2 ** 23 + 300), np.arange(2 ** 23 - 300, 2 ** 23),
                           np.arange(-2 ** 23, 2 ** 23, 4099), np.arange(-300, 301)])


def stem_values():
    """the int32 encode's cases plus multiples of 2^-23 near zero and both ends and their fp32 neighbours: the points
    where the shifted int32 value steps"""
    k = np.concatenate([np.arange(-40, 41), np.arange(2 ** 23 - 40, 2 ** 23 + 41), -np.arange(2 ** 23 - 40, 2 ** 23 + 41)])
    grid = (k.astype(np.float64) / 2 ** 23).astype(np.float32)
    near = np.concatenate([grid, np.nextafter(grid, np.float32(np.inf)), np.nextafter(grid, np.float32(-np.inf))])
    return np.concatenate([fo.i32_stem_values(), near]).astype(np.float32)
