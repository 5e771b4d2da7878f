"""Exact host reference of the int16 PCM conversions and the encode contract of include/dcs.h:

- decode: pcm / float32(32767), IEEE fp32 division (no fast-math in the build);
- downmix: (((a_0 + a_1) + a_2) + ...) * float32(1 / C) in fp32, left to right; the mono modes channel 0,
  (l + r) * 0.5f and l + r;
- encode: v = y * 32767.0f in fp32, truncated toward zero, saturated to int32 (NaN -> 0), then reduced modulo 2^16
  with integer arithmetic -- numpy's astype(int16) for |v| < 2^31, pinned where numpy is platform-dependent;
- the C-channel interleave [nsrc][L][C], and a host emulation of the index formulas of pcm_encode_channels_kernel
  (shift, head, 16-byte middle, tail) so that mutants of those formulas can be run without a device;
- the tile plan of the fused resampling kernels (resample.cu pcm_plan), for lengths at the tile boundaries;
- the case values: every int16, and stem values at and past full scale.
The fused kernels' references are built from these and dcs_resample's own fp32 output (the kernels promise its bits)."""
import numpy as np

MAXV = np.float32(32767)
SENTINEL = np.int16(0x5A5A)        # around every int16 output: must stay unchanged
POISON = np.int16(-0x2153)         # shared memory the emulated kernel never staged


def decode(pcm):
    """int16 [...] -> float32 pcm / 32767"""
    return np.asarray(pcm, dtype=np.int16).astype(np.float32) / MAXV


def downmix(planes):
    """float32 [C, L] -> (((a_0 + a_1) + a_2) + ...) * float32(1 / C)"""
    planes = np.asarray(planes, dtype=np.float32)
    a = planes[0].copy()
    with np.errstate(over="ignore", invalid="ignore"):
        for p in planes[1:]:
            a = a + p
        return a * (np.float32(1) / np.float32(planes.shape[0]))


def decode_mono(pcm, mode):
    """int16 [L, channels] -> float32 [L]: channel 0 (mode 0 or one channel), (l + r) * 0.5f (1), l + r (2)"""
    x = decode(np.asarray(pcm).reshape(len(pcm), -1))
    if x.shape[1] == 1 or mode == 0:
        return x[:, 0].copy()
    l, r = x[:, 0], x[:, 1]
    return (l + r) * np.float32(0.5) if mode == 1 else l + r


def decode_channels(pcm, mix=downmix):
    """int16 [L, C] -> float32 [C + 1, L]: the downmix, then each channel"""
    a = np.ascontiguousarray(decode(pcm).T)
    return np.concatenate([mix(a)[None], a])


def encode(y):
    """float32 [...] -> int16 [...]: the encode of include/dcs.h"""
    with np.errstate(invalid="ignore", over="ignore"):
        v = np.asarray(y, dtype=np.float32) * MAXV
    t = np.trunc(v.astype(np.float64))
    t = np.where(np.isnan(t), 0.0, np.clip(t, -2.0 ** 31, 2.0 ** 31 - 1))
    i = t.astype(np.int64)
    return ((i + 32768) % 65536 - 32768).astype(np.int16)


def interleave(stems, nsrc, enc=encode):
    """stem planes float32 [nsrc * C, L] ordered (source, channel) -> int16 [nsrc, L, C]"""
    P, L = stems.shape
    return np.ascontiguousarray(enc(stems).reshape(nsrc, P // nsrc, L).transpose(0, 2, 1))


# ---------------------------------------------------------------------------------------------- encode kernel indices
ROWS = 256       # kPcmEncodeRows: rows per CTA, one per thread


def kernel_head(n, shift):
    return min(n, (8 - shift) & 7)


def emulate_encode_channels(stems, nsrc, shift0, head=kernel_head, tail_end=lambda n: n, enc=encode):
    """The stores of pcm_encode_channels_kernel, tile by tile, into an int16 buffer whose first value lies shift0
    values past a 16-byte boundary: the tile staged at its destination's offset modulo 16 bytes, `head` values one at a
    time, 16-byte pieces, then the tail up to tail_end(n).  Returns the buffer [nsrc * L * C + 16] from SENTINEL; values
    read from tile slots nothing staged are POISON.  The 16-byte stores must be aligned."""
    P, L = stems.shape
    C = P // nsrc
    vals = interleave(stems, nsrc, enc).reshape(-1)
    buf = np.full(vals.size + 16, SENTINEL, dtype=np.int16)
    for s in range(nsrc):
        for i0 in range(0, L, ROWS):
            rows = min(L - i0, ROWS)
            dst = (s * L + i0) * C
            shift = (shift0 + dst) % 8
            n = rows * C
            tile = np.full(ROWS * 16 + 8 + 16, POISON, dtype=np.int16)
            tile[shift:shift + n] = vals[dst:dst + n]
            h = head(n, shift)
            nvec = (n - h) >> 3
            tail0 = h + nvec * 8
            for k in range(max(nvec, 0)):
                o = h + 8 * k
                assert (shift0 + dst + o) % 8 == 0 and (shift + o) % 8 == 0, "misaligned 16-byte store"
                buf[dst + o:dst + o + 8] = tile[shift + o:shift + o + 8]
            for t in range(h):
                buf[dst + t] = tile[shift + t]
            for th in range(ROWS):
                t = tail0 + th
                if t < tail_end(n):
                    buf[dst + t] = tile[shift + t]
    return buf


# ---------------------------------------------------------------------------------------------- fused kernels' tiles
RS_THREADS, RS_V, RS_SMEM_MAX = 512, 4, 227 * 1024


def pcm_plan(up, down, C, encode_side):
    """resample.cu pcm_plan: (periods per tile, channels per tile) of the fused kernel for C channels"""
    ntaps = 20 * max(up, down) + 1
    Q = -(-ntaps // up)
    half = (ntaps - 1) // 2
    cspan = ((up - 1) * down + half) // up - half // up
    bank = Q * up * 8
    for groups in range(1, (C if encode_side else 1) + 1):
        cn = -(-C // groups) if encode_side else C
        cs = (cn | 1) if encode_side else cn
        tp = max(1, 4 * RS_THREADS // (up * (cn if encode_side else 1))) * RS_V
        while tp >= RS_V:
            if bank + ((tp - 1) * down + cspan + Q) * cs * (4 if encode_side else 2) <= RS_SMEM_MAX:
                return tp, cn
            tp -= RS_V
    raise ValueError("no tile for %d/%d at C = %d" % (up, down, C))


def fused_lengths(up, down, C, encode_side):
    """(num_in, num_out) pairs: 1, 7 and ntaps // 2 input samples at full output length, and outputs of one tile
    +-1 (the shortest input that gives them, its output trimmed to them)"""
    ntaps = 20 * max(up, down) + 1
    tile = pcm_plan(up, down, C, encode_side)[0] * up
    pairs = {(n, -(-n * up // down)) for n in (1, 7, ntaps // 2)}
    for m in (tile - 1, tile, tile + 1):
        pairs.add((-(-m * down // up), m))
    return sorted(pairs)


# ---------------------------------------------------------------------------------------------- case values
def stem_values():
    """float32 stem values for the encode: every k / 32767 in fp32; the fp32 neighbours (4 steps) of each integer
    boundary m / 32767 for m in a spread of [-65537, 65537]; +-1, -32768/32767; past full scale up to +-65537; +-0,
    subnormals; the rule's extremes: NaN, +-inf, +-3e9, +-65538 and the neighbours of +-2^31 / 32767."""
    k = np.arange(-32768, 32768, dtype=np.float32)
    out = [k / MAXV]
    m = np.unique(np.concatenate([np.arange(-40, 41), np.arange(-32770, -32760), np.arange(32760, 32771),
                                  np.arange(-65537, 65538, 997), np.array([-65537, 65536, 65537])]))
    base = m.astype(np.float32) / MAXV
    for d in range(1, 5):
        up_, dn = base.copy(), base.copy()
        for _ in range(d):
            up_ = np.nextafter(up_, np.float32(np.inf))
            dn = np.nextafter(dn, np.float32(-np.inf))
        out += [up_, dn]
    big = np.float32(2.0 ** 31) / MAXV
    edge = [big, np.nextafter(big, np.float32(0)), np.nextafter(big, np.float32(np.inf))]
    special = [1.0, -1.0, np.float32(-32768) / MAXV, 0.0, -0.0, 1e-45, -1e-45, 1.2e-38, -1.2e-38, 1e-40, 3e-6,
               65537.0, -65537.0, 65536.5, -65536.5, 1.5, -1.5, 2.0, -2.0, 1000.25, -1000.25,
               np.nan, np.inf, -np.inf, 3e9, -3e9, 65538.0, -65538.0] + edge + [-e for e in edge]
    out.append(np.array(special, dtype=np.float32))
    out.append(np.frombuffer(np.array([0x7fc0beef, 0xffc00001, 0x7f800001], dtype=np.uint32).tobytes(), np.float32))
    return np.concatenate(out).astype(np.float32)


def full_scale_clip(L, nch, seed):
    """int16 [L, nch] mastered to 0 dBFS: two synthetic sources at different gains per channel plus a square wave,
    clipped to [-32768, 32767], reaching both ends on every channel"""
    from oracle import pipeline
    a, _ = pipeline.synth_mixture(L / 44100.0 + 0.01, seed)
    b, _ = pipeline.synth_mixture(L / 44100.0 + 0.01, seed + 1)
    rng = np.random.default_rng(seed)
    t = np.arange(L)
    cols = []
    for c in range(nch):
        g, h = rng.uniform(0.5, 1.0, 2)
        sq = np.sign(np.sin(2 * np.pi * (110 + 37 * c) * t / 44100.0))
        x = g * a[:L] + h * b[:L] + 0.6 * sq
        cols.append(1.3 * x / np.abs(x).max())
    x = np.round(np.stack(cols, axis=1) * 32768)
    x[rng.integers(0, L, 4), :] = 40000
    x[rng.integers(0, L, 4), :] = -40000
    return np.clip(x, -32768, 32767).astype(np.int16)


def all_int16(C, shift=7919):
    """int16 [65536, C]: channel c holds every int16 value, rotated by c * shift so that rows mix them"""
    v = np.arange(-32768, 32768, dtype=np.int64)
    return np.stack([np.roll(v, c * shift) for c in range(C)], axis=1).astype(np.int16)
