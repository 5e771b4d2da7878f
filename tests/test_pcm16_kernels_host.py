"""The host reference of the int16 conversions (tests/pcm16_oracle.py), pinned without a device:

- its encode is numpy's (y * maxn).astype('int16') -- what the reference project writes -- wherever |y * 32767| < 2^31,
  and follows include/dcs.h's rule beyond (NaN 0, saturating to int32 first);
- its decode is scipy.io.wavfile's samples / 32767 in fp32, and the correctly rounded quotient, for every int16;
- the emulated index formulas of pcm_encode_channels_kernel write every value of the interleaved stems exactly once,
  with aligned 16-byte stores, for every destination shift 0..7, C 1..16 and tile edges;
- every mutant plan below differs from the reference on at least one case of the GPU suite's kinds; the table of
  which case rejects which mutant is printed."""
import io

import numpy as np
import pytest

import pcm16_oracle as po


def _rng(seed):
    return np.random.default_rng(seed)


def test_encode_is_numpy_astype_below_two_to_the_31():
    y = np.concatenate([po.stem_values(), _rng(1).uniform(-70000, 70000, 200000).astype(np.float32)])
    v = y * po.MAXV
    ok = np.abs(v.astype(np.float64)) < 2.0 ** 31
    assert ok.sum() > 200000 and (~ok).sum() >= 10
    with np.errstate(invalid="ignore"):
        want = v[ok].astype(np.int16)
    got = po.encode(y[ok])
    assert np.array_equal(got, want), int(np.sum(got != want))
    # some of them wrapped, and the wrap is modulo 2^16 of the truncated product
    assert np.sum(np.abs(y[ok]) > 1.0) > 1000
    assert po.encode(np.float32([1.5, -1.5, 2.0, 65537.0]))[:3].tolist() == [-16386, 16386, -2]


def test_encode_rule_beyond_two_to_the_31():
    big = np.float32(2.0 ** 31) / po.MAXV
    y = np.float32([np.nan, -np.nan, np.inf, -np.inf, 3e9, -3e9, 65538.0, -65538.0, big, -big])
    v = (y * po.MAXV).astype(np.float64)
    assert all(np.isnan(v[:2])) and all(np.abs(v[2:]) >= 2.0 ** 31)
    # NaN -> 0; the int32 saturation then the low 16 bits: 2^31 - 1 -> -1, -2^31 -> 0
    assert po.encode(y).tolist() == [0, 0, -1, 0, -1, 0, -1, 0, -1, 0]
    # the largest fp32 stem below the saturation still wraps: v = 2^31 - 256 -> -256
    below = np.nextafter(big, np.float32(0))
    assert float(below * po.MAXV) == 2.0 ** 31 - 256 and po.encode(np.float32([below, -below])).tolist() == [-256, 256]


def test_decode_is_wavfile_over_32767():
    from scipy.io import wavfile
    pcm = po.all_int16(2)
    buf = io.BytesIO()
    wavfile.write(buf, 44100, pcm)
    buf.seek(0)
    _, data = wavfile.read(buf)
    assert data.dtype == np.int16 and np.array_equal(data, pcm)
    want = data.astype(np.float32) / np.float32(32767)
    got = po.decode(pcm)
    assert got.tobytes() == want.tobytes()
    # IEEE division: the float64 quotient rounded once to fp32 (exact for fp32 operands)
    assert got.tobytes() == (pcm.astype(np.float64) / 32767.0).astype(np.float32).tobytes()
    assert po.decode(np.int16([-32768, 32767, 0]))[:2].tolist() == [np.float32(-32768) / np.float32(32767), 1.0]


@pytest.mark.parametrize("shift0", range(8))
def test_emulated_interleave_writes_each_value_once(shift0):
    rng = _rng(10 + shift0)
    vals = po.stem_values()
    for C in range(1, 17):
        for L in (1, 3, 255, 256, 257, 513):
            nsrc = 1 + (C + L + shift0) % 4
            stems = rng.choice(vals, (nsrc * C, L)).astype(np.float32)
            buf = po.emulate_encode_channels(stems, nsrc, shift0)
            n = nsrc * L * C
            assert buf[:n].tobytes() == po.interleave(stems, nsrc).tobytes(), (C, L, nsrc)
            assert np.all(buf[n:] == po.SENTINEL), (C, L, nsrc)


# ---------------------------------------------------------------------------------------------- mutants
def _enc_clip(y):
    v = (np.asarray(y, np.float32) * po.MAXV).astype(np.float64)
    return np.clip(np.trunc(np.where(np.isnan(v), 0.0, v)), -32768, 32767).astype(np.int16)


def _enc_rint(y):
    v = np.asarray(y, np.float32) * po.MAXV
    t = np.rint(np.where(np.isnan(v), 0.0, np.clip(v, -2.0 ** 31, 2.0 ** 31 - 1))).astype(np.int64)
    return ((t + 32768) % 65536 - 32768).astype(np.int16)


def _enc_f64(y):
    v = np.asarray(y, np.float32).astype(np.float64) * 32767.0
    t = np.trunc(np.where(np.isnan(v), 0.0, np.clip(v, -2.0 ** 31, 2.0 ** 31 - 1))).astype(np.int64)
    return ((t + 32768) % 65536 - 32768).astype(np.int16)


def _mix_reversed(planes):
    planes = np.asarray(planes, np.float32)
    return po.downmix(planes[::-1])


def _mix_scaled_terms(planes):
    planes = np.asarray(planes, np.float32)
    w = np.float32(1) / np.float32(planes.shape[0])
    a = planes[0] * w
    for p in planes[1:]:
        a = a + p * w
    return a


REFERENCE = dict(encode=po.encode, mix=po.downmix, plane_of=lambda s, c, nsrc, C: s * C + c,
                 head=po.kernel_head, tail_end=lambda n: n)
MUTANTS = {
    "saturating encode": dict(encode=_enc_clip),
    "round to nearest": dict(encode=_enc_rint),
    "fp64 multiply": dict(encode=_enc_f64),
    "downmix reversed": dict(mix=_mix_reversed),
    "downmix as sum of a_c / C": dict(mix=_mix_scaled_terms),
    "interleave (channel, source)": dict(plane_of=lambda s, c, nsrc, C: c * nsrc + s),
    "head = 8 - shift": dict(head=lambda n, shift: 8 - shift),
    "tail one short": dict(tail_end=lambda n: n - 1),
}


def _case_encode(plan):
    return plan["encode"](po.stem_values())


def _case_decode_channels(plan):
    rng = _rng(3)
    return np.concatenate([po.decode_channels(rng.integers(-32768, 32768, (4099, C)).astype(np.int16), plan["mix"])
                           for C in range(1, 17)], axis=None)


def _case_downmix_float(plan):
    """float planes at the fp32 edges: subnormals that halve to a tie, values whose sum overflows"""
    tiny, huge = np.float32(1e-45), np.float32(3e38)
    planes = np.array([[tiny, huge, 1.0, -tiny], [tiny, huge, 2.0 ** -24, tiny]], dtype=np.float32)
    return np.concatenate([plan["mix"](planes[:, :k]) for k in (1, 2, 4)] + [plan["mix"](np.tile(planes, (2, 1)))])


def _case_mono_decode(plan):
    pcm = po.all_int16(2)
    l, r = po.decode(pcm[:, 0]), po.decode(pcm[:, 1])
    return plan["mix"](np.stack([l, r]))


def _case_interleave(plan):
    rng = _rng(4)
    out = []
    for nsrc in (1, 2, 4):
        for C in (1, 2, 5, 16):
            stems = rng.choice(po.stem_values(), (nsrc * C, 257)).astype(np.float32)
            order = [plan["plane_of"](s, c, nsrc, C) for s in range(nsrc) for c in range(C)]
            out.append(po.interleave(stems[order], nsrc, plan["encode"]).reshape(-1))
    return np.concatenate(out)


def _case_kernel_indices(plan):
    rng = _rng(5)
    out = []
    for shift0 in range(8):
        for C in (1, 3, 7, 16):
            for L in (1, 2, 256, 257):
                nsrc = 1 + (shift0 + C) % 3
                stems = rng.choice(po.stem_values(), (nsrc * C, L)).astype(np.float32)
                out.append(po.emulate_encode_channels(stems, nsrc, shift0, plan["head"], plan["tail_end"],
                                                      plan["encode"]))
    return np.concatenate(out)


CASES = {"encode values": _case_encode, "C-channel decode": _case_decode_channels, "downmix fp32 edges": _case_downmix_float,
         "mono decode downmix 1": _case_mono_decode, "interleave": _case_interleave, "kernel indices": _case_kernel_indices}


def _same(a, b):
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def test_every_mutant_is_rejected(capsys):
    want = {name: case(REFERENCE) for name, case in CASES.items()}
    table = {}
    for mname, change in MUTANTS.items():
        plan = dict(REFERENCE, **change)
        table[mname] = [name for name, case in CASES.items() if not _same(case(plan), want[name])]
    with capsys.disabled():
        print("\nmutant -> cases that reject it")
        for mname, names in table.items():
            print("  %-30s %s" % (mname, ", ".join(names) or "NONE"))
    assert all(table.values()), {m: n for m, n in table.items() if not n}
