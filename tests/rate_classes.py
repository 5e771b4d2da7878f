"""A selection of the resampler's accepted rates that stands in for the whole rate policy in the GPU tests
(tests/test_gpu_resample_rates.py), and the host arithmetic that justifies it.

The policy (resample_oracle.accepted, engine.RESAMPLE_RATES) takes 7 379 rates besides 44.1 kHz.  What the kernels do
with a rate depends only on its geometry, in either direction ("in": rate -> 44.1 kHz, the decode side; "back":
44.1 kHz -> rate, the encode side):

- the plain kernel (resample_kernel, dcs_resampler_create): up, down, taps per phase Q, the bank, cspan = c_{up-1} -
  c_0, the periods per tile tp, the staged span and the work-item rounds per CTA, up * tp / RS_V / RS_THREADS;
- the fused kernels (resample_decode_kernel, resample_encode_kernel, pcm_plan) per side, staging (int16 for the int16
  decode, fp32 for the 4-byte decodes and every encode) and C = 1..16: the tile, the channel groups, the shared memory
  and the rounds.

SELECTION holds every rate attaining an extreme of those over all accepted rates (the first in increasing rate where
several tie), the first rates whose encode splits its channels at C = 14, 15 and 16 and the first uneven splits of
either side, the ratio closest to 1, the everyday rates outside the policy's table, the table itself and a fixed-seed
sample of the rest; each with the reasons it is there.  tests/test_resample_rates_host.py recomputes all of it over
every accepted rate, so a change of the policy or the plan fails there instead of leaving the selection stale."""
import numpy as np

import channels_formats_oracle as fo
import resample_oracle as ro

MODEL_RATE = ro.MODEL_RATE
RATE_RANGE = (8000, 192000)                  # engine.RESAMPLE_RATES
RS_THREADS, RS_V, RS_SMEM_MAX = fo.RS_THREADS, fo.RS_V, fo.RS_SMEM_MAX
RS_TILE_WORDS = 8192                         # resample.cu: staged input per plain tile when the period allows
CHANNELS = range(1, 17)
# the fused plans: (side, staging); the I32, F32 and I24 decodes share the 4-byte plan, every encode format the fp32 one
PLANS = (("decode", "i16"), ("decode", "4byte"), ("encode", "4byte"))
SAMPLE_SEED, SAMPLE_SIZE = 2026, 12


def accepted_rates():
    """every rate the policy takes other than the networks' 44.1 kHz, increasing"""
    lo, hi = RATE_RANGE
    return [r for r in range(lo, hi + 1) if r != MODEL_RATE and ro.accepted(r)]


def pair(rate, direction):
    """(up, down) of the resampler the direction uses: "in" rate -> 44.1 kHz, "back" 44.1 kHz -> rate"""
    return ro.ratio(rate, MODEL_RATE) if direction == "in" else ro.ratio(MODEL_RATE, rate)


def plain_geometry(up, down):
    """dcs_resampler_create's constants: Q, cspan, bank bytes, periods per tile tp, staged span, shared memory, and
    the rounds of RS_THREADS the tile's work items take"""
    Q, cspan, bank = fo.resampler_geometry(up, down)
    tp = (RS_TILE_WORDS - cspan - Q) // down + 1
    tp = min(tp, max(1, 4 * RS_THREADS // up) * RS_V)
    tp = max(RS_V, tp // RS_V * RS_V)
    span = (tp - 1) * down + cspan + Q
    return dict(Q=Q, cspan=cspan, bank=bank, tp=tp, span=span, smem=bank + 4 * span,
                rounds=-(-up * (tp // RS_V) // RS_THREADS))


def plain_tile_loop(up, down):
    """the plain tile as a search: the most periods, a multiple of RS_V, within 4 rounds of the CTA, whose span fits
    RS_TILE_WORDS; RS_V when none does"""
    Q, cspan, _ = fo.resampler_geometry(up, down)
    tp = max(1, 4 * RS_THREADS // up) * RS_V
    while tp > RS_V and (tp - 1) * down + cspan + Q > RS_TILE_WORDS:
        tp -= RS_V
    return tp


def fused_geometry(up, down, C, side, staging):
    """pcm_plan's tile for C channels: periods tp, channels per tile cn, groups, staged span, shared memory and the
    rounds of RS_THREADS a tile's work items take (the encode's items count each channel)"""
    encode = side == "encode"
    fmt = fo.I16 if staging == "i16" else fo.F32
    tp, cn, groups = fo.pcm_plan(up, down, C, encode, fmt)
    Q, cspan, bank = fo.resampler_geometry(up, down)
    span = (tp - 1) * down + cspan + Q
    cs = (cn | 1) if encode else cn
    items = up * (tp // RS_V) * (cn if encode else 1)
    return dict(tp=tp, cn=cn, groups=groups, span=span, uneven=C % cn != 0,
                smem=bank + span * cs * (2 if staging == "i16" else 4), rounds=-(-items // RS_THREADS))


def side_direction(side):
    return "in" if side == "decode" else "back"


def group_changes(rate, side, staging):
    """the channel counts C > 1 at which the rate's plan takes another number of channel groups than at C - 1"""
    up, down = pair(rate, side_direction(side))
    g = [fused_geometry(up, down, C, side, staging)["groups"] for C in CHANNELS]
    return [C for C in CHANNELS if C > 1 and g[C - 1] != g[C - 2]]


def measures(rate):
    """{measure name: value} of one rate, the values a selection must attain the extremes of"""
    m = {}
    for d in ("in", "back"):
        up, down = pair(rate, d)
        g = plain_geometry(up, down)
        m["up " + d], m["down " + d] = up, down
        for k in ("Q", "bank", "cspan", "tp", "span", "rounds"):
            m["plain %s %s" % (k, d)] = g[k]
    for side, staging in PLANS:
        up, down = pair(rate, side_direction(side))
        geo = [fused_geometry(up, down, C, side, staging) for C in CHANNELS]
        m["fused smem %s %s" % (side, staging)] = max(g["smem"] for g in geo)
        m["fused rounds %s %s" % (side, staging)] = max(g["rounds"] for g in geo)
        m["groups %s %s" % (side, staging)] = tuple(g["groups"] for g in geo)
        m["uneven %s %s" % (side, staging)] = any(g["uneven"] and g["groups"] > 1 for g in geo)
    up, down = pair(rate, "in")
    m["distance from 1"] = abs(up - down) / max(up, down)
    return m


# (measure, "max" / "min"): the extremes the selection attains
EXTREMES = ([("up " + d, e) for d in ("in", "back") for e in ("max", "min")]
            + [("down " + d, e) for d in ("in", "back") for e in ("max", "min")]
            + [("plain %s %s" % (k, d), e) for k in ("Q", "bank", "cspan") for d in ("in", "back")
               for e in ("max", "min")]
            + [("plain tp " + d, "min") for d in ("in", "back")] + [("plain span " + d, "max") for d in ("in", "back")]
            + [("plain rounds " + d, "max") for d in ("in", "back")]
            + [("fused smem %s %s" % p, "max") for p in PLANS] + [("fused rounds %s %s" % p, "max") for p in PLANS]
            + [("distance from 1", "min")])


def first_extremes(table):
    """{(measure, "max" / "min"): (value, first rate attaining it)} over table = {rate: measures(rate)}"""
    out = {}
    for name, e in EXTREMES:
        sign = 1 if e == "max" else -1
        best = max(sign * table[r][name] for r in table)
        out[name, e] = (sign * best, min(r for r in table if sign * table[r][name] == best))
    return out


def first_splits(table):
    """the first rates whose encode splits at C = 14, 15, 16, and whose encode / 4-byte decode split unevenly"""
    out = {}
    for C in (14, 15, 16):
        out["encode splits at C = %d" % C] = min(r for r in table if table[r]["groups encode 4byte"][C - 1] > 1)
    out["encode splits unevenly"] = min(r for r in table if table[r]["uneven encode 4byte"])
    out["4-byte decode splits unevenly"] = min(r for r in table if table[r]["uneven decode 4byte"])
    return out


def seeded_sample(rates, exclude):
    """SAMPLE_SIZE further accepted rates drawn with SAMPLE_SEED, none of `exclude`"""
    pool = [r for r in rates if r not in exclude]
    rng = np.random.default_rng(SAMPLE_SEED)
    return sorted(int(r) for r in rng.choice(pool, SAMPLE_SIZE, replace=False))


# rates named for their ratio: everyday rates outside the policy's table
EVERYDAY = {44000: "441/440: near unity", 37800: "7/6: CD-ROM XA", 50000: "441/500", 47250: "14/15", 50400: "7/8"}
# rates named for a second instance of an edge the extremes reach first elsewhere (checked on the host)
NAMED = {8148: "encode splits at C = 16 only", 68200: "up 682 back, the largest bank, with down 441",
         46550: "int16 and 4-byte decode tiles at exactly RS_SMEM_MAX (18/19)",
         86450: "4-byte decode tile at exactly RS_SMEM_MAX", 96425: "4-byte decode tile at exactly RS_SMEM_MAX"}


def derive_selection(rates=None):
    """{rate: [reasons]}: SELECTION recomputed from the policy and the plan over every accepted rate"""
    rates = accepted_rates() if rates is None else rates
    table = {r: measures(r) for r in rates}
    reasons = {}

    def add(r, why):
        reasons.setdefault(r, []).append(why)
    for (name, e), (v, r) in first_extremes(table).items():
        add(r, "%s %s = %s" % (e, name, "%.6f" % v if isinstance(v, float) else v))
    for why, r in first_splits(table).items():
        add(r, why)
    for named in (EVERYDAY, NAMED):
        for r, why in named.items():
            add(r, why)
    for r in ro.TABLE_RATES:
        add(r, "table rate")
    for r in seeded_sample(rates, set(reasons)):
        add(r, "seeded sample")
    return {r: reasons[r] for r in sorted(reasons)}


# rate -> why it is selected, written out so that the GPU tests need no enumeration; derive_selection() recomputes it
SELECTION = {
    8000: ['min plain Q in = 21', 'max plain Q back = 111', 'max plain rounds in = 4',
           'max fused rounds decode i16 = 4', 'max fused rounds decode 4byte = 4', 'table rate'],
    8025: ['min plain tp back = 12', 'encode splits at C = 14', 'encode splits at C = 15', 'encode splits at C = 16',
           'encode splits unevenly'],
    8148: ['encode splits at C = 16 only'],
    8330: ['max fused smem encode 4byte = 232436'],
    8470: ['max up in = 630', 'max down back = 630'],
    8820: ['min up back = 1', 'min down in = 1', 'min plain cspan in = 0', 'min plain cspan back = 0'],
    9212: ['max plain span back = 8192'],
    10900: ['seeded sample'],
    11025: ['table rate'],
    16000: ['table rate'],
    16632: ['seeded sample'],
    22050: ['min plain bank back = 328', 'table rate'],
    24000: ['table rate'],
    24710: ['max plain cspan back = 629'],
    27270: ['seeded sample'],
    32000: ['table rate'],
    33390: ['max plain rounds back = 4'],
    36610: ['4-byte decode splits unevenly'],
    36750: ['max fused smem decode 4byte = 232448'],
    37800: ['7/6: CD-ROM XA'],
    42030: ['min plain Q back = 21'],
    44000: ['441/440: near unity'],
    44170: ['min distance from 1 = 0.001585'],
    44492: ['max plain span in = 8192'],
    45990: ['max fused smem decode i16 = 232448'],
    46305: ['seeded sample'],
    46550: ['int16 and 4-byte decode tiles at exactly RS_SMEM_MAX (18/19)'],
    47250: ['14/15'],
    47430: ['seeded sample'],
    48000: ['table rate'],
    48020: ['seeded sample'],
    50000: ['441/500'],
    50400: ['7/8'],
    50775: ['max plain bank in = 112896'],
    57288: ['max up back = 682', 'max down in = 682', 'max plain bank back = 114576', 'max plain cspan in = 681',
            'min plain tp in = 8'],
    59600: ['seeded sample'],
    64000: ['table rate'],
    68200: ['up 682 back, the largest bank, with down 441'],
    70665: ['max fused rounds encode 4byte = 22'],
    86450: ['4-byte decode tile at exactly RS_SMEM_MAX'],
    87808: ['seeded sample'],
    88200: ['min up in = 1', 'min down back = 1', 'min plain bank in = 328', 'table rate'],
    88515: ['seeded sample'],
    96000: ['table rate'],
    96425: ['4-byte decode tile at exactly RS_SMEM_MAX'],
    120330: ['seeded sample'],
    131355: ['seeded sample'],
    137088: ['seeded sample'],
    176400: ['table rate'],
    191835: ['max plain Q in = 88'],
    192000: ['table rate'],
}
