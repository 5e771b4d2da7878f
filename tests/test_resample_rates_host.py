"""The rate selection of tests/rate_classes.py against the whole rate policy, without a GPU:

- SELECTION is what derive_selection() computes over every accepted rate: it attains every extreme it claims of the
  plain and fused geometry, the first encode splits at C = 14, 15 and 16 and the first uneven splits, the ratio
  closest to 1, and the seeded sample is the seed's draw;
- the named rates have the edges they are named for;
- the gap the GPU file closes: no table rate splits the encode, the only direction it runs;
- the plain tile's closed form (dcs_resampler_create) is the search it abbreviates, and the fused plan's closed form
  (channels_formats_oracle.pcm_plan) is pcm16_oracle's loop at every accepted rate, not only the table's."""
import channels_formats_oracle as fo
import pcm16_oracle as po
import rate_classes as rc
import resample_oracle as ro
from deepconvsep_b200 import engine

RATES = rc.accepted_rates()
TABLE = {r: rc.measures(r) for r in RATES}


def test_the_policy_is_the_one_enumerated():
    assert tuple(engine.RESAMPLE_RATES) == rc.RATE_RANGE
    assert len(RATES) == 7379 and set(ro.TABLE_RATES) <= set(RATES)
    assert all(r in RATES for r in rc.SELECTION)


def test_selection_is_derived_from_every_accepted_rate():
    assert rc.SELECTION == rc.derive_selection(RATES)
    assert 45 <= len(rc.SELECTION) <= 55


def test_selection_attains_every_extreme():
    """each extreme over all 7 379 rates is attained inside the selection, whichever rate attains it first"""
    sel = {r: TABLE[r] for r in rc.SELECTION}
    for (name, e), (v, _) in rc.first_extremes(TABLE).items():
        assert v == (max if e == "max" else min)(m[name] for m in sel.values()), (name, e)
    ext = rc.first_extremes(TABLE)
    # the values the kernels' edges are made of
    assert ext["plain bank back", "max"][0] == 114576 and ext["plain bank back", "max"][0] <= ro.MAX_BANK_BYTES
    assert ext["up back", "max"][0] == 682 and ext["down in", "max"][0] == 682
    assert ext["fused smem decode i16", "max"][0] == ext["fused smem decode 4byte", "max"][0] == rc.RS_SMEM_MAX
    assert rc.RS_SMEM_MAX == 232448
    assert ext["fused smem encode 4byte", "max"][0] <= rc.RS_SMEM_MAX
    assert ext["plain span in", "max"][0] == ext["plain span back", "max"][0] == rc.RS_TILE_WORDS
    assert ext["distance from 1", "min"][1] == 44170                                  # 631/630


def test_selection_holds_every_split():
    for why, r in rc.first_splits(TABLE).items():
        assert why in rc.SELECTION[r], why
    splits = {C: [r for r in rc.SELECTION if TABLE[r]["groups encode 4byte"][C - 1] > 1] for C in (14, 15, 16)}
    assert all(splits[C] for C in splits), splits
    uneven = [(r, C) for r in rc.SELECTION for C in rc.CHANNELS
              if rc.fused_geometry(*rc.pair(r, "back"), C, "encode", "4byte")["groups"] > 1
              and rc.fused_geometry(*rc.pair(r, "back"), C, "encode", "4byte")["uneven"]]
    assert (8025, 15) in uneven                                                        # 8 + 7
    assert rc.fused_geometry(*rc.pair(8025, "back"), 15, "encode", "4byte")["cn"] == 8
    dec = [r for r in rc.SELECTION if TABLE[r]["uneven decode 4byte"]]
    assert dec and all(max(TABLE[r]["groups decode i16"]) == 1 for r in rc.SELECTION)   # the int16 decode never splits


def test_named_rates_have_their_edges():
    back = lambda r: rc.pair(r, "back")                                                 # noqa: E731
    assert back(8025) == (107, 588) and back(57288) == (682, 525) and back(68200) == (682, 441)
    assert rc.plain_geometry(*back(68200))["bank"] == rc.plain_geometry(*back(57288))["bank"] == 114576
    assert TABLE[8148]["groups encode 4byte"] == (1,) * 15 + (2,)
    assert back(46550) == (19, 18) and rc.pair(46550, "in") == (18, 19)
    for r in (46550, 86450, 96425):
        assert TABLE[r]["fused smem decode 4byte"] == rc.RS_SMEM_MAX, r
    assert TABLE[46550]["fused smem decode i16"] == rc.RS_SMEM_MAX
    for r, why in rc.EVERYDAY.items():
        assert why.startswith("%d/%d" % rc.pair(r, "in")), (r, why)                 # up / down into the model
    assert not set(rc.EVERYDAY) & set(ro.TABLE_RATES)


def test_no_table_rate_splits_the_encode():
    """the channel-group encode (groups > 1 in resample_encode_kernel) runs at no table rate: only the selection's
    rates exercise it"""
    for r in ro.TABLE_RATES:
        assert TABLE[r]["groups encode 4byte"] == (1,) * 16, r
    split = [(r, C) for r in RATES for C in rc.CHANNELS if TABLE[r]["groups encode 4byte"][C - 1] > 1]
    assert len(split) == 1357 and len({r for r, _ in split}) == 441


def test_plain_tile_is_the_search_it_abbreviates():
    for r in RATES:
        for d in ("in", "back"):
            up, down = rc.pair(r, d)
            g = rc.plain_geometry(up, down)
            assert g["tp"] == rc.plain_tile_loop(up, down), (r, d)
            assert g["tp"] % rc.RS_V == 0 and g["smem"] <= rc.RS_SMEM_MAX and 1 <= g["rounds"] <= 4
            assert g["span"] <= rc.RS_TILE_WORDS or g["tp"] == rc.RS_V
            # where both tiles are bound by the 4 rounds alone, the one-channel 4-byte decode's is the plain one
            f = rc.fused_geometry(up, down, 1, "decode", "4byte")
            cap = max(1, 4 * rc.RS_THREADS // up) * rc.RS_V
            assert f["tp"] >= g["tp"], (r, d)
            if g["tp"] == cap:
                assert f["tp"] == g["tp"], (r, d)


def test_closed_form_plan_is_the_loop_at_every_accepted_rate():
    """channels_formats_oracle's closed form against pcm16_oracle's loop where both apply (int16 decode, encode)"""
    for r in RATES:
        for d in ("in", "back"):
            up, down = rc.pair(r, d)
            for C in rc.CHANNELS:
                for enc in (False, True):
                    tp, cn, _ = fo.pcm_plan(up, down, C, enc, fo.I16)
                    assert (tp, cn) == po.pcm_plan(up, down, C, enc), (r, d, C, enc)
