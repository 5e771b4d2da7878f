"""The note-table path of the score-informed nets without a GPU: score.score_melody is the `melody` half of
score_filters (pinned to the reference's own functions by tests/golden/score_golden.npz), the Python layer refuses
malformed tables, and the long-clip helpers hand each segment the whole table with its first frame."""
import os
import numpy as np
import pytest

from deepconvsep_b200 import score, longclip
from deepconvsep_b200.engine import check_melody

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INSTS = ["bassoon_b", "clarinet_b", "saxophone_b", "violin_b"]


@pytest.fixture(scope="module")
def sg(tmp_path_factory):
    g = np.load(os.path.join(ROOT, "tests", "golden", "score_golden.npz"))
    d = tmp_path_factory.mktemp("scores")
    for k in INSTS:
        open(os.path.join(str(d), k + ".txt"), "wb").write(g["txt_" + k].tobytes())
    return g, str(d)


def test_score_melody_is_the_golden_table(sg):
    g, d = sg
    nframes = int(g["nframes"])
    melody = score.score_melody(d, INSTS, nframes)
    assert melody.dtype == np.float64 and melody.shape == g["melody"].shape
    np.testing.assert_array_equal(melody, g["melody"])


@pytest.mark.parametrize("nframes,F", [(None, 2049), (300, 2049), (None, 1025)])
def test_score_filters_is_filterSpec_of_score_melody(sg, nframes, F):
    g, d = sg
    T = int(g["nframes"]) if nframes is None else nframes
    N = 2 * (F - 1)
    melody = score.score_melody(d, INSTS, T, frameSize=N)
    mask = score.filterSpec(np.zeros((T, F), dtype=np.float32), melody, 0, T)
    planes = score.score_filters(d, INSTS, T, F, frameSize=N)
    np.testing.assert_array_equal(planes, mask.reshape(T, 4, F).transpose(1, 0, 2))
    if nframes is None and F == 2049:
        np.testing.assert_array_equal(planes, g["mask"].reshape(T, 4, F).transpose(1, 0, 2))


def test_filterSpec_window_is_rows_of_the_whole_clip(sg):
    """filterSpec(start, stop) = rows start..stop-1 of the whole-clip filters: what a long-clip segment rasterises"""
    g, _ = sg
    melody, T, F = g["melody"], int(g["nframes"]), 2049
    whole = score.filterSpec(np.zeros((T, F), dtype=np.float32), melody, 0, T)
    for start, n in ((0, 1), (35, 120), (T - 7, 7)):
        part = score.filterSpec(np.zeros((n, F), dtype=np.float32), melody, start, start + n)
        np.testing.assert_array_equal(part, whole[start:start + n])


def test_check_melody_refusals():
    ok = np.zeros((4, 3, 43))
    assert check_melody(ok, 4).flags.c_contiguous and check_melody(ok.astype(np.float32)).dtype == np.float64
    with pytest.raises(ValueError, match="ninst, nnotes, ncols"):
        check_melody(np.zeros((3, 43)))
    with pytest.raises(ValueError, match="instruments"):
        check_melody(np.zeros((5, 2, 43)))
    with pytest.raises(ValueError, match="instruments"):
        check_melody(np.zeros((0, 2, 43)))
    with pytest.raises(ValueError, match="the model takes 4"):
        check_melody(np.zeros((3, 2, 43)), 4)
    with pytest.raises(ValueError, match="columns"):
        check_melody(np.zeros((4, 2, 2)))


def test_long_clip_takes_filters_or_melody_not_both():
    N, H, tc, ov = 1024, 512, 30, 25
    with pytest.raises(ValueError, match="not both"):
        longclip.separate_long(lambda *a: None, np.zeros(1000), filters=np.zeros((4, 4, 513)), melody=np.zeros((4, 1, 43)),
                               geometry=(N, H, tc, ov))
    with pytest.raises(ValueError, match="columns"):
        longclip.separate_long(lambda *a: None, np.zeros(1000), melody=np.zeros((4, 1, 2)), geometry=(N, H, tc, ov))


def test_long_clip_segments_get_the_whole_table_and_their_first_frame():
    """melody= hands every segment the whole note table and its first whole-clip frame; with a stand-in that
    rasterises on the host, the stitched result is that of filters= sliced on the host"""
    N, H, tc, ov = 1024, 512, 30, 25
    F = N // 2 + 1
    L = 44100 * 6 + 5
    T = -(-L // H) + 2
    rng = np.random.default_rng(2)
    melody = np.zeros((4, 6, 43))
    for j in range(4):
        for p in range(5):
            n0 = rng.uniform(0, T - 20)
            melody[j, p, :3] = (n0, n0 + rng.uniform(1, 60), 60 + j)
            lo = rng.integers(1, F - 40, size=20)
            melody[j, p, 3::2], melody[j, p, 4::2] = lo, lo + rng.integers(0, 30, size=20)
    audio = rng.standard_normal(L).astype(np.float32)
    seen = []

    def per_sample(frames, sub):   # [4, Tsub] per-frame weights -> [4, len(sub)], a stand-in for a separation
        return frames[:, :, None].repeat(H, axis=2).reshape(4, -1)[:, :sub.size] * sub

    def notes(sub, mel, frame0):
        Tsub = -(-sub.size // H) + 2
        seen.append((frame0, np.array_equal(mel, melody)))
        f = score.filterSpec(np.zeros((Tsub, F), dtype=np.float32), mel, frame0, frame0 + Tsub)
        return per_sample(np.ascontiguousarray(f.reshape(Tsub, 4, F).transpose(1, 0, 2)).sum(axis=2), sub)

    whole = score.filterSpec(np.zeros((T, F), dtype=np.float32), melody, 0, T).reshape(T, 4, F).transpose(1, 0, 2)

    def filt(sub, f):
        assert f.shape == (4, -(-sub.size // H) + 2, F)
        return per_sample(np.ascontiguousarray(f).sum(axis=2), sub)

    got = longclip.separate_long([notes, notes], audio, parts=3, melody=melody, geometry=(N, H, tc, ov))
    want = longclip.separate_long([filt, filt], audio, parts=3, filters=whole, geometry=(N, H, tc, ov))
    segs = longclip.plan_segments(L, 3, N, H, tc, ov)
    assert len(segs) == 3 and sorted(s[0] for s in seen) == sorted(sg.frame0 for sg in segs) and all(s[1] for s in seen)
    assert max(sg.frame0 for sg in segs) > 0
    np.testing.assert_array_equal(got, want)
