"""The score filters rasterised on the device from the note table (dcs_score_filters, dcs_separate_audio_notes,
csrc/score_notes.cu) against the host's filterSpec (dataset.py:839-862; deepconvsep_b200/score.py), byte for byte:
the reference's own mask of tests/golden/score_golden.npz, randomised tables with every corner of filterSpec's rules,
channels mode, the separation entry point on the three score nets, long clips, the example script, the dataset
runner, and refusals that queue nothing.  The filter path (dcs_separate_audio_score) is held to the float64 oracle
elsewhere; the note path is held to the filter path bit for bit, plus one direct strict-rule oracle check."""
import ctypes as C
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from oracle import dsp, nets, pipeline  # noqa: E402
import score1x1_oracle as s1  # noqa: E402
from parity import strict_check  # noqa: E402
from deepconvsep_b200 import score  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INSTS = ["bassoon_b", "clarinet_b", "saxophone_b", "violin_b"]
SOURCES = ["bassoon", "clarinet", "saxphone", "violin"]


def golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "score_golden.npz"))


def write_scores(d):
    g = golden()
    for k in INSTS:
        open(os.path.join(str(d), k + ".txt"), "wb").write(g["txt_" + k].tobytes())


def host_planes(melody, start, T, F):
    """filterSpec of the window [start, start + T) as planes [ninst, T, F]"""
    m = score.filterSpec(np.zeros((T, F), dtype=np.float32), melody, start, start + T)
    return np.ascontiguousarray(m.reshape(T, melody.shape[0], F).transpose(1, 0, 2))


def same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def random_table(rng, ninst, nnotes, ncols, Ttot, F, empty=None):
    """rows with filterSpec's corner cases: overlapping notes, notes outside the window, sub-frame notes, integral and
    fractional frames, '?' (NaN) and non-positive MIDI numbers with bins, zero padding rows, ranges with lo >= hi,
    ranges reaching F, negative lo in (-1, 0), pairs with hi <= 0 (skipped, lo may be negative), and with an even
    ncols an unpaired last column (ignored; NaN here)"""
    nh = (ncols - 3) // 2
    m = np.zeros((ninst, nnotes, ncols))
    for j in range(ninst):
        if j == empty:
            continue
        for p in range(nnotes - 2):                              # the last two rows stay zero padding
            n0 = rng.uniform(-6, Ttot + 6)
            if rng.random() < 0.5:
                n0 = float(np.floor(n0))
            ln = rng.uniform(0.05, 0.9) if rng.random() < 0.2 else rng.uniform(1, Ttot / 3 + 2)
            u = rng.random()
            midi = np.nan if u < 0.08 else (0.0 if u < 0.12 else (-5.0 if u < 0.15 else float(rng.integers(40, 90))))
            m[j, p, :3] = (n0, n0 + ln, midi)
            for k in range(nh):
                v = rng.random()
                lo = int(rng.integers(0, F))
                hi = min(F, lo + int(rng.integers(-4, 40)))
                if v < 0.1:
                    hi = F
                if v > 0.93:                                         # skipped pair
                    lo, hi = -int(rng.integers(0, 9)), 0
                elif v > 0.88:
                    lo = -rng.uniform(0, 0.99)                        # int() -> 0
                m[j, p, 3 + 2 * k] = lo + (rng.uniform(0, 0.99) if lo >= 0 and v <= 0.88 else 0)
                m[j, p, 4 + 2 * k] = hi + (rng.uniform(0, 0.99) if 0 < hi < F else 0)
        if ncols % 2 == 0:
            m[j, :, ncols - 1] = np.nan
    return m


@pytest.fixture(scope="module")
def ctx():
    from deepconvsep_b200.engine import Context
    return Context(0)


def test_golden_mask_of_the_reference(ctx):
    """dcs_score_filters on the reference's melody = the mask its own filterSpec produced"""
    from deepconvsep_b200.engine import score_filters
    g = golden()
    T, F = int(g["nframes"]), 2049
    out = score_filters(ctx, g["melody"], T, F).cpu().numpy()
    assert out.shape == (4, T, 2056)
    assert same_bits(out[:, :, :F], g["mask"].reshape(T, 4, F).transpose(1, 0, 2))
    assert not out[:, :, F:].any()


@pytest.mark.parametrize("ninst,nnotes,ncols,F,Ttot,start,T,empty,seed", [
    (4, 30, 43, 257, 300, 0, 300, None, 1),
    (4, 40, 44, 300, 500, 37, 200, 2, 2),
    (3, 25, 23, 129, 100, 5, 1, None, 3),
    (1, 20, 23, 513, 80, 0, 80, None, 4),
    (2, 30, 44, 2049, 200, 150, 1, 0, 5),
    (4, 60, 43, 2049, 400, 63, 250, 3, 6),
    (4, 1, 43, 257, 50, 0, 50, None, 7),
])
def test_random_tables_match_filterSpec(ctx, ninst, nnotes, ncols, F, Ttot, start, T, empty, seed):
    from deepconvsep_b200.engine import score_filters
    rng = np.random.default_rng(seed)
    m = random_table(rng, ninst, nnotes, ncols, Ttot, F, empty)
    want = host_planes(m, start, T, F)
    got = score_filters(ctx, m, T, F, start=start).cpu().numpy()
    assert same_bits(got[:, :, :F], want), np.argwhere(got[:, :, :F] != want)[:5]
    assert not got[:, :, F:].any()
    if empty is not None:
        assert (want[empty] < 1e-10).all()
    assert (want > 0.2).any()                           # some notes do sound in the window


@pytest.mark.parametrize("ldf_extra", [0, 13])
def test_channels_mode_is_filters_times_mag(ctx, ldf_extra):
    from deepconvsep_b200.engine import score_filters
    rng = np.random.default_rng(11)
    F, T, start = 513, 120, 9
    m = random_table(rng, 4, 30, 43, 200, F)
    ldf = (F + 7) // 8 * 8 + ldf_extra
    mag = (rng.random((T, ldf)) ** 3).astype(np.float32)      # pad columns non-zero: the output's are 0 anyway
    got = score_filters(ctx, m, T, F, start=start, mag=torch.as_tensor(mag, device="cuda:0")).cpu().numpy()
    want = host_planes(m, start, T, F) * mag[None, :, :F]
    assert got.shape == (4, T, ldf) and same_bits(got[:, :, :F], want.astype(np.float32))
    assert not got[:, :, F:].any()


def score_separators():
    from deepconvsep_b200.engine import Separator
    F = 2049
    p17 = nets.make_synthetic_params("bach10_score", F, seed=4)
    p11 = p17[:10] + [np.ascontiguousarray(p17[16][:4])]
    p22 = s1.make_synthetic_params_1x1(seed=5)
    seps = {}
    for name, p in (("11", p11), ("17", p17), ("22", p22)):
        seps[name] = Separator(p, frame_size=4096, hop=512, window="blackmanharris", overlap=25, patcher="util",
                               scale_factor=0.2, feat_size=F)
    assert [seps[k].model.arch for k in ("11", "17", "22")] == ["bach10_score", "bach10_score", "bach10_score_1x1"]
    return seps


@pytest.fixture(scope="module")
def seps():
    return score_separators()


@pytest.mark.parametrize("net", ["11", "17", "22"])
def test_separate_notes_equals_separate_score(seps, net):
    """stems, spectrum tap and launch count of the note path = those of the filter path, for both patchers at
    overlaps 25 and 28, N = 4096, and one clip whose first frame is table frame 40"""
    from deepconvsep_b200 import _lib
    sep = seps[net]
    melody = golden()["melody"]
    mix, _ = pipeline.synth_mixture(3.0, 500 + int(net))
    T = dsp.num_frames(mix.size, 512)
    cases = [(p, ov, 0) for p in ("util", "standalone") for ov in (25, 28)] + [("util", 25, 40)]
    for patcher, ov, frame0 in cases:
        sep.patcher, sep.overlap = _lib.PATCHER_IDS[patcher], ov
        c0 = sep.ctx.launch_count()
        a, Sa = sep.separate_tapped(mix, host_planes(melody, frame0, T, 2049))
        c1 = sep.ctx.launch_count()
        b, Sb = sep.separate_tapped(mix, melody=melody, frame0=frame0)
        c2 = sep.ctx.launch_count()
        assert np.abs(a).max() > 0
        assert same_bits(a, b) and same_bits(Sa, Sb), (net, patcher, ov, frame0)
        assert c2 - c1 == c1 - c0 > 0, (c0, c1, c2)
    sep.patcher, sep.overlap = _lib.PATCHER_IDS["util"], 25


def test_device_tensor_audio_and_profile_stage(seps):
    sep = seps["17"]
    melody = golden()["melody"]
    mix, _ = pipeline.synth_mixture(2.0, 77)
    x = torch.as_tensor(mix.astype(np.float32), device="cuda:0")
    sep.ctx.profile(True)
    y = sep.separate_notes(x, melody)
    torch.cuda.synchronize()
    names = [n for n, _ in sep.ctx.profile_read()]
    sep.ctx.profile(False)
    assert "score_channels" in names
    assert y.is_cuda and same_bits(y.cpu().numpy(), sep.separate_notes(mix, melody))


def test_strict_oracle_on_the_golden_scores(seps, tmp_path):
    """note path against the float64 oracle under the strict rule, on the 10 s golden-score clip"""
    write_scores(tmp_path)
    N, F = 4096, 2049
    mix, _ = pipeline.synth_mixture(10.0, 4000)
    T = dsp.num_frames(mix.size, 512)
    filters = score.score_filters(str(tmp_path), INSTS, T, F)
    melody = score.score_melody(str(tmp_path), INSTS, T)
    params = nets.make_synthetic_params("bach10_score", F, seed=4)
    want, mag, ph, mm = pipeline.separate_score(mix, filters, params, frameSize=N, hopSize=512, window=dsp.blackmanharris,
                                                scale_factor=0.2, overlap=25, count_kinks=True, return_spec=True)
    kmap = pipeline.separate_score.last_kink_map
    got, S = seps["17"].separate_tapped(mix, melody=melody)
    strict_check("notes_bach10_score_N4096_10s", got, S, want, mag, ph, mm, kmap, N, 512, dsp.blackmanharris, 0.2)


def test_long_clip_melody_equals_filters(seps):
    """3 segments on 2 contexts: melody= (each segment rasterises from its first frame) = filters= (sliced on the host)"""
    from deepconvsep_b200.engine import Separator
    from deepconvsep_b200 import longclip
    p17 = nets.make_synthetic_params("bach10_score", 2049, seed=4)
    two = [seps["17"], Separator(p17, frame_size=4096, hop=512, window="blackmanharris", overlap=25, patcher="util",
                                 scale_factor=0.2, feat_size=2049)]
    melody = golden()["melody"]
    mix, _ = pipeline.synth_mixture(8.0, 8)
    L, T = mix.size, dsp.num_frames(mix.size, 512)
    segs = longclip.plan_segments(L, 3, 4096, 512, 30, 25)
    assert len(segs) == 3 and segs[-1].frame0 > 0
    a = longclip.separate_long(two, mix, parts=3, filters=host_planes(melody, 0, T, 2049))
    b = longclip.separate_long(two, mix, parts=3, melody=melody)
    assert np.abs(a).max() > 0 and same_bits(a, b)


def test_example_script_wavs_equal_the_filter_path(tmp_path):
    import scipy.io.wavfile
    from deepconvsep_b200.examples.bach10_scoreinformed import separate_bach10 as ex
    from deepconvsep_b200.engine import Separator
    from deepconvsep_b200.models import save_model
    from deepconvsep_b200.examples import _common
    write_scores(tmp_path)
    p17 = nets.make_synthetic_params("bach10_score", 513, seed=6)
    p11 = p17[:10] + [np.ascontiguousarray(p17[16][:4])]
    save_model(str(tmp_path / "m.pkl"), p11)
    mix, _ = pipeline.synth_mixture(4.0, 31)
    wav = tmp_path / "01-piece.wav"
    scipy.io.wavfile.write(str(wav), 44100, (mix * 32767).astype(np.int16))
    out = tmp_path / "out"
    out.mkdir()
    paths = ex.train_auto(str(wav), str(out), str(tmp_path / "m.pkl"), 0.3, 30, 25, 32, 513, 1024, 512)
    audio = _common.decode(scipy.io.wavfile.read(str(wav))[1], "bach10")
    T = int(np.ceil(len(audio) / 512.0)) + 2
    filters = score.score_filters(str(tmp_path), ex.SOURCES_MIDI, T, 513, frameSize=1024, hopSize=512)
    sep = Separator(p11, frame_size=1024, hop=512, window="blackmanharris", scale_factor=0.3, time_context=30, overlap=25,
                    patcher="util", feat_size=513)
    stems = sep.separate_score(audio, filters)
    assert len(paths) == 4
    for i, path in enumerate(paths):
        ref = tmp_path / ("ref%d.wav" % i)
        scipy.io.wavfile.write(str(ref), 44100, (stems[i].astype(np.float64) * 32767).astype("int16"))
        assert open(path, "rb").read() == open(str(ref), "rb").read(), path
    assert np.abs(stems).max() > 0


def test_runner_equals_separate_score_on_summed_stems(tmp_path):
    import scipy.io.wavfile
    from deepconvsep_b200 import runner, util
    from deepconvsep_b200.engine import Separator
    p17 = nets.make_synthetic_params("bach10_score", 513, seed=9)
    db, out = tmp_path / "Bach10", tmp_path / "out"
    for k, secs in enumerate((3.0, 2.0)):
        d = db / ("0%d-piece" % (k + 1))
        d.mkdir(parents=True)
        write_scores(d)
        _, stems = pipeline.synth_mixture(secs, 60 + k)
        for s, name in enumerate(SOURCES):
            scipy.io.wavfile.write(str(d / ("0%d-piece-%s.wav" % (k + 1, name))), 44100, (stems[s] * 32767).astype(np.int16))
    secs, njobs = runner.separate_dataset("bach10_score", str(db), str(out), model=p17, frameSize=1024, hopSize=512)
    assert njobs == 2
    sep = Separator(p17, frame_size=1024, hop=512, window="blackmanharris", scale_factor=0.2, overlap=25, patcher="util",
                    feat_size=513)
    for k in (1, 2):
        piece = str(db / ("0%d-piece" % k))
        audio, sr, bitrate = runner.read_piece(piece)
        T = int(np.ceil(len(audio) / 512.0)) + 2
        stems = sep.separate_score(audio, score.score_filters(piece, INSTS, T, 513, frameSize=1024, hopSize=512))
        assert np.abs(stems).max() > 0
        for i, name in enumerate(SOURCES):
            ref = str(tmp_path / "ref.wav")
            util.writeAudioScipy(ref, stems[i].astype(np.float64), sr, bitrate)
            assert open(str(out / ("0%d-piece-%s.wav" % (k, name))), "rb").read() == open(ref, "rb").read()


def _p(t):
    return C.c_void_p(t.data_ptr())


def test_refusals_queue_nothing_and_leave_the_context_intact(seps):
    from deepconvsep_b200.engine import Model
    sep = seps["17"]
    ctx, lib = sep.ctx, sep.lib
    melody = np.ascontiguousarray(golden()["melody"])
    mix, _ = pipeline.synth_mixture(2.0, 12)
    before = sep.separate_notes(mix, melody)
    torch.cuda.synchronize()
    other = Model(ctx, nets.make_synthetic_params("bach10", 2049, seed=1), arch="bach10", feat_size=2049)
    L = mix.size
    a = torch.as_tensor(mix.astype(np.float32), device="cuda:0")
    out = torch.zeros((4, L), dtype=torch.float32, device="cuda:0")
    T, F, ldf = 40, 2049, 2056
    planes = torch.zeros((4, T, ldf), dtype=torch.float32, device="cuda:0")

    def bad(edit):
        m = melody.copy()
        edit(m)
        return m
    live = [int(np.nonzero(melody[j, :, 2] > 0)[0][0]) for j in range(4)]     # a row with a MIDI number > 0
    neg = bad(lambda m: m[0, live[0], 3:5].__setitem__(slice(None), (-3, 5)))
    above = bad(lambda m: m[1, live[1], 3:5].__setitem__(slice(None), (2000, F + 1)))
    nanf = bad(lambda m: m[2, live[2], 0:1].__setitem__(slice(None), np.nan))
    nanb = bad(lambda m: m[3, live[3], 4:5].__setitem__(slice(None), np.inf))

    def filt(m, ninst=4, ncols=None):
        return lib.dcs_score_filters(ctx.handle, m.ctypes.data, ninst, m.shape[1], ncols or m.shape[2], 0, T, F, None, ldf,
                                     _p(planes), T * ldf, None)

    def notes(model, m):
        return lib.dcs_separate_audio_notes(ctx.handle, model.handle, sep.stft.handle, _p(a), L, m.ctypes.data, m.shape[1],
                                            m.shape[2], 0, C.c_float(0.2), 25, 1, _p(out), L, None)
    n0 = ctx.launch_count()
    calls = [("non-score model", lambda: notes(other, melody)),
             ("ninst 0", lambda: filt(melody, ninst=0)), ("ninst 5", lambda: filt(np.concatenate([melody, melody[:1]]), ninst=5)),
             ("ncols 2", lambda: filt(melody, ncols=2)),
             ("negative bin", lambda: filt(neg)), ("bin above F", lambda: filt(above)), ("NaN frame", lambda: filt(nanf)),
             ("inf bin", lambda: filt(nanb)),
             ("negative bin, separation", lambda: notes(sep.model, neg)), ("NaN frame, separation", lambda: notes(sep.model, nanf))]
    for what, f in calls:
        assert f() == -1, what
        assert lib.dcs_launch_count(ctx.handle) == n0, what
    msg = lib.dcs_last_error().decode()
    assert "non-finite frame" in msg, msg
    torch.cuda.synchronize()
    assert same_bits(sep.separate_notes(mix, melody), before)
    # rows whose MIDI number is not > 0 are not checked (filterSpec never reads their bins)
    quiet = melody.copy()
    quiet[0, live[0], 2] = np.nan
    quiet[0, live[0], 3:5] = (-3, 5)
    assert filt(quiet) == 0
