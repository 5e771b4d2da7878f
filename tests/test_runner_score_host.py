"""The dataset runner's score-informed family without a GPU (deepconvsep_b200/runner.py --family bach10_score; the
separation branch of examples/bach10_scoreinformed/trainCNNrwc.py:357-416,646-647): piece directories, the mixture as
the float sum of the four source wavs, the note table from the pieces' scores, the trainer's transform and
scale_factor_test, the reference's output names and the input's bit depth, two ranks covering the dataset once."""
import os
import numpy as np
import pytest
import scipy.io.wavfile
from types import SimpleNamespace

from deepconvsep_b200 import runner, score

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SOURCES = ["bassoon", "clarinet", "saxphone", "violin"]
MIDI = ["bassoon_b", "clarinet_b", "saxophone_b", "violin_b"]


def _piece(db, name, seconds, dtype=np.int16, seed=0):
    g = np.load(os.path.join(ROOT, "tests", "golden", "score_golden.npz"))
    d = db / name
    d.mkdir(parents=True)
    rng = np.random.default_rng(seed)
    n = int(44100 * seconds)
    for s in SOURCES:
        scipy.io.wavfile.write(str(d / (name + "-" + s + ".wav")), 44100,
                               (rng.uniform(-0.2, 0.2, size=n) * np.iinfo(dtype).max).astype(dtype))
    for k in MIDI:
        open(str(d / (k + ".txt")), "wb").write(g["txt_" + k].tobytes())
    return d


def _fake_separator(log, arch="bach10_score"):
    class Fake(object):
        def __init__(self, params, arch=None, frame_size=None, hop=None, window=None, scale_factor=0.3, time_context=None,
                     overlap=None, patcher="standalone", device=0, feat_size=None):
            log.append(("init", dict(arch=arch, frame_size=frame_size, hop=hop, window=window, overlap=overlap, patcher=patcher,
                                     device=device, feat_size=feat_size, scale_factor=scale_factor)))
            self.nsrc = 4
            self.model = SimpleNamespace(arch=fam, tc=30)

        def separate_notes(self, audio, melody, frame0=0):
            log.append(("notes", np.array(audio), np.array(melody), frame0))
            return np.stack([np.asarray(audio, dtype=np.float32) / (s + 2) for s in range(4)])
    fam = arch
    return Fake


def test_jobs_are_the_digit_piece_directories(tmp_path):
    db = tmp_path / "Bach10"
    for name in ("02-AchLiebenChristen", "01-AchGottundHerr", "README", ".hidden"):
        (db / name).mkdir(parents=True)
    (db / "03-notadir.wav").write_bytes(b"")
    jobs = runner.list_jobs("bach10_score", str(db), "/o")
    assert [j[0] for j in jobs] == [str(db / "01-AchGottundHerr"), str(db / "02-AchLiebenChristen")]
    assert jobs[0][1] == ["/o/01-AchGottundHerr-%s.wav" % s for s in SOURCES]     # trainCNNrwc.py:414


def test_mixture_scores_defaults_names_and_bit_depth(tmp_path, monkeypatch):
    log = []
    monkeypatch.setattr(runner, "Separator", _fake_separator(log))
    db, out = tmp_path / "Bach10", tmp_path / "out"
    _piece(db, "01-AchGottundHerr", 0.5, seed=1)
    _piece(db, "05-DieNacht", 0.8, dtype=np.int32, seed=2)
    secs, njobs = runner.separate_dataset("bach10_score", str(db), str(out), model=[np.zeros(1)])
    assert njobs == 2 and abs(secs - 1.3) < 1e-3
    init = log[0][1]
    assert (init["arch"], init["frame_size"], init["hop"], init["window"], init["overlap"], init["patcher"],
            init["feat_size"], init["scale_factor"]) == (None, 4096, 512, "blackmanharris", 25, "util", 2049, 0.2)
    calls = [e for e in log if e[0] == "notes"]
    assert [len(c[1]) for c in calls] == [35280, 22050]                               # longest first
    piece = str(db / "05-DieNacht")
    mix = sum(scipy.io.wavfile.read(os.path.join(piece, "05-DieNacht-%s.wav" % s))[1] / float(np.iinfo(np.int32).max)
              for s in SOURCES)
    assert np.array_equal(calls[0][1], mix) and calls[0][3] == 0                      # float sum of the stems (:367-378)
    T = int(np.ceil(len(mix) / 512.0)) + 2
    np.testing.assert_array_equal(calls[0][2], score.score_melody(piece, MIDI, T))    # 40 s, 20 harmonics, 50 cents, 440 Hz
    for name, dt in (("01-AchGottundHerr", np.int16), ("05-DieNacht", np.int32)):
        for i, s in enumerate(SOURCES):
            sr, y = scipy.io.wavfile.read(str(out / (name + "-" + s + ".wav")))
            assert sr == 44100 and y.dtype == dt and y.ndim == 1                    # the input's bit depth (util.py:56-58)
    sr, y = scipy.io.wavfile.read(str(out / "05-DieNacht-bassoon.wav"))
    assert np.array_equal(y, ((mix.astype(np.float32) / 2).astype(np.float64) * np.iinfo(np.int32).max).astype(np.int32))


def test_two_ranks_cover_the_pieces_once(tmp_path, monkeypatch):
    log = []
    monkeypatch.setattr(runner, "Separator", _fake_separator(log))
    db, out = tmp_path / "Bach10", tmp_path / "out"
    for k, secs in enumerate((0.3, 0.6, 0.4)):
        _piece(db, "0%d-piece" % k, secs, seed=k)
    done = [runner.separate_dataset("bach10_score", str(db), str(out), model=[np.zeros(1)], rank=r, world_size=2, device=r)[0]
            for r in range(2)]
    assert abs(sum(done) - 1.3) < 1e-3 and min(done) > 0.5
    assert [e[1]["device"] for e in log if e[0] == "init"] == [0, 1]
    assert sorted(os.listdir(str(out))) == sorted("0%d-piece-%s.wav" % (k, s) for k in range(3) for s in SOURCES)


def test_refusals_and_cli_default_scale(tmp_path, monkeypatch):
    log = []
    monkeypatch.setattr(runner, "Separator", _fake_separator(log, arch="bach10"))
    db = tmp_path / "Bach10"
    _piece(db, "01-x", 0.1)
    with pytest.raises(ValueError, match="score-informed network"):
        runner.separate_dataset("bach10_score", str(db), str(tmp_path / "o"), model=[np.zeros(1)])
    with pytest.raises(ValueError, match="keep-channels"):
        runner.separate_dataset("bach10_score", str(db), str(tmp_path / "o"), model=[np.zeros(1)], keep_channels=True)
    seen = []
    monkeypatch.setattr(runner, "separate_dataset", lambda *a, **k: (seen.append(a), (0.0, 0))[1])
    monkeypatch.setattr(runner, "reduce_stats", lambda s, ms: (s, max(ms, 1.0), 1))
    runner.main(["--family", "bach10_score", "--db", str(db), "--out", str(tmp_path / "o"), "--model", "m.pkl"])
    assert seen[-1][4] is None                       # separate_dataset picks the family's 0.2
    runner.main(["--family", "dsd", "--db", str(db), "--out", str(tmp_path / "o"), "--model", "m.pkl", "--scale-factor", "0.5"])
    assert seen[-1][4] == 0.5
    log.clear()
    monkeypatch.undo()
    monkeypatch.setattr(runner, "Separator", _fake_separator(log, arch="dsd"))
    (tmp_path / "Mixtures").mkdir()
    runner.separate_dataset("dsd", str(tmp_path / "Mixtures"), str(tmp_path / "o"), model=[np.zeros(1)])
    assert log[0][1]["scale_factor"] == 0.3          # the other trainers keep 0.3
