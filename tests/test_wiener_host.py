"""The --wiener option without a GPU: the scripts pass it to the keep-channels separation and refuse it without
--keep-channels; the runner takes it for --family dsd --keep-channels and --family dsd_ild only."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import scipy.io.wavfile

from deepconvsep_b200 import runner
from deepconvsep_b200.examples import _common
from deepconvsep_b200.models import FAMILY_DEFAULTS


class FakeSeparator(object):
    def __init__(self, family):
        self.model = SimpleNamespace(arch=family, tc=30)
        self.sources = FAMILY_DEFAULTS[family]["sources"]
        self.nsrc = len(self.sources)
        self.calls = []

    def separate_pcm16(self, pcm, downmix=1, keep_channels=False, wiener=0):
        self.calls.append(("pcm16", keep_channels, wiener))
        return np.stack([np.asarray(pcm) // (s + 1) for s in range(self.nsrc)])

    def separate_keep_channels(self, audio, wiener=0):
        self.calls.append(("keep", True, wiener))
        return np.stack([np.asarray(audio, np.float32) / (s + 1) for s in range(self.nsrc)], axis=1)


@pytest.fixture
def fake(monkeypatch):
    made = []

    def get(model, arch, frame_size, hop, window, scale_factor, time_context, overlap, feat_size, device=0, slot=0):
        made.append(FakeSeparator(arch or "ikala"))
        return made[-1]
    monkeypatch.setattr(_common, "get_separator", get)
    return made


def _wav(path, seconds, channels, dtype=np.int16):
    rng = np.random.default_rng(0)
    n = int(44100 * seconds)
    x = rng.uniform(-0.4, 0.4, size=(n, channels) if channels > 1 else (n,))
    scipy.io.wavfile.write(str(path), 44100, (x * np.iinfo(dtype).max).astype(dtype))


@pytest.mark.parametrize("dtype,kind", [(np.int16, "pcm16"), (np.int32, "keep")])
def test_script_passes_wiener_to_the_keep_channels_call(tmp_path, fake, dtype, kind):
    from deepconvsep_b200.examples.dsd100 import separate_dsd
    _wav(tmp_path / "mix.wav", 0.3, 2, dtype)
    out = tmp_path / "o"
    out.mkdir()
    separate_dsd.main(["-i", str(tmp_path / "mix.wav"), "-o", str(out), "-m", "m.pkl", "--keep-channels", "--wiener", "2"])
    assert fake[-1].calls == [(kind, True, 2)]
    assert scipy.io.wavfile.read(str(out / "vocals.wav"))[1].shape == (13230, 2)


def test_script_refuses_wiener_without_keep_channels(tmp_path, fake):
    from deepconvsep_b200.examples.dsd100 import separate_dsd
    _wav(tmp_path / "mix.wav", 0.2, 2)
    out = tmp_path / "o"
    out.mkdir()
    with pytest.raises(SystemExit) as e:
        separate_dsd.main(["-i", str(tmp_path / "mix.wav"), "-o", str(out), "-m", "m.pkl", "--wiener", "1"])
    assert "--wiener needs --keep-channels" in str(e.value.code)
    with pytest.raises(SystemExit):
        separate_dsd.main(["-i", str(tmp_path / "mix.wav"), "-o", str(out), "-m", "m.pkl", "--keep-channels", "--wiener", "-1"])
    assert fake == [] and list(out.iterdir()) == []
    with pytest.raises(ValueError, match="--keep-channels"):
        _common.run("dsd", str(tmp_path / "mix.wav"), str(out), "m.pkl", 0.3, 30, 25, 32, 513, 1024, 512,
                    lambda fn, s: s + ".wav", wiener=2)


def _runner_fake(log):
    class Fake(object):
        def __init__(self, params, arch=None, **kw):
            self.sources = FAMILY_DEFAULTS[arch]["sources"]
            self.nsrc = len(self.sources)

        def separate_keep_channels(self, audio, wiener=0):
            log.append(("keep", wiener))
            return np.stack([np.asarray(audio, np.float32) / (s + 1) for s in range(self.nsrc)], axis=1)

        def separate_stereo(self, audio, wiener=0):
            log.append(("stereo", wiener))
            return np.stack([np.asarray(audio, np.float32) / (s + 1) for s in range(self.nsrc)], axis=1)
    return Fake


@pytest.mark.parametrize("family,keep,kind", [("dsd", True, "keep"), ("dsd_ild", False, "stereo")])
def test_runner_passes_wiener(tmp_path, monkeypatch, family, keep, kind):
    log = []
    monkeypatch.setattr(runner, "Separator", _runner_fake(log))
    db, out = tmp_path / "db", tmp_path / "out"
    song = db / ("Mixtures" if family == "dsd_ild" else "") / "Test" / "001 - A"
    os.makedirs(str(song))
    _wav(song / "mixture.wav", 0.3, 2)
    runner.separate_dataset(family, str(db), str(out), model=[np.zeros(1)], keep_channels=keep, wiener=3)
    assert log == [(kind, 3)]


def test_runner_refuses_wiener_on_mono_stems(tmp_path, monkeypatch):
    with pytest.raises(ValueError, match="--wiener"):
        runner.separate_dataset("dsd", str(tmp_path), str(tmp_path / "o"), model=[np.zeros(1)], wiener=1)
    seen = {}

    def fake_dataset(family, db, out, model, scale_factor, **kw):
        seen.update(family=family, **kw)
        return 1.0, 1
    monkeypatch.setattr(runner, "separate_dataset", fake_dataset)
    runner.main(["--family", "dsd", "--db", "d", "--out", "o", "--model", "m", "--keep-channels", "--wiener", "2"])
    assert seen["wiener"] == 2 and seen["keep_channels"] is True
    runner.main(["--family", "dsd_ild", "--db", "d", "--out", "o", "--model", "m", "--wiener", "1"])
    assert seen["family"] == "dsd_ild" and seen["wiener"] == 1
    for argv in (["--family", "dsd", "--wiener", "1"], ["--family", "ikala", "--wiener", "1"],
                 ["--family", "dsd_ild", "--wiener", "-1"]):
        with pytest.raises(SystemExit):
            runner.main(argv + ["--db", "d", "--out", "o", "--model", "m"])
