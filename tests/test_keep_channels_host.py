"""Keep-channels mode of the DSD100 / hiphopss network without a GPU: the float64 oracle (tests/channels_oracle.py at
C = 2) against the mono oracle, and the --keep-channels flags of the stand-alone scripts and of the dataset runner with
stand-in separators."""
import os
import numpy as np
import pytest
import scipy.io.wavfile
from types import SimpleNamespace

from oracle import dsp, nets, pipeline
from channels_oracle import separate_channels

N, HOP = 512, 256


def _params(seed):
    return nets.make_synthetic_params("dsd", N // 2 + 1, seed=seed)


def _stereo(seconds, seed):
    mix, _ = pipeline.synth_mixture(seconds, seed)
    other, _ = pipeline.synth_mixture(seconds, seed + 1)
    return np.stack([0.7 * mix + 0.3 * other, 0.4 * mix - 0.6 * np.roll(other, 11)], axis=1)


@pytest.mark.parametrize("patcher", ["standalone", "util"])
def test_equal_channels_are_the_mono_oracle_bit_for_bit(patcher):
    params = _params(11)
    mono, _ = pipeline.synth_mixture(1.0, 5)
    kw = dict(frameSize=N, hopSize=HOP, overlap=25, patcher=patcher)
    want, mag, ph, mm = pipeline.separate(mono, params, "dsd", return_spec=True, count_kinks=True, **kw)
    kmap = pipeline.separate.last_kink_map
    stems, mags, phs, mms, _, km = separate_channels(np.stack([mono, mono], axis=1), params, **kw)
    assert stems.shape == (len(mono), 4, 2)
    for c in range(2):
        assert np.array_equal(stems[:, :, c].T, want)
        assert np.array_equal(mags[c], mag) and np.array_equal(phs[c], ph) and np.array_equal(mms[c], mm)
    assert np.array_equal(km, kmap)
    assert np.linalg.norm(want) > 0


def test_different_channels_share_the_downmix_masks():
    params = _params(12)
    audio = _stereo(1.0, 21)
    kw = dict(frameSize=N, hopSize=HOP, overlap=25)
    stems, mags, phs, mms, M, _ = separate_channels(audio, params, **kw)
    T = phs[0].shape[0]
    # per channel: the blended masks of the downmix times that channel's magnitude
    for c in range(2):
        assert np.linalg.norm(mms[c][:, :T] - M[:, :T] * mags[c]) <= 1e-12 * np.linalg.norm(mms[c])
    # the same masks are the mono oracle's: its blended magnitudes are M~ times the downmix's magnitude
    mono = (audio[:, 0] + audio[:, 1]) / 2
    _, mag_m, ph_m, mm_m = pipeline.separate(mono, params, "dsd", return_spec=True, **kw)
    assert np.linalg.norm(mm_m[:, :T] - M[:, :T] * mag_m) <= 1e-12 * np.linalg.norm(mm_m)
    # so (S_L + S_R) / 2 = M~ (X_L + X_R) / 2 is the mono spectra M~ X_mono (the STFT is linear)
    X = [dsp.stft_norm(audio[:, c], window=np.hanning(N), hopsize=HOP, nfft=N, fs=44100) for c in range(2)]
    Xm = dsp.stft_norm(mono, window=np.hanning(N), hopsize=HOP, nfft=N, fs=44100)
    S = [M[:, :T] * X[c][None] for c in range(2)]
    Sm = M[:, :T] * Xm[None]
    assert np.linalg.norm((S[0] + S[1]) / 2 - Sm) <= 1e-12 * np.linalg.norm(Sm)
    # the oracle's own spectra (float32-rounded magnitudes, as the reference rounds them) agree to that rounding
    Sc = [mms[c][:, :T] / 0.3 * np.sqrt(N) * np.exp(1j * phs[c])[None] for c in range(2)]
    Sm_or = mm_m[:, :T] / 0.3 * np.sqrt(N) * np.exp(1j * ph_m)[None]
    assert np.linalg.norm((Sc[0] + Sc[1]) / 2 - Sm_or) <= 1e-6 * np.linalg.norm(Sm_or)
    for i in range(4):
        for c in range(2):
            assert np.linalg.norm(stems[:, i, c]) > 0


def test_anti_phase_channels_give_finite_stems():
    params = _params(13)
    x, _ = pipeline.synth_mixture(0.6, 8)
    stems, mags, phs, mms, _, _ = separate_channels(np.stack([x, -x], axis=1), params, frameSize=N, hopSize=HOP, overlap=25)
    assert np.isfinite(stems).all() and all(np.isfinite(m).all() for m in mms)
    # the downmix is silent, the channels are not: the masks (of a silent input) still carry each channel through
    assert np.linalg.norm(stems) > 0


# ---- command line and dataset runner, with stand-in separators ----------------------------------------------------
from deepconvsep_b200.examples import _common  # noqa: E402
from deepconvsep_b200.models import FAMILY_DEFAULTS  # noqa: E402
from deepconvsep_b200 import runner  # noqa: E402

GAINS = (0.5, 0.25, 0.125, 0.0625)


class FakeSeparator(object):
    def __init__(self, family):
        self.model = SimpleNamespace(arch=family, tc=30)
        self.sources = FAMILY_DEFAULTS[family]["sources"]
        self.nsrc = len(self.sources)
        self.calls = []

    def separate_pcm16(self, pcm, downmix=1, keep_channels=False):
        assert keep_channels
        self.calls.append(("pcm16_keep", pcm.shape))
        p = np.asarray(pcm).astype(np.float32) / np.float32(32767)
        return np.stack([(p * np.float32(g) * np.float32(32767)).astype(np.int16) for g in GAINS[:self.nsrc]])

    def separate_keep_channels(self, audio):
        self.calls.append(("keep", audio.shape))
        a = np.asarray(audio, dtype=np.float32)
        return np.stack([a * np.float32(g) for g in GAINS[:self.nsrc]], axis=1)     # [L, nsrc, 2]


@pytest.fixture
def fake(monkeypatch):
    made = []

    def get(model, arch, frame_size, hop, window, scale_factor, time_context, overlap, feat_size, device=0, slot=0):
        made.append(FakeSeparator(arch or "ikala"))
        return made[-1]
    monkeypatch.setattr(_common, "get_separator", get)
    return made


def _wav(path, seconds, channels, dtype=np.int16, seed=0):
    rng = np.random.default_rng(seed)
    n = int(44100 * seconds)
    x = rng.uniform(-0.4, 0.4, size=(n, channels) if channels > 1 else (n,))
    data = (x * np.iinfo(dtype).max).astype(dtype) if dtype != np.float32 else x.astype(np.float32)
    scipy.io.wavfile.write(str(path), 44100, data)
    return data


def test_dsd_script_keep_channels_writes_stereo_stems(tmp_path, fake):
    from deepconvsep_b200.examples.dsd100 import separate_dsd
    pcm = _wav(tmp_path / "mix.wav", 0.5, 2)
    out = tmp_path / "o"
    out.mkdir()
    separate_dsd.main(["-i", str(tmp_path / "mix.wav"), "-o", str(out), "-m", "m.pkl", "--keep-channels"])
    assert fake[-1].calls == [("pcm16_keep", pcm.shape)]                        # the int16 path
    assert sorted(f.name for f in out.iterdir()) == ["bass.wav", "drums.wav", "other.wav", "vocals.wav"]
    sr, v = scipy.io.wavfile.read(str(out / "bass.wav"))
    want = (pcm.astype(np.float32) / np.float32(32767) * np.float32(0.25) * np.float32(32767)).astype(np.int16)
    assert sr == 44100 and v.dtype == np.int16 and v.shape == pcm.shape and np.array_equal(v, want)
    # hiphopss is the same script
    from deepconvsep_b200.examples.hiphopss import separate_hhds
    out2 = tmp_path / "o2"
    out2.mkdir()
    separate_hhds.main(["-i", str(tmp_path / "mix.wav"), "-o", str(out2), "-m", "m.pkl", "--keep-channels"])
    assert scipy.io.wavfile.read(str(out2 / "vocals.wav"))[1].shape == pcm.shape


def test_dsd_script_keep_channels_float_wav(tmp_path, fake):
    from deepconvsep_b200.examples.dsd100 import separate_dsd
    _wav(tmp_path / "mix.wav", 0.2, 2, dtype=np.int32)
    out = tmp_path / "o"
    out.mkdir()
    separate_dsd.main(["-i", str(tmp_path / "mix.wav"), "-o", str(out), "-m", "m.pkl", "--keep-channels"])
    assert fake[-1].calls[0][0] == "keep"
    v = scipy.io.wavfile.read(str(out / "vocals.wav"))[1]
    assert v.dtype == np.int16 and v.shape == (8820, 2)


def test_keep_channels_refuses_mono_files(tmp_path, fake):
    from deepconvsep_b200.examples.dsd100 import separate_dsd
    _wav(tmp_path / "mono.wav", 0.2, 1)
    out = tmp_path / "o"
    out.mkdir()
    with pytest.raises(ValueError, match="2-channel"):
        separate_dsd.main(["-i", str(tmp_path / "mono.wav"), "-o", str(out), "-m", "m.pkl", "--keep-channels"])
    assert list(out.iterdir()) == []


@pytest.mark.parametrize("script", ["ikala.separate_ikala", "bach10.separate_bach10"])
def test_keep_channels_refused_for_other_families(tmp_path, fake, script):
    import importlib
    mod = importlib.import_module("deepconvsep_b200.examples." + script)
    _wav(tmp_path / "mix.wav", 0.2, 2)
    out = tmp_path / "o"
    out.mkdir()
    with pytest.raises(SystemExit) as e:
        mod.main(["-i", str(tmp_path / "mix.wav"), "-o", str(out), "-m", "m.pkl", "--keep-channels"])
    assert "only the DSD100 / hiphopss network" in str(e.value.code)
    assert fake == [] and list(out.iterdir()) == []
    with pytest.raises(ValueError, match="only the DSD100"):
        _common.run("ikala", str(tmp_path / "mix.wav"), str(out), "m.pkl", 0.3, 30, 20, 32, 513, 1024, 512,
                    lambda fn, s: s + ".wav", keep_channels=True)


def _runner_fake(log):
    class Fake(object):
        def __init__(self, params, arch=None, **kw):
            log.append(("init", arch))
            self.sources = FAMILY_DEFAULTS[arch or "ikala"]["sources"]
            self.nsrc = len(self.sources)

        def separate(self, audio):
            raise AssertionError("the mono path must not run with keep_channels")

        def separate_keep_channels(self, audio):
            log.append(("keep", audio.shape))
            a = np.asarray(audio, dtype=np.float32)
            return np.stack([a / (s + 1) for s in range(self.nsrc)], axis=1)
    return Fake


def test_runner_keep_channels_writes_stereo_stems_in_the_dsd_layout(tmp_path, monkeypatch):
    log = []
    monkeypatch.setattr(runner, "Separator", _runner_fake(log))
    db, out = tmp_path / "Mixtures", tmp_path / "out"
    for sub, song, secs in (("Dev", "051 - A", 0.5), ("Test", "005 - B", 0.3)):
        os.makedirs(str(db / sub / song))
        _wav(db / sub / song / "mixture.wav", secs, 2, seed=len(song))
    secs, njobs = runner.separate_dataset("dsd", str(db), str(out), model=[np.zeros(1)], keep_channels=True)
    assert njobs == 2 and abs(secs - 0.8) < 1e-3
    assert [e[0] for e in log] == ["init", "keep", "keep"]
    mix = scipy.io.wavfile.read(str(db / "Test" / "005 - B" / "mixture.wav"))[1]
    for s, name in enumerate(("vocals", "bass", "drums", "other")):
        sr, y = scipy.io.wavfile.read(str(out / "Test" / "005 - B" / (name + ".wav")))
        assert y.shape == mix.shape and y.dtype == np.int16
        a = (mix / 32767.0).astype(np.float32) / np.float32(s + 1)
        assert np.array_equal(y, (a.astype(np.float64) * 32767).astype(np.int16))


def test_runner_keep_channels_flag(tmp_path, monkeypatch):
    with pytest.raises(ValueError, match="family dsd"):
        runner.separate_dataset("bach10", str(tmp_path), str(tmp_path / "o"), model=[np.zeros(1)], keep_channels=True)
    seen = {}

    def fake_dataset(family, db, out, model, scale_factor, **kw):
        seen.update(family=family, **kw)
        return 1.0, 1
    monkeypatch.setattr(runner, "separate_dataset", fake_dataset)
    runner.main(["--family", "dsd", "--db", "d", "--out", "o", "--model", "m", "--keep-channels"])
    assert seen["family"] == "dsd" and seen["keep_channels"] is True
    runner.main(["--family", "dsd", "--db", "d", "--out", "o", "--model", "m"])
    assert seen["keep_channels"] is False
    with pytest.raises(SystemExit):
        runner.main(["--family", "ikala", "--db", "d", "--out", "o", "--model", "m", "--keep-channels"])
