"""The resampling layer without a GPU: the direct formula of the kernel against scipy.signal.resample_poly, the taps the
engine designs against the oracle's, the rate policy, the lengths, and the scripts' --resample behind a stand-in
separator (in the manner of test_cli_host.py)."""
import numpy as np
import pytest
import scipy.io.wavfile
from scipy.signal import resample_poly
from types import SimpleNamespace

import resample_oracle as ro
from deepconvsep_b200 import engine, _lib
from deepconvsep_b200.examples import _common
from deepconvsep_b200.models import FAMILY_DEFAULTS

DIRECTIONS = ("in", "back")


def _pair(rate, direction):
    return (rate, ro.MODEL_RATE) if direction == "in" else (ro.MODEL_RATE, rate)


def _lengths(rate_in, up, down):
    K = 20 * max(up, down) + 1
    return (1, 7, max(8, K // 3), 3 * rate_in)      # 1, 7, shorter than the filter, 3 s


@pytest.mark.parametrize("direction", DIRECTIONS)
@pytest.mark.parametrize("rate", ro.TABLE_RATES)
def test_direct_formula_is_resample_poly(rate, direction):
    rate_in, rate_out = _pair(rate, direction)
    up, down = ro.ratio(rate_in, rate_out)
    h = ro.taps(up, down)
    rng = np.random.default_rng(rate + (direction == "back"))
    for L in _lengths(rate_in, up, down):
        x = rng.standard_normal(L)
        want = resample_poly(x, up, down)
        got = ro.direct(x, up, down, h)
        assert got.shape == want.shape == (ro.length(L, up, down),)
        assert np.max(np.abs(got - want)) <= 1e-12 * max(np.max(np.abs(want)), 1e-300), (rate, direction, L)


@pytest.mark.parametrize("direction", DIRECTIONS)
@pytest.mark.parametrize("rate", ro.TABLE_RATES)
def test_engine_designs_the_oracles_taps(rate, direction):
    rate_in, rate_out = _pair(rate, direction)
    up, down = engine.resample_ratio(rate_in, rate_out)
    assert (up, down) == ro.ratio(rate_in, rate_out)
    h = engine.resample_taps(up, down)
    want = ro.taps(up, down)
    assert h.dtype == np.float64 and h.flags.c_contiguous and h.shape == want.shape
    assert np.array_equal(h.view(np.uint64), want.view(np.uint64))
    assert engine.resample_bank_bytes(up, down) == ro.bank_bytes(up, down)


# the policy's table: rate -> (taps per phase in, out; bank bytes in, out)
TABLE = {48000: (22, 21), 96000: (44, 21), 192000: (88, 21), 64000: (30, 21), 8000: (21, 111), 16000: (21, 56),
         32000: (21, 28), 24000: (21, 37)}


@pytest.mark.parametrize("rate", ro.TABLE_RATES)
def test_policy_accepts_the_table(rate):
    assert ro.accepted(rate)
    for rate_in, rate_out in (_pair(rate, d) for d in DIRECTIONS):
        up, down = engine.check_resample_rates(rate_in, rate_out)
        assert (up, down) == ro.ratio(rate_in, rate_out)
        assert engine.resample_bank_bytes(up, down) <= _lib.RESAMPLE_MAX_BANK_BYTES
    if rate in TABLE:
        qi, qo = TABLE[rate]
        assert ro.taps_per_phase(*ro.ratio(rate, 44100)) == qi and ro.taps_per_phase(*ro.ratio(44100, rate)) == qo


@pytest.mark.parametrize("rate", [44056, 44099, 7999, 192001, 48000.5, 4000, 384000])
def test_policy_refuses(rate):
    assert not ro.accepted(rate)
    for rate_in, rate_out in ((rate, 44100), (44100, rate)):
        with pytest.raises(ValueError, match=str(int(rate)) if rate == int(rate) else "integer"):
            engine.check_resample_rates(rate_in, rate_out)


def test_policy_names_the_rate_and_the_bank():
    with pytest.raises(ValueError, match=r"44099 Hz.*44100/44099"):
        engine.check_resample_rates(44099, 44100)
    with pytest.raises(ValueError, match="integer"):
        engine.check_resample_rates(True, 44100)


def test_lengths():
    lib = _lib.load()
    for rate in ro.TABLE_RATES:
        up, down = ro.ratio(rate, 44100)
        for L in (1, 2, 7, 160, 161, 48000, 48001, 7938001):
            n44 = lib.dcs_resampled_length(L, up, down)
            assert n44 == ro.length(L, up, down) == -(-L * up // down)
            if L < 100000:
                assert n44 == resample_poly(np.zeros(L), up, down).size
            # the way back covers the input: trimming to L is always possible
            assert lib.dcs_resampled_length(n44, down, up) >= L
    assert lib.dcs_resampled_length(-1, 1, 1) == -1 and lib.dcs_resampled_length(5, 0, 1) == -1


def test_score_and_masks_calls_refuse_other_rates():
    """the refusals come before anything touches the device: a stand-in with only the model description will do"""
    sep = SimpleNamespace(model=SimpleNamespace(arch="dsd"))
    for name, args in (("separate_score", (None, None)), ("separate_notes", (None, None)), ("separate_masks", (None,)),
                       ("apply_masks", (None, None))):
        with pytest.raises(ValueError, match="Resampler"):
            getattr(engine.Separator, name)(sep, *args, sample_rate=48000)


# ---- the scripts' --resample -----------------------------------------------------------------------------------
GAINS = (0.5, 0.25, 0.125, 0.0625)


class FakeSeparator(object):
    """scales its input per source and records every call with its sample_rate"""

    def __init__(self, family, calls):
        self.model = SimpleNamespace(arch=family, tc=30)
        self.sources = FAMILY_DEFAULTS[family]["sources"]
        self.nsrc = len(self.sources)
        self.calls = calls

    def separate(self, audio, sample_rate=44100):
        self.calls.append(("separate", np.shape(audio), sample_rate))
        return np.stack([np.asarray(audio, dtype=np.float32) * np.float32(g) for g in GAINS[:self.nsrc]])

    def separate_pcm16(self, pcm, downmix=1, **kw):
        self.calls.append(("separate_pcm16", np.shape(pcm), 44100))
        p = np.asarray(pcm)
        mono = p.astype(np.float32) / np.float32(32767) if p.ndim == 1 else \
            (p[:, 0].astype(np.float32) + p[:, 1].astype(np.float32)) / np.float32(2 * 32767)
        return np.stack([(mono * np.float32(g) * np.float32(32767)).astype(np.int16) for g in GAINS[:self.nsrc]])

    def _channels(self, name, audio, sample_rate, kw):
        self.calls.append((name, np.shape(audio), sample_rate) + ((kw,) if kw else ()))
        a = np.asarray(audio, dtype=np.float32)
        return np.stack([a * np.float32(g) for g in GAINS[:self.nsrc]], axis=1)     # [L, nsrc, C]

    def separate_channels(self, audio, sample_rate=44100, **kw):
        return self._channels("separate_channels", audio, sample_rate, kw)

    def separate_keep_channels(self, audio, sample_rate=44100, **kw):
        return self._channels("separate_keep_channels", audio, sample_rate, kw)


@pytest.fixture
def seen(monkeypatch):
    record = SimpleNamespace(get=[], calls=[])

    def fake(model, arch, frame_size, hop, window, scale_factor, time_context, overlap, feat_size, device=0, slot=0):
        record.get.append(dict(model=model, arch=arch, frame_size=frame_size, hop=hop, window=str(window),
                               scale_factor=scale_factor, time_context=time_context, overlap=overlap, feat_size=feat_size,
                               device=device, slot=slot))
        return FakeSeparator(arch or "ikala", record.calls)
    monkeypatch.setattr(_common, "get_separator", fake)
    return record


def _wav(tmp_path, name, rate, seconds=0.5, channels=1, seed=0):
    rng = np.random.default_rng(seed)
    L = int(rate * seconds)
    pcm = (rng.uniform(-0.4, 0.4, size=(L, channels) if channels > 1 else (L,)) * 32767).astype(np.int16)
    p = tmp_path / name
    scipy.io.wavfile.write(str(p), rate, pcm)
    return str(p), pcm


def _dsd(argv):
    from deepconvsep_b200.examples.dsd100 import separate_dsd
    return separate_dsd.main(argv)


@pytest.mark.parametrize("channels", [1, 2])
def test_resample_flag_separates_a_48k_wav_at_its_rate(tmp_path, seen, channels):
    wav, pcm = _wav(tmp_path, "mix.wav", 48000, channels=channels)
    out = tmp_path / "o"
    out.mkdir()
    _dsd(["-i", wav, "-o", str(out), "-m", "m.pkl", "--resample"])
    assert seen.calls == [("separate", (len(pcm),), 48000)]
    sr, v = scipy.io.wavfile.read(str(out / "vocals.wav"))
    assert sr == 48000 and v.dtype == np.int16 and v.shape == (len(pcm),)
    # the decode of the existing float path: /iinfo.max, (L + R) / 2; the int16 truncation of the stems
    a = pcm.astype("float") / 32767
    mono = a if channels == 1 else (a[:, 0] + a[:, 1]) / 2
    want = ((mono.astype(np.float32) * np.float32(0.5)).astype(np.float64) * 32767).astype(np.int16)
    assert np.array_equal(v, want)


def test_resample_flag_keeps_six_channels(tmp_path, seen):
    wav, pcm = _wav(tmp_path, "surround.wav", 48000, channels=6, seed=1)
    out = tmp_path / "o"
    out.mkdir()
    _dsd(["-i", wav, "-o", str(out), "-m", "m.pkl", "--keep-channels", "--resample"])
    assert seen.calls == [("separate_channels", (len(pcm), 6), 48000)]
    sr, v = scipy.io.wavfile.read(str(out / "bass.wav"))
    assert sr == 48000 and v.shape == (len(pcm), 6)
    want = ((pcm.astype("float") / 32767).astype(np.float32) * np.float32(0.25)).astype(np.float64) * 32767
    assert np.array_equal(v, want.astype(np.int16))


def test_resample_flag_keeps_two_channels_with_the_wiener_filter(tmp_path, seen):
    wav, pcm = _wav(tmp_path, "st.wav", 96000, channels=2, seed=2)
    out = tmp_path / "o"
    out.mkdir()
    _dsd(["-i", wav, "-o", str(out), "-m", "m.pkl", "--keep-channels", "--wiener", "2", "--resample"])
    assert seen.calls == [("separate_keep_channels", (len(pcm), 2), 96000, {"wiener": 2})]
    sr, v = scipy.io.wavfile.read(str(out / "drums.wav"))
    assert sr == 96000 and v.shape == (len(pcm), 2)


@pytest.mark.parametrize("extra", [[], ["--keep-channels"]])
def test_resample_flag_changes_nothing_at_44100(tmp_path, monkeypatch, extra):
    wav, _ = _wav(tmp_path, "mix.wav", 44100, channels=2, seed=3)
    runs = []
    for flags in ([], ["--resample"]):
        record = SimpleNamespace(get=[], calls=[])

        def fake(model, arch, frame_size, hop, window, scale_factor, time_context, overlap, feat_size, device=0, slot=0):
            record.get.append((model, arch, frame_size, hop, str(window), scale_factor, time_context, overlap, feat_size,
                               device, slot))
            return FakeSeparator(arch or "ikala", record.calls)
        monkeypatch.setattr(_common, "get_separator", fake)
        out = tmp_path / ("o%d" % len(runs))
        out.mkdir()
        _dsd(["-i", wav, "-o", str(out), "-m", "m.pkl"] + extra + flags)
        runs.append((record.get, record.calls, {f.name: scipy.io.wavfile.read(str(f))[1].tobytes()
                                                for f in out.iterdir()}))
    assert runs[0] == runs[1]
    assert runs[0][1][0][2] == 44100


def test_one_wav_over_several_devices_at_48k_is_refused_before_a_model_loads(tmp_path, seen):
    wav, _ = _wav(tmp_path, "mix.wav", 48000, channels=2)
    out = tmp_path / "o"
    out.mkdir()
    with pytest.raises(SystemExit, match="48000 Hz"):
        _dsd(["-i", wav, "-o", str(out), "-m", "m.pkl", "--devices", "0,1", "--resample"])
    assert seen.get == [] and list(out.iterdir()) == []
    with pytest.raises(ValueError, match="48000 Hz"):
        _common.run("dsd", wav, str(out), "m.pkl", 0.3, 30, 25, 32, 513, 1024, 512, lambda fn, s: s + ".wav",
                    device=[0, 1], resample=True)
    assert seen.get == []


def test_a_rate_outside_the_policy_is_refused_before_a_model_loads(tmp_path, seen):
    wav, _ = _wav(tmp_path, "odd.wav", 44099, channels=1)
    out = tmp_path / "o"
    out.mkdir()
    with pytest.raises(ValueError, match="44099 Hz"):
        _dsd(["-i", wav, "-o", str(out), "-m", "m.pkl", "--resample"])
    assert seen.get == []


def test_other_scripts_take_the_flag(tmp_path, seen):
    from deepconvsep_b200.examples.ikala import separate_ikala
    from deepconvsep_b200.examples.bach10 import separate_bach10
    wav, pcm = _wav(tmp_path, "song.wav", 32000, channels=2, seed=4)
    out = tmp_path / "o"
    out.mkdir()
    separate_ikala.main(["-i", wav, "-o", str(out), "-m", "m.pkl", "--resample"])
    separate_bach10.main(["-i", wav, "-o", str(out), "-m", "m.pkl", "--resample"])
    assert seen.calls == [("separate", (len(pcm),), 32000)] * 2
    assert scipy.io.wavfile.read(str(out / "song-voice.wav"))[0] == 32000
    assert scipy.io.wavfile.read(str(out / "song_violin.wav"))[0] == 32000
