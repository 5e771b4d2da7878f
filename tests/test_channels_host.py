"""C-channel stems without a GPU: the float64 oracle (tests/channels_oracle.py) against the mono oracle, the shape
and layout marshalling of Separator.separate_channels / apply_masks and Stft.inverse_masked against a stand-in library
working on host memory, and the option rules of --keep-channels on recordings of more than two channels in
check_stereo_options, clip_call, the stand-alone scripts and the dataset runner."""
import ctypes as C
import os
from types import SimpleNamespace

import numpy as np
import pytest
import scipy.io.wavfile

from oracle import nets, pipeline
import channels_oracle as co

from deepconvsep_b200 import engine, runner
from deepconvsep_b200.engine import Separator, Stft, check_stereo_options, clip_call
from deepconvsep_b200.examples import _common
from deepconvsep_b200.models import FAMILY_DEFAULTS


# ---------------------------------------------------------------------------------------------- the oracle
def test_oracle_one_channel_is_the_mono_oracle_and_six_share_the_masks():
    N, hop = 512, 256
    params = nets.make_synthetic_params("dsd", N // 2 + 1, seed=3)
    a, _ = pipeline.synth_mixture(0.8, 5)
    kw = dict(frameSize=N, hopSize=hop, overlap=25)
    want = pipeline.separate(a, params, "dsd", **kw)
    assert np.array_equal(co.separate_channels(a[:, None], params, **kw)[0][:, :, 0].T, want)
    audio = np.stack([g * np.roll(a, d) for g, d in ((1.0, 0), (0.5, 3), (-0.7, 40), (0.2, 7), (0.9, 111), (0.3, 1))], axis=1)
    stems, mags, _, mms, masks, _ = co.separate_channels(audio, params, **kw)
    assert stems.shape == (len(a), 4, 6)
    for c in range(6):
        assert np.linalg.norm(mms[c][:, :masks.shape[1]] - masks * mags[c]) <= 1e-12 * np.linalg.norm(mms[c])


# ---------------------------------------------------------------------------------------------- marshalling
def _host(ptr, n):
    """the n floats at address ptr"""
    return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_float)), shape=(n,))


class FakeLib(object):
    """the three entry points on host memory: stems plane (s * nx + c) = (s + 1) * channel c (times mask_s[0, 0])"""

    def __init__(self):
        self.calls = []

    def dcs_separate_audio_channels(self, ctx, model, plan, x, nx, stride, L, scale, overlap, patcher, out, ostride, stream):
        self.calls.append(("channels", nx, stride, L, scale, overlap, patcher, ostride))
        a = _host(x, nx * stride).reshape(nx, stride)
        o = _host(out, 4 * nx * ostride).reshape(4 * nx, ostride)
        for s in range(4):
            for c in range(nx):
                o[s * nx + c, :L] = (s + 1) * a[c, :L]
        return 0

    def dcs_apply_masks(self, ctx, plan, x, nx, stride, L, m, nsrc, m_stride, out, ostride, stream):
        self.calls.append(("apply", nx, stride, L, nsrc, m_stride, ostride))
        a = _host(x, nx * stride).reshape(nx, stride)
        mk = _host(m, nsrc * m_stride).reshape(nsrc, m_stride)
        o = _host(out, nsrc * nx * ostride).reshape(nsrc * nx, ostride)
        for s in range(nsrc):
            for c in range(nx):
                o[s * nx + c, :L] = mk[s, 0] * a[c, :L]
        return 0

    def dcs_istft_masked(self, plan, X, nx, x_plane, M, nsrc, m_stride, T, ldf, out, n, ostride, stream):
        self.calls.append(("istft_masked", nx, x_plane, nsrc, m_stride, T, ldf, n, ostride))
        _host(out, nsrc * nx * ostride)[:] = 1.0
        return 0


@pytest.fixture
def sep(monkeypatch):
    torch = pytest.importorskip("torch")
    monkeypatch.setattr(engine, "_stream_ptr", lambda stream=None, device=None: None)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))     # host tensors stand for device planes
    lib = FakeLib()
    N, hop = 1024, 512
    s = object.__new__(Separator)
    s.lib, s.nsrc, s.scale_factor, s.overlap, s.patcher = lib, 4, 0.3, 25, 0
    s.ctx = SimpleNamespace(handle=1, device=0, lib=lib)
    s.model = SimpleNamespace(arch="dsd", handle=2, F=N // 2 + 1)
    st = object.__new__(Stft)
    st.ctx, st.lib, st.N, st.hop, st.device, st.F, st.ldf, st.handle = s.ctx, lib, N, hop, 0, N // 2 + 1, 520, 3
    st.num_frames = lambda L: (int(L) + hop - 1) // hop + 2
    monkeypatch.setattr(Stft, "dev", property(lambda self: torch.device("cpu")))
    s.stft = st
    return s


@pytest.mark.parametrize("nch", [1, 2, 6])
def test_separate_channels_layouts(sep, nch):
    import torch
    L = 3000
    audio = np.random.default_rng(nch).uniform(-1, 1, (L, nch))
    got = sep.separate_channels(audio)
    assert got.shape == (L, 4, nch) and got.dtype == np.float32 and got.flags.c_contiguous
    for s in range(4):
        assert np.array_equal(got[:, s, :], (s + 1) * audio.astype(np.float32))
    assert sep.lib.calls[-1] == ("channels", nch, L, L, 0.3, 25, 0, L)
    x = torch.as_tensor(np.ascontiguousarray(audio.T.astype(np.float32)))
    planes = sep.separate_channels(x)
    assert tuple(planes.shape) == (4 * nch, L)
    assert np.array_equal(planes.numpy().reshape(4, nch, L).transpose(2, 0, 1), got)
    out = np.empty((L, 4, nch), dtype=np.float32)
    assert sep.separate_channels(audio, out=out) is out and np.array_equal(out, got)


def test_separate_channels_refusals(sep):
    with pytest.raises(ValueError, match="1 to 16"):
        sep.separate_channels(np.zeros(1000))
    with pytest.raises(ValueError, match="1 to 16"):
        sep.separate_channels(np.zeros((1000, 17)))
    n = len(sep.lib.calls)
    for arch in ("dsd_ild", "bach10_score", "bach10_score_1x1"):
        sep.model.arch = arch
        with pytest.raises(ValueError, match="separate_masks.*apply_masks"):
            sep.separate_channels(np.zeros((1000, 3)))
    assert len(sep.lib.calls) == n


def test_apply_masks_layouts(sep):
    import torch
    L, nch, nsrc = 2000, 3, 5
    T, F, ldf = sep.stft.num_frames(L), sep.stft.F, sep.stft.ldf
    audio = np.random.default_rng(1).uniform(-1, 1, (L, nch))
    masks = np.random.default_rng(2).uniform(0, 1, (nsrc, T, F))
    got = sep.apply_masks(audio, masks)
    assert got.shape == (L, nsrc, nch) and got.dtype == np.float32
    for s in range(nsrc):
        assert np.array_equal(got[:, s, :], np.float32(masks[s, 0, 0]) * audio.astype(np.float32))
    assert sep.lib.calls[-1] == ("apply", nch, L, L, nsrc, T * ldf, L)
    # device layout: masks [nsrc, T, ldf] as a view with a gap between planes
    buf = torch.zeros((nsrc, T * ldf + 24))
    md = buf[:, :T * ldf].view(nsrc, T, ldf)
    md[:, :, :F] = torch.as_tensor(masks.astype(np.float32))
    planes = sep.apply_masks(torch.as_tensor(np.ascontiguousarray(audio.T.astype(np.float32))), md)
    assert tuple(planes.shape) == (nsrc * nch, L) and sep.lib.calls[-1] == ("apply", nch, L, L, nsrc, T * ldf + 24, L)
    assert np.array_equal(planes.numpy().reshape(nsrc, nch, L).transpose(2, 0, 1), got)
    with pytest.raises(ValueError, match=r"\[nsrc, %d, %d\]" % (T, F)):
        sep.apply_masks(audio, masks[:, :-1])
    with pytest.raises(ValueError, match="1 to 16"):
        sep.apply_masks(audio[:, 0], masks)


def test_inverse_masked_strides(sep):
    import torch
    st = sep.stft
    X = torch.zeros((2, 9, st.ldf), dtype=torch.complex64)
    M = torch.zeros((3, 9 * st.ldf + 8))[:, :9 * st.ldf].view(3, 9, st.ldf)
    out = st.inverse_masked(X, M, num_out=700)
    assert tuple(out.shape) == (6, 700) and bool((out == 1).all())
    assert sep.lib.calls[-1] == ("istft_masked", 2, 9 * st.ldf, 3, 9 * st.ldf + 8, 9, st.ldf, 700, 700)
    assert tuple(st.inverse_masked(X[0], M[0]).shape) == (1, 8 * 512 + 512)
    with pytest.raises(ValueError):
        st.inverse_masked(X, M[:, :8])


# ---------------------------------------------------------------------------------------------- option rules
def test_check_stereo_options_by_channel_count():
    with pytest.raises(ValueError, match="at least a 2-channel"):
        check_stereo_options("dsd", True, channels=1)
    for fam in ("dsd", "ikala", "ikala_nopool", "bach10"):
        check_stereo_options(fam, True, channels=6)
        with pytest.raises(ValueError, match="--wiener 2.*two-channel stems.*6 channels"):
            check_stereo_options(fam, True, wiener=2, channels=6)
    for fam in ("dsd_ild", "bach10_score", "bach10_score_1x1"):
        with pytest.raises(ValueError, match="separate_masks.*apply_masks"):
            check_stereo_options(fam, True, channels=6)
    # two channels, or a count not known: the rule as it was
    check_stereo_options("dsd", True, wiener=2, channels=2)
    with pytest.raises(ValueError, match="only the DSD100"):
        check_stereo_options("ikala", True, channels=2)
    with pytest.raises(ValueError, match="only the DSD100"):
        check_stereo_options("ikala", True)


def test_clip_call_routes_by_channel_count():
    s = SimpleNamespace(model=SimpleNamespace(arch="dsd"), separate_channels="channels", separate_keep_channels=lambda a, wiener=0: "keep")
    assert clip_call(s, keep_channels=True, channels=6) == "channels"
    assert clip_call(s, keep_channels=True, channels=2)(None) == "keep"
    assert clip_call(s, keep_channels=True)(None) == "keep"
    with pytest.raises(ValueError, match="two-channel stems"):
        clip_call(s, keep_channels=True, wiener=1, channels=3)
    s.model.arch = "dsd_ild"
    with pytest.raises(ValueError, match="apply_masks"):
        clip_call(s, keep_channels=True, channels=3)


class FakeSeparator(object):
    def __init__(self, family):
        self.model = SimpleNamespace(arch=family, tc=30)
        self.sources = FAMILY_DEFAULTS[family]["sources"]
        self.nsrc = len(self.sources)
        self.calls = []

    def separate_pcm16(self, pcm, downmix=1, keep_channels=False):
        self.calls.append(("pcm16_keep" if keep_channels else "pcm16", pcm.shape))
        return np.stack([np.asarray(pcm) // (s + 1) for s in range(self.nsrc)]).astype(np.int16)

    def separate_channels(self, audio):
        self.calls.append(("channels", audio.shape))
        return np.stack([np.asarray(audio, np.float32) / (s + 1) for s in range(self.nsrc)], axis=1)


@pytest.fixture
def fake(monkeypatch):
    made = []

    def get(model, arch, frame_size, hop, window, scale_factor, time_context, overlap, feat_size, device=0, slot=0):
        made.append(FakeSeparator(arch or "ikala"))
        return made[-1]
    monkeypatch.setattr(_common, "get_separator", get)
    return made


def _wav(path, seconds, channels, seed=0):
    n = int(44100 * seconds)
    x = np.random.default_rng(seed).uniform(-0.4, 0.4, size=(n, channels) if channels > 1 else (n,))
    pcm = (x * 32767).astype(np.int16)
    scipy.io.wavfile.write(str(path), 44100, pcm)
    return pcm


@pytest.mark.parametrize("script,first", [("dsd100.separate_dsd", "bass.wav"), ("ikala.separate_ikala", "mix-music.wav"),
                                          ("bach10.separate_bach10", "mix_bassoon.wav")])
def test_scripts_write_six_channel_stems(tmp_path, fake, script, first):
    import importlib
    mod = importlib.import_module("deepconvsep_b200.examples." + script)
    pcm = _wav(tmp_path / "mix.wav", 0.2, 6)
    out = tmp_path / "o"
    out.mkdir()
    mod.main(["-i", str(tmp_path / "mix.wav"), "-o", str(out), "-m", "m.pkl", "--keep-channels"])
    assert fake[-1].calls == [("channels", pcm.shape)]
    names = sorted(f.name for f in out.iterdir())
    assert names[0] == first and len(names) == fake[-1].nsrc
    v = scipy.io.wavfile.read(str(out / first))[1]
    assert v.dtype == np.int16 and v.shape == pcm.shape
    with pytest.raises(SystemExit) as e:
        mod.main(["-i", str(tmp_path / "mix.wav"), "-o", str(out), "-m", "m.pkl", "--keep-channels", "--wiener", "1"])
    assert "two-channel stems" in str(e.value.code) or "only the DSD100" in str(e.value.code) or "--wiener" in str(e.value.code)
    assert len(fake) == 1


def test_dsd_script_keeps_the_stereo_path_for_two_channels(tmp_path, fake):
    from deepconvsep_b200.examples.dsd100 import separate_dsd
    pcm = _wav(tmp_path / "mix.wav", 0.2, 2)
    out = tmp_path / "o"
    out.mkdir()
    separate_dsd.main(["-i", str(tmp_path / "mix.wav"), "-o", str(out), "-m", "m.pkl", "--keep-channels"])
    assert fake[-1].calls == [("pcm16_keep", pcm.shape)]
    _wav(tmp_path / "mono.wav", 0.2, 1)
    with pytest.raises(ValueError, match="2-channel"):
        _common.run("dsd", str(tmp_path / "mono.wav"), str(out), "m.pkl", 0.3, 30, 25, 32, 513, 1024, 512,
                    lambda fn, s: s + ".wav", keep_channels=True)
    with pytest.raises(ValueError, match="--wiener 1"):
        _wav(tmp_path / "five.wav", 0.1, 5)
        _common.run("dsd", str(tmp_path / "five.wav"), str(out), "m.pkl", 0.3, 30, 25, 32, 513, 1024, 512,
                    lambda fn, s: s + ".wav", keep_channels=True, wiener=1)
    assert len(fake) == 1


def _runner_fake(log):
    class Fake(object):
        def __init__(self, params, arch=None, **kw):
            self.sources = FAMILY_DEFAULTS[arch or "ikala"]["sources"]
            self.nsrc = len(self.sources)
            self.model = SimpleNamespace(arch=arch or "ikala")

        def separate_channels(self, audio):
            log.append(("channels", audio.shape))
            return np.stack([np.asarray(audio, np.float32) / (s + 1) for s in range(self.nsrc)], axis=1)

        def separate_keep_channels(self, audio):
            log.append(("keep", audio.shape))
            return np.stack([np.asarray(audio, np.float32) / (s + 1) for s in range(self.nsrc)], axis=1)
    return Fake


@pytest.mark.parametrize("family,nch,kind", [("dsd", 6, "channels"), ("dsd", 2, "keep"), ("bach10", 4, "channels")])
def test_runner_routes_by_channel_count(tmp_path, monkeypatch, family, nch, kind):
    log = []
    monkeypatch.setattr(runner, "Separator", _runner_fake(log))
    db, out = tmp_path / "db", tmp_path / "out"
    if family == "dsd":
        os.makedirs(str(db / "Test" / "001 - A"))
        wav = db / "Test" / "001 - A" / "mixture.wav"
    else:
        os.makedirs(str(db))
        wav = db / "piece.wav"
    pcm = _wav(wav, 0.2, nch)
    runner.separate_dataset(family, str(db), str(out), model=[np.zeros(1)], keep_channels=True)
    assert log == [(kind, pcm.shape)]
    first = out / "Test" / "001 - A" / "vocals.wav" if family == "dsd" else out / "piece_bassoon.wav"
    assert scipy.io.wavfile.read(str(first))[1].shape == pcm.shape
    if nch > 2:
        with pytest.raises(ValueError, match="two-channel stems"):
            runner.separate_dataset(family, str(db), str(out), model=[np.zeros(1)], keep_channels=True, wiener=1)
        seen = {}
        monkeypatch.setattr(runner, "separate_dataset", lambda fam, *a, **kw: (seen.update(kw), (1.0, 1))[1])
        runner.main(["--family", family, "--db", str(db), "--out", str(out), "--model", "m", "--keep-channels"])
        assert seen["keep_channels"] is True
