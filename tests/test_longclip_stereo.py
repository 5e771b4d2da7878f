"""Stereo stems of one long recording cut into segments (deepconvsep_b200.longclip with keep_channels / wiener /
wiener_radius), with the float64 keep-channels oracle and the float64 sliding-window Wiener filter as the engine: the
stitched stems are the whole-clip stems bit for bit, the Wiener margins are tight to one chunk, segments start on the
chunk grid, whole-clip covariances over several segments are refused, and the scripts cut one stereo wav over devices."""
import math
import os
import socket
from types import SimpleNamespace

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

from deepconvsep_b200 import longclip
from oracle import dsp, nets, pipeline
import channels_oracle as co
import wiener_local_oracle as WL

CHUNK = WL.CHUNK


class OracleKeepSeparator(object):
    """The Separator's keep-channels call in float64: the keep-channels oracle's spectra, the sliding-window Wiener
    filter on them against the float64 STFT of each channel, the inverse STFT -> [L, nsrc, 2]"""

    def __init__(self, N, H, overlap, seed=3):
        self.model = SimpleNamespace(arch="dsd", tc=30)
        self.frame_size, self.hop, self.overlap = N, H, overlap
        self.params = nets.make_synthetic_params("dsd", N // 2 + 1, seed=seed)
        self.calls = []

    def separate_keep_channels(self, audio, wiener=0, wiener_radius=0):
        audio = np.asarray(audio, dtype=np.float64)
        self.calls.append((audio.shape[0], wiener, wiener_radius))
        N, H = self.frame_size, self.hop
        stems, _, phs, mms, _, _ = co.separate_channels(audio, self.params, frameSize=N, hopSize=H, overlap=self.overlap)
        if not wiener:
            return stems
        win = np.hanning(N)
        T = phs[0].shape[0]
        X = np.stack([dsp.stft_norm(audio[:, c], win, H, N) for c in range(2)])
        S0 = np.stack([[mms[c][j, :T] / 0.3 * np.sqrt(N) * np.exp(1j * phs[c]) for c in range(2)] for j in range(4)])
        Y = WL.wiener_windowed(X, S0, wiener, wiener_radius)
        L = audio.shape[0]
        for j in range(4):
            for c in range(2):
                stems[:, j, c] = dsp.istft_norm(Y[j, c], win, hopsize=H, nfft=N)[:L]
        return stems


def stereo_mix(L, seed):
    mix, _ = pipeline.synth_mixture(L / 44100.0 + 0.1, seed)
    other, _ = pipeline.synth_mixture(L / 44100.0 + 0.1, seed + 1)
    return np.stack([0.7 * mix[:L] + 0.3 * other[:L], 0.4 * mix[:L] + 0.6 * np.roll(other, 11)[:L]], axis=1)


def clip_for(parts, N, H, ov, reach, extra=77):
    left, right = longclip.margins(N, H, 30, ov, reach)
    return parts * 2 * (left + right) + extra


@pytest.mark.parametrize("N,H,overlap,K,W,parts", [
    (256, 128, 25, 1, 1, 3),     # N / H = 2
    (256, 32, 20, 2, 3, 2),      # N / H = 8, step 10
    (256, 128, 20, 2, 1, 3),
    (256, 32, 25, 1, 3, 2),
    (256, 128, 25, 0, 0, 3),     # keep-channels without the filter: the plain margins
])
def test_stitched_equals_whole_bit_for_bit(N, H, overlap, K, W, parts):
    sep = OracleKeepSeparator(N, H, overlap)
    L = clip_for(parts, N, H, overlap, K * W)
    audio = stereo_mix(L, 40 + K + W)
    whole = sep.separate_keep_channels(audio, wiener=K, wiener_radius=W)
    segs = longclip.plan_segments(L, parts, N, H, 30, overlap, wiener_reach=K * W)
    assert len(segs) == parts
    got = longclip.separate_long([sep, sep], audio, parts=parts, keep_channels=True, wiener=K, wiener_radius=W)
    assert got.shape == whole.shape == (L, 4, 2)
    assert np.array_equal(got, whole), np.abs(got - whole).max()
    assert [c[1:] for c in sep.calls[1:]] == [(K, W)] * parts
    if K:
        plain = sep.separate_keep_channels(audio)
        assert np.abs(whole - plain).max() > 1e-3 * np.abs(plain).max()       # the filter did something


def test_wiener_margins_are_tight_to_one_chunk():
    """at the exact margins the stitched stems are the whole clip's; one chunk less on the left (the cut moved left by
    CHUNK hops, segment inputs unchanged) or on the right (the first segment's input ends CHUNK hops earlier) and they
    differ"""
    N, H, ov, K, W = 256, 128, 25, 2, 1
    sep = OracleKeepSeparator(N, H, ov)
    L = clip_for(2, N, H, ov, K * W)
    audio = stereo_mix(L, 9)
    whole = sep.separate_keep_channels(audio, wiener=K, wiener_radius=W)
    a, b = longclip.plan_segments(L, 2, N, H, 30, ov, wiener_reach=K * W)
    left, _ = longclip.margins(N, H, 30, ov, K * W)
    o = b.in_start + left                                      # the first sample segment b may keep
    assert o <= b.out_start

    def stitched(segs):
        pieces = [sep.separate_keep_channels(audio[s.in_start:s.in_stop], wiener=K, wiener_radius=W) for s in segs]
        return longclip.stitch(segs, [np.moveaxis(p, 0, -1) for p in pieces], L, dtype=np.float64)

    want = np.moveaxis(whole, 0, -1)
    exact = [a._replace(out_stop=o), b._replace(out_start=o)]
    assert np.array_equal(stitched(exact), want)
    short_left = [a._replace(out_stop=o - CHUNK * H), b._replace(out_start=o - CHUNK * H)]
    short_right = [a._replace(in_stop=a.in_stop - CHUNK * H), b]
    for bad in (short_left, short_right):
        assert not np.array_equal(stitched(bad), want)


def test_the_chunk_length_is_the_headers():
    import re
    from deepconvsep_b200 import _lib
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "dcs.h")).read()
    assert int(re.search(r"#define DCS_WIENER_CHUNK_FRAMES (\d+)", hdr).group(1)) == _lib.WIENER_CHUNK_FRAMES == CHUNK


def test_segment_starts_are_on_the_patch_and_chunk_grids():
    for (N, H, tc, ov) in ((1024, 512, 30, 25), (2048, 512, 30, 25), (1024, 128, 30, 20), (256, 32, 30, 23)):
        for reach in (1, 2, 6):
            align = math.lcm(tc - ov, CHUNK)
            for L in (5000, 44100 * 60 + 13, 44100 * 600):
                for parts in (1, 2, 3, 8):
                    segs = longclip.plan_segments(L, parts, N, H, tc, ov, wiener_reach=reach)
                    assert segs[0].in_start == 0 and segs[-1].in_stop == L
                    for x, y in zip(segs, segs[1:]):
                        assert x.out_stop == y.out_start
                    for s in segs:
                        assert s.frame0 % align == 0 and s.in_start == s.frame0 * H
                        assert s.in_start <= s.out_start < s.out_stop <= s.in_stop


def test_whole_clip_covariances_over_several_segments_are_refused_before_any_segment_runs():
    N, H, ov = 256, 128, 25
    sep = OracleKeepSeparator(N, H, ov)
    L = clip_for(3, N, H, ov, 1)
    audio = np.zeros((L, 2))
    with pytest.raises(ValueError, match="wiener_radius"):
        longclip.separate_long([sep, sep], audio, parts=3, keep_channels=True, wiener=2)
    for bad in (dict(wiener=0, wiener_radius=1), dict(wiener=1, wiener_radius=-1)):
        with pytest.raises(ValueError, match="--wiener-radius"):
            longclip.separate_long([sep, sep], audio, parts=3, keep_channels=True, **bad)
    assert sep.calls == []
    # one segment: the whole-clip filter is that of the whole-clip call
    short = stereo_mix(20000, 3)
    got = longclip.separate_long(sep, short, parts=1, keep_channels=True, wiener=1)
    assert np.array_equal(got, sep.separate_keep_channels(short, wiener=1))


def _worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    N, H, ov, K, W = 256, 128, 20, 2, 1
    sep = OracleKeepSeparator(N, H, ov)
    audio = stereo_mix(clip_for(2, N, H, ov, K * W), 12)
    out = longclip.separate_long_distributed(sep, audio, keep_channels=True, wiener=K, wiener_radius=W)
    dist.barrier()
    if rank == 0:
        q.put(bool(np.array_equal(out, sep.separate_keep_channels(audio, wiener=K, wiener_radius=W))))
    else:
        assert out is None
    dist.destroy_process_group()


def test_two_rank_gloo_stereo_long_clip():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    equal = q.get(timeout=600)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert equal


class ScalingKeepSeparator(object):
    """stand-in for the CUDA Separator: source s = the input times 2^-(s+1), as [L, nsrc, 2]"""
    calls = []

    def __init__(self, device):
        self.device = device
        self.model = SimpleNamespace(arch="dsd", tc=30)
        self.frame_size, self.hop, self.overlap = 1024, 512, 25
        self.sources = ["vocals", "bass", "drums", "other"]

    def separate_keep_channels(self, sub, wiener=0, wiener_radius=0):
        self.calls.append((self.device, len(sub), wiener, wiener_radius))
        return np.stack([np.asarray(sub, dtype=np.float32) * g for g in (0.5, 0.25, 0.125, 0.0625)], axis=1)


def test_cli_cuts_one_stereo_wav_over_the_listed_devices(tmp_path, monkeypatch):
    import scipy.io.wavfile
    from deepconvsep_b200.examples import _common
    from deepconvsep_b200.examples.dsd100 import separate_dsd

    calls = ScalingKeepSeparator.calls = []
    monkeypatch.setattr(_common, "get_separator", lambda *a, device=0, slot=0, **k: ScalingKeepSeparator(device))
    rng = np.random.default_rng(0)
    pcm = (rng.uniform(-0.5, 0.5, size=(44100 * 40, 2)) * 32767).astype(np.int16)
    wav = tmp_path / "one.wav"
    scipy.io.wavfile.write(str(wav), 44100, pcm)
    out = tmp_path / "out"
    out.mkdir()
    separate_dsd.main(["-i", str(wav), "-o", str(out), "-m", "unused.pkl", "--devices", "0,1", "--keep-channels",
                       "--wiener", "2", "--wiener-radius", "1"])
    assert sorted(c[0] for c in calls) == [0, 1] and all(n < len(pcm) for _, n, _, _ in calls)
    assert all(c[2:] == (2, 1) for c in calls)
    for name, g in zip(("vocals", "bass", "drums", "other"), (0.5, 0.25, 0.125, 0.0625)):
        sr, got = scipy.io.wavfile.read(str(out / (name + ".wav")))
        want = (((pcm / 32767.0).astype(np.float32) * np.float32(g)).astype(np.float64) * 32767).astype(np.int16)
        assert sr == 44100 and got.shape == pcm.shape and np.array_equal(got, want)
    # whole-clip covariances cannot be cut: refused with the reason, before anything runs
    calls.clear()
    for extra in (["--wiener", "2"],):
        with pytest.raises(SystemExit) as e:
            separate_dsd.main(["-i", str(wav), "-o", str(out), "-m", "unused.pkl", "--devices", "0,1", "--keep-channels"]
                              + extra)
        assert "--wiener-radius" in str(e.value.code)
    assert calls == []
