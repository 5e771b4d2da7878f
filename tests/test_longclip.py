"""One recording cut into segments, separated independently and stitched (deepconvsep_b200.longclip):
the planner's margins are exact -- with the float64 oracle as the engine the stitched stems ARE the
whole-clip stems -- for both patchers, overlaps 25 and 20, N/hop = 2 and 8, and over two gloo ranks."""
import os
import socket
import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

from deepconvsep_b200 import longclip
from oracle import nets, pipeline, dsp


def _engine(params, arch, N, H, overlap, patcher, window=np.hanning):
    def fn(sub, filt):
        return pipeline.separate(np.asarray(sub, dtype=np.float64), params, arch, frameSize=N, hopSize=H, window=window,
                                 overlap=overlap, patcher=patcher)
    return fn


def test_plan_covers_the_clip_once_and_respects_the_grids():
    for (N, H, tc, ov) in ((1024, 512, 30, 25), (2048, 512, 30, 25), (4096, 512, 30, 25), (1024, 512, 30, 20), (2048, 256, 30, 25)):
        for L in (0, 1, 5000, 44100 * 7 + 13, 44100 * 60):
            for parts in (1, 2, 3, 8):
                segs = longclip.plan_segments(L, parts, N, H, tc, ov)
                if L == 0:
                    assert segs == []
                    continue
                assert segs[0].in_start == 0 and segs[0].out_start == 0
                assert segs[-1].in_stop == L and segs[-1].out_stop == L
                for a, b in zip(segs, segs[1:]):
                    assert a.out_stop == b.out_start
                for s in segs:
                    assert s.in_start <= s.out_start < s.out_stop <= s.in_stop
                    assert s.in_start == s.frame0 * H and s.frame0 % (tc - ov) == 0
                    assert s.in_stop == L or (s.in_stop - s.in_start) % H == 0
    # a clip too short for its margins stays in one piece
    assert len(longclip.plan_segments(44100, 8, 1024, 512, 30, 25)) == 1


@pytest.mark.parametrize("arch,N,H,overlap,patcher,seconds,parts", [
    ("dsd", 1024, 512, 25, "standalone", 5.0, 3),
    ("dsd", 1024, 512, 25, "util", 4.0, 2),
    ("dsd", 2048, 256, 25, "standalone", 4.0, 2),          # N / (2 hop) = 4 padded frames at either end
    ("ikala", 1024, 512, 20, "standalone", 4.5, 3),        # step 10, max-pool routing
])
def test_stitched_equals_whole_with_the_oracle_as_engine(arch, N, H, overlap, patcher, seconds, parts):
    F = N // 2 + 1
    params = nets.make_synthetic_params(arch, F, seed=3)
    mix, _ = pipeline.synth_mixture(seconds, 5)
    mix = mix[:len(mix) - 77]                              # a length off every grid
    fn = _engine(params, arch, N, H, overlap, patcher)
    whole = fn(mix, None)
    segs = longclip.plan_segments(len(mix), parts, N, H, 30, overlap)
    assert len(segs) == parts
    got = longclip.separate_long([fn] * 2, mix, parts=parts, geometry=(N, H, 30, overlap))
    assert got.shape == whole.shape
    scale = np.abs(whole).max()
    assert np.abs(got - whole).max() <= 1e-13 * scale, np.abs(got - whole).max() / scale


def test_margins_are_tight_enough_to_matter():
    """One patch step less on the left, four hops less on the right, and the stitched result differs: the test above
    is not vacuous (the right bound has two hops of slack: the newest patch enters a frame at offset 0 with weight 0)."""
    N, H, tc, ov = 1024, 512, 30, 25
    params = nets.make_synthetic_params("dsd", 513, seed=3)
    mix, _ = pipeline.synth_mixture(5.0, 5)
    fn = _engine(params, "dsd", N, H, ov, "standalone")
    whole = fn(mix, None)
    segs = longclip.plan_segments(len(mix), 2, N, H, tc, ov)
    a, b = segs
    step = tc - ov
    bad_left = [a, b._replace(in_start=b.in_start + step * H, frame0=b.frame0 + step)]
    bad_right = [a._replace(in_stop=a.in_stop - 4 * H), b]
    for bad in (bad_left, bad_right):
        pieces = [fn(mix[s.in_start:s.in_stop], None) for s in bad]
        got = longclip.stitch(bad, pieces, len(mix), dtype=np.float64)
        assert np.abs(got - whole).max() > 1e-9 * np.abs(whole).max()


def test_score_filters_travel_with_their_frames():
    N, H, tc, ov = 1024, 512, 30, 25
    L = 44100 * 4 + 5
    T = int(np.ceil(L / float(H))) + 2
    filt = np.arange(4 * T * 3, dtype=np.float32).reshape(4, T, 3)
    seen = []

    def fn(sub, f):
        Ts = int(np.ceil(len(sub) / float(H))) + 2
        assert f.shape == (4, Ts, 3)
        seen.append(f[0, 0, 0])
        return np.zeros((4, len(sub)), dtype=np.float32)
    longclip.separate_long(fn, np.zeros(L), parts=2, filters=filt, geometry=(N, H, tc, ov))
    segs = longclip.plan_segments(L, 2, N, H, tc, ov)
    assert seen == [filt[0, s.frame0, 0] for s in segs]


def _worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    N, H, tc, ov = 1024, 512, 30, 25
    params = nets.make_synthetic_params("dsd", 513, seed=3)
    mix, _ = pipeline.synth_mixture(4.0, 5)
    fn = _engine(params, "dsd", N, H, ov, "standalone")
    out = longclip.separate_long_distributed(fn, mix, geometry=(N, H, tc, ov))
    dist.barrier()
    if rank == 0:
        whole = fn(mix, None)
        q.put(float(np.abs(out - whole).max() / np.abs(whole).max()))
    else:
        assert out is None
    dist.destroy_process_group()


def test_two_rank_gloo_long_clip():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    err = q.get(timeout=300)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert err <= 1e-13


def test_cli_splits_one_recording_over_the_listed_devices(tmp_path, monkeypatch):
    """`separate_dsd.py -i one.wav --devices 0,1`: the recording (not a file list) is cut over the devices; with a
    stand-in for the CUDA Separator that scales its input per source, the wavs are those of a whole-clip call."""
    import scipy.io.wavfile
    from types import SimpleNamespace
    from deepconvsep_b200.examples import _common
    from deepconvsep_b200.examples.dsd100 import separate_dsd

    calls = []

    class FakeSeparator(object):
        def __init__(self, device):
            self.device = device
            self.model = SimpleNamespace(arch="dsd", tc=30)
            self.frame_size, self.hop, self.overlap = 1024, 512, 25
            self.sources = ["vocals", "bass", "drums", "other"]

        def separate(self, sub):
            calls.append((self.device, len(sub)))
            return np.stack([np.asarray(sub, dtype=np.float32) * g for g in (0.5, 0.25, 0.125, 0.0625)])

    monkeypatch.setattr(_common, "get_separator", lambda *a, device=0, slot=0, **k: FakeSeparator(device))
    rng = np.random.default_rng(0)
    pcm = (rng.uniform(-0.5, 0.5, size=(44100 * 6, 2)) * 32767).astype(np.int16)
    wav = tmp_path / "one.wav"
    scipy.io.wavfile.write(str(wav), 44100, pcm)
    out = tmp_path / "out"
    out.mkdir()
    separate_dsd.main(["-i", str(wav), "-o", str(out), "-m", "unused.pkl", "--devices", "0,1"])
    assert sorted(d for d, _ in calls) == [0, 1] and all(n < len(pcm) for _, n in calls)
    mono = (pcm[:, 0] / 32767.0 + pcm[:, 1] / 32767.0) / 2
    for name, g in zip(("vocals", "bass", "drums", "other"), (0.5, 0.25, 0.125, 0.0625)):
        sr, got = scipy.io.wavfile.read(str(out / (name + ".wav")))
        want = ((mono.astype(np.float32) * np.float32(g)).astype(np.float64) * 32767).astype(np.int16)
        assert sr == 44100 and np.array_equal(got, want)


def test_the_1x1_score_net_is_refused_before_any_segment_runs():
    """long clips are not built for the score-informed build_ca_1x1 network: with either kind of score, on one host or
    over ranks, a separator of that network is refused before any segment is separated"""
    from types import SimpleNamespace
    picked = []

    class FakeSeparator(object):
        def __init__(self):
            self.model = SimpleNamespace(arch="bach10_score_1x1", tc=30)
            self.frame_size, self.hop, self.overlap = 4096, 512, 25

        def separate_score(self, sub, filters):
            picked.append("score")
            return np.zeros((4, len(sub)), dtype=np.float32)

        def separate_notes(self, sub, melody, frame0=0):
            picked.append("notes")
            return np.zeros((4, len(sub)), dtype=np.float32)

    L = 44100 * 20
    T = -(-L // 512) + 2
    for score in ({"filters": np.zeros((4, T, 2049), dtype=np.float32)}, {"melody": np.zeros((4, 1, 43))}):
        with pytest.raises(ValueError, match="build_ca_1x1"):
            longclip.separate_long([FakeSeparator(), FakeSeparator()], np.zeros(L), parts=2, **score)
        with pytest.raises(ValueError, match="build_ca_1x1"):
            longclip.separate_long_distributed(FakeSeparator(), np.zeros(L), **score)
    assert picked == []


def _toy_engine(N, H, tc, ov, patcher):
    """The pipeline's time structure with a toy network: every output frame of a patch depends on ALL frames of the
    patch (so one contaminated frame spoils the whole patch), two sources, the real patchers / cross-fade / STFTs."""
    from oracle import patch
    gen = patch.generate_overlapadd if patcher == "standalone" else patch.generate_overlapadd_util

    def fn(sub, filt):
        sub = np.asarray(sub, dtype=np.float64)
        mag, ph = dsp.compute_file(sub, phase=True, frameSize=N, hopSize=H, window=np.hanning)
        batches, n = gen(mag, input_size=mag.shape[-1], time_context=tc, overlap=ov, batch_size=4)
        if n == 0:
            mm = np.zeros((2, len(ph), mag.shape[-1]))
        else:
            g = 1.0 / (1.0 + np.exp(-20.0 * batches.mean(axis=(2, 3, 4), keepdims=True)))      # one number per patch
            out = np.stack([batches * g, batches * (1.0 - g)], axis=1)                        # [nb, 2, B, 1, tc, F]
            mm = patch.overlapadd_multi(out, batches, n, overlap=ov)
        stems = []
        for s in range(2):
            m = mm[s, :len(ph)]
            if m.shape[0] < len(ph):
                m = np.concatenate([m, np.zeros((len(ph) - m.shape[0], m.shape[1]))])
            stems.append(dsp.compute_inverse(m, ph, frameSize=N, hopSize=H, window=np.hanning)[:len(sub)])
        return np.stack(stems)
    return fn


def test_margins_are_exact_for_many_geometries():
    """frame sizes / hops / contexts / overlaps the reference never uses (N/2 not a multiple of the hop, step 1,
    step = time_context - 1, overlap 1 ...), both patchers, clip lengths on and off the grids"""
    rng = np.random.default_rng(7)
    cases = 0
    for N, H in ((64, 16), (64, 32), (96, 20), (128, 8), (32, 32)):
        for tc, ov in ((6, 4), (6, 5), (5, 1), (8, 3), (30, 25)):
            for patcher in ("standalone", "util"):
                left, right = longclip.margins(N, H, tc, ov)
                L = int(3.2 * 2 * (left + right)) + int(rng.integers(0, 3 * H))
                x = rng.standard_normal(L) * np.hanning(L) + 0.1 * np.sin(np.arange(L) * 0.05)
                fn = _toy_engine(N, H, tc, ov, patcher)
                whole = fn(x, None)
                segs = longclip.plan_segments(L, 3, N, H, tc, ov)
                assert len(segs) == 3, (N, H, tc, ov, L)
                got = longclip.separate_long(fn, x, parts=3, geometry=(N, H, tc, ov))
                err = np.abs(got - whole).max() / np.abs(whole).max()
                assert err <= 1e-12, (N, H, tc, ov, patcher, err)
                cases += 1
    assert cases == 50
