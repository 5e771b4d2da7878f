"""C-channel int16 clips through the multi-clip scheduler (dcs_separate_batch_pcm16_channels_host,
Separator.separate_pcm16_channels_batch): one launch decodes an interleaved clip into the downmix and C float planes,
the clip is separated as separate_channels(wiener=K, wiener_radius=W), one launch encodes the nsrc x C stem planes as
interleaved int16.

- bit for bit against the encode of the float path, for C in {1, 2, 3, 6, 16}, every FFT dispatch path and both
  patchers;
- C = 1 is the mono int16 batch, C = 2 with the DSD100 net is the keep-channels int16 batch;
- the Wiener post-filter for C in {3, 6, 8};
- batches against one-clip calls (pinned and pageable host buffers), the launch count, the workspace formula of
  include/dcs.h, the refusals before anything is queued.

Clips are at 0.8 of full scale, so that no stem wraps in the int16 encode."""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from oracle import nets, pipeline  # noqa: E402

MB = 1 << 20


def separator(arch="dsd", N=1024, hop=512, seed=5, overlap=25, patcher="standalone", win="hanning"):
    from deepconvsep_b200.engine import Separator
    F = N // 2 + 1
    params = nets.make_synthetic_params(arch, F, seed=seed)
    return Separator(params, arch=arch, frame_size=N, hop=hop, window=win, overlap=overlap, patcher=patcher, feat_size=F)


def pcm_clip(seconds, nch, seed):
    """int16 [L, nch]: different gains and delays of two sources, peak at 0.8 of full scale"""
    a, _ = pipeline.synth_mixture(seconds, seed)
    b, _ = pipeline.synth_mixture(seconds, seed + 1)
    rng = np.random.default_rng(seed)
    cols = []
    for c in range(nch):
        g, h = rng.uniform(-1.0, 1.0, 2)
        cols.append(g * np.roll(a, int(rng.integers(0, 60))) + h * np.roll(b, int(rng.integers(0, 60))))
    x = np.stack(cols, axis=1)
    return np.round(x * (0.8 / np.abs(x).max()) * 32767).astype(np.int16)


def float_route(sep, pcm, wiener=0, wiener_radius=0):
    """the stems the int16 batch must give: separate_channels on pcm / 32767 (fp32), times 32767 in fp32, truncated"""
    x = torch.tensor(np.ascontiguousarray(pcm.T).astype(np.float32) / np.float32(32767), device="cuda")
    stems = sep.separate_channels(x, wiener=wiener, wiener_radius=wiener_radius).cpu().numpy()    # [nsrc * C, L]
    L, nch = pcm.shape
    return (stems * np.float32(32767)).astype(np.int16).reshape(sep.nsrc, nch, L).transpose(0, 2, 1)


def same_bytes(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def rounded(nbytes):
    return (nbytes + MB - 1) // MB * MB


# ---------------------------------------------------------------------------------------------- 1. float path
@pytest.mark.parametrize("arch,N,win,overlap", [("dsd", 1024, "hanning", 25), ("dsd", 2048, "hanning", 25),
                                                ("ikala", 1024, "hanning", 20), ("bach10", 4096, "blackmanharris", 25)])
@pytest.mark.parametrize("patcher", ["standalone", "util"])
def test_bits_of_the_float_path(arch, N, win, overlap, patcher):
    sep = separator(arch, N, win=win, overlap=overlap, patcher=patcher, seed=N + len(arch))
    for k, nch in enumerate((1, 2, 3, 6, 16)):
        pcm = pcm_clip(1.5 + 0.1 * k, nch, 300 + 7 * k + N)
        got = sep.separate_pcm16_channels_batch([pcm])[0]
        want = float_route(sep, pcm)
        assert got.shape == (sep.nsrc, pcm.shape[0], nch) and got.dtype == np.int16
        assert np.abs(want.astype(np.int64)).sum() > 0, nch
        assert same_bytes(got, want), (nch, int(np.sum(got != want)))


# ---------------------------------------------------------------------------------------------- 2. identities
@pytest.mark.parametrize("arch,N,win,overlap", [("dsd", 2048, "hanning", 25), ("ikala", 1024, "hanning", 20),
                                                ("bach10", 4096, "blackmanharris", 25)])
def test_one_channel_is_the_mono_batch(arch, N, win, overlap):
    sep = separator(arch, N, win=win, overlap=overlap, seed=21)
    clips = [pcm_clip(s, 1, 40 + k) for k, s in enumerate((2.2, 1.3, 3.1))]
    got = sep.separate_pcm16_channels_batch(clips)
    want = sep.separate_pcm16_batch([c[:, 0] for c in clips])
    for g, w, c in zip(got, want, clips):
        assert g.shape == (sep.nsrc, c.shape[0], 1) and w.shape == (sep.nsrc, c.shape[0])
        assert np.abs(w.astype(np.int64)).sum() > 0
        assert same_bytes(g[:, :, 0], w)


@pytest.mark.parametrize("N", [1024, 2048])
@pytest.mark.parametrize("wiener,radius", [(0, 0), (2, 0), (2, 1)])
def test_two_channels_are_the_keep_channels_batch(N, wiener, radius):
    sep = separator("dsd", N, seed=23)
    clips = [pcm_clip(s, 2, 60 + k) for k, s in enumerate((4.0, 2.5))]      # 4 s: three chunks of the filter's windows
    got = sep.separate_pcm16_channels_batch(clips, wiener=wiener, wiener_radius=radius)
    want = sep.separate_pcm16_batch(clips, keep_channels=True, wiener=wiener, wiener_radius=radius)
    for g, w in zip(got, want):
        assert np.abs(w.astype(np.int64)).sum() > 0
        assert same_bytes(g, w)


# ---------------------------------------------------------------------------------------------- 3. Wiener post-filter
@pytest.mark.parametrize("nch", [3, 6, 8])
def test_wiener_is_the_encode_of_the_float_path(nch):
    sep = separator("dsd", 1024, seed=25)
    pcm = pcm_clip(4.0, nch, 80 + nch)
    for wiener in (1, 2):
        for radius in (0, 2):
            got = sep.separate_pcm16_channels_batch([pcm], wiener=wiener, wiener_radius=radius)[0]
            want = float_route(sep, pcm, wiener, radius)
            assert np.abs(want.astype(np.int64)).sum() > 0
            assert same_bytes(got, want), (nch, wiener, radius, int(np.sum(got != want)))
    # the filter changes the stems
    assert not same_bytes(got, float_route(sep, pcm))


# ---------------------------------------------------------------------------------------------- 4. batches
@pytest.mark.parametrize("pinned", [True, False])
def test_batch_is_one_clip_calls(pinned):
    sep = separator("dsd", 2048, seed=27)
    nch = 6
    # not longest first: both staging buffers are reused by a longer clip than the one before
    clips = [pcm_clip(s, nch, 90 + k) for k, s in enumerate((2.0, 3.5, 1.2, 2.7))]
    if pinned:
        pin = [torch.empty(c.shape, dtype=torch.int16, pin_memory=True).numpy() for c in clips]
        for p_, c in zip(pin, clips):
            p_[...] = c
        clips = pin
        outs = [torch.empty((sep.nsrc, c.shape[0], nch), dtype=torch.int16, pin_memory=True).numpy() for c in clips]
    else:
        outs = None
    got = sep.separate_pcm16_channels_batch(clips, outs=outs)
    if outs is not None:
        assert all(g is o for g, o in zip(got, outs))
    for g, c in zip(got, clips):
        one = sep.separate_pcm16_channels_batch([np.array(c)])[0]
        assert np.abs(one.astype(np.int64)).sum() > 0
        assert same_bytes(g, one)
    assert same_bytes(got[1], float_route(sep, np.array(clips[1])))


def test_launch_count_is_the_float_call_plus_one():
    """the decode forms the downmix in place of separate_channels' downmix launch, and the encode is one launch more"""
    sep = separator("dsd", 1024, seed=29)
    for nch, wiener in ((6, 0), (3, 2)):
        pcm = pcm_clip(2.0, nch, 100 + nch)
        x = torch.tensor(np.ascontiguousarray(pcm.T).astype(np.float32) / np.float32(32767), device="cuda")
        n0 = sep.ctx.launch_count()
        sep.separate_channels(x, wiener=wiener)
        n1 = sep.ctx.launch_count()
        sep.separate_pcm16_channels_batch([pcm, pcm], wiener=wiener)
        n2 = sep.ctx.launch_count()
        assert n2 - n1 == 2 * (n1 - n0 + 1), (nch, wiener, n1 - n0, n2 - n1)


# ---------------------------------------------------------------------------------------------- 5. workspace
@pytest.mark.parametrize("nch,wiener,radius", [(6, 0, 0), (8, 2, 2)])
def test_workspace_formula(nch, wiener, radius):
    clips = [pcm_clip(s, nch, 110 + k) for k, s in enumerate((1.7, 3.3, 2.1))]
    Lmax = max(c.shape[0] for c in clips)
    batch = separator("dsd", 2048, seed=31)                  # a fresh context each
    batch.separate_pcm16_channels_batch(clips, wiener=wiener, wiener_radius=radius)
    single = separator("dsd", 2048, seed=31)
    longest = next(c for c in clips if c.shape[0] == Lmax)
    single.separate_channels(np.ascontiguousarray(longest).astype(np.float32) / np.float32(32767), wiener=wiener,
                             wiener_radius=radius)
    nsrc, n = batch.nsrc, min(len(clips), 2)
    want = (single.ctx.workspace_bytes() - rounded(4 * Lmax) + rounded(4 * (nch + 1) * Lmax) + rounded(4 * nsrc * nch * Lmax)
            + n * rounded(2 * nch * Lmax) + n * rounded(2 * nsrc * nch * Lmax))
    assert batch.ctx.workspace_bytes() == want, (batch.ctx.workspace_bytes(), want)


# ---------------------------------------------------------------------------------------------- 6. refusals
def test_refusals_queue_nothing():
    from deepconvsep_b200 import _lib
    from deepconvsep_b200.engine import Model, _ptr
    sep = separator("dsd", 1024, seed=33)
    ctx, lib = sep.ctx, sep.lib
    nch = 3
    clips = [pcm_clip(1.0, nch, 120), pcm_clip(0.7, nch, 121)]
    ref = sep.separate_pcm16_channels_batch(clips)
    others = {a: Model(ctx, nets.make_synthetic_params(a, F, seed=3), arch=a, feat_size=F)
              for a, F in (("dsd_ild", 513), ("bach10_score", 129))}
    Ls = np.array([c.shape[0] for c in clips], dtype=np.int64)
    outs = [np.empty((4, c.shape[0], nch), dtype=np.int16) for c in clips]

    def call(model=None, channels=nch, iterations=0, radius=0, pin=None, lens=None, strides=None):
        pin = pin or [c.ctypes.data for c in clips]
        lens = Ls if lens is None else lens
        strides = Ls if strides is None else strides
        return lib.dcs_separate_batch_pcm16_channels_host(
            ctx.handle, (model or sep.model).handle, sep.stft.handle, 2, (C.c_void_p * 2)(*pin), lens.ctypes.data, channels,
            iterations, radius, C.c_float(0.3), 25, 0, (C.c_void_p * 2)(*[o.ctypes.data for o in outs]), strides.ctypes.data,
            None)

    short = Ls.copy()
    short[1] -= 1
    zero = Ls.copy()
    zero[1] = 0
    refused = {
        "channels 0": (lambda: call(channels=0), "channels 0"),
        "channels 17": (lambda: call(channels=17), "channels 17"),
        "iterations -1": (lambda: call(iterations=-1), "iterations -1"),
        "radius -1": (lambda: call(radius=-1), "radius -1"),
        "filter on 1 channel": (lambda: call(channels=1, iterations=1), "Wiener"),
        "filter on 9 channels": (lambda: call(channels=9, iterations=1), "Wiener"),
        "clip 1 NULL": (lambda: call(pin=[clips[0].ctypes.data, None]), "clip 1"),
        "clip 1 length 0": (lambda: call(lens=zero), "clip 1"),
        "clip 1 stride < length": (lambda: call(strides=short), "clip 1"),
        "overlap = time_context": (lambda: lib.dcs_separate_batch_pcm16_channels_host(
            ctx.handle, sep.model.handle, sep.stft.handle, 1, (C.c_void_p * 1)(clips[0].ctypes.data), Ls.ctypes.data, nch,
            0, 0, C.c_float(0.3), sep.model.tc, 0, (C.c_void_p * 1)(outs[0].ctypes.data), Ls.ctypes.data, None), "overlap"),
    }
    for a, m in others.items():
        refused["architecture " + a] = (lambda m=m: call(model=m), "dcs_separate_masks")
    tap = torch.zeros((4 * nch, sep.stft.num_frames(int(Ls.max())), sep.stft.ldf), dtype=torch.complex64, device="cuda")

    def tapped():
        _lib.check(lib.dcs_set_spectrum_tap(ctx.handle, _ptr(tap), tap.numel()))
        try:
            return call()
        finally:
            _lib.check(lib.dcs_set_spectrum_tap(ctx.handle, None, 0))
    refused["spectrum tap without the filter"] = (tapped, "spectrum tap")
    for name, (fn, msg) in refused.items():
        torch.cuda.synchronize()
        n0 = ctx.launch_count()
        with pytest.raises(_lib.DcsError) as e:
            _lib.check(fn())
        assert ctx.launch_count() == n0, name
        assert msg in str(e.value), (name, str(e.value))
    # the filter's settings on the ctx are not read
    sep.ctx.set_wiener(2)
    got = sep.separate_pcm16_channels_batch(clips)
    sep.ctx.set_wiener(0)
    for g, r in zip(got, ref):
        assert same_bytes(g, r)
