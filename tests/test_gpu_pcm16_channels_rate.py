"""C-channel int16 clips at 8-192 kHz through the multi-clip scheduler (dcs_separate_batch_pcm16_channels_resampled_host,
Separator.separate_pcm16_channels_batch(sample_rate=fs)): one launch resamples and decodes a clip into the downmix and C
float planes at 44.1 kHz, the clip is separated as separate_channels(wiener=K, wiener_radius=W), one launch resamples the
nsrc x C stem planes back and encodes them as interleaved int16.

- bit for bit against the encode of the float route at the rate (separate_channels(pcm / 32767, sample_rate=fs)), for
  every rate class of the resampler, C in {1, 2, 6, 16}, the DSD network at N = 1024 and 2048 and the iKala network,
  both patchers, and clips of 1, 7, fewer than the filter's taps and tile-boundary +-1 samples;
- the Wiener post-filter for C in {2, 6, 8} at 48 kHz;
- batches against one-clip calls (pinned and pageable), 44.1 kHz as the call without the keyword, the launch count, the
  workspace formula of include/dcs.h, the refusals before anything is queued.

Clips are at 0.8 of full scale, so that no stem wraps in the int16 encode."""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from oracle import nets, pipeline  # noqa: E402

MB = 1 << 20
RS_THREADS, RS_V, RS_SMEM_MAX = 512, 4, 227 * 1024       # resample.cu's tile rule, for the tile-boundary lengths
RATES = [8000, 22050, 32000, 48000, 64000, 96000, 192000]


def separator(arch="dsd", N=1024, hop=512, seed=5, overlap=25, patcher="standalone"):
    from deepconvsep_b200.engine import Separator
    F = N // 2 + 1
    params = nets.make_synthetic_params(arch, F, seed=seed)
    return Separator(params, arch=arch, frame_size=N, hop=hop, window="hanning", overlap=overlap, patcher=patcher,
                     feat_size=F)


def pcm_clip(L, nch, seed):
    """int16 [L, nch]: different gains and delays of two sources, peak at 0.8 of full scale"""
    n = max(L, 4410) + 64
    a, _ = pipeline.synth_mixture(n / 44100.0, seed)
    b, _ = pipeline.synth_mixture(n / 44100.0, seed + 1)
    rng = np.random.default_rng(seed)
    cols = []
    for c in range(nch):
        g, h = rng.uniform(-1.0, 1.0, 2)
        cols.append(g * np.roll(a, int(rng.integers(0, 60))) + h * np.roll(b, int(rng.integers(0, 60))))
    x = np.stack(cols, axis=1)[:L]
    return np.round(x * (0.8 / max(np.abs(x).max(), 1e-9)) * 32767).astype(np.int16)


def float_route(sep, pcm, rate, wiener=0, wiener_radius=0):
    """the stems the int16 batch must give: separate_channels at the rate on pcm / 32767 (fp32), times 32767 in fp32,
    truncated"""
    x = torch.tensor(np.ascontiguousarray(pcm.T).astype(np.float32) / np.float32(32767), device="cuda")
    stems = sep.separate_channels(x, wiener=wiener, wiener_radius=wiener_radius, sample_rate=rate).cpu().numpy()
    L, nch = pcm.shape
    return (stems * np.float32(32767)).astype(np.int16).reshape(sep.nsrc, nch, L).transpose(0, 2, 1)


def same_bytes(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def rounded(nbytes):
    return (nbytes + MB - 1) // MB * MB


def _bank(up, down):
    ntaps = 20 * max(up, down) + 1
    Q = -(-ntaps // up)
    half = (ntaps - 1) // 2
    cspan = ((up - 1) * down + half) // up - half // up
    return ntaps, Q, cspan, Q * up * 8


def _periods_per_tile(up, down, nch, encode):
    """resample.cu's periods per tile of the fused kernels (the channels of one encode tile: all of them at these rates)"""
    _, Q, cspan, bank = _bank(up, down)
    tp = max(1, 4 * RS_THREADS // (up * (nch if encode else 1))) * RS_V
    cs = (nch | 1) if encode else nch
    while tp > RS_V and bank + ((tp - 1) * down + cspan + Q) * cs * (4 if encode else 2) > RS_SMEM_MAX:
        tp -= RS_V
    return tp


def edge_lengths(rate, nch):
    """1, 7, fewer than the filter's taps, and +-1 around the first tile boundary of the decode (at 44.1 kHz) and of
    the encode (at the rate)"""
    from deepconvsep_b200.engine import resample_ratio
    up, down = resample_ratio(rate, 44100)
    ntaps = _bank(up, down)[0]
    out_tile = _periods_per_tile(up, down, nch, False) * up                 # outputs of one decode tile
    first = -(-out_tile * down // up)                                         # the shortest clip with L' >= out_tile
    enc_tile = _periods_per_tile(down, up, nch, True) * down                  # outputs of one encode tile
    Ls = {1, 7, ntaps // 2, first - 1, first, first + 1, enc_tile - 1, enc_tile, enc_tile + 1}
    return sorted(L for L in Ls if L >= 1)


# ---------------------------------------------------------------------------------------------- 1. float route
NETS = [("dsd", 1024, 25), ("dsd", 2048, 25), ("ikala", 1024, 20)]


@pytest.mark.parametrize("rate", RATES)
@pytest.mark.parametrize("net", range(len(NETS)), ids=["dsd1024", "dsd2048", "ikala"])
def test_bits_of_the_float_route(rate, net):
    arch, N, overlap = NETS[net]
    patcher = ("standalone", "util")[(RATES.index(rate) + net) % 2]
    sep = separator(arch, N, overlap=overlap, patcher=patcher, seed=N + len(arch) + rate % 97)
    for k, nch in enumerate((1, 2, 6, 16)):
        lengths = [int(0.6 * rate) + 13 * k] + edge_lengths(rate, nch)
        clips = [pcm_clip(L, nch, 300 + 7 * k + i + rate % 1009) for i, L in enumerate(lengths)]
        got = sep.separate_pcm16_channels_batch(clips, sample_rate=rate)
        nonzero = 0
        for g, c in zip(got, clips):
            want = float_route(sep, c, rate)
            assert g.shape == (sep.nsrc, c.shape[0], nch) and g.dtype == np.int16
            assert same_bytes(g, want), (nch, c.shape[0], int(np.sum(g != want)))
            nonzero += int(np.abs(want.astype(np.int64)).sum() > 0)
        assert np.abs(got[0].astype(np.int64)).sum() > 0 and nonzero >= 1, nch


# ---------------------------------------------------------------------------------------------- 2. Wiener post-filter
@pytest.mark.parametrize("nch", [2, 6, 8])
def test_wiener_is_the_encode_of_the_float_route(nch):
    sep = separator("dsd", 1024, seed=25)
    pcm = pcm_clip(4 * 48000, nch, 80 + nch)           # 4 s: three chunks of the filter's windows
    plain = sep.separate_pcm16_channels_batch([pcm], sample_rate=48000)[0]
    for wiener in (1, 2):
        for radius in (0, 2):
            got = sep.separate_pcm16_channels_batch([pcm], wiener=wiener, wiener_radius=radius, sample_rate=48000)[0]
            want = float_route(sep, pcm, 48000, wiener, radius)
            assert np.abs(want.astype(np.int64)).sum() > 0
            assert same_bytes(got, want), (nch, wiener, radius, int(np.sum(got != want)))
            assert not same_bytes(got, plain), (nch, wiener, radius)


# ---------------------------------------------------------------------------------------------- 3. batches
@pytest.mark.parametrize("pinned", [True, False])
def test_batch_is_one_clip_calls(pinned):
    sep = separator("dsd", 2048, seed=27)
    nch, rate = 6, 48000
    # not longest first: both staging buffers are reused by a longer clip than the one before
    clips = [pcm_clip(int(s * rate), nch, 90 + k) for k, s in enumerate((2.0, 3.5, 1.2, 2.7))]
    if pinned:
        pin = [torch.empty(c.shape, dtype=torch.int16, pin_memory=True).numpy() for c in clips]
        for p_, c in zip(pin, clips):
            p_[...] = c
        clips = pin
        outs = [torch.empty((sep.nsrc, c.shape[0], nch), dtype=torch.int16, pin_memory=True).numpy() for c in clips]
    else:
        outs = None
    got = sep.separate_pcm16_channels_batch(clips, outs=outs, sample_rate=rate)
    if outs is not None:
        assert all(g is o for g, o in zip(got, outs))
    for g, c in zip(got, clips):
        one = sep.separate_pcm16_channels_batch([np.array(c)], sample_rate=rate)[0]
        assert np.abs(one.astype(np.int64)).sum() > 0
        assert same_bytes(g, one)
    assert same_bytes(got[1], float_route(sep, np.array(clips[1]), rate))


def test_model_rate_keyword_changes_nothing():
    sep = separator("dsd", 1024, seed=28)
    clips = [pcm_clip(n, 6, 95 + n % 7) for n in (70000, 40000)]
    n0 = sep.ctx.launch_count()
    plain = sep.separate_pcm16_channels_batch(clips)
    n1 = sep.ctx.launch_count()
    keyed = sep.separate_pcm16_channels_batch(clips, sample_rate=44100)
    n2 = sep.ctx.launch_count()
    assert n2 - n1 == n1 - n0
    assert sep._resamplers == {}
    for a, b in zip(plain, keyed):
        assert np.abs(a.astype(np.int64)).sum() > 0 and same_bytes(a, b)


# ---------------------------------------------------------------------------------------------- 4. launches, workspace
@pytest.mark.parametrize("rate", [48000, 96000])
def test_launch_count(rate):
    """per clip: separate_channels at L' plus one, one fewer than the float route at the rate"""
    sep = separator("dsd", 1024, seed=29)
    for nch, wiener in ((6, 0), (3, 2)):
        pcm = pcm_clip(2 * rate, nch, 100 + nch)
        sep.separate_pcm16_channels_batch([pcm], wiener=wiener, sample_rate=rate)     # resamplers made
        Lm = sep.resampler(rate, 44100).length(pcm.shape[0])
        x44 = torch.zeros((nch, Lm), dtype=torch.float32, device="cuda")
        x = torch.tensor(np.ascontiguousarray(pcm.T).astype(np.float32) / np.float32(32767), device="cuda")
        n0 = sep.ctx.launch_count()
        sep.separate_channels(x44, wiener=wiener)
        n1 = sep.ctx.launch_count()
        sep.separate_channels(x, wiener=wiener, sample_rate=rate)
        n2 = sep.ctx.launch_count()
        sep.separate_pcm16_channels_batch([pcm, pcm], wiener=wiener, sample_rate=rate)
        n3 = sep.ctx.launch_count()
        assert n3 - n2 == 2 * (n1 - n0 + 1) == 2 * (n2 - n1 - 1), (nch, wiener, n1 - n0, n2 - n1, n3 - n2)


@pytest.mark.parametrize("rate,nch,wiener,radius", [(48000, 6, 0, 0), (96000, 8, 2, 2), (48000, 8, 2, 2)])
def test_workspace_formula(rate, nch, wiener, radius):
    clips = [pcm_clip(int(s * rate), nch, 110 + k) for k, s in enumerate((1.7, 3.3, 2.1))]
    Lmax = max(c.shape[0] for c in clips)
    batch = separator("dsd", 2048, seed=31)                  # a fresh context each
    batch.separate_pcm16_channels_batch(clips, wiener=wiener, wiener_radius=radius, sample_rate=rate)
    Lm = batch.resampler(rate, 44100).length(Lmax)
    single = separator("dsd", 2048, seed=31)
    single.separate_channels(torch.zeros((nch, Lm), dtype=torch.float32, device="cuda"), wiener=wiener,
                             wiener_radius=radius)
    nsrc, n = batch.nsrc, min(len(clips), 2)
    want = (single.ctx.workspace_bytes() - rounded(4 * Lm) + rounded(4 * (nch + 1) * Lm) + rounded(4 * nsrc * nch * Lm)
            + n * rounded(2 * nch * Lmax) + n * rounded(2 * nsrc * nch * Lmax))
    assert batch.ctx.workspace_bytes() == want, (batch.ctx.workspace_bytes(), want)


# ---------------------------------------------------------------------------------------------- 5. refusals
def test_refusals_queue_nothing():
    from deepconvsep_b200 import _lib
    from deepconvsep_b200.engine import Model
    sep = separator("dsd", 1024, seed=33)
    ctx, lib = sep.ctx, sep.lib
    rate, nch = 48000, 3
    clips = [pcm_clip(48000, nch, 120), pcm_clip(33600, nch, 121)]
    to, back = sep.resampler(rate, 44100), sep.resampler(44100, rate)
    to96 = sep.resampler(96000, 44100)
    other = separator("dsd", 1024, seed=34)
    foreign = other.resampler(44100, rate)
    models = {a: Model(ctx, nets.make_synthetic_params(a, F, seed=3), arch=a, feat_size=F)
              for a, F in (("dsd_ild", 513), ("bach10_score", 129))}
    Ls = np.array([c.shape[0] for c in clips], dtype=np.int64)
    outs = [np.empty((4, c.shape[0], 16), dtype=np.int16) for c in clips]
    wide = [pcm_clip(int(L), 17, 122) for L in Ls]

    def call(model=None, pair=(to, back), channels=nch, iterations=0, lens=None, pcm=None):
        lens = Ls if lens is None else lens
        pcm = pcm or clips
        h = [None if r is None else r.handle for r in pair]
        return lib.dcs_separate_batch_pcm16_channels_resampled_host(
            ctx.handle, (model or sep.model).handle, sep.stft.handle, h[0], h[1], 2,
            (C.c_void_p * 2)(*[c.ctypes.data for c in pcm]), lens.ctypes.data, channels, iterations, 0, C.c_float(0.3),
            25, 0, (C.c_void_p * 2)(*[o.ctypes.data for o in outs]), lens.ctypes.data, None)

    zero = Ls.copy()
    zero[1] = 0
    refused = {
        "NULL to_model": (lambda: call(pair=(None, back)), "NULL resampler"),
        "NULL from_model": (lambda: call(pair=(to, None)), "NULL resampler"),
        "not inverse": (lambda: call(pair=(to96, back)), "not inverse"),
        "same direction twice": (lambda: call(pair=(to, to)), "not inverse"),
        "another ctx": (lambda: call(pair=(to, foreign)), "another ctx"),
        "channels 17": (lambda: call(channels=17, pcm=wide), "channels 17"),
        "filter on 9 channels": (lambda: call(channels=9, iterations=1, pcm=wide), "Wiener"),
        "clip 1 length 0": (lambda: call(lens=zero), "clip 1"),
    }
    for a, m in models.items():
        refused["architecture " + a] = (lambda m=m: call(model=m), "dcs_separate_masks")
    for name, (fn, msg) in refused.items():
        torch.cuda.synchronize()
        n0 = ctx.launch_count()
        with pytest.raises(_lib.DcsError) as e:
            _lib.check(fn())
        assert ctx.launch_count() == n0, name
        assert msg in str(e.value), (name, str(e.value))
    n0 = ctx.launch_count()
    with pytest.raises(ValueError, match="44099"):
        sep.separate_pcm16_channels_batch(clips, sample_rate=44099)
    with pytest.raises(ValueError, match="channel count"):
        sep.separate_pcm16_channels_batch([clips[0], wide[1]], sample_rate=rate)
    assert ctx.launch_count() == n0 and (44099, 44100) not in sep._resamplers
    got = sep.separate_pcm16_channels_batch(clips, sample_rate=rate)
    for g, c in zip(got, clips):
        want = float_route(sep, c, rate)
        assert np.abs(want.astype(np.int64)).sum() > 0 and same_bytes(g, want)
