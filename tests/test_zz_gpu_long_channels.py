"""30 minutes of 6-channel int16 audio with the Wiener post-filter through dcs_separate_long_channels_host: the
workspace is the formula's bytes for 120 s segments, far below the whole-recording call's, and a segment in the middle
is, byte for byte, its kept part of the batch call on that segment's samples."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import channels_formats_oracle as fo  # noqa: E402
from test_gpu_channels_formats import separator, rounded  # noqa: E402


def test_thirty_minutes_six_channels_with_the_filter():
    rate, nch, seconds = 44100, 6, 30 * 60
    L = seconds * rate
    rng = np.random.default_rng(7)
    # a cheap full-length signal: a few tones and noise per channel, at half scale
    t = np.arange(L, dtype=np.float64) / rate
    rec = np.empty((L, nch), dtype=np.int16)
    for c in range(nch):
        x = 0.2 * np.sin(2 * np.pi * (110 + 37 * c) * t) + 0.1 * np.sin(2 * np.pi * 1234.5 * t + c)
        x += 0.05 * rng.standard_normal(L)
        rec[:, c] = np.round(x * 32767).astype(np.int16)
    del t
    sep = separator("dsd", 2048, seed=70)
    out = sep.separate_long_channels(rec, wiener=2, wiener_radius=2)
    segs = sep.long_segments(L, 2, 2)
    assert len(segs) == 15 and out.shape == (sep.nsrc, L, nch)
    Sw = max(s.model_stop - s.model_start for s in segs)
    Smax = max(s.in_stop - s.in_start for s in segs)
    Kmax = max(s.out_stop - s.out_start for s in segs)
    single = separator("dsd", 2048, seed=70)
    single.separate_channels(torch.zeros((nch, Sw), dtype=torch.float32, device="cuda"), wiener=2, wiener_radius=2)
    want = (single.ctx.workspace_bytes() - rounded(4 * Sw) + rounded(4 * (nch + 1) * Sw) + rounded(4 * 4 * nch * Sw)
            + 2 * rounded(2 * nch * Smax) + 2 * rounded(2 * 4 * nch * Kmax))
    assert sep.ctx.workspace_bytes() == want, (sep.ctx.workspace_bytes(), want)
    sg = segs[7]
    clip = np.ascontiguousarray(rec[sg.in_start:sg.in_stop])
    one = sep.separate_channels_batch([clip], wiener=2, wiener_radius=2)[0]
    assert fo.same_bits(out[:, sg.out_start:sg.out_stop], one[:, sg.out_start - sg.in_start:sg.out_stop - sg.in_start])
    assert np.abs(out[:, sg.out_start:sg.out_stop].astype(np.int64)).sum() > 0
