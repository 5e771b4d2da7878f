"""Float64 oracle of C-channel stems from a single-channel network (TEST INFRASTRUCTURE: built on oracle/).

The network sees the downmix (((a_0 + a_1) + a_2) + ...) / C exactly as `oracle.pipeline.separate` runs it (float32
scaled magnitude, the patcher, batches of 32, the soft-mask rule); its per-patch soft masks are applied to the patches
of each channel's scaled magnitude, cross-faded with `overlapadd_multi`, and inverted with that channel's phase.  That
is M~_s * X_c per (source, channel), M~_s = overlapadd_multi of the per-patch masks, formed without dividing anything by
the downmix's magnitude (which vanishes where the channels are in anti-phase).  At C = 2 with the DSD100 network this is
the keep-channels mode.  The blended masks and the kink map are those of tests/masks_oracle.separate_masks on the
downmix."""
import numpy as np

from oracle import dsp, patch, nets
import masks_oracle as mo


def downmix(audio):
    """float64 [L, C] -> the mean of the channels, summed in channel order"""
    audio = np.asarray(audio, dtype=np.float64)
    mono = audio[:, 0].copy()
    for c in range(1, audio.shape[1]):
        mono = mono + audio[:, c]
    return mono / audio.shape[1]


def separate_channels(audio, params, arch="dsd", frameSize=1024, hopSize=512, window=np.hanning, scale_factor=0.3,
                      time_context=30, overlap=25, batch_size=32, patcher="standalone"):
    """audio float [L, C] -> (stems float64 [L, nsrc, C], mags [C] of [T, F] (scaled float32 magnitude per channel),
    phs [C] of [T, F], mms [C] of [nsrc, T, F] (the blended masks times the channel's scaled magnitude, formed patch by
    patch), masks float64 [nsrc, T, F], kink map bool [T, F] of the downmix)."""
    a = nets.ARCHS[arch]
    nsrc = a["nsrc"]
    audio = np.asarray(audio, dtype=np.float64)
    assert audio.ndim == 2, audio.shape
    L, C = audio.shape
    kw = dict(frameSize=frameSize, hopSize=hopSize, window=window)
    gen = patch.generate_overlapadd if patcher == "standalone" else patch.generate_overlapadd_util

    def scaled(x):
        m, p = dsp.compute_file(x, phase=True, **kw)
        return scale_factor * m.astype(np.float32), p

    mono = downmix(audio)
    mag, _ = scaled(mono)
    T, F = mag.shape
    batches, nchunks = gen(mag, input_size=F, time_context=time_context, overlap=overlap, batch_size=batch_size)
    pres = [nets.predict(params, b, arch, return_pre=True) for b in batches]
    ms = [nets.soft_masks(nets.relu(p), a["mask"], nsrc) for p in pres]
    masks = mo._blend([[m[:, i:i + 1] for i in range(nsrc)] for m in ms], batches, nchunks, overlap, T, F, nsrc)
    kmap = mo._kink_map(pres, a["mask"], nsrc, nchunks, batch_size, time_context - overlap, time_context, T, F)
    stems = np.zeros((L, nsrc, C))
    mags, phs, mms = [], [], []
    for c in range(C):
        mag_c, ph_c = scaled(audio[:, c])
        cb, _ = gen(mag_c, input_size=F, time_context=time_context, overlap=overlap, batch_size=batch_size)
        if nchunks == 0:
            mm = np.zeros((nsrc, T, F))
        else:
            mm = patch.overlapadd_multi(np.array([[m[:, i:i + 1] * b[:, 0:1] for i in range(nsrc)] for m, b in zip(ms, cb)]),
                                        batches, nchunks, overlap=overlap)
        for i in range(nsrc):
            rows = mm[i, :T]
            if rows.shape[0] < T:
                rows = np.concatenate([rows, np.zeros((T - rows.shape[0], F))])
            stems[:, i, c] = dsp.compute_inverse(rows / scale_factor, ph_c, **kw)[:L]
        mags.append(mag_c)
        phs.append(ph_c)
        mms.append(mm)
    return stems, mags, phs, mms, masks, kmap
