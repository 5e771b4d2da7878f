"""Float64 oracle of the keep-channels mode of the DSD100 / hiphopss network (TEST INFRASTRUCTURE: built on oracle/).

The network sees the downmix (l + r) / 2 exactly as `oracle.pipeline.separate` runs it (float32 scaled magnitude, the
patcher, batches of 32, the soft-mask rule); its per-patch soft masks are then applied to the patches of each channel's
scaled magnitude, cross-faded with the same `overlapadd_multi`, and inverted with that channel's phase.  That is
M~_s * X_c per (source, channel), M~_s = overlapadd_multi of the per-patch masks, formed without dividing anything by
the downmix's magnitude (which vanishes where the channels are in anti-phase)."""
import numpy as np

from oracle import dsp, patch, nets


def separate_keep_channels(audio, params, frameSize=1024, hopSize=512, window=np.hanning, scale_factor=0.3,
                           time_context=30, overlap=25, batch_size=32, patcher="standalone"):
    """audio float [L, 2] -> (stems float64 [L, nsrc, 2], mags [2] of [T, F] (scaled float32 magnitude per channel),
    phs [2] of [T, F], mms [2] of [nsrc, T', F] (M~ times the channel's scaled magnitude), kink map bool [T, F] of the
    downmix).  Per channel c, (stems[:, :, c].T, mags[c], phs[c], mms[c], kmap) is what tests/parity.strict_check takes.
    separate_keep_channels.last_masks: the blended masks M~ [nsrc, T', F]."""
    arch = "dsd"
    a = nets.ARCHS[arch]
    nsrc = a["nsrc"]
    audio = np.asarray(audio, dtype=np.float64)
    assert audio.ndim == 2 and audio.shape[1] == 2, audio.shape
    L = audio.shape[0]
    kw = dict(frameSize=frameSize, hopSize=hopSize, window=window)
    gen = patch.generate_overlapadd if patcher == "standalone" else patch.generate_overlapadd_util

    def scaled(x):
        m, p = dsp.compute_file(x, phase=True, **kw)
        return scale_factor * m.astype(np.float32), p           # separate_dsd.py:290 (float32)

    mag, ph = scaled((audio[:, 0] + audio[:, 1]) / 2)
    T, F = mag.shape
    batches, nchunks = gen(mag, input_size=F, time_context=time_context, overlap=overlap, batch_size=batch_size)
    pres = [nets.predict(params, b, arch, return_pre=True) for b in batches]
    masks = [nets.soft_masks(nets.relu(p), a["mask"], nsrc) for p in pres]            # [B, nsrc, tc, F] per batch

    # kink map of the downmix (as oracle.pipeline.separate(count_kinks=True) builds it): applies to both channels
    step = time_context - overlap
    kmap = np.zeros((max(T, nchunks * step + time_context), F), dtype=bool)
    left = nchunks
    for bi, b in enumerate(batches):
        nb = max(0, min(left, batch_size))
        flag = nets.near_kink(pres[bi][:nb], a["mask"], nsrc)
        for i in np.nonzero(flag.reshape(nb, -1).any(axis=1))[0]:
            k0 = (bi * batch_size + int(i)) * step
            kmap[k0:k0 + time_context] |= flag[i]
        left -= batch_size
    kmap = kmap[:T]

    def blend(per_batch):
        if nchunks == 0:
            return np.zeros((nsrc, T, F))
        return patch.overlapadd_multi(np.array(per_batch), batches, nchunks, overlap=overlap)

    separate_keep_channels.last_masks = blend([[m[:, i:i + 1] for i in range(nsrc)] for m in masks])

    stems = np.zeros((L, nsrc, 2))
    mags, phs, mms = [], [], []
    for c in range(2):
        mag_c, ph_c = scaled(audio[:, c])
        cb, _ = gen(mag_c, input_size=F, time_context=time_context, overlap=overlap, batch_size=batch_size)
        # mask times the channel's patch, then the cross-fade: with l == r these are the mono oracle's operations
        mm = blend([[m[:, i:i + 1] * b[:, 0:1] for i in range(nsrc)] for m, b in zip(masks, cb)])
        for i in range(nsrc):
            out = dsp.compute_inverse(mm[i, :T] / scale_factor, ph_c, **kw)
            stems[:, i, c] = out[:L]
        mags.append(mag_c)
        phs.append(ph_c)
        mms.append(mm)
    return stems, mags, phs, mms, kmap
