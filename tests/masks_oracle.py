"""Oracle (TEST INFRASTRUCTURE ONLY): the blended soft masks sum_k w_k m_{s,k} of every network family in float64 --
the quantity the masks output (dcs_separate_masks*) returns -- computed from the same predictions, patcher and
cross-fade as the separation oracles (oracle.pipeline.separate / separate_score / separate_stereo and
score1x1_oracle.separate_score_1x1), which are left as they are.  The masks are cross-faded directly, not recovered as
mm / mag: that quotient is undefined where |X| = 0.

Each function returns (masks, mix, mm, kmap): masks float64 [nsrc, T, F] ([nsrc, 2, T, F] for the stereo net), the
mixture the network's masks multiply in the oracle (mag; the sum of the input channels for the score-informed nets;
per channel [2, T, F] for the stereo net), the oracle's blended masked magnitudes mm computed the pipeline's way
(sum_k w_k (m_{s,k} * mix)), and the bins near_kink flags (bool [T, F], [2, T, F] for the stereo net)."""
import numpy as np

from oracle import dsp, patch, nets
import score1x1_oracle as s1


def _blend(parts, batches, nchunks, overlap, T, F, nsrc):
    """overlapadd_multi of per-batch lists of nsrc arrays [B, 1, tc, F], cut or zero-padded to T frames"""
    if nchunks == 0:
        return np.zeros((nsrc, T, F))
    mm = patch.overlapadd_multi(np.array(parts), batches, nchunks, overlap=overlap)[:, :T]
    if mm.shape[1] < T:
        mm = np.concatenate([mm, np.zeros((nsrc, T - mm.shape[1], F))], axis=1)
    return mm


def _kink_map(pres, rule, nsrc, nchunks, batch_size, step, time_context, T, F, sel=slice(None)):
    kmap = np.zeros((max(T, nchunks * step + time_context), F), dtype=bool)
    left = nchunks
    for bi, pre in enumerate(pres):
        nb = max(0, min(left, batch_size))
        flag = nets.near_kink(pre[:nb][:, sel], rule, nsrc)
        for i in np.nonzero(flag.reshape(nb, -1).any(axis=1))[0]:
            k0 = (bi * batch_size + int(i)) * step
            kmap[k0:k0 + time_context] |= flag[i]
        left -= batch_size
    return kmap[:T]


def _pool_dev(pool_bits, batch_size, nchunks, step, time_context, T):
    """the device's tie bits uint8 [T, WP, C] -> predict's pool_dev of batch bi (as oracle.pipeline.separate builds it)"""
    bits = np.asarray(pool_bits)[:, :, :30]
    dev = np.stack([(bits >> r) & 1 for r in range(4)], axis=-1).astype(bool).transpose(2, 0, 1, 3)   # [C, T, WP, 4]

    def of(bi, b):
        C_, T2, WP_, _ = dev.shape
        out = np.zeros((b.shape[0], C_, time_context, WP_, 4), dtype=bool)
        valid = np.zeros((b.shape[0], 1, time_context, 1, 1), dtype=bool)
        for i in range(b.shape[0]):
            k = bi * batch_size + i
            if k >= nchunks:
                break
            t0 = k * step
            n = max(0, min(time_context, T - t0, T2 - t0))
            out[i, :, :n] = dev[:, t0:t0 + n]
            valid[i, 0, :n] = True
        return out, valid
    return of


def separate_masks(audio, params, arch, frameSize=1024, hopSize=512, window=np.hanning, scale_factor=0.3,
                   time_context=30, overlap=25, batch_size=32, patcher="standalone", pool_bits=None):
    """the single-channel nets (oracle.pipeline.separate); pool_bits: the max-pool net's device routing, adopted in the
    ill-conditioned windows only"""
    a = nets.ARCHS[arch]
    mag, ph = dsp.compute_file(audio, phase=True, frameSize=frameSize, hopSize=hopSize, window=window)
    mag = scale_factor * mag.astype(np.float32)
    T, F = mag.shape
    gen = patch.generate_overlapadd if patcher == "standalone" else patch.generate_overlapadd_util
    batches, nchunks = gen(mag, input_size=F, time_context=time_context, overlap=overlap, batch_size=batch_size)
    step = time_context - overlap
    pd = None if pool_bits is None else _pool_dev(pool_bits, batch_size, nchunks, step, time_context, T)
    pres = [nets.predict(params, b, arch, return_pre=True, pool_dev=None if pd is None else pd(bi, b))
            for bi, b in enumerate(batches)]
    ms = [nets.soft_masks(nets.relu(p), a["mask"], a["nsrc"]) for p in pres]
    masks = _blend([[m[:, i:i + 1] for i in range(a["nsrc"])] for m in ms], batches, nchunks, overlap, T, F, a["nsrc"])
    mm = _blend([[m[:, i:i + 1] * b[:, 0:1] for i in range(a["nsrc"])] for m, b in zip(ms, batches)], batches, nchunks,
                overlap, T, F, a["nsrc"])
    kmap = _kink_map(pres, a["mask"], a["nsrc"], nchunks, batch_size, step, time_context, T, F)
    return masks, np.asarray(mag, dtype=np.float64), mm, kmap


def _score_chans(audio, filters, frameSize, hopSize, window, scale_factor):
    mag, _ = dsp.compute_file(audio, phase=True, frameSize=frameSize, hopSize=hopSize, window=window)
    mag = scale_factor * mag.astype(np.float32)
    chans = np.ones((4, mag.shape[0], mag.shape[1]))
    for j in range(4):
        chans[j] = np.asarray(filters[j], dtype=np.float32) * mag
    return chans


def _score_result(pres, batches, nchunks, overlap, batch_size, time_context, T, F):
    ms = [nets.soft_masks(nets.relu(p), "bach10", 4) for p in pres]
    masks = _blend([[m[:, i:i + 1] for i in range(4)] for m in ms], batches, nchunks, overlap, T, F, 4)
    mm = _blend([[m[:, i:i + 1] * b.sum(axis=1, keepdims=True) for i in range(4)] for m, b in zip(ms, batches)], batches,
                nchunks, overlap, T, F, 4)
    kmap = _kink_map(pres, "bach10", 4, nchunks, batch_size, time_context - overlap, time_context, T, F)
    return masks, mm, kmap


def separate_score_masks(audio, filters, params, frameSize=4096, hopSize=512, window=None, scale_factor=0.2,
                         time_context=30, overlap=25, batch_size=32):
    """the score-informed build_ca (oracle.pipeline.separate_score): util patcher on the channels filter * mag"""
    window = dsp.blackmanharris if window is None else window
    chans = _score_chans(audio, filters, frameSize, hopSize, window, scale_factor)
    T, F = chans.shape[1:]
    batches, nchunks = patch.generate_overlapadd_util(chans, input_size=F, time_context=time_context, overlap=overlap,
                                                      batch_size=batch_size)
    pres = [nets.predict(params, b, "bach10_score", return_pre=True) for b in batches]
    masks, mm, kmap = _score_result(pres, batches, nchunks, overlap, batch_size, time_context, T, F)
    return masks, chans.sum(axis=0), mm, kmap


def separate_score_1x1_masks(audio, filters, params, frameSize=4096, hopSize=512, window=None, scale_factor=0.2,
                             time_context=30, overlap=25, batch_size=32, gate_codes_dev=None, patcher="util"):
    """build_ca_1x1 (score1x1_oracle.separate_score_1x1); gate_codes_dev: the device's gate codes (routing tap),
    adopted where near_gate flags the pre-activation"""
    window = dsp.blackmanharris if window is None else window
    chans = _score_chans(audio, filters, frameSize, hopSize, window, scale_factor)
    T, F = chans.shape[1:]
    batches, nchunks = s1.patches(chans, time_context, overlap, batch_size, patcher)
    step = time_context - overlap
    pres = [s1.predict_1x1(params, b, return_pre=True,
                           gate_dev=None if gate_codes_dev is None else s1.device_gates(gate_codes_dev, bi, b.shape[0], nchunks,
                                                                                        step, time_context))
            for bi, b in enumerate(batches)]
    masks, mm, kmap = _score_result(pres, batches, nchunks, overlap, batch_size, time_context, T, F)
    return masks, chans.sum(axis=0), mm, kmap


def separate_stereo_masks(audio, params, frameSize=1024, hopSize=512, window=np.hanning, scale_factor=0.3,
                          time_context=30, overlap=25, batch_size=32):
    """the stereo / ILD net (oracle.pipeline.separate_stereo): audio [L, 2]; per channel the masks normalised over the
    sources, masks [nsrc, 2, T, F]"""
    a = nets.ARCHS["dsd_ild"]
    nch, nsrc = a["nch"], a["nsrc"]
    mag = scale_factor * np.stack([dsp.compute_file(audio[:, j], phase=True, frameSize=frameSize, hopSize=hopSize,
                                                    window=window)[0] for j in range(nch)]).astype(np.float32)
    _, T, F = mag.shape
    batches, nchunks = patch.generate_overlapadd_util(mag, input_size=F, time_context=time_context, overlap=overlap,
                                                      batch_size=batch_size)
    pres = [nets.predict(params, b, "dsd_ild", return_pre=True) for b in batches]
    masks, mms, kmaps = np.zeros((nsrc, nch, T, F)), np.zeros((nsrc, nch, T, F)), []
    for j in range(nch):
        ms = []
        for p in pres:
            pj = nets.relu(p)[:, j::nch]
            tot = pj.sum(axis=1, keepdims=True)
            ms.append(pj / np.where(tot > 0, tot, 1.0))
        masks[:, j] = _blend([[m[:, i:i + 1] for i in range(nsrc)] for m in ms], batches, nchunks, overlap, T, F, nsrc)
        mms[:, j] = _blend([[m[:, i:i + 1] * b[:, j:j + 1] for i in range(nsrc)] for m, b in zip(ms, batches)], batches,
                           nchunks, overlap, T, F, nsrc)
        kmaps.append(_kink_map(pres, a["mask"], nsrc, nchunks, batch_size, time_context - overlap, time_context, T, F,
                               sel=slice(j, None, nch)))
    return masks, np.asarray(mag, dtype=np.float64), mms, np.stack(kmaps)
