"""Oracle (TEST INFRASTRUCTURE ONLY): float64 numpy restatement of the score-informed network build_ca_1x1
and of its separation branch, built on the layer functions of oracle/nets.py and the patcher of oracle/patch.py.

  network          examples/bach10_scoreinformed/trainCNNrwc.py:66-132 (trainCNNrwc_samp.py:66-132)
  separation       examples/bach10_scoreinformed/trainCNNrwc.py:357-416 (the branch oracle.pipeline.separate_score
                   restates for build_ca: util patcher, channels filter * magnitude, Bach10 mask on channels 0..3)
"""
import numpy as np

from oracle import dsp, patch
from oracle.nets import conv2d, conv2d_inverse, relu, near_kink, soft_masks, _as_float64

# Score-informed net selected with `--function build_ca_1x1` (examples/bach10_scoreinformed/trainCNNrwc.py:66-132,
# :629; trainCNNrwc_samp.py:66-132,675).  conv_l = Conv2DLayer(num_filters, (kh, 5), stride (1, 2), rectify) followed
# by a BiasLayer, so h_l = relu(W_l * h_{l-1} + b_l) + c_l; then Conv2DLayer(800, (1, 1), rectify) + BiasLayer sliced
# into four 200-channel sources.  Decoder d = InverseLayer(conv6) ... InverseLayer(conv1) of source d; InverseLayer
# is the gradient of the layer's output -- after its rectifier -- so inv_l(g) = conv_l^T(g * relu'(pre_l)), with
# Theano's relu = 0.5*(x + |x|): relu'(0) = 0.5 (-0.0 included).  ConcatLayer (16 channels) + BiasLayer + rectify;
# the Bach10 mask reads channels 0..3, all of decoder 1, so decoders 2-4 and 1x1 channels 200..799 are dead.
S1X1 = ((30, 1), (50, 1), (70, 1), (100, 1), (200, 10), (200, 10))   # conv1..conv6: (filters, kernel height)
GATE_TAU = 1e-5    # near_gate: relative distance to the rectifier's kink, in units of sum|w*x| + |b|


def param_shapes_1x1():
    """the 22 arrays of get_all_param_values(build_ca_1x1(...)): (W, b, c) of conv1..conv6 and the 1x1 conv, final bias"""
    shp, cin = [], 4
    for C, kh in S1X1:
        shp += [(C, cin, kh, 5), (C,), (C,)]
        cin = C
    return shp + [(800, 200, 1, 1), (800,), (800,), (16,)]


def make_synthetic_params_1x1(seed=0, dtype=np.float32, bias=0.02, out_bias=1e-4):
    """Seeded stand-in for a trained build_ca_1x1 .pkl: GlorotUniform filters, U(+-bias) biases on both sides of each
    rectifier, final bias U(0.5, 1.5) * out_bias: the decoder output is ~1e-4, so the masks vary strongly while few bins
    sit on the mask's all-zero discontinuity."""
    rng = np.random.default_rng(seed)
    out = []
    shapes = param_shapes_1x1()
    for i, s in enumerate(shapes):
        if i == len(shapes) - 1:
            out.append(rng.uniform(0.5 * out_bias, 1.5 * out_bias, size=s).astype(dtype))
            continue
        a = np.sqrt(6.0 / ((s[0] + s[1]) * s[2] * s[3])) if len(s) == 4 else bias
        out.append(rng.uniform(-a, a, size=s).astype(dtype))
    return out


def widths_1x1(F):
    """output widths of conv1..conv6 (F = 2049: 1023, 510, 253, 125, 61, 29)"""
    w, out = F, []
    for _ in S1X1:
        w = (w - 5) // 2 + 1
        out.append(w)
    return out


def gate_codes(pre):
    """2 * relu'(pre) of Theano's 0.5*(x + |x|): 2 above 0, 1 at exactly 0 (either sign), 0 below"""
    return np.where(pre > 0, 2, np.where(pre == 0, 1, 0)).astype(np.uint8)


def near_gate(pre, scale, tau=GATE_TAU):
    """Pre-activations whose rectifier decision is ill-conditioned: within tau * (sum|w*x| + |b|) of the kink, where
    no fp32 evaluation can be expected to land on float64's side.  An exact 0 of an all-zero sum (scale 0: silence and
    zero biases) is exact in every evaluation and is not flagged: there the device must give the 0.5 code too."""
    return np.abs(pre) < tau * scale


def predict_1x1(params, x, return_pre=False, gate_dev=None, gate_stats=None, all_decoders=False, tau=GATE_TAU):
    """`get_output(build_ca_1x1(...), deterministic=True)` in float64: x [B, 4, tc, F] -> rectified output (channels
    0..3 = decoder 1; all_decoders: all 16 concat channels) or the value before the final rectify (return_pre).
    gate_dev: per layer the device's gate codes [B, C, rows, W] and a per-patch validity mask [B]; at positions
    near_gate flags the device's code is adopted, everywhere else float64's is used and gate_stats counts the
    disagreements (and the flagged / total positions)."""
    p = _as_float64(params)
    h = np.asarray(x, dtype=np.float64)
    shapes, codes = [], []
    for l in range(6):
        W, b, c = p[3 * l], p[3 * l + 1], p[3 * l + 2]
        shapes.append(h.shape)
        pre = conv2d(h, W, (1, 2)) + b[None, :, None, None]
        code = gate_codes(pre)
        if gate_dev is not None:
            dev, valid = gate_dev[l]
            near = near_gate(pre, conv2d(np.abs(h), np.abs(W), (1, 2)) + np.abs(b)[None, :, None, None], tau)
            v = np.asarray(valid, dtype=bool)[:, None, None, None]
            if gate_stats is not None:
                gate_stats["positions"] = gate_stats.get("positions", 0) + int(v.sum()) * int(np.prod(pre.shape[1:]))
                gate_stats["flagged"] = gate_stats.get("flagged", 0) + int((near & v).sum())
                gate_stats["disagree_unflagged"] = gate_stats.get("disagree_unflagged", 0) + int(((dev != code) & ~near & v).sum())
                gate_stats["half"] = gate_stats.get("half", 0) + int(((np.where(near, dev, code) == 1) & v).sum())
            code = np.where(near & v, dev, code)
        codes.append(code)
        h = relu(pre) + c[None, :, None, None]
    s = relu(conv2d(h, p[18]) + p[19][None, :, None, None]) + p[20][None, :, None, None]
    decs = []
    for d in range(4 if all_decoders else 1):
        g = s[:, 200 * d:200 * (d + 1)]
        for l in range(5, -1, -1):
            g = conv2d_inverse(g * (0.5 * codes[l]), p[3 * l], shapes[l], (1, 2))
        decs.append(g)
    merged = np.concatenate(decs, axis=1)
    pre = merged + p[21][None, :merged.shape[1], None, None]
    return pre if return_pre else relu(pre)



def device_gates(codes_dev, bi, B, nchunks, step, time_context):
    """the device's gate codes of the whole clip (six uint8 [rows, W, C], the routing tap) -> predict_1x1's gate_dev for
    batch bi of B patches: row r of patch k is frame k*step + r; patches past nchunks (batch padding) are not valid"""
    dev = []
    for l, codes in enumerate(codes_dev):
        h = time_context - 9 * max(0, l - 3)       # rows of conv l+1 in a patch
        out = np.zeros((B, codes.shape[2], h, codes.shape[1]), dtype=np.uint8)
        valid = np.zeros(B, dtype=bool)
        for i in range(B):
            k = bi * B + i
            if k >= nchunks:
                break
            out[i] = codes[k * step:k * step + h].transpose(2, 0, 1)
            valid[i] = True
        dev.append((out, valid))
    return dev


def patches(chans, time_context, overlap, batch_size, patcher="util"):
    """the patcher on the [4, T, F] channel tensor: util's zero-padded one (util.py:220-248), or the stand-alone
    scripts' one (separate_dsd.py:114-135, tail dropped) channel by channel"""
    if patcher == "util":
        return patch.generate_overlapadd_util(chans, input_size=chans.shape[-1], time_context=time_context, overlap=overlap,
                                              batch_size=batch_size)
    per = [patch.generate_overlapadd(c, input_size=chans.shape[-1], time_context=time_context, overlap=overlap,
                                     batch_size=batch_size) for c in chans]
    return np.concatenate([b for b, _ in per], axis=2), per[0][1]


def separate_score_1x1(audio, filters, params, frameSize=4096, hopSize=512, window=None, scale_factor=0.2,
                       time_context=30, overlap=25, batch_size=32, gate_codes_dev=None, return_spec=False, patcher="util"):
    """The separation branch of trainCNNrwc.py:384-416 with build_ca_1x1, structured like oracle.pipeline.separate_score:
    filters [4, T, F] -> channels filter * mag (float32 products), util's zero-padded patcher, the network per batch of
    32 patches, Bach10 mask on the SUM of the channels, cross-fade, inverse STFT with the mixture phase.
    gate_codes_dev: the device's gate codes of the whole clip (a list of six uint8 [rows, W, C], the routing tap); row r of
    patch k is frame k*step + r.  separate_score_1x1.last_kink_map / last_gate_stats hold the flagged bins and counts."""
    if window is None:
        window = dsp.blackmanharris
    mag, ph = dsp.compute_file(audio, phase=True, frameSize=frameSize, hopSize=hopSize, window=window)
    mag = scale_factor * mag.astype(np.float32)
    chans = np.ones((4, mag.shape[0], mag.shape[1]))
    for j in range(4):
        chans[j] = np.asarray(filters[j], dtype=np.float32) * mag
    batches, nchunks = patches(chans, time_context, overlap, batch_size, patcher)
    step = time_context - overlap
    stats = {}
    pres = [predict_1x1(params, b, return_pre=True, gate_stats=stats,
                        gate_dev=None if gate_codes_dev is None else device_gates(gate_codes_dev, bi, b.shape[0], nchunks, step,
                                                                                  time_context))
            for bi, b in enumerate(batches)]
    separate_score_1x1.last_gate_stats = stats
    output = []
    for b, pre in zip(batches, pres):
        m = soft_masks(relu(pre), "bach10", 4)
        mix = b.sum(axis=1, keepdims=True)         # trainCNNrwc.py:258
        output.append([m[:, i:i + 1] * mix for i in range(4)])
    output = np.array(output)
    kmap = np.zeros((max(len(ph), nchunks * step + time_context), mag.shape[-1]), dtype=bool)
    left = nchunks
    for bi, b in enumerate(batches):
        nb = max(0, min(left, batch_size))
        flag = near_kink(pres[bi][:nb], "bach10", 4)
        for i in np.nonzero(flag.reshape(nb, -1).any(axis=1))[0]:
            k0 = (bi * batch_size + int(i)) * step
            kmap[k0:k0 + time_context] |= flag[i]
        left -= batch_size
    separate_score_1x1.last_kink_map = kmap[:len(ph)]
    if nchunks == 0:
        mm = np.zeros((4, len(ph), mag.shape[-1]))
    else:
        mm = patch.overlapadd_multi(output, batches, nchunks, overlap=overlap)
    stems = []
    for i in range(4):
        out = dsp.compute_inverse(mm[i, :len(ph)] / scale_factor, ph, frameSize=frameSize, hopSize=hopSize, window=window)
        stems.append(out[:len(audio)] if len(out) > len(audio) else out)
    if return_spec:
        return np.stack(stems), mag, ph, mm
    return np.stack(stems)
