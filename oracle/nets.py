"""Oracle (TEST INFRASTRUCTURE ONLY): float64 numpy restatement of the four `build_ca`
networks and of the soft-mask graph.  **Parity unpinned** (see oracle/__init__.py): the
arithmetic lives in Theano 0.9 / Lasagne master, which are not in /root/reference.

Reference call sites restated here:
  DSD100 / hiphopss  examples/dsd100/separate_dsd.py:172-236 (net), :252-271 (mask)
  iKala (max-pool)   examples/ikala/separate_ikala.py:172-192 (net), :207-216 (mask)
  iKala (no pool)    examples/ikala/trainCNN.py:66-110
  Bach10             examples/bach10/separate_bach10.py:172-229 (net), :245-264 (mask)
  Score-informed     examples/bach10_scoreinformed/trainCNNrwc.py:134-193 (net), :248-263 (mask)
  Stereo / ILD       examples/dsd100_2ch_ILD/trainCNN_ILD_DSD100.py:66-113 (net), :176-189 (mask)
Lasagne layer semantics: SURVEY.md App. A.2 (Conv2DLayer flips filters; DenseLayer defaults
to rectify; InverseLayer = gradient of the layer output wrt its input, tied weights).
"""
import numpy as np
from numpy.lib.stride_tricks import sliding_window_view

EPS = 1e-18  # separate_dsd.py:245

# name -> (nsrc, in-channels, conv1 (filters, kh, kw, sh, sw), pool_w, conv2 (filters, kh, kw),
#          bottleneck, decoder index feeding each concatenated output, mask rule)
ARCHS = {
    # conv1 kw == feat_size, conv2 kh == time_context // 2 (separate_dsd.py:198,202)
    "dsd": dict(nsrc=4, nch=1, c1=(50, 1, "F", 1, 1), pool=0, c2=(50, "T/2", 1), nfc=128,
                dec_of_out=(0, 1, 2, 1), ndec=3, mask="dsd"),
    "ikala": dict(nsrc=2, nch=1, c1=(30, 1, 30, 1, 3), pool=4, c2=(30, 10, 20), nfc=256,
                  dec_of_out=(0, 1), ndec=2, mask="dsd"),
    "ikala_nopool": dict(nsrc=2, nch=1, c1=(30, 1, 30, 1, 3), pool=0, c2=(30, 10, 20), nfc=256,
                         dec_of_out=(0, 1), ndec=2, mask="dsd"),
    # conv2 kh == int(2 * time_context / 3) (separate_bach10.py:200)
    "bach10": dict(nsrc=4, nch=1, c1=(30, 1, 30, 1, 4), pool=0, c2=(30, "2T/3", 1), nfc=256,
                   dec_of_out=(0, 1, 2, 3), ndec=4, mask="bach10"),
    "bach10_score": dict(nsrc=4, nch=4, c1=(30, 1, 30, 1, 4), pool=0, c2=(30, "2T/3", 1), nfc=256,
                         dec_of_out=(0, 1, 2, 3), ndec=4, mask="bach10"),
    # stereo DSD100 with the inter-aural level difference loss: 2 input channels, one decoder per
    # source, each InverseLayer(conv1) returns both channels -> 8 outputs ordered (source, channel)
    # (trainCNN_ILD_DSD100.py:88-106); masks are normalised per channel over the sources (:183-186)
    "dsd_ild": dict(nsrc=4, nch=2, c1=(50, 1, "F", 1, 1), pool=0, c2=(50, "T/2", 1), nfc=256,
                    dec_of_out=(0, 1, 2, 3), ndec=4, mask="ild"),
}

EPS_ILD = 1e-12  # trainCNN_ILD_DSD100.py:153


def arch_dims(arch, F, tc):
    a = ARCHS[arch]
    f1, kh1, kw1, sh1, sw1 = a["c1"]
    if kw1 == "F":
        kw1 = F
    f2, kh2, kw2 = a["c2"]
    if kh2 == "T/2":
        kh2 = int(tc / 2)
    elif kh2 == "2T/3":
        kh2 = int(2 * tc / 3)
    h1, w1 = (tc - kh1) // sh1 + 1, (F - kw1) // sw1 + 1
    wp = w1 // a["pool"] if a["pool"] else w1
    h2, w2 = h1 - kh2 + 1, wp - kw2 + 1
    return dict(f1=f1, kh1=kh1, kw1=kw1, sh1=sh1, sw1=sw1, h1=h1, w1=w1, wp=wp,
                f2=f2, kh2=kh2, kw2=kw2, h2=h2, w2=w2, flat=f2 * h2 * w2, nfc=a["nfc"],
                nch=a["nch"], ndec=a["ndec"], nsrc=a["nsrc"], nout=len(a["dec_of_out"]) * a["nch"])


def param_shapes(arch, F, tc=30):
    """Shapes of `lasagne.layers.get_all_param_values(net)` (SURVEY.md App. A.4)."""
    d = arch_dims(arch, F, tc)
    shp = [(d["f1"], d["nch"], d["kh1"], d["kw1"]), (d["f1"],), (d["f1"],),
           (d["f2"], d["f1"], d["kh2"], d["kw2"]), (d["f2"],), (d["f2"],),
           (d["flat"], d["nfc"]), (d["nfc"],)]
    for _ in range(d["ndec"]):
        shp += [(d["nfc"], d["flat"]), (d["flat"],)]
    shp.append((d["nout"],))
    return shp


def make_synthetic_params(arch, F, tc=30, seed=0, dtype=np.float32, out_bias=0.002):
    """Seeded stand-in for a trained .pkl: Lasagne GlorotUniform weights, U(+-0.1) biases.
    The final per-source bias is U(+-out_bias): with Glorot weights the decoder output has a
    standard deviation of ~2.5e-3 for |x| ~ 1e-2, so a +-0.1 output bias would swamp it and
    every mask would be a constant -- a parity test that exercises nothing.  +-0.002 gives
    ~50 % ReLU zeros per source, strongly varying masks and some all-zero bins."""
    rng = np.random.default_rng(seed)
    out = []
    shapes = param_shapes(arch, F, tc)
    for i, s in enumerate(shapes):
        if len(s) == 4:
            a = np.sqrt(6.0 / ((s[0] + s[1]) * s[2] * s[3]))
        elif len(s) == 2:
            a = np.sqrt(6.0 / (s[0] + s[1]))
        else:
            a = out_bias if i == len(shapes) - 1 else 0.1
        out.append(rng.uniform(-a, a, size=s).astype(dtype))
    return out


def infer_arch(params):
    """Infer (arch, F, time_context) from the shapes in a parameter list."""
    n = len(params)
    w1, w2, wfc = params[0].shape, params[3].shape, params[6].shape
    # DSD nets: conv2 has kh2 = int(tc / 2) taps and leaves h2 = tc - kh2 + 1 rows, fc.W has 50 * h2 rows, so
    # tc = h2 + kh2 - 1 (2 * kh2 is wrong for an odd time_context)
    if n == 15 and w1[0] == 50:
        return "dsd", w1[3], wfc[0] // 50 + w2[2] - 1
    if n == 13 and w1[0] == 30:
        # fc.W rows disambiguate the pool / no-pool iKala nets (SURVEY.md 0.7); F is not
        # recoverable from the parameters (conv1 is 30 wide) -> iKala default 513.
        for arch in ("ikala", "ikala_nopool"):
            if arch_dims(arch, 513, 30)["flat"] == wfc[0]:
                return arch, 513, 30
    if n == 17 and w1[0] == 50 and w1[1] == 2:
        return "dsd_ild", w1[3], wfc[0] // 50 + w2[2] - 1
    if n == 17 and w1[0] == 30:
        arch = "bach10_score" if w1[1] == 4 else "bach10"
        for F in (2049, 1025, 513):
            if arch_dims(arch, F, 30)["flat"] == wfc[0]:
                return arch, F, 30
    raise ValueError("unrecognised parameter list (%d arrays, conv1.W %s, fc.W %s)" % (n, w1, wfc))


# ----------------------------------------------------------------------------- layers
def conv2d(x, W, stride=(1, 1)):
    """lasagne Conv2DLayer(pad='valid', flip_filters=True), no bias:
    out[b,f,i,j] = sum_{c,p,q} W[f,c,p,q] * x[b,c,i*sh+(kh-1-p), j*sw+(kw-1-q)]"""
    sh, sw = stride
    F_, C, kh, kw = W.shape
    Wf = W[:, :, ::-1, ::-1]
    win = sliding_window_view(x, (kh, kw), axis=(2, 3))[:, :, ::sh, ::sw]  # [B,C,oh,ow,kh,kw]
    out = np.tensordot(win, Wf, axes=([1, 4, 5], [1, 2, 3]))               # [B,oh,ow,F]
    return np.ascontiguousarray(out.transpose(0, 3, 1, 2))


def conv2d_inverse(g, W, in_shape, stride=(1, 1)):
    """lasagne InverseLayer(g, conv): d(sum(conv(x) * g))/dx -- transposed convolution with
    the same (tied) W; input positions no stride window covers stay 0."""
    sh, sw = stride
    F_, C, kh, kw = W.shape
    B, _, oh, ow = g.shape
    Wf = W[:, :, ::-1, ::-1]
    gx = np.zeros((B,) + tuple(in_shape[1:]))
    if kh * kw > oh * ow:
        cols = np.tensordot(g, Wf, axes=([1], [0]))        # [B,oh,ow,C,kh,kw]
        for i in range(oh):
            for j in range(ow):
                gx[:, :, i * sh:i * sh + kh, j * sw:j * sw + kw] += cols[:, i, j]
    else:
        for p in range(kh):
            for q in range(kw):
                t = np.tensordot(g, Wf[:, :, p, q], axes=([1], [0]))  # [B,oh,ow,C]
                gx[:, :, p:p + sh * oh:sh, q:q + sw * ow:sw] += t.transpose(0, 3, 1, 2)
    return gx


def maxpool_w(x, pw):
    """MaxPool2DLayer(pool_size=(1,pw)), stride = pool size, ignore_border=True."""
    B, C, H, W = x.shape
    wp = W // pw
    return x[:, :, :, :wp * pw].reshape(B, C, H, wp, pw).max(axis=4)


def maxpool_w_inverse(g, x, pw, dev_hits=None, tau_rel=4e-6, stats=None):
    """InverseLayer(g, pool): Theano MaxPoolGrad -- the value goes to every position of the
    window equal to the window maximum (ties all receive it); dropped border columns get 0.

    The routing is a DISCRETE decision: where two positions of a window differ by less than the rounding
    noise of any float32 evaluation (or of the float32 STFT feeding it) the argmax is ill-conditioned --
    the same kind of discontinuity as the soft mask's (near_kink).  For the parity tests `dev_hits` =
    (hits [B,C,H,wp,pw], valid [B,1,H,1,1]) (the device's own tie bits per patch row) may be supplied: in windows where some non-maximal position
    lies within tau of the maximum (tau = tau_rel * (|max| + 0.05)) the device's choice is adopted --
    after checking it only selects positions inside that near-maximal set -- and everywhere else the
    float64 argmax is used and the device is REQUIRED to agree (`stats` collects the counts)."""
    B, C, H, W = x.shape
    wp = W // pw
    xr = x[:, :, :, :wp * pw].reshape(B, C, H, wp, pw)
    top = xr.max(axis=4, keepdims=True)
    hit = (xr == top)
    if dev_hits is not None:
        near = (top - xr) <= tau_rel * (np.abs(top) + 0.05)
        amb = near.sum(axis=4, keepdims=True) > hit.sum(axis=4, keepdims=True)     # an ill-conditioned window
        dev, valid = dev_hits
        dev = np.where(valid, dev.astype(bool), hit)      # rows without a device decision keep the float64 one
        if stats is not None:
            stats["windows"] = stats.get("windows", 0) + int(amb.size)
            stats["ambiguous"] = stats.get("ambiguous", 0) + int(amb.sum())
            stats["disagree_well_conditioned"] = stats.get("disagree_well_conditioned", 0) + int(((dev != hit).any(axis=4, keepdims=True) & ~amb).sum())
            stats["inadmissible"] = stats.get("inadmissible", 0) + int(((dev & ~near).any(axis=4, keepdims=True) & amb).sum()) \
                + int((~dev.any(axis=4, keepdims=True) & amb).sum())
        hit = np.where(amb, dev, hit)
    gx = np.zeros_like(x)
    gx[:, :, :, :wp * pw] = (hit * g[..., None]).reshape(B, C, H, wp * pw)
    return gx


def relu(x):
    return np.maximum(x, 0.0)


# ----------------------------------------------------------------------------- networks
_F64_CACHE = {"key": None, "val": None}


def _as_float64(params):
    """float64 copies of a parameter list, kept for the last list seen (the Bach10 nets have 214 M
    parameters: converting them once per 32-patch batch dominated the oracle's run time)."""
    key = tuple((id(v), getattr(v, "shape", None)) for v in params)
    if _F64_CACHE["key"] != key:
        _F64_CACHE["val"] = [np.asarray(v, dtype=np.float64) for v in params]
        _F64_CACHE["key"] = key
    return _F64_CACHE["val"]


def predict(params, x, arch, return_pre=False, pool_dev=None, pool_stats=None):
    """`lasagne.layers.get_output(build_ca(...), deterministic=True)`: x [B,nch,tc,F] ->
    rectified concat output [B, nout, tc, F] (return_pre: the value before the final rectify).
    pool_dev: see maxpool_w_inverse (parity tests of the max-pool net only)."""
    a = ARCHS[arch]
    p = _as_float64(params)
    x = np.asarray(x, dtype=np.float64)
    B, nch, tc, F = x.shape
    d = arch_dims(arch, F, tc)
    s1 = (d["sh1"], d["sw1"])
    W1, W2 = p[0], p[3]
    h1 = conv2d(x, W1, s1) + (p[1] + p[2])[None, :, None, None]          # conv1 + b, BiasLayer
    hp = maxpool_w(h1, a["pool"]) if a["pool"] else h1
    h2 = conv2d(hp, W2) + (p[4] + p[5])[None, :, None, None]            # conv2 + b, BiasLayer
    z = relu(h2.reshape(B, -1) @ p[6] + p[7])                            # DenseLayer (rectify)
    decs = []
    for s in range(d["ndec"]):
        Ws, bs = p[8 + 2 * s], p[9 + 2 * s]
        r = relu(z @ Ws + bs).reshape(B, d["f2"], d["h2"], d["w2"])      # DenseLayer + Reshape
        g = conv2d_inverse(r, W2, hp.shape)                              # InverseLayer(., conv2)
        if a["pool"]:
            g = maxpool_w_inverse(g, h1, a["pool"], dev_hits=pool_dev, stats=pool_stats)   # InverseLayer(., pool1)
        decs.append(conv2d_inverse(g, W1, x.shape, s1))                  # InverseLayer(., conv1)
    merged = np.concatenate([decs[i] for i in a["dec_of_out"]], axis=1)  # ConcatLayer(axis=1)
    pre = merged + p[-1][None, :, None, None]                            # BiasLayer
    return pre if return_pre else relu(pre)                              # + rectify


def near_kink(pre, rule, nsrc, tau=None):
    """Bins where the reference's soft mask is DISCONTINUOUS and the float64 value sits within
    `tau` of the jump: all rectified outputs vanish on one side ('dsd' rule: masks jump from
    (1/nsrc, ...) to (1, 0, ...); 'bach10' rule: from 0 to 1).  No finite-precision evaluation
    can be expected to land on the oracle's side there.  Default tau = 1e-5 x the mean absolute
    pre-activation (>= 2e-8): a chain of six fp32-accurate contractions reproduces a
    pre-activation to a few 1e-6 of its typical magnitude, not of its own (near-zero) value."""
    x = pre[:, :nsrc]
    if tau is None:
        tau = max(2e-8, 1e-5 * float(np.mean(np.abs(x))))
    s = np.sort(x, axis=1)
    top, second = s[:, -1], s[:, -2]
    return (np.abs(top) < tau) & (second <= tau)


def soft_masks(pred, rule, nsrc, rand=None):
    """Mask graph.  `rand` None -> the closed forms of SURVEY.md 0.5 (the unseeded uniform
    `rand_num` cancels): 'dsd' rule: all-zero bins get 1/nsrc; 'bach10' rule: they get 0."""
    s = pred[:, :nsrc]
    if rand is not None:
        if rule == "dsd":     # separate_dsd.py:258-266
            v = s + EPS * rand
            return v / v.sum(axis=1, keepdims=True)
        return s / (s.sum(axis=1, keepdims=True) + EPS * rand)  # separate_bach10.py:256-259
    tot = s.sum(axis=1, keepdims=True)
    safe = np.where(tot > 0, tot, 1.0)
    m = s / safe
    if rule == "dsd":
        m = np.where(tot > 0, m, 1.0 / nsrc)
    return m


def predict_function2(params, x, arch, rand=None, pred=None):
    """The compiled Theano function of train_auto (separate_dsd.py:273): batch -> list of
    nsrc arrays [B,1,tc,F] = mask_s * mixture.  (`pred`: the rectified network output if the
    caller already evaluated it.)"""
    a = ARCHS[arch]
    x = np.asarray(x, dtype=np.float64)
    if pred is None:
        pred = predict(params, x, arch)
    m = soft_masks(pred, a["mask"], a["nsrc"], rand)
    # score-informed: mixture estimate = sum of the input channels (trainCNNrwc.py:258)
    mix = x.sum(axis=1, keepdims=True) if a["nch"] > 1 else x[:, 0:1]
    return [m[:, i:i + 1] * mix for i in range(a["nsrc"])]


def predict_function_ild(params, x, rand=None, pred=None):
    """`predict_function` of the stereo / ILD trainer (trainCNN_ILD_DSD100.py:176-189,232):
    x [B, 2, tc, F] -> list over the input channels j of [B, nsrc, tc, F] = mask_j * x[:, j].
    The network's outputs are ordered (source, channel); channel j's masks are outputs j::nch
    divided by their sum over the sources (+ eps * N(0, 0.1) noise with eps = 1e-12: `rand` None
    uses the closed form -- an all-zero bin has numerator 0, so its mask is 0 -- and drops the
    additive eps * noise on the estimate, 1e-13 absolute)."""
    a = ARCHS["dsd_ild"]
    x = np.asarray(x, dtype=np.float64)
    if pred is None:
        pred = predict(params, x, "dsd_ild")
    nch, nsrc = a["nch"], a["nsrc"]
    out = []
    for j in range(nch):
        pj = pred[:, j::nch]
        tot = pj.sum(axis=1, keepdims=True)
        if rand is not None:
            mask = pj / (tot + EPS_ILD * rand)
            out.append(mask * x[:, j:j + 1] + EPS_ILD * rand)
        else:
            mask = pj / np.where(tot > 0, tot, 1.0)
            out.append(mask * x[:, j:j + 1])
    return out
