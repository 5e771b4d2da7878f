"""Weight-loading surface: the `.pkl` files of the reference are
`cPickle.dump(lasagne.layers.get_all_param_values(net))` -- a Python list of numpy arrays in layer
order (examples/dsd100/trainCNN.py:53-64; loaded by separate_dsd.py:17-21,249-250).  The list
layout per architecture is SURVEY.md App. A.4."""
import pickle
import numpy as np

# family defaults of the stand-alone scripts: (frameSize, hop, window name, overlap, source names)
FAMILY_DEFAULTS = {
    "dsd": dict(frameSize=1024, hopSize=512, window="hanning", overlap=25,
                sources=["vocals", "bass", "drums", "other"]),            # separate_dsd.py:243,332
    "ikala": dict(frameSize=1024, hopSize=512, window="hanning", overlap=20,
                  sources=["voice", "music"]),                             # separate_ikala.py:253-275
    "ikala_nopool": dict(frameSize=1024, hopSize=512, window="hanning", overlap=20,
                         sources=["voice", "music"]),
    "bach10": dict(frameSize=4096, hopSize=512, window="blackmanharris", overlap=25,
                   sources=["bassoon", "clarinet", "saxphone", "violin"]),  # separate_bach10.py:236,325
    "bach10_score": dict(frameSize=4096, hopSize=512, window="blackmanharris", overlap=25,
                         sources=["bassoon", "clarinet", "saxphone", "violin"]),
    # --function build_ca_1x1 of the same trainer (trainCNNrwc.py:66-132,629,655): N=4096 / hop 512, tc 30
    "bach10_score_1x1": dict(frameSize=4096, hopSize=512, window="blackmanharris", overlap=25,
                             sources=["bassoon", "clarinet", "saxphone", "violin"]),
    # stereo / ILD trainer: transform and overlap come from its __main__ defaults
    # (examples/dsd100_2ch_ILD/trainCNN_ILD_DSD100.py:118,147-148)
    "dsd_ild": dict(frameSize=1024, hopSize=512, window="hanning", overlap=25,
                    sources=["vocals", "bass", "drums", "other"]),
}


def load_model(filename):
    """separate_dsd.py:17-21.  Python-2 pickles of numpy arrays need encoding='latin1'."""
    with open(filename, "rb") as f:
        try:
            params = pickle.load(f)
        except UnicodeDecodeError:
            f.seek(0)
            params = pickle.load(f, encoding="latin1")
    return [np.asarray(p) for p in params]


def save_model(filename, params):
    """examples/dsd100/trainCNN.py:59-64 (protocol 2 keeps the file readable from Python 2)."""
    with open(filename, "wb") as f:
        pickle.dump([np.asarray(p) for p in params], f, protocol=2)


def _flat(arch, F, tc=30):
    if arch == "dsd":
        return 50 * (tc - tc // 2 + 1)
    w1 = (F - 30) // (3 if arch.startswith("ikala") else 4) + 1
    if arch == "ikala":
        return 30 * (tc - 10 + 1) * (w1 // 4 - 20 + 1)
    if arch == "ikala_nopool":
        return 30 * (tc - 10 + 1) * (w1 - 20 + 1)
    return 30 * (tc - int(2 * tc / 3) + 1) * w1


# build_ca_1x1: conv1..conv6 (filters, kernel height); every kernel is 5 wide with stride (1, 2)
S1X1_LAYERS = ((30, 1), (50, 1), (70, 1), (100, 1), (200, 10), (200, 10))


def check_1x1_geometry(feat_size, time_context):
    """build_ca_1x1 keeps no column of conv6 below 253 bins and no row below 19 frames; neither is in the weights."""
    if feat_size < 253:
        raise ValueError("build_ca_1x1 needs feat_size >= 253 (conv6 would have no columns), got %d" % feat_size)
    if time_context < 19:
        raise ValueError("build_ca_1x1 needs time_context >= 19 (conv6 would have no rows), got %d" % time_context)


def gate_code_layout(feat_size, time_context, Tp):
    """[(rows, width, channels)] of the ReLU gate codes of conv1..conv6 the routing tap holds for the 1x1 score net
    (include/dcs.h, dcs_set_pool_tap): Tp frames for conv1..conv4, Tp-9 and Tp-18 for conv5 and conv6."""
    out, W, rows = [], feat_size, Tp
    for C, kh in S1X1_LAYERS:
        W = (W - 5) // 2 + 1
        rows -= kh - 1
        out.append((rows, W, C))
    return out


def infer_arch(params, feat_size=None, time_context=None):
    """(arch, feat_size, time_context) from the parameter shapes (the .pkl carries no names).  For the 1x1 score net
    neither feat_size nor time_context is in the weights: the trainer's 2049 and 30 unless given."""
    n = len(params)
    s0 = params[0].shape
    if n == 22 and tuple(s0) == (30, 4, 1, 5):
        F, tc = int(feat_size or 2049), int(time_context or 30)
        check_1x1_geometry(F, tc)
        return "bach10_score_1x1", F, tc
    s3, s6 = params[3].shape, params[6].shape
    # DSD nets: conv2 has kh2 = int(tc/2) taps and leaves h2 = tc - kh2 + 1 rows, fc.W has 50*h2 rows: tc = h2 + kh2 - 1
    # (2*kh2 would be wrong for an odd time_context)
    if n == 15 and len(s0) == 4 and s0[0] == 50:
        return "dsd", int(s0[3]), int(s6[0]) // 50 + int(s3[2]) - 1
    if n == 17 and len(s0) == 4 and s0[0] == 50 and s0[1] == 2:
        return "dsd_ild", int(s0[3]), int(s6[0]) // 50 + int(s3[2]) - 1
    cands = (513, 1025, 2049, 257, 129, 65) if feat_size is None else (feat_size,)
    if n == 13 and s0[0] == 30:
        for F in cands:
            for arch in ("ikala", "ikala_nopool"):
                if _flat(arch, F) == s6[0]:
                    return arch, F, 30
    # the one-decoder score net (default build_ca of trainCNNrwc_samp.py:195-235) is decoder 1 of the 17-array one
    if (n == 17 or (n == 11 and s0[1] == 4)) and s0[0] == 30:
        arch = "bach10_score" if s0[1] == 4 else "bach10"
        for F in cands[::-1] if feat_size is None else cands:
            if _flat(arch, F) == s6[0]:
                return arch, F, 30
    raise ValueError("unrecognised parameter list: %d arrays, conv1.W %s, fc.W %s" % (n, s0, s6))
