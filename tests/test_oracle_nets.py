"""Cross-check oracle.nets against an independent torch-autograd formulation of the Lasagne
semantics (Conv2DLayer flips filters; InverseLayer == gradient wrt the layer's input)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as Fn
from oracle import nets


def torch_predict(params, x, arch):
    a = nets.ARCHS[arch]
    p = [torch.tensor(np.asarray(v, dtype=np.float64)) for v in params]
    x = torch.tensor(x, dtype=torch.float64, requires_grad=True)
    B, nch, tc, F = x.shape
    d = nets.arch_dims(arch, F, tc)
    conv1 = lambda v: Fn.conv2d(v, p[0].flip(2, 3), stride=(d["sh1"], d["sw1"]))
    conv2 = lambda v: Fn.conv2d(v, p[3].flip(2, 3))
    h1 = conv1(x) + (p[1] + p[2])[None, :, None, None]
    h1d = h1.detach().requires_grad_(True)
    if a["pool"]:
        # Theano MaxPoolGrad routes to ALL tied maxima; torch routes to one -> build the
        # tie-aware un-pool explicitly so that the two formulations only share the definition.
        wp = h1d.shape[3] // a["pool"]
        xr = h1d[..., :wp * a["pool"]].reshape(B, -1, tc, wp, a["pool"])
        hp = xr.max(dim=4).values
        hit = (xr == hp[..., None]).to(torch.float64)
    else:
        hp = h1d
    hpd = hp.detach().requires_grad_(True)
    h2 = conv2(hpd) + (p[4] + p[5])[None, :, None, None]
    z = torch.relu(h2.reshape(B, -1) @ p[6] + p[7])
    decs = []
    for s in range(d["ndec"]):
        r = torch.relu(z @ p[8 + 2 * s] + p[9 + 2 * s]).reshape(h2.shape).detach()
        g, = torch.autograd.grad(conv2(hpd), hpd, grad_outputs=r)
        if a["pool"]:
            gx = torch.zeros_like(h1d)
            gx[..., :wp * a["pool"]] = (hit * g[..., None]).reshape(B, -1, tc, wp * a["pool"])
            g = gx
        gin, = torch.autograd.grad(conv1(x), x, grad_outputs=g.detach())
        decs.append(gin)
    merged = torch.cat([decs[i] for i in a["dec_of_out"]], dim=1)
    return torch.relu(merged + p[-1][None, :, None, None]).detach().numpy()


@pytest.mark.parametrize("arch,F", [("dsd", 513), ("dsd", 65), ("ikala", 513), ("ikala_nopool", 129),
                                    ("bach10", 257), ("bach10_score", 129), ("dsd_ild", 129)])
def test_predict_matches_torch_autograd(arch, F):
    rng = np.random.default_rng(3)
    params = nets.make_synthetic_params(arch, F, seed=1)
    assert [v.shape for v in params] == nets.param_shapes(arch, F)
    nch = nets.ARCHS[arch]["nch"]
    x = 0.3 * np.abs(rng.standard_normal((3, nch, 30, F)))
    x[1, :, 10:20] = 0.0          # silent frames: constant conv1 output -> max-pool ties
    got = nets.predict(params, x, arch)
    ref = torch_predict(params, x, arch)
    assert got.shape == ref.shape == (3, nets.arch_dims(arch, F, 30)["nout"], 30, F)
    np.testing.assert_allclose(got, ref, rtol=0, atol=1e-12)


def test_param_counts():
    # SURVEY.md App. A.4
    assert sum(int(np.prod(s)) for s in nets.param_shapes("dsd", 513)) == 475482
    assert len(nets.param_shapes("dsd", 513)) == 15
    assert len(nets.param_shapes("ikala", 513)) == 13
    assert len(nets.param_shapes("bach10", 2049)) == 17
    assert nets.param_shapes("ikala", 513)[6] == (13230, 256)
    assert nets.param_shapes("ikala_nopool", 513)[6] == (90090, 256)
    assert nets.param_shapes("bach10", 2049)[6] == (166650, 256)
    for arch, F in [("dsd", 513), ("dsd", 1025), ("ikala", 513), ("ikala_nopool", 513), ("bach10", 2049)]:
        shapes = nets.param_shapes(arch, F)
        fake = [np.zeros(s, dtype=np.float32) if len(s) < 2 or s[0] * s[1] < 10 ** 6 else
                np.lib.stride_tricks.as_strided(np.zeros(1, np.float32), s, (0,) * len(s)) for s in shapes]
        assert nets.infer_arch(fake)[:2] == (arch, F)


@pytest.mark.parametrize("arch", ["dsd", "dsd_ild"])
@pytest.mark.parametrize("tc", [4, 17, 30, 31, 64])
def test_infer_arch_recovers_time_context(arch, tc):
    """conv2 has int(tc / 2) taps and leaves h2 = tc - int(tc / 2) + 1 rows: tc = h2 + kh2 - 1, odd tc included"""
    shapes = nets.param_shapes(arch, 129, tc)
    assert nets.infer_arch([np.zeros(s, dtype=np.float32) for s in shapes]) == (arch, 129, tc)


def test_mask_rules_closed_form():
    """eps*rand cancels: 'dsd' rule -> 1/nsrc on all-zero bins, 'bach10' rule -> 0 there;
    elsewhere both equal p/sum(p) to float64 rounding."""
    rng = np.random.default_rng(0)
    pred = np.maximum(rng.standard_normal((2, 4, 5, 7)), 0)
    pred[0, :, 2, 3] = 0
    r = rng.uniform(size=(2, 1, 5, 7))
    for rule in ("dsd", "bach10"):
        a = nets.soft_masks(pred, rule, 4, rand=r)
        b = nets.soft_masks(pred, rule, 4)
        np.testing.assert_allclose(a, b, rtol=1e-12, atol=1e-15)
    assert np.all(nets.soft_masks(pred, "dsd", 4)[0, :, 2, 3] == 0.25)
    assert np.all(nets.soft_masks(pred, "bach10", 4)[0, :, 2, 3] == 0.0)


def test_dsd_fourth_source_is_decoder_two():
    """separate_dsd.py:228 builds l_reshape4 from l_fc12: before the output bias, 'other' ==
    'bass' (SURVEY.md 0.3)."""
    params = nets.make_synthetic_params("dsd", 65, seed=5)
    params[-1][:] = 0
    x = 0.3 * np.abs(np.random.default_rng(1).standard_normal((2, 1, 30, 65)))
    pred = nets.predict(params, x, "dsd")
    np.testing.assert_array_equal(pred[:, 1], pred[:, 3])
    outs = nets.predict_function2(params, x, "dsd")
    np.testing.assert_allclose(sum(outs), x, rtol=1e-12, atol=1e-15)


def test_stereo_ild_masks_and_pipeline():
    """stereo / ILD variant (examples/dsd100_2ch_ILD/trainCNN_ILD_DSD100.py): outputs ordered
    (source, channel), masks normalised per channel, closed form == the seeded-noise graph, and the
    dataset loop of :299-327 gives stems whose per-channel sum is the mixture wherever the masks
    cover it."""
    from oracle import pipeline
    rng = np.random.default_rng(7)
    F = 65
    params = nets.make_synthetic_params("dsd_ild", F, seed=2)
    assert nets.infer_arch(params) == ("dsd_ild", F, 30)
    assert params[0].shape == (50, 2, 1, F) and params[-1].shape == (8,) and len(params) == 17
    x = 0.3 * np.abs(rng.standard_normal((2, 2, 30, F)))
    out = nets.predict_function_ild(params, x)
    assert len(out) == 2 and out[0].shape == (2, 4, 30, F)
    pred = nets.predict(params, x, "dsd_ild")
    for j in range(2):
        tot = pred[:, j::2].sum(axis=1)
        est = out[j].sum(axis=1)
        # where any source is active the four estimates of channel j add up to the channel's input
        np.testing.assert_allclose(est[tot > 0], x[:, j][tot > 0], rtol=1e-12)
        assert np.all(est[tot == 0] == 0)
    # the reference graph with its noise terms: eps * N(0, 0.1) with eps = 1e-12 perturbs a mask by
    # eps * |noise| / (sum of the outputs) -- below 1e-6 relative for sums above 1e-6
    noise = 0.1 * rng.standard_normal((2, 4, 30, F))
    noisy = nets.predict_function_ild(params, x, rand=noise)
    for j in range(2):
        tot = pred[:, j::2].sum(axis=1, keepdims=True)
        bound = 1e-12 * np.abs(noise) * (1.0 + x[:, j:j + 1] / np.where(tot > 0, tot, np.inf)) * 1.01
        assert np.all(np.abs(noisy[j] - out[j]) <= bound + 1e-300)
    # whole loop on a short stereo clip
    mix, _ = pipeline.synth_mixture(1.5, 3)
    audio = np.stack([mix, 0.6 * np.roll(mix, 7)], axis=1)
    N = 2 * (F - 1)
    sep = pipeline.separate_stereo(audio, params, frameSize=N, hopSize=N // 2)
    assert sep.shape == (len(mix), 4, 2) and np.isfinite(sep).all()
    # every (source, channel) carries energy with these weights, and the channels differ
    e = (sep ** 2).sum(axis=0)
    assert e.min() > 1e-4 * e.max()
    assert not np.allclose(sep[:, :, 0], sep[:, :, 1])
    # linearity in the channel gain is NOT expected (the net sees both channels); permuting the input
    # channels permutes nothing trivially either -- but a silent channel must give silent stems
    audio0 = audio.copy(); audio0[:, 1] = 0.0
    sep0 = pipeline.separate_stereo(audio0, params, frameSize=N, hopSize=N // 2)
    assert np.max(np.abs(sep0[:, :, 1])) < 1e-9
