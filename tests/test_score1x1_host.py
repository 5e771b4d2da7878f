"""Host tests of the score-informed build_ca_1x1 network (examples/bach10_scoreinformed/trainCNNrwc.py:66-132): the
float64 oracle (tests/score1x1_oracle.py) against an independent torch-autograd formulation of the same Lasagne graph, the
0.5 derivative of Theano's rectifier at 0, the dead decoders, and the parameter-list inference of deepconvsep_b200.models."""
import numpy as np
import pytest

import score1x1_oracle as s1
from oracle.nets import conv2d
from deepconvsep_b200 import models

torch = pytest.importorskip("torch")


def torch_1x1(params, x, theano_relu=True):
    """get_output(build_ca_1x1(...)) with torch autograd: Conv2DLayer flips its filters, rectify is Theano's
    0.5*(x + |x|), and each InverseLayer(incoming, layer) is the vector-Jacobian product of the layer's output (after
    its rectifier) with respect to its input.  All four decoders; returns the rectified 16-channel concat.
    theano_relu=False: the encoder uses torch.relu, whose derivative at 0 is 0 instead of 0.5."""
    P = [torch.tensor(np.asarray(p, dtype=np.float64)) for p in params]
    h = torch.tensor(np.asarray(x, dtype=np.float64), requires_grad=True)
    ins, outs = [], []
    for l in range(6):
        ins.append(h)
        pre = torch.nn.functional.conv2d(h, P[3 * l].flip(2, 3), stride=(1, 2)) + P[3 * l + 1][None, :, None, None]
        out = 0.5 * (pre + pre.abs()) if theano_relu else torch.relu(pre)
        outs.append(out)
        h = out + P[3 * l + 2][None, :, None, None]
    pre = torch.nn.functional.conv2d(h, P[18].flip(2, 3)) + P[19][None, :, None, None]
    s = (0.5 * (pre + pre.abs()) + P[20][None, :, None, None]).detach()
    decs = []
    for d in range(4):
        g = s[:, 200 * d:200 * (d + 1)]
        for l in range(5, -1, -1):
            g, = torch.autograd.grad(outs[l], ins[l], grad_outputs=g, retain_graph=True)
        decs.append(g)
    m = torch.cat(decs, dim=1) + P[21][None, :, None, None]
    return (0.5 * (m + m.abs())).numpy()


def patch_input(F, tc=30, seed=0, B=2):
    rng = np.random.default_rng(seed)
    return (rng.random((B, 4, tc, F)) * rng.random((B, 1, tc, F)) ** 3 * 0.05).astype(np.float32)


@pytest.mark.parametrize("F,tc", [(257, 30), (300, 30), (300, 19), (257, 31)])
def test_oracle_matches_torch_autograd(F, tc):
    """F = 300 leaves columns uncovered by the next layer's windows in five of the six layers (their gradient is 0)"""
    params = s1.make_synthetic_params_1x1(seed=11)
    params[21][:] = np.random.default_rng(2).uniform(-1e-4, 1e-4, 16)      # both sides of the final rectifier
    x = patch_input(F, tc)
    ref = torch_1x1(params, x)
    got = s1.predict_1x1(params, x, all_decoders=True)
    assert got.shape == ref.shape == (2, 16, tc, F)
    assert np.abs(got - ref).max() <= 1e-12 * np.abs(ref).max()
    assert (ref[:, :4] > 0).mean() > 0.05 and (ref[:, :4] == 0).mean() > 0.05   # the masks see both sides of the ReLU
    if F == 300:
        w = [F] + s1.widths_1x1(F)
        assert sum((w[l] - 5) % 2 == 1 for l in range(6)) == 5


def test_rectifier_derivative_is_half_at_zero():
    """a silent input with a zeroed conv1 bias pair puts every conv1 pre-activation exactly at 0: both formulations give
    it the derivative 0.5 of 0.5*(x + |x|)"""
    params = s1.make_synthetic_params_1x1(seed=12)
    params[1][:] = 0
    params[2][:] = 0
    x = np.zeros((1, 4, 30, 257), dtype=np.float32)
    x[:, :, :, :100] = patch_input(100, seed=3, B=1)        # silent above bin 100
    pre1 = conv2d(x.astype(np.float64), params[0].astype(np.float64), (1, 2))
    assert (s1.gate_codes(pre1) == 1).mean() > 0.4
    ref = torch_1x1(params, x)
    got = s1.predict_1x1(params, x, all_decoders=True)
    assert np.abs(got - ref).max() <= 1e-12 * np.abs(ref).max()
    # the rule matters: with relu'(0) = 0 the output changes
    assert not np.allclose(torch_1x1(params, x, theano_relu=False), ref)


def test_dead_decoders_do_not_change_the_output():
    """decoders 2-4 and 1x1 channels 200..799 never reach the mask: perturbing them leaves channels 0..3 bit-identical"""
    params = s1.make_synthetic_params_1x1(seed=13)
    x = patch_input(257, seed=5)
    base = torch_1x1(params, x)[:, :4]
    pert = [p.copy() for p in params]
    rng = np.random.default_rng(1)
    for i in (18, 19, 20):
        pert[i][200:] = rng.uniform(-1, 1, size=pert[i][200:].shape).astype(np.float32)
    pert[21][4:] = 7.0
    assert np.array_equal(torch_1x1(pert, x)[:, :4], base)
    assert np.array_equal(s1.predict_1x1(pert, x), s1.predict_1x1(params, x))


def test_infer_arch_1x1_and_one_decoder():
    p22 = s1.make_synthetic_params_1x1(seed=1)
    assert models.infer_arch(p22) == ("bach10_score_1x1", 2049, 30)
    assert models.infer_arch(p22, 1025) == ("bach10_score_1x1", 1025, 30)
    assert models.infer_arch(p22, 300, 19) == ("bach10_score_1x1", 300, 19)
    with pytest.raises(ValueError, match="feat_size >= 253"):
        models.infer_arch(p22, 252)
    with pytest.raises(ValueError, match="time_context >= 19"):
        models.infer_arch(p22, 2049, 18)
    with pytest.raises(ValueError):
        models.check_1x1_geometry(513, 18)
    from oracle import nets
    p17 = nets.make_synthetic_params("bach10_score", 513)
    p11 = p17[:10] + [p17[16][:4]]
    assert models.infer_arch(p11) == ("bach10_score", 513, 30)
    assert models.infer_arch(p11, 513) == ("bach10_score", 513, 30)
    assert models.infer_arch(p17) == ("bach10_score", 513, 30)
    assert models.FAMILY_DEFAULTS["bach10_score_1x1"]["frameSize"] == 4096


def test_gate_code_layout():
    lay = models.gate_code_layout(2049, 30, 100)
    assert lay == [(100, 1023, 30), (100, 510, 50), (100, 253, 70), (100, 125, 100), (91, 61, 200), (82, 29, 200)]
    assert [w for _, w, _ in lay] == s1.widths_1x1(2049)


def test_arch_id_is_in_the_abi():
    import os
    from deepconvsep_b200 import _lib
    assert _lib.ARCH_IDS["bach10_score_1x1"] == 6
    h = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "dcs.h")).read()
    assert "DCS_ARCH_BACH10_SCORE_1X1 = 6" in h
