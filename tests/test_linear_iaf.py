"""The linear IAF posteriors ``down_iaf2`` / ``up_iaf2`` (models.py:55-56, 79-82, 152-161, 246-259): one masked conv
``ar.conv2d(n_z, 2 n_z)`` whose interleaved rows are the two heads, run by the operator as a stack without hidden
layers.  On the CPU:

* the fp64 oracle (tests/linear_oracle.py) against tests/golden/cvae_layer_linear.npz, i.e. the reference's own
  models.py executed (tests/golden/make_golden_linear.py), both posteriors, priors diag and made, with and without
  downsampling, and made with depth_ar = 0;
* the mask of ``ar.conv2d(n_z, 2 n_z)``, de-interleaved, is the mask of the depth-0 stack's heads;
* the Theano model through ``CudaIAF(path="simt")`` over the emulated ABI against the fixture, the training gradients
  of ``CudaIAFTrain`` against fp64 autograd (masked taps exactly zero), and ``decode``;
* every other unsupported posterior is still refused.
"""
import os

import numpy as np
import pytest
import torch

from iaf_b200 import elbo_theano as ET
from iaf_b200 import masks
from iaf_b200.weights import deinterleave_heads
from oracle import iaf_oracle as O
from tests import flipmask_oracle as FO
from tests import linear_oracle as LO
from tests.emu.harness import EmuOperator
from tests.test_made_prior import _emulated_abi, _rel, _setup
from tests.test_made_sample import _emulated_abi as _emulated_abi_with_inverse

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cvae_layer_linear.npz")
HPS = dict(n_z=4, n_h1=8, n_h2=8, depths=[2, 2], nl="elu", kl_min=0.0, image_size=16)
CASES = ([(p, pr, 1, n) for p in ET.LINEAR for pr in ET.PRIORS for n in ("0_1", "1_0")] +
         [("down_iaf2", "made", 0, "0_1")])


def _layer(posterior, prior, depth_ar, name, iaf_cls, dtype, device):
    g = np.load(GOLD)
    pre = "%s:%s:%d:%s/" % (posterior, prior, depth_ar, name)
    hps = dict(HPS, posterior=posterior, prior=prior, depth_ar=depth_ar)
    T = lambda a: torch.from_numpy(np.asarray(a)).to(dtype).to(device)
    w = {k[len(pre) + 2:]: T(g[k]) for k in g.files if k.startswith(pre + "w/")}
    iaf = iaf_cls(w, hps)
    ds = bool(g[pre + "downsample"])
    eps = T(g[pre + "eps"])
    up_out, up_state = ET.layer_up(w, name, T(g[pre + "up_in"]), hps, ds, eps, iaf)
    out, kl_bc, kl_sum = ET.layer_down_q(w, name, T(g[pre + "down_in"]), up_state, eps, iaf, hps, ds)
    got = dict(up_out=up_out, down_out=out, kl_bc=kl_bc, kl_sum=kl_sum)
    ref = dict(up_out=g[pre + "up_out"], down_out=g[pre + "down_out"], kl_bc=g[pre + "kl"].sum(axis=(2, 3)),
               kl_sum=g[pre + "kl"].sum(axis=(1, 2, 3)))
    return {k: v.detach().double().cpu().numpy() for k, v in got.items()}, ref, w, iaf


@pytest.mark.parametrize("posterior,prior,depth_ar,name", CASES)
def test_linear_layer_oracle_matches_reference_models_py(posterior, prior, depth_ar, name):
    for cls in (LO.OracleIAFTheanoLinear, LO.TorchIAFTheanoLinear):
        got, ref, _, _ = _layer(posterior, prior, depth_ar, name, cls, torch.float64, "cpu")
        for k in ref:
            np.testing.assert_allclose(got[k], ref[k], rtol=1e-9, atol=1e-9, err_msg=k)


def test_linear_fixture_has_the_reference_parameter_layout():
    g = np.load(GOLD)
    nz, nh2 = HPS["n_z"], HPS["n_h2"]
    for posterior, prior, depth_ar, name in CASES:
        pre = "%s:%s:%d:%s/w/%s_" % (posterior, prior, depth_ar, name, name)
        assert g[pre + "posterior_conv1_w"].shape == (2 * nz, nz + 1, 3, 3)
        assert not any(k.startswith(pre + "posterior_conv1_") and k[len(pre + "posterior_conv1_")].isdigit()
                       for k in g.files)
        ds = "2" if name == "1_0" else "1"
        assert g[pre + "up_conv1_" + ds + "_w"].shape[0] == nh2 + 2 * nz                       # no up context
        assert g[pre + "up_conv2_w"].shape[1] == (nh2 + nz if posterior == "up_iaf2" else nh2) + 1
        n_prior = 2 * nh2 if prior == "made" else nh2 + 2 * nz
        assert g[pre + "down_conv1_w"].shape[0] == n_prior + (2 * nz if posterior == "down_iaf2" else 0)
        assert (pre + "prior_conv1_out_1_w" in g.files) == (prior == "made")
        assert (pre + "prior_conv1_0_w" in g.files) == (prior == "made" and depth_ar > 0)


@pytest.mark.parametrize("n_z", [1, 4, 16, 48])
def test_deinterleaved_mask_is_the_depth0_heads_mask(n_z):
    """ar.py:241-281: rows 2i, 2i + 1 of ar.conv2d(n_z, 2 n_z) (zerodiagonal, k = 2) see the centre of inputs < i and never
    the pad channel's; that is row i of a head ar.conv2d(n_z, n_z, zerodiagonal=True), the rule iaf_tap_rule applies to
    the heads of a stack (the host restatement iaf_b200.masks is pinned to the device's by tests/test_host_cpu.py).
    l2normalize's extra zeroing of rows [0, 2) at the centre is a no-op: those taps are masked already."""
    full = O.theano_conv_ar_mask(n_z, 2 * n_z, zerodiagonal=True, pad_channel=True)
    head = masks.theano_conv_ar_mask(n_z, n_z, zerodiagonal=True)
    for k in range(2):
        assert np.array_equal(full[k::2], head)
    assert not full[:FO.zero_rows(n_z, 2 * n_z), :, 1, 1].any()


def _linear_params(n_z, seed):
    rng = np.random.RandomState(seed)
    # unmasked weights: any tap the kernel wrongly keeps or drops shows in its outputs
    return dict(w=(0.3 * rng.randn(2 * n_z, n_z + 1, 3, 3)).astype(np.float32),
                s=rng.uniform(-0.2, 0.2, size=(2 * n_z,)).astype(np.float32),
                b=(0.1 * rng.randn(2 * n_z)).astype(np.float32))


@pytest.mark.parametrize("n_z,H,W,B", [(4, 5, 7, 2), (16, 4, 4, 2), (8, 1, 1, 3)])
def test_emulated_depth0_step_with_deinterleaved_rows_is_the_linear_step(n_z, H, W, B):
    """The SIMT kernels under host emulation, a depth-0 plan fed the de-interleaved rows: forward against the reference
    form (conv, then out[:, ::2] / out[:, 1::2]), backward against fp64 autograd with the gradients interleaved back."""
    p = _linear_params(n_z, 3)
    op = EmuOperator("theano", n_z, [], [n_z, n_z], H, W).set_weights(deinterleave_heads(p["w"], p["s"], p["b"]))
    z = np.random.RandomState(4).randn(B, n_z, H, W).astype(np.float32)
    z_ref, ls_ref = LO.step(z.astype(np.float64), {k: v.astype(np.float64) for k, v in p.items()})
    zo, ls, ld = op.step(z, None)
    assert _rel(zo, z_ref) < 1e-5 and _rel(ls, ls_ref) < 1e-5 and _rel(ld, -ls_ref.sum(axis=(1, 2, 3))) < 1e-5
    tp = {k: torch.from_numpy(v).double().requires_grad_(True) for k, v in p.items()}
    zt = torch.from_numpy(z).double().requires_grad_(True)
    rng = np.random.RandomState(5)
    g_zo, g_ls = rng.randn(*z.shape).astype(np.float32), rng.randn(*z.shape).astype(np.float32)
    zn, als = LO.t_step(zt, tp)
    ((zn * torch.from_numpy(g_zo)).sum() + (als * torch.from_numpy(g_ls)).sum()).backward()
    g_z, g_ctx, gw, gs, gb = op.step_bwd(z, None, g_zo, g_ls)
    assert g_ctx is None and _rel(g_z, zt.grad) < 2e-5
    for got, k in zip((gw, gs, gb), "wsb"):
        full = np.empty_like(p[k])
        full[0::2], full[1::2] = got
        assert _rel(full, tp[k].grad) < 2e-5, k
        if k == "w":
            mask = O.theano_conv_ar_mask(n_z, 2 * n_z, zerodiagonal=True, pad_channel=True)
            assert (full[mask == 0] == 0).all()


@pytest.mark.parametrize("posterior,prior,depth_ar,name", CASES)
def test_linear_layer_through_the_emulated_abi(posterior, prior, depth_ar, name, monkeypatch):
    with _emulated_abi(monkeypatch):
        got, ref, _, iaf = _layer(posterior, prior, depth_ar, name, lambda w, hps: ET.CudaIAF(w, hps, path="simt"),
                                  torch.float32, "cpu")
        op = iaf.ops[(name, 1)]
        assert op.hidden == [] and op.heads == [4, 4]
        if prior == "made":
            assert iaf.prior_ops[name].hidden == depth_ar * [HPS["n_h2"]]
    for k in ref:
        assert _rel(got[k], ref[k]) < 1e-4, k


@pytest.mark.parametrize("posterior", ET.LINEAR)
@pytest.mark.parametrize("prior", ET.PRIORS)
def test_linear_elbo_and_training_gradients_over_the_emulated_abi(posterior, prior, monkeypatch):
    """cvae1 with a linear posterior: cost against the fp64 oracle, and d(cost)/d(every parameter) through CudaIAFTrain
    against fp64 autograd, the posterior conv's gradient interleaved with masked taps exactly zero (ar.py:369-373)."""
    hps = dict(HPS, depths=[1, 1], image_size=8, posterior=posterior, prior=prior, depth_ar=1)
    w32, x, n32 = _setup(hps, 2, 7, torch.float32, "cpu")
    w64, _, n64 = _setup(hps, 2, 7, torch.float64, "cpu")
    ref0 = ET.forward(w64, x, n64, LO.OracleIAFTheanoLinear(w64, hps), hps)
    for w in (w32, w64):
        for v in w.values():
            v.requires_grad_(True)
    with _emulated_abi(monkeypatch):
        iaf = ET.CudaIAFTrain(w32, hps, path="simt")
        got = ET.forward(w32, x, n32, iaf, hps)
        got["cost"].sum().backward()
    ref = ET.forward(w64, x, n64, LO.TorchIAFTheanoLinear(w64, hps), hps)
    np.testing.assert_allclose(ref["cost"].detach().numpy(), ref0["cost"].numpy(), rtol=1e-12)
    np.testing.assert_allclose(got["cost"].detach().numpy(), ref["cost"].detach().numpy(), rtol=2e-5)
    ref["cost"].sum().backward()
    checked = 0
    for k in w64:
        g, r = w32[k].grad, w64[k].grad
        assert (g is None) == (r is None), k
        if r is None:
            continue
        err = float((g.double() - r).abs().max()) / max(float(r.abs().max()), 1e-12)
        assert err < 5e-4, (k, err)   # fp32 torch plumbing around the operators
        if k.endswith("_posterior_conv1_w"):
            mask = O.theano_conv_ar_mask(hps["n_z"], 2 * hps["n_z"], zerodiagonal=True, pad_channel=True)
            assert bool((g.numpy()[mask == 0] == 0).all()), k
            assert bool((g.numpy()[mask == 1] != 0).all()), k
            checked += 1
    assert checked == len(hps["depths"])


@pytest.mark.parametrize("posterior", ET.LINEAR)
@pytest.mark.parametrize("prior", ET.PRIORS)
def test_decode_runs_for_the_linear_posteriors(posterior, prior, monkeypatch):
    """decode / layer_down_p depend only on down_conv1's prior channels: the same as for the other posteriors."""
    hps = dict(HPS, depths=[1, 1], image_size=8, posterior=posterior, prior=prior, depth_ar=1)
    w, _, noise = _setup(hps, 2, 9, torch.float32, "cpu")
    with _emulated_abi_with_inverse(monkeypatch):
        img = ET.decode(w, noise, ET.CudaIAF(w, hps, path="simt"), hps)
    assert img.shape == (2, 3, 8, 8) and img.dtype == torch.uint8
    if prior == "diag":   # the diagonal prior's sample needs no operator: the torch restatement gives the same image
        assert torch.equal(img, ET.decode(w, noise, None, hps))


def test_other_posteriors_are_still_refused():
    for posterior in ("down_iaf1", "up_iaf1", "down_iaf1_nl", "up_iaf1_nl", "down_iaf2_deep", "down_iaf1_deep",
                      "down_diag", "up_diag", "down_tim", "down_bernoulli", "iaf2"):
        hps = dict(HPS, posterior=posterior, prior="diag", depth_ar=1)
        with pytest.raises(ValueError):
            ET.make_params(hps, seed=0)
        w, x, noise = _setup(dict(hps, posterior="down_iaf2"), 2, 3, torch.float64, "cpu")
        with pytest.raises(ValueError):
            ET.forward(w, x, noise, LO.OracleIAFTheanoLinear(w, hps), hps)
