"""The two-step posterior ``posterior='down_iaf2_nl2'`` of the Theano front-end (models.py:93-98, 273-291): sample ->
step(posterior_conv1) -> step(posterior_conv2, flipmask=True) -> KL, both arw_logsd in log q.

* the restated cvae_layer with the fp64 oracle block against tests/golden/cvae_layer_nl2.npz, i.e. the reference's own
  models.py executed (tests/golden/make_golden_flipmask.py);
* the same layer through the CUDA operators' C ABI: on the CPU over the host-emulated library (tests/emu), on the GPU
  over libiaf_b200.so;
* bits/dim of small nl2 models, CUDA operators vs oracle, and the training gradients over the emulated ABI;
* posterior names the front-end does not implement are refused.
"""
import contextlib
import ctypes as C
import os

import numpy as np
import pytest
import torch

from iaf_b200 import elbo_theano as ET
from tests.flipmask_oracle import OracleIAFTheanoNL2, TorchIAFTheanoNL2, conv_ar_mask

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cvae_layer_nl2.npz")
HPS = dict(n_z=4, n_h1=8, n_h2=8, depths=[2, 2], depth_ar=1, nl="elu", kl_min=0.0, image_size=16,
           posterior="down_iaf2_nl2")


def _layer(name, iaf_cls, dtype, device):
    g = np.load(GOLD)
    pre = name + "/"
    T = lambda a: torch.from_numpy(np.asarray(a)).to(dtype).to(device)
    w = {k[len(pre) + 2:]: T(g[k]) for k in g.files if k.startswith(pre + "w/")}
    iaf = iaf_cls(w, HPS)
    ds = bool(g[pre + "downsample"])
    up_out, up_state = ET.layer_up(w, name, T(g[pre + "up_in"]), HPS, ds, None, iaf)
    out, kl_bc, kl_sum = ET.layer_down_q(w, name, T(g[pre + "down_in"]), up_state, T(g[pre + "eps"]), iaf, HPS, ds)
    got = dict(up_out=up_out, down_out=out, kl_bc=kl_bc, kl_sum=kl_sum)
    ref = dict(up_out=g[pre + "up_out"], down_out=g[pre + "down_out"], kl_bc=g[pre + "kl"].sum(axis=(2, 3)),
               kl_sum=g[pre + "kl"].sum(axis=(1, 2, 3)))
    return {k: v.detach().double().cpu().numpy() for k, v in got.items()}, ref


def _rel(a, ref):
    return float(np.abs(a - ref).max() / max(np.abs(ref).max(), 1.0))


@contextlib.contextmanager
def _emulated_abi(monkeypatch):
    """Point the ctypes binding at the host-emulated library (test only; the product refuses CPU tensors)."""
    from iaf_b200 import _lib as L
    from iaf_b200 import ops
    from tests.emu.harness import emu

    def check_input(t, name, shape=None):
        assert isinstance(t, torch.Tensor) and t.dtype == torch.float32
        if shape is not None:
            assert tuple(t.shape) == tuple(shape)
        return t.contiguous()
    monkeypatch.setattr(L, "lib", emu)
    monkeypatch.setattr(ops, "_check_input", check_input)
    monkeypatch.setattr(ops, "_stream", lambda device: C.c_void_p(0))
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    yield


@pytest.mark.parametrize("name", ["0_1", "1_0"])
def test_nl2_layer_matches_reference_models_py(name):
    got, ref = _layer(name, OracleIAFTheanoNL2, torch.float64, "cpu")
    for k in ref:
        np.testing.assert_allclose(got[k], ref[k], rtol=1e-9, atol=1e-9, err_msg=k)


@pytest.mark.parametrize("name", ["0_1", "1_0"])
def test_nl2_layer_through_the_emulated_abi(name, monkeypatch):
    with _emulated_abi(monkeypatch):
        got, ref = _layer(name, lambda w, hps: ET.CudaIAF(w, hps, path="simt"), torch.float32, "cpu")
    for k in ref:
        assert _rel(got[k], ref[k]) < 1e-4, k


def _setup(hps, B, seed, dtype, device):
    w = {k: torch.from_numpy(np.asarray(v)).to(dtype).to(device) for k, v in ET.make_params(hps, seed=seed).items()}
    rng = np.random.RandomState(seed + 1)
    S = hps["image_size"]
    x = torch.from_numpy(rng.randint(0, 256, size=(B, 3, S, S)).astype(np.uint8)).to(device)
    noise = {}
    for i in range(len(hps["depths"])):
        s = S // 2 ** (i + 1)
        for j in range(hps["depths"][i]):
            noise[(i, j)] = torch.from_numpy(rng.randn(B, hps["n_z"], s, s)).to(dtype).to(device)
    return w, x, noise


def test_nl2_parameters_and_unknown_posteriors():
    w = ET.make_params(dict(HPS, depths=[1, 1]), seed=0)
    assert "0_0_posterior_conv2_0_w" in w and "1_0_posterior_conv2_out_1_w" in w
    assert not any("_posterior_conv2_" in k for k in ET.make_params(dict(HPS, posterior="down_iaf2_nl"), seed=0))
    for posterior in ("down_iaf2_deep", "up_iaf1_nl"):
        hps = dict(HPS, posterior=posterior)
        with pytest.raises(ValueError):
            ET.make_params(hps, seed=0)
        wd, x, noise = _setup(dict(HPS, posterior="down_iaf2_nl"), 2, 3, torch.float64, "cpu")
        with pytest.raises(ValueError):
            ET.forward(wd, x, noise, OracleIAFTheanoNL2(wd, hps), hps)


def test_nl2_second_step_matters_cpu():
    """The nl2 objective differs from the one-step objective on the same conv1 weights (the second step runs)."""
    w, x, noise = _setup(HPS, 2, 5, torch.float64, "cpu")
    a = ET.forward(w, x, noise, OracleIAFTheanoNL2(w, HPS), HPS)
    h1 = dict(HPS, posterior="down_iaf2_nl")
    b = ET.forward(w, x, noise, OracleIAFTheanoNL2(w, h1), h1)
    assert abs(float(a["bits_per_dim"]) - float(b["bits_per_dim"])) > 1e-6
    c = ET.forward(w, x, noise, TorchIAFTheanoNL2(w, HPS), HPS)
    np.testing.assert_allclose(a["cost"].numpy(), c["cost"].numpy(), rtol=1e-12)


def test_nl2_training_gradients_over_the_emulated_abi(monkeypatch):
    """d(cost)/d(every parameter) through CudaIAFTrain (two operator autograd nodes per layer, the second flipped)
    against fp64 autograd through the oracle block."""
    hps = dict(HPS, depths=[1, 1], image_size=8)
    w32, x, n32 = _setup(hps, 2, 7, torch.float32, "cpu")
    w64, _, n64 = _setup(hps, 2, 7, torch.float64, "cpu")
    for w in (w32, w64):
        for v in w.values():
            v.requires_grad_(True)
    with _emulated_abi(monkeypatch):
        got = ET.forward(w32, x, n32, ET.CudaIAFTrain(w32, hps, path="simt"), hps)
        got["cost"].sum().backward()
    ref = ET.forward(w64, x, n64, TorchIAFTheanoNL2(w64, hps), hps)
    np.testing.assert_allclose(got["cost"].detach().numpy(), ref["cost"].detach().numpy(), rtol=2e-5)
    ref["cost"].sum().backward()
    checked = 0
    for k in w64:
        g, r = w32[k].grad, w64[k].grad
        if r is None:
            assert g is None, k
            continue
        err = float((g.double() - r).abs().max()) / max(float(r.abs().max()), 1e-12)
        assert err < 5e-4, (k, err)   # fp32 torch plumbing around the operator
        if "_posterior_conv2_" in k and k.endswith("_w"):
            mask = conv_ar_mask(g.shape[1] - 1, g.shape[0], "_out_" in k, True)
            assert bool((g.numpy()[mask == 0] == 0).all()), k   # masked taps: exactly zero (ar.py:369-373)
            checked += 1
    assert checked >= 3 * len(hps["depths"])


@pytest.mark.gpu
def test_nl2_training_gradients_on_the_tensor_cores():
    """d(cost)/d(every parameter) through CudaIAFTrain on the GPU, at a shape where both convs of every layer run the
    tensor-core forward and backward (the second one flipped), against fp64 autograd through the oracle block."""
    hps = dict(HPS, n_z=16, n_h1=32, n_h2=32, depths=[1, 1], depth_ar=1, image_size=16)
    w32, x, n32 = _setup(hps, 2, 7, torch.float32, "cuda")
    w64, _, n64 = _setup(hps, 2, 7, torch.float64, "cpu")
    for w in (w32, w64):
        for v in w.values():
            v.requires_grad_(True)
    iaf = ET.CudaIAFTrain(w32, hps)
    got = ET.forward(w32, x, n32, iaf, hps)
    got["cost"].sum().backward()
    assert sorted(iaf.ops) == [("0_0", 1), ("0_0", 2), ("1_0", 1), ("1_0", 2)]
    for (name, conv), op in iaf.ops.items():
        s = hps["image_size"] // 2 ** (int(name[0]) + 1)
        assert op.flipmask == (conv == 2), (name, conv)
        assert op.path_used(s, s, "cuda:0", "step") == "tc", (name, conv)
        assert op.backward_path(s, s, "cuda:0") == "tc", (name, conv)
    ref = ET.forward(w64, x.cpu(), n64, TorchIAFTheanoNL2(w64, hps), hps)
    np.testing.assert_allclose(got["cost"].detach().cpu().numpy(), ref["cost"].detach().numpy(), rtol=2e-5)
    ref["cost"].sum().backward()
    checked = 0
    for k in w64:
        g, r = w32[k].grad, w64[k].grad
        if r is None:
            assert g is None, k
            continue
        g = g.cpu()
        err = float((g.double() - r).abs().max()) / max(float(r.abs().max()), 1e-12)
        assert err < 5e-4, (k, err)   # fp32 torch plumbing around the operator
        if "_posterior_conv2_" in k and k.endswith("_w"):
            mask = conv_ar_mask(g.shape[1] - 1, g.shape[0], "_out_" in k, True)
            assert bool((g.numpy()[mask == 0] == 0).all()), k   # masked taps: exactly zero (ar.py:369-373)
            checked += 1
    assert checked == 3 * len(hps["depths"])


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["0_1", "1_0"])
def test_nl2_layer_on_the_gpu(name):
    got, ref = _layer(name, ET.CudaIAF, torch.float32, "cuda")
    for k in ref:
        assert _rel(got[k], ref[k]) < 1e-4, k


@pytest.mark.gpu
@pytest.mark.parametrize("hps,B", [
    # C1 shapes (n_h 64, depth_ar 1): the tensor-core one-launch step for both convs
    (dict(n_z=32, n_h1=64, n_h2=64, depths=[2, 2], depth_ar=1, nl="elu", kl_min=0.25, image_size=32,
          posterior="down_iaf2_nl2"), 4),
    # n_h 160, depth_ar 2: the per-stage tensor-core kernels
    (dict(n_z=32, n_h1=160, n_h2=160, depths=[1, 1], depth_ar=2, nl="elu", kl_min=0.0, image_size=32,
          posterior="down_iaf2_nl2"), 2),
])
def test_nl2_bits_per_dim_parity(hps, B):
    wg, xg, ng = _setup(hps, B, 9, torch.float32, "cuda")
    wc, xc, nc = _setup(hps, B, 9, torch.float64, "cpu")
    iaf = ET.CudaIAF(wg, hps)
    got = ET.forward(wg, xg, ng, iaf, hps)
    ref = ET.forward(wc, xc, nc, OracleIAFTheanoNL2(wc, hps), hps)
    assert sorted(n for n, conv in iaf.ops if conv == 2) == sorted(n for n, conv in iaf.ops if conv == 1)
    assert all(op.flipmask == (conv == 2) and op.path_used(8, 8, "cuda:0", "step") == "tc" for (n, conv), op in iaf.ops.items())
    rel = abs(float(got["bits_per_dim"]) - float(ref["bits_per_dim"])) / abs(float(ref["bits_per_dim"]))
    assert rel < 1e-4, (float(got["bits_per_dim"]), float(ref["bits_per_dim"]))
    for k in ref:
        if k.startswith("cost_z"):
            np.testing.assert_allclose(got[k].cpu().numpy(), ref[k].numpy(), rtol=2e-4, atol=1e-2)
    np.testing.assert_allclose(got["cost"].cpu().numpy(), ref["cost"].numpy(), rtol=1e-4)
