"""Theano front-end ELBO (SURVEY 8f-2, configs C1 / C4): the restated `cvae_layer` / `cvae1.f_encode_decode` plumbing is
pinned against vectors produced by executing the reference's own models.py (tests/golden/make_golden_theano_layer.py),
and bits/dim computed with the CUDA operator equals bits/dim computed with the oracle operator."""
import os

import numpy as np
import pytest
import torch

from iaf_b200 import elbo_theano as ET
from oracle.elbo_oracle import OracleIAFTheano

GOLD = os.path.join(os.path.dirname(__file__), "golden", "cvae_layer_down.npz")


@pytest.mark.parametrize("name", ["0_1", "1_0", "u0_1", "u1_0"])
def test_layer_matches_reference_models_py(name):
    """cvae_layer.up / down_q (models.py:133-328) for down_iaf2_nl and up_iaf2_nl ("u" cases) + diag prior, incl.
    conv.py's weight-normed convs with pad channel, stride-2 / depth-to-space resampling, nearest-neighbour skip paths,
    and the IAF step."""
    g = np.load(GOLD)
    pre = name + "/"
    w = {k[len(pre) + 2:]: torch.from_numpy(g[k]) for k in g.files if k.startswith(pre + "w/")}
    hps = dict(n_z=4, n_h1=8, n_h2=8, depths=[2, 2], depth_ar=1, nl="elu", kl_min=0.0, image_size=16,
               posterior="up_iaf2_nl" if name[0] == "u" else "down_iaf2_nl")
    ds = bool(g[pre + "downsample"])
    up_out, up_state = ET.layer_up(w, name, torch.from_numpy(g[pre + "up_in"]), hps, ds, torch.from_numpy(g[pre + "eps"]),
                                   OracleIAFTheano(w, hps))
    np.testing.assert_allclose(up_out.numpy(), g[pre + "up_out"], rtol=1e-10, atol=1e-10)
    out, kl_bc, kl_sum = ET.layer_down_q(w, name, torch.from_numpy(g[pre + "down_in"]), up_state,
                                         torch.from_numpy(g[pre + "eps"]), OracleIAFTheano(w, hps), hps, ds)
    np.testing.assert_allclose(out.numpy(), g[pre + "down_out"], rtol=1e-9, atol=1e-9)
    np.testing.assert_allclose(kl_bc.numpy(), g[pre + "kl"].sum(axis=(2, 3)), rtol=1e-9, atol=1e-9)
    np.testing.assert_allclose(kl_sum.numpy(), g[pre + "kl"].sum(axis=(1, 2, 3)), rtol=1e-9, atol=1e-9)


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


@pytest.mark.parametrize("posterior", ["down_iaf2_nl", "up_iaf2_nl"])
def test_forward_free_bits_and_shapes_cpu(posterior):
    hps = dict(n_z=4, n_h1=8, n_h2=8, depths=[2, 2], depth_ar=1, nl="elu", kl_min=0.25, image_size=16, posterior=posterior)
    w, x, noise = _setup(hps, 3, 5, torch.float64, "cpu")
    r = ET.forward(w, x, noise, OracleIAFTheano(w, hps), hps)
    assert r["cost"].shape == (3,) and np.isfinite(float(r["bits_per_dim"]))
    assert sorted(k for k in r if k.startswith("cost_z")) == ["cost_z000_000", "cost_z000_001", "cost_z001_000", "cost_z001_001"]
    # kl_min = 0: the objective is the plain per-sample sum (models.py:465-466); with free bits it is >= that
    hps0 = dict(hps, kl_min=0.0)
    r0 = ET.forward(w, x, noise, OracleIAFTheano(w, hps0), hps0)
    kl = sum(r0[k] for k in r0 if k.startswith("cost_z"))
    np.testing.assert_allclose(r0["cost"].numpy(), ((r0["cost_x"] + kl) / (3 * 16 * 16 * np.log(2.0))).numpy(), rtol=1e-12)
    assert float(r["bits_per_dim"]) >= float(r0["bits_per_dim"]) - 1e-12


@pytest.mark.gpu
@pytest.mark.parametrize("hps,B", [
    # C1 shapes (README.md:30): n_h 64, depth_ar 1, three levels -> 16x16, 8x8, 4x4 latents; tensor-core kernel
    (dict(n_z=32, n_h1=64, n_h2=64, depths=[2, 2, 2], depth_ar=1, nl="elu", kl_min=0.25, image_size=32), 4),
    # C4 shapes (README.md:55-58): n_h 160, depth_ar 2, two levels; tensor-core kernel
    (dict(n_z=32, n_h1=160, n_h2=160, depths=[2, 2], depth_ar=2, nl="elu", kl_min=0.25, image_size=32), 2),
    # cvae1's default nonlinearity (models.py:384) runs on the exact-fp32 kernel's run-time switch as well
    (dict(n_z=32, n_h1=64, n_h2=64, depths=[1, 1], depth_ar=1, nl="softplus", kl_min=0.0, image_size=32), 2),
    # the bottom-up placement (up_iaf2_nl, models.py:169-178): the bare step, KL assembled in the top-down pass
    (dict(n_z=32, n_h1=64, n_h2=64, depths=[2, 2], depth_ar=1, nl="elu", kl_min=0.25, image_size=32,
          posterior="up_iaf2_nl"), 4),
    (dict(n_z=32, n_h1=160, n_h2=160, depths=[1, 1], depth_ar=2, nl="elu", kl_min=0.0, image_size=32,
          posterior="up_iaf2_nl"), 2),
])
def test_bits_per_dim_parity_theano(hps, B):
    wg, xg, ng = _setup(hps, B, 9, torch.float32, "cuda")
    wc, xc, nc = _setup(hps, B, 9, torch.float64, "cpu")
    got = ET.forward(wg, xg, ng, ET.CudaIAF(wg, hps), hps)
    ref = ET.forward(wc, xc, nc, OracleIAFTheano(wc, hps), hps)
    rel = abs(float(got["bits_per_dim"]) - float(ref["bits_per_dim"])) / abs(float(ref["bits_per_dim"]))
    assert rel < 1e-4, (float(got["bits_per_dim"]), float(ref["bits_per_dim"]))
    for k in ref:
        if k.startswith("cost_z"):
            np.testing.assert_allclose(got[k].cpu().numpy(), ref[k].numpy(), rtol=2e-4, atol=1e-2)
    np.testing.assert_allclose(got["cost"].cpu().numpy(), ref["cost"].numpy(), rtol=1e-4)


@pytest.mark.parametrize("posterior", ["down_iaf2_nl", "up_iaf2_nl"])
def test_torch_oracle_block_equals_numpy_oracle_block_cpu(posterior):
    """The differentiable oracle block (TorchIAFTheano) reproduces the pinned numpy block on the same inputs."""
    from oracle.elbo_oracle import TorchIAFTheano
    hps = dict(n_z=4, n_h1=8, n_h2=8, depths=[1, 2], depth_ar=1, nl="elu", kl_min=0.25, image_size=16, posterior=posterior)
    w, x, noise = _setup(hps, 3, 5, torch.float64, "cpu")
    a = ET.forward(w, x, noise, OracleIAFTheano(w, hps), hps)
    b = ET.forward(w, x, noise, TorchIAFTheano(w, hps), hps)
    np.testing.assert_allclose(a["cost"].numpy(), b["cost"].numpy(), rtol=1e-12)


@pytest.mark.parametrize("posterior", ["down_iaf2_nl", "up_iaf2_nl"])
def test_theano_training_gradients_over_the_emulated_abi(posterior, monkeypatch):
    """d(cost)/d(every parameter) of the Theano front-end through elbo_theano.CudaIAFTrain -- the operator's autograd node
    (iaf_step_fwd_train / iaf_step_bwd_saved) -- against fp64 autograd through the oracle block.  Runs on the CPU by
    pointing the ctypes binding at the host-emulated library (tests/emu): the kernels' real source is executed, the
    python glue is the product's.  Test-only monkeypatching; the product refuses CPU tensors."""
    import contextlib
    import ctypes as C
    from iaf_b200 import _lib as L
    from iaf_b200 import ops
    from oracle import iaf_oracle as O
    from oracle.elbo_oracle import TorchIAFTheano
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

    hps = dict(n_z=4, n_h1=8, n_h2=8, depths=[1, 1], depth_ar=1, nl="elu", kl_min=0.0, image_size=8, posterior=posterior)
    w32, x, n32 = _setup(hps, 2, 7, torch.float32, "cpu")
    w64, _, n64 = _setup(hps, 2, 7, torch.float64, "cpu")
    for w in (w32, w64):
        for v in w.values():
            v.requires_grad_(True)
    got = ET.forward(w32, x, n32, ET.CudaIAFTrain(w32, hps, path="simt"), hps)
    ref = ET.forward(w64, x, n64, TorchIAFTheano(w64, hps), hps)
    np.testing.assert_allclose(got["cost"].detach().numpy(), ref["cost"].detach().numpy(), rtol=2e-5)
    got["cost"].sum().backward()
    ref["cost"].sum().backward()
    checked = 0
    for k in w64:
        g, r = w32[k].grad, w64[k].grad
        if r is None:
            assert g is None, k
            continue
        err = float((g.double() - r).abs().max()) / max(float(r.abs().max()), 1e-12)
        assert err < 5e-4, (k, err)   # fp32 torch plumbing around the operator; the operator alone is held to 2e-5
        if "_posterior_conv1_" in k and k.endswith("_w"):
            mask = O.theano_conv_ar_mask(g.shape[1] - 1, g.shape[0], (3, 3), "_out_" in k)
            assert bool((g.numpy()[mask == 0] == 0).all()), k   # the postup contract (ar.py:369-373)
            checked += 1
    assert checked >= 3 * len(hps["depths"])
