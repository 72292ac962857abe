"""bits/dim parity (BASELINE.json metric, SURVEY 8f-2): the restated ELBO forward evaluated with the CUDA
operator equals the same forward evaluated with the oracle operator on identical weights, inputs and noise."""
import numpy as np
import pytest
import torch

from iaf_b200 import elbo
from oracle import iaf_oracle as O
from oracle.elbo_oracle import OracleIAF


def _setup(hps, B, seed, dtype, device):
    p = elbo.make_params(hps, seed=seed)
    params = {k: torch.from_numpy(np.asarray(v)).to(dtype).to(device) for k, v in p.items()}
    rng = np.random.RandomState(seed + 1)
    x = torch.from_numpy(rng.randint(0, 256, size=(B, 3, hps["image_size"], hps["image_size"])).astype(np.uint8)).to(device)
    noise = {}
    for i in range(hps["depth"]):
        size = hps["image_size"] // 2 ** (i + 1)
        for j in range(hps["num_blocks"]):
            noise[(i, j)] = torch.from_numpy(rng.randn(B, hps["z_size"], size, size).astype(np.float32)).to(dtype).to(device)
    return params, x, noise


def test_plumbing_against_oracle_primitives_cpu():
    hps = dict(z_size=4, h_size=8, depth=2, num_blocks=2, kl_min=0.25, image_size=16)
    params, x, noise = _setup(hps, 2, 3, torch.float64, "cpu")
    # conv2d (stride 1) equals the oracle's weight-normed cross-correlation with an all-ones mask
    h = torch.randn(2, 8, 8, 8, dtype=torch.float64)
    got = elbo.conv2d(params, "IAF_0_0/up_conv3", h).numpy()
    V, g, b = (params["IAF_0_0/up_conv3/" + k].numpy() for k in "Vgb")
    w = O.tf_effective_weight(V, g, np.ones_like(V))
    np.testing.assert_allclose(got, O.xcorr2d_same(h.numpy(), w) + b.reshape(1, -1, 1, 1), atol=1e-12)
    # deconv2d is the adjoint of the SAME stride-2 conv with the same filter: <conv(a), c> == <a, deconv(c)>
    pz = {"t/V": params["IAF_1_0/down_deconv2/V"], "t/g": torch.zeros(8, dtype=torch.float64), "t/b": torch.zeros(8, dtype=torch.float64)}
    a = torch.randn(1, 8, 8, 8, dtype=torch.float64)
    c = torch.randn(1, 12, 4, 4, dtype=torch.float64)
    Vn = pz["t/V"] * torch.rsqrt((pz["t/V"] ** 2).sum(dim=(0, 1, 2), keepdim=True))
    fwd = torch.nn.functional.conv2d(torch.nn.functional.pad(a, (0, 1, 0, 1)), Vn.permute(3, 2, 0, 1), stride=2)
    assert abs(float((fwd * c).sum()) - float((a * elbo.deconv2d(pz, "t", c)).sum())) < 1e-9
    out = elbo.forward(params, x, noise, OracleIAF(params, hps), hps)
    assert np.isfinite(float(out["bits_per_dim"])) and out["kl_cost"].shape == (2,)
    # free bits: kl_obj >= kl_cost can differ, and the objective uses the local batch mean (tf_train.py:77-83)
    assert float(out["obj"]) != float((out["kl_cost"] - out["log_pxz"]).sum())


@pytest.mark.gpu
@pytest.mark.parametrize("hps,B", [
    (dict(z_size=32, h_size=64, depth=2, num_blocks=2, kl_min=0.25, image_size=32), 4),   # tensor-core path, two levels
    (dict(z_size=32, h_size=160, depth=1, num_blocks=3, kl_min=0.1, image_size=32), 2),   # C3 shapes: tensor-core path
])
def test_bits_per_dim_parity(hps, B):
    pg, xg, ng = _setup(hps, B, 7, torch.float32, "cuda")
    pc, xc, nc = _setup(hps, B, 7, torch.float64, "cpu")
    got = elbo.forward(pg, xg, ng, elbo.CudaIAF(pg, hps), hps)
    ref = elbo.forward(pc, xc, nc, OracleIAF(pc, hps), hps)
    rel = abs(float(got["bits_per_dim"]) - float(ref["bits_per_dim"])) / abs(float(ref["bits_per_dim"]))
    assert rel < 1e-4, (float(got["bits_per_dim"]), float(ref["bits_per_dim"]))
    np.testing.assert_allclose(got["kl_cost"].cpu().numpy(), ref["kl_cost"].numpy(), rtol=2e-4, atol=1e-2)
    np.testing.assert_allclose(float(got["obj"]), float(ref["obj"]), rtol=1e-4)


def _dp_worker(rank, world, port, q):
    import os
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    hps = dict(z_size=4, h_size=8, depth=1, num_blocks=2, kl_min=0.0, image_size=8)
    params, x, noise = _setup(hps, 4, 11, torch.float64, "cpu")
    bpd = elbo.sharded_bits_per_dim(params, x, noise, OracleIAF(params, hps), hps)
    q.put((rank, float(bpd)))
    dist.destroy_process_group()


def test_sharded_elbo_equals_single_process_gloo_world2():
    """C5's structure on CPU: 2 ranks, batch sharded, one all-reduce of the scalar (tf_train.py:126-142)."""
    import os
    import torch.multiprocessing as mp
    hps = dict(z_size=4, h_size=8, depth=1, num_blocks=2, kl_min=0.0, image_size=8)
    params, x, noise = _setup(hps, 4, 11, torch.float64, "cpu")
    single = float(elbo.forward(params, x, noise, OracleIAF(params, hps), hps)["bits_per_dim"])
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 31500 + os.getpid() % 2000
    ps = [ctx.Process(target=_dp_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in ps:
        p.start()
    res = sorted(q.get(timeout=180) for _ in ps)
    for p in ps:
        p.join(timeout=60)
        assert p.exitcode == 0
    for _, v in res:
        assert abs(v - single) < 1e-12 * max(1.0, abs(single))


def test_torch_oracle_layer_equals_numpy_oracle_layer_cpu():
    """The differentiable oracle block (TorchIAF) reproduces the pinned numpy oracle block on the same inputs."""
    from oracle.elbo_oracle import TorchIAF
    hps = dict(z_size=4, h_size=8, depth=1, num_blocks=2, kl_min=0.25, image_size=8)
    params, x, noise = _setup(hps, 3, 5, torch.float64, "cpu")
    a = elbo.forward(params, x, noise, OracleIAF(params, hps), hps)
    b = elbo.forward(params, x, noise, TorchIAF(params, hps), hps)
    assert abs(float(a["bits_per_dim"]) - float(b["bits_per_dim"])) < 1e-12
    np.testing.assert_allclose(a["kl_obj"].numpy(), b["kl_obj"].numpy(), rtol=1e-12)


@pytest.mark.gpu
@pytest.mark.parametrize("hps,B", [
    (dict(z_size=32, h_size=64, depth=2, num_blocks=1, kl_min=0.25, image_size=32), 3),
    (dict(z_size=8, h_size=16, depth=1, num_blocks=2, kl_min=0.0, image_size=16), 4),
])
def test_training_objective_gradient_parity(hps, B):
    """SURVEY 8f-4: d(objective)/d(every parameter) through the CUDA operator's autograd node (iaf_step_fwd /
    iaf_step_bwd) equals torch autograd through the oracle block, in fp64 on the CPU."""
    from oracle.elbo_oracle import TorchIAF
    pg, xg, ng = _setup(hps, B, 9, torch.float32, "cuda")
    pc, xc, nc = _setup(hps, B, 9, torch.float64, "cpu")
    for p in (pg, pc):
        for v in p.values():
            v.requires_grad_(True)
    got = elbo.forward(pg, xg, ng, elbo.CudaIAFTrain(pg, hps), hps)
    ref = elbo.forward(pc, xc, nc, TorchIAF(pc, hps), hps)
    np.testing.assert_allclose(float(got["obj"]), float(ref["obj"]), rtol=1e-4)
    got["obj"].backward()
    ref["obj"].backward()
    for k in pc:
        g, r = pg[k].grad, pc[k].grad
        if r is None:   # e.g. the last up-layer's up_conv3: its output is discarded (tf_train.py:186-190)
            assert g is None, k
            continue
        assert g is not None, k
        err = float((g.double().cpu() - r).abs().max()) / max(float(r.abs().max()), 1e-12)
        assert err < 2e-3, (k, err)   # fp32 plumbing (cuDNN convs) dominates; the operator's own gradients are
        #                               checked to 1e-4 in tests/test_gpu_parity.py
        if "ar_multiconv2d" in k and k.endswith("/V"):
            zd = "layer_out" in k
            mask = O.get_conv_ar_mask(3, 3, g.shape[2], g.shape[3], zd)
            assert bool((g.cpu().numpy()[mask == 0] == 0).all())   # the postup contract (ar.py:369-373)


def _dp_grad_worker(rank, world, port, q):
    import os
    import torch.distributed as dist
    from iaf_b200.parallel import allreduce_grads, shard_range
    from oracle.elbo_oracle import TorchIAF
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    hps = dict(z_size=4, h_size=8, depth=1, num_blocks=2, kl_min=0.0, image_size=8)
    params, x, noise = _setup(hps, 4, 11, torch.float64, "cpu")
    for v in params.values():
        v.requires_grad_(True)
    lo, hi = shard_range(4, rank, world)
    out = elbo.forward(params, x[lo:hi], {k: v[lo:hi] for k, v in noise.items()}, TorchIAF(params, hps), hps)
    out["obj"].backward()
    allreduce_grads(params, average=False)
    q.put((rank, {k: v.grad.numpy().copy() for k, v in params.items() if v.grad is not None}))
    dist.destroy_process_group()


def test_sharded_gradients_allreduce_equals_single_process_gloo_world2():
    """Data-parallel training step on CPU (tf_train.py:126-147, common.py:78-115): with kl_min = 0 the objective is a
    sum over samples, so the summed gradients of two half-batch ranks equal the full-batch gradient."""
    import os
    import torch.multiprocessing as mp
    from oracle.elbo_oracle import TorchIAF
    hps = dict(z_size=4, h_size=8, depth=1, num_blocks=2, kl_min=0.0, image_size=8)
    params, x, noise = _setup(hps, 4, 11, torch.float64, "cpu")
    for v in params.values():
        v.requires_grad_(True)
    elbo.forward(params, x, noise, TorchIAF(params, hps), hps)["obj"].backward()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 33500 + os.getpid() % 2000
    ps = [ctx.Process(target=_dp_grad_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in ps:
        p.start()
    res = sorted((q.get(timeout=180) for _ in ps), key=lambda t: t[0])
    for p in ps:
        p.join(timeout=60)
        assert p.exitcode == 0
    for _, grads in res:
        for k, g in grads.items():
            np.testing.assert_allclose(g, params[k].grad.numpy(), rtol=1e-9, atol=1e-12)


@pytest.mark.parametrize("fused", [False, True])
def test_tf_training_gradients_over_the_emulated_abi(monkeypatch, fused):
    """CPU twin of test_training_objective_gradient_parity: elbo.CudaIAFTrain (autograd node -> iaf_step_fwd_train /
    iaf_step_bwd_saved) with the ctypes binding pointed at the host-emulated library (tests/emu), against fp64 autograd
    through the oracle block.  Test-only monkeypatching; the product refuses CPU tensors."""
    import contextlib
    import ctypes as C
    from iaf_b200 import _lib as L
    from iaf_b200 import ops
    from oracle.elbo_oracle import TorchIAF
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

    hps = dict(z_size=4, h_size=8, depth=1, num_blocks=2, kl_min=0.25, image_size=8)
    p32, x, n32 = _setup(hps, 3, 9, torch.float32, "cpu")
    p64, _, n64 = _setup(hps, 3, 9, torch.float64, "cpu")
    for p in (p32, p64):
        for v in p.values():
            v.requires_grad_(True)
    got = elbo.forward(p32, x, n32, elbo.CudaIAFTrain(p32, hps, path="simt", fused=fused), hps)
    ref = elbo.forward(p64, x, n64, TorchIAF(p64, hps), hps)
    np.testing.assert_allclose(float(got["obj"].detach()), float(ref["obj"].detach()), rtol=2e-5)
    got["obj"].backward()
    ref["obj"].backward()
    for k in p64:
        g, r = p32[k].grad, p64[k].grad
        if r is None:
            assert g is None, k
            continue
        err = float((g.double() - r).abs().max()) / max(float(r.abs().max()), 1e-12)
        assert err < 5e-4, (k, err)
        if "ar_multiconv2d" in k and k.endswith("/V"):
            mask = O.get_conv_ar_mask(3, 3, g.shape[2], g.shape[3], "layer_out" in k)
            assert bool((g.numpy()[mask == 0] == 0).all()), k


def test_forward_against_reference_executed_cvae1_forward():
    """elbo.forward (the restatement used for every bits/dim parity number) against what the reference's OWN
    `CVAE1._forward` (tf_train.py:161-219, with IAFLayer.up/down, conv2d/deconv2d/ar_multiconv2d, discretized_logistic,
    compute_lowerbound executed from the reference source by tests/golden/make_golden_cvae1.py) produced on the same
    parameters, image and noise: the objective, the loss and bits/dim."""
    import os
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "cvae1_forward.npz"))
    for tag in ("", "kl40_"):    # free bits idle / binding (tf_train.py:77-83)
        hps = dict(z_size=4, h_size=8, depth=2, num_blocks=2, kl_min=float(g[tag + "kl_min"]), image_size=16)
        params = {k: torch.from_numpy(np.asarray(v, dtype=np.float64)) for k, v in elbo.make_params(hps, seed=int(g["seed"])).items()}
        x = torch.from_numpy(g["x"])
        noise = {(i, j): torch.from_numpy(g["noise_%d_%d" % (i, j)].astype(np.float64)) for i in range(2) for j in range(2)}
        out = elbo.forward(params, x, noise, OracleIAF(params, hps), hps)
        np.testing.assert_allclose(float(out["obj"]), float(g[tag + "obj"]), rtol=1e-10)
        np.testing.assert_allclose(float((out["kl_cost"] - out["log_pxz"]).sum()), float(g[tag + "loss"]), rtol=1e-10)
        np.testing.assert_allclose(float(out["bits_per_dim"]), float(g[tag + "bits_per_dim"]), rtol=1e-10)
    assert float(g["kl40_obj"]) > float(g["kl40_loss"]) and float(g["obj"]) == float(g["loss"])
