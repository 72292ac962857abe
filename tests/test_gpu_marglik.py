"""The importance-sampled log-likelihood on the GPU: ``log_likelihood`` of both restated models through the CUDA operator
(CudaIAF, fp32) against the same estimator through the fp64 oracle blocks on the CPU, per image, on identical weights,
images and noise; chunk invariance on the GPU; a call whose B * chunk samples span several waves of CTAs; and the
operator launches per chunk."""
import numpy as np
import pytest
import torch

from iaf_b200 import elbo
from iaf_b200 import elbo_theano as ET
from oracle.elbo_oracle import OracleIAF
from tests.test_marglik import fixed_noise, tf_setup, tf_shapes, th_oracle, th_setup, th_shapes

DEV = "cuda:0"


def rel_err(got, ref):
    """max over images of |got - ref| / max(|ref|, 1)."""
    got, ref = got.double().cpu().numpy(), ref.double().cpu().numpy()
    return float((np.abs(got - ref) / np.maximum(np.abs(ref), 1.0)).max())


def _tf_pair(hps, B, k, seed):
    pg, xg = tf_setup(hps, B, seed, torch.float32, DEV)
    pc, xc = tf_setup(hps, B, seed, torch.float64, "cpu")
    ng, _ = fixed_noise(tf_shapes(hps, B), k, seed + 2, torch.float32, DEV)
    nc, _ = fixed_noise(tf_shapes(hps, B), k, seed + 2, torch.float64, "cpu")
    return (pg, xg, ng), (pc, xc, nc)


@pytest.mark.gpu
@pytest.mark.parametrize("hps,B,k,chunk", [
    (dict(z_size=32, h_size=64, depth=2, num_blocks=2, kl_min=0.25, image_size=32), 2, 4, 3),    # two levels
    (dict(z_size=32, h_size=160, depth=1, num_blocks=2, kl_min=0.1, image_size=32), 2, 3, None),  # the C3 stack
])
def test_tf_log_likelihood_against_fp64_oracle(hps, B, k, chunk):
    (pg, xg, ng), (pc, xc, nc) = _tf_pair(hps, B, k, 3)
    iaf = elbo.CudaIAF(pg, hps)
    got = elbo.log_likelihood(pg, xg, iaf, hps, k, chunk=chunk, noise=ng)
    ref = elbo.log_likelihood(pc, xc, OracleIAF(pc, hps), hps, k, chunk=chunk, noise=nc)
    assert got["log_px"].dtype == torch.float64 and got["log_px"].device.type == "cuda"
    for sc, op in iaf.ops.items():
        s = hps["image_size"] // 2 ** (int(sc.split("_")[1]) + 1)
        assert op.path_used(s, s, DEV, "layer") == "tc", sc
    assert rel_err(got["log_px"], ref["log_px"]) <= 1e-4
    assert rel_err(got["elbo"], ref["elbo"]) <= 1e-4
    assert abs(float(got["bits_per_dim"]) - float(ref["bits_per_dim"])) <= 1e-4 * abs(float(ref["bits_per_dim"]))


@pytest.mark.gpu
@pytest.mark.parametrize("posterior", ["down_iaf2_nl", "down_iaf2_nl2", "up_iaf2_nl", "down_iaf2"])
def test_theano_made_log_likelihood_against_fp64_oracle(posterior):
    B, k = 2, 3
    hps = dict(n_z=32, n_h1=64, n_h2=64, depths=[1, 1], depth_ar=1, nl="elu", kl_min=0.25, image_size=32,
               posterior=posterior, prior="made")
    wg, xg = th_setup(hps, B, 5, torch.float32, DEV)
    wc, xc = th_setup(hps, B, 5, torch.float64, "cpu")
    ng, _ = fixed_noise(th_shapes(hps, B), k, 6, torch.float32, DEV)
    nc, _ = fixed_noise(th_shapes(hps, B), k, 6, torch.float64, "cpu")
    iaf = ET.CudaIAF(wg, hps)
    got = ET.log_likelihood(wg, xg, iaf, hps, k, chunk=2, noise=ng)
    ref = ET.log_likelihood(wc, xc, th_oracle(wc, hps), hps, k, chunk=2, noise=nc)
    for (name, conv), op in iaf.ops.items():
        s = hps["image_size"] // 2 ** (int(name[0]) + 1)
        assert op.path_used(s, s, DEV, "step") == "tc", (name, conv)
    assert rel_err(got["log_px"], ref["log_px"]) <= 1e-4
    assert rel_err(got["elbo"], ref["elbo"]) <= 1e-4


@pytest.mark.gpu
def test_chunk_invariance_on_the_gpu():
    """Same noise, chunks 1, 3 and k: equal to 1e-6 relative (a sample's tiles depend on its position in the batch, so
    this is not bitwise).  Theano up_iaf2_nl too: its up pass runs per sample."""
    hps = dict(z_size=32, h_size=64, depth=1, num_blocks=2, kl_min=0.0, image_size=32)
    B, k = 3, 7
    (pg, xg, ng), _ = _tf_pair(hps, B, k, 9)
    iaf = elbo.CudaIAF(pg, hps)
    runs = [elbo.log_likelihood(pg, xg, iaf, hps, k, chunk=c, noise=ng)["log_px"] for c in (1, 3, k)]
    for r in runs[1:]:
        assert rel_err(r, runs[0]) <= 1e-6
    th = dict(n_z=32, n_h1=64, n_h2=64, depths=[1, 1], depth_ar=1, nl="elu", kl_min=0.0, image_size=32,
              posterior="up_iaf2_nl")
    wg, xg = th_setup(th, B, 10, torch.float32, DEV)
    ng, _ = fixed_noise(th_shapes(th, B), k, 11, torch.float32, DEV)
    iaf = ET.CudaIAF(wg, th)
    runs = [ET.log_likelihood(wg, xg, iaf, th, k, chunk=c, noise=ng)["log_px"] for c in (1, 3, k)]
    for r in runs[1:]:
        assert rel_err(r, runs[0]) <= 1e-6


@pytest.mark.gpu
def test_one_call_spanning_several_waves():
    """B * chunk = 4 * 64 = 256 samples of 16x16 latents in ONE call: about 578 tensor-core tiles of 128 slots,
    several waves over the H100's 132 SMs.  Against the fp64 oracle, and against small chunks on the GPU."""
    hps = dict(z_size=32, h_size=64, depth=1, num_blocks=1, kl_min=0.0, image_size=32)
    B, k = 4, 64
    (pg, xg, ng), (pc, xc, nc) = _tf_pair(hps, B, k, 13)
    iaf = elbo.CudaIAF(pg, hps)
    got = elbo.log_likelihood(pg, xg, iaf, hps, k, chunk=k, noise=ng)
    (op,) = iaf.ops.values()
    assert op.path_used(16, 16, DEV, "layer") == "tc"
    ref = elbo.log_likelihood(pc, xc, OracleIAF(pc, hps), hps, k, chunk=k, noise=nc)
    assert rel_err(got["log_px"], ref["log_px"]) <= 1e-4
    small = elbo.log_likelihood(pg, xg, iaf, hps, k, chunk=5, noise=ng)
    assert rel_err(got["log_px"], small["log_px"]) <= 1e-6


@pytest.mark.gpu
def test_operator_launches_per_chunk():
    """Every chunk runs each layer's operator entry exactly once: the launches of a call with 3 chunks are
    3 x layers x the entry's launches (TF: the fused layer entry; Theano down_iaf2_nl2 + made: two steps and the
    prior's log-density per layer)."""
    hps = dict(z_size=32, h_size=64, depth=2, num_blocks=1, kl_min=0.0, image_size=32)
    B, k, chunk = 2, 6, 2
    (pg, xg, ng), _ = _tf_pair(hps, B, k, 15)
    iaf = elbo.CudaIAF(pg, hps)
    elbo.log_likelihood(pg, xg, iaf, hps, 1, noise=ng)           # creates every operator and plan
    before = {sc: op.launch_count() for sc, op in iaf.ops.items()}
    elbo.log_likelihood(pg, xg, iaf, hps, k, chunk=chunk, noise=ng)
    per_chunk = {sc: (op.launch_count() - before[sc]) / (k // chunk) for sc, op in iaf.ops.items()}
    assert len(per_chunk) == hps["depth"] * hps["num_blocks"]
    for sc, op in iaf.ops.items():
        s = int(sc.split("_")[1])
        size = hps["image_size"] // 2 ** (s + 1)
        t = lambda *shape: torch.randn(*shape, device=DEV)
        l0 = op.launch_count()
        op.layer(t(B * chunk, 32, size, size), t(B * chunk, 32, size, size), 0.1 * t(B * chunk, 32, size, size),
                 t(B * chunk, 32, size, size), 0.1 * t(B * chunk, 32, size, size), t(B * chunk, 64, size, size),
                 want_kl=False)
        assert per_chunk[sc] == op.launch_count() - l0 >= 1, sc

    th = dict(n_z=32, n_h1=64, n_h2=64, depths=[1, 1], depth_ar=1, nl="elu", kl_min=0.0, image_size=32,
              posterior="down_iaf2_nl2", prior="made")
    wg, xg = th_setup(th, B, 16, torch.float32, DEV)
    ng, _ = fixed_noise(th_shapes(th, B), k, 17, torch.float32, DEV)
    iaf = ET.CudaIAF(wg, th)
    ET.log_likelihood(wg, xg, iaf, th, 1, noise=ng)
    ops = list(iaf.ops.values()) + list(iaf.prior_ops.values())
    assert len(ops) == 3 * len(th["depths"])
    before = [op.launch_count() for op in ops]
    ET.log_likelihood(wg, xg, iaf, th, k, chunk=chunk, noise=ng)
    per_chunk = [(op.launch_count() - b) / (k // chunk) for op, b in zip(ops, before)]
    entry = []
    for (name, conv), op in iaf.ops.items():
        size = th["image_size"] // 2 ** (int(name[0]) + 1)
        l0 = op.launch_count()
        op.step(torch.randn(B * chunk, 32, size, size, device=DEV), torch.randn(B * chunk, 64, size, size, device=DEV))
        entry.append(op.launch_count() - l0)
    for name, op in iaf.prior_ops.items():
        size = th["image_size"] // 2 ** (int(name[0]) + 1)
        l0 = op.launch_count()
        op.ar_logp(torch.randn(B * chunk, 32, size, size, device=DEV), torch.randn(B * chunk, 64, size, size, device=DEV))
        entry.append(op.launch_count() - l0)
    assert per_chunk == entry and min(entry) >= 1, (per_chunk, entry)
