"""The importance-sampled log-likelihood of both restated models (``elbo.log_likelihood``, ``elbo_theano.log_likelihood``)
in fp64 on the CPU with the oracle blocks: the reference's estimators (``compute_lowerbound`` over ``forward`` on
``repeat(x, k)``, tf_train.py:167-170, 218; train.py:187-205 over k calls of ``forward``), chunk invariance, Jensen,
the streaming reduction at extreme log-weights, sharding over two gloo ranks, and the refused model names."""
import math
import os

import numpy as np
import pytest
import torch
from scipy.special import logsumexp

from iaf_b200 import elbo
from iaf_b200 import elbo_theano as ET
from oracle import iaf_oracle as O
from oracle.elbo_oracle import OracleIAF
from tests.linear_oracle import OracleIAFTheanoLinear
from tests.made_oracle import OracleIAFTheanoMade

TF_HPS = dict(z_size=4, h_size=8, depth=2, num_blocks=2, kl_min=0.25, image_size=16)
TH_HPS = dict(n_z=4, n_h1=8, n_h2=8, depths=[1, 1], depth_ar=1, nl="elu", kl_min=0.0, image_size=8)
POSTERIORS = ["down_iaf2_nl", "up_iaf2_nl", "down_iaf2_nl2", "down_iaf2", "up_iaf2"]


def tf_setup(hps, B, seed, dtype=torch.float64, device="cpu"):
    p = elbo.make_params(hps, seed=seed)
    params = {k: torch.from_numpy(np.asarray(v)).to(dtype).to(device) for k, v in p.items()}
    rng = np.random.RandomState(seed + 1)
    S = hps["image_size"]
    x = torch.from_numpy(rng.randint(0, 256, size=(B, 3, S, S)).astype(np.uint8)).to(device)
    return params, x


def th_setup(hps, B, seed, dtype=torch.float64, device="cpu"):
    w = {k: torch.from_numpy(np.asarray(v)).to(dtype).to(device) for k, v in ET.make_params(hps, seed=seed).items()}
    rng = np.random.RandomState(seed + 1)
    S = hps["image_size"]
    x = torch.from_numpy(rng.randint(0, 256, size=(B, 3, S, S)).astype(np.uint8)).to(device)
    return w, x


def fixed_noise(shapes, k, seed, dtype=torch.float64, device="cpu"):
    """All k samples of every image drawn up front: noise(start, count) slices them, image-major, so that every chunk
    size sees the same draws.  Returns (noise callable, {(i, j): [B, k, C, H, W]})."""
    rng = np.random.RandomState(seed)
    full = {key: torch.from_numpy(rng.randn(B, k, *s)).to(dtype).to(device) for key, (B, *s) in sorted(shapes.items())}

    def noise(start, count):
        return {key: v[:, start:start + count].reshape((-1,) + tuple(v.shape[2:])) for key, v in full.items()}
    return noise, full


def tf_shapes(hps, B):
    S = hps["image_size"]
    return {(i, j): (B, hps["z_size"], S // 2 ** (i + 1), S // 2 ** (i + 1))
            for i in range(hps["depth"]) for j in range(hps["num_blocks"])}


def th_shapes(hps, B):
    S = hps["image_size"]
    return {(i, j): (B, hps["n_z"], S // 2 ** (i + 1), S // 2 ** (i + 1))
            for i in range(len(hps["depths"])) for j in range(hps["depths"][i])}


def th_oracle(w, hps):
    cls = OracleIAFTheanoLinear if hps["posterior"] in ET.LINEAR else OracleIAFTheanoMade
    return cls(w, hps)


def test_tf_one_sample_is_the_elbo_of_forward():
    B = 3
    params, x = tf_setup(TF_HPS, B, 3)
    noise, full = fixed_noise(tf_shapes(TF_HPS, B), 1, 5)
    iaf = OracleIAF(params, TF_HPS)
    got = elbo.log_likelihood(params, x, iaf, TF_HPS, 1, noise=noise)
    ref = elbo.forward(params, x, noise(0, 1), iaf, TF_HPS)
    w = (ref["log_pxz"] - ref["kl_cost"]).numpy()
    np.testing.assert_allclose(got["log_px"].numpy(), w, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(got["elbo"].numpy(), w, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(float(got["bits_per_dim"]), float(ref["bits_per_dim"]), rtol=1e-12)


@pytest.mark.parametrize("chunk", [1, 3, 4])
def test_tf_equals_compute_lowerbound_over_repeat(chunk):
    """k = 4: -compute_lowerbound(log_pxz, kl_cost, 4) of forward on repeat(x, 4), whatever the chunk (1, 3 or k)."""
    B, k = 3, 4
    params, x = tf_setup(TF_HPS, B, 3)
    noise, full = fixed_noise(tf_shapes(TF_HPS, B), k, 5)
    iaf = OracleIAF(params, TF_HPS)
    ref = elbo.forward(params, torch.from_numpy(O.repeat(x.numpy(), k)), noise(0, k), iaf, TF_HPS)
    lb = O.compute_lowerbound(ref["log_pxz"].numpy(), ref["kl_cost"].numpy(), k)
    got = elbo.log_likelihood(params, x, iaf, TF_HPS, k, chunk=chunk, noise=noise)
    np.testing.assert_allclose(got["log_px"].numpy(), -lb, rtol=1e-12, atol=1e-12)
    w = (ref["log_pxz"] - ref["kl_cost"]).numpy().reshape(B, k)
    np.testing.assert_allclose(got["elbo"].numpy(), w.mean(axis=1), rtol=1e-12, atol=1e-12)
    bpd = (lb.sum()) / (math.log(2.0) * 3 * TF_HPS["image_size"] ** 2 * B)
    np.testing.assert_allclose(float(got["bits_per_dim"]), bpd, rtol=1e-12)
    # Jensen, exact for any fixed noise: log mean exp >= mean
    assert bool((got["log_px"] >= got["elbo"] - 1e-12 * got["elbo"].abs()).all())
    assert bool((got["log_px"] > got["elbo"]).any())


def test_tf_free_bits_do_not_enter_the_estimate():
    B, k = 2, 3
    params, x = tf_setup(TF_HPS, B, 4)
    noise, _ = fixed_noise(tf_shapes(TF_HPS, B), k, 6)
    a = elbo.log_likelihood(params, x, OracleIAF(params, TF_HPS), TF_HPS, k, noise=noise)
    h0 = dict(TF_HPS, kl_min=0.0)
    b = elbo.log_likelihood(params, x, OracleIAF(params, h0), h0, k, noise=noise)
    np.testing.assert_array_equal(a["log_px"].numpy(), b["log_px"].numpy())


def test_tf_default_noise_and_chunk():
    """The default noise is seeded (same seed, same estimate) and the default chunk covers k at these sizes; the
    estimator records no autograd graph."""
    B, k = 2, 3
    params, x = tf_setup(TF_HPS, B, 4)
    for v in params.values():
        v.requires_grad_(True)
    iaf = OracleIAF(params, TF_HPS)
    a = elbo.log_likelihood(params, x, iaf, TF_HPS, k, seed=1)
    b = elbo.log_likelihood(params, x, iaf, TF_HPS, k, seed=1)
    c = elbo.log_likelihood(params, x, iaf, TF_HPS, k, seed=2)
    assert not a["log_px"].requires_grad and a["log_px"].dtype == torch.float64 and a["log_px"].shape == (B,)
    np.testing.assert_array_equal(a["log_px"].numpy(), b["log_px"].numpy())
    assert not np.array_equal(a["log_px"].numpy(), c["log_px"].numpy())
    assert elbo.default_chunk(B, k, elbo._elems_per_sample(TF_HPS)) == k
    with pytest.raises(ValueError):
        elbo.log_likelihood(params, x, iaf, TF_HPS, 0)


def test_default_chunk_keeps_every_tensor_below_2_31():
    hps = dict(z_size=32, h_size=160, depth=1, num_blocks=20, kl_min=0.0, image_size=32)   # the README's eval config
    e = elbo._elems_per_sample(hps)
    assert e >= (4 * 32 + 2 * 160) * 16 * 16 and e >= 3 * 35 * 35   # down_conv1's output, x_dec's full output
    assert elbo.default_chunk(100, 10 ** 4, e) == elbo.MAX_SAMPLES // 100          # the samples-per-call cap binds
    assert 100 * (elbo.MAX_SAMPLES // 100) * e < 2 ** 31
    c = elbo.default_chunk(1, 10 ** 6, 2 ** 31 // 1000)                             # the index bound binds
    assert c * (2 ** 31 // 1000) < 2 ** 31 <= (c + 1) * (2 ** 31 // 1000) and c < elbo.MAX_SAMPLES
    assert elbo.default_chunk(100, 5, e) == 5 and elbo.default_chunk(10 ** 7, 5, e) == 1
    th = dict(n_z=32, n_h1=64, n_h2=64, depths=[2, 2, 2], depth_ar=1, nl="elu", kl_min=0.0, image_size=32)
    e = ET._elems_per_sample(th)
    assert e >= (2 * 64 + 4 * 32) * 16 * 16 and e >= (64 + 1) * 18 * 18 and e >= 4 * 36 * 36


def test_streaming_reduction_at_extreme_log_weights():
    """Log-weights near -1e4 with a spread of 1e3, fed in uneven chunks: neither overflow nor underflow, and the
    result is scipy's logsumexp - log k."""
    rng = np.random.RandomState(0)
    B, k = 5, 40
    w = -1e4 - 1e3 * rng.rand(B, k)
    w[:, 7] = -1e4 - 1e3          # the spread's far end
    w[2] = -1e4 + 0.0             # equal weights: log mean exp == the weight
    acc = elbo.LogMeanExp(B, "cpu")
    for lo, hi in ((0, 1), (1, 4), (4, 17), (17, 40)):
        acc.add(torch.from_numpy(w[:, lo:hi]))
    log_px, mean_w = acc.result()
    ref = logsumexp(w, axis=1) - math.log(k)
    assert np.isfinite(log_px.numpy()).all()
    np.testing.assert_allclose(log_px.numpy(), ref, rtol=1e-14)
    np.testing.assert_allclose(mean_w.numpy(), w.mean(axis=1), rtol=1e-14)
    assert abs(float(log_px[2]) + 1e4) < 1e-9
    # the maximum arriving in the last chunk rescales the earlier ones
    acc = elbo.LogMeanExp(1, "cpu")
    acc.add(torch.tensor([[-1.1e4, -1.05e4]], dtype=torch.float64))
    acc.add(torch.tensor([[-1e4]], dtype=torch.float64))
    np.testing.assert_allclose(float(acc.result()[0][0]), logsumexp([-1.1e4, -1.05e4, -1e4]) - math.log(3), rtol=1e-14)


@pytest.mark.parametrize("prior", ["diag", "made"])
@pytest.mark.parametrize("posterior", POSTERIORS)
def test_theano_equals_est_marglik_over_k_forward_calls(posterior, prior):
    """kl_min = 0: the train.py:196-201 running log-mean-exp over k calls of forward(...)["cost"] (in nats, through
    the correction factor), with chunks 1, 3 and k; kl_min > 0 gives the same estimate (the true KL sums)."""
    B, k = 2, 4
    hps = dict(TH_HPS, posterior=posterior, prior=prior)
    w, x = th_setup(hps, B, 7)
    noise, _ = fixed_noise(th_shapes(hps, B), k, 8)
    iaf = th_oracle(w, hps)
    correction = -(3 * hps["image_size"] ** 2 * np.log(2.0))
    obj = np.vstack([ET.forward(w, x, noise(j, 1), iaf, hps)["cost"].numpy() * correction for j in range(k)])
    mx = obj.max(axis=0)
    est = np.log(np.exp(obj - mx).mean(axis=0)) + mx
    for chunk in (1, 3, k):
        got = ET.log_likelihood(w, x, iaf, hps, k, chunk=chunk, noise=noise)
        np.testing.assert_allclose(got["log_px"].numpy(), est, rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(got["elbo"].numpy(), obj.mean(axis=0), rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(float(got["bits_per_dim"]), est.mean() / correction, rtol=1e-12)
        assert bool((got["log_px"] >= got["elbo"] - 1e-12 * got["elbo"].abs()).all())
    hk = dict(hps, kl_min=0.5)
    got = ET.log_likelihood(w, x, th_oracle(w, hk), hk, k, chunk=3, noise=noise)
    np.testing.assert_allclose(got["log_px"].numpy(), est, rtol=1e-12, atol=1e-12)
    # ... where the reference's own estimate, over the free-bits cost, differs
    cost = np.vstack([ET.forward(w, x, noise(j, 1), iaf, hk)["cost"].numpy() * correction for j in range(k)])
    assert not np.allclose(cost, obj, rtol=1e-9)


def _sharded_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    B, k = 3, 3
    params, x = tf_setup(TF_HPS, B, 11)
    noise, _ = fixed_noise(tf_shapes(TF_HPS, B), k, 12)
    tf = elbo.sharded_log_likelihood(params, x, OracleIAF(params, TF_HPS), TF_HPS, k, chunk=2, noise=noise)
    hps = dict(TH_HPS, posterior="down_iaf2_nl", prior="made")
    w, xt = th_setup(hps, B, 13)
    tnoise, _ = fixed_noise(th_shapes(hps, B), k, 14)
    th = elbo.sharded_log_likelihood(w, xt, th_oracle(w, hps), hps, k, chunk=2, noise=tnoise,
                                     estimator=ET.log_likelihood)
    q.put((rank, float(tf), float(th)))
    dist.destroy_process_group()


def test_sharded_log_likelihood_equals_single_process_gloo_world2():
    """Images split over two ranks (3 images: 2 + 1), each running all k samples of its own, one all-reduce of the
    summed -log_px: the global bits/dim of one process, for both models."""
    import torch.multiprocessing as mp
    B, k = 3, 3
    params, x = tf_setup(TF_HPS, B, 11)
    noise, _ = fixed_noise(tf_shapes(TF_HPS, B), k, 12)
    single_tf = float(elbo.log_likelihood(params, x, OracleIAF(params, TF_HPS), TF_HPS, k, noise=noise)["bits_per_dim"])
    hps = dict(TH_HPS, posterior="down_iaf2_nl", prior="made")
    w, xt = th_setup(hps, B, 13)
    tnoise, _ = fixed_noise(th_shapes(hps, B), k, 14)
    single_th = float(ET.log_likelihood(w, xt, th_oracle(w, hps), hps, k, noise=tnoise)["bits_per_dim"])
    assert single_tf == float(elbo.sharded_log_likelihood(params, x, OracleIAF(params, TF_HPS), TF_HPS, k,
                                                           noise=noise))   # one process: no collective
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 35500 + os.getpid() % 2000
    ps = [ctx.Process(target=_sharded_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in ps:
        p.start()
    res = sorted(q.get(timeout=300) for _ in ps)
    for p in ps:
        p.join(timeout=60)
        assert p.exitcode == 0
    for _, tf, th in res:
        assert abs(tf - single_tf) < 1e-12 * max(1.0, abs(single_tf))
        assert abs(th - single_th) < 1e-12 * max(1.0, abs(single_th))


@pytest.mark.parametrize("name", ["posterior", "prior"])
def test_refused_names_raise_value_error(name):
    bad = {"posterior": ("down_iaf1_nl", "up_iaf1_nl", "down_iaf2_deep", "up_iaf2_deep", "down_diag", "up_diag",
                         "down_tim", "down_bernoulli"),
           "prior": ("diag2", "bernoulli")}[name]
    w, x = th_setup(TH_HPS, 2, 3)
    for v in bad:
        hps = dict(TH_HPS, **{name: v})
        with pytest.raises(ValueError):
            ET.log_likelihood(w, x, OracleIAFTheanoMade(w, hps), hps, 2)
