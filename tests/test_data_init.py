"""The data-dependent initialisation of both restated models (elbo.data_init: tf_train.py mode "init";
elbo_theano.data_init: cvae1 with data_init) against what the reference's own init passes produced
(tests/golden/make_golden_init.py), in fp64 on the CPU; and the run-time paths left exactly as they were."""
import hashlib
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from iaf_b200 import elbo
from iaf_b200 import elbo_theano as ET
from oracle.elbo_oracle import OracleIAF

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
TF_HPS = dict(z_size=4, h_size=8, depth=2, num_blocks=2, kl_min=0.25, image_size=16)
TH_HPS = dict(n_z=4, n_h1=4, n_h2=8, depths=[1, 1], depth_ar=2, nl="elu", kl_min=0.25, image_size=16)
TH_CASES = [(p, q) for p in ET.POSTERIORS for q in ET.PRIORS]


def _t(a):
    return torch.from_numpy(np.asarray(a, dtype=np.float64))


def _rel(got, ref):
    got, ref = np.asarray(got, dtype=np.float64), np.asarray(ref, dtype=np.float64)
    return float(np.abs(got - ref).max()) / max(float(np.abs(ref).max()), 1e-300)


def _tf_inputs():
    g = np.load(os.path.join(GOLDEN, "init_tf.npz"))
    # the reference creates g and b inside the init branch; here they start at make_params' values, which the pass
    # must overwrite, every one
    params = {k: _t(v) for k, v in elbo.make_params(TF_HPS, seed=1).items()}
    for k in g.files:
        if k.startswith("V/"):
            params[k[2:]] = _t(g[k])
    params["h_top"] = torch.zeros(TF_HPS["h_size"], dtype=torch.float64)   # tf_train.py:190
    params["dec_log_stdv"] = torch.zeros((), dtype=torch.float64)           # tf_train.py:122
    noise = {(i, j): _t(g["noise_%d_%d" % (i, j)]) for i in range(2) for j in range(2)}
    return g, params, torch.from_numpy(g["x"]), noise


def test_tf_data_init_matches_reference_init_pass():
    g, params, x, noise = _tf_inputs()
    new, out, stacks = elbo.data_init_pass(params, x, TF_HPS, noise)
    init = [k for k in g.files if k.startswith("init/")]
    assert len(init) == 2 * sum(k.startswith("V/") for k in g.files) == 68
    for k in init:
        assert _rel(new[k[5:]], g[k]) <= 1e-6, (k, _rel(new[k[5:]], g[k]))
    for k, v in params.items():                     # V, h_top, dec_log_stdv pass through untouched
        if not k.endswith(("/g", "/b")):
            assert new[k] is v, k
    # the init-mode ELBO terms (tf_train.py:210-218 in mode "init")
    np.testing.assert_allclose(float(out["obj"]), float(g["obj"]), rtol=1e-9)
    np.testing.assert_allclose(float((out["kl_cost"] - out["log_pxz"]).sum()), float(g["loss"]), rtol=1e-9)
    assert sorted(stacks) == sorted("IAF_%d_%d/ar_multiconv2d" % k for k in noise)
    # data_init is the same pass, and leaves its input dict alone
    assert all(torch.equal(v, new[k]) for k, v in elbo.data_init(params, x, TF_HPS, noise).items())
    assert float((params["x_enc/g"] - new["x_enc/g"]).abs().max()) > 0


def test_tf_cube_root_gain_after_init():
    """layers.py:49, 60: g = log(scale) / 3 while the run-time branch applies exp(g), so a layer initialised on the
    batch runs at scale^(1/3), not at the standardising scale.  x_enc sees the image directly: after init, its
    run-time output is exp(g) x_init + b, with std scale^(1/3) std(x_init) = 0.1^(1/3) std(x_init)^(2/3)."""
    _, params, x, noise = _tf_inputs()
    new = elbo.data_init(params, x, TF_HPS, noise)
    img = elbo._image(new, x)
    y = elbo.conv2d(new, "x_enc", img, stride=2)
    x_init = elbo.conv2d(dict(new, **{"x_enc/g": torch.zeros_like(new["x_enc/g"]),
                                      "x_enc/b": torch.zeros_like(new["x_enc/b"])}), "x_enc", img, stride=2)
    sd_init = x_init.std(dim=(0, 2, 3), unbiased=False)
    sd = y.std(dim=(0, 2, 3), unbiased=False)
    np.testing.assert_allclose(sd.numpy(), (0.1 ** (1 / 3) * sd_init ** (2 / 3)).numpy(), rtol=1e-9)
    assert float((sd - 0.1).abs().min()) > 1e-3      # not the standardised init-mode output


def _unflatten(vec, names, shapes):
    out, i = {}, 0
    for k in names:
        n = int(np.prod(shapes[k]))
        out[k] = np.asarray(vec[i:i + n], dtype=np.float64).reshape(shapes[k])
        i += n
    assert i == vec.size
    return out


def _th_inputs(g, posterior, prior):
    """The case's initial parameters (tensors), the reference's initialised values of every parameter but the kernels
    (arrays), its image batch and noise.  The fixture stores both as flat vectors in sorted name order."""
    tag = "%s_%s/" % (posterior, prior)
    hps = dict(TH_HPS, posterior=posterior, prior=prior)
    shapes = {k: v.shape for k, v in ET.make_params(hps).items()}
    names = sorted(shapes)
    w0 = {k: _t(v) for k, v in _unflatten(g[tag + "w0"], names, shapes).items()}
    ref = _unflatten(g[tag + "w"], [k for k in names if not k.endswith("_w")], shapes)
    noise = {(i, j): _t(g[tag + "eps_%d_%d" % (i, j)]) for i in range(2) for j in range(1)}
    return tag, hps, w0, ref, torch.from_numpy(g[tag + "x"]), noise


@pytest.mark.parametrize("posterior,prior", TH_CASES)
def test_theano_data_init_matches_reference_init_pass(posterior, prior):
    g = np.load(os.path.join(GOLDEN, "init_theano.npz"))
    tag, hps, w, refs, x, noise = _th_inputs(g, posterior, prior)
    new, results, stacks = ET.data_init_pass(w, x, hps, noise)
    n_set = 0
    for k in w:
        if k.endswith("_w"):
            assert new[k] is w[k], k
            continue
        ref = refs[k]
        n_set += not np.array_equal(ref, w[k].numpy())
        if ref.ndim == 0 or not np.any(ref):
            np.testing.assert_array_equal(new[k].numpy(), ref, err_msg=k)     # h_top, logsd_x: passed through
        else:
            assert _rel(new[k], ref) <= 1e-6, (k, _rel(new[k], ref))
    assert n_set == 2 * sum(k.endswith("_w") for k in w)                      # every conv was initialised
    for k in ("cost", "cost_x", "cost_z000_000", "cost_z001_000"):           # the init-mode ELBO terms
        np.testing.assert_allclose(results[k].numpy(), g[tag + "results/" + k], rtol=1e-6, err_msg=k)
    expect = {"0_0_posterior_conv1", "1_0_posterior_conv1"}
    if posterior == "down_iaf2_nl2":
        expect |= {"0_0_posterior_conv2", "1_0_posterior_conv2"}
    if prior == "made":
        expect |= {"0_0_prior_conv1", "1_0_prior_conv1"}
    assert set(stacks) == expect


def test_theano_zero_std_skips_the_conv():
    """conv.py:229-231 / ar.py:335-337: a conv with a channel of std exactly 0 keeps its parameters (and passes its
    output on unstandardised), with the reference's warning; the other convs are still initialised."""
    g = np.load(os.path.join(GOLDEN, "init_theano.npz"))
    tag, hps, w, refs, x, noise = _th_inputs(g, "down_iaf2_nl", "diag")
    w["0_0_posterior_conv1_out_1_w"] = w["0_0_posterior_conv1_out_1_w"].clone()
    w["0_0_posterior_conv1_out_1_w"][2] = 0.0        # that channel's output is its bias: std 0 (ar.py:280: norm + 1e-8)
    w["0_0_posterior_conv1_out_1_s"] = torch.full((4,), 0.05, dtype=torch.float64)
    with pytest.warns(UserWarning, match="Stdev=0 for 1 features in 0_0_posterior_conv1_out_1. Skipping"):
        new = ET.data_init(w, x, hps, noise)
    for k in "sb":
        assert new["0_0_posterior_conv1_out_1_" + k] is w["0_0_posterior_conv1_out_1_" + k]
    # convs before it in the pass are as in the reference's run; its sibling head is initialised as usual
    assert _rel(new["0_0_posterior_conv1_out_0_s"], refs["0_0_posterior_conv1_out_0_s"]) <= 1e-6
    assert _rel(new["1_0_posterior_conv1_1_s"], refs["1_0_posterior_conv1_1_s"]) <= 1e-6
    assert not torch.equal(new["x_dec_s"], w["x_dec_s"])

    # the datainit convs: a constant input gives every output channel std 0
    plain = {"c_w": torch.randn(3, 2, 1, 1, dtype=torch.float64), "c_s": torch.zeros(3, dtype=torch.float64),
             "c_b": torch.zeros(3, dtype=torch.float64)}
    with pytest.warns(UserWarning, match="Stdev=0 for 3 features in c"):
        y = ET.conv2d(elbo.InitPass(plain), "c", torch.ones(2, 2, 4, 4, dtype=torch.float64))
    np.testing.assert_array_equal(y.numpy(), ET.conv2d(plain, "c", torch.ones(2, 2, 4, 4, dtype=torch.float64)).numpy())


def test_data_init_default_noise_is_seeded():
    _, params, x, _ = _tf_inputs()
    a, b, c = (elbo.data_init(params, x, TF_HPS, seed=s) for s in (4, 4, 5))
    assert all(torch.equal(a[k], b[k]) for k in a)
    assert not torch.equal(a["x_dec/b"], c["x_dec/b"]) and torch.equal(a["x_enc/b"], c["x_enc/b"])


def _digest(d):
    m = hashlib.sha256()
    for k in sorted(d):
        m.update(k.encode())
        m.update(np.ascontiguousarray(d[k]).tobytes())
    return m.hexdigest()


def test_make_params_unchanged():
    """make_params draws what it drew before data_init existed (digests of the arrays it returned then)."""
    assert _digest(elbo.make_params(TF_HPS, seed=3)) == "3be2317b8cfdfb4ddd22bd56091e4e66aa989007cebbe8aacc17b5f44ac6aa6e"
    expect = {"down_iaf2_nl": "30fcbc625ce0e6bc7b168c2b5a08925ec3545f8e271d78db8686c5a1cf9e48a6",
              "up_iaf2_nl": "f13520591fd29d5a320466ff332fa116236e2b4e28ddbb966ec0494926a56605",
              "down_iaf2_nl2": "be170344b516302d85ee47be7cd0af2f908e06829ff0026c83fb77759795a6b2",
              "down_iaf2": "b30da3882f95cc9a238d880cf4558d501845fad9bfec6e17b0726192881beec1",
              "up_iaf2": "63ce25df218a00be22726d0d16c56218a5acf03ebe2c0353b468c9c0217abe4e"}
    hps = dict(n_z=4, n_h1=8, n_h2=8, depths=[1, 1], depth_ar=2, nl="elu", kl_min=0.25, image_size=16, prior="made")
    for post, h in expect.items():
        assert _digest(ET.make_params(dict(hps, posterior=post), seed=3)) == h, post


def _conv2d_before(params, name, x, stride=1):
    """elbo.conv2d as it was before the init branch: the run-time path must compute bit for bit the same."""
    V, g, b = params[name + "/V"], params[name + "/g"], params[name + "/b"]
    w = torch.exp(g).reshape(1, 1, 1, -1) * V * torch.rsqrt(torch.clamp((V * V).sum(dim=(0, 1, 2), keepdim=True), min=1e-12))
    kh, kw = V.shape[0], V.shape[1]
    pt, pb = elbo._same_pad(x.shape[2], kh, stride)
    pl, pr = elbo._same_pad(x.shape[3], kw, stride)
    x = F.pad(x, (pl, pr, pt, pb))
    return F.conv2d(x, w.permute(3, 2, 0, 1), stride=stride) + b.reshape(1, -1, 1, 1)


def _deconv2d_before(params, name, x, stride=2):
    V, g, b = params[name + "/V"], params[name + "/g"], params[name + "/b"]
    w = torch.exp(g).reshape(1, 1, -1, 1) * V * torch.rsqrt(torch.clamp((V * V).sum(dim=(0, 1, 2), keepdim=True), min=1e-12))
    kh, kw = V.shape[0], V.shape[1]
    H, W = x.shape[2] * stride, x.shape[3] * stride
    y = F.conv_transpose2d(x, w.permute(3, 2, 0, 1), stride=stride)
    pt, _ = elbo._same_pad(H, kh, stride)
    pl, _ = elbo._same_pad(W, kw, stride)
    return y[:, :, pt:pt + H, pl:pl + W] + b.reshape(1, -1, 1, 1)


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_tf_forward_bit_identical_to_before(monkeypatch, dtype):
    params = {k: torch.from_numpy(np.asarray(v)).to(dtype) for k, v in elbo.make_params(TF_HPS, seed=3).items()}
    rng = np.random.RandomState(4)
    x = torch.from_numpy(rng.randint(0, 256, size=(3, 3, 16, 16)).astype(np.uint8))
    noise = {(i, j): torch.from_numpy(rng.randn(3, 4, 16 // 2 ** (i + 1), 16 // 2 ** (i + 1))).to(dtype)
             for i in range(2) for j in range(2)}
    got = elbo.forward(params, x, noise, OracleIAF(params, TF_HPS), TF_HPS)
    monkeypatch.setattr(elbo, "conv2d", _conv2d_before)
    monkeypatch.setattr(elbo, "deconv2d", _deconv2d_before)
    ref = elbo.forward(params, x, noise, OracleIAF(params, TF_HPS), TF_HPS)
    for k in ref:
        assert torch.equal(got[k], ref[k]), k
