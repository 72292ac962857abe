"""H100 checks of the fused Adamax step (iaf_b200.optim.Adamax, iaf_adamax_kernel) and of both models' train_step:

* 50 steps are bit-identical to the op-by-op fp32 restatement (tests/adamax_oracle.py) on the GPU, for both rules, at
  the TF default parameter set (104 tensors, 8.33 M elements) and at a c2a-shaped Theano set; one launch per step;
* a captured step replayed 10 times equals 10 eager steps bit for bit, on a side stream too;
* after a step, CudaIAF bound to the live parameters and to ``averaged()`` equals a freshly built CudaIAF (the step
  bumps the version counters its packed-weight cache keys on);
* 100 training steps leave every masked tap of every AR weight at exactly zero, its first moment too;
* 20 ``train_step``s of each model at small shapes follow an fp64 oracle training loop (oracle gradients, fp64
  restated optimiser) in the parameters, the averages and the bits/dim evaluated at ``averaged()``.
TF32 is off throughout, so the models' stock convs run in fp32."""
import numpy as np
import pytest
import torch

from iaf_b200 import _lib
from iaf_b200 import elbo
from iaf_b200 import elbo_theano as ET
from iaf_b200.masks import tf_conv_ar_mask, theano_conv_ar_mask
from iaf_b200.optim import Adamax
from oracle.elbo_oracle import TorchIAF, TorchIAFTheano
from tests.adamax_oracle import RestatedAdamax

pytestmark = pytest.mark.gpu

TF_DEFAULT = dict(z_size=32, h_size=160, depth=2, num_blocks=2, kl_min=0.25, image_size=32)  # tf_train.py:98-113
TH_C2A = dict(n_z=32, n_h1=64, n_h2=64, depths=[2, 2, 2], depth_ar=1, nl="elu", kl_min=0.25, image_size=32)
TF_SMALL = dict(z_size=4, h_size=8, depth=2, num_blocks=1, kl_min=0.1, image_size=8)
TH_SMALL = dict(n_z=4, n_h1=4, n_h2=8, depths=[1, 1], depth_ar=1, nl="elu", kl_min=0.1, image_size=8)


@pytest.fixture(autouse=True)
def _no_tf32():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def _params(rule, hps, seed=0, dtype=torch.float32, device="cuda"):
    mp = elbo.make_params if rule == "tf" else ET.make_params
    return {k: torch.tensor(np.asarray(v), dtype=dtype, device=device).requires_grad_()
            for k, v in mp(hps, seed=seed).items()}


def _clone(p):
    return {k: v.detach().clone().requires_grad_() for k, v in p.items()}


def _set_grads(params, gen, step):
    for i, p in enumerate(params.values()):
        scale = 10.0 ** ((i + step) % 7 - 3)
        g = torch.randn(p.shape, generator=gen, device=p.device) * scale
        if (i + step) % 11 == 0:
            g = torch.zeros_like(g)
        p.grad = g


def _assert_same(a, b, what):
    for k in a:
        assert torch.equal(a[k].detach(), b[k].detach()), "%s: %s differs" % (what, k)


@pytest.mark.parametrize("rule,hps", [("tf", TF_DEFAULT), ("theano", TH_C2A)], ids=["tf_default", "theano_c2a"])
def test_fused_step_bit_identical_to_restatement(rule, hps):
    p = _params(rule, hps)
    if rule == "tf":
        assert len(p) == 104 and sum(t.numel() for t in p.values()) == 8_331_175
    q = _clone(p)
    opt, ref = Adamax(p, rule), RestatedAdamax(q, rule)
    gen = torch.Generator(device="cuda").manual_seed(1)
    lib = _lib.lib()
    for step in range(50):
        _set_grads(p, gen, step)
        for k in p:
            q[k].grad = p[k].grad.clone()
        if step % 9 == 4:                      # a missing gradient: skipped (TF) / zero (Theano)
            p["h_top"].grad = q["h_top"].grad = None
        before = lib.iaf_adamax_launch_count()
        opt.step()
        assert lib.iaf_adamax_launch_count() - before == 1
        ref.step()
    torch.cuda.synchronize()
    _assert_same(p, q, "parameters")
    _assert_same(opt.averaged(), ref.averaged(), "averages")


@pytest.mark.parametrize("side", [False, True], ids=["current_stream", "side_stream"])
def test_captured_step_replays_like_eager_steps(side):
    p = _params("tf", TF_SMALL)
    q, p0 = _clone(p), _clone(p)
    gen = torch.Generator(device="cuda").manual_seed(2)
    _set_grads(p, gen, 0)
    for k in p:
        q[k].grad = p[k].grad.clone()
    opt, eager = Adamax(p, "tf"), Adamax(q, "tf")
    warm = {"w": torch.zeros(5, device="cuda", requires_grad=True)}
    warm["w"].grad = torch.ones(5, device="cuda")
    Adamax(warm, "tf").step()                  # the kernel's module is loaded before the capture
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        opt.step()
    with torch.cuda.stream(s if side else torch.cuda.current_stream()):
        for _ in range(10):
            graph.replay()
            eager.step()
    torch.cuda.synchronize()
    _assert_same(p, q, "parameters")
    _assert_same(opt.averaged(), eager.averaged(), "averages")
    assert sum(not torch.equal(p[k], p0[k]) for k in p) > len(p) // 2   # the replays did update


def _layer_inputs(hps, seed=3):
    g = torch.Generator(device="cuda").manual_seed(seed)
    zs, hs, S = hps["z_size"], hps["h_size"], hps["image_size"] // 2
    r = lambda c, s=1.0: s * torch.randn((2, c, S, S), generator=g, device="cuda")
    return r(zs), r(zs), r(zs, 0.1), r(zs), r(zs, 0.1), r(hs)


def test_step_bumps_the_versions_cudaiaf_caches_on():
    p = _params("tf", TF_SMALL)
    opt = Adamax(p, "tf")
    live, avg = elbo.CudaIAF(p, TF_SMALL), elbo.CudaIAF(opt.averaged(), TF_SMALL)
    args = _layer_inputs(TF_SMALL)
    with torch.no_grad():
        live("IAF_0_0", *args), avg("IAF_0_0", *args)     # pack the weights
        gen = torch.Generator(device="cuda").manual_seed(4)
        for step in range(3):
            _set_grads(p, gen, step)
            opt.step()
        for layer, params in ((live, p), (avg, opt.averaged())):
            got = layer("IAF_0_0", *args)
            want = elbo.CudaIAF(params, TF_SMALL)("IAF_0_0", *args)
            for a, b in zip(got, want):
                assert torch.equal(a, b)


def _ar_masks(rule, params):
    """{name: mask} of every AR weight (raw layouts) of the small models."""
    out = {}
    for k, v in params.items():
        if rule == "tf" and "/ar_multiconv2d/" in k and k.endswith("/V"):
            out[k] = tf_conv_ar_mask(v.shape[2], v.shape[3], "layer_out" in k)
        elif rule == "theano" and "_posterior_conv1_" in k and k.endswith("_w"):
            out[k] = theano_conv_ar_mask(v.shape[1] - 1, v.shape[0], zerodiagonal="_out_" in k)
    return {k: torch.from_numpy(m).to(params[k].device) for k, m in out.items()}


def _batch(hps, seed, dtype=torch.float32, device="cuda"):
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(0, 256, (4, 3, hps["image_size"], hps["image_size"]), generator=g, dtype=torch.uint8)
    if "z_size" in hps:
        shapes = elbo._noise_shapes(hps, 4)
    else:
        S = hps["image_size"]
        shapes = {(i, j): (4, hps["n_z"], S // 2 ** (i + 1), S // 2 ** (i + 1))
                  for i in range(len(hps["depths"])) for j in range(hps["depths"][i])}
    noise = {k: torch.randn(s, generator=g, dtype=torch.float64) for k, s in sorted(shapes.items())}
    return x.to(device), {k: v.to(device=device, dtype=dtype) for k, v in noise.items()}


@pytest.mark.parametrize("rule", ["tf", "theano"])
def test_masked_taps_stay_zero(rule):
    hps = TF_SMALL if rule == "tf" else TH_SMALL
    p = _params(rule, hps)
    masks = _ar_masks(rule, p)
    assert masks
    with torch.no_grad():
        for k, m in masks.items():
            p[k].mul_(m)                       # postup's re-mask (ar.py:369-373) on the initial weights
    p0 = {k: v.detach().clone() for k, v in p.items()}
    opt = Adamax(p, rule)
    mod = elbo if rule == "tf" else ET
    layer = elbo.CudaIAFTrain(p, hps) if rule == "tf" else ET.CudaIAFTrain(p, hps)
    for step in range(100):
        x, noise = _batch(hps, step)
        mod.train_step(p, x, opt, hps, noise=noise, iaf_layer=layer)
    torch.cuda.synchronize()
    names = list(p)
    for k, m in masks.items():
        assert (p[k][m == 0] == 0).all(), k
        assert (opt.averaged()[k][m == 0] == 0).all(), k
        i = names.index(k)
        off = sum(-(-p[n].numel() // 4) * 4 for n in names[:i])
        mom1 = opt.mom1[off:off + p[k].numel()].view(p[k].shape)
        assert (mom1[m == 0] == 0).all(), k
        assert not torch.equal(p[k][m != 0], p0[k][m != 0]), k   # the live taps did train


def _rel_l2(a, b, scale):
    return float((a.double().cpu() - b.double().cpu()).norm() / max(float(scale), 1e-30))


@pytest.mark.parametrize("rule", ["tf", "theano"])
def test_train_steps_follow_fp64_oracle_loop(rule):
    """Tolerance: the parameters' and averages' distance to the fp64 loop is below 1e-3 of how far the fp64 loop moved
    them (Adamax's step is lr v / m: an fp32 gradient that flips the sign of a near-zero component moves that one
    element by up to 2 lr b1, so a max-norm bound would only restate lr); bits/dim at averaged() to 1e-5 relative."""
    hps = TF_SMALL if rule == "tf" else TH_SMALL
    mod = elbo if rule == "tf" else ET
    p = _params(rule, hps)
    r = _params(rule, hps, dtype=torch.float64, device="cpu")
    p0 = {k: v.detach().clone() for k, v in r.items()}
    opt, ropt = Adamax(p, rule), RestatedAdamax(r, rule)
    layer = elbo.CudaIAFTrain(p, hps) if rule == "tf" else ET.CudaIAFTrain(p, hps)
    rlayer = TorchIAF(r, hps) if rule == "tf" else TorchIAFTheano(r, hps)
    for step in range(20):
        x, noise = _batch(hps, 100 + step)
        b = mod.train_step(p, x, opt, hps, noise=noise, iaf_layer=layer)
        xr, nr = _batch(hps, 100 + step, torch.float64, "cpu")
        rb = mod.train_step(r, xr, ropt, hps, noise=nr, iaf_layer=rlayer)
        assert abs(float(b) - float(rb)) < 1e-4 * abs(float(rb))
    torch.cuda.synchronize()
    moved = torch.sqrt(sum(((r[k].detach() - p0[k]) ** 2).sum() for k in r))
    dp = torch.sqrt(sum(((p[k].detach().double().cpu() - r[k].detach()) ** 2).sum() for k in r))
    avg, ravg = opt.averaged(), ropt.averaged()
    moved_avg = torch.sqrt(sum(((ravg[k] - p0[k]) ** 2).sum() for k in r))
    da = torch.sqrt(sum(((avg[k].double().cpu() - ravg[k]) ** 2).sum() for k in r))
    print("%s: |dp| / |moved| = %.3e, |davg| / |moved avg| = %.3e" % (rule, dp / moved, da / moved_avg))
    assert dp < 1e-3 * moved and da < 1e-3 * moved_avg

    x, noise = _batch(hps, 999)
    xr, nr = _batch(hps, 999, torch.float64, "cpu")
    with torch.no_grad():
        if rule == "tf":
            got = elbo.forward(avg, x, noise, elbo.CudaIAF(avg, hps), hps)["bits_per_dim"]
            want = elbo.forward(ravg, xr, nr, TorchIAF(ravg, hps), hps)["bits_per_dim"]
        else:
            got = ET.forward(avg, x, noise, ET.CudaIAF(avg, hps), hps)["bits_per_dim"]
            want = ET.forward(ravg, xr, nr, TorchIAFTheano(ravg, hps), hps)["bits_per_dim"]
    print("%s: bits/dim at averaged() %.8f vs fp64 %.8f" % (rule, float(got), float(want)))
    assert abs(float(got) - float(want)) < 1e-5 * abs(float(want))
