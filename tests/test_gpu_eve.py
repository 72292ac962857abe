"""H100 checks of the fused Eve step (iaf_b200.optim.Eve, iaf_eve_kernel) and of the Theano model's Eve train_step:

* 50 steps are bit-identical to the op-by-op fp32 restatement (tests/eve_oracle.py) on the GPU, in the parameters,
  every state buffer, the averages and the lookahead, at a c2a-shaped Theano set (134 tensors, 2.84 M elements) and at
  a small one; one launch per step;
* a captured step replayed 10 times equals 10 eager steps bit for bit, on a side stream too;
* after a step, CudaIAF on ``averaged()`` and CudaIAFTrain on ``lookahead()`` equal freshly built ones (the step bumps
  the version counters their packed-weight caches key on);
* 100 training steps leave every masked tap of every AR weight at exactly zero in w, w', mom1 and delta;
* 20 Eve ``train_step``s at small shapes follow an fp64 oracle training loop (oracle gradients, fp64 restated Eve) in
  the parameters, the lookahead, the averages and the bits/dim evaluated at ``averaged()``.
TF32 is off throughout, so the model's stock convs run in fp32."""
import numpy as np
import pytest
import torch

from iaf_b200 import _lib
from iaf_b200 import elbo_theano as ET
from iaf_b200.masks import theano_conv_ar_mask
from iaf_b200.optim import Eve
from oracle.elbo_oracle import TorchIAFTheano
from tests.eve_oracle import RestatedEve

pytestmark = pytest.mark.gpu

TH_C2A = dict(n_z=32, n_h1=64, n_h2=64, depths=[2, 2, 2], depth_ar=1, nl="elu", kl_min=0.25, image_size=32)
TH_SMALL = dict(n_z=4, n_h1=4, n_h2=8, depths=[1, 1], depth_ar=1, nl="elu", kl_min=0.1, image_size=8)
STATE = ("mom1", "mom_max", "delta", "avg")


@pytest.fixture(autouse=True)
def _no_tf32():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def _params(hps, seed=0, dtype=torch.float32, device="cuda"):
    return {k: torch.tensor(np.asarray(v), dtype=dtype, device=device) for k, v in ET.make_params(hps, seed=seed).items()}


def _clone(p):
    return {k: v.detach().clone() for k, v in p.items()}


def _set_grads(la, gen, step):
    out = {}
    for i, (k, p) in enumerate(la.items()):
        scale = 10.0 ** ((i + step) % 7 - 3)
        g = torch.randn(p.shape, generator=gen, device=p.device) * scale
        if (i + step) % 11 == 0:
            g = torch.zeros_like(g)
        p.grad = g
        out[k] = g
    return out


def _state(opt, name):
    """{name: opt's slice of the flat state buffer ``name``} (the optimiser's offsets: 4-element aligned slices)."""
    buf, out, off = getattr(opt, name), {}, 0
    for k, p in zip(opt.names, opt.params):
        out[k] = buf[off:off + p.numel()].view(p.shape)
        off += -(-p.numel() // 4) * 4
    return out


def _assert_same(a, b, what):
    for k in a:
        assert torch.equal(a[k].detach(), b[k].detach()), "%s: %s differs" % (what, k)


def _assert_all_same(opt, p, ref, q):
    _assert_same(p, q, "parameters")
    _assert_same(opt.lookahead(), ref.lookahead(), "lookahead")
    _assert_same(opt.averaged(), ref.averaged(), "averages")
    for name in STATE:
        _assert_same(_state(opt, name), getattr(ref, name), name)


@pytest.mark.parametrize("hps", [TH_C2A, TH_SMALL], ids=["theano_c2a", "theano_small"])
def test_fused_step_bit_identical_to_restatement(hps):
    p = _params(hps)
    if hps is TH_C2A:
        assert len(p) == 134 and sum(t.numel() for t in p.values()) == 2_841_605
    q = _clone(p)
    opt, ref = Eve(p), RestatedEve(q)
    _assert_same(opt.lookahead(), ref.lookahead(), "initial lookahead")
    gen = torch.Generator(device="cuda").manual_seed(1)
    lib = _lib.lib()
    rla = ref.lookahead()
    for step in range(50):
        grads = _set_grads(opt.lookahead(), gen, step)
        for k in rla:
            rla[k].grad = grads[k].clone()
        if step % 9 == 4:                      # a missing gradient: a zero gradient
            opt.lookahead()["h_top"].grad = rla["h_top"].grad = None
        before = lib.iaf_adamax_launch_count()
        opt.step()
        assert lib.iaf_adamax_launch_count() - before == 1
        ref.step()
    torch.cuda.synchronize()
    _assert_all_same(opt, p, ref, q)
    assert not torch.equal(opt.lookahead()["h_top"], p["h_top"])


@pytest.mark.parametrize("side", [False, True], ids=["current_stream", "side_stream"])
def test_captured_step_replays_like_eager_steps(side):
    p = _params(TH_SMALL)
    q, p0 = _clone(p), _clone(p)
    opt, eager = Eve(p), Eve(q)
    gen = torch.Generator(device="cuda").manual_seed(2)
    grads = _set_grads(opt.lookahead(), gen, 0)
    for k, t in eager.lookahead().items():
        t.grad = grads[k].clone()
    warm = Eve({"w": torch.zeros(5, device="cuda")})
    warm.lookahead()["w"].grad = torch.ones(5, device="cuda")
    warm.step()                                # the kernel's module is loaded before the capture
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
    _assert_same(opt.lookahead(), eager.lookahead(), "lookahead")
    _assert_same(opt.averaged(), eager.averaged(), "averages")
    for name in STATE:
        assert torch.equal(getattr(opt, name), getattr(eager, name)), name
    assert sum(not torch.equal(p[k], p0[k]) for k in p) > len(p) // 2   # the replays did update


def _layer_inputs(hps, seed=3):
    g = torch.Generator(device="cuda").manual_seed(seed)
    nz, nh, S = hps["n_z"], hps["n_h2"], hps["image_size"] // 2
    r = lambda c, s=1.0: s * torch.randn((2, c, S, S), generator=g, device="cuda")
    return r(nz), r(nz), r(nz, 0.1), r(nz), r(nz, 0.1), r(nh)


def test_step_bumps_the_versions_the_layers_cache_on():
    p = _params(TH_SMALL)
    opt = Eve(p)
    avg, train = ET.CudaIAF(opt.averaged(), TH_SMALL), ET.CudaIAFTrain(opt.lookahead(), TH_SMALL)
    args = _layer_inputs(TH_SMALL)
    with torch.no_grad():
        avg("0_0", *args), train("0_0", *args)   # pack the weights
        gen = torch.Generator(device="cuda").manual_seed(4)
        for step in range(3):
            _set_grads(opt.lookahead(), gen, step)
            opt.step()
        for layer, fresh in ((avg, ET.CudaIAF(opt.averaged(), TH_SMALL)),
                             (train, ET.CudaIAFTrain(opt.lookahead(), TH_SMALL))):
            for a, b in zip(layer("0_0", *args), fresh("0_0", *args)):
                assert torch.equal(a, b)
    # and the training layer's autograd node sees the new lookahead too
    la = opt.lookahead()
    z = train("0_0", *args)[0]
    z.sum().backward()
    assert la["0_0_posterior_conv1_0_w"].grad is not None


def _ar_masks(params):
    """{name: mask} of every AR weight of the Theano posterior (raw layouts)."""
    out = {}
    for k, v in params.items():
        if "_posterior_conv1_" in k and k.endswith("_w"):
            out[k] = theano_conv_ar_mask(v.shape[1] - 1, v.shape[0], zerodiagonal="_out_" in k)
    return {k: torch.from_numpy(m).to(params[k].device) for k, m in out.items()}


def _batch(hps, seed, dtype=torch.float32, device="cuda"):
    g = torch.Generator().manual_seed(seed)
    S = hps["image_size"]
    x = torch.randint(0, 256, (4, 3, S, S), generator=g, dtype=torch.uint8)
    shapes = {(i, j): (4, hps["n_z"], S // 2 ** (i + 1), S // 2 ** (i + 1))
              for i in range(len(hps["depths"])) for j in range(hps["depths"][i])}
    noise = {k: torch.randn(s, generator=g, dtype=torch.float64) for k, s in sorted(shapes.items())}
    return x.to(device), {k: v.to(device=device, dtype=dtype) for k, v in noise.items()}


def test_masked_taps_stay_zero():
    p = _params(TH_SMALL)
    masks = _ar_masks(p)
    assert masks
    with torch.no_grad():
        for k, m in masks.items():
            p[k].mul_(m)                       # postup's re-mask (ar.py:369-373) on the initial weights
    p0 = _clone(p)
    opt = Eve(p)
    layer = ET.CudaIAFTrain(opt.lookahead(), TH_SMALL)
    for step in range(100):
        x, noise = _batch(TH_SMALL, step)
        ET.train_step(p, x, opt, TH_SMALL, noise=noise, iaf_layer=layer)
    torch.cuda.synchronize()
    mom1, delta = _state(opt, "mom1"), _state(opt, "delta")
    for k, m in masks.items():
        for what, t in (("w", p[k]), ("w'", opt.lookahead()[k]), ("mom1", mom1[k]), ("delta", delta[k]),
                        ("avg", opt.averaged()[k])):
            assert (t[m == 0] == 0).all(), "%s %s" % (what, k)
        assert not torch.equal(p[k][m != 0], p0[k][m != 0]), k   # the live taps did train


def _dist(a, b):
    return torch.sqrt(sum(((a[k].detach().double().cpu() - b[k].detach().double().cpu()) ** 2).sum() for k in a))


def test_train_steps_follow_fp64_oracle_loop():
    """Tolerances of the Adamax loop (tests/test_gpu_train.py): the parameters', lookahead's and averages' distance to
    the fp64 loop below 1e-3 of how far the fp64 loop moved them, the step's bits/dim to 1e-4 and the bits/dim at
    averaged() to 1e-5 relative."""
    hps = TH_SMALL
    p = _params(hps)
    r = _params(hps, dtype=torch.float64, device="cpu")
    p0 = _clone(r)
    opt, ropt = Eve(p), RestatedEve(r)
    layer = ET.CudaIAFTrain(opt.lookahead(), hps)
    rlayer = TorchIAFTheano(ropt.lookahead(), hps)
    for step in range(20):
        x, noise = _batch(hps, 100 + step)
        b = ET.train_step(p, x, opt, hps, noise=noise, iaf_layer=layer)
        xr, nr = _batch(hps, 100 + step, torch.float64, "cpu")
        rb = ET.train_step(r, xr, ropt, hps, noise=nr, iaf_layer=rlayer)
        assert abs(float(b) - float(rb)) < 1e-4 * abs(float(rb))
    torch.cuda.synchronize()
    for what, got, want in (("params", p, r), ("lookahead", opt.lookahead(), ropt.lookahead()),
                            ("averages", opt.averaged(), ropt.averaged())):
        moved, d = _dist(want, p0), _dist(got, want)
        print("|d %s| / |moved| = %.3e" % (what, d / moved))
        assert d < 1e-3 * moved, what

    avg, ravg = opt.averaged(), ropt.averaged()
    x, noise = _batch(hps, 999)
    xr, nr = _batch(hps, 999, torch.float64, "cpu")
    with torch.no_grad():
        got = ET.forward(avg, x, noise, ET.CudaIAF(avg, hps), hps)["bits_per_dim"]
        want = ET.forward(ravg, xr, nr, TorchIAFTheano(ravg, hps), hps)["bits_per_dim"]
    print("bits/dim at averaged() %.8f vs fp64 %.8f" % (float(got), float(want)))
    assert abs(float(got) - float(want)) < 1e-5 * abs(float(want))


def test_make_optimizer_builds_both():
    p = _params(TH_SMALL)
    a = ET.make_optimizer(p, dict(TH_SMALL, alpha=0.003))
    e = ET.make_optimizer(_clone(p), dict(TH_SMALL, optim="eve", beta1=0.2))
    assert a.rule == "theano" and a.lr == 0.003 and a.avg_decay == 1.0 - 0.001
    assert isinstance(e, Eve) and (e.lr, e.beta1, e.beta2, e.beta3) == (0.002, 0.2, 0.001, 0.01)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two CUDA devices")
def test_optimizer_refuses_mixed_devices():
    with pytest.raises(ValueError, match="the others on"):
        Eve({"a": torch.zeros(3, device="cuda:0"), "b": torch.zeros(3, device="cuda:1")})
