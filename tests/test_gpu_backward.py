"""GPU parity of the backward (SURVEY 8f-4): iaf_step_bwd / iaf_multiconv_bwd through the C ABI and through the
python operator's autograd node, against torch autograd (fp64, CPU) over oracle/iaf_oracle_torch.py -- i.e. what
theano.grad / tf.gradients derive for models.py:281-285 + ar.py:396-416 | tf_train.py:69-72 + layers.py:158-166,
weight normalisation and mask included.  The same comparisons run on the CPU under host emulation in
tests/test_emu_kernels.py; tolerance here: ||delta||_inf / ||ref||_inf <= 1e-4 per tensor."""
import numpy as np
import pytest
import torch

from oracle import iaf_oracle as O
from oracle import iaf_oracle_torch as OT

pytestmark = pytest.mark.gpu
TOL = 1e-4


def _keys(variant):
    return ("V", "g", "b") if variant == "tf" else ("w", "s", "b")


def _rel(a, ref):
    a = a.detach().double().cpu().numpy()
    ref = ref.detach().numpy()
    assert np.isfinite(a).all()
    return float(np.abs(a - ref).max() / max(np.abs(ref).max(), 1e-30))


def _build(variant, n_z, hidden, heads, H, W, B, nl, path="auto"):
    from iaf_b200 import IAFOperator
    hid, hd = O.make_params(variant, n_z, hidden, heads, seed=1)
    z, ctx = O.make_inputs(B, n_z, hidden[0] if hidden else 1, H, W, seed=0)
    keys = _keys(variant)
    dev = [tuple(torch.from_numpy(np.ascontiguousarray(l[k])).cuda().requires_grad_(True) for k in keys) for l in hid + hd]
    op = IAFOperator(variant, n_z, hidden, heads, nl=nl, path=path).set_weights(dev)
    f64 = lambda ls: O.cast_params(ls, np.float64)
    th, thh = OT.to_torch(f64(hid), torch.float64), OT.to_torch(f64(hd), torch.float64)
    for l in th + thh:
        for k in l:
            l[k].requires_grad_(True)
    return op, dev, th, thh, z, (ctx if hidden else None)


BWD_CASES = [
    # variant, n_z, hidden, H, W, B, nl
    ("tf", 32, [64], 16, 16, 4, "elu"),            # C2a shape (forward on the tensor cores)
    ("tf", 32, [160, 160], 16, 16, 2, "elu"),      # C2b / C3 shape (forward on the tensor cores)
    ("theano", 32, [64], 8, 8, 3, "elu"),          # C1 level 1
    ("theano", 32, [160, 160], 16, 16, 2, "softplus"),  # C4 shape, cvae1's default nl
    ("tf", 8, [16, 16], 5, 7, 2, "elu"),
    ("tf", 6, [12], 3, 5, 2, "tanh"),              # channel counts off the vector widths
    ("theano", 6, [12], 3, 19, 2, "relu"),         # three pixel segments
    ("theano", 4, [], 4, 4, 2, "elu"),             # depth_ar = 0 (SURVEY F8)
    ("tf", 4, [8], 40, 24, 1, "leakyrelu"),        # several row bands
    ("theano", 4, [4], 2, 2, 70, "elu"),           # more (sample, band) units than weight-gradient CTAs
    ("tf", 16, [32], 16, 16, 3, "elu"),            # tensor cores, padded column groups (one-launch forward)
    ("theano", 16, [48, 48], 8, 8, 2, "elu"),      # tensor cores, padded column groups (per-stage forward, 48-wide data
                                                   # gradient and weight gradient)
]


@pytest.mark.parametrize("case", BWD_CASES, ids=lambda c: "%s-%s-%dx%d" % (c[0], "x".join(map(str, c[2])) or "0", c[3], c[4]))
def test_step_backward_through_autograd(case):
    variant, n_z, hidden, H, W, B, nl = case
    op, dev, th, thh, z, ctx = _build(variant, n_z, hidden, [n_z, n_z], H, W, B, nl)
    zg = torch.from_numpy(z).cuda().requires_grad_(True)
    cg = torch.from_numpy(ctx).cuda().requires_grad_(True) if ctx is not None else None
    zt = torch.from_numpy(z).double().requires_grad_(True)
    ct = torch.from_numpy(ctx).double().requires_grad_(True) if ctx is not None else None
    rng = np.random.RandomState(5)
    gzo, gls = rng.randn(*z.shape).astype(np.float32), rng.randn(*z.shape).astype(np.float32)
    gld = rng.randn(B).astype(np.float32)
    zo, ls, ld = op.step(zg, cg)
    (zo * torch.from_numpy(gzo).cuda()).sum().add((ls * torch.from_numpy(gls).cuda()).sum()).add(
        (ld * torch.from_numpy(gld).cuda()).sum()).backward()
    zn, lsd, ldt = OT.iaf_step(variant, zt, ct, th, thh, nl=nl)
    ((zn * torch.from_numpy(gzo)).sum() + (lsd * torch.from_numpy(gls)).sum() + (ldt * torch.from_numpy(gld)).sum()).backward()
    assert _rel(zg.grad, zt.grad) < TOL
    if ctx is not None:
        assert _rel(cg.grad, ct.grad) < TOL
    keys = _keys(variant)
    for i, l in enumerate(th + thh):
        for t, k in zip(dev[i], keys):
            assert t.grad is not None and _rel(t.grad, l[k].grad) < TOL, (i, k)
        zd = i >= len(hidden)
        gw = dev[i][0].grad.cpu().numpy()
        mask = (O.get_conv_ar_mask(3, 3, gw.shape[2], gw.shape[3], zd) if variant == "tf"
                else O.theano_conv_ar_mask(gw.shape[1] - 1, gw.shape[0], (3, 3), zd))
        assert (gw[mask == 0] == 0).all()   # masked taps: exactly zero (the postup contract, ar.py:369-373)


@pytest.mark.parametrize("variant,n_z,hidden,heads", [("tf", 32, [64], [32, 32]), ("theano", 4, [8], [8]),
                                                       ("theano", 6, [12], [6])])
def test_multiconv_backward_through_autograd(variant, n_z, hidden, heads):
    H, W, B = 8, 8, 2
    op, dev, th, thh, z, ctx = _build(variant, n_z, hidden, heads, H, W, B, "elu")
    zg, cg = torch.from_numpy(z).cuda().requires_grad_(True), torch.from_numpy(ctx).cuda().requires_grad_(True)
    zt, ct = torch.from_numpy(z).double().requires_grad_(True), torch.from_numpy(ctx).double().requires_grad_(True)
    outs = op.multiconv(zg, cg)
    ref = OT.multiconv(variant, zt, ct, th, thh)
    rng = np.random.RandomState(3)
    gs = [rng.randn(*o.shape).astype(np.float32) for o in outs]
    sum((o * torch.from_numpy(g).cuda()).sum() for o, g in zip(outs, gs)).backward()
    sum((r * torch.from_numpy(g)).sum() for r, g in zip(ref, gs)).backward()
    assert _rel(zg.grad, zt.grad) < TOL and _rel(cg.grad, ct.grad) < TOL
    for i, l in enumerate(th + thh):
        for t, k in zip(dev[i], _keys(variant)):
            assert _rel(t.grad, l[k].grad) < TOL, (i, k)


def test_theano_factory_is_differentiable_and_postup_keeps_the_mask():
    """multiconv2d(...) (ar.py:378-423): gradients flow to the {name}_{i}_w/_b/_s entries of w, and a plain SGD update
    followed by postup() leaves the masked taps at zero."""
    from iaf_b200 import multiconv2d
    w = {}
    f = multiconv2d("pc", 4, [8], [4, 4], w=w, nl="elu")
    for k in w:
        w[k].requires_grad_(True)
    z, ctx = torch.randn(2, 4, 6, 6, device="cuda"), 0.1 * torch.randn(2, 8, 6, 6, device="cuda")
    m, s = f(z, ctx, w)
    (m.square().sum() + s.sum()).backward()
    assert all(w[k].grad is not None and torch.isfinite(w[k].grad).all() for k in w)
    upd = f.postup({k: (w[k] - 0.1 * w[k].grad).detach() for k in w if k.endswith("_w")}, w)
    for n in f.names:
        zd = "_out_" in n
        mask = O.theano_conv_ar_mask(w[n + "_w"].shape[1] - 1, w[n + "_w"].shape[0], (3, 3), zd)
        assert bool((upd[n + "_w"].cpu().numpy()[mask == 0] == 0).all())


@pytest.mark.parametrize("hidden", [[64], [160, 160]], ids=["c2a", "c2b"])
def test_backward_full_size_properties(hidden):
    """B = 256 (BASELINE.json's batch), where the fp64 oracle is too slow: the backward is linear in the upstream
    gradients, per-sample input gradients do not depend on the rest of the batch (bit-equal on a sub-batch), repeated
    runs are bit-identical (fixed-order reductions), and parameter gradients are the sum over sub-batches."""
    from iaf_b200 import IAFOperator
    n_z, H, W, B = 32, 16, 16, 256
    hid, hd = O.make_params("tf", n_z, hidden, [n_z, n_z], seed=1)
    z, ctx = O.make_inputs(B, n_z, hidden[0], H, W, seed=0)
    dev = [tuple(torch.from_numpy(np.ascontiguousarray(l[k])).cuda() for k in "Vgb") for l in hid + hd]
    op = IAFOperator("tf", n_z, hidden, [n_z, n_z], nl="elu").set_weights(dev)
    zg, cg = torch.from_numpy(z).cuda(), torch.from_numpy(ctx).cuda()
    g = torch.Generator(device="cuda").manual_seed(3)
    g1, g2 = (torch.randn(z.shape, device="cuda", generator=g) for _ in range(2))
    l1 = torch.randn(B, device="cuda", generator=g)
    a = op.step_backward(zg, cg, g1, None, l1)
    b = op.step_backward(zg, cg, g1, None, l1)
    flat = lambda r: [r[0], r[1]] + list(r[2]) + list(r[3]) + list(r[4])
    for x, y in zip(flat(a), flat(b)):
        assert torch.equal(x, y)
    c = op.step_backward(zg, cg, g2, g1, None)
    d = op.step_backward(zg, cg, 2.0 * g1 - 0.5 * g2, -0.5 * g1, 2.0 * l1)
    for x, y, w_ in zip(flat(a), flat(c), flat(d)):
        ref = 2.0 * x.double() - 0.5 * y.double()
        assert float((w_.double() - ref).abs().max()) <= 1e-4 * max(float(ref.abs().max()), 1e-6)
    # the autograd node (training forward on the tensor-core kernels keeps the activations, backward without recompute)
    # agrees with the recompute path
    zr, cr = zg.clone().requires_grad_(True), cg.clone().requires_grad_(True)
    pr = [tuple(t.clone().requires_grad_(True) for t in l) for l in dev]
    op2 = IAFOperator("tf", n_z, hidden, [n_z, n_z], nl="elu").set_weights(pr)
    zo, ls, ld = op2.step(zr, cr)
    ((zo * g1).sum() + (ld * l1).sum()).backward()
    got = [zr.grad, cr.grad] + [l[0].grad for l in pr] + [l[1].grad for l in pr] + [l[2].grad for l in pr]
    for x, y in zip(got, flat(a)):
        assert float((x.double() - y.double()).abs().max()) <= 1e-4 * max(float(y.abs().max()), 1e-6)
    # sub-batches: input gradients bit-equal, parameter gradients add up
    h = B // 2
    lo = op.step_backward(zg[:h].contiguous(), cg[:h].contiguous(), g1[:h].contiguous(), None, l1[:h].contiguous())
    hi = op.step_backward(zg[h:].contiguous(), cg[h:].contiguous(), g1[h:].contiguous(), None, l1[h:].contiguous())
    assert torch.equal(lo[0], a[0][:h]) and torch.equal(hi[1], a[1][h:])
    for x, y, w_ in zip(flat(lo)[2:], flat(hi)[2:], flat(a)[2:]):
        ref = x.double() + y.double()
        assert float((w_.double() - ref).abs().max()) <= 1e-4 * max(float(ref.abs().max()), 1e-6)


def test_backward_error_behaviour():
    from iaf_b200 import IAFOperator
    hid, hd = O.make_params("tf", 4, [8], [4, 4], seed=1)
    dev = [tuple(torch.from_numpy(np.ascontiguousarray(l[k])).cuda() for k in "Vgb") for l in hid + hd]
    op = IAFOperator("tf", 4, [8], [4, 4]).set_weights(dev)
    z, ctx = torch.randn(2, 4, 4, 4, device="cuda"), torch.randn(2, 8, 4, 4, device="cuda")
    with pytest.raises((ValueError, RuntimeError, TypeError)):
        op.step_backward(z, ctx, torch.randn(2, 4, 4, 4))            # CPU gradient: no CPU fallback
    with pytest.raises((ValueError, TypeError)):
        op.step_backward(z, ctx, torch.randn(2, 4, 4, 4, device="cuda", dtype=torch.float64))
    # no gradient requested anywhere: the forward is not recorded
    zo, _, _ = op.step(z, ctx)
    assert not zo.requires_grad


@pytest.mark.parametrize("variant,hidden,H,W,nl", [("tf", [64], 16, 16, "elu"), ("theano", [160, 160], 16, 16, "softplus"),
                                                   ("tf", [160, 160], 8, 8, "elu")],
                         ids=["c2a", "c4-softplus", "c3-8x8"])
def test_tensor_core_backward_is_taken_and_matches_the_simt_backward(variant, hidden, H, W, nl, monkeypatch):
    """The backward of a tensor-core plan runs its data gradient (layered-kernel stage on the point-reflected stream) and
    its weight gradient (MN-major wgmma over the slot stream) on the tensor cores -- `backward_path` says so -- and agrees
    with the exact-fp32 SIMT backward of the same operator (IAF_BWD_TC=0) within the parity tolerance; a plan pinned to the
    SIMT path keeps the SIMT backward."""
    n_z, B = 32, 5
    rng = np.random.RandomState(11)

    def grads(env):
        if env is not None:
            monkeypatch.setenv("IAF_BWD_TC", env)
        else:
            monkeypatch.delenv("IAF_BWD_TC", raising=False)
        op, dev, _, _, z, ctx = _build(variant, n_z, hidden, [n_z, n_z], H, W, B, nl)
        path = op.backward_path(H, W, "cuda")
        zg = torch.from_numpy(z).cuda().requires_grad_(True)
        cg = torch.from_numpy(ctx).cuda().requires_grad_(True)
        r = np.random.RandomState(5)
        gzo, gls = r.randn(*z.shape).astype(np.float32), r.randn(*z.shape).astype(np.float32)
        gld = r.randn(B).astype(np.float32)
        zo, ls, ld = op.step(zg, cg)
        (zo * torch.from_numpy(gzo).cuda()).sum().add((ls * torch.from_numpy(gls).cuda()).sum()).add(
            (ld * torch.from_numpy(gld).cuda()).sum()).backward()
        return path, [zg.grad, cg.grad] + [t.grad for l in dev for t in l]

    p_tc, g_tc = grads(None)
    p_simt, g_simt = grads("0")
    assert p_tc == "tc" and p_simt == "simt", (p_tc, p_simt)
    for a, b in zip(g_tc, g_simt):
        assert torch.isfinite(a).all()
        assert float((a.double() - b.double()).abs().max()) <= TOL * max(float(b.abs().max()), 1e-30)
    monkeypatch.delenv("IAF_BWD_TC", raising=False)
    op = _build(variant, n_z, hidden, [n_z, n_z], H, W, B, nl, path="simt")[0]
    assert op.backward_path(H, W, "cuda") == "simt"
    del rng


def test_tensor_core_backward_is_scale_invariant():
    """Gradients 2^-40 and 2^+20 times the usual size go through the fp16 operand images unharmed: every sample is scaled by
    a power of two taken from its own largest gradient (exact to undo), so the result is the usual one times that factor."""
    variant, n_z, hidden, H, W, B, nl = "tf", 32, [64], 16, 16, 3, "elu"
    op, dev, _, _, z, ctx = _build(variant, n_z, hidden, [n_z, n_z], H, W, B, nl)
    assert op.backward_path(H, W, "cuda") == "tc"
    r = np.random.RandomState(5)
    gzo = torch.from_numpy(r.randn(*z.shape).astype(np.float32)).cuda()
    out = []
    for f in (1.0, 2.0 ** -40, 2.0 ** 20):
        zg = torch.from_numpy(z).cuda().requires_grad_(True)
        cg = torch.from_numpy(ctx).cuda().requires_grad_(True)
        for l in dev:
            for t in l:
                t.grad = None
        zo, ls, ld = op.step(zg, cg)
        (zo * (gzo * f)).sum().backward()
        out.append([zg.grad / f, cg.grad / f] + [t.grad / f for l in dev for t in l])
    for other in out[1:]:
        for a, b in zip(out[0], other):
            assert torch.isfinite(b).all()
            assert float((a.double() - b.double()).abs().max()) <= 1e-5 * max(float(a.abs().max()), 1e-30)


def test_tensor_core_backward_after_a_larger_batch():
    """The operand images of the tensor-core backward outlive a call: a smaller batch after a larger one must give what a
    fresh operator gives (the weight gradient sums over every slot of every K tile, so stale slots would show up there)."""
    variant, n_z, hidden, H, W, nl = "tf", 32, [64], 16, 16, "elu"

    def run(op, dev, B):
        z, ctx = O.make_inputs(B, n_z, hidden[0], H, W, seed=3)
        zg = torch.from_numpy(z).cuda().requires_grad_(True)
        cg = torch.from_numpy(ctx).cuda().requires_grad_(True)
        for l in dev:
            for t in l:
                t.grad = None
        zo, ls, ld = op.step(zg, cg)
        (zo.sum() + 0.5 * ls.sum() - ld.sum()).backward()
        return [zg.grad.clone(), cg.grad.clone()] + [t.grad.clone() for l in dev for t in l]

    op, dev = _build(variant, n_z, hidden, [n_z, n_z], H, W, 2, nl)[:2]
    assert op.backward_path(H, W, "cuda") == "tc"
    run(op, dev, 9)
    got = run(op, dev, 5)
    op2, dev2 = _build(variant, n_z, hidden, [n_z, n_z], H, W, 2, nl)[:2]
    want = run(op2, dev2, 5)
    # not bit-equal: the number of split-K groups of the weight gradient is fixed when the scratch is sized (for the larger
    # batch here), so the summation order differs; slots left over from the larger batch would be an O(1) error
    for a, b in zip(got, want):
        assert float((a.double() - b.double()).abs().max()) <= 1e-5 * max(float(b.abs().max()), 1e-30)


@pytest.mark.parametrize("variant,hidden,H,W", [("tf", [32], 16, 16), ("theano", [48, 48], 8, 8)],
                         ids=["one-launch", "per-stage"])
def test_padded_column_group_shapes_run_on_the_tensor_cores(variant, hidden, H, W):
    """The n_z = 16 cases of BWD_CASES (and of test_gpu_parity's STEP_CASES) exercise the padded column groups of the wgmma
    kernels -- stages whose width is an odd multiple of 16 -- only if they run there: forward and backward of both shapes
    are on the tensor cores."""
    op = _build(variant, 16, hidden, [16, 16], H, W, 2, "elu")[0]
    assert op.path_used(H, W, "cuda") == "tc"
    assert op.backward_path(H, W, "cuda") == "tc"
