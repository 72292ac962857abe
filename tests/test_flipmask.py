"""The reversed-order IAF step (``multiconv2d(..., flipmask=True)``, IAF_VARIANT_THEANO_FLIPMASK) on the CPU.

* the oracle (tests/flipmask_oracle.py) and the host masks against tests/golden/flipmask.npz, i.e. the reference's
  graphy/nodes/ar.py executed with flipmask=True (tests/golden/make_golden_flipmask.py);
* strict triangularity of the flipped step in the reversed order, by fp64 autograd;
* the SIMT kernels under host emulation (tests/emu) against fp64 autograd: step, multiconv and layer, forward and
  backward, the training pairs, the pad channel's centre gradient and the exact zeros;
* the Python front-end's argument checks.
"""
import os

import numpy as np
import pytest
import torch

from iaf_b200 import masks as M
from oracle import iaf_oracle as O
from tests import flipmask_oracle as FO
from tests.emu.harness import EmuOperator
from tests.golden.cases import checksum
from tests.golden.make_golden_flipmask import FLIP_CASES, MASK_SHAPES, case_inputs

TOL = 2e-5  # fp32 kernels vs fp64 autograd, relative to the largest entry of each tensor (as tests/test_emu_kernels.py)
GOLDEN = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "flipmask.npz"))


def _rel(a, b):
    b = b.detach().numpy() if hasattr(b, "detach") else np.asarray(b)
    assert np.isfinite(a).all()
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def _torch_params(ls, grad=True):
    out = [{k: torch.from_numpy(np.asarray(v, np.float64)).requires_grad_(grad) for k, v in l.items()} for l in ls]
    return out


# ---------------------------------------------------------------------------------------------------------------------
# against the reference
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_in,n_out", MASK_SHAPES)
@pytest.mark.parametrize("zd", [False, True])
def test_masks_and_postup_match_the_reference(n_in, n_out, zd):
    ref = GOLDEN["mask_%d_%d_%d" % (n_in, n_out, zd)]
    assert np.array_equal(M.theano_conv_ar_mask(n_in, n_out, (3, 3), zd, flipmask=True), ref)
    assert np.array_equal(FO.conv_ar_mask(n_in, n_out, zd, True), ref)
    # the pad channel (last) inherits channel 0's centre column; channel 0 never sees the centre
    assert not ref[:, 0, 1, 1].any()
    if not zd:
        assert ref[:, n_in, 1, 1].all()


def test_postup_of_the_factory_applies_the_flipped_mask():
    from iaf_b200 import multiconv2d
    w = {}
    try:
        f = multiconv2d("pf", 4, [8], [4, 4], flipmask=True, nl="elu", w=w, device="cpu")
    except (RuntimeError, OSError):
        pytest.skip("the operator library is not built")
    upd = {n + "_w": torch.ones_like(w[n + "_w"]) for n in f.names}
    upd = f.postup(upd, w)
    for n, (cin, cout, zd) in zip(f.names, ((4, 8, False), (8, 4, True), (8, 4, True))):
        assert np.array_equal(upd[n + "_w"].numpy(), GOLDEN["mask_%d_%d_%d" % (cin, cout, zd)])
        assert not (w[n + "_w"].numpy()[GOLDEN["mask_%d_%d_%d" % (cin, cout, zd)] == 0]).any()  # ar.py:288


@pytest.mark.parametrize("ci", range(len(FLIP_CASES)), ids=[c[0] for c in FLIP_CASES])
def test_oracle_matches_the_reference(ci):
    name, B, n_z, hidden, heads, H, W, nl = FLIP_CASES[ci]
    hid, hd, z, ctx = case_inputs(ci, B, n_z, hidden, heads, H, W)
    assert checksum(z, ctx, *[v for l in hid + hd for v in l.values()]) == pytest.approx(float(GOLDEN[name + "_insum"]), rel=1e-12)
    f64 = lambda ls: O.cast_params(ls, np.float64)
    outs = FO.multiconv(z.astype(np.float64), ctx.astype(np.float64), f64(hid), f64(hd), nl)
    touts = FO.t_multiconv(torch.from_numpy(z).double(), torch.from_numpy(ctx).double(), _torch_params(hid, False),
                           _torch_params(hd, False), nl)
    for k in range(len(heads)):
        ref = GOLDEN["%s_out%d" % (name, k)]
        assert np.abs(outs[k] - ref).max() <= 1e-12 * max(np.abs(ref).max(), 1.0)
        assert np.abs(touts[k].numpy() - ref).max() <= 1e-12 * max(np.abs(ref).max(), 1.0)


def test_flipped_step_is_strictly_triangular_in_the_reversed_order():
    """d z'[c, y, x] / d z[c', y', x'] is zero unless (c', y', x') comes strictly before (c, y, x) in the flipped order
    (reverse raster, then descending channel): a later pixel in raster order, or the same pixel and a higher channel."""
    n_z, hidden, H, W = 4, [8], 3, 4
    hid, hd = O.make_params("theano", n_z, hidden, [n_z, n_z], seed=4)
    z = torch.from_numpy(np.random.RandomState(2).randn(1, n_z, H, W)).double().requires_grad_(True)
    ctx = torch.zeros(1, hidden[0], H, W, dtype=torch.float64)
    th, thh = _torch_params(hid, False), _torch_params(hd, False)
    f = lambda x: FO.t_iaf_step(x, ctx, th, thh)[0]
    J = torch.autograd.functional.jacobian(f, z).reshape(n_z, H, W, n_z, H, W).numpy()
    for c in range(n_z):
        for y in range(H):
            for x in range(W):
                for c2 in range(n_z):
                    for y2 in range(H):
                        for x2 in range(W):
                            before = (y2, x2) > (y, x) or ((y2, x2) == (y, x) and c2 > c)
                            if (c2, y2, x2) == (c, y, x):
                                assert J[c, y, x, c2, y2, x2] != 0  # the affine term
                            elif not before:
                                assert J[c, y, x, c2, y2, x2] == 0, (c, y, x, c2, y2, x2)
    # the channel dependence at one pixel is not empty (the test above would pass for a purely spatial mask)
    assert np.abs(J[:, 1, 1, :, 1, 1] - np.diag(np.diag(J[:, 1, 1, :, 1, 1]))).sum() > 0


# ---------------------------------------------------------------------------------------------------------------------
# the SIMT kernels under host emulation
# ---------------------------------------------------------------------------------------------------------------------
STEP_CASES = [
    # n_z, hidden, H, W, B, nl  (the shape mix of tests/test_emu_kernels.STEP_CASES, flipped)
    (4, [8], 4, 4, 2, "elu"),
    (8, [16, 16], 6, 9, 1, "softplus"),   # two hidden layers, W > 8: two pixel segments
    (8, [16, 16], 5, 7, 2, "elu"),        # non-square
    (6, [12], 3, 5, 2, "relu"),           # channel counts off the vector widths
    (4, [], 4, 4, 2, "elu"),              # depth_ar = 0
    (16, [80], 4, 4, 1, "elu"),           # > 64 channels: several ci / column blocks in the weight gradient
    (4, [8], 12, 24, 1, "leakyrelu"),     # several row bands
    (4, [4], 2, 2, 40, "elu"),            # more (sample, band) units than weight-gradient CTAs
    (8, [4], 5, 6, 2, "elu"),             # hidden narrower than z
]


def _setup(n_z, hidden, heads, H, W, B, nl, seed=1):
    hid, hd = O.make_params("theano", n_z, hidden, heads, seed=seed)
    z, ctx = O.make_inputs(B, n_z, hidden[0] if hidden else 1, H, W, seed=0)
    op = EmuOperator("theano_flipmask", n_z, hidden, heads, H, W, nl=nl).set_weights(
        [tuple(l[k] for k in "wsb") for l in hid + hd])
    return op, hid, hd, z, (ctx if hidden else None)


def _check_param_grads(gw, gs, gb, th, n_hidden):
    for i, l in enumerate(th):
        for g, k in zip((gw[i], gs[i], gb[i]), "wsb"):
            assert _rel(g, l[k].grad) < TOL, (i, k)
        zd = i >= n_hidden
        cin, cout = gw[i].shape[1] - 1, gw[i].shape[0]
        mask = FO.conv_ar_mask(cin, cout, zd, True)
        assert (gw[i][mask == 0] == 0).all()                         # masked taps: exactly zero
        if zd:
            assert (gw[i][:FO.zero_rows(cin, cout), :, 1, 1] == 0).all()  # l2normalize's zeroed rows: exactly zero
        # the pad channel's centre: live in the mask, reaches no output, gradient -k*v through the norm (nonzero)
        live = mask[:, cin, 1, 1] > 0
        if zd:
            live[:FO.zero_rows(cin, cout)] = False
        if live.any():
            assert (gw[i][live, cin, 1, 1] != 0).all()


@pytest.mark.parametrize("n_z,hidden,H,W,B,nl", STEP_CASES)
def test_emulated_flipped_step_forward_and_backward(n_z, hidden, H, W, B, nl):
    op, hid, hd, z, ctx = _setup(n_z, hidden, [n_z, n_z], H, W, B, nl)
    zo, ls, ld = op.step(z, ctx)
    th, thh = _torch_params(hid), _torch_params(hd)
    zt = torch.from_numpy(z).double().requires_grad_(True)
    ct = torch.from_numpy(ctx).double().requires_grad_(True) if ctx is not None else None
    zn, lsd, ldt = FO.t_iaf_step(zt, ct, th, thh, nl=nl)
    assert _rel(zo, zn) < 1e-5 and _rel(ls, lsd) < 1e-5 and _rel(ld, ldt) < 1e-5
    rng = np.random.RandomState(5)
    gzo, gls = rng.randn(*z.shape).astype(np.float32), rng.randn(*z.shape).astype(np.float32)
    gld = rng.randn(B).astype(np.float32)
    g_z, g_ctx, gw, gs, gb = op.step_bwd(z, ctx, gzo, gls, gld)
    ((zn * torch.from_numpy(gzo)).sum() + (lsd * torch.from_numpy(gls)).sum() + (ldt * torch.from_numpy(gld)).sum()).backward()
    assert _rel(g_z, zt.grad) < TOL and (ctx is None or _rel(g_ctx, ct.grad) < TOL)
    _check_param_grads(gw, gs, gb, th + thh, len(hidden))
    # training pair
    zo2, ls2, ld2, hs = op.step_train(z, ctx)
    assert np.array_equal(zo2, zo) and np.array_equal(ls2, ls) and np.array_equal(ld2, ld)
    s_z, s_ctx, sw, ss, sb = op.step_bwd_saved(z, ctx, zo2, ls2, hs, gzo, gls, gld)
    assert _rel(s_z, zt.grad) < TOL and (ctx is None or _rel(s_ctx, ct.grad) < TOL)
    _check_param_grads(sw, ss, sb, th + thh, len(hidden))


@pytest.mark.parametrize("n_z,hidden,heads", [(4, [8], [4, 4]), (4, [4], [8]), (8, [4], [8, 8]), (6, [12], [6])])
def test_emulated_flipped_multiconv_forward_and_backward(n_z, hidden, heads):
    H, W, B = 4, 5, 2
    op, hid, hd, z, ctx = _setup(n_z, hidden, heads, H, W, B, "elu")
    outs = op.multiconv(z, ctx)
    th, thh = _torch_params(hid), _torch_params(hd)
    zt, ct = torch.from_numpy(z).double().requires_grad_(True), torch.from_numpy(ctx).double().requires_grad_(True)
    ref = FO.t_multiconv(zt, ct, th, thh)
    for o, r in zip(outs, ref):
        assert _rel(o, r) < 1e-5
    rng = np.random.RandomState(3)
    g_outs = [rng.randn(*o.shape).astype(np.float32) for o in outs]
    sum((r * torch.from_numpy(g)).sum() for r, g in zip(ref, g_outs)).backward()
    g_z, g_ctx, gw, gs, gb = op.multiconv_bwd(z, ctx, g_outs)
    assert _rel(g_z, zt.grad) < TOL and _rel(g_ctx, ct.grad) < TOL
    _check_param_grads(gw, gs, gb, th + thh, len(hidden))
    outs2, hs = op.multiconv_train(z, ctx)
    assert all(np.array_equal(a, b) for a, b in zip(outs2, outs))
    s = op.multiconv_bwd_saved(z, ctx, hs, g_outs)
    assert _rel(s[0], zt.grad) < TOL and _rel(s[1], ct.grad) < TOL
    _check_param_grads(s[2], s[3], s[4], th + thh, len(hidden))


@pytest.mark.parametrize("n_z,hidden,H,W,B", [(4, [8], 4, 5, 2), (4, [], 3, 3, 2)])
def test_emulated_flipped_layer_forward_and_backward(n_z, hidden, H, W, B):
    op, hid, hd, _, _ = _setup(n_z, hidden, [n_z, n_z], H, W, B, "elu")
    rng = np.random.RandomState(11)
    a = [rng.randn(B, n_z, H, W), 0.5 * rng.randn(B, n_z, H, W), 0.3 * rng.randn(B, n_z, H, W),
         0.5 * rng.randn(B, n_z, H, W), 0.3 * rng.randn(B, n_z, H, W)]
    ctx = 0.1 * rng.randn(B, hidden[0] if hidden else 1, H, W)
    a32 = [x.astype(np.float32) for x in a] + [ctx.astype(np.float32)]
    zo, kl, kl_bc, kl_cost = op.layer(*a32)
    ts = [torch.from_numpy(x.astype(np.float64)).requires_grad_(True) for x in a32]
    th, thh = _torch_params(hid), _torch_params(hd)
    ref = FO.t_stochastic_layer(*ts[:5], ts[5] if hidden else None, th, thh)
    for o, r in zip((zo, kl, kl_bc, kl_cost), ref):
        assert _rel(o, r) < 1e-5
    g = [rng.randn(*o.shape).astype(np.float32) for o in (zo, kl, kl_bc, kl_cost)]
    sum((r * torch.from_numpy(x)).sum() for r, x in zip(ref, g)).backward()
    outs, g_ctx, gw, gs, gb = op.layer_bwd(*a32, *g)
    for o, t in zip(outs, (ts[1], ts[2], ts[3], ts[4], ts[0])):  # post_mean, post_logsd, prior_mean, prior_logsd, eps
        assert _rel(o, t.grad) < TOL
    if hidden:
        assert _rel(g_ctx, ts[5].grad) < TOL
    _check_param_grads(gw, gs, gb, th + thh, len(hidden))


def test_emulated_algorithmic_flops_count_the_flipped_mask():
    from tests.emu.harness import emu
    import ctypes as C
    for n_z, hidden in ((4, [8]), (8, [4]), (32, [64])):
        op, _, _, _, _ = _setup(n_z, hidden, [n_z, n_z], 4, 4, 1, "elu")
        sizes, nnz = [n_z] + hidden, 0
        for i in range(len(hidden) + 2):
            cin, cout, zd = (sizes[i], sizes[i + 1], False) if i < len(hidden) else (sizes[-1], n_z, True)
            m = FO.conv_ar_mask(cin, cout, zd, True).copy()
            if zd:
                m[:FO.zero_rows(cin, cout), :, 1, 1] = 0
            nnz += int(m[:, :cin].sum())   # real input channels (the pad channel only ever meets the border)
        flops = emu().iaf_plan_algorithmic_flops(op.plan, C.c_int(3))
        assert flops == 2.0 * 3 * 4 * 4 * nnz


def test_flipmask_front_end_checks():
    from iaf_b200 import ops
    with pytest.raises(ValueError):
        ops.IAFOperator("tf", 4, [8], [4, 4], flipmask=True)
    with pytest.raises(ValueError):
        ops.IAFOperator("theano_flipmask", 4, [8], [4, 4])
