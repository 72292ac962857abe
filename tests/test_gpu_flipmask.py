"""GPU parity of the reversed-order IAF step (``multiconv2d(..., flipmask=True)``, IAF_VARIANT_THEANO_FLIPMASK) on both
kernel families, against the fp64 oracle of tests/flipmask_oracle.py (pinned to the reference by
tests/golden/flipmask.npz).  The flipped step runs the Theano parameterisation (pad-channel table) on the unreflected
image: on the tensor cores that combination exists only here.  Forward tolerance: ||delta||_inf / max(||ref||_inf, 1)
<= 1e-4 per sample; gradients: ||delta||_inf / ||ref||_inf <= 1e-4 per tensor."""
import numpy as np
import pytest
import torch

from oracle import iaf_oracle as O
from tests import flipmask_oracle as FO

pytestmark = pytest.mark.gpu
TOL = 1e-4


def _f64(ls):
    return O.cast_params(ls, np.float64)


def _per_sample(a, ref):
    a = a.detach().double().cpu().numpy() if hasattr(a, "detach") else np.asarray(a, np.float64)
    assert np.isfinite(a).all()
    a, ref = a.reshape(a.shape[0], -1), np.asarray(ref).reshape(a.shape[0], -1)
    return float((np.abs(a - ref).max(axis=1) / np.maximum(np.abs(ref).max(axis=1), 1.0)).max())


def _rel(a, ref):
    a = a.detach().double().cpu().numpy()
    ref = ref.detach().numpy()
    assert np.isfinite(a).all()
    return float(np.abs(a - ref).max() / max(np.abs(ref).max(), 1e-30))


def _op(n_z, hidden, heads, path, grad=False, seed=1, nl="elu"):
    from iaf_b200 import IAFOperator
    hid, hd = O.make_params("theano", n_z, hidden, heads, seed=seed)
    dev = [tuple(torch.from_numpy(np.ascontiguousarray(l[k])).cuda().requires_grad_(grad) for k in "wsb") for l in hid + hd]
    op = IAFOperator("theano", n_z, hidden, heads, nl=nl, path=path, flipmask=True).set_weights(dev)
    return op, dev, hid, hd


FWD_CASES = [
    # id, n_z, hidden, H, W, B, path, fused (IAF_TC_FUSED), expected path
    ("c1-onelaunch", 32, [64], 16, 16, 8, "tc", "1", "tc"),
    ("c1-perstage", 32, [64], 16, 16, 8, "tc", "0", "tc"),
    ("c1-simt", 32, [64], 16, 16, 4, "simt", "1", "simt"),
    ("160x160-16", 32, [160, 160], 16, 16, 4, "tc", "1", "tc"),
    ("160x160-8", 32, [160, 160], 8, 8, 8, "tc", "1", "tc"),
    ("160x160-8-simt", 32, [160, 160], 8, 8, 2, "simt", "1", "simt"),
    ("nonsquare-tc", 32, [64], 12, 20, 4, "tc", "1", "tc"),
    ("nonsquare-simt", 16, [32], 5, 11, 3, "simt", "1", "simt"),
]


@pytest.mark.parametrize("case", FWD_CASES, ids=lambda c: c[0])
def test_flipped_step_and_multiconv_forward(case, monkeypatch):
    _, n_z, hidden, H, W, B, path, fused, expect = case
    monkeypatch.setenv("IAF_TC_FUSED", fused)  # read when the plan is created
    op, _, hid, hd = _op(n_z, hidden, [n_z, n_z], path)
    z, ctx = O.make_inputs(B, n_z, hidden[0], H, W, seed=0)
    zr, lr, ldr = FO.iaf_step(z.astype(np.float64), ctx.astype(np.float64), _f64(hid), _f64(hd))
    zc, cc = torch.from_numpy(z).cuda(), torch.from_numpy(ctx).cuda()
    assert op.path_used(H, W, "cuda:0", "step") == expect  # (creates the plan and packs the weights)
    n0 = op.launch_count()
    zo, ls, ld = op.step(zc, cc)
    torch.cuda.synchronize()
    if expect == "tc" and fused == "1" and len(hidden) == 1:
        assert op.launch_count() - n0 == 1  # the one-launch step kernel
    assert _per_sample(zo, zr) < TOL and _per_sample(ls, lr) < TOL and _per_sample(ld[:, None], ldr[:, None]) < TOL
    m, s = op.multiconv(zc, cc)
    mr, sr = FO.multiconv(z.astype(np.float64), ctx.astype(np.float64), _f64(hid), _f64(hd))
    assert _per_sample(m, mr) < TOL and _per_sample(s, sr) < TOL
    # the flipped step is a different transform from the unflipped one
    zu, _, _ = O.iaf_step("theano", z.astype(np.float64), ctx.astype(np.float64), _f64(hid), _f64(hd))
    assert np.abs(zu - zr).max() > 1e-3


@pytest.mark.parametrize("path", ["tc", "simt"])
def test_flipped_fused_layer(path):
    n_z, hidden, H, W, B = 32, [64], 8, 8, 4
    op, _, hid, hd = _op(n_z, hidden, [n_z, n_z], path)
    rng = np.random.RandomState(11)
    eps, pm = rng.randn(B, n_z, H, W), 0.5 * rng.randn(B, n_z, H, W)
    pls, prm, prl = 0.3 * rng.randn(B, n_z, H, W), 0.5 * rng.randn(B, n_z, H, W), 0.3 * rng.randn(B, n_z, H, W)
    ctx = 0.1 * rng.randn(B, hidden[0], H, W)
    ins = [torch.from_numpy(a.astype(np.float32)).cuda() for a in (eps, pm, pls, prm, prl, ctx)]
    z, kl, kl_bc, kl_cost = op.layer(*ins)
    torch.cuda.synchronize()
    assert op.path_used(H, W, "cuda:0", "layer") == path
    T = lambda a: torch.from_numpy(a.astype(np.float32).astype(np.float64))
    th, thh = (OT_params(hid), OT_params(hd))
    ref = FO.t_stochastic_layer(*[T(a) for a in (eps, pm, pls, prm, prl, ctx)], th, thh)
    for a, r in zip((z, kl, kl_bc, kl_cost), ref):
        assert _per_sample(a, r.numpy()) < TOL


def OT_params(ls, grad=False):
    from oracle import iaf_oracle_torch as OT
    out = OT.to_torch(_f64(ls), torch.float64)
    for l in out:
        for k in l:
            l[k].requires_grad_(grad)
    return out


BWD_CASES = [
    # id, n_z, hidden, H, W, B, path, backward path
    ("c1-tc", 32, [64], 16, 16, 3, "tc", "tc"),
    ("160x160-tc", 32, [160, 160], 8, 8, 2, "tc", "tc"),
    ("nonsquare-tc", 16, [32], 10, 22, 2, "tc", "tc"),
    ("c1-simt", 32, [64], 8, 8, 2, "simt", "simt"),
    ("small-simt", 6, [12], 3, 19, 2, "simt", "simt"),
]


@pytest.mark.parametrize("case", BWD_CASES, ids=lambda c: c[0])
def test_flipped_step_backward(case):
    _, n_z, hidden, H, W, B, path, bpath = case
    op, dev, hid, hd = _op(n_z, hidden, [n_z, n_z], path, grad=True)
    assert op.backward_path(H, W, "cuda:0") == bpath
    z, ctx = O.make_inputs(B, n_z, hidden[0], H, W, seed=0)
    zg, cg = torch.from_numpy(z).cuda().requires_grad_(True), torch.from_numpy(ctx).cuda().requires_grad_(True)
    zt, ct = torch.from_numpy(z).double().requires_grad_(True), torch.from_numpy(ctx).double().requires_grad_(True)
    th, thh = OT_params(hid, True), OT_params(hd, True)
    rng = np.random.RandomState(5)
    gzo, gls, gld = rng.randn(*z.shape), rng.randn(*z.shape), rng.randn(B)
    zo, ls, ld = op.step(zg, cg)
    G = lambda a: torch.from_numpy(a.astype(np.float32))
    ((zo * G(gzo).cuda()).sum() + (ls * G(gls).cuda()).sum() + (ld * G(gld).cuda()).sum()).backward()
    zn, lsd, ldt = FO.t_iaf_step(zt, ct, th, thh)
    ((zn * G(gzo)).sum() + (lsd * G(gls)).sum() + (ldt * G(gld)).sum()).backward()
    assert _rel(zg.grad, zt.grad) < TOL and _rel(cg.grad, ct.grad) < TOL
    for i, l in enumerate(th + thh):
        for t, k in zip(dev[i], "wsb"):
            assert _rel(t.grad, l[k].grad) < TOL, (i, k)
        gw = dev[i][0].grad.cpu().numpy()
        zd = i >= len(hidden)
        mask = FO.conv_ar_mask(gw.shape[1] - 1, gw.shape[0], zd, True)
        assert (gw[mask == 0] == 0).all()
        # the pad channel's centre: live in the mask, reaches no output, gradient -k*v through the norm
        assert (gw[:, -1, 1, 1][mask[:, -1, 1, 1] > 0] != 0).any()
        if zd:
            assert (gw[:FO.zero_rows(gw.shape[1] - 1, gw.shape[0]), :, 1, 1] == 0).all()


def test_flipped_step_graph_capture_and_replay():
    n_z, hidden, H, W, B = 32, [64], 16, 16, 4
    op, _, hid, hd = _op(n_z, hidden, [n_z, n_z], "tc")
    z, ctx = O.make_inputs(B, n_z, hidden[0], H, W, seed=0)
    zc, cc = torch.from_numpy(z).cuda(), torch.from_numpy(ctx).cuda()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        eager = op.step(zc, cc)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = op.step(zc, cc)
    g.replay()
    torch.cuda.synchronize()
    for a, b in zip(out, eager):
        assert torch.equal(a, b)
    zr, _, _ = FO.iaf_step(z.astype(np.float64), ctx.astype(np.float64), _f64(hid), _f64(hd))
    zc.copy_(torch.from_numpy(z[::-1].copy()))  # new inputs, same buffers
    cc.copy_(torch.from_numpy(ctx[::-1].copy()))
    g.replay()
    torch.cuda.synchronize()
    assert _per_sample(out[0], zr[::-1]) < TOL
