"""The tensor-core (wgmma) kernels over the whole shape envelope ``path="auto"`` sends to them, against the fp64 oracle.

The SIMT kernels are pinned to the oracle on the CPU (tests/emu); the tensor-core kernels cannot be emulated, so this
file runs them on the GPU at the shapes where hand-written wgmma code goes wrong: stage widths of every column-group
count (padded groups, streamed vs. resident weights), the one-launch / per-stage boundary, the widest maps the tile
window accepts, many samples per tile, deep stacks, every nonlinearity, the fused-layer backward, and weight / gradient
magnitudes far from the defaults.  Every case asserts which kernels ran (``path_used`` / ``backward_path`` /
``launch_count``), so that a later plan change cannot quietly move it onto the SIMT path.

Tolerances: forward ``|d|_inf / max(|ref|_inf, 1) <= 1e-4`` (per sample for per-sample reductions), backward
``|d|_inf / |ref|_inf <= 1e-4`` per tensor."""
import math

import numpy as np
import pytest
import torch

from oracle import iaf_oracle as O
from oracle import iaf_oracle_torch as OT

pytestmark = pytest.mark.gpu
TOL = 1e-4
DEV = "cuda:0"  # the plans that path_used / launch_count look at are keyed by device index: the same one the calls use


# ---------------------------------------------------------------------------------------------------------------------
# helpers
# ---------------------------------------------------------------------------------------------------------------------
def _np(t):
    return t.detach().double().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t, dtype=np.float64)


def fwd_err(a, ref):
    a, ref = _np(a), _np(ref)
    assert np.isfinite(a).all()
    return float(np.abs(a - ref).max() / max(np.abs(ref).max(), 1.0))


def per_sample_fwd_err(a, ref):
    """Worst sample of ``|d_n|_inf / max(|ref_n|_inf, 1)`` over the leading (batch) axis."""
    a, ref = _np(a), _np(ref)
    assert np.isfinite(a).all()
    d = np.abs(a - ref).reshape(a.shape[0], -1).max(axis=1)
    r = np.maximum(np.abs(ref).reshape(a.shape[0], -1).max(axis=1), 1.0)
    return float((d / r).max())


def bwd_err(a, ref):
    a, ref = _np(a), _np(ref)
    assert np.isfinite(a).all()
    m = np.abs(ref).max()
    assert m > 0
    return float(np.abs(a - ref).max() / m)


def _keys(variant):
    return ("V", "g", "b") if variant == "tf" else ("w", "s", "b")


def make_params(variant, n_z, hidden, seed=1, spread=False, heads_gain=None):
    """Raw parameters (oracle.make_params).  ``spread``: gains spread like a trained model's: hidden layers tf
    g ~ U(-3, 3), theano s ~ U(-1, 1) (column gains between 0.05 and 20), heads over the lower half of that range (gains
    up to 1: with heads of gain 20 behind such hidden layers arw_logsd reaches ~90 and z' leaves the fp32 range even in
    the fp64 reference).  ``heads_gain``: every head column's gain set to it (tf g = log(gain), theano
    s = log(gain) / 3), the rest at the defaults."""
    hid, hd = O.make_params(variant, n_z, hidden, [n_z, n_z], seed=seed)
    k = "g" if variant == "tf" else "s"
    if spread:
        rng = np.random.RandomState(seed + 1000)
        lim = 3.0 if variant == "tf" else 1.0
        for l in hid:
            l[k] = rng.uniform(-lim, lim, size=l[k].shape).astype(np.float32)
        for l in hd:
            l[k] = rng.uniform(-lim, 0.0, size=l[k].shape).astype(np.float32)
    if heads_gain is not None:
        v = math.log(heads_gain) / (1.0 if variant == "tf" else 3.0)
        for l in hd:
            l[k] = np.full_like(l[k], v)
    return hid, hd


def dev_layers(variant, layers, grad=False):
    return [tuple(torch.from_numpy(np.ascontiguousarray(l[k])).to(DEV).requires_grad_(grad) for k in _keys(variant))
            for l in layers]


def f64_layers(layers, grad=False):
    out = OT.to_torch(O.cast_params(layers, np.float64), torch.float64)
    for l in out:
        for t in l.values():
            t.requires_grad_(grad)
    return out


def make_op(variant, n_z, hidden, nl, path, layers, grad=False):
    from iaf_b200 import IAFOperator
    dev = dev_layers(variant, layers, grad)
    return IAFOperator(variant, n_z, hidden, [n_z, n_z], nl=nl, path=path).set_weights(dev), dev


def layer_inputs(B, n_z, hidden, H, W, seed):
    rng = np.random.RandomState(seed)
    shp = (B, n_z, H, W)
    eps, pm, prm = (rng.randn(*shp).astype(np.float32) for _ in range(3))
    pls, prl = ((0.3 * rng.randn(*shp)).astype(np.float32) for _ in range(2))
    ctx = (0.1 * rng.randn(B, hidden[0], H, W)).astype(np.float32)
    return eps, pm, pls, prm, prl, ctx


def layer_ref(variant, nl, th, thh, eps, pm, pls, prm, prl, ctx):
    """The fused stochastic-layer block in fp64 torch: posterior sample -> IAF step -> logqs - logps -> kl and its
    per-(sample, channel) and per-sample sums (tf_train.py:56-85, models.py:273-328)."""
    c = 0.5 * math.log(2.0 * math.pi)
    z0 = pm + torch.exp(pls) * eps
    zn, lsd, _ = OT.iaf_step(variant, z0, ctx, th, thh, nl=nl)
    kl = (-c - pls - 0.5 * eps * eps + lsd) - (-c - prl - 0.5 * (zn - prm) ** 2 * torch.exp(-2.0 * prl))
    return zn, kl, kl.sum(dim=(2, 3)), kl.sum(dim=(1, 2, 3))


def check_masked_taps_zero(variant, dev, n_hidden):
    for i, l in enumerate(dev):
        gw = l[0].grad.cpu().numpy()
        zd = i >= n_hidden
        mask = (O.get_conv_ar_mask(3, 3, gw.shape[2], gw.shape[3], zd) if variant == "tf"
                else O.theano_conv_ar_mask(gw.shape[1] - 1, gw.shape[0], (3, 3), zd))
        assert (gw[mask == 0] == 0).all(), i


def step_backward_pairs(variant, n_z, hidden, H, W, B, nl, hid, hd, path="auto", g_seed=5, g_scale=None):
    """Gradients of one step's autograd node and of fp64 torch autograd over the oracle, for the same random upstream
    gradients of (z', arw_logsd, logdet).  ``g_scale[n]`` multiplies sample n's upstream gradients.
    Returns (op, dev, [(name, got, ref)])."""
    op, dev = make_op(variant, n_z, hidden, nl, path, hid + hd, grad=True)
    z, ctx = O.make_inputs(B, n_z, hidden[0], H, W, seed=0)
    r = np.random.RandomState(g_seed)
    gzo, gls = r.randn(*z.shape).astype(np.float32), r.randn(*z.shape).astype(np.float32)
    gld = r.randn(B).astype(np.float32)
    if g_scale is not None:
        f = np.asarray(g_scale, dtype=np.float32)
        gzo, gls, gld = gzo * f[:, None, None, None], gls * f[:, None, None, None], gld * f
    zg = torch.from_numpy(z).to(DEV).requires_grad_(True)
    cg = torch.from_numpy(ctx).to(DEV).requires_grad_(True)
    zo, ls, ld = op.step(zg, cg)
    ((zo * torch.from_numpy(gzo).to(DEV)).sum() + (ls * torch.from_numpy(gls).to(DEV)).sum()
     + (ld * torch.from_numpy(gld).to(DEV)).sum()).backward()
    th, thh = f64_layers(hid, True), f64_layers(hd, True)
    zt = torch.from_numpy(z).double().requires_grad_(True)
    ct = torch.from_numpy(ctx).double().requires_grad_(True)
    zn, lsd, ldt = OT.iaf_step(variant, zt, ct, th, thh, nl=nl)
    ((zn * torch.from_numpy(gzo)).sum() + (lsd * torch.from_numpy(gls)).sum() + (ldt * torch.from_numpy(gld)).sum()).backward()
    pairs = [("g_z", zg.grad, zt.grad), ("g_context", cg.grad, ct.grad)]
    for i, l in enumerate(th + thh):
        for t, k in zip(dev[i], _keys(variant)):
            pairs.append(("layer%d.%s" % (i, k), t.grad, l[k].grad))
    return op, dev, pairs


def _cid(c):
    return "%s-z%d-%s-%dx%d" % (c[0], c[1], "x".join(map(str, c[2])), c[3], c[4])


# ---------------------------------------------------------------------------------------------------------------------
# 1. forward shape envelope
# ---------------------------------------------------------------------------------------------------------------------
# (adjacent widths divide one another, ar.py:250,257: 80 / 112 / 176 wide stages sit on n_z = 16)
FWD_CASES = [
    # variant, n_z, hidden, H, W, B, one_launch
    ("tf", 16, [80], 16, 16, 2, False),             # NGW 3 with a padded group (80 = 2.5 x 32)
    ("tf", 16, [112], 8, 8, 2, False),              # NGW 4 with a padded group
    ("theano", 32, [96, 32], 8, 8, 2, False),       # NGW 3 -> 1 -> 2: width changes between stages
    ("theano", 32, [128, 64], 8, 8, 2, False),      # NGW 4 -> 2
    ("tf", 16, [176, 176], 16, 16, 2, False),       # NGW 6 padded, the widest accepted stage, streamed weight ring
    ("theano", 48, [96], 16, 16, 2, False),         # heads N = 96
    ("tf", 16, [64], 16, 32, 2, True),              # non-square, one launch
    ("theano", 32, [64], 3, 46, 2, True),           # the widest map of the one-launch kernel (shared memory)
    ("theano", 32, [64], 3, 47, 2, False),          # one column more: per-stage
    ("tf", 16, [32], 5, 62, 2, True),               # one launch at the smallest tile advance TS = 64 (MIR = 64)
    ("tf", 32, [64], 3, 126, 2, False),             # per-stage, MIR = 128: the z window is exactly full
    ("theano", 32, [64, 64], 1, 1, 70, False),      # 33 samples per tile: per-sample log-det / KL sums
    ("tf", 16, [16], 2, 2, 50, True),               # 15 samples per tile, one launch
    ("tf", 16, [48, 96, 48, 16], 8, 8, 2, False),   # four hidden layers: operand-image ping-pong over five stages
]


@pytest.mark.parametrize("case", FWD_CASES, ids=_cid)
def test_forward_envelope_against_fp64_oracle(case):
    """Step, multiconv and layer entries of an ``auto`` operator: each on the tensor cores, through the expected kernel
    (one launch, or one launch per stage), and each within the forward tolerance of the fp64 oracle."""
    variant, n_z, hidden, H, W, B, one_launch = case
    nl = "elu"
    hid, hd = make_params(variant, n_z, hidden, seed=21)
    op, _ = make_op(variant, n_z, hidden, nl, "auto", hid + hd)
    for entry in ("step", "multiconv", "layer"):
        assert op.path_used(H, W, DEV, entry=entry) == "tc", entry
    z, ctx = O.make_inputs(B, n_z, hidden[0], H, W, seed=22)
    zc, cc = torch.from_numpy(z).to(DEV), torch.from_numpy(ctx).to(DEV)
    f64 = lambda ls: O.cast_params(ls, np.float64)

    l0 = op.launch_count()
    z1, logsd, logdet = op.step(zc, cc)
    assert op.launch_count() - l0 == (1 if one_launch else len(hidden) + 1)
    z_ref, logsd_ref, logdet_ref = O.iaf_step(variant, z.astype(np.float64), ctx.astype(np.float64), f64(hid), f64(hd), nl)
    assert fwd_err(z1, z_ref) < TOL
    assert fwd_err(logsd, logsd_ref) < TOL
    assert per_sample_fwd_err(logdet[:, None], logdet_ref[:, None]) < TOL

    th, thh = f64_layers(hid), f64_layers(hd)
    zt, ct = torch.from_numpy(z).double(), torch.from_numpy(ctx).double()
    m, s = op.multiconv(zc, cc)
    m_ref, s_ref = OT.multiconv(variant, zt, ct, th, thh, nl)
    assert fwd_err(m, m_ref) < TOL and fwd_err(s, s_ref) < TOL

    eps, pm, pls, prm, prl, lctx = layer_inputs(B, n_z, hidden, H, W, seed=23)
    t = lambda a: torch.from_numpy(a).to(DEV)
    zo, kl, kl_bc, kl_cost = op.layer(t(eps), t(pm), t(pls), t(prm), t(prl), t(lctx))
    d = lambda a: torch.from_numpy(a).double()
    zr, klr, bcr, costr = layer_ref(variant, nl, th, thh, d(eps), d(pm), d(pls), d(prm), d(prl), d(lctx))
    assert fwd_err(zo, zr) < TOL
    assert fwd_err(kl, klr) < TOL
    assert per_sample_fwd_err(kl_bc, bcr) < TOL
    assert per_sample_fwd_err(kl_cost[:, None], costr[:, None]) < TOL


@pytest.mark.parametrize("variant,hidden,H,W", [("tf", [64], 16, 16), ("theano", [64, 64], 8, 8)],
                         ids=["one-launch", "per-stage"])
def test_optional_outputs_may_be_null_on_a_tensor_core_plan(variant, hidden, H, W):
    """want_logsd / want_logdet / want_kl = False pass null pointers to the tensor-core kernels: the outputs that are
    still written are bit-identical to the full call."""
    n_z, B = 32, 3
    hid, hd = make_params(variant, n_z, hidden, seed=3)
    op, _ = make_op(variant, n_z, hidden, "elu", "tc", hid + hd)
    assert op.path_used(H, W, DEV, entry="step") == "tc" and op.path_used(H, W, DEV, entry="layer") == "tc"
    z, ctx = O.make_inputs(B, n_z, hidden[0], H, W, seed=4)
    zc, cc = torch.from_numpy(z).to(DEV), torch.from_numpy(ctx).to(DEV)
    full = op.step(zc, cc)
    for wl, wd in ((False, True), (True, False), (False, False)):
        part = op.step(zc, cc, want_logsd=wl, want_logdet=wd)
        assert torch.equal(part[0], full[0])
        assert (part[1] is None) == (not wl) and (part[2] is None) == (not wd)
        if wl:
            assert torch.equal(part[1], full[1])
        if wd:
            assert torch.equal(part[2], full[2])
    t = lambda a: torch.from_numpy(a).to(DEV)
    ins = [t(a) for a in layer_inputs(B, n_z, hidden, H, W, seed=5)]
    a = op.layer(*ins)
    b = op.layer(*ins, want_kl=False)
    assert b[1] is None
    assert torch.equal(a[0], b[0]) and torch.equal(a[2], b[2]) and torch.equal(a[3], b[3])


# ---------------------------------------------------------------------------------------------------------------------
# 2. plan boundaries (plans only: nothing outside the envelope is launched on the tensor cores)
# ---------------------------------------------------------------------------------------------------------------------
BOUNDARY_CASES = [
    # variant, n_z, hidden, H, W, expected path
    ("tf", 16, [176], 16, 16, "tc"),
    ("tf", 16, [192], 16, 16, "simt"),   # a 192-column stage and its accumulator tile leave no room for two ring stages
    ("tf", 16, [192], 1, 1, "simt"),
    ("tf", 32, [192], 4, 4, "simt"),
    ("theano", 32, [192], 32, 32, "simt"),
    ("tf", 32, [256], 16, 16, "simt"),
    ("tf", 48, [96], 16, 16, "tc"),
    ("tf", 64, [64], 16, 16, "simt"),    # the z window (n_z / 8 chunks x 128 + MIR slots) exceeds 1024 items
    ("tf", 32, [64], 2, 126, "tc"),
    ("tf", 32, [64], 2, 127, "simt"),    # MIR = 136 > 128: a tap reaches past the next tile
]


@pytest.mark.parametrize("case", BOUNDARY_CASES, ids=lambda c: _cid(c) + "-" + c[5])
def test_plan_boundaries(case):
    """``auto`` puts the shape on the pinned kernel family; ``path="tc"`` refuses what the tensor cores cannot take."""
    variant, n_z, hidden, H, W, want = case
    hid, hd = make_params(variant, n_z, hidden, seed=1)
    op, _ = make_op(variant, n_z, hidden, "elu", "auto", hid + hd)
    assert op.path_used(H, W, DEV) == want
    for entry in ("step", "multiconv", "layer"):
        assert op.path_used(H, W, DEV, entry=entry) == want, entry
    op_tc, _ = make_op(variant, n_z, hidden, "elu", "tc", hid + hd)
    if want == "tc":
        assert op_tc.path_used(H, W, DEV) == "tc"
    else:
        with pytest.raises(NotImplementedError):
            op_tc.path_used(H, W, DEV)


# ---------------------------------------------------------------------------------------------------------------------
# 3. nonlinearities (the generic epilogue NLT = -1 forward, dg_nl_grad backward)
# ---------------------------------------------------------------------------------------------------------------------
NL_SHAPES = [("tf", 32, [64], 16, 16, True), ("theano", 32, [64, 64], 8, 8, False)]


@pytest.mark.parametrize("nl", ["relu", "tanh", "leakyrelu", "softplus"])
@pytest.mark.parametrize("shape", NL_SHAPES, ids=["one-launch", "per-stage"])
def test_nonlinearity_forward_and_backward(shape, nl):
    variant, n_z, hidden, H, W, one_launch = shape
    B = 2
    hid, hd = make_params(variant, n_z, hidden, seed=31)
    op, _ = make_op(variant, n_z, hidden, nl, "auto", hid + hd)
    assert op.path_used(H, W, DEV, entry="step") == "tc"
    assert op.backward_path(H, W, DEV) == "tc"
    z, ctx = O.make_inputs(B, n_z, hidden[0], H, W, seed=32)
    l0 = op.launch_count()
    z1, logsd, logdet = op.step(torch.from_numpy(z).to(DEV), torch.from_numpy(ctx).to(DEV))
    assert op.launch_count() - l0 == (1 if one_launch else len(hidden) + 1)
    f64 = lambda ls: O.cast_params(ls, np.float64)
    z_ref, logsd_ref, logdet_ref = O.iaf_step(variant, z.astype(np.float64), ctx.astype(np.float64), f64(hid), f64(hd), nl)
    assert fwd_err(z1, z_ref) < TOL and fwd_err(logsd, logsd_ref) < TOL
    assert per_sample_fwd_err(logdet[:, None], logdet_ref[:, None]) < TOL

    op2, dev, pairs = step_backward_pairs(variant, n_z, hidden, H, W, B, nl, hid, hd)
    assert op2.backward_path(H, W, DEV) == "tc"
    for name, got, ref in pairs:
        assert bwd_err(got, ref) < TOL, name
    check_masked_taps_zero(variant, dev, len(hidden))


# ---------------------------------------------------------------------------------------------------------------------
# 4. backward envelope
# ---------------------------------------------------------------------------------------------------------------------
BWD_CASES = [
    # variant, n_z, hidden, H, W, B, backward path
    ("tf", 16, [80], 16, 16, 2, "tc"),
    ("tf", 16, [112], 8, 8, 2, "tc"),
    ("theano", 32, [96, 32], 8, 8, 2, "tc"),
    ("theano", 32, [128, 64], 8, 8, 2, "tc"),       # weight gradient of a 128-channel input
    ("tf", 16, [176, 176], 16, 16, 2, "tc"),        # weight-gradient column blocks of 16 (Np = 16), cin 176 > 128
    ("theano", 48, [96], 16, 16, 2, "tc"),
    ("theano", 32, [64, 64], 1, 1, 70, "tc"),
    ("tf", 16, [16], 2, 2, 50, "tc"),
    ("tf", 16, [48, 96, 48, 16], 8, 8, 2, "tc"),    # G[j & 1] buffers over three hidden-layer gradients
    ("theano", 48, [96], 22, 22, 2, "tc"),          # W = 22: Wp + 1 = WG_HALO; cp H W 4 > 160 KB: non-fused prologue
    ("tf", 32, [64], 4, 22, 2, "tc"),               # the weight gradient's halo edge
    ("tf", 32, [64], 4, 23, 2, "simt"),             # one column more: the exact-fp32 backward
    ("tf", 32, [64], 40, 20, 2, "tc"),              # cp H W 4 = 200 KB > 160 KB: non-fused step prologue
]


@pytest.mark.parametrize("case", BWD_CASES, ids=_cid)
def test_backward_envelope_against_fp64_autograd(case):
    variant, n_z, hidden, H, W, B, want = case
    hid, hd = make_params(variant, n_z, hidden, seed=1)
    op, dev, pairs = step_backward_pairs(variant, n_z, hidden, H, W, B, "elu", hid, hd)
    assert op.path_used(H, W, DEV, entry="step") == "tc"
    assert op.backward_path(H, W, DEV) == want
    for name, got, ref in pairs:
        assert bwd_err(got, ref) < TOL, name
    check_masked_taps_zero(variant, dev, len(hidden))


# ---------------------------------------------------------------------------------------------------------------------
# 5. fused-layer backward (iaf_layer_bwd: op.layer's autograd node)
# ---------------------------------------------------------------------------------------------------------------------
LAYER_SHAPES = [("tf", 32, [64], 16, 16), ("tf", 32, [64, 64], 8, 8), ("theano", 16, [48, 48], 8, 8)]
UPSTREAM = ["all", "kl_bc", "kl_cost", "z"]


@pytest.mark.parametrize("which", UPSTREAM)
@pytest.mark.parametrize("path", ["tc", "simt"])
@pytest.mark.parametrize("shape", LAYER_SHAPES, ids=["c2a", "tf-64x64-8x8", "theano-z16-48x48"])
def test_fused_layer_backward_against_fp64_autograd(shape, path, which):
    """Every gradient of op.layer's autograd node (the five elementwise inputs, the context and every raw parameter) for
    each set of upstream gradients; outputs whose gradient is None reach the backward as null pointers."""
    variant, n_z, hidden, H, W = shape
    B, nl = 2, "elu"
    hid, hd = make_params(variant, n_z, hidden, seed=41)
    op, dev = make_op(variant, n_z, hidden, nl, path, hid + hd, grad=True)
    if path == "tc":
        assert op.path_used(H, W, DEV, entry="layer") == "tc"
        assert op.backward_path(H, W, DEV) == "tc"
    else:
        assert op.path_used(H, W, DEV, entry="layer") == "simt"
        assert op.backward_path(H, W, DEV) == "simt"
    ins = layer_inputs(B, n_z, hidden, H, W, seed=42)
    rng = np.random.RandomState(43)
    shp = (B, n_z, H, W)
    g_z = rng.randn(*shp).astype(np.float32) if which in ("all", "z") else None
    g_kl = rng.randn(*shp).astype(np.float32) if which == "all" else None
    g_bc = rng.randn(B, n_z).astype(np.float32) if which in ("all", "kl_bc") else None
    g_cost = rng.randn(B).astype(np.float32) if which in ("all", "kl_cost") else None

    def loss(outs, to):
        terms = [(o * to(g)).sum() for o, g in zip(outs, (g_z, g_kl, g_bc, g_cost)) if g is not None]
        return sum(terms[1:], terms[0])

    gi = [torch.from_numpy(a).to(DEV).requires_grad_(True) for a in ins]
    loss(op.layer(*gi), lambda g: torch.from_numpy(g).to(DEV)).backward()
    ti = [torch.from_numpy(a).double().requires_grad_(True) for a in ins]
    th, thh = f64_layers(hid, True), f64_layers(hd, True)
    loss(layer_ref(variant, nl, th, thh, *ti), torch.from_numpy).backward()
    names = ("eps", "post_mean", "post_logsd", "prior_mean", "prior_logsd", "context")
    pairs = [(n, g.grad, t.grad) for n, g, t in zip(names, gi, ti)]
    for i, l in enumerate(th + thh):
        for t, k in zip(dev[i], _keys(variant)):
            pairs.append(("layer%d.%s" % (i, k), t.grad, l[k].grad))
    for name, got, ref in pairs:
        if ref is None or float(ref.abs().max()) == 0.0:
            assert got is None or float(got.abs().max()) == 0.0, name
        else:
            assert got is not None, name
            assert bwd_err(got, ref) < TOL, name
    check_masked_taps_zero(variant, dev, len(hidden))


# ---------------------------------------------------------------------------------------------------------------------
# 6. numerical regimes
# ---------------------------------------------------------------------------------------------------------------------
REGIME_SHAPES = [("tf", 32, [64], 16, 16), ("theano", 32, [64, 64], 8, 8)]


@pytest.mark.parametrize("shape", REGIME_SHAPES, ids=["one-launch", "per-stage"])
def test_trained_gain_spread_forward_and_backward(shape):
    """Gains spread like a trained model's (column gains between 0.05 and 20)."""
    variant, n_z, hidden, H, W = shape
    B = 2
    hid, hd = make_params(variant, n_z, hidden, seed=51, spread=True)
    op, _ = make_op(variant, n_z, hidden, "elu", "auto", hid + hd)
    assert op.path_used(H, W, DEV, entry="step") == "tc"
    z, ctx = O.make_inputs(B, n_z, hidden[0], H, W, seed=52)
    z1, logsd, logdet = op.step(torch.from_numpy(z).to(DEV), torch.from_numpy(ctx).to(DEV))
    f64 = lambda ls: O.cast_params(ls, np.float64)
    z_ref, logsd_ref, logdet_ref = O.iaf_step(variant, z.astype(np.float64), ctx.astype(np.float64), f64(hid), f64(hd))
    assert fwd_err(z1, z_ref) < TOL and fwd_err(logsd, logsd_ref) < TOL
    assert per_sample_fwd_err(logdet[:, None], logdet_ref[:, None]) < TOL
    op2, _, pairs = step_backward_pairs(variant, n_z, hidden, H, W, B, "elu", hid, hd)
    assert op2.backward_path(H, W, DEV) == "tc"
    for name, got, ref in pairs:
        assert bwd_err(got, ref) < TOL, name


@pytest.mark.parametrize("gain", [1e-2, 1e-3])
@pytest.mark.parametrize("shape", REGIME_SHAPES, ids=["one-launch", "per-stage"])
def test_small_heads_gain_backward(shape, gain):
    """Heads of gain 1e-2 / 1e-3 (a data-dependent init gives heads an output std near 0.1): weights of O(gain / sqrt(K))
    must keep their precision in the fp16 operand images of the data gradient.  Per tensor against fp64 autograd and
    against the exact-fp32 SIMT backward."""
    variant, n_z, hidden, H, W = shape
    B = 2
    hid, hd = make_params(variant, n_z, hidden, seed=61, heads_gain=gain)
    op, _, pairs = step_backward_pairs(variant, n_z, hidden, H, W, B, "elu", hid, hd)
    assert op.backward_path(H, W, DEV) == "tc"
    op_s, _, pairs_s = step_backward_pairs(variant, n_z, hidden, H, W, B, "elu", hid, hd, path="simt")
    assert op_s.backward_path(H, W, DEV) == "simt"
    for (name, got, ref), (_, got_s, _) in zip(pairs, pairs_s):
        assert bwd_err(got, ref) < TOL, name
        assert bwd_err(got, got_s) < TOL, name


@pytest.mark.parametrize("shape", REGIME_SHAPES, ids=["one-launch", "per-stage"])
def test_per_sample_gradient_scale_is_independent_of_the_batch(shape):
    """One sample's upstream gradients scaled by 2^-30 and one sample's set to zero: every sample's g_z and g_context are
    accurate relative to that sample's own largest value (the per-sample power-of-two scale of the operand images), and
    the zero sample's are exactly zero."""
    variant, n_z, hidden, H, W = shape
    B = 4
    hid, hd = make_params(variant, n_z, hidden, seed=71)
    scale = [1.0, 2.0 ** -30, 0.0, 1.0]
    op, _, pairs = step_backward_pairs(variant, n_z, hidden, H, W, B, "elu", hid, hd, g_scale=scale)
    assert op.backward_path(H, W, DEV) == "tc"
    for name, got, ref in pairs[:2]:
        got, ref = _np(got), _np(ref)
        assert np.isfinite(got).all()
        assert (got[2] == 0).all(), name
        for n in (0, 1, 3):
            m = np.abs(ref[n]).max()
            assert m > 0
            assert np.abs(got[n] - ref[n]).max() / m < TOL, (name, n)
    for name, got, ref in pairs[2:]:
        assert bwd_err(got, ref) < TOL, name
