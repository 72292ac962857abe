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


def col_err(a, ref, abs_err=0.0):
    """Worst channel of ``max_{n,y,x} |d| / max_{n,y,x} |ref|`` over axis 1: each channel judged at its own scale, so a
    head or layer of small gain gets no absolute error floor.  ``abs_err``: an absolute error every element may carry on
    top (subtracted from |d| first)."""
    a, ref = _np(a), _np(ref)
    assert np.isfinite(a).all()
    r = np.abs(ref).max(axis=(0, 2, 3))
    assert (r > 0).all()
    return float((np.maximum(np.abs(a - ref) - abs_err, 0.0).max(axis=(0, 2, 3)) / r).max())


def logdet_err(logdet, logdet_ref, logsd_ref):
    """Worst sample of ``|d logdet_n| / sum |arw_logsd_ref[n]|``: the log-det against the size of what it sums."""
    a, ref, ls = _np(logdet), _np(logdet_ref), _np(logsd_ref)
    assert np.isfinite(a).all()
    return float((np.abs(a - ref) / np.abs(ls).reshape(ls.shape[0], -1).sum(axis=1)).max())


def bwd_err(a, ref):
    a, ref = _np(a), _np(ref)
    assert np.isfinite(a).all()
    m = np.abs(ref).max()
    assert m > 0
    return float(np.abs(a - ref).max() / m)


def _keys(variant):
    return ("V", "g", "b") if variant == "tf" else ("w", "s", "b")


def make_params(variant, n_z, hidden, seed=1, spread=False, heads_gain=None, hidden0_gain=None, zero_bias=False):
    """Raw parameters (oracle.make_params).  ``spread``: gains spread like a trained model's: hidden layers tf
    g ~ U(-3, 3), theano s ~ U(-1, 1) (column gains between 0.05 and 20), heads over the lower half of that range (gains
    up to 1: with heads of gain 20 behind such hidden layers arw_logsd reaches ~90 and z' leaves the fp32 range even in
    the fp64 reference).  ``heads_gain`` / ``hidden0_gain``: every column's gain of the heads / of the first hidden layer
    set to it (tf g = log(gain), theano s = log(gain) / 3), the rest at the defaults.  ``zero_bias``: the layers whose
    gain is set get zero biases too, so that a small output is not hidden behind its bias."""
    hid, hd = O.make_params(variant, n_z, hidden, [n_z, n_z], seed=seed)
    k = "g" if variant == "tf" else "s"
    if spread:
        rng = np.random.RandomState(seed + 1000)
        lim = 3.0 if variant == "tf" else 1.0
        for l in hid:
            l[k] = rng.uniform(-lim, lim, size=l[k].shape).astype(np.float32)
        for l in hd:
            l[k] = rng.uniform(-lim, 0.0, size=l[k].shape).astype(np.float32)
    for gain, ls in ((heads_gain, hd), (hidden0_gain, hid[:1])):
        if gain is None:
            continue
        v = math.log(gain) / (1.0 if variant == "tf" else 3.0)
        for l in ls:
            l[k] = np.full_like(l[k], v)
            if zero_bias:
                l["b"] = np.zeros_like(l["b"])
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


# Forward precision per output channel, and non-finite samples.  Shapes: the one-launch step, the per-stage step, C2b and
# the streamed weight ring.  Every case also runs on the exact-fp32 SIMT kernel, which meets the same bounds: they ask for
# fp32-level accuracy of each channel at its own scale.  Measured errors go to the JUnit report (record_property).
GAIN_SHAPES = [
    # variant, n_z, hidden, H, W, launches of one tensor-core step
    ("tf", 32, [64], 16, 16, 1),
    ("theano", 32, [64, 64], 8, 8, 3),
    ("tf", 32, [160, 160], 16, 16, 3),
    ("tf", 16, [176, 176], 16, 16, 3),
]
GAIN_IDS = ["one-launch", "per-stage", "c2b", "ring"]
COL_TOL = 1e-5     # col_err
LOGDET_TOL = 2e-6  # logdet_err
# absolute error of the tensor-core epilogue's elu for a negative input: exp(v) - 1 with ex2.approx (2 ulp of a result
# near 1).  It is most of an activation of ~1e-3 and is allowed on top of COL_TOL for hidden activations.
ELU_ABS = 3e-7


def checked_op(shape, path, hid, hd, checknan=None):
    """Operator on ``path`` ("auto": the tensor cores, or "simt"), asserting where every entry and the backward run.
    Returns (op, launches of one step)."""
    from iaf_b200 import IAFOperator
    variant, n_z, hidden, H, W, launches = shape
    op = IAFOperator(variant, n_z, hidden, [n_z, n_z], nl="elu", path=path, checknan=checknan)
    op.set_weights(dev_layers(variant, hid + hd))
    want = "tc" if path == "auto" else "simt"
    for entry in ("step", "multiconv", "layer"):
        assert op.path_used(H, W, DEV, entry=entry) == want, entry
    assert op.backward_path(H, W, DEV) == want
    return op, (launches if path == "auto" else 1)


def counted_step(op, launches, z, ctx, train=False):
    """op.step (or the training forward, which also returns the hidden activations) through the expected kernels."""
    l0 = op.launch_count()
    out = op._step_train_raw(z, ctx) if train else op.step(z, ctx)
    assert op.launch_count() - l0 == launches
    return out


def within(record_property, name, err, tol):
    record_property(name, err)
    assert err <= tol, (name, err)


@pytest.mark.parametrize("path", ["auto", "simt"])
@pytest.mark.parametrize("gain", [1e-2, 1e-3, 1e-4])
@pytest.mark.parametrize("shape", GAIN_SHAPES, ids=GAIN_IDS)
def test_small_heads_gain_forward_per_channel(shape, gain, path, record_property):
    """Heads of gain 1e-2 .. 1e-4 with zero biases: weights of O(gain / sqrt(K)), far below the range where the fp16 lo
    half of a weight is a normal number.  m, s and arw_logsd per channel, the log-det against sum |arw_logsd|, z' and the
    layer entry at the usual tolerance."""
    variant, n_z, hidden, H, W, _ = shape
    B = 2
    hid, hd = make_params(variant, n_z, hidden, seed=81, heads_gain=gain, zero_bias=True)
    op, launches = checked_op(shape, path, hid, hd)
    z, ctx = O.make_inputs(B, n_z, hidden[0], H, W, seed=82)
    zc, cc = torch.from_numpy(z).to(DEV), torch.from_numpy(ctx).to(DEV)
    th, thh = f64_layers(hid), f64_layers(hd)
    zt, ct = torch.from_numpy(z).double(), torch.from_numpy(ctx).double()

    z1, logsd, logdet = counted_step(op, launches, zc, cc)
    z_ref, logsd_ref, logdet_ref = OT.iaf_step(variant, zt, ct, th, thh)
    within(record_property, "arw_logsd", col_err(logsd, logsd_ref), COL_TOL)
    within(record_property, "logdet", logdet_err(logdet, logdet_ref, logsd_ref), LOGDET_TOL)
    assert fwd_err(z1, z_ref) < TOL
    m, s = op.multiconv(zc, cc)
    m_ref, s_ref = OT.multiconv(variant, zt, ct, th, thh)
    within(record_property, "m", col_err(m, m_ref), COL_TOL)
    within(record_property, "s", col_err(s, s_ref), COL_TOL)

    eps, pm, pls, prm, prl, lctx = layer_inputs(B, n_z, hidden, H, W, seed=83)
    t = lambda a: torch.from_numpy(a).to(DEV)
    zo, kl, kl_bc, kl_cost = op.layer(t(eps), t(pm), t(pls), t(prm), t(prl), t(lctx))
    d = lambda a: torch.from_numpy(a).double()
    zr, klr, bcr, costr = layer_ref(variant, "elu", th, thh, d(eps), d(pm), d(pls), d(prm), d(prl), d(lctx))
    assert fwd_err(zo, zr) < TOL and fwd_err(kl, klr) < TOL
    assert per_sample_fwd_err(kl_bc, bcr) < TOL
    assert per_sample_fwd_err(kl_cost[:, None], costr[:, None]) < TOL


@pytest.mark.parametrize("path", ["auto", "simt"])
@pytest.mark.parametrize("gain", [1e-2, 1e-3])
@pytest.mark.parametrize("shape", GAIN_SHAPES, ids=GAIN_IDS)
def test_small_first_hidden_gain_forward_per_channel(shape, gain, path, record_property):
    """First hidden layer of gain 1e-2 / 1e-3 with zero bias and zero context: its activations (kept by the training
    forward) per channel, beyond the elu's absolute error ELU_ABS, and the step's outputs at the usual tolerance.  The
    heads see activations of ~gain here, whose own fp16 split has an absolute floor (activations are not scaled), so they
    get no per-channel bound."""
    variant, n_z, hidden, H, W, _ = shape
    B = 2
    hid, hd = make_params(variant, n_z, hidden, seed=91, hidden0_gain=gain, zero_bias=True)
    op, launches = checked_op(shape, path, hid, hd)
    z, _ = O.make_inputs(B, n_z, hidden[0], H, W, seed=92)
    ctx = np.zeros((B, hidden[0], H, W), dtype=np.float32)
    th, thh = f64_layers(hid), f64_layers(hd)
    zt, ct = torch.from_numpy(z).double(), torch.from_numpy(ctx).double()

    z1, logsd, logdet, hs = counted_step(op, launches, torch.from_numpy(z).to(DEV), torch.from_numpy(ctx).to(DEV),
                                         train=True)
    conv = OT.tf_ar_conv2d if variant == "tf" else OT.theano_ar_conv2d
    h_ref = torch.nn.functional.elu(conv(zt, th[0], False) + ct)
    record_property("hidden0_raw", col_err(hs[0], h_ref))
    within(record_property, "hidden0", col_err(hs[0], h_ref, ELU_ABS), COL_TOL)
    z_ref, logsd_ref, logdet_ref = OT.iaf_step(variant, zt, ct, th, thh)
    assert fwd_err(z1, z_ref) < TOL and fwd_err(logsd, logsd_ref) < TOL
    assert per_sample_fwd_err(logdet[:, None], logdet_ref[:, None]) < TOL


@pytest.mark.parametrize("path", ["auto", "simt"])
@pytest.mark.parametrize("shape", GAIN_SHAPES, ids=GAIN_IDS)
def test_heads_column_beyond_fp16_range(shape, path, record_property):
    """One column of the m head with gain e^15 (tf g = 15, theano s = 5): most of its weights are larger than the
    largest fp16 number and must still come out exact."""
    variant, n_z, hidden, H, W, _ = shape
    B = 2
    hid, hd = make_params(variant, n_z, hidden, seed=101)
    c = n_z // 2 + 3
    hd[0]["g" if variant == "tf" else "s"][c] = 15.0 if variant == "tf" else 5.0
    op, launches = checked_op(shape, path, hid, hd)
    z, ctx = O.make_inputs(B, n_z, hidden[0], H, W, seed=102)
    zc, cc = torch.from_numpy(z).to(DEV), torch.from_numpy(ctx).to(DEV)
    th, thh = f64_layers(hid), f64_layers(hd)
    zt, ct = torch.from_numpy(z).double(), torch.from_numpy(ctx).double()

    m, _ = op.multiconv(zc, cc)
    m_ref, _ = OT.multiconv(variant, zt, ct, th, thh)
    assert float(m_ref[:, c].abs().max()) > 65504.0  # the column really is beyond the fp16 range
    within(record_property, "m_column", col_err(m[:, c:c + 1], m_ref[:, c:c + 1]), COL_TOL)
    z1, _, _ = counted_step(op, launches, zc, cc)
    z_ref, _, _ = OT.iaf_step(variant, zt, ct, th, thh)
    within(record_property, "z", fwd_err(z1, z_ref), TOL)


ISO_SHAPES = GAIN_SHAPES + [("tf", 16, [16], 2, 2, 1)]
ISO_IDS = GAIN_IDS + ["2x2-b50"]


@pytest.mark.parametrize("path", ["auto", "simt"])
@pytest.mark.parametrize("poison", ["1e5", "nan"])
@pytest.mark.parametrize("shape", ISO_SHAPES, ids=ISO_IDS)
def test_non_finite_sample_stays_in_its_sample(shape, poison, path):
    """One channel plane of one middle sample set to 1e5 (inf in the fp16 operand split of the tensor cores) or NaN:
    every other sample's outputs of step, multiconv, layer (eps poisoned) and the step's autograd node (g_z, g_context)
    are bit-identical to a clean run at the same batch positions.  On the tensor cores the poisoned sample's log-det is
    non-finite (loud), and checknan="raise" raises on the poisoned batch only."""
    variant, n_z, hidden, H, W, _ = shape
    B = 50 if H == 2 else 3      # 2x2: 15 samples per tile
    pn, pc = B // 2, 3
    val = 1e5 if poison == "1e5" else float("nan")
    hid, hd = make_params(variant, n_z, hidden, seed=111)
    op, launches = checked_op(shape, path, hid, hd)
    z, ctx = O.make_inputs(B, n_z, hidden[0], H, W, seed=112)
    zp = z.copy()
    zp[pn, pc] = val
    t = lambda a: torch.from_numpy(a).to(DEV)
    keep = torch.tensor([n for n in range(B) if n != pn], device=DEV)

    def same(clean, bad):
        for i, (a, b) in enumerate(zip(clean, bad)):
            assert torch.equal(a[keep], b[keep]), i
            assert torch.isfinite(a).all(), i

    clean = counted_step(op, launches, t(z), t(ctx))
    bad = op.step(t(zp), t(ctx))
    same(clean, bad)
    if path == "auto":
        assert not bool(torch.isfinite(bad[2][pn]))
    same(op.multiconv(t(z), t(ctx)), op.multiconv(t(zp), t(ctx)))

    ins = layer_inputs(B, n_z, hidden, H, W, seed=113)
    eps_p = ins[0].copy()
    eps_p[pn, pc] = val
    same(op.layer(*map(t, ins)), op.layer(t(eps_p), *map(t, ins[1:])))

    r = np.random.RandomState(114)
    gzo, gls = t(r.randn(*z.shape).astype(np.float32)), t(r.randn(*z.shape).astype(np.float32))
    gld = t(r.randn(B).astype(np.float32))

    def grads(zz):
        zg, cg = t(zz).requires_grad_(True), t(ctx).requires_grad_(True)
        zo, ls, ld = op.step(zg, cg)
        ((zo * gzo).sum() + (ls * gls).sum() + (ld * gld).sum()).backward()
        return zg.grad, cg.grad

    same(grads(z), grads(zp))

    opn, _ = checked_op(shape, path, hid, hd, checknan="raise")
    opn.step(t(z), t(ctx))
    if path == "auto" or bool(torch.isnan(bad[2].sum())):
        with pytest.raises(FloatingPointError):
            opn.step(t(zp), t(ctx))
    else:
        opn.step(t(zp), t(ctx))  # the exact-fp32 kernel may carry 1e5 through to a finite log-det


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
