"""The reversed-order IAF step (``IAFOperator(..., flipmask=True)``, IAF_VARIANT_THEANO_FLIPMASK) over the whole
tensor-core envelope, and every backward kernel combination of all three variants, against fp64 references.

The flipped step is the only variant whose tensor-core forward runs on the unreflected image with the pad-channel table,
and whose backward runs on the reflected gradient stream with pad-channel sums (the fused step prologue with
``img_flip = 1, fwd_flip = 0``, ``iaf_bwd_bias_kernel<true>`` with ``flip = 1``).  Sections 1-4 mirror
tests/test_gpu_tc_envelope.py for it: forward shapes and plan boundaries, the backward envelope, the nonlinearities and
the fused-layer backward, and the numerical regimes.  Section 5 runs each of the four backward configurations
(tensor cores; "tc-dgrad": data gradient on the tensor cores, weight gradient on SIMT; the three-kernel step prologue;
SIMT) through each backward route, for tf, theano and the flipped step.  Weight gradients are also judged at their own
scale: the pad-channel slice ``g_w[:, -1]`` (a sum over border pixels) and, under the trained-gain spread and small heads
gains, each output channel's row.

The fp64 reference of the flipped step is tests/flipmask_oracle.py (pinned to the reference by tests/golden/flipmask.npz).
Tolerances are those of tests/test_gpu_tc_envelope.py: forward ``|d|_inf / max(|ref|_inf, 1) <= 1e-4`` per sample,
backward ``|d|_inf / |ref|_inf <= 1e-4`` per tensor (per slice, per row), and the per-channel bounds of its section 6.
Every case asserts where it ran (``path_used``, ``backward_path``, the launch count) and records its measured errors
with ``record_property``."""
import numpy as np
import pytest
import torch

from oracle import iaf_oracle as O
from oracle import iaf_oracle_torch as OT
from tests import flipmask_oracle as FO
from tests.test_gpu_tc_envelope import (COL_TOL, DEV, ELU_ABS, GAIN_IDS, GAIN_SHAPES, LOGDET_TOL, TOL, _keys, _np,
                                        bwd_err, check_masked_taps_zero, col_err, dev_layers, f64_layers, fwd_err,
                                        layer_inputs, layer_ref, logdet_err, make_params, per_sample_fwd_err, within)

pytestmark = pytest.mark.gpu
BWD_ENV = ("IAF_BWD_TC", "IAF_BWD_WG_TC", "IAF_BWD_FUSED_PROLOGUE", "IAF_TC_FUSED")


# ---------------------------------------------------------------------------------------------------------------------
# helpers.  ``variant`` is "tf", "theano" or "flip" (the Theano parameterisation with flipmask=True).
# ---------------------------------------------------------------------------------------------------------------------
def _pv(variant):
    """Parameterisation of a variant."""
    return "theano" if variant == "flip" else variant


def v_op(variant, n_z, hidden, path, layers, nl="elu", grad=False, checknan=None):
    from iaf_b200 import IAFOperator
    dev = dev_layers(_pv(variant), layers, grad)
    op = IAFOperator(_pv(variant), n_z, hidden, [n_z, n_z], nl=nl, path=path, checknan=checknan,
                     flipmask=variant == "flip")
    return op.set_weights(dev), dev


def ref_step(variant, zt, ct, th, thh, nl="elu"):
    if variant == "flip":
        return FO.t_iaf_step(zt, ct, th, thh, nl)
    return OT.iaf_step(variant, zt, ct, th, thh, nl=nl)


def ref_layer(variant, nl, th, thh, *ins):
    if variant == "flip":
        return FO.t_stochastic_layer(*ins, th, thh, nl)
    return layer_ref(variant, nl, th, thh, *ins)


def row_err(a, ref):
    """Worst output channel (axis 0) of ``|d_co|_inf / |ref_co|_inf``: each row of a weight gradient (or each entry of a
    scale / bias gradient) at its own scale.  Rows whose reference is zero must be exactly zero."""
    a, ref = _np(a), _np(ref)
    assert np.isfinite(a).all()
    a, ref = a.reshape(a.shape[0], -1), ref.reshape(ref.shape[0], -1)
    m = np.abs(ref).max(axis=1)
    assert (a[m == 0] == 0).all()
    return float((np.abs(a - ref).max(axis=1)[m > 0] / m[m > 0]).max())


def check_flipped_masks(dev, n_hidden):
    """Masked taps and the heads' zero-diagonal centre rows get exactly zero gradient; every layer's live pad-channel
    centre (it enters the norm but reaches no output: gradient -k*w) gets a nonzero one."""
    for i, l in enumerate(dev):
        gw = l[0].grad.cpu().numpy()
        zd = i >= n_hidden
        mask = FO.conv_ar_mask(gw.shape[1] - 1, gw.shape[0], zd, True)
        assert (gw[mask == 0] == 0).all(), i
        assert (gw[:, -1, 1, 1][mask[:, -1, 1, 1] > 0] != 0).any(), i
        if zd:
            assert (gw[:FO.zero_rows(gw.shape[1] - 1, gw.shape[0]), :, 1, 1] == 0).all(), i


def check_masks(variant, dev, n_hidden):
    if variant == "flip":
        check_flipped_masks(dev, n_hidden)
    else:
        check_masked_taps_zero(variant, dev, n_hidden)


def check_grads(rec, variant, pairs, rows=False, tag=""):
    """Every gradient per tensor; for the Theano variants the pad-channel slice of every weight gradient at its own
    maximum; with ``rows`` every output channel's row of g_w at its own maximum.  Records every error and returns the
    ones beyond the tolerance.

    With ``rows`` the error of each g_s[co] and g_b[co] relative to itself is recorded too, but not bounded: each is one
    sum over every pixel of every sample (g_b of the pre-activation gradient, g_s of its product with the kernel) that
    can cancel to far below its terms, and fp32 summation then has no relative bound.  Measured on an NVIDIA H100 80GB
    HBM3 (700 W power limit) under the
    trained-gain spread and heads gain 1e-3: up to 3.4e-3 on the exact-fp32 SIMT kernels, 2.8e-2 on the tensor cores,
    while every g_w row stays within 3.2e-5."""
    errs = []
    for name, got, ref in pairs:
        errs.append((tag + name, bwd_err(got, ref)))
        if not name.startswith("layer"):
            continue
        if variant != "tf" and name.endswith(".w"):
            errs.append((tag + name + "[:,pad]", bwd_err(got[:, -1], ref[:, -1])))
        if rows and name.endswith(".w"):
            errs.append((tag + name + "[row]", row_err(got, ref)))
        elif rows:
            rec(tag + name + "[entry]", row_err(got, ref))
    for name, err in errs:
        rec(name, err)
    return [(n, e) for n, e in errs if e > TOL]


def backward_pairs(variant, n_z, hidden, H, W, B, nl, hid, hd, path="auto", g_seed=5):
    """Gradients of one step's autograd node and of fp64 autograd over the reference, for the same random upstream
    gradients of (z', arw_logsd, logdet).  Returns (op, dev, [(name, got, ref)], launches of the backward)."""
    op, dev = v_op(variant, n_z, hidden, path, hid + hd, nl, grad=True)
    z, ctx = O.make_inputs(B, n_z, hidden[0], H, W, seed=0)
    r = np.random.RandomState(g_seed)
    gzo, gls = r.randn(*z.shape).astype(np.float32), r.randn(*z.shape).astype(np.float32)
    gld = r.randn(B).astype(np.float32)
    zg = torch.from_numpy(z).to(DEV).requires_grad_(True)
    cg = torch.from_numpy(ctx).to(DEV).requires_grad_(True)
    zo, ls, ld = op.step(zg, cg)
    l0 = op.launch_count()
    ((zo * torch.from_numpy(gzo).to(DEV)).sum() + (ls * torch.from_numpy(gls).to(DEV)).sum()
     + (ld * torch.from_numpy(gld).to(DEV)).sum()).backward()
    launches = op.launch_count() - l0
    th, thh = f64_layers(hid, True), f64_layers(hd, True)
    zt = torch.from_numpy(z).double().requires_grad_(True)
    ct = torch.from_numpy(ctx).double().requires_grad_(True)
    zn, lsd, ldt = ref_step(variant, zt, ct, th, thh, nl)
    ((zn * torch.from_numpy(gzo)).sum() + (lsd * torch.from_numpy(gls)).sum() + (ldt * torch.from_numpy(gld)).sum()).backward()
    pairs = [("g_z", zg.grad, zt.grad), ("g_context", cg.grad, ct.grad)]
    for i, l in enumerate(th + thh):
        for t, k in zip(dev[i], _keys(_pv(variant))):
            pairs.append(("layer%d.%s" % (i, k), t.grad, l[k].grad))
    return op, dev, pairs, launches


def fused_prologue_fits(n_z, H, W):
    """The one-launch step prologue holds one sample's heads gradient (2 n_z planes) in shared memory
    (iaf_dg_step_supported)."""
    return 2 * n_z * H * W * 4 <= 160 * 1024


def bwd_launches(bpath, route, n_z, hidden, H, W, fwd_launches, fused_prologue=True):
    """Kernel launches of one backward call (iaf_bwd_run, plus the tensor-core recompute of op.step_backward), for the
    backward kernels ``bpath`` ("tc", "tc-dgrad", "simt") and the route: "step" (the autograd node, kept activations),
    "recompute" (op.step_backward) or "layer" (op.layer's autograd node)."""
    nst = len(hidden) + 1
    n = 2                                     # the heads' gradient, the weight-norm backward
    if route == "recompute":
        n += fwd_launches if bpath != "simt" else nst  # tensor-core training forward, or the SIMT layer convs
    if route == "layer":
        n += 2 + nst                          # layer pre / post kernels, the SIMT layer convs
    if bpath == "simt":
        return n + 4 * nst                    # weight gradient + reduce, transposed weights + data gradient per stage
    if bpath == "tc-dgrad":
        return n + 1 + 5 * nst                # operand image; weight gradient + reduce, dg stage (3) per stage
    fused = route != "layer" and fused_prologue and fused_prologue_fits(n_z, H, W)
    return n + 8 * nst + (-1 if fused else 1)  # per stage wgrad (2) + bias (2) + reduce + dg stage (3)


def _cid(c):
    return "z%d-%s-%dx%d-b%d" % (c[0], "x".join(map(str, c[1])), c[2], c[3], c[4])


# ---------------------------------------------------------------------------------------------------------------------
# 1. flipped forward envelope
# ---------------------------------------------------------------------------------------------------------------------
FWD_CASES = [
    # n_z, hidden, H, W, B, one_launch
    (16, [80], 16, 16, 2, False),             # padded column groups
    (16, [112], 8, 8, 2, False),
    (32, [96, 32], 8, 8, 2, False),           # width changes between stages
    (32, [128, 64], 8, 8, 2, False),
    (16, [176, 176], 16, 16, 2, False),       # streamed weight ring
    (48, [96], 16, 16, 2, False),             # heads N = 96
    (16, [64], 16, 32, 2, True),              # non-square, one launch
    (32, [64], 3, 46, 2, True),               # the widest map of the one-launch kernel
    (32, [64], 3, 47, 2, False),              # one column more: per-stage
    (16, [32], 5, 62, 2, True),               # one launch at MIR = 64
    (32, [64], 3, 126, 2, False),             # MIR = 128
    (32, [64, 64], 1, 1, 70, False),          # many samples per tile
    (16, [16], 2, 2, 50, True),               # many samples per tile, one launch
    (16, [48, 96, 48, 16], 8, 8, 2, False),   # four hidden layers
]


@pytest.mark.parametrize("case", FWD_CASES, ids=_cid)
def test_flipped_forward_envelope(case, record_property):
    """Step, multiconv and layer entries of a flipped ``auto`` operator on the tensor cores, through the expected
    kernels, per sample within 1e-4 of the fp64 reference."""
    n_z, hidden, H, W, B, one_launch = case
    hid, hd = make_params("theano", n_z, hidden, seed=21)
    op, _ = v_op("flip", n_z, hidden, "auto", hid + hd)
    for entry in ("step", "multiconv", "layer"):
        assert op.path_used(H, W, DEV, entry=entry) == "tc", entry
    z, ctx = O.make_inputs(B, n_z, hidden[0], H, W, seed=22)
    zc, cc = torch.from_numpy(z).to(DEV), torch.from_numpy(ctx).to(DEV)
    th, thh = f64_layers(hid), f64_layers(hd)
    zt, ct = torch.from_numpy(z).double(), torch.from_numpy(ctx).double()
    chk = lambda name, err: within(record_property, name, err, TOL)

    l0 = op.launch_count()
    z1, logsd, logdet = op.step(zc, cc)
    assert op.launch_count() - l0 == (1 if one_launch else len(hidden) + 1)
    z_ref, logsd_ref, logdet_ref = FO.iaf_step(z.astype(np.float64), ctx.astype(np.float64),
                                               O.cast_params(hid, np.float64), O.cast_params(hd, np.float64))
    chk("z", per_sample_fwd_err(z1, z_ref))
    chk("arw_logsd", per_sample_fwd_err(logsd, logsd_ref))
    chk("logdet", per_sample_fwd_err(logdet[:, None], logdet_ref[:, None]))

    l0 = op.launch_count()
    m, s = op.multiconv(zc, cc)
    assert op.launch_count() - l0 == (1 if one_launch else len(hidden) + 1)
    m_ref, s_ref = FO.t_multiconv(zt, ct, th, thh)
    chk("m", per_sample_fwd_err(m, m_ref))
    chk("s", per_sample_fwd_err(s, s_ref))

    eps, pm, pls, prm, prl, lctx = layer_inputs(B, n_z, hidden, H, W, seed=23)
    t = lambda a: torch.from_numpy(a).to(DEV)
    l0 = op.launch_count()
    zo, kl, kl_bc, kl_cost = op.layer(t(eps), t(pm), t(pls), t(prm), t(prl), t(lctx))
    assert op.launch_count() - l0 == (1 if one_launch else len(hidden) + 1)
    d = lambda a: torch.from_numpy(a).double()
    zr, klr, bcr, costr = FO.t_stochastic_layer(d(eps), d(pm), d(pls), d(prm), d(prl), d(lctx), th, thh)
    chk("layer.z", per_sample_fwd_err(zo, zr))
    chk("layer.kl", per_sample_fwd_err(kl, klr))
    chk("layer.kl_bc", per_sample_fwd_err(kl_bc, bcr))
    chk("layer.kl_cost", per_sample_fwd_err(kl_cost[:, None], costr[:, None]))


BOUNDARY_CASES = [
    # n_z, hidden, H, W, expected path
    (16, [176], 16, 16, "tc"),
    (16, [192], 16, 16, "simt"),     # a 192-column stage leaves no room for two ring stages
    (32, [192], 32, 32, "simt"),
    (48, [96], 16, 16, "tc"),
    (64, [64], 16, 16, "simt"),      # the z window exceeds 1024 items
    (32, [64], 2, 126, "tc"),
    (32, [64], 2, 127, "simt"),      # MIR = 136 > 128
]


@pytest.mark.parametrize("case", BOUNDARY_CASES, ids=lambda c: "z%d-%s-%dx%d-%s" % (c[0], "x".join(map(str, c[1])),
                                                                                    c[2], c[3], c[4]))
def test_flipped_plan_boundaries(case):
    """``auto`` puts the flipped shape on the pinned kernel family; ``path="tc"`` refuses what the tensor cores cannot
    take."""
    n_z, hidden, H, W, want = case
    hid, hd = make_params("theano", n_z, hidden, seed=1)
    op, _ = v_op("flip", n_z, hidden, "auto", hid + hd)
    assert op.path_used(H, W, DEV) == want
    for entry in ("step", "multiconv", "layer"):
        assert op.path_used(H, W, DEV, entry=entry) == want, entry
    op_tc, _ = v_op("flip", n_z, hidden, "tc", hid + hd)
    if want == "tc":
        assert op_tc.path_used(H, W, DEV) == "tc"
    else:
        with pytest.raises(NotImplementedError):
            op_tc.path_used(H, W, DEV)


# ---------------------------------------------------------------------------------------------------------------------
# 2. flipped backward envelope
# ---------------------------------------------------------------------------------------------------------------------
BWD_CASES = [
    # n_z, hidden, H, W, B, backward path
    (16, [80], 16, 16, 2, "tc"),
    (16, [112], 8, 8, 2, "tc"),
    (32, [96, 32], 8, 8, 2, "tc"),
    (32, [128, 64], 8, 8, 2, "tc"),
    (16, [176, 176], 16, 16, 2, "tc"),
    (48, [96], 16, 16, 2, "tc"),
    (32, [64, 64], 1, 1, 70, "tc"),
    (16, [16], 2, 2, 50, "tc"),
    (16, [48, 96, 48, 16], 8, 8, 2, "tc"),
    (48, [96], 22, 22, 2, "tc"),        # cp H W 4 > 160 KB: the three-kernel step prologue
    (32, [64], 4, 22, 2, "tc"),         # the weight gradient's halo edge
    (32, [64], 4, 23, 2, "simt"),       # one column more: the exact-fp32 backward
    (32, [64], 40, 20, 2, "tc"),        # cp H W 4 = 200 KB: the three-kernel step prologue
]


@pytest.mark.parametrize("case", BWD_CASES, ids=_cid)
def test_flipped_backward_envelope(case, record_property):
    """Every gradient of the flipped step's autograd node against fp64 autograd, per tensor and (pad channel) per
    slice; masked taps, zero-diagonal centre rows exactly zero, pad centres nonzero."""
    n_z, hidden, H, W, B, want = case
    hid, hd = make_params("theano", n_z, hidden, seed=1)
    op, dev, pairs, launches = backward_pairs("flip", n_z, hidden, H, W, B, "elu", hid, hd)
    assert op.path_used(H, W, DEV, entry="step") == "tc"
    assert op.backward_path(H, W, DEV) == want
    assert launches == bwd_launches(want, "step", n_z, hidden, H, W, None), launches
    fails = check_grads(record_property, "flip", pairs)
    assert not fails, fails
    check_flipped_masks(dev, len(hidden))


# ---------------------------------------------------------------------------------------------------------------------
# 3. nonlinearities and the fused-layer backward, flipped
# ---------------------------------------------------------------------------------------------------------------------
NL_SHAPES = [(32, [64], 16, 16, True), (32, [64, 64], 8, 8, False)]


@pytest.mark.parametrize("nl", ["relu", "tanh", "leakyrelu", "softplus"])
@pytest.mark.parametrize("shape", NL_SHAPES, ids=["one-launch", "per-stage"])
def test_flipped_nonlinearity_forward_and_backward(shape, nl, record_property):
    n_z, hidden, H, W, one_launch = shape
    B = 2
    hid, hd = make_params("theano", n_z, hidden, seed=31)
    op, _ = v_op("flip", n_z, hidden, "auto", hid + hd, nl)
    assert op.path_used(H, W, DEV, entry="step") == "tc"
    assert op.backward_path(H, W, DEV) == "tc"
    z, ctx = O.make_inputs(B, n_z, hidden[0], H, W, seed=32)
    l0 = op.launch_count()
    z1, logsd, logdet = op.step(torch.from_numpy(z).to(DEV), torch.from_numpy(ctx).to(DEV))
    assert op.launch_count() - l0 == (1 if one_launch else len(hidden) + 1)
    z_ref, logsd_ref, logdet_ref = FO.iaf_step(z.astype(np.float64), ctx.astype(np.float64),
                                               O.cast_params(hid, np.float64), O.cast_params(hd, np.float64), nl)
    within(record_property, "z", per_sample_fwd_err(z1, z_ref), TOL)
    within(record_property, "arw_logsd", per_sample_fwd_err(logsd, logsd_ref), TOL)
    within(record_property, "logdet", per_sample_fwd_err(logdet[:, None], logdet_ref[:, None]), TOL)

    op2, dev, pairs, launches = backward_pairs("flip", n_z, hidden, H, W, B, nl, hid, hd)
    assert op2.backward_path(H, W, DEV) == "tc"
    assert launches == bwd_launches("tc", "step", n_z, hidden, H, W, None), launches
    fails = check_grads(record_property, "flip", pairs)
    assert not fails, fails
    check_flipped_masks(dev, len(hidden))


LAYER_SHAPES = [(32, [64], 16, 16), (16, [48, 48], 8, 8)]
UPSTREAM = ["all", "kl_bc", "kl_cost", "z"]


@pytest.mark.parametrize("which", UPSTREAM)
@pytest.mark.parametrize("path", ["tc", "simt"])
@pytest.mark.parametrize("shape", LAYER_SHAPES, ids=["one-launch", "per-stage"])
def test_flipped_fused_layer_backward(shape, path, which, record_property):
    """Every gradient of the flipped op.layer autograd node for each set of upstream gradients, against fp64 autograd
    of t_stochastic_layer."""
    n_z, hidden, H, W = shape
    B, nl = 2, "elu"
    hid, hd = make_params("theano", n_z, hidden, seed=41)
    op, dev = v_op("flip", n_z, hidden, path, hid + hd, nl, grad=True)
    assert op.path_used(H, W, DEV, entry="layer") == path
    assert op.backward_path(H, W, DEV) == path
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
    outs = op.layer(*gi)
    l0 = op.launch_count()
    loss(outs, lambda g: torch.from_numpy(g).to(DEV)).backward()
    assert op.launch_count() - l0 == bwd_launches(path, "layer", n_z, hidden, H, W, None)
    ti = [torch.from_numpy(a).double().requires_grad_(True) for a in ins]
    th, thh = f64_layers(hid, True), f64_layers(hd, True)
    loss(FO.t_stochastic_layer(*ti, th, thh, nl), torch.from_numpy).backward()
    names = ("eps", "post_mean", "post_logsd", "prior_mean", "prior_logsd", "context")
    pairs = [(n, g.grad, t.grad) for n, g, t in zip(names, gi, ti)]
    for i, l in enumerate(th + thh):
        for t, k in zip(dev[i], "wsb"):
            pairs.append(("layer%d.%s" % (i, k), t.grad, l[k].grad))
    for name, got, ref in pairs:
        if ref is None or float(ref.abs().max()) == 0.0:
            assert got is None or float(got.abs().max()) == 0.0, name
            pairs = [p for p in pairs if p[0] != name]
        else:
            assert got is not None, name
    fails = check_grads(record_property, "flip", pairs)
    assert not fails, fails
    check_flipped_masks(dev, len(hidden))


# ---------------------------------------------------------------------------------------------------------------------
# 4. flipped numerical regimes (tests/test_gpu_tc_envelope.py section 6)
# ---------------------------------------------------------------------------------------------------------------------
def checked_op(variant, shape, path, hid, hd, checknan=None):
    """Operator on ``path`` ("auto": the tensor cores, or "simt"), asserting where every entry and the backward run.
    Returns (op, launches of one step)."""
    _, n_z, hidden, H, W, launches = shape
    op, _ = v_op(variant, n_z, hidden, path, hid + hd, checknan=checknan)
    want = "tc" if path == "auto" else "simt"
    for entry in ("step", "multiconv", "layer"):
        assert op.path_used(H, W, DEV, entry=entry) == want, entry
    assert op.backward_path(H, W, DEV) == want
    return op, (launches if path == "auto" else 1)


def counted(op, launches, fn, *args):
    l0 = op.launch_count()
    out = fn(*args)
    assert op.launch_count() - l0 == launches
    return out


@pytest.mark.parametrize("path", ["auto", "simt"])
@pytest.mark.parametrize("gain", [1e-2, 1e-3, 1e-4])
@pytest.mark.parametrize("shape", GAIN_SHAPES, ids=GAIN_IDS)
def test_flipped_small_heads_gain_forward_per_channel(shape, gain, path, record_property):
    """Heads of gain 1e-2 .. 1e-4 with zero biases: m, s and arw_logsd per channel (each column's norm includes its
    live pad centre), the log-det against sum |arw_logsd|, z' and the layer entry at the usual tolerance."""
    _, n_z, hidden, H, W, _ = shape
    B = 2
    hid, hd = make_params("theano", n_z, hidden, seed=81, heads_gain=gain, zero_bias=True)
    op, launches = checked_op("flip", shape, path, hid, hd)
    z, ctx = O.make_inputs(B, n_z, hidden[0], H, W, seed=82)
    zc, cc = torch.from_numpy(z).to(DEV), torch.from_numpy(ctx).to(DEV)
    th, thh = f64_layers(hid), f64_layers(hd)
    zt, ct = torch.from_numpy(z).double(), torch.from_numpy(ctx).double()

    z1, logsd, logdet = counted(op, launches, op.step, zc, cc)
    z_ref, logsd_ref, logdet_ref = FO.t_iaf_step(zt, ct, th, thh)
    within(record_property, "arw_logsd", col_err(logsd, logsd_ref), COL_TOL)
    within(record_property, "logdet", logdet_err(logdet, logdet_ref, logsd_ref), LOGDET_TOL)
    within(record_property, "z", per_sample_fwd_err(z1, z_ref), TOL)
    m, s = counted(op, launches, op.multiconv, zc, cc)
    m_ref, s_ref = FO.t_multiconv(zt, ct, th, thh)
    within(record_property, "m", col_err(m, m_ref), COL_TOL)
    within(record_property, "s", col_err(s, s_ref), COL_TOL)

    eps, pm, pls, prm, prl, lctx = layer_inputs(B, n_z, hidden, H, W, seed=83)
    t = lambda a: torch.from_numpy(a).to(DEV)
    zo, kl, kl_bc, kl_cost = op.layer(t(eps), t(pm), t(pls), t(prm), t(prl), t(lctx))
    d = lambda a: torch.from_numpy(a).double()
    zr, klr, bcr, costr = FO.t_stochastic_layer(d(eps), d(pm), d(pls), d(prm), d(prl), d(lctx), th, thh)
    within(record_property, "layer.z", per_sample_fwd_err(zo, zr), TOL)
    within(record_property, "layer.kl", per_sample_fwd_err(kl, klr), TOL)
    within(record_property, "layer.kl_bc", per_sample_fwd_err(kl_bc, bcr), TOL)
    within(record_property, "layer.kl_cost", per_sample_fwd_err(kl_cost[:, None], costr[:, None]), TOL)


@pytest.mark.parametrize("path", ["auto", "simt"])
@pytest.mark.parametrize("gain", [1e-2, 1e-3])
@pytest.mark.parametrize("shape", GAIN_SHAPES, ids=GAIN_IDS)
def test_flipped_small_first_hidden_gain_forward_per_channel(shape, gain, path, record_property):
    """First hidden layer of gain 1e-2 / 1e-3 with zero bias and zero context: its activations (kept by the training
    forward) per channel beyond the elu's absolute error ELU_ABS, and the step's outputs at the usual tolerance."""
    _, n_z, hidden, H, W, _ = shape
    B = 2
    hid, hd = make_params("theano", n_z, hidden, seed=91, hidden0_gain=gain, zero_bias=True)
    op, launches = checked_op("flip", shape, path, hid, hd)
    z, _ = O.make_inputs(B, n_z, hidden[0], H, W, seed=92)
    ctx = np.zeros((B, hidden[0], H, W), dtype=np.float32)
    th, thh = f64_layers(hid), f64_layers(hd)
    zt, ct = torch.from_numpy(z).double(), torch.from_numpy(ctx).double()

    z1, logsd, logdet, hs = counted(op, launches, op._step_train_raw, torch.from_numpy(z).to(DEV),
                                    torch.from_numpy(ctx).to(DEV))
    h_ref = torch.nn.functional.elu(FO.t_ar_conv2d(zt, th[0], False, True) + ct)
    record_property("hidden0_raw", col_err(hs[0], h_ref))
    within(record_property, "hidden0", col_err(hs[0], h_ref, ELU_ABS), COL_TOL)
    z_ref, logsd_ref, logdet_ref = FO.t_iaf_step(zt, ct, th, thh)
    within(record_property, "z", per_sample_fwd_err(z1, z_ref), TOL)
    within(record_property, "arw_logsd", per_sample_fwd_err(logsd, logsd_ref), TOL)
    within(record_property, "logdet", per_sample_fwd_err(logdet[:, None], logdet_ref[:, None]), TOL)


@pytest.mark.parametrize("path", ["auto", "simt"])
@pytest.mark.parametrize("shape", GAIN_SHAPES, ids=GAIN_IDS)
def test_flipped_heads_column_beyond_fp16_range(shape, path, record_property):
    """One column of the m head with gain e^15 (s = 5): most of its weights are beyond the fp16 range."""
    _, n_z, hidden, H, W, _ = shape
    B = 2
    hid, hd = make_params("theano", n_z, hidden, seed=101)
    c = n_z // 2 + 3
    hd[0]["s"][c] = 5.0
    op, launches = checked_op("flip", shape, path, hid, hd)
    z, ctx = O.make_inputs(B, n_z, hidden[0], H, W, seed=102)
    zc, cc = torch.from_numpy(z).to(DEV), torch.from_numpy(ctx).to(DEV)
    th, thh = f64_layers(hid), f64_layers(hd)
    zt, ct = torch.from_numpy(z).double(), torch.from_numpy(ctx).double()

    m, _ = counted(op, launches, op.multiconv, zc, cc)
    m_ref, _ = FO.t_multiconv(zt, ct, th, thh)
    assert float(m_ref[:, c].abs().max()) > 65504.0
    within(record_property, "m_column", col_err(m[:, c:c + 1], m_ref[:, c:c + 1]), COL_TOL)
    z1, _, _ = counted(op, launches, op.step, zc, cc)
    z_ref, _, _ = FO.t_iaf_step(zt, ct, th, thh)
    within(record_property, "z", fwd_err(z1, z_ref), TOL)


ISO_SHAPES = GAIN_SHAPES + [("theano", 16, [16], 2, 2, 1)]
ISO_IDS = GAIN_IDS + ["2x2-b50"]


@pytest.mark.parametrize("path", ["auto", "simt"])
@pytest.mark.parametrize("poison", ["1e5", "nan"])
@pytest.mark.parametrize("shape", ISO_SHAPES, ids=ISO_IDS)
def test_flipped_non_finite_sample_stays_in_its_sample(shape, poison, path):
    """One channel plane of one middle sample set to 1e5 or NaN: every other sample's outputs of step, multiconv, layer
    and the step's autograd node are bit-identical to a clean run; checknan="raise" raises on the poisoned batch."""
    _, n_z, hidden, H, W, _ = shape
    B = 50 if H == 2 else 3
    pn, pc = B // 2, 3
    val = 1e5 if poison == "1e5" else float("nan")
    hid, hd = make_params("theano", n_z, hidden, seed=111)
    op, launches = checked_op("flip", shape, path, hid, hd)
    z, ctx = O.make_inputs(B, n_z, hidden[0], H, W, seed=112)
    zp = z.copy()
    zp[pn, pc] = val
    t = lambda a: torch.from_numpy(a).to(DEV)
    keep = torch.tensor([n for n in range(B) if n != pn], device=DEV)

    def same(clean, bad):
        for i, (a, b) in enumerate(zip(clean, bad)):
            assert torch.equal(a[keep], b[keep]), i
            assert torch.isfinite(a).all(), i

    clean = counted(op, launches, op.step, t(z), t(ctx))
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

    opn, _ = checked_op("flip", shape, path, hid, hd, checknan="raise")
    opn.step(t(z), t(ctx))
    if path == "auto" or bool(torch.isnan(bad[2].sum())):
        with pytest.raises(FloatingPointError):
            opn.step(t(zp), t(ctx))
    else:
        opn.step(t(zp), t(ctx))  # the exact-fp32 kernel may carry 1e5 through to a finite log-det


@pytest.mark.parametrize("path", ["auto", "simt"])
@pytest.mark.parametrize("variant", ["theano", "flip"])
@pytest.mark.parametrize("shape", GAIN_SHAPES, ids=GAIN_IDS)
def test_trained_gain_spread_gradients_per_row(shape, variant, path, record_property):
    """Gains spread like a trained model's (column gains between 0.05 and 20): the forward, and every gradient per
    tensor, per pad-channel slice and per output channel's row (a column whose gradient is far below its sample's
    largest one is where the per-sample fp16 scale of the gradient images loses bits)."""
    _, n_z, hidden, H, W, _ = shape
    B = 2
    hid, hd = make_params("theano", n_z, hidden, seed=51, spread=True)
    op, launches = checked_op(variant, shape, path, hid, hd)
    z, ctx = O.make_inputs(B, n_z, hidden[0], H, W, seed=52)
    z1, logsd, logdet = counted(op, launches, op.step, torch.from_numpy(z).to(DEV), torch.from_numpy(ctx).to(DEV))
    th, thh = f64_layers(hid), f64_layers(hd)
    z_ref, logsd_ref, logdet_ref = ref_step(variant, torch.from_numpy(z).double(), torch.from_numpy(ctx).double(), th, thh)
    within(record_property, "z", per_sample_fwd_err(z1, z_ref), TOL)
    within(record_property, "arw_logsd", per_sample_fwd_err(logsd, logsd_ref), TOL)
    within(record_property, "logdet", per_sample_fwd_err(logdet[:, None], logdet_ref[:, None]), TOL)
    op2, dev, pairs, _ = backward_pairs(variant, n_z, hidden, H, W, B, "elu", hid, hd, path=path)
    assert op2.backward_path(H, W, DEV) == ("tc" if path == "auto" else "simt")
    fails = check_grads(record_property, variant, pairs, rows=True)
    assert not fails, fails
    check_masks(variant, dev, len(hidden))


@pytest.mark.parametrize("gain", [1e-2, 1e-3])
@pytest.mark.parametrize("variant", ["theano", "flip"])
@pytest.mark.parametrize("shape", GAIN_SHAPES, ids=GAIN_IDS)
def test_small_heads_gain_gradients(shape, variant, gain, record_property):
    """Heads of gain 1e-2 / 1e-3: every gradient per tensor and per pad-channel slice against fp64 autograd and against
    the exact-fp32 SIMT backward, and at gain 1e-3 per output channel's row."""
    _, n_z, hidden, H, W, _ = shape
    B = 2
    hid, hd = make_params("theano", n_z, hidden, seed=61, heads_gain=gain)
    op, dev, pairs, _ = backward_pairs(variant, n_z, hidden, H, W, B, "elu", hid, hd)
    assert op.path_used(H, W, DEV, entry="step") == "tc" and op.backward_path(H, W, DEV) == "tc"
    op_s, _, pairs_s, _ = backward_pairs(variant, n_z, hidden, H, W, B, "elu", hid, hd, path="simt")
    assert op_s.backward_path(H, W, DEV) == "simt"
    rows = gain == 1e-3
    fails = check_grads(record_property, variant, pairs, rows=rows)
    fails += check_grads(record_property, variant, pairs_s, rows=rows, tag="simt.")
    assert not fails, fails
    for (name, got, _), (_, got_s, _) in zip(pairs, pairs_s):
        within(record_property, "tc-vs-simt." + name, bwd_err(got, got_s), TOL)
    check_masks(variant, dev, len(hidden))


# ---------------------------------------------------------------------------------------------------------------------
# 5. every backward kernel combination, all three variants
# ---------------------------------------------------------------------------------------------------------------------
# name, environment, backward path.  IAF_BWD_TC / IAF_BWD_WG_TC are read when the backward plan is created (a fresh
# operator per combination), IAF_BWD_FUSED_PROLOGUE on every call.
COMBOS = [
    ("tc", {}, "tc"),
    ("tc-dgrad", {"IAF_BWD_WG_TC": "0"}, "tc-dgrad"),
    ("three-kernel-prologue", {"IAF_BWD_FUSED_PROLOGUE": "0"}, "tc"),
    ("simt", {"IAF_BWD_TC": "0"}, "simt"),
]
COMBO_SHAPES = [
    # n_z, hidden, H, W, launches of one tensor-core step
    (32, [64], 16, 16, 1),
    (32, [64, 64], 8, 8, 3),
    (32, [160, 160], 16, 16, 3),
]
LAYER_NAMES = ("eps", "post_mean", "post_logsd", "prior_mean", "prior_logsd", "context")


def route_grads(op, dev, variant, route, ins, ups):
    """(names, gradients, launches of the backward) of one backward route: "step" (the step's autograd node, kept
    activations), "recompute" (op.step_backward) or "layer" (op.layer's autograd node)."""
    t = lambda a: torch.from_numpy(a).to(DEV)
    flat = [x for l in dev for x in l]
    pnames = ["layer%d.%s" % (i, k) for i in range(len(dev)) for k in _keys(_pv(variant))]
    if route == "recompute":
        l0 = op.launch_count()
        g_z, g_ctx, gw, gs, gb = op.step_backward(t(ins[0]), t(ins[1]), *map(t, ups))
        n = op.launch_count() - l0
        return ["g_z", "g_context"] + pnames, [g_z, g_ctx] + [x for i in range(len(gw)) for x in (gw[i], gs[i], gb[i])], n
    gi = [t(a).requires_grad_(True) for a in ins]
    outs = op.layer(*gi) if route == "layer" else op.step(*gi)
    loss = sum((o * t(g)).sum() for o, g in zip(outs, ups))
    l0 = op.launch_count()
    grads = torch.autograd.grad(loss, gi + flat)
    n = op.launch_count() - l0
    names = list(LAYER_NAMES) if route == "layer" else ["g_z", "g_context"]
    return names + pnames, list(grads), n


def route_ref(variant, route, ins, ups, hid, hd):
    th, thh = f64_layers(hid, True), f64_layers(hd, True)
    ti = [torch.from_numpy(a).double().requires_grad_(True) for a in ins]
    outs = ref_layer(variant, "elu", th, thh, *ti) if route == "layer" else ref_step(variant, *ti, th, thh)
    loss = sum((o * torch.from_numpy(g).double()).sum() for o, g in zip(outs, ups))
    flat = [l[k] for l in th + thh for k in _keys(_pv(variant))]
    return list(torch.autograd.grad(loss, ti + flat))


@pytest.mark.parametrize("route", ["step", "recompute", "layer"])
@pytest.mark.parametrize("variant", ["tf", "theano", "flip"])
@pytest.mark.parametrize("shape", COMBO_SHAPES, ids=["one-launch", "per-stage", "c2b"])
def test_backward_kernel_combinations(shape, variant, route, monkeypatch, record_property):
    """Each backward configuration on a fresh operator, through one route: the expected kernels ran (backward_path and
    the launch count), every gradient is within 1e-4 of fp64 autograd (pad-channel slices at their own scale), a
    repeated call is bit-identical, and the configurations agree with one another."""
    n_z, hidden, H, W, fwd_launches = shape
    B = 2
    hid, hd = make_params(_pv(variant), n_z, hidden, seed=121)
    r = np.random.RandomState(122)
    if route == "layer":
        ins = layer_inputs(B, n_z, hidden, H, W, seed=123)
        shp = (B, n_z, H, W)
        ups = [r.randn(*shp).astype(np.float32), r.randn(*shp).astype(np.float32),
               r.randn(B, n_z).astype(np.float32), r.randn(B).astype(np.float32)]
    else:
        ins = list(O.make_inputs(B, n_z, hidden[0], H, W, seed=123))
        ups = [r.randn(B, n_z, H, W).astype(np.float32), r.randn(B, n_z, H, W).astype(np.float32),
               r.randn(B).astype(np.float32)]
    ref = route_ref(variant, route, ins, ups, hid, hd)
    got = {}
    for combo, env, bpath in COMBOS:
        for k in BWD_ENV:
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        op, dev = v_op(variant, n_z, hidden, "auto", hid + hd, grad=True)
        for entry in ("step", "layer"):
            assert op.path_used(H, W, DEV, entry=entry) == "tc", (combo, entry)
        assert op.backward_path(H, W, DEV) == bpath, combo
        want_n = bwd_launches(bpath, route, n_z, hidden, H, W, fwd_launches, fused_prologue=combo != "three-kernel-prologue")
        names, g1, n1 = route_grads(op, dev, variant, route, ins, ups)
        _, g2, n2 = route_grads(op, dev, variant, route, ins, ups)
        assert n1 == want_n and n2 == want_n, (combo, n1, n2, want_n)
        for name, a, b in zip(names, g1, g2):
            assert torch.equal(a, b), (combo, name)
        fails = check_grads(record_property, variant, list(zip(names, g1, ref)), tag=combo + ".")
        assert not fails, fails
        got[combo] = g1
    base = COMBOS[0][0]
    for combo, _, _ in COMBOS[1:]:
        for name, a, b in zip(names, got[combo], got[base]):
            within(record_property, "%s-vs-%s.%s" % (combo, base, name), bwd_err(a, b), TOL)
