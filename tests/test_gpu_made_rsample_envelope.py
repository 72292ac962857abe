"""The backward of the step's inverse on the H100 over its own envelope: the adjoint kernel (``iaf_inv_adj_kernel``) and
the autograd node of ``IAFOperator.step_inverse(..., differentiable=True)`` / ``ar_rsample``, against the settled fp64
adjoint (tests/test_made_rsample_envelope.py).

The node's backward runs the step's training forward at z for the hidden activations (on a tensor-core plan, the
tensor-core kernels), the adjoint for the gradient at u (one CTA per sample, on the SIMT pack, whatever the plan), and
the step's saved backward at z for the context and parameter gradients.  The cases:
* the sampler's stack matrix at 3x5 in every variant, on whatever plan ``auto`` picks, and flipped [8, 4, 8];
* every nonlinearity on the SIMT path and on two tensor-core stacks (the adjoint evaluates nl' on the activations of
  the tensor-core training forward);
* maps one pixel wide or one row high, non-square maps, a 1x300 row, c2a at 64x64, c2b at 32x32, and 16x40;
* the adjoint's window at its widest map and one column past it, on three stacks;
* tensor-core against SIMT plans, every backward route, and the tile schedule (``IAF_NUM_SMS``);
* new weights between nodes and between a node's forward and its backward, two nodes of one operator with different
  weights, and a few SGD steps;
* batches past the first wave, one sample, non-finite samples, and a side stream.

Every fp64 case asserts z and g_u per sample within ``TOL`` (``|d_n|_inf / max(|ref_n|_inf, 1)``), g_context per sample
and each parameter gradient as a whole tensor, ``path_used`` / ``backward_path``, and the launches of the node's
backward: the training forward at z, one adjoint launch and the step's saved backward, nothing else.  The reference
starts cold on small maps; on the 1x300 row, the large maps and the window edges its inverse starts warm from the
kernel's z and both fixed points stop once they move by at most ``SETTLE``.  Each case records its worst errors with
``record_property``."""
import numpy as np
import pytest
import torch

from iaf_b200 import IAFOperator
from oracle import iaf_oracle as O
from tests import test_made_sample_envelope as E
from tests.test_made_rsample import adj_w_max, upstream
from tests.test_made_rsample_envelope import settled_grads

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
VARIANTS = ("tf", "theano", "theano_flipmask")
NLS = ("none", "elu", "softplus", "relu", "tanh", "leakyrelu")
TOL = 1e-4
# 1e-13 of the sample's scale: nine orders below TOL, reached within a few tens of iterations (E.inverse)
SETTLE = 1e-13
ROUTES = {None: "tc", "IAF_BWD_WG_TC": "tc-dgrad", "IAF_BWD_TC": "simt"}

_record = []


@pytest.fixture(autouse=True)
def _recorder(record_property):
    _record.append(record_property)
    yield
    _record.pop()


def _np(t):
    return t.detach().double().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t, dtype=np.float64)


def err(a, ref, whole=False):
    """Per sample (or, with ``whole``, over the tensor): max |a - ref| / max(|ref|_inf, 1)."""
    a, ref = _np(a), _np(ref)
    return E.per_sample_err(a[None], ref[None]) if whole else E.per_sample_err(a, ref)


class Case(object):
    def __init__(self, variant, n_z, hidden, H, W, nl="elu", path="auto", seed=1, frozen=False):
        """``frozen``: the parameters do not require grad."""
        self.variant, self.n_z, self.hidden, self.H, self.W, self.nl = variant, n_z, list(hidden), H, W, nl
        self.frozen = frozen
        self.base = "tf" if variant == "tf" else "theano"
        self.keys = "Vgb" if variant == "tf" else "wsb"
        self.layers = self.params(seed)
        self.op = IAFOperator(self.base, n_z, hidden, [n_z, n_z], nl=nl, path=path,
                              flipmask=variant == "theano_flipmask").set_weights(self.layers)

    def params(self, seed):
        hid, hd = O.make_params(self.base, self.n_z, self.hidden, [self.n_z, self.n_z], seed=seed)
        return [tuple(torch.from_numpy(np.ascontiguousarray(l[k])).to(DEV).requires_grad_(not self.frozen)
                      for k in self.keys)
                for l in hid + hd]

    def ref_params(self, layers):
        """(hid, hd) of the fp64 reference from the values of ``layers``."""
        ls = [{k: t.detach().cpu().numpy() for k, t in zip(self.keys, l)} for l in layers]
        return ls[:len(self.hidden)], ls[len(self.hidden):]

    def inputs(self, B, seed=0):
        u, ctx = O.make_inputs(B, self.n_z, self.hidden[0] if self.hidden else 1, self.H, self.W, seed=seed)
        return u, (ctx if self.hidden else None)

    def dev(self, a, grad=False):
        return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(DEV).requires_grad_(grad)


def forward(k, u, ctx, ctx_grad=True):
    """The node's forward: (outputs, u and context leaves)."""
    ut, ct = k.dev(u, True), k.dev(ctx, ctx_grad)
    for l in k.layers:
        for t in l:
            t.grad = None
    return k.op.step_inverse(ut, ct, differentiable=True), ut, ct


def backward(k, fwd, g, layers=None):
    """The node's backward from ``forward``'s result: (z, g_u, g_ctx, [per layer [grads]], launches)."""
    outs, ut, ct = fwd
    layers = k.layers if layers is None else layers
    loss = sum((o * k.dev(gi)).sum() for o, gi in zip(outs, g) if gi is not None)
    n0 = k.op.launch_count()
    loss.backward()
    n = k.op.launch_count() - n0
    return outs[0].detach(), ut.grad, None if ct is None else ct.grad, [[t.grad for t in l] for l in layers], n


def launch_model(k, u, ctx, outs, g, layers=None, eps_only=False):
    """Launches of the three calls the node's backward makes, each issued on its own (the step's backward only when
    the context or the parameters need a gradient)."""
    layers = [tuple(t.detach() for t in l) for l in (k.layers if layers is None else layers)]
    ut, ct = k.dev(u), k.dev(ctx)
    z, ls = outs[0].detach(), outs[1].detach()
    with torch.no_grad():
        n0 = k.op.launch_count()
        hidden = k.op._step_train_raw(z, ct, layers)[3]
        n1 = k.op.launch_count()
        g_u = k.op._step_inverse_adjoint_raw(ut, ls, hidden, *(k.dev(a) for a in g), layers=layers)
        n2 = k.op.launch_count()
        if eps_only:
            return n2 - n0, g_u
        k.op._backward("step", z, ct, layers, (-g_u, k.dev(g[1]), k.dev(g[2])), True, saved=(ut, ls, hidden))
        n3 = k.op.launch_count()
    assert n2 - n1 == 1
    return n3 - n0, g_u


def compare(k, got, u, ctx, g, layers=None, warm=False, tag=""):
    """``got`` (from ``backward``) against the settled fp64 adjoint of the values of ``layers``."""
    z, g_u, g_ctx, g_par, _ = got
    hid, hd = k.ref_params(k.layers if layers is None else layers)
    start = _np(z) if warm else None
    zr, g_u_ref, g_ctx_ref, g_par_ref, iters = settled_grads(k.variant, u, ctx, hid, hd, k.nl, *g, start=start,
                                                             settle=SETTLE if warm else 0.0)
    assert iters <= k.n_z * k.H * k.W + 1
    errs = {"z": err(z, zr), "g_u": err(g_u, g_u_ref)}
    if ctx is not None and not k.frozen:
        errs["g_ctx"] = err(g_ctx, g_ctx_ref)
    if not k.frozen:
        errs["params"] = max(err(t, ref[key], whole=True) for got_l, ref in zip(g_par, g_par_ref)
                             for t, key in zip(got_l, k.keys))
    for name, e in errs.items():
        _record[-1](tag + name, "%.3e" % e)
    for name, e in errs.items():
        assert e < TOL, (name, e)
    return errs


def check(k, B=2, which="all", warm=False, path=None, route=None, eps_only=False):
    """One node against fp64, its plan and backward route, and the launches of its backward.  ``eps_only``: only u
    requires grad (the Case's parameters are frozen)."""
    assert k.frozen == eps_only
    if path is not None:
        assert k.op.path_used(k.H, k.W, DEV) == path
    if route is not None:
        assert k.op.backward_path(k.H, k.W, DEV) == route
    _record[-1]("path", k.op.path_used(k.H, k.W, DEV))
    u, ctx = k.inputs(B)
    g = upstream(u.shape, which)
    fwd = forward(k, u, ctx, ctx_grad=not eps_only)
    got = backward(k, fwd, g)
    if eps_only:
        assert got[2] is None and all(t is None for l in got[3] for t in l)
    compare(k, got, u, ctx, g, warm=warm)
    n_model, g_u = launch_model(k, u, ctx, fwd[0], g, eps_only=eps_only)
    assert got[4] == n_model, (got[4], n_model)
    assert torch.equal(g_u, got[1])
    return got


# ---------------------------------------------------------------------------------------------------------------------
# stack shapes (cold start; maps of 3x5)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("n_z,hidden", [s[:2] for s in E.STACKS])
def test_stack_shapes(variant, n_z, hidden):
    check(Case(variant, n_z, hidden, 3, 5))


def test_stack_that_steps_up_again():
    check(Case("theano_flipmask", 16, [8, 4, 8], 3, 5))


# ---------------------------------------------------------------------------------------------------------------------
# nonlinearities, on SIMT and on the tensor cores (cold start)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("nl", NLS)
@pytest.mark.parametrize("n_z,hidden,path", [(8, [16, 16], "simt"), (32, [64], "tc"), (32, [32, 64], "tc")])
def test_every_nonlinearity(variant, nl, n_z, hidden, path):
    check(Case(variant, n_z, hidden, 3, 4, nl=nl), path=path)


# ---------------------------------------------------------------------------------------------------------------------
# maps
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("H,W", E.MAPS)
def test_maps(variant, H, W):
    check(Case(variant, 4, [8], H, W))


def refuses_before_launching(k, u, ctx):
    """The context or the parameters require grad on a map the step's backward does not take: the node raises before
    it launches anything."""
    k.op.path_used(k.H, k.W, DEV)
    n0 = k.op.launch_count()
    with pytest.raises(NotImplementedError, match="not supported"):
        k.op.backward_path(k.H, k.W, DEV)
    with pytest.raises(NotImplementedError, match="not supported"):
        k.op.ar_rsample(k.dev(u, True), k.dev(ctx, True))
    assert k.op.launch_count() == n0


@pytest.mark.parametrize("variant", VARIANTS)
def test_a_wide_row(variant):
    """1x300 is past the step's backward on one row (tests/test_made_rsample_envelope.py: W <= 124 for this stack), not
    past the adjoint: the gradient at u matches fp64, and a node that would need the step's backward refuses up
    front."""
    check(Case(variant, 4, [8], 1, 300, frozen=True), warm=True, eps_only=True)
    k = Case(variant, 4, [8], 1, 300)
    refuses_before_launching(k, *k.inputs(2))


@pytest.mark.parametrize("variant", VARIANTS)
def test_64x64_on_c2a_stack(variant):
    check(Case(variant, 32, [64], 64, 64), warm=True, path="tc")


def test_32x32_on_c2b_stack():
    check(Case("theano", 32, [160, 160], 32, 32), warm=True, path="tc")


def test_non_square_16x40_on_c2a_stack():
    check(Case("theano", 32, [64], 16, 40), warm=True, path="tc")


# ---------------------------------------------------------------------------------------------------------------------
# the adjoint's window
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant,n_z,hidden,H,w_adj,w_inv", [("tf", 16, [64] * 4, 2, 97, 103),
                                                              ("theano_flipmask", 32, [128] * 4, 2, 47, 50),
                                                              ("theano", 48, [], 1, 297, None)])
def test_the_widest_map_the_adjoint_takes_and_the_first_it_does_not(variant, n_z, hidden, H, w_adj, w_inv):
    """The adjoint's window (inv_tables): per stage two rows over W + 2 columns of its output gradients (each hidden
    width, the heads' 2 n_z) and the gradient accumulators of its input (n_z, each hidden width), in floats
    2 (W + 2) (2 n_z + sum hidden) + n_z + sum hidden <= 57600 (225 KiB):
    * tf n_z 16 [64]*4: 576 (W + 2) + 272; W = 97: 57296, W = 98: 57872.  The inverse takes up to 103.
    * flipped n_z 32 [128]*4: 1152 (W + 2) + 544; W = 47: 56992, W = 48: 58144.  The inverse takes up to 50.
    * n_z 48 without a hidden layer: 192 (W + 2) + 48; W = 297: 57456, W = 298: 57648.  This row is past the step's
      backward, so there the node runs with frozen parameters (the gradient at u only).
    At the widest map the node matches fp64; one column more the inverse still runs, and the differentiable call raises
    before anything is launched."""
    assert adj_w_max(n_z, hidden) == w_adj
    if w_inv is not None:
        assert E.inv_w_max(n_z, hidden) == w_inv
        check(Case(variant, n_z, hidden, H, w_adj), warm=True)
    else:
        check(Case(variant, n_z, hidden, H, w_adj, frozen=True), warm=True, eps_only=True)
        k = Case(variant, n_z, hidden, H, w_adj)
        refuses_before_launching(k, *k.inputs(2))
    k = Case(variant, n_z, hidden, H, w_adj + 1)
    u, ctx = k.inputs(2)
    with torch.no_grad():
        z = k.op.step_inverse(k.dev(u), k.dev(ctx))[0]
    assert torch.isfinite(z).all()
    n0 = k.op.launch_count()
    with pytest.raises(NotImplementedError, match="not supported"):
        k.op.step_inverse(k.dev(u, True), k.dev(ctx), differentiable=True)
    with pytest.raises(NotImplementedError, match="not supported"):
        k.op.ar_rsample(k.dev(u, True), k.dev(ctx))
    assert k.op.launch_count() == n0


# ---------------------------------------------------------------------------------------------------------------------
# tensor-core and SIMT plans, the backward routes, the tile schedule
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant,n_z,hidden", [("theano", 32, [64]), ("theano_flipmask", 32, [32, 64])])
def test_tensor_core_and_simt_plans(variant, n_z, hidden):
    """The raw adjoint on identical inputs is bit-identical on both plans (the same SIMT pack, the same kernel), and
    both nodes match fp64."""
    tc, simt = Case(variant, n_z, hidden, 8, 8), Case(variant, n_z, hidden, 8, 8, path="simt")
    check(tc, B=3, path="tc")
    check(simt, B=3, path="simt")
    u, ctx = tc.inputs(3)
    g = [tc.dev(a) for a in upstream(u.shape, "all")]
    ut, ct = tc.dev(u), tc.dev(ctx)
    with torch.no_grad():
        z, ls, _ = tc.op.step_inverse(ut, ct)
        hidden_act = tc.op._step_train_raw(z, ct)[3]
        a = tc.op._step_inverse_adjoint_raw(ut, ls, hidden_act, *g)
        b = simt.op._step_inverse_adjoint_raw(ut, ls, hidden_act, *g)
    assert torch.equal(a, b)


@pytest.mark.parametrize("env", list(ROUTES))
@pytest.mark.parametrize("variant,n_z,hidden", [("theano_flipmask", 32, [64]), ("theano", 32, [])])
def test_every_backward_route(variant, n_z, hidden, env, monkeypatch):
    if env:
        monkeypatch.setenv(env, "0")
    check(Case(variant, n_z, hidden, 4, 4), B=3, path="tc", route=ROUTES[env])


def test_the_tile_schedule(monkeypatch):
    """IAF_NUM_SMS caps the SMs the tensor-core training forward and backward schedule for (read at plan creation): at
    1 one CTA runs every tile.  g_u and g_context are bit-identical across caps, the parameter gradients (reductions
    whose order follows the schedule) within TOL, and each cap matches fp64."""
    runs = []
    for cap in (None, 1, 3):
        if cap is None:
            monkeypatch.delenv("IAF_NUM_SMS", raising=False)
        else:
            monkeypatch.setenv("IAF_NUM_SMS", str(cap))
        runs.append(check(Case("theano", 32, [64], 8, 8), B=4, path="tc", route="tc"))
    for r in runs[1:]:
        assert torch.equal(r[1], runs[0][1]) and torch.equal(r[2], runs[0][2])
        for a, b in zip(r[3], runs[0][3]):
            for x, y in zip(a, b):
                assert err(x, y, whole=True) < TOL


# ---------------------------------------------------------------------------------------------------------------------
# weights
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("how", ("set_weights", "invalidate"))
def test_new_weights_between_nodes(how):
    k = Case("theano", 8, [16, 16], 4, 5)
    u, ctx = k.inputs(2)
    g = upstream(u.shape, "all")
    old = backward(k, forward(k, u, ctx), g)
    compare(k, old, u, ctx, g)
    new = k.params(2)
    if how == "set_weights":
        k.layers = new
        k.op.set_weights(new)
    else:
        with torch.no_grad():
            for l, n in zip(k.layers, new):
                for t, s in zip(l, n):
                    t.data.copy_(s)
        k.op.invalidate()
    got = backward(k, forward(k, u, ctx), g)
    assert not torch.equal(got[1], old[1])
    compare(k, got, u, ctx, g)


def test_new_weights_between_a_nodes_forward_and_its_backward():
    """The node keeps the parameter tensors of its forward: set_weights with other tensors before its backward changes
    nothing about that backward, and the next node uses the new ones."""
    k = Case("tf", 8, [16], 4, 5)
    u, ctx = k.inputs(2)
    g = upstream(u.shape, "all")
    a = k.layers
    fwd = forward(k, u, ctx)
    k.layers = k.params(2)
    k.op.set_weights(k.layers)
    compare(k, backward(k, fwd, g, layers=a), u, ctx, g, layers=a)
    compare(k, backward(k, forward(k, u, ctx), g), u, ctx, g)


def test_two_nodes_of_one_operator_with_different_weights():
    """Weights A, the first node's forward; weights B, the second node's forward; then the first node's backward before
    the second's.  Each matches the fp64 adjoint of its own weights."""
    k = Case("theano_flipmask", 5, [10], 4, 5)
    u, ctx = k.inputs(2)
    g = upstream(u.shape, "all")
    a = k.layers
    fa = forward(k, u, ctx)
    b = k.params(2)
    k.layers = b
    k.op.set_weights(b)
    fb = forward(k, u, ctx)
    compare(k, backward(k, fa, g, layers=a), u, ctx, g, layers=a, tag="a_")
    compare(k, backward(k, fb, g, layers=b), u, ctx, g, layers=b, tag="b_")


def test_three_sgd_steps():
    """ar_rsample -> loss -> backward -> optimizer.step(), three times, each step's gradients against fp64 at the
    parameters of that step.  loss = sum(z * G) + sum(logp): logp = sum(-0.5 log 2 pi - arw_logsd - 0.5 eps^2), so its
    upstream is g_logsd = -1 and eps also gets -eps directly."""
    k = Case("theano", 32, [64], 4, 4)
    assert k.op.path_used(4, 4, DEV) == "tc"
    u, ctx = k.inputs(2)
    G = upstream(u.shape, "z")[0]
    # the loss is unbounded, so SGD runs away at larger rates (at 0.01 the third step's weights give a NaN sample)
    opt = torch.optim.SGD([t for l in k.layers for t in l], lr=1e-3)
    last = None
    for step in range(3):
        opt.zero_grad()
        e, c = k.dev(u, True), k.dev(ctx, True)
        z, _, lp = k.op.ar_rsample(e, c)
        ((z * k.dev(G)).sum() + lp.sum()).backward()
        hid, hd = k.ref_params(k.layers)
        zr, g_u_ref, g_ctx_ref, g_par_ref, _ = settled_grads("theano", u, ctx, hid, hd, "elu", G,
                                                             -np.ones_like(u), None, start=_np(z), settle=SETTLE)
        assert last is None or not torch.equal(z, last)  # the step moved the parameters
        last = z.detach().clone()
        assert err(z, zr) < TOL
        assert err(e.grad, g_u_ref - u) < TOL, err(e.grad, g_u_ref - u)
        assert err(c.grad, g_ctx_ref) < TOL, err(c.grad, g_ctx_ref)
        for l, ref in zip(k.layers, g_par_ref):
            for t, key in zip(l, k.keys):
                assert err(t.grad, ref[key], whole=True) < TOL, (step, key)
        opt.step()


# ---------------------------------------------------------------------------------------------------------------------
# batches, non-finite samples, streams
# ---------------------------------------------------------------------------------------------------------------------
def test_more_samples_than_the_first_wave():
    """g_u and g_context of each sample of a batch of 3 waves + 1 are bit-identical to a batch of that sample alone."""
    k = Case("theano", 4, [8], 2, 2)
    B = 3 * torch.cuda.get_device_properties(DEV).multi_processor_count + 1
    u, ctx = k.inputs(B)
    g = upstream(u.shape, "all")
    full = backward(k, forward(k, u, ctx), g)
    sl = lambda a, b: None if a is None else a[b:b + 1]
    for b in range(B):
        one = backward(k, forward(k, sl(u, b), sl(ctx, b)), [sl(a, b) for a in g])
        assert torch.equal(one[1], full[1][b:b + 1]) and torch.equal(one[2], full[2][b:b + 1]), b


def test_one_sample():
    check(Case("theano_flipmask", 8, [16], 5, 6), B=1)


@pytest.mark.parametrize("variant,n_z,hidden", [("tf", 8, [16]), ("theano", 32, [64])])
def test_non_finite_samples_leave_the_others_alone(variant, n_z, hidden):
    """NaN or inf in one sample's eps, context or g_z: the other samples' g_u and g_context are bit-identical to a
    clean run."""
    k = Case(variant, n_z, hidden, 4, 5)
    u, ctx = k.inputs(5)
    g = upstream(u.shape, "all")
    clean = backward(k, forward(k, u, ctx), g)
    u2, c2, gz2 = u.copy(), ctx.copy(), g[0].copy()
    u2[1] = np.nan
    c2[2, 3, 1, 2] = np.inf
    gz2[3, 0, 2, 2] = np.nan
    dirty = backward(k, forward(k, u2, c2), (gz2,) + tuple(g[1:]))
    for b in (0, 4):
        assert torch.equal(dirty[1][b], clean[1][b]) and torch.equal(dirty[2][b], clean[2][b]), b
    for b in (1, 2, 3):
        assert not torch.isfinite(dirty[1][b]).all(), b


def test_a_side_stream():
    """The node's forward and backward on a side stream give the default stream's bits."""
    k = Case("theano", 32, [64], 8, 8)
    u, ctx = k.inputs(3)
    g = upstream(u.shape, "all")
    ref = backward(k, forward(k, u, ctx), g)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        got = backward(k, forward(k, u, ctx), g)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1]) and torch.equal(got[2], ref[2])
    for a, b in zip(got[3], ref[3]):
        assert all(torch.equal(x, y) for x, y in zip(a, b))
