"""The backward of the step's inverse on the H100: the adjoint kernel (``iaf_inv_adj_kernel``) and the autograd node of
``IAFOperator.step_inverse(..., differentiable=True)`` / ``ar_rsample``.

* every gradient (u, context, parameters) against fp64 autograd through the unrolled fixed point
  (tests/test_made_rsample.py), on SIMT and tensor-core plans, n_z 16/32/48 with hidden [], [64], [48, 96];
* both backward routes of the step's backward (IAF_BWD_TC=0, IAF_BWD_WG_TC=0) under the node, with its launches
  counted: the hidden activations at z, one adjoint launch, the step's saved backward, nothing else;
* at the benchmark's prior shapes (c2a, c2b): the adjoint's identity through the step's backward, and two routes to
  the same gradient: ``ar_rsample``'s own logp against ``ar_logp`` evaluated at ``ar_rsample``'s z;
* determinism, batch independence, the adjoint inside a CUDA graph, and the widest map whose window fits.
"""
import numpy as np
import pytest
import torch

from iaf_b200 import IAFOperator
from oracle import iaf_oracle as O
from tests.test_made_rsample import adj_w_max, oracle_grads, upstream
from tests.test_made_sample_envelope import per_sample_err

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
VARIANTS = ("tf", "theano", "theano_flipmask")
TOL = 1e-4


class Case(object):
    def __init__(self, variant, n_z, hidden, H, W, path="auto", nl="elu"):
        base = "tf" if variant == "tf" else "theano"
        self.variant, self.n_z, self.hidden, self.H, self.W, self.nl = variant, n_z, hidden, H, W, nl
        self.hid, self.hd = O.make_params(base, n_z, hidden, [n_z, n_z], seed=1)
        keys = "Vgb" if variant == "tf" else "wsb"
        self.keys = keys
        self.layers = [tuple(torch.from_numpy(np.ascontiguousarray(l[k])).to(DEV).requires_grad_(True) for k in keys)
                       for l in self.hid + self.hd]
        self.op = IAFOperator(base, n_z, hidden, [n_z, n_z], nl=nl, path=path,
                              flipmask=variant == "theano_flipmask").set_weights(self.layers)

    def inputs(self, B, seed=0):
        u, ctx = O.make_inputs(B, self.n_z, self.hidden[0] if self.hidden else 1, self.H, self.W, seed=seed)
        return u, (ctx if self.hidden else None)

    def dev(self, a, grad=False):
        return None if a is None else torch.from_numpy(a).to(DEV).requires_grad_(grad)

    def zero_grads(self):
        for l in self.layers:
            for t in l:
                t.grad = None


def node_grads(k, u, ctx, g):
    """step_inverse(differentiable=True) on the GPU: (z, g_u, g_ctx, [per layer {key: grad}]) as numpy."""
    k.zero_grads()
    ut, ct = k.dev(u, True), k.dev(ctx, True)
    outs = k.op.step_inverse(ut, ct, differentiable=True)
    loss = sum((o * k.dev(gi)).sum() for o, gi in zip(outs, g) if gi is not None)
    loss.backward()
    np_ = lambda t: t.detach().cpu().numpy()
    return (np_(outs[0]), np_(ut.grad), None if ct is None else np_(ct.grad),
            [{key: np_(t.grad) for key, t in zip(k.keys, l)} for l in k.layers])


def assert_matches_fp64(k, u, ctx, g):
    z, g_u, g_ctx, g_par = node_grads(k, u, ctx, g)
    zr, g_u_ref, g_ctx_ref, g_par_ref = oracle_grads(k.variant, u, ctx, k.hid, k.hd, k.nl, *g)
    assert per_sample_err(z, zr) < TOL
    assert per_sample_err(g_u, g_u_ref) < TOL, per_sample_err(g_u, g_u_ref)
    if ctx is not None:
        assert per_sample_err(g_ctx, g_ctx_ref) < TOL, per_sample_err(g_ctx, g_ctx_ref)
    for got, ref in zip(g_par, g_par_ref):
        for key in got:
            err = per_sample_err(got[key][None], ref[key][None])
            assert err < TOL, (key, err)


# ---------------------------------------------------------------------------------------------------------------------
# fp64
# ---------------------------------------------------------------------------------------------------------------------
STACKS = [(16, []), (16, [64]), (16, [48, 96]), (32, []), (32, [64]), (48, []), (48, [48, 96])]


@pytest.mark.parametrize("path", ("simt", "tc"))
@pytest.mark.parametrize("n_z,hidden", STACKS)
@pytest.mark.parametrize("variant", VARIANTS)
def test_every_gradient_matches_fp64(variant, n_z, hidden, path):
    k = Case(variant, n_z, hidden, 2, 3, path=path)
    assert k.op.path_used(2, 3, DEV) == path
    u, ctx = k.inputs(2)
    assert_matches_fp64(k, u, ctx, upstream(u.shape, "all"))


@pytest.mark.parametrize("which", ("z", "logsd", "logdet"))
def test_partial_upstreams_on_the_tensor_cores(which):
    k = Case("theano", 32, [64], 3, 3)
    assert k.op.path_used(3, 3, DEV) == "tc"
    u, ctx = k.inputs(2)
    assert_matches_fp64(k, u, ctx, upstream(u.shape, which))


# ---------------------------------------------------------------------------------------------------------------------
# the backward routes, with launches counted
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("env,route", ((None, "tc"), ("IAF_BWD_WG_TC", "tc-dgrad"), ("IAF_BWD_TC", "simt")))
def test_both_backward_routes_with_launch_counts(env, route, monkeypatch):
    if env:
        monkeypatch.setenv(env, "0")
    k = Case("theano", 32, [64], 4, 4)
    assert k.op.path_used(4, 4, DEV) == "tc" and k.op.backward_path(4, 4, DEV) == route
    u, ctx = k.inputs(3)
    g = upstream(u.shape, "all")
    assert_matches_fp64(k, u, ctx, g)
    # the node's backward = the hidden activations at z + one adjoint launch + the step's saved backward
    ut, ct = k.dev(u, True), k.dev(ctx, True)
    outs = k.op.step_inverse(ut, ct, differentiable=True)
    loss = sum((o * k.dev(gi)).sum() for o, gi in zip(outs, g))
    n0 = k.op.launch_count()
    loss.backward()
    n_node = k.op.launch_count() - n0
    layers = [tuple(t.detach() for t in l) for l in k.layers]
    z, ls = outs[0].detach(), outs[1].detach()
    with torch.no_grad():
        n0 = k.op.launch_count()
        hidden = k.op._step_train_raw(z, ct.detach(), layers)[3]
        n_train = k.op.launch_count() - n0
        n0 = k.op.launch_count()
        g_u = k.op._step_inverse_adjoint_raw(ut.detach(), ls, hidden, *(k.dev(a) for a in g), layers=layers)
        assert k.op.launch_count() == n0 + 1
        n0 = k.op.launch_count()
        k.op._backward("step", z, ct.detach(), layers, (-g_u, k.dev(g[1]), k.dev(g[2])), True,
                       saved=(ut.detach(), ls, hidden))
        n_bwd = k.op.launch_count() - n0
    assert n_node == n_train + 1 + n_bwd, (n_node, n_train, n_bwd)
    assert torch.equal(g_u, ut.grad)


# ---------------------------------------------------------------------------------------------------------------------
# the benchmark's prior shapes
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hidden", ([64], [160, 160]), ids=("c2a", "c2b"))
def test_identity_and_two_routes_at_the_benchmark_shapes(hidden):
    k = Case("theano", 32, hidden, 16, 16)
    assert k.op.path_used(16, 16, DEV) == "tc"
    u, ctx = k.inputs(8)
    g = upstream(u.shape, "all")
    ut, ct = k.dev(u), k.dev(ctx)
    with torch.no_grad():
        z, ls, _ = k.op.step_inverse(ut, ct)
        hidden_act = k.op._step_train_raw(z, ct)[3]
        g_u = k.op._step_inverse_adjoint_raw(ut, ls, hidden_act, *(k.dev(a) for a in g))
        g_zs = k.op._backward("step", z, ct, k.op._layers, (-g_u, k.dev(g[1]), k.dev(g[2])), False,
                              saved=(ut, ls, hidden_act))[0]
    assert per_sample_err(g_zs.cpu(), -g[0]) < TOL, per_sample_err(g_zs.cpu(), -g[0])
    # d logp / d (eps, context, parameters): ar_rsample's own logp, and ar_logp at its sample
    grads = []
    for route in ("own", "ar_logp"):
        k.zero_grads()
        e, c = k.dev(u, True), k.dev(ctx, True)
        zs, _, lp = k.op.ar_rsample(e, c)
        if route == "ar_logp":
            lp = k.op.ar_logp(zs, c)[2]
        lp.sum().backward()
        grads.append([e.grad.cpu(), c.grad.cpu()] + [t.grad.cpu() for l in k.layers for t in l])
    # eps and context per sample, each parameter as a whole
    for i, (a, b) in enumerate(zip(*grads)):
        err = per_sample_err(a, b) if i < 2 else per_sample_err(a[None], b[None])
        assert err < TOL, (i, err)


# ---------------------------------------------------------------------------------------------------------------------
# determinism, graphs, the window
# ---------------------------------------------------------------------------------------------------------------------
def _adjoint_inputs(k, B):
    u, ctx = k.inputs(B)
    g = upstream(u.shape, "all")
    ut, ct = k.dev(u), k.dev(ctx)
    with torch.no_grad():
        z, ls, _ = k.op.step_inverse(ut, ct)
        hidden = k.op._step_train_raw(z, ct)[3]
    return ut, ls, hidden, [k.dev(a) for a in g]


@pytest.mark.parametrize("variant", VARIANTS)
def test_adjoint_is_deterministic_and_batch_independent(variant):
    k = Case(variant, 32, [64], 16, 16)
    ut, ls, hidden, g = _adjoint_inputs(k, 40)
    with torch.no_grad():
        a = k.op._step_inverse_adjoint_raw(ut, ls, hidden, *g)
        assert torch.equal(a, k.op._step_inverse_adjoint_raw(ut, ls, hidden, *g))
        for lo, hi in ((0, 1), (5, 6), (17, 40)):
            sl = lambda t: t[lo:hi].contiguous()
            s = k.op._step_inverse_adjoint_raw(sl(ut), sl(ls), [sl(h) for h in hidden], *(sl(t) for t in g))
            assert torch.equal(s, a[lo:hi])
        # the whole node, twice
        e, c = ut.clone().requires_grad_(True), k.dev(k.inputs(40)[1], True)
        outs = []
        for _ in range(2):
            e.grad = c.grad = None
            with torch.enable_grad():
                k.op.ar_rsample(e, c)[2].sum().backward()
            outs.append((e.grad.clone(), c.grad.clone()))
        assert all(torch.equal(x, y) for x, y in zip(*outs))


def test_adjoint_in_a_cuda_graph():
    k = Case("theano", 32, [64], 16, 16)
    ut, ls, hidden, g = _adjoint_inputs(k, 32)
    with torch.no_grad():
        ref = k.op._step_inverse_adjoint_raw(ut, ls, hidden, *g)
        out = torch.empty_like(ut)
        launches = k.op.launch_count()
        graph = torch.cuda.CUDAGraph()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            with torch.cuda.graph(graph, stream=s):
                out.copy_(k.op._step_inverse_adjoint_raw(ut, ls, hidden, *g))
        torch.cuda.current_stream().wait_stream(s)
        assert k.op.launch_count() == launches + 1  # one kernel, nothing allocated
        out.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, ref)


def test_the_widest_map_that_fits_and_the_first_that_does_not():
    """c2b's stack (n_z 32, [160, 160]): the adjoint's window fits at W = 72 and not at 73 (test_made_rsample.py derives
    both); at 73 the inverse still runs, and the differentiable call refuses before launching anything."""
    w = adj_w_max(32, [160, 160])
    assert w == 72
    k = Case("theano", 32, [160, 160], 2, w)
    ut, ls, hidden, g = _adjoint_inputs(k, 2)
    with torch.no_grad():
        g_u = k.op._step_inverse_adjoint_raw(ut, ls, hidden, *g)
        z = k.op.step_inverse(ut, k.dev(k.inputs(2)[1]))[0]
        g_zs = k.op._backward("step", z, k.dev(k.inputs(2)[1]), k.op._layers, (-g_u, g[1], g[2]), False,
                              saved=(ut, ls, hidden))[0]
    assert per_sample_err(g_zs.cpu(), -g[0].cpu()) < TOL
    wide = Case("theano", 32, [160, 160], 2, w + 1)
    u, ctx = wide.inputs(2)
    with torch.no_grad():
        wide.op.step_inverse(wide.dev(u), wide.dev(ctx))
    n0 = wide.op.launch_count()
    with pytest.raises(NotImplementedError, match="not supported"):
        wide.op.ar_rsample(wide.dev(u, True), wide.dev(ctx))
    assert wide.op.launch_count() == n0
