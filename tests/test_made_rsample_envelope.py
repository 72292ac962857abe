"""The backward of the step's inverse over its own envelope on the CPU: the adjoint kernel (``iaf_inv_adj_kernel``,
iaf_inv.cu) under host emulation and the autograd node of ``step_inverse(..., differentiable=True)`` over the emulated
ABI, against a settled fp64 adjoint, and the host table (``inv_tables``, iaf_capi.cu) that says after which z channel's
step a hidden unit's gradient is final.

The adjoint's envelope: one CTA of 128 threads per sample; per pixel one pass over every stage's inputs that gathers the
non-centre taps of its output gradients from a two-row ring (the heads' 2 n_z entries mapped onto the packed columns
interleaved in groups of four over ``round_up(n_z, 4)``); then a chain over the z channels in the reverse of the mask's
order whose hidden stages read a table of "gradient final at step k" and the hidden activations at z.  The cases run it
where that logic has edges:
* the stacks of the sampler's envelope (tests/test_made_sample_envelope.py): padded heads (n_z 1, 3, 5, 7), heads wider
  than the CTA (n_z 80 and 128), three and four hidden layers, widths that step down, no hidden layer, and flipped
  [8, 4, 8];
* all six nonlinearities (the chain evaluates nl' from the kept activations);
* maps one pixel wide or one row high and non-square maps;
* the table itself, restated (``adjoint_steps``): stages whose tables differ, and the "step C" group of units no head
  depends on at the centre;
* the window on stacks without a tensor-core plan: the SIMT plan is refused at a narrower map than the adjoint's;
* the node with each combination of inputs that require grad, frozen parameters included.

The reference, ``settled_grads``: z* from the fp64 inverse, then the gradient at u as the fixed point of the transposed
chain at z*, then the context and parameter gradients from one fp64 backward of the step at z*.  It costs a few tens
of VJPs where the unrolled reference of tests/test_made_rsample.py needs n_z*H*W + 1 iterations, so it reaches the
large maps of tests/test_gpu_made_rsample_envelope.py; it is pinned to the unrolled reference here.

Every case: g_u (and z) per sample within ``TOL`` (``|d_n|_inf / max(|ref_n|_inf, 1)``), the identity of the adjoint
(the step's backward at z with upstream (-g_u, g_logsd, g_logdet) returns -g_z), and for the node g_context per sample
and every parameter gradient as a whole.  The emulation is slow (about 1 ms per barrier per sample): B = 2, small maps."""
import itertools

import numpy as np
import pytest
import torch

from iaf_b200 import _lib as L
from oracle import iaf_oracle as O
from oracle import iaf_oracle_torch as OT
from tests import flipmask_oracle as FO
from tests import test_made_sample_envelope as E
from tests.test_made_rsample import _emulated_abi, _op, _torch_op, adj_w_max, emu_adjoint, oracle_grads, upstream

VARIANTS = ("tf", "theano", "theano_flipmask")
NLS = ("none", "elu", "softplus", "relu", "tanh", "leakyrelu")
TOL = 1e-4
per_sample_err = E.per_sample_err


# ---------------------------------------------------------------------------------------------------------------------
# the settled fp64 adjoint and the restated table (tests/test_gpu_made_rsample_envelope.py uses them too)
# ---------------------------------------------------------------------------------------------------------------------
def settled_grads(variant, u, ctx, hid, hd, nl, g_z, g_logsd, g_logdet, start=None, settle=0.0):
    """fp64: (z, g_u, g_context or None, [per layer {key: grad}], iterations of the adjoint), as ``oracle_grads``.

    z* = E.inverse(u) (cold, or warm from ``start`` with the same ``settle``).  At z*, with a = 0.1 s(z*) and
    G_a = g_logsd - g_logdet, the gradient at u is the fixed point of the transposed chain
        v <- exp(a) (g_z + VJP_stack(z*)[gm = 0.1 exp(-a) v, gs = 0.1 (u v + G_a)]),
    started from v = exp(a) g_z, on one fp64 torch graph of the heads at z*.  The stack's Jacobian is strictly
    triangular in the mask's order, so every iteration makes at least one more position final and the iterate stops
    changing within n_z*H*W + 1 iterations; it stops once no element moves by more than ``settle * max(|v|_inf, 1)``,
    and raises when it has not settled by then.  The context and parameter gradients are one backward of the step at z*,
    ``((z - 0.1 m) exp(-a), a, -sum a)``, with upstream (-v, g_logsd, g_logdet)."""
    zs = E.inverse(variant, u, ctx, hid, hd, nl, start=start, settle=settle)[0]
    T = lambda a, grad=False: torch.tensor(np.asarray(a, np.float64), requires_grad=grad)
    layers = [{k: T(v, True) for k, v in l.items()} for l in hid + hd]
    hl, hh = layers[:len(hid)], layers[len(hid):]
    zt = T(zs, True)
    cc = T(ctx, True) if ctx is not None else None
    if variant == "theano_flipmask":
        m, s = FO.t_multiconv(zt, cc, hl, hh, nl, flipmask=True)
    else:
        m, s = OT.multiconv(variant, zt, cc, hl, hh, nl)
    a = 0.1 * s
    ut = T(u)
    with torch.no_grad():
        ea, ema = torch.exp(a), torch.exp(-a)
        gz = T(g_z) if g_z is not None else torch.zeros_like(ut)
        G_a = (T(g_logsd) if g_logsd is not None else torch.zeros_like(ut)) - \
            (T(g_logdet)[:, None, None, None] if g_logdet is not None else 0.0)
    v = ea * gz
    for it in range(1, u[0].size + 2):
        vjp = torch.autograd.grad((m, s), zt, (0.1 * ema * v, 0.1 * (ut * v + G_a)), retain_graph=True)[0]
        vn = ea * (gz + vjp)
        moved = float((vn - v).abs().max())
        v = vn
        if moved <= settle * max(float(v.abs().max()), 1.0):
            break
    else:
        raise AssertionError("the adjoint did not settle within n_z*H*W + 1 iterations: not the mask's order")
    outs = [((zt - 0.1 * m) * torch.exp(-a), -v)]
    if g_logsd is not None:
        outs.append((a, T(g_logsd)))
    if g_logdet is not None:
        outs.append((-a.sum(dim=(1, 2, 3)), T(g_logdet)))
    params = [t for l in layers for t in l.values()]
    inputs = ([cc] if cc is not None else []) + params
    got = torch.autograd.grad([o for o, _ in outs], inputs, [g for _, g in outs], allow_unused=True)
    got = [np.zeros(t.shape) if g is None else g.numpy() for g, t in zip(got, inputs)]
    g_ctx = got.pop(0) if cc is not None else None
    rest = iter(got)
    return zs, v.numpy(), g_ctx, [{k: next(rest) for k in l} for l in layers], it


def adjoint_steps(variant, n_z, hidden):
    """The adjoint's table restated from the mask oracles: per hidden layer an int array, the step (in the mask's order)
    at which the unit's gradient is final, i.e. the earliest step among its live centre consumers in the stage above;
    n_z ("step C", before the chain) when no unit above reads it at the centre."""
    pos = np.arange(n_z)[::-1] if variant == "theano_flipmask" else np.arange(n_z)
    sizes, steps, nxt = [n_z] + list(hidden), [None] * len(hidden), pos
    for j in range(len(hidden) - 1, -1, -1):
        m = E.centre_mask(variant, sizes[j + 1], hidden[j + 1] if j + 1 < len(hidden) else n_z, j + 1 == len(hidden))
        nxt = np.array([nxt[m[u]].min() if m[u].any() else n_z for u in range(sizes[j + 1])])
        steps[j] = nxt
    return steps


# ---------------------------------------------------------------------------------------------------------------------
# checks
# ---------------------------------------------------------------------------------------------------------------------
def _case(variant, n_z, hidden, H, W, B=2):
    base = "tf" if variant == "tf" else "theano"
    hid, hd = O.make_params(base, n_z, hidden, [n_z, n_z], seed=1)
    u, ctx = O.make_inputs(B, n_z, hidden[0] if hidden else 1, H, W, seed=0)
    return hid, hd, u, (ctx if hidden else None)


def check_emulated(variant, n_z, hidden, H, W, nl="elu", which="all", B=2):
    """The emulated adjoint (one launch) against the settled fp64 adjoint, and its identity through the step's
    backward."""
    hid, hd, u, ctx = _case(variant, n_z, hidden, H, W, B)
    op = _op(variant, n_z, hidden, H, W, nl)[0]
    g = upstream(u.shape, which)
    z, ls, hidden_act, g_u = emu_adjoint(op, u, ctx, *g)
    zr, g_u_ref, _, _, _ = settled_grads(variant, u, ctx, hid, hd, nl, *g)
    assert per_sample_err(z, zr) < TOL, per_sample_err(z, zr)
    assert per_sample_err(g_u, g_u_ref) < TOL, per_sample_err(g_u, g_u_ref)
    g_zs = op.step_bwd_saved(z, ctx, u, ls, hidden_act, np.ascontiguousarray(-g_u), g[1], g[2], params=False)[0]
    minus_gz = -g[0] if g[0] is not None else np.zeros_like(u)
    assert per_sample_err(g_zs, minus_gz) < TOL, per_sample_err(g_zs, minus_gz)


def node_grads(variant, n_z, hidden, nl, hid, hd, u, ctx, g, eps=True, context=True, params=True):
    """step_inverse(differentiable=True) over the emulated ABI with the chosen inputs requiring grad: (z, g_u, g_ctx,
    [per layer (grads)], launches of the backward, the operator); a gradient not asked for is None."""
    op, layers = _torch_op(variant, n_z, hidden, hid, hd, nl, grad=params)
    ut = torch.from_numpy(u).requires_grad_(eps)
    ct = torch.from_numpy(ctx).requires_grad_(context) if ctx is not None else None
    outs = op.step_inverse(ut, ct, differentiable=True)
    loss = sum((o * torch.from_numpy(gi)).sum() for o, gi in zip(outs, g) if gi is not None)
    n0 = op.launch_count()
    loss.backward()
    n_bwd = op.launch_count() - n0
    return (outs[0].detach(), ut.grad, None if ct is None else ct.grad, [[t.grad for t in l] for l in layers], n_bwd,
            op)


def check_node(variant, n_z, hidden, H, W, nl="elu", which="all", B=2):
    """The node over the emulated ABI: z, g_u, g_context and every parameter gradient against the settled fp64
    adjoint."""
    hid, hd, u, ctx = _case(variant, n_z, hidden, H, W, B)
    g = upstream(u.shape, which)
    z, g_u, g_ctx, g_par, _, _ = node_grads(variant, n_z, hidden, nl, hid, hd, u, ctx, g)
    zr, g_u_ref, g_ctx_ref, g_par_ref, _ = settled_grads(variant, u, ctx, hid, hd, nl, *g)
    assert per_sample_err(z, zr) < TOL
    assert per_sample_err(g_u, g_u_ref) < TOL, per_sample_err(g_u, g_u_ref)
    if ctx is not None:
        assert per_sample_err(g_ctx, g_ctx_ref) < TOL, per_sample_err(g_ctx, g_ctx_ref)
    keys = "Vgb" if variant == "tf" else "wsb"
    for got, ref in zip(g_par, g_par_ref):
        for t, k in zip(got, keys):
            err = per_sample_err(t[None], ref[k][None])
            assert err < TOL, (k, err)


# ---------------------------------------------------------------------------------------------------------------------
# the reference
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("settle", (0.0, 1e-13))
@pytest.mark.parametrize("n_z,hidden,H,W", [(4, [8], 3, 3), (5, [10], 2, 3), (4, [], 2, 3)])
@pytest.mark.parametrize("variant", VARIANTS)
def test_the_settled_adjoint_matches_the_unrolled_fixed_point(variant, n_z, hidden, H, W, settle):
    """Two fp64 references that share nothing but the forward oracles: autograd through the unrolled fixed point, and
    the settled adjoint at z*.  They agree to a few ulp of fp64, and the adjoint settles well within its bound."""
    hid, hd, u, ctx = _case(variant, n_z, hidden, H, W)
    g = upstream(u.shape, "all")
    zu, g_u_u, g_ctx_u, g_par_u = oracle_grads(variant, u, ctx, hid, hd, "elu", *g)
    zs, g_u_s, g_ctx_s, g_par_s, iters = settled_grads(variant, u, ctx, hid, hd, "elu", *g, settle=settle)
    assert iters <= n_z * H * W + 1
    rel = lambda a, b: float(np.abs(a - b).max() / max(np.abs(b).max(), 1.0))
    assert rel(zs, zu) < 1e-12
    assert rel(g_u_s, g_u_u) < 1e-12, rel(g_u_s, g_u_u)
    if ctx is not None:
        assert rel(g_ctx_s, g_ctx_u) < 1e-12, rel(g_ctx_s, g_ctx_u)
    for a, b in zip(g_par_s, g_par_u):
        for k in a:
            assert rel(a[k], b[k]) < 1e-12, (k, rel(a[k], b[k]))


# ---------------------------------------------------------------------------------------------------------------------
# stack shapes: the sampler's matrix, and [8, 4, 8] flipped
# ---------------------------------------------------------------------------------------------------------------------
FLIP_ONLY = (16, [8, 4, 8], 2, 2)  # triangular only in the reversed order (tests/test_made_sample_envelope.py)


def _stack_cases():
    for v, s in itertools.product(VARIANTS, E.STACKS + [FLIP_ONLY]):
        if s != FLIP_ONLY or v == "theano_flipmask":
            yield (v,) + s


@pytest.mark.parametrize("variant,n_z,hidden,H,W", list(_stack_cases()))
def test_stack_shapes(variant, n_z, hidden, H, W, monkeypatch):
    check_emulated(variant, n_z, hidden, H, W)
    with _emulated_abi(monkeypatch):
        check_node(variant, n_z, hidden, H, W)


# ---------------------------------------------------------------------------------------------------------------------
# nonlinearities and maps
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("nl", NLS)
@pytest.mark.parametrize("n_z,hidden,H,W", [(8, [16, 16], 2, 2), (4, [8], 2, 3)])
def test_every_nonlinearity(variant, nl, n_z, hidden, H, W, monkeypatch):
    check_emulated(variant, n_z, hidden, H, W, nl)
    with _emulated_abi(monkeypatch):
        check_node(variant, n_z, hidden, H, W, nl)


# 1x1: one pixel on all four borders; 1xW: every pixel on the top border of the adjoint's raster order; Hx1: every
# pixel on both x borders; 3x17 and 17x3: rows that wrap the ring many times, and the transposed shape
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("H,W", E.MAPS)
def test_maps(variant, H, W, monkeypatch):
    check_emulated(variant, 4, [8], H, W)
    with _emulated_abi(monkeypatch):
        check_node(variant, 4, [8], H, W)


# ---------------------------------------------------------------------------------------------------------------------
# the adjoint's table
# ---------------------------------------------------------------------------------------------------------------------
def test_the_table_of_every_stack_of_the_matrix():
    """Every hidden unit's gradient is final no earlier than (in the chain's backward order) the step after which the
    unit itself is final in the inverse (E.final_steps), which is what lets the chain read each z channel's
    accumulator complete; and every stage is spread over more than one step."""
    for v, (n_z, hidden, _, _) in itertools.product(VARIANTS, E.STACKS):
        fwd, tri = E.final_steps(v, n_z, hidden)
        assert tri
        adj = adjoint_steps(v, n_z, hidden)
        for j, (f, a) in enumerate(zip(fwd, adj)):
            assert len(a) == hidden[j] and (a > f).all(), (v, n_z, hidden, j)
            if n_z > 1:
                assert len(set(a.tolist())) > 1, (v, n_z, hidden, j)


def test_stages_whose_tables_differ_from_stage_one():
    """A kernel that read stage 1's table at a later stage would finalise the wrong units.  In [16, 32, 16, 8] stages 2
    and 3 have tables of their own in every variant; unflipped, [8, 8, 8], [32, 32, 32] and stages 1-2 of [8, 4, 4]
    share one table, so only a stack like the former (or flipmask) can tell the two kernels apart."""
    for v in VARIANTS:
        steps = adjoint_steps(v, 8, [16, 32, 16, 8])
        for j in (2, 3):
            assert not np.array_equal(steps[j], steps[1]), (v, j)
    for v in ("tf", "theano"):
        for n_z, hidden in ((4, [8, 8, 8]), (16, [32, 32, 32])):
            steps = adjoint_steps(v, n_z, hidden)
            assert all(np.array_equal(s, steps[1]) for s in steps), (v, n_z, hidden)
        steps = adjoint_steps(v, 16, [8, 4, 4])
        assert np.array_equal(steps[1], steps[2])


def test_step_c_groups_run_at_every_stage_where_they_occur():
    """Units that no head depends on at the centre get their gradient before the chain (the table's "step C" group).
    Every variant has them; for each variant and each stage index at which any legal stack of up to four hidden layers
    has such a group, some stack of the matrix runs one there."""
    in_matrix = {v: set() for v in VARIANTS}
    for v, (n_z, hidden, _, _) in itertools.product(VARIANTS, E.STACKS + [FLIP_ONLY]):
        if (n_z, hidden) == FLIP_ONLY[:2] and v != "theano_flipmask":
            continue
        in_matrix[v] |= {j for j, s in enumerate(adjoint_steps(v, n_z, hidden)) if (s == n_z).any()}
    for v in VARIANTS:
        legal = set()
        for n_z, hidden in itertools.chain(E._legal_stacks(8, 2), [(s[0], s[1]) for s in E.STACKS]):
            if E.final_steps(v, n_z, hidden)[1]:
                legal |= {j for j, s in enumerate(adjoint_steps(v, n_z, hidden)) if (s == n_z).any()}
        assert legal, v
        assert legal <= in_matrix[v], (v, legal, in_matrix[v])
        assert in_matrix[v] == {0, 1, 2, 3}, (v, in_matrix[v])


# ---------------------------------------------------------------------------------------------------------------------
# the window on stacks without a tensor-core plan
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_z,hidden,w_simt,w_adj", [(8, [16, 32, 16, 8], 168, 324), (80, [160], 72, 87)])
def test_the_simt_plan_is_refused_before_the_adjoint_window_could_overflow(n_z, hidden, w_simt, w_adj):
    """The SIMT step keeps at least 2 + n_hidden rows; the adjoint keeps two rows of every stage's output gradients.
    On these stacks, which the tensor cores do not take, the SIMT plan's one-row limit (E.simt_smem) is narrower than
    the adjoint's (adj_w_max), so the adjoint never refuses on its own there: at the SIMT plan's widest map the adjoint
    is available, and one column more there is no plan at all."""
    assert adj_w_max(n_z, hidden) == w_adj
    assert max(W for W in range(1, w_adj + 2) if E.simt_smem(n_z, hidden, W) <= E.SMEM_LIMIT) == w_simt
    for v in VARIANTS:
        op = _op(v, n_z, hidden, 2, w_simt)[0]
        assert op.lib.iaf_step_inverse_adjoint(op.plan, None, None, None, None, None, None, None, 0, None) == L.OK
        for W in (w_simt + 1, w_adj + 1):
            with pytest.raises(RuntimeError, match="status %d" % L.ERR_UNSUPPORTED):
                _op(v, n_z, hidden, 2, W)


# ---------------------------------------------------------------------------------------------------------------------
# the node's inputs
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("eps,context,params", [(True, False, False), (False, True, False), (False, False, True),
                                                (True, True, False)],
                         ids=("eps", "context", "params", "eps+context"))
def test_each_combination_of_inputs_that_require_grad(variant, eps, context, params, monkeypatch):
    """The gradients asked for match fp64 and the others are None.  With only eps requiring grad the backward is the
    training forward at z and one adjoint launch, without the step's backward."""
    n_z, hidden, H, W = 4, [8], 2, 3
    hid, hd, u, ctx = _case(variant, n_z, hidden, H, W)
    g = upstream(u.shape, "all")
    zr, g_u_ref, g_ctx_ref, g_par_ref, _ = settled_grads(variant, u, ctx, hid, hd, "elu", *g)
    with _emulated_abi(monkeypatch):
        z, g_u, g_ctx, g_par, n_bwd, op = node_grads(variant, n_z, hidden, "elu", hid, hd, u, ctx, g, eps, context,
                                                     params)
        with torch.no_grad():
            n0 = op.launch_count()
            op._step_train_raw(z, torch.from_numpy(ctx))
            n_train = op.launch_count() - n0
    assert per_sample_err(z, zr) < TOL
    if eps:
        assert per_sample_err(g_u, g_u_ref) < TOL, per_sample_err(g_u, g_u_ref)
    else:
        assert g_u is None
    if context:
        assert per_sample_err(g_ctx, g_ctx_ref) < TOL, per_sample_err(g_ctx, g_ctx_ref)
    else:
        assert g_ctx is None
    keys = "Vgb" if variant == "tf" else "wsb"
    for got, ref in zip(g_par, g_par_ref):
        for t, k in zip(got, keys):
            if params:
                assert per_sample_err(t[None], ref[k][None]) < TOL, k
            else:
                assert t is None
    if eps and not context and not params:
        assert n_bwd == n_train + 1, (n_bwd, n_train)
    else:
        assert n_bwd > n_train + 1, (n_bwd, n_train)


def test_a_map_the_step_backward_does_not_take(monkeypatch):
    """On one row the step's backward plan takes (4, [8]) up to W = 124 (its weight-gradient window), the adjoint up to
    W = 1797.  At W = 125 the node still gives the gradient at u, which needs no step backward, and it refuses before
    launching anything when the context or the parameters require grad, instead of failing half-way through its
    backward."""
    n_z, hidden, W = 4, [8], 125
    for w, rc in ((W - 1, L.OK), (W, L.ERR_UNSUPPORTED)):
        op = _op("theano", n_z, hidden, 1, w)[0]
        assert min(op.lib.iaf_plan_bwd_path(op.plan), 0) == rc
    assert adj_w_max(n_z, hidden) == 1797
    hid, hd, u, ctx = _case("theano", n_z, hidden, 1, W, B=1)
    g = upstream(u.shape, "all")
    zr, g_u_ref, _, _, _ = settled_grads("theano", u, ctx, hid, hd, "elu", *g)
    with _emulated_abi(monkeypatch):
        z, g_u, g_ctx, g_par, _, op = node_grads("theano", n_z, hidden, "elu", hid, hd, u, ctx, g, context=False,
                                                 params=False)
        assert per_sample_err(z, zr) < TOL and per_sample_err(g_u, g_u_ref) < TOL
        assert g_ctx is None and all(t is None for l in g_par for t in l)
        for context, params in ((True, False), (False, True)):
            op, _ = _torch_op("theano", n_z, hidden, hid, hd, "elu", grad=params)
            op.path_used(1, W, "cpu")
            n0 = op.launch_count()
            with pytest.raises(NotImplementedError, match="not supported"):
                op.ar_rsample(torch.from_numpy(u).requires_grad_(True), torch.from_numpy(ctx).requires_grad_(context))
            assert op.launch_count() == n0
