"""The backward of the step's inverse on the CPU: the adjoint kernel (``iaf_inv_adj_kernel``, iaf_inv.cu) under host
emulation, and the autograd node of ``IAFOperator.step_inverse(..., differentiable=True)`` / ``ar_rsample`` over the
emulated ABI, against the fp64 gradient of the inverse.

The fp64 reference is torch autograd through the unrolled fixed point ``z <- 0.1 m(z) + exp(0.1 s(z)) u`` on the
forward oracles (``oracle/iaf_oracle_torch``, ``tests/flipmask_oracle``).  After n_z*H*W + 1 iterations the iterate
equals the inverse as a function of (u, context, parameters), not only at the one point (each iteration makes one more
position of the triangular chain exact, values and derivatives alike), so its gradient is the inverse's exactly.

Every case: ``|d_n|_inf / max(|ref_n|_inf, 1) <= TOL`` per sample n for g_u and g_context, the same over the whole
tensor for each parameter gradient, and the identity of the adjoint: the step's own backward at z with upstream
(-g_u, g_logsd, g_logdet) returns -g_z.  The emulation is slow (about 1 ms per barrier per sample): B = 2, small maps.
tests/test_gpu_made_rsample.py runs the same comparison on the H100."""
import contextlib
import ctypes as C
import itertools

import numpy as np
import pytest
import torch

from iaf_b200 import _lib as L
from oracle import iaf_oracle as O
from oracle import iaf_oracle_torch as OT
from tests import flipmask_oracle as FO
from tests.emu.harness import EmuOperator, _arr, _check, _p
from tests.emu.inverse import EmuInvOperator
from tests.test_made_sample_envelope import SMEM_LIMIT, final_steps, per_sample_err

VARIANTS = ("tf", "theano", "theano_flipmask")
NLS = ("none", "elu", "softplus", "relu", "tanh", "leakyrelu")
UPSTREAMS = ("z", "logsd", "logdet", "all")
TOL = 1e-4


# ---------------------------------------------------------------------------------------------------------------------
# fp64 reference, restated window (tests/test_gpu_made_rsample.py uses them too)
# ---------------------------------------------------------------------------------------------------------------------
def upstream(shape, which, seed=3):
    """(g_z, g_logsd, g_logdet) float32, None where ``which`` ("z" | "logsd" | "logdet" | "all") leaves it out."""
    rng = np.random.RandomState(seed)
    g = [rng.randn(*shape).astype(np.float32), rng.randn(*shape).astype(np.float32),
         rng.randn(shape[0]).astype(np.float32)]
    keep = {"z": (0,), "logsd": (1,), "logdet": (2,), "all": (0, 1, 2)}[which]
    return tuple(t if i in keep else None for i, t in enumerate(g))


def oracle_grads(variant, u, ctx, hid, hd, nl, g_z, g_logsd, g_logdet):
    """fp64 autograd through the unrolled fixed point: (z, g_u, g_context or None, [per layer {key: grad}])."""
    T = lambda a: torch.tensor(np.asarray(a, np.float64), requires_grad=True)
    layers = [{k: T(v) for k, v in l.items()} for l in hid + hd]
    hl, hh = layers[:len(hid)], layers[len(hid):]
    uu = T(u)
    cc = T(ctx) if ctx is not None else None

    def heads(z):
        if variant == "theano_flipmask":
            return FO.t_multiconv(z, cc, hl, hh, nl, flipmask=True)
        return OT.multiconv(variant, z, cc, hl, hh, nl)
    z = uu
    for _ in range(u[0].size + 1):
        m, s = heads(z)
        z = 0.1 * m + torch.exp(0.1 * s) * uu
    a = 0.1 * heads(z)[1]
    loss = 0.0
    for out, g in ((z, g_z), (a, g_logsd), (-a.sum(dim=(1, 2, 3)), g_logdet)):
        if g is not None:
            loss = loss + (out * torch.from_numpy(np.asarray(g, np.float64))).sum()
    params = [t for l in layers for t in l.values()]
    inputs = [uu] + ([cc] if cc is not None else []) + params
    got = torch.autograd.grad(loss, inputs, allow_unused=True)
    got = [np.zeros(t.shape) if g is None else g.numpy() for g, t in zip(got, inputs)]
    g_u, rest = got[0], got[1:]
    g_ctx = rest.pop(0) if cc is not None else None
    it = iter(rest)
    return z.detach().numpy(), g_u, g_ctx, [{k: next(it) for k in l} for l in layers]


def adj_smem(n_z, hidden, W):
    """Bytes of the adjoint's window (inv_tables): per stage two rows of its output gradients over W + 2 columns (the
    heads' 2 n_z, the hidden layers' own widths), per stage the accumulators of its input (n_z, then each hidden
    width)."""
    return 4 * (2 * (W + 2) * (2 * n_z + sum(hidden)) + n_z + sum(hidden))


def adj_w_max(n_z, hidden):
    """The widest map whose adjoint window fits."""
    return (SMEM_LIMIT // 4 - n_z - sum(hidden)) // (2 * (2 * n_z + sum(hidden))) - 2


# ---------------------------------------------------------------------------------------------------------------------
# the emulated ABI
# ---------------------------------------------------------------------------------------------------------------------
def _op(variant, n_z, hidden, H, W, nl="elu", seed=1):
    base = "tf" if variant == "tf" else "theano"
    hid, hd = O.make_params(base, n_z, hidden, [n_z, n_z], seed=seed)
    keys = "Vgb" if variant == "tf" else "wsb"
    op = EmuInvOperator(variant, n_z, hidden, [n_z, n_z], H, W, nl=nl).set_weights(
        [tuple(l[k] for k in keys) for l in hid + hd])
    return op, hid, hd


def emu_adjoint(op, u, ctx, g_z, g_logsd, g_logdet):
    """inverse, the hidden activations at z, the adjoint: (z, logsd, hidden, g_u); one launch for the adjoint."""
    B = u.shape[0]
    z, ls = np.full_like(u, np.nan), np.full_like(u, np.nan)
    _check(op.lib.iaf_step_inverse(op.plan, _p(u), _p(ctx), _p(z), _p(ls), None, B, None))
    hidden = op.step_train(z, ctx)[3]
    g_u = np.full_like(u, np.nan)
    gz = g_z if g_z is not None else np.zeros_like(u)
    n0 = op.lib.iaf_plan_launch_count(op.plan)
    _check(op.lib.iaf_step_inverse_adjoint(op.plan, _p(u), _p(ls), _arr(hidden) if hidden else None, _p(gz),
                                           _p(g_logsd), _p(g_logdet), _p(g_u), B, None))
    assert op.lib.iaf_plan_launch_count(op.plan) == n0 + 1
    return z, ls, hidden, g_u


def check_emulated(variant, n_z, hidden, H, W, nl="elu", which="all", B=2):
    """The emulated adjoint's g_u against fp64, and the identity through the step's backward."""
    op, hid, hd = _op(variant, n_z, hidden, H, W, nl)
    u, ctx = O.make_inputs(B, n_z, hidden[0] if hidden else 1, H, W, seed=0)
    ctx = ctx if hidden else None
    g = upstream(u.shape, which)
    z, ls, hidden_act, g_u = emu_adjoint(op, u, ctx, *g)
    zr, g_u_ref, _, _ = oracle_grads(variant, u, ctx, hid, hd, nl, *g)
    assert per_sample_err(z, zr) < TOL
    assert per_sample_err(g_u, g_u_ref) < TOL, per_sample_err(g_u, g_u_ref)
    # the step's backward at z with upstream -g_u returns -g_z (zero without a g_z upstream)
    g_zs = op.step_bwd_saved(z, ctx, u, ls, hidden_act, np.ascontiguousarray(-g_u), g[1], g[2], params=False)[0]
    minus_gz = -g[0] if g[0] is not None else np.zeros_like(u)
    assert per_sample_err(g_zs, minus_gz) < TOL, per_sample_err(g_zs, minus_gz)
    return op, u, ctx, g


# ---------------------------------------------------------------------------------------------------------------------
# the Python node over the emulated ABI
# ---------------------------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def _emulated_abi(monkeypatch):
    """Point the ctypes binding at the host-emulated library (test only; the product refuses CPU tensors)."""
    from iaf_b200 import ops
    from tests.emu.inverse import emu

    def check_input(t, name, shape=None):
        assert isinstance(t, torch.Tensor) and t.dtype == torch.float32
        if shape is not None:
            assert tuple(t.shape) == tuple(shape)
        return t.contiguous()
    monkeypatch.setattr(L, "lib", emu)
    monkeypatch.setattr(ops, "_check_input", check_input)
    monkeypatch.setattr(ops, "_stream", lambda device: C.c_void_p(0))
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    yield


def _torch_op(variant, n_z, hidden, hid, hd, nl, grad=True):
    from iaf_b200 import ops
    keys = "Vgb" if variant == "tf" else "wsb"
    layers = [tuple(torch.from_numpy(np.ascontiguousarray(l[k])).requires_grad_(grad) for k in keys) for l in hid + hd]
    op = ops.IAFOperator("tf" if variant == "tf" else "theano", n_z, hidden, [n_z, n_z], nl=nl, path="simt",
                         flipmask=variant == "theano_flipmask").set_weights(layers)
    return op, layers


def check_node(variant, n_z, hidden, H, W, nl="elu", which="all", B=2):
    """step_inverse(differentiable=True) over the emulated ABI: every gradient against fp64."""
    base = "tf" if variant == "tf" else "theano"
    hid, hd = O.make_params(base, n_z, hidden, [n_z, n_z], seed=1)
    u, ctx = O.make_inputs(B, n_z, hidden[0] if hidden else 1, H, W, seed=0)
    ctx = ctx if hidden else None
    g = upstream(u.shape, which)
    op, layers = _torch_op(variant, n_z, hidden, hid, hd, nl)
    ut = torch.from_numpy(u).requires_grad_(True)
    ct = torch.from_numpy(ctx).requires_grad_(True) if ctx is not None else None
    outs = op.step_inverse(ut, ct, differentiable=True)
    loss = sum((o * torch.from_numpy(gi)).sum() for o, gi in zip(outs, g) if gi is not None)
    loss.backward()
    zr, g_u_ref, g_ctx_ref, g_par_ref = oracle_grads(variant, u, ctx, hid, hd, nl, *g)
    assert per_sample_err(outs[0].detach(), zr) < TOL
    assert per_sample_err(ut.grad, g_u_ref) < TOL, per_sample_err(ut.grad, g_u_ref)
    if ct is not None:
        assert per_sample_err(ct.grad, g_ctx_ref) < TOL, per_sample_err(ct.grad, g_ctx_ref)
    keys = "Vgb" if variant == "tf" else "wsb"
    for l, ref in zip(layers, g_par_ref):
        for t, k in zip(l, keys):
            err = per_sample_err(t.grad[None], ref[k][None])
            assert err < TOL, (k, err)


# ---------------------------------------------------------------------------------------------------------------------
# the matrix
# ---------------------------------------------------------------------------------------------------------------------
STACKS = [
    # n_z, hidden, H, W
    (4, [], 3, 3),
    (4, [8], 3, 3),
    (8, [16, 16], 2, 3),
    (4, [8, 8, 8], 2, 3),
]
FLIP_ONLY = (16, [8, 4, 8], 2, 2)  # triangular only in the reversed order (test_made_sample_envelope.py)


def _stack_cases():
    for v, s in itertools.product(VARIANTS, STACKS + [FLIP_ONLY]):
        if s != FLIP_ONLY or v == "theano_flipmask":
            yield (v,) + s


@pytest.mark.parametrize("variant,n_z,hidden,H,W", list(_stack_cases()))
def test_stack_shapes(variant, n_z, hidden, H, W, monkeypatch):
    check_emulated(variant, n_z, hidden, H, W)
    with _emulated_abi(monkeypatch):
        check_node(variant, n_z, hidden, H, W)


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("nl", NLS)
def test_every_nonlinearity(variant, nl):
    check_emulated(variant, 4, [8, 8], 2, 3, nl)


# 1x1: one pixel on all four borders; 1x9: every pixel on the top and bottom border; 9x1: on both x borders
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("H,W", [(1, 1), (1, 9), (9, 1), (3, 5)])
def test_maps(variant, H, W):
    check_emulated(variant, 4, [8], H, W)


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("which", UPSTREAMS)
def test_partial_upstreams(variant, which, monkeypatch):
    check_emulated(variant, 4, [8], 2, 3, which=which)
    with _emulated_abi(monkeypatch):
        check_node(variant, 4, [8], 2, 3, which=which)


def test_the_table_restated():
    """The adjoint's "final after step k" table in Python, from the mask oracles: the unit's earliest live centre
    consumer in the mask's order.  Every stack above is triangular, and every hidden unit is final at or before (in the
    backward chain: no earlier than) the step of the last z channel it reads, which is what lets the chain read each
    z channel's accumulator complete."""
    for v, (n_z, hidden, _, _) in itertools.product(VARIANTS, STACKS):
        fwd, tri = final_steps(v, n_z, hidden)
        assert tri
        pos = np.arange(n_z)[::-1] if v == "theano_flipmask" else np.arange(n_z)
        sizes = [n_z] + list(hidden)
        from tests.test_made_sample_envelope import centre_mask
        nxt = pos
        for j in range(len(hidden) - 1, -1, -1):
            m = centre_mask(v, sizes[j + 1], hidden[j + 1] if j + 1 < len(hidden) else n_z, j + 1 == len(hidden))
            adj = np.array([nxt[m[u]].min() if m[u].any() else n_z for u in range(sizes[j + 1])])
            assert (adj > fwd[j]).all(), (v, n_z, hidden, j)
            nxt = adj


@pytest.mark.parametrize("variant", VARIANTS)
def test_g_u_is_bit_identical_across_batch_sizes(variant):
    op, hid, hd = _op(variant, 8, [16], 3, 4)
    u, ctx = O.make_inputs(3, 8, 16, 3, 4, seed=0)
    g = upstream(u.shape, "all")
    full = emu_adjoint(op, u, ctx, *g)[3]
    for b in range(3):
        sl = lambda a: None if a is None else np.ascontiguousarray(a[b:b + 1])
        one = emu_adjoint(op, sl(u), sl(ctx), sl(g[0]), sl(g[1]), sl(g[2]))[3]
        assert np.array_equal(one[0], full[b])


# ---------------------------------------------------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------------------------------------------------
def test_the_window_formula_and_its_boundary():
    """adj_smem: 4 (2 (W + 2) (2 n_z + sum hidden) + n_z + sum hidden) bytes, limit 225 KiB = 57600 floats.
    c2b (n_z 32, [160, 160]): 2 n_z + sum hidden = 384, so 768 (W + 2) + 352 <= 57600, W + 2 <= 74.5: W <= 72
    (W 72: 56832 + 352 = 57184 floats; W 73: 57600 + 352 = 57952).  c2a (n_z 32, [64]): 256 (W + 2) + 96 <= 57600,
    W <= 222.  n_z 48 without a hidden layer: 192 (W + 2) + 48 <= 57600, W <= 297 (W 298: 57648 floats)."""
    for (n_z, hidden), w in (((32, [160, 160]), 72), ((32, [64]), 222), ((48, []), 297)):
        assert adj_w_max(n_z, hidden) == w
        assert adj_smem(n_z, hidden, w) <= SMEM_LIMIT < adj_smem(n_z, hidden, w + 1)
    assert adj_smem(32, [160, 160], 72) == 4 * 57184 and adj_smem(48, [], 298) == 4 * 57648


def _query(op):
    return op.lib.iaf_step_inverse_adjoint(op.plan, None, None, None, None, None, None, None, 0, None)


def test_the_adjoint_refuses_where_its_window_does_not_fit(monkeypatch):
    """Without a hidden layer the SIMT plan and the inverse still fit at W = 298 on one row (the inverse's window is
    half the adjoint's rings); the adjoint refuses there, and takes W = 297."""
    n_z = 48
    ok = _op("theano", n_z, [], 1, adj_w_max(n_z, []))[0]
    assert _query(ok) == L.OK
    wide = _op("theano", n_z, [], 1, adj_w_max(n_z, []) + 1)[0]
    assert _query(wide) == L.ERR_UNSUPPORTED
    u = np.zeros((1, n_z, 1, 299), np.float32)
    g_u = np.empty_like(u)
    assert wide.lib.iaf_step_inverse_adjoint(wide.plan, _p(u), _p(u), None, _p(u), None, None, _p(g_u), 1, None) == \
        L.ERR_UNSUPPORTED
    # the Python node refuses before launching anything
    with _emulated_abi(monkeypatch):
        hid, hd = O.make_params("theano", n_z, [], [n_z, n_z], seed=1)
        op, _ = _torch_op("theano", n_z, [], hid, hd, "elu")
        e = torch.zeros((1, n_z, 1, 298), requires_grad=True)
        op.path_used(1, 298, "cpu")  # plan and packed weights
        n0 = op.launch_count()
        with pytest.raises(NotImplementedError, match="not supported"):
            op.step_inverse(e, None, differentiable=True)
        with pytest.raises(NotImplementedError, match="not supported"):
            op.ar_rsample(e, None)
        assert op.launch_count() == n0


def test_the_adjoint_checks_its_plan_and_arguments():
    op, hid, hd = _op("theano", 4, [8], 3, 3)
    u, ctx = O.make_inputs(2, 4, 8, 3, 3, seed=0)
    g_u = np.empty_like(u)
    h = [np.zeros((2, 8, 3, 3), np.float32)]
    call = lambda o, hidden, gz, B=2: o.lib.iaf_step_inverse_adjoint(o.plan, _p(u), _p(u), hidden, _p(gz), None, None,
                                                                     _p(g_u), B, None)
    assert call(op, None, u) == L.ERR_BAD_ARG                 # hidden activations
    assert call(op, _arr(h), None) == L.ERR_BAD_ARG           # g_z
    assert call(op, _arr(h), u, B=-1) == L.ERR_BAD_ARG
    fresh = EmuInvOperator("theano", 4, [8], [4, 4], 3, 3)
    assert _query(fresh) == L.ERR_NOT_PACKED
    # one head: no step, no inverse
    one = EmuInvOperator("theano", 4, [8], [4], 3, 3)
    p1, h1 = O.make_params("theano", 4, [8], [4], seed=1)
    one.set_weights([tuple(l[k] for k in "wsb") for l in p1 + h1])
    assert _query(one) == L.ERR_BAD_SHAPE
    # a stack that is not triangular in the mask's order has no inverse, so no adjoint
    nt = _op("theano", 16, [8, 4, 8], 2, 2)[0]
    assert not final_steps("theano", 16, [8, 4, 8])[1]
    assert _query(nt) == L.ERR_UNSUPPORTED
    # the C ABI built without iaf_inv.cu refuses, it does not fall back
    plain = EmuOperator("theano", 4, [8], [4, 4], 3, 3).set_weights([tuple(l[k] for k in "wsb") for l in hid + hd])
    assert _query(plain) == L.ERR_UNSUPPORTED


def test_default_behaviour_is_unchanged_under_autograd(monkeypatch):
    """Without differentiable=True the inverse still refuses under autograd, and ar_sample always does; outside
    autograd ar_rsample is ar_sample."""
    with _emulated_abi(monkeypatch):
        hid, hd = O.make_params("theano", 4, [8], [4, 4], seed=1)
        op, _ = _torch_op("theano", 4, [8], hid, hd, "elu")
        eps, ctx = (torch.from_numpy(a) for a in O.make_inputs(2, 4, 8, 3, 3, seed=0))
        with pytest.raises(NotImplementedError, match="no_grad"):
            op.step_inverse(eps, ctx)
        with pytest.raises(NotImplementedError, match="no_grad"):
            op.ar_sample(eps, ctx)
        with torch.no_grad():
            a, b = op.ar_sample(eps, ctx), op.ar_rsample(eps, ctx)
        assert all(torch.equal(x, y) for x, y in zip(a, b))
        z, bc, lp = op.ar_rsample(eps, ctx)
        assert z.requires_grad and lp.requires_grad
        assert torch.equal(z.detach(), a[0]) and torch.equal(lp.detach(), a[2])
