"""The inverse of the IAF step (``iaf_inv_kernel``: ``IAFOperator.step_inverse`` / ``ar_sample``) on the H100 over its
own envelope, against fp64.

The kernel runs one CTA of 128 threads per sample, keeps per stage a two-row ring of its input in shared memory (at
most 225 KiB), reads a host table of which hidden units become final after which z channel, and finds the heads
interleaved in groups of four columns over ``head_pad = round_up(n_z, 4)``.  Every plan runs it, tensor-core plans
included, on the SIMT pack.  The cases: stack shapes (padded heads, heads of 160 and 256 columns, three and four
hidden layers, widths that step down, no hidden layer), every nonlinearity, maps one pixel wide or one row high, a
1x300 row and 64x64, the shared-memory limit of two more tensor-core stacks, and the refusal of a SIMT-only stack's
plan before its window could overflow, tensor-core plans (the same bits as a SIMT plan, and the sample's density
against the tensor-core ``ar_logp``), re-packing after ``set_weights`` / ``invalidate()``, two operators alternating,
batches past the first wave, non-finite samples, and the NULL-output combinations.

Every fp64 case asserts: z, arw_logsd and logdet per sample within ``TOL`` (``|d_n|_inf / max(|ref_n|_inf, 1)``), the
round trip step(z) == u on the same operator, and exactly one launch per ``step_inverse``.  The reference is
``E.inverse``: from the cold start z_0 = u until the iterate stops changing on small maps (``check(warm=False)``); on
the 1x300 row, 64x64 and the shared-memory limits warm-started from the kernel's z until it moves by at most
``SETTLE`` (``check(warm=True)``).  Both must settle within n_z*H*W + 1 iterations."""
import numpy as np
import pytest
import torch

from iaf_b200 import IAFOperator
from oracle import iaf_oracle as O
from tests import test_made_sample_envelope as E

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-4
VARIANTS = ("tf", "theano", "theano_flipmask")
NLS = ("none", "elu", "softplus", "relu", "tanh", "leakyrelu")
# The warm start stops once no element moves by more than 1e-13 of the sample's scale: about 500 ulp of fp64, nine
# orders below TOL, and reached within a few tens of iterations where exact settling takes hundreds (E.inverse).
SETTLE = 1e-13


def _np(t):
    return t.detach().double().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t, dtype=np.float64)


def per_sample_err(a, ref):
    a, ref = _np(a), _np(ref)
    assert np.isfinite(a).all()
    d = np.abs(a - ref).reshape(a.shape[0], -1).max(axis=1)
    r = np.maximum(np.abs(ref).reshape(a.shape[0], -1).max(axis=1), 1.0)
    return float((d / r).max())


def within(err, tol=TOL):
    assert err < tol, err


class Case(object):
    def __init__(self, variant, n_z, hidden, H, W, nl="elu", seed=1):
        self.variant, self.n_z, self.hidden, self.H, self.W, self.nl = variant, n_z, list(hidden), H, W, nl
        self.base = "tf" if variant == "tf" else "theano"
        self.keys = "Vgb" if variant == "tf" else "wsb"
        self.params(seed)

    def params(self, seed):
        self.hid, self.hd = O.make_params(self.base, self.n_z, self.hidden, [self.n_z, self.n_z], seed=seed)
        return [tuple(torch.from_numpy(l[k]).to(DEV) for k in self.keys) for l in self.hid + self.hd]

    def op(self, path="auto", seed=None):
        layers = self.params(seed) if seed is not None else self.params(1)
        return IAFOperator(self.base, self.n_z, self.hidden, [self.n_z, self.n_z], nl=self.nl, path=path,
                           flipmask=self.variant == "theano_flipmask").set_weights(layers)

    def inputs(self, B, seed=0):
        u, ctx = O.make_inputs(B, self.n_z, self.hidden[0] if self.hidden else 1, self.H, self.W, seed=seed)
        return torch.from_numpy(u).to(DEV), (torch.from_numpy(ctx).to(DEV) if self.hidden else None)


def inverse1(op, u, ctx, **kw):
    """One step_inverse, asserting it is one launch (the plan and the pack happen before, in path_used)."""
    op.path_used(u.shape[2], u.shape[3], DEV)
    n0 = op.launch_count()
    with torch.no_grad():
        out = op.step_inverse(u, ctx, **kw)
    assert op.launch_count() == n0 + 1
    return out


def check(k, B=2, path="auto", warm=False, op=None, logdet_scale=False):
    """The inverse against fp64 (cold start, or warm from the kernel's z), and the round trip.  Returns the outputs."""
    op = op if op is not None else k.op(path)
    u, ctx = k.inputs(B)
    z, ls, ld = inverse1(op, u, ctx)
    un, cn = u.cpu().numpy(), None if ctx is None else ctx.cpu().numpy()
    if warm:
        zr, ar, ldr, iters = E.inverse(k.variant, un, cn, k.hid, k.hd, k.nl, start=z.cpu().numpy(), settle=SETTLE)
    else:
        zr, ar, ldr, iters = E.inverse(k.variant, un, cn, k.hid, k.hd, k.nl)
    assert iters <= k.n_z * k.H * k.W + 1
    within(per_sample_err(z, zr))
    within(per_sample_err(ls, ar))
    if logdet_scale:
        # logdet sums n_z*H*W terms in fp32: its error scales with sum |arw_logsd|, not with |logdet|
        within(float((np.abs(_np(ld) - ldr) / np.abs(ar).sum(axis=(1, 2, 3))).max()))
    else:
        within(per_sample_err(ld[:, None], ldr[:, None]))
    with torch.no_grad():
        zs = op.step(z, ctx)[0]
    within(per_sample_err(zs, u))
    return z, ls, ld


# ---------------------------------------------------------------------------------------------------------------------
# stack shapes (cold start; maps of 3x5)
# ---------------------------------------------------------------------------------------------------------------------
STACKS = [
    (1, [2]), (3, [6]), (5, [10]),   # head_pad 4, 4, 8: padded head columns; widths not multiples of 8
    (6, [12, 3]),                    # steps down to 3 units
    (7, []),                         # no hidden layer, head_pad 8
    (16, [8, 4, 4]),                 # hidden narrower than n_z over three stages
    (8, [16, 32, 16, 8]),            # four hidden layers
    (16, [32, 32, 32]),              # three
    (80, [160]), (128, [128]),       # heads of 160 and 256 columns: two passes of the 128 threads
    (16, []), (48, []),              # depth 0 on a tensor-core plan
]


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("n_z,hidden", STACKS)
def test_stack_shapes(variant, n_z, hidden):
    check(Case(variant, n_z, hidden, 3, 5))


def test_stack_that_steps_up_again():
    """[8, 4, 8] at n_z 16: triangular only in the flipped order (E.final_steps); unflipped the plan has no inverse."""
    check(Case("theano_flipmask", 16, [8, 4, 8], 3, 5))
    for v in ("tf", "theano"):
        k = Case(v, 16, [8, 4, 8], 3, 5)
        assert not E.final_steps(v, 16, [8, 4, 8])[1]
        with torch.no_grad(), pytest.raises(NotImplementedError):
            k.op().step_inverse(*k.inputs(2))


# ---------------------------------------------------------------------------------------------------------------------
# nonlinearities (cold start)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("nl", NLS)
@pytest.mark.parametrize("n_z,hidden", [(8, [16, 16]), (4, [8])])
def test_every_nonlinearity(variant, nl, n_z, hidden):
    check(Case(variant, n_z, hidden, 3, 4, nl=nl))


# ---------------------------------------------------------------------------------------------------------------------
# maps
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("H,W", [(1, 1), (1, 9), (9, 1), (2, 2), (3, 17), (17, 3)])
def test_maps(variant, H, W):
    check(Case(variant, 4, [8], H, W))          # cold start


@pytest.mark.parametrize("variant", VARIANTS)
def test_a_wide_row(variant):
    check(Case(variant, 4, [8], 1, 300), warm=True)


@pytest.mark.parametrize("variant", VARIANTS)
def test_64x64_on_c2a_stack(variant):
    check(Case(variant, 32, [64], 64, 64), warm=True, logdet_scale=True)


# ---------------------------------------------------------------------------------------------------------------------
# the shared-memory limit
# ---------------------------------------------------------------------------------------------------------------------
# Only a tensor-core plan exists at the inverse's W_max + 1 (see the SIMT-only case below), so the limit is reached on
# wide tensor-core stacks; c2b's ([160, 160], W_max 79) is in tests/test_gpu_made_sample.py.
@pytest.mark.parametrize("variant,n_z,hidden", [("tf", 16, [64] * 4), ("theano_flipmask", 32, [128] * 4)])
def test_the_widest_map_that_fits_and_the_first_that_does_not(variant, n_z, hidden):
    w_max = E.inv_w_max(n_z, hidden)
    assert E.inv_smem(n_z, hidden, w_max) <= E.SMEM_LIMIT < E.inv_smem(n_z, hidden, w_max + 1)
    assert w_max == {16: 103, 32: 50}[n_z]     # the formula's value, as derived by hand from inv_tables
    check(Case(variant, n_z, hidden, 2, w_max), warm=True)
    k = Case(variant, n_z, hidden, 2, w_max + 1)
    op = k.op()
    assert op.path_used(2, w_max + 1, DEV) == "tc"
    with torch.no_grad(), pytest.raises(NotImplementedError):
        op.step_inverse(*k.inputs(2))


def test_a_simt_only_plan_is_refused_before_its_inverse_could_be():
    """n_z 8 has no tensor-core plan: the SIMT band (at least 2 + n_hidden rows) outgrows shared memory at a narrower
    map than the inverse's two-row window.  At the SIMT plan's widest map the inverse runs (warm start); at the
    inverse's W_max + 1 there is no plan at all."""
    n_z, hidden = 8, [16, 32, 16, 8]
    w_inv = E.inv_w_max(n_z, hidden)
    w_simt = max(W for W in range(1, w_inv + 2) if E.simt_smem(n_z, hidden, W) <= E.SMEM_LIMIT)
    assert w_simt < w_inv
    k = Case("theano", n_z, hidden, 2, w_simt)
    op = k.op()
    assert op.path_used(2, w_simt, DEV) == "simt"
    check(k, op=op, warm=True)
    for W in (w_simt + 1, w_inv + 1):
        with pytest.raises(NotImplementedError):
            Case("theano", n_z, hidden, 2, W).op().path_used(2, W, DEV)


# ---------------------------------------------------------------------------------------------------------------------
# tensor-core plans
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant,n_z,hidden", [("tf", 16, []), ("theano", 32, [64]), ("theano", 48, [48, 96]),
                                                ("theano_flipmask", 32, [32, 64])])
def test_tensor_core_plans_run_the_same_inverse(variant, n_z, hidden):
    k = Case(variant, n_z, hidden, 8, 8)
    tc, simt = k.op("auto"), k.op("simt")
    assert tc.path_used(8, 8, DEV) == "tc" and simt.path_used(8, 8, DEV) == "simt"
    a = check(k, B=3, op=tc)
    b = inverse1(simt, *k.inputs(3))
    # the same SIMT pack and the same kernel: bit-identical
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    # the sample's density against the tensor-core density entry, an independent kernel
    u, ctx = k.inputs(3)
    with torch.no_grad():
        z, bc, lp = tc.ar_sample(u, ctx)
        _, bc_ref, lp_ref = tc.ar_logp(z, ctx)
    assert tc.path_used(8, 8, DEV, "ar_logp") == "tc"
    assert torch.equal(z, a[0])
    within(per_sample_err(bc, bc_ref))
    within(per_sample_err(lp[:, None], lp_ref[:, None]))


# ---------------------------------------------------------------------------------------------------------------------
# weights
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("how", ("set_weights", "invalidate"))
def test_new_weights_are_packed_before_the_next_inverse(how):
    k = Case("theano", 8, [16, 16], 4, 5)
    layers = k.params(1)
    op = IAFOperator("theano", 8, [16, 16], [8, 8]).set_weights(layers)
    u, ctx = k.inputs(2)
    old = inverse1(op, u, ctx)
    new = k.params(2)
    if how == "set_weights":
        op.set_weights(new)
    else:
        for l, n in zip(layers, new):
            for t, s in zip(l, n):
                t.data.copy_(s)
        op.invalidate()
    fresh = inverse1(k.op(seed=2), u, ctx)
    got = inverse1(op, u, ctx)
    assert not torch.equal(got[0], old[0])
    assert all(torch.equal(x, y) for x, y in zip(got, fresh))


def test_two_operators_alternate_on_one_map():
    ka, kb = Case("theano", 4, [8], 4, 5), Case("tf", 8, [16, 32, 16, 8], 4, 5)
    oa, ob = ka.op(), kb.op()
    ra, rb = check(ka, op=oa), check(kb, op=ob)
    for _ in range(2):
        assert all(torch.equal(x, y) for x, y in zip(inverse1(oa, *ka.inputs(2)), ra))
        assert all(torch.equal(x, y) for x, y in zip(inverse1(ob, *kb.inputs(2)), rb))


# ---------------------------------------------------------------------------------------------------------------------
# batches
# ---------------------------------------------------------------------------------------------------------------------
def test_one_sample():
    check(Case("theano_flipmask", 8, [16], 5, 6), B=1)


def test_more_samples_than_the_first_wave():
    k = Case("theano", 4, [8], 2, 2)
    op = k.op()
    B = 3 * torch.cuda.get_device_properties(DEV).multi_processor_count + 1
    u, ctx = k.inputs(B)
    full = inverse1(op, u, ctx)
    with torch.no_grad():
        for b in range(B):
            one = op.step_inverse(u[b:b + 1].contiguous(), ctx[b:b + 1].contiguous())
            assert all(torch.equal(x, y[b:b + 1]) for x, y in zip(one, full)), b


def test_non_finite_samples_leave_the_others_alone():
    k = Case("tf", 8, [16], 4, 5)
    op = k.op()
    u, ctx = k.inputs(5)
    clean = inverse1(op, u, ctx)
    u2, c2 = u.clone(), ctx.clone()
    u2[1] = float("nan")
    u2[2, 3, 1, 2] = float("inf")
    c2[3] = float("nan")
    dirty = inverse1(op, u2, c2)
    for b in (0, 4):
        assert all(torch.equal(x[b], y[b]) for x, y in zip(dirty, clean))
    for b in (1, 2, 3):
        assert not torch.isfinite(dirty[0][b]).all()


def test_null_outputs():
    k = Case("theano_flipmask", 5, [10], 4, 5)
    op = k.op()
    u, ctx = k.inputs(2)
    full = inverse1(op, u, ctx)
    for want_logsd in (False, True):
        for want_logdet in (False, True):
            got = inverse1(op, u, ctx, want_logsd=want_logsd, want_logdet=want_logdet)
            assert torch.equal(got[0], full[0])
            for g, f, w in zip(got[1:], full[1:], (want_logsd, want_logdet)):
                assert (g is None) if not w else torch.equal(g, f)
