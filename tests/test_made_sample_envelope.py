"""The inverse of the IAF step (``iaf_inv_kernel``, iaf_inv.cu) over its own envelope on the CPU: the kernel under host
emulation (tests/emu/inverse.py) against the fp64 fixed point, and the host table (``inv_tables``, iaf_capi.cu) that
says which hidden units become final after which z channel.

The kernel's envelope: one CTA of 128 threads per sample, the heads interleaved in groups of four columns over
``head_pad = round_up(n_z, 4)``, per stage a two-row ring of its input in shared memory, and a table of "units final
after step k" per hidden stage.  The cases run it where that logic has edges:
* stacks with n_z not a multiple of 4 (padded head columns), heads wider than the CTA (n_z 80 and 128: 160 and 256
  columns), three and four hidden layers, widths that step down, and no hidden layer (tf included);
* all six nonlinearities, on a stack with two hidden layers and on one with one;
* maps one pixel wide (on both x borders at once) or one row high (every pixel on the bottom border);
* the tables themselves, restated in Python from the mask oracles (``final_steps``);
* the shared-memory limit of a stack the tensor cores do not take: the SIMT plan is refused at a narrower map than the
  inverse's window would be.
tests/test_gpu_made_sample_envelope.py runs the same matrix and more on the H100.

Every case: z, arw_logsd and logdet against fp64 (``inverse`` from the cold start z_0 = u: all maps here are small)
with ``|d_n|_inf / max(|ref_n|_inf, 1) < TOL`` per sample n, the round trip step(z) == u on the same plan, and exactly
one launch per inverse.  The emulation is slow (about 1 ms per barrier per sample), so B = 2 and the maps are small."""
import itertools

import numpy as np
import pytest

from iaf_b200 import _lib as L
from oracle import iaf_oracle as O
from tests import flipmask_oracle as FO
from tests import made_sample_oracle as MS
from tests.emu.harness import _check, _p
from tests.emu.inverse import EmuInvOperator

VARIANTS = ("tf", "theano", "theano_flipmask")
TOL = 1e-4
NLS = ("none", "elu", "softplus", "relu", "tanh", "leakyrelu")


# ---------------------------------------------------------------------------------------------------------------------
# fp64 references and the restated tables and layouts (tests/test_gpu_made_sample_envelope.py uses them too)
# ---------------------------------------------------------------------------------------------------------------------
def inverse(variant, u, ctx, hidden, hd, nl="elu", start=None, settle=0.0):
    """fp64: (z, arw_logsd, logdet, iterations) with step(z) = u: ``MS.inverse`` with a warm start and a settle
    threshold.

    ``start``: the warm start, e.g. the kernel's fp32 z, instead of ``z_0 = u``.  The map is triangular in the mask's
    order, so its fixed point is unique and the same n_z*H*W + 1 bound holds from any start: started from a wrong
    kernel output, the iteration either settles on the true inverse, which the comparison with that output then
    rejects, or does not settle in time.

    ``settle``: stop once no element moves by more than ``settle * max(|z|_inf, 1)`` instead of not at all.  On large
    maps the iterate reaches fp64 accuracy within a few tens of iterations from either start, and then keeps flipping
    last bits (each iteration's rounding feeds the next) until the triangular front has crossed the whole map: at 64x64
    with n_z 32, about 220 iterations either way.  A step of at most ``settle`` leaves z within a small multiple of it of
    the fixed point (the step's Jacobian is strictly triangular with entries scaled by 0.1), far below the fp32 kernel's
    error."""
    f64 = lambda ls: O.cast_params(ls, np.float64)
    hidden, hd = f64(hidden), f64(hd)
    u = np.asarray(u, np.float64)
    ctx = None if ctx is None else np.asarray(ctx, np.float64)
    bound = u[0].size + 1
    z = u.copy() if start is None else np.array(start, dtype=np.float64)
    for it in range(1, bound + 1):
        m, s = MS.heads(variant, z, ctx, hidden, hd, nl)
        zn = 0.1 * m + np.exp(0.1 * s) * u
        if np.abs(zn - z).max() <= settle * max(np.abs(z).max(), 1.0):
            a = 0.1 * s
            return z, a, -a.sum(axis=(1, 2, 3)), it
        z = zn
    raise AssertionError("the fixed point did not settle within n_z*H*W + 1 iterations: not the mask's order")


def centre_mask(variant, n_in, n_out, zerodiagonal):
    """[n_in, n_out] bool: the live centre taps of one masked conv, read off the forward oracles' own masks."""
    if variant == "tf":
        return O.get_conv_ar_mask(3, 3, n_in, n_out, zerodiagonal)[1, 1] != 0
    m = FO.conv_ar_mask(n_in, n_out, zerodiagonal, variant == "theano_flipmask")
    return m[:, :n_in, 1, 1].T != 0


def final_steps(variant, n_z, hidden):
    """When each hidden unit becomes final in a pixel's chain of z-channel steps: (per hidden layer an int array, the
    step after which the unit's last live centre input is final, -1 when it has none; whether every head channel's
    live centre inputs are final before that channel's own step, i.e. whether the step is triangular in the mask's
    order).  z channel c is solved at step c, or n_z - 1 - c with flipmask."""
    pos = np.arange(n_z)[::-1] if variant == "theano_flipmask" else np.arange(n_z)
    prev, steps, sizes = pos, [], [n_z] + list(hidden)
    for j, h in enumerate(hidden):
        m = centre_mask(variant, sizes[j], h, False)
        prev = np.array([prev[m[:, u]].max() if m[:, u].any() else -1 for u in range(h)])
        steps.append(prev)
    m = centre_mask(variant, sizes[-1], n_z, True)
    triangular = all(not m[:, c].any() or prev[m[:, c]].max() < pos[c] for c in range(n_z))
    return steps, triangular


# The shared-memory layouts of iaf_capi.cu, restated (limit: 225 KiB of opt-in shared memory per CTA).
SMEM_LIMIT = 225 * 1024


def _r(x, m):
    return (x + m - 1) // m * m


def inv_smem(n_z, hidden, W):
    """Bytes of the inverse's window (inv_tables): per stage two rows of its input over W + 2 columns, per stage its
    accumulators (hidden widths padded to 8, the interleaved head pair to 2 * round_up(n_z, 4)), the per-channel sums."""
    cin = [n_z] + list(hidden)
    cout_pad = [_r(h, 8) for h in hidden] + [2 * _r(n_z, 4)]
    return 4 * (sum(cin) * 2 * (W + 2) + sum(cout_pad) + n_z)


def inv_w_max(n_z, hidden):
    """The widest map whose window fits."""
    fixed = inv_smem(n_z, hidden, -2)  # the accumulators and sums
    return (SMEM_LIMIT - fixed) // (8 * (n_z + sum(hidden))) - 2


def simt_smem(n_z, hidden, W, band_rows=1):
    """Bytes of the SIMT step's band (simt_geometry) at ``band_rows`` rows; at one row it is the least the SIMT plan can
    ask for, which iaf_plan_create reaches on maps of one row and on every map whose height is a power of two."""
    nseg = (W + 7) // 8
    P, rows = 8 * nseg + 2, band_rows + len(hidden) + 1
    ca = max([h for j, h in enumerate(hidden) if j % 2 == 0], default=0)
    cb = max([h for j, h in enumerate(hidden) if j % 2 == 1], default=0)
    tile = band_rows * nseg * (2 * _r(n_z, 4) // 8) * 4
    return 4 * (_r(n_z * rows * P, 4) + _r(ca * rows * P, 4) + _r(cb * rows * P, 4) + tile)


def per_sample_err(a, ref):
    a, ref = np.asarray(a, np.float64), np.asarray(ref, np.float64)
    assert np.isfinite(a).all()
    d = np.abs(a - ref).reshape(a.shape[0], -1).max(axis=1)
    r = np.maximum(np.abs(ref).reshape(a.shape[0], -1).max(axis=1), 1.0)
    return float((d / r).max())


def _op(variant, n_z, hidden, H, W, nl="elu", seed=1):
    base = "tf" if variant == "tf" else "theano"
    hid, hd = O.make_params(base, n_z, hidden, [n_z, n_z], seed=seed)
    keys = "Vgb" if variant == "tf" else "wsb"
    op = EmuInvOperator(variant, n_z, hidden, [n_z, n_z], H, W, nl=nl).set_weights(
        [tuple(l[k] for k in keys) for l in hid + hd])
    return op, hid, hd


def _inverse(op, u, ctx):
    z, ls, ld = np.full_like(u, np.nan), np.full_like(u, np.nan), np.full((u.shape[0],), np.nan, np.float32)
    n0 = op.lib.iaf_plan_launch_count(op.plan)
    _check(op.lib.iaf_step_inverse(op.plan, _p(u), _p(ctx), _p(z), _p(ls), _p(ld), u.shape[0], None))
    assert op.lib.iaf_plan_launch_count(op.plan) == n0 + 1
    return z, ls, ld


def check(variant, n_z, hidden, H, W, nl="elu", B=2):
    """The emulated inverse against the cold-start fp64 fixed point, and the round trip through the step."""
    op, hid, hd = _op(variant, n_z, hidden, H, W, nl)
    u, ctx = O.make_inputs(B, n_z, hidden[0] if hidden else 1, H, W, seed=0)
    ctx = ctx if hidden else None
    z, ls, ld = _inverse(op, u, ctx)
    zr, ar, ldr, iters = inverse(variant, u, ctx, hid, hd, nl)
    assert iters <= n_z * H * W + 1
    assert per_sample_err(z, zr) < TOL, per_sample_err(z, zr)
    assert per_sample_err(ls, ar) < TOL, per_sample_err(ls, ar)
    assert per_sample_err(ld[:, None], ldr[:, None]) < TOL, per_sample_err(ld[:, None], ldr[:, None])
    zs = op.step(z, ctx)[0]
    assert per_sample_err(zs, u) < TOL, per_sample_err(zs, u)


# ---------------------------------------------------------------------------------------------------------------------
# stack shapes
# ---------------------------------------------------------------------------------------------------------------------
# n_z, hidden, H, W.  Maps of 2x2 or 2x3 (1x2 for the widest heads) keep the emulation's barrier count small; the maps
# cases below cover the geometry.
STACKS = [
    (1, [2], 2, 3),                 # head_pad 4: three padded columns per head
    (3, [6], 2, 3),
    (5, [10], 2, 3),                # head_pad 8, hidden 10: neither a multiple of 8
    (6, [12, 3], 2, 3),             # steps down to 3 units
    (7, [], 2, 3),                  # no hidden layer, head_pad 8
    (16, [8, 4, 4], 2, 2),          # hidden narrower than n_z over three stages
    (8, [16, 32, 16, 8], 2, 2),     # four hidden layers, each stage's table different from stage 1's
    (16, [32, 32, 32], 2, 2),       # three hidden layers
    (80, [160], 1, 2),              # heads of 160 columns: two passes of the 128 threads
    (128, [128], 1, 2),             # heads of 256 columns
    (16, [], 2, 2),
    (48, [], 2, 2),
]
# Unflipped, [8, 4, 8] is not triangular in the mask's order: head channel 2 sees, through the units that step up
# again, z channel 3 (final_steps).  The step is then no autoregressive flow, and the plan has no inverse; flipped,
# the reversed order keeps it triangular.
NOT_TRIANGULAR = (16, [8, 4, 8], 2, 2)


def _stack_cases():
    for v, s in itertools.product(VARIANTS, STACKS + [NOT_TRIANGULAR]):
        if s == NOT_TRIANGULAR and v != "theano_flipmask":
            continue
        yield (v,) + s


@pytest.mark.parametrize("variant,n_z,hidden,H,W", list(_stack_cases()))
def test_stack_shapes_match_the_fp64_fixed_point(variant, n_z, hidden, H, W):
    check(variant, n_z, hidden, H, W)


@pytest.mark.parametrize("variant", ("tf", "theano"))
def test_a_stack_that_is_not_triangular_has_no_inverse(variant):
    n_z, hidden, H, W = NOT_TRIANGULAR
    assert not final_steps(variant, n_z, hidden)[1]
    op, hid, hd = _op(variant, n_z, hidden, H, W)
    u, ctx = O.make_inputs(2, n_z, hidden[0], H, W, seed=0)
    z = np.empty_like(u)
    assert op.lib.iaf_step_inverse(op.plan, _p(u), _p(ctx), _p(z), None, None, 2, None) == L.ERR_UNSUPPORTED


# ---------------------------------------------------------------------------------------------------------------------
# nonlinearities
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("nl", NLS)
@pytest.mark.parametrize("n_z,hidden,H,W", [(8, [16, 16], 2, 2), (4, [8], 2, 3)])
def test_every_nonlinearity(variant, nl, n_z, hidden, H, W):
    check(variant, n_z, hidden, H, W, nl)


# ---------------------------------------------------------------------------------------------------------------------
# maps
# ---------------------------------------------------------------------------------------------------------------------
# 1x1: one pixel on all four borders; 1xW: every pixel on the bottom border; Hx1: every pixel on both x borders
MAPS = [(1, 1), (1, 9), (9, 1), (2, 2), (3, 17), (17, 3)]


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("H,W", MAPS)
def test_maps(variant, H, W):
    check(variant, 4, [8], H, W)


# ---------------------------------------------------------------------------------------------------------------------
# the tables
# ---------------------------------------------------------------------------------------------------------------------
def test_every_stack_of_the_matrix_is_triangular_and_has_groups_at_every_stage():
    """The Python restatement of inv_tables on the stacks above: each is triangular (so the plan has an inverse), every
    hidden stage becomes final over more than one step, and the four- and three-hidden-layer stacks give stages 2 and 3
    tables of their own (a kernel that read stage 1's table there would compute wrong units)."""
    for v, (n_z, hidden, _, _) in itertools.product(VARIANTS, STACKS):
        steps, tri = final_steps(v, n_z, hidden)
        assert tri, (v, n_z, hidden)
        assert len(steps) == len(hidden)
        for j, s in enumerate(steps):
            assert len(s) == hidden[j] and s.max() <= n_z - 1
            if n_z > 1:
                assert len(set(s.tolist())) > 1, (v, n_z, hidden, j)
    for v in VARIANTS:
        steps, _ = final_steps(v, 8, [16, 32, 16, 8])
        for j in (2, 3):
            assert not np.array_equal(steps[j], steps[1])
        # [32, 32, 32] has the same table at every stage past the first; [8, 4, 4] at stages 1 and 2
        steps, _ = final_steps(v, 16, [8, 4, 4])
        assert not np.array_equal(steps[0], steps[1])


def _legal_stacks(max_nz=16, depth=2):
    """Every stack with n_z <= max_nz, up to ``depth`` hidden layers of widths n_z * 2^k (k in -3..2, integral), in
    which each adjacent pair of widths divides (iaf_plan_create)."""
    for n_z in range(1, max_nz + 1):
        widths = sorted({int(n_z * 2.0 ** k) for k in range(-3, 3) if n_z * 2.0 ** k >= 1 and
                         float(n_z * 2.0 ** k).is_integer()})
        for d in range(depth + 1):
            for hidden in itertools.product(widths, repeat=d):
                sizes = [n_z] + list(hidden) + [n_z]
                if all(a % b == 0 or b % a == 0 for a, b in zip(sizes, sizes[1:])):
                    yield n_z, list(hidden)


def test_step_minus_one_groups_occur_only_with_flipmask():
    """A hidden unit with no live centre input is final before the first z channel (the table's "step -1" group).
    Unflipped, no legal stack has one: input channel 0 reaches every hidden unit's centre (iaf_tap_rule: c <= i, or
    c < (o + 1) k).  Flipped, channel 0 never sees the centre, so the first hidden layer's last units (and, through
    them, later layers' units) see no z channel: the kernel runs that group at every pixel."""
    seen_flip = False
    for n_z, hidden in _legal_stacks():
        for v in VARIANTS:
            steps, _ = final_steps(v, n_z, hidden)
            minus = any((s == -1).any() for s in steps)
            if v == "theano_flipmask":
                seen_flip |= minus
            else:
                assert not minus, (v, n_z, hidden)
    assert seen_flip
    # and some stack of the matrix runs such a group
    assert any((s == -1).any() for s in final_steps("theano_flipmask", 5, [10])[0])


# ---------------------------------------------------------------------------------------------------------------------
# the shared-memory limit on a stack the tensor cores do not take
# ---------------------------------------------------------------------------------------------------------------------
SIMT_ONLY = (8, [16, 32, 16, 8])


def test_the_simt_plan_is_refused_before_the_inverse_window_could_overflow():
    """The SIMT step keeps at least 2 + n_hidden rows of z and of two hidden buffers; the inverse keeps two rows per
    stage.  So where no tensor-core plan exists, plan creation refuses a map before the inverse's window stops fitting,
    and the inverse never refuses on its own there.  The restated layouts (simt_smem, inv_smem) are pinned to
    iaf_plan_create at the SIMT plan's widest map of H = 2 (whose band can be one row)."""
    n_z, hidden = SIMT_ONLY
    w_inv = inv_w_max(n_z, hidden)
    assert inv_smem(n_z, hidden, w_inv) <= SMEM_LIMIT < inv_smem(n_z, hidden, w_inv + 1)
    w_simt = max(W for W in range(1, w_inv + 2) if simt_smem(n_z, hidden, W) <= SMEM_LIMIT)
    assert w_simt < w_inv
    for v in VARIANTS:
        _op(v, n_z, hidden, 2, w_simt)
        for W in (w_simt + 1, w_inv + 1):
            with pytest.raises(RuntimeError, match="status %d" % L.ERR_UNSUPPORTED):
                _op(v, n_z, hidden, 2, W)
    # the same ordering for every stack of the matrix and every legal small stack (on a one-row band)
    for n_z, hidden in [s[:2] for s in STACKS] + list(_legal_stacks(8, 2)):
        assert simt_smem(n_z, hidden, inv_w_max(n_z, hidden) + 1) > SMEM_LIMIT, (n_z, hidden)
