"""The inverse of the IAF step (``iaf_step_inverse``), sampling the autoregressive (MADE) prior with it, and the Theano
model's decoder (``cvae_layer.down_p``, ``cvae1.f_decoder``: models.py:330-359, 499-521), on the CPU.

* the kernel under host emulation against the fp64 fixed-point inverse (tests/made_sample_oracle.py), for the three
  variants: z, arw_logsd and logdet; the round trips with the step; every NULL-output combination; batch independence;
  the argument checks;
* ``IAFOperator.step_inverse`` / ``ar_sample`` over the emulated ABI: the density identity with ``ar_logp`` at the
  sample, and the refusal under autograd;
* ``layer_down_p`` with prior='diag' against tests/golden/cvae_layer_down_p.npz (the reference's own down_p executed,
  tests/golden/make_golden_down_p.py), and ``decode`` with prior='made' through the emulated ABI against the fp64 oracle.
"""
import contextlib
import ctypes as C
import itertools
import math
import os

import numpy as np
import pytest
import torch

from iaf_b200 import elbo_theano as ET
from oracle import iaf_oracle as O
from tests import made_sample_oracle as MS
from tests.emu.harness import EmuOperator, _check, _p
from tests.emu.inverse import EmuInvOperator

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cvae_layer_down_p.npz")
POSTERIORS = ("down_iaf2_nl", "up_iaf2_nl", "down_iaf2_nl2")
VARIANTS = ("tf", "theano", "theano_flipmask")
SHAPES = [
    # n_z, hidden, H, W, B, nl
    (4, [8], 4, 4, 2, "elu"),
    (8, [16, 16], 5, 7, 2, "softplus"),   # two hidden layers, non-square
    (4, [], 3, 6, 2, "elu"),              # no hidden layer (Theano only)
    (4, [8], 12, 9, 1, "relu"),           # W not a multiple of 8
    (8, [4], 4, 5, 2, "tanh"),            # cout < cin
]
TOL = 1e-5
# The round trips compose the inverse with the step, two fp32 evaluations of the same stack; each agrees with fp64 to
# a few 1e-7 relative (the oracle comparison above asks 1e-5), so their composition is held to the same 1e-5.
RT_TOL = 1e-5
LOG2PI = math.log(2 * math.pi)


def _rel(a, b):
    a = a.detach().numpy() if hasattr(a, "detach") else np.asarray(a)
    b = b.detach().numpy() if hasattr(b, "detach") else np.asarray(b)
    assert np.isfinite(a).all()
    return float(np.abs(a.astype(np.float64) - b).max() / max(np.abs(b).max(), 1e-30))


def _cases():
    for v, s in itertools.product(VARIANTS, SHAPES):
        if v == "tf" and not s[1]:
            continue
        yield (v,) + s


def _emu(variant, n_z, hidden, H, W, B, nl, seed=1):
    hid, hd = O.make_params("tf" if variant == "tf" else "theano", n_z, hidden, [n_z, n_z], seed=seed)
    keys = "Vgb" if variant == "tf" else "wsb"
    u, ctx = O.make_inputs(B, n_z, hidden[0] if hidden else 1, H, W, seed=0)
    op = EmuInvOperator(variant, n_z, hidden, [n_z, n_z], H, W, nl=nl).set_weights(
        [tuple(l[k] for k in keys) for l in hid + hd])
    return op, hid, hd, u, (ctx if hidden else None)


def emu_inverse(op, u, ctx, want=(True, True)):
    B = u.shape[0]
    z = np.full_like(u, np.nan)
    ls = np.full_like(u, np.nan) if want[0] else None
    ld = np.full((B,), np.nan, np.float32) if want[1] else None
    _check(op.lib.iaf_step_inverse(op.plan, _p(u), _p(ctx), _p(z), _p(ls), _p(ld), B, None))
    return z, ls, ld


@pytest.mark.parametrize("variant,n_z,hidden,H,W,B,nl", list(_cases()))
def test_emulated_inverse_matches_the_fp64_fixed_point(variant, n_z, hidden, H, W, B, nl):
    op, hid, hd, u, ctx = _emu(variant, n_z, hidden, H, W, B, nl)
    zr, ar, ldr, iters = MS.inverse(variant, u, ctx, hid, hd, nl)
    assert iters <= n_z * H * W + 1
    z, ls, ld = emu_inverse(op, u, ctx)
    assert _rel(z, zr) < TOL and _rel(ls, ar) < TOL and _rel(ld, ldr) < TOL
    # step(inverse(u)) == u, and the inverse's arw_logsd / logdet are the step's own at z
    zs, lss, lds = op.step(z, ctx)
    assert _rel(zs, u) < RT_TOL and _rel(lss, ls) < RT_TOL and _rel(lds, ld) < RT_TOL
    # inverse(step(z)) == z, from an independent z
    z2 = np.random.RandomState(3).randn(*u.shape).astype(np.float32)
    u2, _, _ = op.step(z2, ctx)
    assert _rel(emu_inverse(op, u2, ctx)[0], z2) < RT_TOL
    # every NULL-output combination: bit-identical to the full call
    for want in itertools.product((False, True), repeat=2):
        got = emu_inverse(op, u, ctx, want)
        assert np.array_equal(got[0], z)
        for g, full, w in zip(got[1:], (ls, ld), want):
            assert (g is None) if not w else np.array_equal(g, full)


@pytest.mark.parametrize("variant", VARIANTS)
def test_emulated_inverse_is_batch_independent(variant):
    op, hid, hd, u, ctx = _emu(variant, 8, [16], 4, 5, 3, "elu")
    full = emu_inverse(op, u, ctx)
    for b in range(u.shape[0]):
        one = emu_inverse(op, np.ascontiguousarray(u[b:b + 1]), None if ctx is None else np.ascontiguousarray(ctx[b:b + 1]))
        assert np.array_equal(one[0][0], full[0][b]) and np.array_equal(one[1][0], full[1][b])
        assert np.array_equal(one[2][0], full[2][b])


def test_emulated_inverse_checks_its_arguments():
    from iaf_b200 import _lib as L
    op, hid, hd, u, ctx = _emu("theano", 4, [8], 4, 4, 2, "elu")
    B = u.shape[0]
    z = np.empty_like(u)
    assert op.lib.iaf_step_inverse(op.plan, _p(u), _p(None), _p(z), None, None, B, None) == L.ERR_BAD_ARG  # context
    assert op.lib.iaf_step_inverse(op.plan, _p(u), _p(ctx), _p(None), None, None, B, None) == L.ERR_BAD_ARG  # z_out
    one = EmuInvOperator("theano", 4, [8], [4], 4, 4)
    p1, h1 = O.make_params("theano", 4, [8], [4], seed=1)
    one.set_weights([tuple(l[k] for k in "wsb") for l in p1 + h1])
    assert one.lib.iaf_step_inverse(one.plan, _p(u), _p(ctx), _p(z), None, None, B, None) == L.ERR_BAD_SHAPE  # one head
    fresh = EmuInvOperator("theano", 4, [8], [4, 4], 4, 4)
    assert fresh.lib.iaf_step_inverse(fresh.plan, _p(u), _p(ctx), _p(z), None, None, B, None) == L.ERR_NOT_PACKED
    # the C ABI built without iaf_inv.cu (the emulated library of tests/emu/build_emu.py) refuses, it does not fall back
    plain = EmuOperator("theano", 4, [8], [4, 4], 4, 4).set_weights([tuple(l[k] for k in "wsb") for l in hid + hd])
    assert plain.lib.iaf_step_inverse(plain.plan, _p(u), _p(ctx), _p(z), None, None, B, None) == L.ERR_UNSUPPORTED
    # the ABI facts that stay as they are
    assert op.lib.iaf_plan_path_for_entry(op.plan, 4) == L.ERR_BAD_ARG
    assert op.lib.iaf_version() == 201


# ---------------------------------------------------------------------------------------------------------------------
# the Python layer over the emulated ABI
# ---------------------------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def _emulated_abi(monkeypatch):
    """Point the ctypes binding at the host-emulated library (test only; the product refuses CPU tensors)."""
    from iaf_b200 import _lib as L
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


def test_python_step_inverse_and_ar_sample_over_the_emulated_abi(monkeypatch):
    from iaf_b200 import ops
    with _emulated_abi(monkeypatch):
        variant, n_z, hidden, H, W, B = "theano", 4, [8], 4, 5, 2
        hid, hd = O.make_params(variant, n_z, hidden, [n_z, n_z], seed=1)
        eps, ctx = O.make_inputs(B, n_z, hidden[0], H, W, seed=0)
        dev = [tuple(torch.from_numpy(l[k].copy()) for k in "wsb") for l in hid + hd]
        op = ops.IAFOperator(variant, n_z, hidden, [n_z, n_z], nl="elu", path="simt").set_weights(dev)
        e, c = torch.from_numpy(eps), torch.from_numpy(ctx)
        z, ls, ld = op.step_inverse(e, c)
        zr, ar, ldr, _ = MS.inverse(variant, eps, ctx, hid, hd, "elu")
        assert _rel(z, zr) < TOL and _rel(ls, ar) < TOL and _rel(ld, ldr) < TOL
        z1, none1, none2 = op.step_inverse(e, c, want_logsd=False, want_logdet=False)
        assert torch.equal(z1, z) and none1 is None and none2 is None
        zs, bc, lp = op.ar_sample(e, c)
        assert torch.equal(zs, z)
        # the prior's density at its own sample: what ar_logp computes there
        _, bc_ref, lp_ref = op.ar_logp(zs, c)
        assert _rel(bc, bc_ref.numpy().astype(np.float64)) < TOL and _rel(lp, lp_ref.numpy().astype(np.float64)) < TOL
        ident = -0.5 * LOG2PI * n_z * H * W + ldr - 0.5 * (eps.astype(np.float64) ** 2).sum(axis=(1, 2, 3))
        assert _rel(lp, ident) < TOL
        # not differentiable: refused under autograd, never detached silently
        with pytest.raises(NotImplementedError, match="no_grad"):
            op.ar_sample(e.clone().requires_grad_(True), c)
        with pytest.raises(NotImplementedError, match="no_grad"):
            op.step_inverse(e, c.clone().requires_grad_(True))
        grad_op = ops.IAFOperator(variant, n_z, hidden, [n_z, n_z], nl="elu", path="simt").set_weights(
            [tuple(t.clone().requires_grad_(True) for t in l) for l in dev])
        with pytest.raises(NotImplementedError):
            grad_op.ar_sample(e, c)
        with torch.no_grad():
            assert torch.equal(grad_op.ar_sample(e, c)[0], z)


# ---------------------------------------------------------------------------------------------------------------------
# the decoder
# ---------------------------------------------------------------------------------------------------------------------
HPS = dict(n_z=4, n_h1=8, n_h2=8, depths=[2, 2], depth_ar=1, nl="elu", kl_min=0.0, image_size=16)
CASES = [(p, n) for p in POSTERIORS for n in ("0_1", "1_0")]


@pytest.mark.parametrize("posterior,name", CASES)
def test_layer_down_p_diag_matches_reference_models_py(posterior, name):
    g = np.load(GOLD)
    pre = "%s:%s/" % (posterior, name)
    T = lambda a: torch.from_numpy(np.asarray(a)).double()
    w = {k[len(pre) + 2:]: T(g[k]) for k in g.files if k.startswith(pre + "w/")}
    hps = dict(HPS, posterior=posterior, prior="diag")
    out = ET.layer_down_p(w, name, T(g[pre + "down_in"]), T(g[pre + "eps"]), None, hps, bool(g[pre + "downsample"]))
    np.testing.assert_allclose(out.numpy(), g[pre + "down_out"], rtol=1e-9, atol=1e-9)


class _Recording(object):
    """Wraps an iaf_layer and keeps every prior sample with its noise and context."""

    def __init__(self, inner):
        self.inner, self.samples = inner, {}

    def prior_sample(self, name, eps, context):
        z = self.inner.prior_sample(name, eps, context)
        self.samples[name] = (eps, context, z)
        return z


def _decoder_setup(hps, B, seed):
    w = {k: torch.from_numpy(np.asarray(v)) for k, v in ET.make_params(hps, seed=seed).items()}
    rng = np.random.RandomState(seed + 1)
    eps = {}
    for i in range(len(hps["depths"])):
        s = hps["image_size"] // 2 ** (i + 1)
        for j in range(hps["depths"][i]):
            eps[(i, j)] = torch.from_numpy(rng.randn(B, hps["n_z"], s, s).astype(np.float32))
    return w, eps


@pytest.mark.parametrize("posterior", POSTERIORS)
def test_made_decoder_over_the_emulated_abi_matches_the_fp64_oracle(posterior, monkeypatch):
    hps = dict(HPS, depths=[1, 1], image_size=8, posterior=posterior, prior="made")
    w, eps = _decoder_setup(hps, 2, 5)
    ref_layer = _Recording(MS.OracleIAFTheanoMadeSample(w, hps))
    ref = ET.decode(w, eps, ref_layer, hps)
    with _emulated_abi(monkeypatch):
        cuda_layer = _Recording(ET.CudaIAF(w, hps, path="simt"))
        got = ET.decode(w, eps, cuda_layer, hps)
        assert got.dtype == torch.uint8 and got.shape == (2, 3, 8, 8)
        assert sorted(cuda_layer.samples) == ["0_0", "1_0"]
        for name, (e, c, z) in cuda_layer.samples.items():
            # every layer's sample round-trips to its noise through the prior's own step
            u, _, _ = cuda_layer.inner._prior_op(name, e.device).step(z, c)
            assert _rel(u, e.numpy().astype(np.float64)) < RT_TOL, name
    for name in ("0_0", "1_0"):
        # the latents: the fp32 kernel against the fp64 fixed point on the same context
        e, c, z = cuda_layer.samples[name]
        hidden, hd = MS._prior_layers(w, name, hps["depth_ar"], lambda t: t.numpy().astype(np.float64))
        zr = MS.inverse("theano", e.numpy(), c.numpy(), hidden, hd, hps["nl"])[0]
        assert _rel(z, zr) < TOL, name
    # the images: fp32 plumbing on both sides; the latents differ by a few ulp, which may move a pixel across one
    # quantisation boundary
    d = (got.int() - ref.int()).abs()
    assert int(d.max()) <= 1 and float((d > 0).float().mean()) < 0.01
    # the prior is sampled, not replaced by the reference's placeholder z = eps
    hd_layer = _Recording(type("EpsPrior", (), {"prior_sample": lambda self, n, e, c: e})())
    assert not torch.equal(ET.decode(w, eps, hd_layer, hps), ref)


def test_diag_decoder_needs_no_prior_sampler():
    hps = dict(HPS, depths=[1, 1], image_size=8, posterior="down_iaf2_nl", prior="diag")
    w, eps = _decoder_setup(hps, 2, 9)
    img = ET.decode(w, eps, None, hps)
    assert img.dtype == torch.uint8 and img.shape == (2, 3, 8, 8)
