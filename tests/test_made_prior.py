"""The autoregressive (MADE) prior, ``cvae_layer(..., prior='made', ...)`` (models.py:36-38, 304-309, 328): the fused
prior log-density entry ``iaf_ar_logp_*`` and the Theano ELBO with ``prior='made'``, on the CPU.

* the fp64 oracle (tests/made_oracle.py) against tests/golden/cvae_layer_made.npz, i.e. the reference's own models.py
  executed (tests/golden/make_golden_made.py), for all three posteriors with and without downsampling;
* the SIMT kernels under host emulation: the forward against the fp64 density, every NULL-output combination, the
  identity with the step's outputs, and the training pair against fp64 autograd;
* the Python autograd node over the emulated ABI, and the ELBO with prior='made' through it.
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
from oracle import iaf_oracle_torch as OT
from tests import flipmask_oracle as FO
from tests.emu.harness import EmuOperator, _arr, _check, _p
from tests.made_oracle import OracleIAFTheanoMade, TorchIAFTheanoMade

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cvae_layer_made.npz")
POSTERIORS = ("down_iaf2_nl", "up_iaf2_nl", "down_iaf2_nl2")
HPS = dict(n_z=4, n_h1=8, n_h2=8, depths=[2, 2], depth_ar=1, nl="elu", kl_min=0.0, image_size=16, prior="made")
TOL = 2e-5  # fp32 kernels vs fp64 autograd, relative to the largest entry of each tensor (as tests/test_emu_kernels.py)
LOG2PI = math.log(2 * math.pi)


def _rel(a, b):
    b = b.detach().numpy() if hasattr(b, "detach") else np.asarray(b)
    a = a.detach().numpy() if hasattr(a, "detach") else np.asarray(a)
    assert np.isfinite(a).all()
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


# ---------------------------------------------------------------------------------------------------------------------
# the oracle against the reference
# ---------------------------------------------------------------------------------------------------------------------
def _layer(posterior, name, iaf_cls, dtype, device):
    g = np.load(GOLD)
    pre = "%s:%s/" % (posterior, name)
    hps = dict(HPS, posterior=posterior)
    T = lambda a: torch.from_numpy(np.asarray(a)).to(dtype).to(device)
    w = {k[len(pre) + 2:]: T(g[k]) for k in g.files if k.startswith(pre + "w/")}
    iaf = iaf_cls(w, hps)
    ds = bool(g[pre + "downsample"])
    eps = T(g[pre + "eps"])
    up_out, up_state = ET.layer_up(w, name, T(g[pre + "up_in"]), hps, ds, eps, iaf)
    out, kl_bc, kl_sum = ET.layer_down_q(w, name, T(g[pre + "down_in"]), up_state, eps, iaf, hps, ds)
    got = dict(up_out=up_out, down_out=out, kl_bc=kl_bc, kl_sum=kl_sum)
    ref = dict(up_out=g[pre + "up_out"], down_out=g[pre + "down_out"], kl_bc=g[pre + "kl"].sum(axis=(2, 3)),
               kl_sum=g[pre + "kl"].sum(axis=(1, 2, 3)))
    return {k: v.detach().double().cpu().numpy() for k, v in got.items()}, ref


CASES = [(p, n) for p in POSTERIORS for n in ("0_1", "1_0")]


@pytest.mark.parametrize("posterior,name", CASES)
def test_made_layer_oracle_matches_reference_models_py(posterior, name):
    for cls in (OracleIAFTheanoMade, TorchIAFTheanoMade):
        got, ref = _layer(posterior, name, cls, torch.float64, "cpu")
        for k in ref:
            np.testing.assert_allclose(got[k], ref[k], rtol=1e-9, atol=1e-9, err_msg=k)


def test_made_fixture_has_the_prior_stack_and_channel_map():
    g = np.load(GOLD)
    for posterior, name in CASES:
        pre = "%s:%s/w/%s_" % (posterior, name, name)
        assert pre + "prior_conv1_0_w" in g.files and pre + "prior_conv1_out_1_w" in g.files
        n_down = g[pre + "down_conv1_w"].shape[0]
        assert n_down == 2 * 8 + (0 if posterior == "up_iaf2_nl" else 2 * 4 + 8)   # models.py:36-38, 84-96


# ---------------------------------------------------------------------------------------------------------------------
# the SIMT kernels under host emulation
# ---------------------------------------------------------------------------------------------------------------------
VARIANTS = ("tf", "theano", "theano_flipmask")
SHAPES = [
    # n_z, hidden, H, W, B, nl
    (4, [8], 4, 4, 2, "elu"),
    (8, [16, 16], 5, 7, 2, "softplus"),   # two hidden layers, non-square
    (4, [], 3, 6, 2, "elu"),              # depth_ar = 0 (Theano only: the TF front-end always has hidden layers)
    (4, [8], 12, 9, 1, "relu"),           # several row bands, two pixel segments
]


def _params(variant, n_z, hidden, seed=1):
    hid, hd = O.make_params("tf" if variant == "tf" else "theano", n_z, hidden, [n_z, n_z], seed=seed)
    return hid, hd, ("Vgb" if variant == "tf" else "wsb")


def _np_logps(variant, z, ctx, hid, hd, nl):
    """fp64: the heads of the stack, .1 each, rand.py:83 (models.py:304-309)."""
    f64 = lambda ls: O.cast_params(ls, np.float64)
    z, ctx = z.astype(np.float64), (ctx.astype(np.float64) if ctx is not None else None)
    if variant == "theano_flipmask":
        m, s = FO.multiconv(z, ctx, f64(hid), f64(hd), nl, flipmask=True)
    else:
        m, s = O.multiconv(variant, z, ctx, f64(hid), f64(hd), nl)
    return O.gaussian_diag_logps(0.1 * m, 2 * (0.1 * s), z)


def _t_logps(variant, z, ctx, th, thh, nl):
    if variant == "theano_flipmask":
        m, s = FO.t_multiconv(z, ctx, th, thh, nl, flipmask=True)
    else:
        m, s = OT.multiconv(variant, z, ctx, th, thh, nl)
    mean, logvar = 0.1 * m, 2 * (0.1 * s)
    return -0.5 * (LOG2PI + logvar + (z - mean) ** 2 / torch.exp(logvar))


def _emu(variant, n_z, hidden, H, W, B, nl, seed=1):
    hid, hd, keys = _params(variant, n_z, hidden, seed)
    z, ctx = O.make_inputs(B, n_z, hidden[0] if hidden else 1, H, W, seed=0)
    op = EmuOperator(variant, n_z, hidden, [n_z, n_z], H, W, nl=nl).set_weights(
        [tuple(l[k] for k in keys) for l in hid + hd])
    return op, hid, hd, keys, z, (ctx if hidden else None)


def emu_ar_logp(op, z, ctx, want=(True, True, True)):
    B = z.shape[0]
    lps = np.full_like(z, np.nan) if want[0] else None
    bc = np.full((B, op.n_z), np.nan, np.float32) if want[1] else None
    lp = np.full((B,), np.nan, np.float32) if want[2] else None
    _check(op.lib.iaf_ar_logp_fwd(op.plan, _p(z), _p(ctx), _p(lps), _p(bc), _p(lp), B, None))
    return lps, bc, lp


def emu_ar_logp_train(op, z, ctx):
    B = z.shape[0]
    lps, zo, ls = (np.full_like(z, np.nan) for _ in range(3))
    bc, lp = np.full((B, op.n_z), np.nan, np.float32), np.full((B,), np.nan, np.float32)
    hidden = [np.full((B, h, op.H, op.W), np.nan, np.float32) for h in op.hidden]
    _check(op.lib.iaf_ar_logp_fwd_train(op.plan, _p(z), _p(ctx), _p(lps), _p(bc), _p(lp), _p(zo), _p(ls),
                                        _arr(hidden) if hidden else None, B, None))
    return lps, bc, lp, zo, ls, hidden


def emu_ar_logp_bwd_saved(op, z, ctx, zo, ls, hidden, g_lps, g_bc, g_lp, params=True):
    B = z.shape[0]
    g_z, g_ctx, gw, gs, gb = op._grad_bufs(z, ctx, params)
    _check(op.lib.iaf_ar_logp_bwd_saved(op.plan, _p(z), _p(zo), _p(ls), _arr(hidden) if hidden else None,
                                        _arr([l[0] for l in op.layers]), _arr([l[1] for l in op.layers]), _p(g_lps),
                                        _p(g_bc), _p(g_lp), _p(g_z), _p(g_ctx), _arr(gw) if params else None,
                                        _arr(gs) if params else None, _arr(gb) if params else None, B, None))
    return g_z, g_ctx, gw, gs, gb


def _cases():
    for v, s in itertools.product(VARIANTS, SHAPES):
        if v == "tf" and not s[1]:
            continue
        yield (v,) + s


@pytest.mark.parametrize("variant,n_z,hidden,H,W,B,nl", list(_cases()))
def test_emulated_ar_logp_forward(variant, n_z, hidden, H, W, B, nl):
    op, hid, hd, _, z, ctx = _emu(variant, n_z, hidden, H, W, B, nl)
    ref = _np_logps(variant, z, ctx, hid, hd, nl)
    lps, bc, lp = emu_ar_logp(op, z, ctx)
    assert _rel(lps, ref) < 1e-5
    assert _rel(bc, ref.sum(axis=(2, 3))) < 1e-5 and _rel(lp, ref.sum(axis=(1, 2, 3))) < 1e-5
    # every NULL-output combination: the outputs that are asked for are bit-identical, nothing else is touched
    for want in itertools.product((False, True), repeat=3):
        got = emu_ar_logp(op, z, ctx, want)
        for g, full, w in zip(got, (lps, bc, lp), want):
            assert (g is None) if not w else np.array_equal(g, full)
    # the identity with the step's outputs: logp = -0.5 log 2pi n_z H W + logdet - 0.5 sum z'^2
    zo, _, logdet = op.step(z, ctx)
    ident = -0.5 * LOG2PI * n_z * H * W + logdet.astype(np.float64) - 0.5 * (zo.astype(np.float64) ** 2).sum(axis=(1, 2, 3))
    assert _rel(lp, ident) < 1e-5


def _check_param_grads(gw, gs, gb, th, keys, variant, n_hidden):
    for i, l in enumerate(th):
        for g, k in zip((gw[i], gs[i], gb[i]), keys):
            assert _rel(g, l[k].grad) < TOL, (i, k)
        zd = i >= n_hidden
        if variant == "tf":
            cin, cout = gw[i].shape[2], gw[i].shape[3]
            mask = O.get_conv_ar_mask(3, 3, cin, cout, zd)
        else:
            cin, cout = gw[i].shape[1] - 1, gw[i].shape[0]
            mask = FO.conv_ar_mask(cin, cout, zd, variant == "theano_flipmask")
        assert (gw[i][mask == 0] == 0).all(), i                       # masked taps: exactly zero


@pytest.mark.parametrize("variant,n_z,hidden,H,W,B,nl", list(_cases()))
def test_emulated_ar_logp_training_pair(variant, n_z, hidden, H, W, B, nl):
    op, hid, hd, keys, z, ctx = _emu(variant, n_z, hidden, H, W, B, nl)
    lps0, bc0, lp0 = emu_ar_logp(op, z, ctx)
    lps, bc, lp, zo, ls, hs = emu_ar_logp_train(op, z, ctx)
    assert np.array_equal(lps, lps0) and np.array_equal(bc, bc0) and np.array_equal(lp, lp0)
    zs, lss, _ = op.step(z, ctx)
    assert np.array_equal(zo, zs) and np.array_equal(ls, lss)      # what the backward keeps: the step's own z', logsd
    rng = np.random.RandomState(5)
    ups = (rng.randn(*z.shape).astype(np.float32), rng.randn(B, n_z).astype(np.float32), rng.randn(B).astype(np.float32))
    for sel in ((0,), (1,), (2,), (0, 1, 2)):
        g_in = [ups[k] if k in sel else None for k in range(3)]
        th, thh = OT.to_torch(O.cast_params(hid, np.float64), torch.float64), OT.to_torch(O.cast_params(hd, np.float64), torch.float64)
        for l in th + thh:
            for t in l.values():
                t.requires_grad_(True)
        zt = torch.from_numpy(z).double().requires_grad_(True)
        ct = torch.from_numpy(ctx).double().requires_grad_(True) if ctx is not None else None
        lt = _t_logps(variant, zt, ct, th, thh, nl)
        obj = 0.0
        if 0 in sel:
            obj = obj + (lt * torch.from_numpy(ups[0])).sum()
        if 1 in sel:
            obj = obj + (lt.sum(dim=(2, 3)) * torch.from_numpy(ups[1])).sum()
        if 2 in sel:
            obj = obj + (lt.sum(dim=(1, 2, 3)) * torch.from_numpy(ups[2])).sum()
        obj.backward()
        g_z, g_ctx, gw, gs, gb = emu_ar_logp_bwd_saved(op, z, ctx, zo, ls, hs, *g_in)
        assert _rel(g_z, zt.grad) < TOL and (ctx is None or _rel(g_ctx, ct.grad) < TOL), sel
        _check_param_grads(gw, gs, gb, th + thh, keys, variant, len(hidden))
        again = emu_ar_logp_bwd_saved(op, z, ctx, zo, ls, hs, *g_in)
        assert all(np.array_equal(a, b) for a, b in zip(again[:2] + tuple(again[2] + again[3] + again[4]),
                                                         (g_z, g_ctx) + tuple(gw + gs + gb)) if a is not None)


def test_emulated_ar_logp_checks_its_arguments():
    op, hid, hd, keys, z, ctx = _emu("theano", 4, [8], 4, 4, 2, "elu")
    B = z.shape[0]
    with pytest.raises(RuntimeError):
        _check(op.lib.iaf_ar_logp_fwd(op.plan, _p(z), _p(None), None, None, None, B, None))   # context is required
    with pytest.raises(RuntimeError):  # the training forward must keep z' and made_logsd
        _check(op.lib.iaf_ar_logp_fwd_train(op.plan, _p(z), _p(ctx), None, None, None, None, None, None, B, None))
    one = EmuOperator("theano", 4, [8], [4], 4, 4)
    one.set_weights([tuple(l[k] for k in "wsb") for l in O.make_params("theano", 4, [8], [4], seed=1)[0] +
                     O.make_params("theano", 4, [8], [4], seed=1)[1]])
    assert one.lib.iaf_ar_logp_fwd(one.plan, _p(z), _p(ctx), None, None, None, B, None) == -2   # needs two heads of n_z
    from iaf_b200 import _lib as L
    assert op.lib.iaf_plan_path_for_entry(op.plan, L.ENTRIES["ar_logp"]) == L.PATHS["simt"]
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
    from tests.emu.harness import emu

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


def test_python_ar_logp_autograd_glue_over_the_emulated_abi(monkeypatch):
    """IAFOperator.ar_logp: the plain call and the _ArLogpFn node (argument order, saved tensors, None upstreams)."""
    from iaf_b200 import ops
    with _emulated_abi(monkeypatch):
        variant, n_z, hidden, H, W, B = "theano", 4, [8], 4, 5, 2
        hid, hd = O.make_params(variant, n_z, hidden, [n_z, n_z], seed=1)
        z, ctx = O.make_inputs(B, n_z, hidden[0], H, W, seed=0)
        dev = [tuple(torch.from_numpy(l[k].copy()).requires_grad_(True) for k in "wsb") for l in hid + hd]
        op = ops.IAFOperator(variant, n_z, hidden, [n_z, n_z], nl="elu", path="simt").set_weights(dev)
        assert op.path_used(H, W, "cpu", entry="ar_logp") == "simt"
        ref = _np_logps(variant, z, ctx, hid, hd, "elu")
        with torch.no_grad():
            lps, bc, lp = op.ar_logp(torch.from_numpy(z), torch.from_numpy(ctx), want_logps=True)
            none, bc2, lp2 = op.ar_logp(torch.from_numpy(z), torch.from_numpy(ctx))
        assert none is None and torch.equal(bc, bc2) and torch.equal(lp, lp2)
        assert _rel(lps, ref) < 1e-5 and _rel(lp, ref.sum(axis=(1, 2, 3))) < 1e-5
        # only logp_bc and logp are used downstream: the logps gradient arrives as None
        zg, cg = torch.from_numpy(z).requires_grad_(True), torch.from_numpy(ctx).requires_grad_(True)
        _, bc, lp = op.ar_logp(zg, cg)
        assert bc.grad_fn is not None and type(bc.grad_fn).__name__.startswith("_ArLogpFn")
        (bc.square().sum() + 3.0 * lp.sum()).backward()
    th = OT.to_torch(O.cast_params(hid, np.float64), torch.float64)
    thh = OT.to_torch(O.cast_params(hd, np.float64), torch.float64)
    for l in th + thh:
        for t in l.values():
            t.requires_grad_(True)
    zt, ct = torch.from_numpy(z).double().requires_grad_(True), torch.from_numpy(ctx).double().requires_grad_(True)
    lt = _t_logps(variant, zt, ct, th, thh, "elu")
    (lt.sum(dim=(2, 3)).square().sum() + 3.0 * lt.sum(dim=(1, 2, 3)).sum()).backward()
    assert _rel(zg.grad, zt.grad) < TOL and _rel(cg.grad, ct.grad) < TOL
    for i, l in enumerate(th + thh):
        for t, k in zip(dev[i], "wsb"):
            assert _rel(t.grad, l[k].grad) < TOL, (i, k)


def _setup(hps, B, seed, dtype, device):
    w = {k: torch.from_numpy(np.asarray(v)).to(dtype).to(device) for k, v in ET.make_params(hps, seed=seed).items()}
    rng = np.random.RandomState(seed + 1)
    S = hps["image_size"]
    x = torch.from_numpy(rng.randint(0, 256, size=(B, 3, S, S)).astype(np.uint8)).to(device)
    noise = {}
    for i in range(len(hps["depths"])):
        s = S // 2 ** (i + 1)
        for j in range(hps["depths"][i]):
            noise[(i, j)] = torch.from_numpy(rng.randn(B, hps["n_z"], s, s)).to(dtype).to(device)
    return w, x, noise


@pytest.mark.parametrize("posterior,name", CASES)
def test_made_layer_through_the_emulated_abi(posterior, name, monkeypatch):
    with _emulated_abi(monkeypatch):
        got, ref = _layer(posterior, name, lambda w, hps: ET.CudaIAF(w, hps, path="simt"), torch.float32, "cpu")
    for k in ref:
        assert _rel(got[k], ref[k]) < 1e-4, k


@pytest.mark.parametrize("posterior", POSTERIORS)
def test_made_elbo_and_training_gradients_over_the_emulated_abi(posterior, monkeypatch):
    """cvae1 with prior='made': cost against the fp64 oracle, and d(cost)/d(every parameter) through CudaIAFTrain (the
    prior's own autograd node included) against fp64 autograd."""
    hps = dict(HPS, depths=[1, 1], image_size=8, posterior=posterior)
    w32, x, n32 = _setup(hps, 2, 7, torch.float32, "cpu")
    w64, _, n64 = _setup(hps, 2, 7, torch.float64, "cpu")
    assert any("_prior_conv1_out_1_" in k for k in w32)
    ref0 = ET.forward(w64, x, n64, OracleIAFTheanoMade(w64, hps), hps)
    for w in (w32, w64):
        for v in w.values():
            v.requires_grad_(True)
    with _emulated_abi(monkeypatch):
        iaf = ET.CudaIAFTrain(w32, hps, path="simt")
        got = ET.forward(w32, x, n32, iaf, hps)
        got["cost"].sum().backward()
    assert sorted(iaf.prior_ops) == ["0_0", "1_0"]
    ref = ET.forward(w64, x, n64, TorchIAFTheanoMade(w64, hps), hps)
    np.testing.assert_allclose(ref["cost"].detach().numpy(), ref0["cost"].numpy(), rtol=1e-12)
    np.testing.assert_allclose(got["cost"].detach().numpy(), ref["cost"].detach().numpy(), rtol=2e-5)
    ref["cost"].sum().backward()
    checked = 0
    for k in w64:
        g, r = w32[k].grad, w64[k].grad
        if r is None:
            assert g is None, k
            continue
        err = float((g.double() - r).abs().max()) / max(float(r.abs().max()), 1e-12)
        assert err < 5e-4, (k, err)   # fp32 torch plumbing around the operators
        if "_prior_conv1_" in k and k.endswith("_w"):
            mask = FO.conv_ar_mask(g.shape[1] - 1, g.shape[0], "_out_" in k, False)
            assert bool((g.numpy()[mask == 0] == 0).all()), k   # masked taps: exactly zero (ar.py:369-373)
            checked += 1
    assert checked == 3 * len(hps["depths"])
    # the made objective is not the diagonal-prior one
    hd = dict(hps, prior="diag")
    wd, xd, nd = _setup(hd, 2, 7, torch.float64, "cpu")
    assert abs(float(ET.forward(wd, xd, nd, OracleIAFTheanoMade(wd, hd), hd)["bits_per_dim"]) -
               float(ref0["bits_per_dim"])) > 1e-6


def test_unknown_priors_are_refused():
    for prior in ("diag2", "bernoulli", "made2"):
        hps = dict(HPS, prior=prior, posterior="down_iaf2_nl")
        with pytest.raises(ValueError):
            ET.make_params(hps, seed=0)
        wd, x, noise = _setup(dict(hps, prior="diag"), 2, 3, torch.float64, "cpu")
        with pytest.raises(ValueError):
            ET.forward(wd, x, noise, OracleIAFTheanoMade(wd, hps), hps)
    # the default stays the diagonal prior: no prior stack, down_conv1 unchanged
    w = ET.make_params(dict(HPS, prior="diag", posterior="down_iaf2_nl"), seed=0)
    assert not any("_prior_conv1_" in k for k in w)
    assert w["0_0_down_conv1_w"].shape[0] == (8 + 2 * 4) + (2 * 4 + 8)
