"""Stacks without a hidden layer (depth_ar = 0, and the linear IAF posteriors down_iaf2 / up_iaf2) on the H100's tensor
cores: the per-stage kernel's heads stage fed from fp32 z, in all four modes (step, multiconv, layer, logp) against fp64
per sample, the tile schedule, the envelope, the backward under every backward-kernel setting, the inverse on such a
plan, and the Theano ELBO with the linear posteriors and its training gradients."""
import math

import numpy as np
import pytest
import torch

from iaf_b200 import IAFOperator
from iaf_b200 import elbo_theano as ET
from oracle import iaf_oracle as O
from oracle import iaf_oracle_torch as OT
from tests import flipmask_oracle as FO
from tests import linear_oracle as LO

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-4
LOG2PI = math.log(2 * math.pi)
VARIANTS = ("tf", "theano", "theano_flipmask")
ENTRIES = ("step", "multiconv", "layer", "ar_logp")


def _np(t):
    return t.detach().double().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t, dtype=np.float64)


def per_sample_err(a, ref):
    a, ref = _np(a), _np(ref)
    assert np.isfinite(a).all()
    d = np.abs(a - ref).reshape(a.shape[0], -1).max(axis=1)
    r = np.maximum(np.abs(ref).reshape(a.shape[0], -1).max(axis=1), 1.0)
    return float((d / r).max())


def bwd_err(a, ref):
    a, ref = _np(a), _np(ref)
    assert np.isfinite(a).all()
    m = np.abs(ref).max()
    assert m > 0
    return float(np.abs(a - ref).max() / m)


class Case(object):
    """A depth-0 stack: two heads of n_z straight on z, no context."""

    def __init__(self, variant, n_z, path="auto", seed=1):
        self.variant, self.n_z = variant, n_z
        self.keys = "Vgb" if variant == "tf" else "wsb"
        self.hid, self.hd = O.make_params("tf" if variant == "tf" else "theano", n_z, [], [n_z, n_z], seed=seed)
        self.layers = [tuple(torch.from_numpy(l[k]).to(DEV) for k in self.keys) for l in self.hd]
        self.op = IAFOperator("tf" if variant == "tf" else "theano", n_z, [], [n_z, n_z], nl="elu", path=path,
                              flipmask=variant == "theano_flipmask").set_weights(self.layers)

    def f64_heads(self, grad=False):
        thh = OT.to_torch(O.cast_params(self.hd, np.float64), torch.float64)
        for l in thh:
            for t in l.values():
                t.requires_grad_(grad)
        return thh

    def heads(self, z, thh):
        if self.variant == "theano_flipmask":
            return FO.t_multiconv(z, None, [], thh, "elu", flipmask=True)
        return OT.multiconv(self.variant, z, None, [], thh, "elu")

    def step(self, z, thh):
        m, s = self.heads(z, thh)
        a = 0.1 * s
        return (z - 0.1 * m) / torch.exp(a), a

    def logps(self, z, thh):
        m, s = self.heads(z, thh)
        mean, logvar = 0.1 * m, 2 * (0.1 * s)
        return -0.5 * (LOG2PI + logvar + (z - mean) ** 2 / torch.exp(logvar))   # rand.py:83

    def layer(self, eps, pm, pls, qm, qls, thh):
        z0 = pm + torch.exp(pls) * eps
        z, a = self.step(z0, thh)
        logqs = -0.5 * LOG2PI - pls - 0.5 * eps * eps + a
        logps = -0.5 * LOG2PI - qls - 0.5 * (z - qm) ** 2 * torch.exp(-2 * qls)
        return z, logqs - logps


def _inputs(n_z, B, H, W, seed=0):
    rng = np.random.RandomState(seed)
    f = lambda scale, off=0.0: torch.from_numpy((off + scale * rng.randn(B, n_z, H, W)).astype(np.float32)).to(DEV)
    return dict(z=f(1.0), pm=f(0.3), pls=f(0.2, -0.3), qm=f(0.3), qls=f(0.2, -0.2))


def _all_entries(op, x):
    """Every forward entry once: {entry: tuple of outputs}."""
    z = x["z"]
    with torch.no_grad():
        return dict(step=op.step(z, None), multiconv=tuple(op.multiconv(z, None)),
                    layer=op.layer(z, x["pm"], x["pls"], x["qm"], x["qls"], None),
                    ar_logp=op.ar_logp(z, None, want_logps=True))


MAPS = [(1, 1), (4, 4), (16, 16), (12, 20), (2, 126)]


def _maps(n_z):
    # the z window holds n_z / 8 chunks of 128 + MIR slots, at most 1024 items: n_z = 48 reaches W = 38, not 126
    return [m for m in MAPS if n_z < 48 or m[1] <= 38] + ([(2, 38)] if n_z == 48 else [])


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("n_z,H,W", [(n, h, w) for n in (16, 32, 48) for h, w in _maps(n)])
def test_depth0_forward_all_entries_on_the_tensor_cores(variant, n_z, H, W):
    c = Case(variant, n_z)
    for e in ENTRIES:
        assert c.op.path_used(H, W, DEV, entry=e) == "tc", e
    x = _inputs(n_z, 3, H, W)
    thh = c.f64_heads()
    zt = torch.from_numpy(_np(x["z"]))
    _all_entries(c.op, x)                                               # packs the weights
    n0 = c.op.launch_count()
    got = _all_entries(c.op, x)
    assert c.op.launch_count() - n0 == len(ENTRIES)                     # one launch per forward: the heads stage
    with torch.no_grad():
        torch.cuda.synchronize()
        z_ref, a_ref = c.step(zt, thh)
        zo, ls, ld = got["step"]
        assert per_sample_err(zo, z_ref) < TOL and per_sample_err(ls, a_ref) < TOL
        assert per_sample_err(ld[:, None], -a_ref.sum(dim=(1, 2, 3))[:, None]) < TOL
        m_ref, s_ref = c.heads(zt, thh)
        assert per_sample_err(got["multiconv"][0], m_ref) < TOL and per_sample_err(got["multiconv"][1], s_ref) < TOL
        f = lambda k: torch.from_numpy(_np(x[k]))
        zl_ref, kl_ref = c.layer(zt, f("pm"), f("pls"), f("qm"), f("qls"), thh)
        zl, kl, kl_bc, kl_cost = got["layer"]
        assert per_sample_err(zl, zl_ref) < TOL and per_sample_err(kl, kl_ref) < TOL
        assert per_sample_err(kl_bc, kl_ref.sum(dim=(2, 3))) < TOL
        assert per_sample_err(kl_cost[:, None], kl_ref.sum(dim=(1, 2, 3))[:, None]) < TOL
        lps_ref = c.logps(zt, thh)
        lps, bc, lp = got["ar_logp"]
        assert per_sample_err(lps, lps_ref) < TOL and per_sample_err(bc, lps_ref.sum(dim=(2, 3))) < TOL
        assert per_sample_err(lp[:, None], lps_ref.sum(dim=(1, 2, 3))[:, None]) < TOL


@pytest.mark.parametrize("variant,n_z,H,W", [("theano", 32, 16, 16), ("tf", 16, 12, 20), ("theano_flipmask", 48, 8, 8)])
def test_depth0_tile_schedule_is_bit_identical(variant, n_z, H, W, monkeypatch):
    """B = 32 spans tens of tiles: one CTA per SM, one CTA in all, three CTAs; the outputs do not move."""
    outs = []
    x = _inputs(n_z, 32, H, W, seed=2)
    for n in ("1", "3", None):
        if n is None:
            monkeypatch.delenv("IAF_NUM_SMS", raising=False)
        else:
            monkeypatch.setenv("IAF_NUM_SMS", n)
        c = Case(variant, n_z)
        assert all(c.op.path_used(H, W, DEV, entry=e) == "tc" for e in ENTRIES)
        outs.append({e: [t.cpu() for t in v if t is not None] for e, v in _all_entries(c.op, x).items()})
    for o in outs[1:]:
        for e in ENTRIES:
            assert all(torch.equal(a, b) for a, b in zip(o[e], outs[0][e])), e


@pytest.mark.parametrize("n_z,H,W", [(64, 16, 16), (8, 16, 16), (48, 2, 126), (32, 2, 127)])
def test_depth0_shapes_outside_the_tensor_cores(n_z, H, W):
    """``auto`` keeps them on the SIMT kernels; ``path="tc"`` refuses instead of slowing down."""
    c = Case("theano", n_z)
    for e in ENTRIES:
        assert c.op.path_used(H, W, DEV, entry=e) == "simt", e
    with pytest.raises(NotImplementedError):
        Case("theano", n_z, path="tc").op.path_used(H, W, DEV)


BWD_SETTINGS = [({}, "tc"), ({"IAF_BWD_FUSED_PROLOGUE": "0"}, "tc"), ({"IAF_BWD_WG_TC": "0"}, "tc-dgrad"),
                ({"IAF_BWD_TC": "0"}, "simt")]


@pytest.mark.parametrize("env,bwd_path", BWD_SETTINGS, ids=["default", "no_fused_prologue", "no_wg_tc", "no_tc"])
@pytest.mark.parametrize("variant,n_z,H,W", [("theano", 32, 16, 16), ("tf", 16, 12, 20), ("theano_flipmask", 48, 8, 8),
                                             ("theano", 32, 4, 22)])
def test_depth0_backward(variant, n_z, H, W, env, bwd_path, monkeypatch):
    """Every entry's backward against fp64 autograd: the single stage's data gradient lands in g_z on top of the affine
    term, the weight gradient runs over z; no context gradient exists."""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    c = Case(variant, n_z)
    assert c.op.backward_path(H, W, DEV) == bwd_path
    assert c.op.path_used(H, W, DEV, entry="step") == "tc"
    x = _inputs(n_z, 3, H, W, seed=4)
    rng = np.random.RandomState(6)
    up = lambda *s: torch.from_numpy(rng.randn(*s).astype(np.float32)).to(DEV)
    B = 3
    for entry in ENTRIES:
        params = [tuple(t.clone().requires_grad_(True) for t in l) for l in c.layers]
        c.op.set_weights(params)
        ins = {k: v.clone().requires_grad_(True) for k, v in x.items()}
        thh = c.f64_heads(True)
        ref_ins = {k: torch.from_numpy(_np(v)).requires_grad_(True) for k, v in x.items()}
        if entry == "step":
            u = [up(B, n_z, H, W), up(B, n_z, H, W), up(B)]
            zo, ls, ld = c.op.step(ins["z"], None)
            zr, ar = c.step(ref_ins["z"], thh)
            outs, refs = (zo, ls, ld), (zr, ar, -ar.sum(dim=(1, 2, 3)))
        elif entry == "multiconv":
            u = [up(B, n_z, H, W), up(B, n_z, H, W)]
            outs, refs = tuple(c.op.multiconv(ins["z"], None)), tuple(c.heads(ref_ins["z"], thh))
        elif entry == "layer":
            u = [up(B, n_z, H, W), up(B, n_z, H, W), up(B, n_z), up(B)]
            outs = c.op.layer(ins["z"], ins["pm"], ins["pls"], ins["qm"], ins["qls"], None)
            zr, klr = c.layer(ref_ins["z"], ref_ins["pm"], ref_ins["pls"], ref_ins["qm"], ref_ins["qls"], thh)
            refs = (zr, klr, klr.sum(dim=(2, 3)), klr.sum(dim=(1, 2, 3)))
        else:
            u = [up(B, n_z, H, W), up(B, n_z), up(B)]
            outs = c.op.ar_logp(ins["z"], None, want_logps=True)
            lr = c.logps(ref_ins["z"], thh)
            refs = (lr, lr.sum(dim=(2, 3)), lr.sum(dim=(1, 2, 3)))
        sum(((o * g).sum() for o, g in zip(outs, u)), torch.zeros((), device=DEV)).backward()
        sum(((r * g.cpu().double()).sum() for r, g in zip(refs, u)), torch.zeros((), dtype=torch.float64)).backward()
        used = ("z", "pm", "pls", "qm", "qls") if entry == "layer" else ("z",)
        for k in used:
            assert bwd_err(ins[k].grad, ref_ins[k].grad) < TOL, (entry, k)
        for i, (l, r) in enumerate(zip(params, thh)):
            for t, k in zip(l, c.keys):
                assert bwd_err(t.grad, r[k].grad) < TOL, (entry, i, k)
            g = _np(l[0].grad)
            if variant == "tf":
                mask = O.get_conv_ar_mask(3, 3, n_z, n_z, True)
            else:
                mask = FO.conv_ar_mask(n_z, n_z, True, variant == "theano_flipmask")
            assert (g[mask == 0] == 0).all(), (entry, i)      # masked taps: exactly zero


@pytest.mark.parametrize("variant", VARIANTS)
def test_step_inverse_on_a_depth0_tensor_core_plan(variant):
    c = Case(variant, 32)
    H = W = 8
    assert c.op.path_used(H, W, DEV, entry="step") == "tc"
    u = _inputs(32, 4, H, W, seed=8)["z"]
    with torch.no_grad():
        z, ls, ld = c.op.step_inverse(u, None)
        u2, ls2, ld2 = c.op.step(z, None)
    assert per_sample_err(u2, u) < 1e-5
    assert per_sample_err(ls, ls2) < 1e-5 and per_sample_err(ld[:, None], ld2[:, None]) < 1e-5


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


@pytest.mark.parametrize("posterior", ET.LINEAR)
@pytest.mark.parametrize("prior", ET.PRIORS)
def test_linear_elbo_and_training_gradients_on_the_tensor_cores(posterior, prior):
    """The Theano ELBO with a linear posterior at n_z = 32, every posterior operator on the tensor cores forward and
    backward: the cost against the fp64 oracle (inference and training wrappers), d(cost)/d(every parameter) against
    fp64 autograd, the posterior conv's gradient interleaved with masked taps exactly zero."""
    hps = dict(n_z=32, n_h1=32, n_h2=32, depths=[1, 1], depth_ar=1, nl="elu", kl_min=0.0, image_size=16,
               posterior=posterior, prior=prior)
    w32, x, n32 = _setup(hps, 2, 7, torch.float32, "cuda")
    w64, _, n64 = _setup(hps, 2, 7, torch.float64, "cpu")
    ref0 = ET.forward(w64, x.cpu(), n64, LO.OracleIAFTheanoLinear(w64, hps), hps)
    inf = ET.CudaIAF(w32, hps)
    with torch.no_grad():
        got0 = ET.forward(w32, x, n32, inf, hps)
    np.testing.assert_allclose(got0["cost"].cpu().numpy(), ref0["cost"].numpy(), rtol=2e-5)
    for w in (w32, w64):
        for v in w.values():
            v.requires_grad_(True)
    iaf = ET.CudaIAFTrain(w32, hps)
    got = ET.forward(w32, x, n32, iaf, hps)
    got["cost"].sum().backward()
    for ops in (inf.ops, iaf.ops):
        assert sorted(ops) == [("0_0", 1), ("1_0", 1)]
        for (name, _), op in ops.items():
            s = hps["image_size"] // 2 ** (int(name[0]) + 1)
            assert op.hidden == [] and op.path_used(s, s, DEV, "step") == "tc" and op.path_used(s, s, DEV, "layer") == "tc"
            assert op.backward_path(s, s, DEV) == "tc", name
    ref = ET.forward(w64, x.cpu(), n64, LO.TorchIAFTheanoLinear(w64, hps), hps)
    np.testing.assert_allclose(got["cost"].detach().cpu().numpy(), ref["cost"].detach().numpy(), rtol=2e-5)
    ref["cost"].sum().backward()
    checked = 0
    for k in w64:
        g, r = w32[k].grad, w64[k].grad
        assert (g is None) == (r is None), k
        if r is None:
            continue
        g = g.cpu()
        err = float((g.double() - r).abs().max()) / max(float(r.abs().max()), 1e-12)
        assert err < 5e-4, (k, err)   # fp32 torch plumbing around the operators
        if k.endswith("_posterior_conv1_w"):
            mask = O.theano_conv_ar_mask(32, 64, zerodiagonal=True, pad_channel=True)
            assert bool((g.numpy()[mask == 0] == 0).all()), k
            checked += 1
    assert checked == len(hps["depths"])
