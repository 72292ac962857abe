"""CPU checks of the reference's Eve optimiser (iaf_b200.optim.Eve, iaf_eve_step, elbo_theano's optim='eve'):

* the op-by-op fp32 restatement (tests/eve_oracle.py) reproduces tests/golden/eve.npz, the trajectory of the
  reference's own Eve source, bit for bit, taking its gradients at its own lookahead; and the fixture does exercise the
  lookahead: the gradients taken at w instead give another trajectory;
* the kernel, run under the host emulation (tests/emu), is bit-identical to the restatement: tensor sizes around the
  4096-element tile, views at odd storage offsets, missing gradients, a gradient scale with other hyperparameters, and
  a table that needs a second launch;
* the C entry refuses bad arguments, the library without the kernel refuses after validating, and the Python side
  refuses what it cannot take;
* a 2-rank gloo sharded Theano ``train_step`` with Eve equals one process running the same towers on the global batch's
  mean cost, at an even and an uneven split.
"""
import ctypes as C
import math
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from iaf_b200 import _lib as L
from iaf_b200 import elbo, elbo_theano
from iaf_b200 import optim
from iaf_b200.optim import EVE_DEFAULTS, Eve
from tests.adamax_oracle import RestatedAdamax
from tests.emu import harness
from tests.emu.optim import emu
from tests.eve_oracle import RestatedEve

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "eve.npz")
NAMES = ("a", "b", "c")
STATE = ("mom1", "mom_max", "delta", "avg")


# ---------------------------------------------------------------------------------------------------------------------
# the restatement against the reference's own trajectory
def _gradient_at(f, k, point, t):
    """tests/golden/make_golden_eve.py's stand-in objective: its gradient at ``point`` on step t (float32)."""
    n = f["noise/" + k][t]
    if not f["has_c"][t] and k == "c":
        return None
    if t in f["edge_steps"]:
        return torch.from_numpy(n.copy())
    g = n + f["kappa"] * (point.numpy() - f["target/" + k])
    g[n == 0] = 0.0
    return torch.from_numpy(g.astype(np.float32))


def _run_fixture(at_lookahead):
    f = np.load(GOLDEN)
    params = {k: torch.from_numpy(f["param0/" + k].copy()) for k in NAMES}
    opt = RestatedEve(params)
    flat = lambda d: np.concatenate([d[k].detach().numpy().ravel() for k in NAMES])
    out = {key: [] for key in ("grad", "param", "lookahead") + STATE}
    for t in range(f["has_c"].shape[0]):
        point = opt.lookahead() if at_lookahead else params
        grads = {k: _gradient_at(f, k, point[k].detach(), t) for k in NAMES}
        out["grad"].append(flat({k: torch.zeros(params[k].shape) if g is None else g for k, g in grads.items()}))
        opt.step(grads=grads)
        out["param"].append(flat(params))
        out["lookahead"].append(flat(opt.lookahead()))
        for name in STATE:
            out[name].append(flat(getattr(opt, name)))
    return f, {k: np.stack(v) for k, v in out.items()}


def test_restatement_matches_reference_trajectory():
    f, got = _run_fixture(at_lookahead=True)
    for name, v in got.items():
        for t in range(v.shape[0]):
            np.testing.assert_array_equal(v[t], f["eve/" + name][t], err_msg="%s step %d" % (name, t))


def test_fixture_exercises_the_lookahead():
    """The gradients of the fixture depend on where they are taken: at w instead of w' they differ from step 1 on (at
    step 0 the two points are equal), and so does the whole trajectory."""
    f, got = _run_fixture(at_lookahead=False)
    np.testing.assert_array_equal(got["grad"][0], f["eve/grad"][0])
    assert not np.array_equal(got["grad"][1], f["eve/grad"][1])
    for name in ("param", "lookahead", "avg", "delta"):
        assert not np.array_equal(got[name][-1], f["eve/" + name][-1]), name
    # and the lookahead really is away from w: c = (1 - b1) / b1 = 9 times the last update
    assert (f["eve/lookahead"] != f["eve/param"]).sum() > f["eve/param"].size // 2


def test_golden_sequence_covers_the_edges():
    f = np.load(GOLDEN)
    g = f["eve/grad"]
    assert (g[3] == 0).all() and (g == 0).any(axis=0).all()
    live = g[10:13] != 0
    assert np.isclose(np.abs(g[10:13][live]), 1e-30, rtol=1e-6).all() and (np.abs(g[20][g[20] != 0]) == 1e4).all()
    assert (np.sign(g[8]) == -np.sign(g[7]))[(g[7] != 0) & (g[8] != 0)].all()
    assert not f["has_c"].all()
    assert (g[:, 0] == 0).all()                                 # an element that never sees a gradient


# ---------------------------------------------------------------------------------------------------------------------
# the kernel under the host emulation
class EveEmuSet(object):
    """A parameter set in numpy buffers, stepped by the emulated iaf_eve_step.  ``shift``: each parameter and gradient
    is a view one float into its buffer (an odd storage offset, 4-byte aligned only); state slices start at odd
    offsets then too."""

    def __init__(self, params, shift=0, **hp):
        self.shift = shift
        self.hp = {k: (EVE_DEFAULTS[k] if hp.get(k) is None else hp[k]) for k in EVE_DEFAULTS}
        self.bufs = [np.zeros(p.size + shift, np.float32) for p in params]
        self.params = [b[shift:] for b in self.bufs]
        for dst, p in zip(self.params, params):
            dst[...] = p.ravel()
        self.offsets, total = [], 0
        for p in params:
            self.offsets.append(total + shift)
            total += p.size + shift if shift else -(-p.size // 4) * 4
        self.mom1 = np.zeros(total, np.float32)
        self.mom_max = np.full(total, 1e-8, np.float32)
        self.delta = np.zeros(total, np.float32)
        self.avg = np.zeros(total, np.float32)
        self.lookahead = np.zeros(total, np.float32)
        for p, off in zip(self.params, self.offsets):
            self.avg[off:off + p.size] = p
            self.lookahead[off:off + p.size] = p
        self.gbufs = [np.zeros(p.size + shift, np.float32) for p in params]

    def table(self, grads):
        t = (L.AdamaxTensor * len(self.params))()
        for e, p, gb, g, off in zip(t, self.params, self.gbufs, grads, self.offsets):
            e.param, e.numel, e.offset = p.ctypes.data, p.size, off
            if g is not None:
                gb[self.shift:] = g.ravel()
                e.grad = gb.ctypes.data + 4 * self.shift
        return t

    def step(self, grads, grad_scale=1.0):
        t = self.table(grads)
        h = self.hp
        ptr = lambda a: C.c_void_p(a.ctypes.data)
        return emu().iaf_eve_step(t, len(t), ptr(self.mom1), ptr(self.mom_max), ptr(self.delta), ptr(self.avg),
                                  ptr(self.lookahead), h["lr"], h["beta1"], h["beta2"], h["beta3"], grad_scale, None)

    def state(self, name, i):
        return getattr(self, name)[self.offsets[i]:self.offsets[i] + self.params[i].size]


def _grads(rng, sizes, step, missing):
    out = []
    for i, n in enumerate(sizes):
        if i in missing and step % 2 == 1:
            out.append(None)
            continue
        g = (rng.randn(n) * np.exp(rng.uniform(-4, 4, size=n))).astype(np.float32)
        g[rng.rand(n) < 0.1] = 0.0
        out.append(g)
    return out


def _compare(sizes, shift=0, steps=4, missing=(), grad_scale=1.0, seed=0, **hp):
    rng = np.random.RandomState(seed)
    p0 = [(0.3 * rng.randn(n)).astype(np.float32) for n in sizes]
    es = EveEmuSet(p0, shift, **hp)
    tp = {str(i): torch.from_numpy(p.copy()) for i, p in enumerate(p0)}
    ref = RestatedEve(tp, **hp)
    before = emu().iaf_adamax_launch_count()
    for s in range(steps):
        gs = _grads(rng, sizes, s, missing)
        assert es.step(gs, grad_scale) == 0
        ref.step(grad_scale, grads={str(i): None if g is None else torch.from_numpy(g) for i, g in enumerate(gs)})
    for i in range(len(sizes)):
        k = str(i)
        np.testing.assert_array_equal(es.params[i], tp[k].numpy(), err_msg="param %d" % i)
        np.testing.assert_array_equal(es.state("lookahead", i), ref.la[k].detach().numpy(), err_msg="lookahead %d" % i)
        for name in STATE:
            np.testing.assert_array_equal(es.state(name, i), getattr(ref, name)[k].numpy(), err_msg="%s %d" % (name, i))
    return emu().iaf_adamax_launch_count() - before


@pytest.mark.parametrize("shift", [0, 1], ids=["aligned", "odd_offset"])
def test_emulated_kernel_equals_restatement(shift):
    assert _compare([1, 3, 4095, 4096, 4097, 9000], shift=shift, missing=(1, 4)) == 4


def test_emulated_kernel_grad_scale_and_hyperparameters():
    _compare([7, 4100], grad_scale=0.5, lr=0.003, beta1=0.2, beta2=0.01, beta3=0.05, seed=1)
    _compare([5, 4099], shift=1, grad_scale=3.0, lr=0.01, beta1=0.7, beta2=0.1, beta3=0.5, seed=2)


def test_emulated_kernel_missing_gradient_is_a_zero_gradient():
    p0 = [np.linspace(-1, 1, 6).astype(np.float32)]
    a, b = EveEmuSet(p0), EveEmuSet(p0)
    for es in (a, b):
        assert es.step([np.ones(6, np.float32)]) == 0
    assert a.step([None]) == 0 and b.step([np.zeros(6, np.float32)]) == 0
    for name in ("params",):
        np.testing.assert_array_equal(getattr(a, name)[0], getattr(b, name)[0])
    for name in STATE + ("lookahead",):
        np.testing.assert_array_equal(getattr(a, name), getattr(b, name), err_msg=name)
    assert (np.abs(a.state("mom1", 0)) < 1.0).all() and not np.array_equal(a.state("delta", 0), 0)


def test_emulated_kernel_table_needing_a_second_launch():
    n = L.ADAMAX_MAX_TENSORS + 5
    sizes = [1 + i % 3 for i in range(n)]
    assert _compare(sizes, steps=1) == 2
    assert _compare(sizes, steps=2, missing=(3, 801)) == 4


def test_eve_step_rejects_bad_arguments():
    lib = emu()
    p = np.zeros(8, np.float32)
    st = np.zeros(8, np.float32)
    ptr = lambda a, off=0: a.ctypes.data + off

    def call(entries, n=None, state=True, bad_state=None, lr=0.002, beta1=0.1, beta3=0.01, grad_scale=1.0):
        t = (L.AdamaxTensor * max(len(entries), 1))()
        for e, (param, grad, numel, offset) in zip(t, entries):
            e.param, e.grad, e.numel, e.offset = param, grad, numel, offset
        s = [C.c_void_p(ptr(st)) if state else None] * 5
        if bad_state is not None:
            s[bad_state[0]] = bad_state[1]
        return lib.iaf_eve_step(t, len(entries) if n is None else n, *s, lr, beta1, 0.001, beta3, grad_scale, None)

    good = (ptr(p), ptr(p), 8, 0)
    before = lib.iaf_adamax_launch_count()
    assert call([good], n=-1) == L.ERR_BAD_ARG
    assert call([good], state=False) == L.ERR_BAD_ARG
    for i in range(5):                                         # each state buffer: NULL, or not 4-byte aligned
        assert call([good], bad_state=(i, None)) == L.ERR_BAD_ARG
        assert call([good], bad_state=(i, C.c_void_p(ptr(st, 2)))) == L.ERR_BAD_ARG
    assert call([(None, ptr(p), 8, 0)]) == L.ERR_BAD_ARG
    assert call([(ptr(p), ptr(p), 0, 0)]) == L.ERR_BAD_ARG
    assert call([(ptr(p), ptr(p), 8, -1)]) == L.ERR_BAD_ARG
    assert call([(ptr(p, 2), ptr(p), 4, 0)]) == L.ERR_BAD_ARG    # not 4-byte aligned
    assert call([(ptr(p), ptr(p, 1), 4, 0)]) == L.ERR_BAD_ARG
    assert call([good], lr=math.nan) == L.ERR_BAD_ARG
    assert call([good], beta3=math.inf) == L.ERR_BAD_ARG
    assert call([good], grad_scale=math.inf) == L.ERR_BAD_ARG
    assert call([good], beta1=0.0) == L.ERR_BAD_ARG              # the lookahead's (1 - b1) / b1
    assert call([good, (None, None, 1, 0)]) == L.ERR_BAD_ARG       # a bad entry anywhere: nothing launched
    assert call([], n=0) == L.OK
    assert lib.iaf_adamax_launch_count() == before
    np.testing.assert_array_equal(p, 0.0)
    np.testing.assert_array_equal(st, 0.0)


def test_library_without_the_kernel_checks_then_refuses():
    """The C ABI built without iaf_optim.cu (tests/emu/build_emu.py's library) still validates the arguments, and then
    refuses a valid call with IAF_ERR_UNSUPPORTED instead of launching anything."""
    lib = harness.emu()
    p = np.zeros(8, np.float32)
    t = (L.AdamaxTensor * 1)()
    t[0].param, t[0].grad, t[0].numel, t[0].offset = p.ctypes.data, p.ctypes.data, 8, 0
    s = [C.c_void_p(np.zeros(8, np.float32).ctypes.data)] * 5
    before = lib.iaf_adamax_launch_count()
    assert lib.iaf_eve_step(t, 1, *s, 0.002, 0.1, 0.001, 0.01, 1.0, None) == L.ERR_UNSUPPORTED
    assert lib.iaf_eve_step(t, 1, *s, 0.002, 0.0, 0.001, 0.01, 1.0, None) == L.ERR_BAD_ARG
    t[0].numel = 0
    assert lib.iaf_eve_step(t, 1, *s, 0.002, 0.1, 0.001, 0.01, 1.0, None) == L.ERR_BAD_ARG
    assert lib.iaf_adamax_launch_count() == before
    np.testing.assert_array_equal(p, 0.0)


# ---------------------------------------------------------------------------------------------------------------------
# the Python side
def test_optimizer_refuses_what_it_cannot_take():
    with pytest.raises(ValueError, match="CUDA"):
        Eve({"w": torch.zeros(3)})
    with pytest.raises(ValueError, match="non-empty"):
        Eve({})
    with pytest.raises(ValueError):
        Eve([torch.zeros(3)])
    with pytest.raises(ValueError, match="beta1"):
        Eve({"w": torch.zeros(3)}, beta1=0.0)


def test_make_optimizer_maps_cvae1s_arguments(monkeypatch):
    made = []
    monkeypatch.setattr(optim, "Adamax", lambda w, **kw: made.append(("adamax", kw)) or "adamax")
    monkeypatch.setattr(optim, "Eve", lambda w, **kw: made.append(("eve", kw)) or "eve")
    w = {"w": torch.zeros(3)}
    assert elbo_theano.make_optimizer(w, dict(n_z=4)) == "adamax"
    assert elbo_theano.make_optimizer(w, dict(optim="adamax", alpha=0.003)) == "adamax"
    assert elbo_theano.make_optimizer(w, dict(optim="eve", alpha=0.001, beta1=0.2, beta2=0.01)) == "eve"
    assert made == [("adamax", dict(rule="theano", lr=None, beta1=None, beta2=None)),
                    ("adamax", dict(rule="theano", lr=0.003, beta1=None, beta2=None)),
                    ("eve", dict(lr=0.001, beta1=0.2, beta2=0.01))]
    with pytest.raises(ValueError, match="unknown optim"):
        elbo_theano.make_optimizer(w, dict(optim="adam"))


TF_HPS = dict(z_size=4, h_size=8, depth=2, num_blocks=1, kl_min=0.1, image_size=8)
TH_HPS = dict(n_z=4, n_h1=4, n_h2=8, depths=[1, 1], depth_ar=1, nl="elu", kl_min=0.1, image_size=8)


def _theano_model(seed=2):
    return {k: torch.from_numpy(np.asarray(v, np.float64)) for k, v in elbo_theano.make_params(TH_HPS, seed=seed).items()}


def _batch(B):
    S = TH_HPS["image_size"]
    g = torch.Generator().manual_seed(5)
    x = torch.randint(0, 256, (B, 3, S, S), generator=g, dtype=torch.uint8)
    noise = {(i, 0): torch.randn((B, TH_HPS["n_z"], S // 2 ** (i + 1), S // 2 ** (i + 1)), generator=g,
                                 dtype=torch.float64) for i in range(2)}
    return x, noise


def test_tf_train_step_refuses_eve():
    from oracle.elbo_oracle import TorchIAF
    p = {k: torch.from_numpy(np.asarray(v, np.float64)).requires_grad_() for k, v in
         elbo.make_params(TF_HPS, seed=2).items()}
    x = torch.zeros((2, 3, 8, 8), dtype=torch.uint8)
    with pytest.raises(ValueError, match="Adamax only"):
        elbo.train_step(p, x, RestatedEve(p), TF_HPS, iaf_layer=TorchIAF(p, TF_HPS))


def test_theano_train_step_refuses_a_layer_not_on_the_lookahead():
    from oracle.elbo_oracle import TorchIAFTheano
    w = _theano_model()
    opt = RestatedEve(w)
    x, noise = _batch(2)
    with pytest.raises(ValueError, match="lookahead"):
        elbo_theano.train_step(w, x, opt, TH_HPS, noise=noise, iaf_layer=TorchIAFTheano(w, TH_HPS))


def test_theano_train_step_with_eve_takes_the_mean_at_the_lookahead():
    """One process, fp64: train_step differentiates mean(cost) at opt.lookahead() and returns the bits/dim there; with
    Adamax it still differentiates the sum at w."""
    from oracle.elbo_oracle import TorchIAFTheano
    x, noise = _batch(3)
    w, v = _theano_model(), _theano_model()
    opt, ref = RestatedEve(w), RestatedEve(v)
    for _ in range(3):
        bpd = elbo_theano.train_step(w, x, opt, TH_HPS, noise=noise, iaf_layer=TorchIAFTheano(opt.lookahead(), TH_HPS))
        la = ref.lookahead()
        for t in la.values():
            t.grad = None
        out = elbo_theano.forward(la, x, noise, TorchIAFTheano(la, TH_HPS), TH_HPS)
        out["cost"].mean().backward()
        ref.step()
        assert abs(float(bpd) - float(out["bits_per_dim"].detach())) <= 1e-14 * abs(float(bpd))
    for k in w:
        np.testing.assert_allclose(w[k].numpy(), v[k].numpy(), rtol=1e-12, atol=1e-15, err_msg=k)
    # the Adamax path is untouched: the sum's gradient at w
    wa = {k: t.clone().requires_grad_() for k, t in _theano_model().items()}
    va = {k: t.clone().requires_grad_() for k, t in _theano_model().items()}
    oa, ra = RestatedAdamax(wa, "theano"), RestatedAdamax(va, "theano")
    elbo_theano.train_step(wa, x, oa, TH_HPS, noise=noise, iaf_layer=TorchIAFTheano(wa, TH_HPS))
    elbo_theano.forward(va, x, noise, TorchIAFTheano(va, TH_HPS), TH_HPS)["cost"].sum().backward()
    ra.step()
    for k in wa:
        np.testing.assert_array_equal(wa[k].detach().numpy(), va[k].detach().numpy(), err_msg=k)


# ---------------------------------------------------------------------------------------------------------------------
# sharded train_step
def _sharded_worker(rank, world, port, B, out):
    from oracle.elbo_oracle import TorchIAFTheano
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        w = _theano_model()
        x, noise = _batch(B)
        opt = RestatedEve(w)
        layer = TorchIAFTheano(opt.lookahead(), TH_HPS)
        bpd = [float(elbo_theano.train_step(w, x, opt, TH_HPS, noise=noise, iaf_layer=layer, sharded=True))
               for _ in range(2)]
        if rank == 0:
            torch.save((dict(w), opt.averaged(), {k: v.detach() for k, v in opt.lookahead().items()}, bpd), out)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("B", [4, 5], ids=["even", "uneven"])
def test_sharded_train_step_equals_towers_in_one_process(B, tmp_path):
    """Each rank takes its contiguous rows; the gradients averaged over the ranks are those of the global batch's mean
    cost at the lookahead, for any shard sizes.  One process summing both towers' costs, dividing by B and stepping
    once must give the same parameters, averages, lookahead and bits/dim (fp64, oracle iaf_layer)."""
    from oracle.elbo_oracle import TorchIAFTheano
    from iaf_b200.parallel import shard_range
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    out = str(tmp_path / "rank0.pt")
    mp.spawn(_sharded_worker, args=(2, port, B, out), nprocs=2, join=True)
    got_w, got_avg, got_la, got_bpd = torch.load(out)

    w = _theano_model()
    x, noise = _batch(B)
    opt = RestatedEve(w)
    for _ in range(2):
        la = opt.lookahead()
        layer = TorchIAFTheano(la, TH_HPS)
        for t in la.values():
            t.grad = None
        total, bpd = 0.0, 0.0
        for r in range(2):
            lo, hi = shard_range(B, r, 2)
            o = elbo_theano.forward(la, x[lo:hi], {k: v[lo:hi] for k, v in noise.items()}, layer, TH_HPS)
            total = total + o["cost"].sum()
            bpd = bpd + float(o["bits_per_dim"].detach()) * (hi - lo) / B
        (total / B).backward()
        opt.step()
    for name, got, want in (("param", got_w, w), ("avg", got_avg, opt.averaged()), ("lookahead", got_la, opt.lookahead())):
        for k in want:
            np.testing.assert_allclose(got[k].numpy(), want[k].detach().numpy(), rtol=1e-12, atol=1e-14,
                                       err_msg="%s %s" % (name, k))
    assert abs(got_bpd[1] - bpd) < 1e-12 * abs(bpd)
