"""CPU checks of the reference's Adamax rules and weight averages (iaf_b200.optim, iaf_adamax_step):

* the op-by-op fp32 restatement (tests/adamax_oracle.py) reproduces tests/golden/optim.npz, the trajectories of the
  reference's own update code, bit for bit;
* the kernel, run under the host emulation (tests/emu), is bit-identical to the restatement for both rules: tensor
  sizes around the 4096-element tile, views at odd storage offsets, missing gradients, a gradient scale, and a table
  that needs a second launch;
* the C entry refuses bad arguments with its status codes, and the Python optimiser refuses what it cannot take;
* a 2-rank gloo sharded ``train_step`` of either model equals one process running the same two towers.
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
from iaf_b200.optim import DEFAULTS, Adamax
from tests.adamax_oracle import RestatedAdamax
from tests.emu import harness
from tests.emu.optim import emu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "optim.npz")
NAMES = ("a", "b", "c")


# ---------------------------------------------------------------------------------------------------------------------
# the restatement against the reference's own trajectories
@pytest.mark.parametrize("rule", ["tf", "theano"])
def test_restatement_matches_reference_trajectory(rule):
    f = np.load(GOLDEN)
    params = {k: torch.from_numpy(f["param0/" + k].copy()) for k in NAMES}
    opt = RestatedAdamax(params, rule)
    for t in range(f["has_c"].shape[0]):
        grads = {k: torch.from_numpy(f["grads/" + k][t].copy()) for k in NAMES}
        if not f["has_c"][t]:
            grads["c"] = None
        opt.step(grads=grads)
        flat = lambda d: np.concatenate([d[k].numpy().ravel() for k in NAMES])
        for name, got in (("param", flat(params)), ("mom1", flat(opt.mom1)), ("mom_max", flat(opt.mom_max)),
                          ("avg", flat(opt.avg))):
            np.testing.assert_array_equal(got, f["%s/%s" % (rule, name)][t], err_msg="%s %s step %d" % (rule, name, t))


def test_golden_sequence_covers_the_edges():
    f = np.load(GOLDEN)
    g = np.concatenate([f["grads/" + k].reshape(30, -1) for k in NAMES], axis=1)
    assert (g[3] == 0).all() and (g == 0).any(axis=0).all()
    live = g[10:13] != 0
    assert np.isclose(np.abs(g[10:13][live]), 1e-30, rtol=1e-6).all() and (np.abs(g[20][g[20] != 0]) == 1e4).all()
    assert (np.sign(g[8]) == -np.sign(g[7]))[(g[7] != 0) & (g[8] != 0)].all()
    assert not f["has_c"].all()


# ---------------------------------------------------------------------------------------------------------------------
# the kernel under the host emulation
class EmuSet(object):
    """A parameter set in numpy buffers, stepped by the emulated iaf_adamax_step.  ``shift``: each parameter and gradient
    is a view one float into its buffer (an odd storage offset, 4-byte aligned only); state slices start at odd
    offsets then too."""

    def __init__(self, params, rule, shift=0, **hp):
        self.rule, self.shift = rule, shift
        d = dict(DEFAULTS[rule])
        d.update({k: v for k, v in hp.items() if v is not None})
        if d["avg_decay"] is None:
            d["avg_decay"] = 1.0 - d["beta2"]
        self.hp = d
        self.bufs = [np.zeros(p.size + shift, np.float32) for p in params]
        self.params = [b[shift:] for b in self.bufs]
        for dst, p in zip(self.params, params):
            dst[...] = p.ravel()
        self.offsets, total = [], 0
        for p in params:
            self.offsets.append(total + shift)
            total += p.size + shift if shift else -(-p.size // 4) * 4   # aligned: slices on 16-byte boundaries
        self.mom1 = np.zeros(total, np.float32)
        self.mom_max = np.full(total, 1e-8 if rule == "theano" else 0.0, np.float32)
        self.avg = np.zeros(total, np.float32)
        for p, off in zip(self.params, self.offsets):
            self.avg[off:off + p.size] = p
        self.gbufs = [np.zeros(p.size + shift, np.float32) for p in params]

    def table(self, grads):
        t = (L.AdamaxTensor * len(self.params))()
        for e, p, gb, g, off in zip(t, self.params, self.gbufs, grads, self.offsets):
            e.param, e.numel, e.offset = p.ctypes.data, p.size, off
            if g is not None:
                gb[self.shift:] = g.ravel()
                e.grad = gb.ctypes.data + 4 * self.shift
        return t

    def step(self, grads, grad_scale=1.0, rule=None):
        t = self.table(grads)
        h = self.hp
        return emu().iaf_adamax_step(L.ADAMAX_RULES[self.rule] if rule is None else rule, t, len(t),
                                     C.c_void_p(self.mom1.ctypes.data), C.c_void_p(self.mom_max.ctypes.data),
                                     C.c_void_p(self.avg.ctypes.data), h["lr"], h["beta1"], h["beta2"],
                                     h["avg_decay"], grad_scale, None)

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


def _compare(rule, sizes, shift=0, steps=4, missing=(), grad_scale=1.0, seed=0, **hp):
    rng = np.random.RandomState(seed)
    p0 = [(0.3 * rng.randn(n)).astype(np.float32) for n in sizes]
    es = EmuSet(p0, rule, shift, **hp)
    tp = {str(i): torch.from_numpy(p.copy()) for i, p in enumerate(p0)}
    ref = RestatedAdamax(tp, rule, **hp)
    before = emu().iaf_adamax_launch_count()
    for s in range(steps):
        gs = _grads(rng, sizes, s, missing)
        assert es.step(gs, grad_scale) == 0
        ref.step(grad_scale, grads={str(i): None if g is None else torch.from_numpy(g) for i, g in enumerate(gs)})
    for i in range(len(sizes)):
        k = str(i)
        np.testing.assert_array_equal(es.params[i], tp[k].numpy(), err_msg="param %d" % i)
        np.testing.assert_array_equal(es.state("avg", i), ref.avg[k].numpy(), err_msg="avg %d" % i)
        np.testing.assert_array_equal(es.state("mom1", i), ref.mom1[k].numpy(), err_msg="mom1 %d" % i)
        np.testing.assert_array_equal(es.state("mom_max", i), ref.mom_max[k].numpy(), err_msg="max %d" % i)
    return emu().iaf_adamax_launch_count() - before


@pytest.mark.parametrize("rule", ["tf", "theano"])
@pytest.mark.parametrize("shift", [0, 1], ids=["aligned", "odd_offset"])
def test_emulated_kernel_equals_restatement(rule, shift):
    launches = _compare(rule, [1, 3, 4095, 4096, 4097, 9000], shift=shift, missing=(1, 4))
    assert launches == 4


@pytest.mark.parametrize("rule", ["tf", "theano"])
def test_emulated_kernel_grad_scale_and_hyperparameters(rule):
    _compare(rule, [7, 4100], grad_scale=0.5, lr=0.003, beta1=0.8 if rule == "tf" else 0.2, beta2=0.99 if rule == "tf"
             else 0.01, avg_decay=0.9, seed=1)


@pytest.mark.parametrize("rule", ["tf", "theano"])
def test_emulated_kernel_missing_gradient(rule):
    """TF skips the tensor (apply_gradients with a None gradient) but moves its average; Theano steps it with zero."""
    p0 = [np.linspace(-1, 1, 6).astype(np.float32)]
    es = EmuSet(p0, rule)
    assert es.step([np.ones(6, np.float32)]) == 0
    p1, m1, mx, a1 = es.params[0].copy(), es.mom1.copy(), es.mom_max.copy(), es.avg.copy()
    assert es.step([None]) == 0
    if rule == "tf":
        np.testing.assert_array_equal(es.params[0], p1)
        np.testing.assert_array_equal(es.mom1, m1)
        np.testing.assert_array_equal(es.mom_max, mx)
    else:
        assert not np.array_equal(es.params[0], p1) and (np.abs(es.state("mom1", 0)) < np.abs(m1[:6])).all()
    assert not np.array_equal(es.avg, a1)


def test_emulated_kernel_table_needing_a_second_launch():
    n = L.ADAMAX_MAX_TENSORS + 5
    sizes = [1 + i % 3 for i in range(n)]
    assert _compare("tf", sizes, steps=1) == 2
    assert _compare("theano", sizes, steps=2, missing=(3, 801)) == 4


def test_adamax_step_rejects_bad_arguments():
    lib = emu()
    p = np.zeros(8, np.float32)
    st = np.zeros(8, np.float32)
    ptr = lambda a, off=0: a.ctypes.data + off

    def call(entries, rule=0, n=None, state=True, lr=0.01, grad_scale=1.0):
        t = (L.AdamaxTensor * max(len(entries), 1))()
        for e, (param, grad, numel, offset) in zip(t, entries):
            e.param, e.grad, e.numel, e.offset = param, grad, numel, offset
        s = C.c_void_p(ptr(st)) if state else None
        return lib.iaf_adamax_step(rule, t, len(entries) if n is None else n, s, s, s, lr, 0.9, 0.999, 0.999,
                                   grad_scale, None)

    good = (ptr(p), ptr(p), 8, 0)
    before = lib.iaf_adamax_launch_count()
    assert call([good], rule=2) == L.ERR_UNSUPPORTED
    assert call([good], n=-1) == L.ERR_BAD_ARG
    assert call([good], state=False) == L.ERR_BAD_ARG
    assert call([(None, ptr(p), 8, 0)]) == L.ERR_BAD_ARG
    assert call([(ptr(p), ptr(p), 0, 0)]) == L.ERR_BAD_ARG
    assert call([(ptr(p), ptr(p), 8, -1)]) == L.ERR_BAD_ARG
    assert call([(ptr(p, 2), ptr(p), 4, 0)]) == L.ERR_BAD_ARG    # not 4-byte aligned
    assert call([(ptr(p), ptr(p, 1), 4, 0)]) == L.ERR_BAD_ARG
    assert call([good], lr=math.nan) == L.ERR_BAD_ARG
    assert call([good], grad_scale=math.inf) == L.ERR_BAD_ARG
    assert call([good, (None, None, 1, 0)]) == L.ERR_BAD_ARG       # a bad entry anywhere: nothing launched
    assert call([], n=0) == L.OK
    assert lib.iaf_adamax_launch_count() == before


def test_library_without_the_kernel_checks_then_refuses():
    """The C ABI built without iaf_optim.cu (tests/emu/build_emu.py's library) still validates the arguments, and then
    refuses a valid call with IAF_ERR_UNSUPPORTED instead of launching anything."""
    lib = harness.emu()
    p = np.zeros(8, np.float32)
    t = (L.AdamaxTensor * 1)()
    t[0].param, t[0].grad, t[0].numel, t[0].offset = p.ctypes.data, p.ctypes.data, 8, 0
    s = C.c_void_p(np.zeros(8, np.float32).ctypes.data)
    before = lib.iaf_adamax_launch_count()
    assert lib.iaf_adamax_step(0, t, 1, s, s, s, 0.01, 0.9, 0.999, 0.999, 1.0, None) == L.ERR_UNSUPPORTED
    t[0].numel = 0
    assert lib.iaf_adamax_step(0, t, 1, s, s, s, 0.01, 0.9, 0.999, 0.999, 1.0, None) == L.ERR_BAD_ARG
    assert lib.iaf_adamax_launch_count() == before
    np.testing.assert_array_equal(p, 0.0)


def test_optimizer_refuses_what_it_cannot_take():
    cpu = {"w": torch.zeros(3)}
    with pytest.raises(ValueError, match="unknown rule"):
        Adamax(cpu, rule="adam")
    with pytest.raises(ValueError, match="CUDA"):
        Adamax(cpu)
    with pytest.raises(ValueError):
        Adamax({})
    with pytest.raises(ValueError):
        Adamax([torch.zeros(3)])


# ---------------------------------------------------------------------------------------------------------------------
# sharded train_step
TF_HPS = dict(z_size=4, h_size=8, depth=2, num_blocks=1, kl_min=0.1, image_size=8)
TH_HPS = dict(n_z=4, n_h1=4, n_h2=8, depths=[1, 1], depth_ar=1, nl="elu", kl_min=0.1, image_size=8)
B = 4


def _model(which):
    from oracle.elbo_oracle import TorchIAF, TorchIAFTheano
    if which == "tf":
        p = {k: torch.from_numpy(np.asarray(v, np.float64)).requires_grad_() for k, v in
             elbo.make_params(TF_HPS, seed=2).items()}
        shapes = elbo._noise_shapes(TF_HPS, B)
        return p, TF_HPS, TorchIAF(p, TF_HPS), shapes, elbo
    w = {k: torch.from_numpy(np.asarray(v, np.float64)).requires_grad_() for k, v in
         elbo_theano.make_params(TH_HPS, seed=2).items()}
    S = TH_HPS["image_size"]
    shapes = {(i, 0): (B, TH_HPS["n_z"], S // 2 ** (i + 1), S // 2 ** (i + 1)) for i in range(2)}
    return w, TH_HPS, TorchIAFTheano(w, TH_HPS), shapes, elbo_theano


def _batch(shapes):
    g = torch.Generator().manual_seed(5)
    x = torch.randint(0, 256, (B, 3, 8, 8), generator=g, dtype=torch.uint8)
    noise = {k: torch.randn(s, generator=g, dtype=torch.float64) for k, s in sorted(shapes.items())}
    return x, noise


def _sharded_worker(rank, world, port, which, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        p, hps, layer, shapes, mod = _model(which)
        x, noise = _batch(shapes)
        opt = RestatedAdamax(p, which)
        bpd = [float(mod.train_step(p, x, opt, hps, noise=noise, iaf_layer=layer, sharded=True)) for _ in range(2)]
        if rank == 0:
            torch.save(({k: v.detach() for k, v in p.items()}, {k: v for k, v in opt.averaged().items()}, bpd), out)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("which", ["tf", "theano"])
def test_sharded_train_step_equals_two_towers_in_one_process(which, tmp_path):
    """Each rank is one tower (tf_train.py:126-147): its half of the batch, its own free-bits batch mean, and the
    towers' gradients averaged (average_grads).  One process running both towers, summing their objectives and
    stepping with grad_scale 1/2, must give the same parameters, averages and bits/dim (fp64, oracle iaf_layer)."""
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    out = str(tmp_path / "rank0.pt")
    mp.spawn(_sharded_worker, args=(2, port, which, out), nprocs=2, join=True)
    got_p, got_avg, got_bpd = torch.load(out)

    p, hps, layer, shapes, mod = _model(which)
    x, noise = _batch(shapes)
    opt = RestatedAdamax(p, which)
    for _ in range(2):
        for t in p.values():
            t.grad = None
        obj, bpd = 0.0, 0.0
        for lo, hi in ((0, B // 2), (B // 2, B)):
            o = mod.forward(p, x[lo:hi], {k: v[lo:hi] for k, v in noise.items()}, layer, hps)
            obj = obj + (o["obj"] if which == "tf" else o["cost"].sum())
            bpd = bpd + float(o["bits_per_dim"].detach()) / 2
        obj.backward()
        opt.step(grad_scale=0.5)
    for k in p:
        np.testing.assert_allclose(got_p[k].numpy(), p[k].detach().numpy(), rtol=1e-12, atol=1e-14, err_msg=k)
        np.testing.assert_allclose(got_avg[k].numpy(), opt.averaged()[k].numpy(), rtol=1e-12, atol=1e-14, err_msg=k)
    assert abs(got_bpd[1] - bpd) < 1e-12 * abs(bpd)


def test_every_readme_model_fits_one_launch():
    """The table of the largest parameter set the README runs (the TF eval model: depth 1, num_blocks 20) fits in one
    launch's parameter space."""
    n = len(elbo.make_params(dict(z_size=32, h_size=160, depth=1, num_blocks=20, kl_min=0.0, image_size=32)))
    assert n <= L.ADAMAX_MAX_TENSORS
