"""The operator under CUDA-graph capture, on side streams, and with one plan's scratch shared by every entry point.

bench.py measures the step as graph replays captured on a side stream, and a training loop may capture its whole step;
the tests in test_gpu_tc_envelope.py and test_gpu_backward.py only make eager calls on the default stream.  Here every
test runs on three plans (one-launch tensor-core step, per-stage tensor-core step, exact-fp32 SIMT step) and asserts
where it ran (``path_used`` / ``backward_path`` / the ``launch_count`` change).  It covers:

* replays of captured forwards and training pairs, bit-equal to eager calls and within tolerance of the fp64 oracle,
  also after the inputs are overwritten in place (a graph reads its inputs live);
* a whole training step (forward, backward, SGD update, and the re-pack inside the autograd node) in one graph;
* a fresh operator whose first calls (plan, packing, scratch, backward plan) run on a side stream while the default
  stream is busy, over memory that was filled with 0xFF bytes: scratch zero-fills must be ordered on the caller's stream;
* two side streams sharing one operator without caller synchronisation;
* scratch sized by one entry point and batch size and reused by another;
* the refusals that keep graphs valid: no allocation inside a capture, no re-allocation after one.  Nothing is replayed
  unless the refusal held, so no replay ever touches freed memory.

Tolerances: forward ``|d|_inf / max(|ref|_inf, 1) <= 1e-4`` (per sample for per-sample sums), backward
``|d|_inf / |ref|_inf <= 1e-4`` per tensor."""
import collections
import math

import numpy as np
import pytest
import torch

from oracle import iaf_oracle as O
from oracle import iaf_oracle_torch as OT

pytestmark = pytest.mark.gpu
TOL = 1e-4
DEV = "cuda:0"
N_Z = 32
REFUSED = "largest batch size"  # in the message of every capture refusal

Plan = collections.namedtuple("Plan", "variant hidden H W path fwd_path launches bwd_path")
PLANS = {
    "one-launch": Plan("tf", [64], 16, 16, "auto", "tc", 1, "tc"),
    "per-stage": Plan("theano", [64, 64], 8, 8, "auto", "tc", 3, "tc"),
    "simt": Plan("tf", [64], 16, 16, "simt", "simt", 1, "simt"),
}
plans = pytest.mark.parametrize("plan", list(PLANS))


# ---------------------------------------------------------------------------------------------------------------------
# helpers
# ---------------------------------------------------------------------------------------------------------------------
def _np(t):
    return t.detach().double().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t, dtype=np.float64)


def fwd_err(a, ref):
    a, ref = _np(a), _np(ref)
    assert np.isfinite(a).all()
    return float(np.abs(a - ref).max() / max(np.abs(ref).max(), 1.0))


def per_sample_fwd_err(a, ref):
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


def _keys(variant):
    return ("V", "g", "b") if variant == "tf" else ("w", "s", "b")


def _mask(variant, w, zerodiag):
    if variant == "tf":
        return O.get_conv_ar_mask(3, 3, w.shape[2], w.shape[3], zerodiag)
    return O.theano_conv_ar_mask(w.shape[1] - 1, w.shape[0], (3, 3), zerodiag)


def _d(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _leaf(t):
    return t.detach().clone().requires_grad_(True)


def _flat(grads):
    """(g_z, g_context, [g_w], [g_scale], [g_bias]) of IAFOperator._backward -> one list of tensors."""
    g_z, g_ctx, gw, gs, gb = grads
    return [g_z, g_ctx] + [t for i in range(len(gw)) for t in (gw[i], gs[i], gb[i])]


class Case(object):
    """One operator of plan ``name`` with the oracle's parameters.  ``masked``: the weights' masked taps start at zero
    (as the reference initialises them), so that a training step can be checked to keep them there."""

    def __init__(self, name, grad=False, masked=False, seed=1):
        from iaf_b200 import IAFOperator
        self.name, self.p = name, PLANS[name]
        p = self.p
        self.hid, self.hd = O.make_params(p.variant, N_Z, p.hidden, [N_Z, N_Z], seed=seed)
        if masked:
            k = _keys(p.variant)[0]
            for i, l in enumerate(self.hid + self.hd):
                l[k] = (l[k] * _mask(p.variant, l[k], i >= len(p.hidden))).astype(np.float32)
        self.dev = [tuple(_d(l[k]).requires_grad_(grad) for k in _keys(p.variant)) for l in self.hid + self.hd]
        self.params = [t for l in self.dev for t in l]
        self.op = IAFOperator(p.variant, N_Z, p.hidden, [N_Z, N_Z], nl="elu", path=p.path).set_weights(self.dev)

    def step_inputs(self, B, seed):
        z, ctx = O.make_inputs(B, N_Z, self.p.hidden[0], self.p.H, self.p.W, seed=seed)
        return [_d(z), _d(ctx)]

    def layer_inputs(self, B, seed):
        rng = np.random.RandomState(seed)
        shp = (B, N_Z, self.p.H, self.p.W)
        eps, pm, prm = (rng.randn(*shp).astype(np.float32) for _ in range(3))
        pls, prl = ((0.3 * rng.randn(*shp)).astype(np.float32) for _ in range(2))
        ctx = (0.1 * rng.randn(B, self.p.hidden[0], self.p.H, self.p.W)).astype(np.float32)
        return [_d(a) for a in (eps, pm, pls, prm, prl, ctx)]

    def inputs(self, entry, B, seed):
        return self.layer_inputs(B, seed) if entry.startswith("layer") else self.step_inputs(B, seed)

    def step_grads(self, B, seed):
        r = np.random.RandomState(seed)
        shp = (B, N_Z, self.p.H, self.p.W)
        return [_d(r.randn(*shp).astype(np.float32)), _d(r.randn(*shp).astype(np.float32)), _d(r.randn(B).astype(np.float32))]

    def layer_grads(self, B, seed):
        r = np.random.RandomState(seed)
        shp = (B, N_Z, self.p.H, self.p.W)
        return [_d(r.randn(*shp).astype(np.float32)), _d(r.randn(*shp).astype(np.float32)),
                _d(r.randn(B, N_Z).astype(np.float32)), _d(r.randn(B).astype(np.float32))]

    def assert_paths(self, entries=("step", "multiconv", "layer"), backward=False):
        p = self.p
        for e in entries:
            assert self.op.path_used(p.H, p.W, DEV, entry=e) == p.fwd_path, e
        if backward:
            assert self.op.backward_path(p.H, p.W, DEV) == p.bwd_path

    # ---- fp64 references --------------------------------------------------------------------------------------
    def f64_layers(self, grad=False):
        th = OT.to_torch(O.cast_params(self.hid, np.float64), torch.float64)
        thh = OT.to_torch(O.cast_params(self.hd, np.float64), torch.float64)
        for l in th + thh:
            for t in l.values():
                t.requires_grad_(grad)
        return th, thh

    def layer_ref(self, th, thh, eps, pm, pls, prm, prl, ctx):
        c = 0.5 * math.log(2.0 * math.pi)
        z0 = pm + torch.exp(pls) * eps
        zn, lsd, _ = OT.iaf_step(self.p.variant, z0, ctx, th, thh)
        kl = (-c - pls - 0.5 * eps * eps + lsd) - (-c - prl - 0.5 * (zn - prm) ** 2 * torch.exp(-2.0 * prl))
        return [zn, kl, kl.sum(dim=(2, 3)), kl.sum(dim=(1, 2, 3))]

    def check_forward(self, entry, ins, outs):
        """Outputs of one forward call of ``entry`` against the fp64 oracle."""
        th, thh = self.f64_layers()
        x = [torch.from_numpy(_np(t)) for t in ins]
        if entry.startswith("step"):
            zn, lsd, ld = OT.iaf_step(self.p.variant, x[0], x[1], th, thh)
            assert fwd_err(outs[0], zn) < TOL
            if entry == "step":
                assert fwd_err(outs[1], lsd) < TOL
                assert per_sample_fwd_err(outs[2][:, None], ld[:, None]) < TOL
        elif entry == "multiconv":
            for o, r in zip(outs, OT.multiconv(self.p.variant, x[0], x[1], th, thh)):
                assert fwd_err(o, r) < TOL
        else:
            zn, kl, bc, cost = self.layer_ref(th, thh, *x)
            assert fwd_err(outs[0], zn) < TOL and fwd_err(outs[1], kl) < TOL
            assert per_sample_fwd_err(outs[2], bc) < TOL
            assert per_sample_fwd_err(outs[3][:, None], cost[:, None]) < TOL

    def check_backward(self, entry, ins, g_up, got):
        """Gradients ``got`` (inputs in ``ins`` order, then every raw parameter in (w, scale, bias) order) of the loss
        sum(output * upstream gradient) of ``entry`` against fp64 autograd over the oracle."""
        th, thh = self.f64_layers(True)
        x = [torch.from_numpy(_np(t)).requires_grad_(True) for t in ins]
        u = [torch.from_numpy(_np(g)) for g in g_up]
        if entry == "step":
            outs = OT.iaf_step(self.p.variant, x[0], x[1], th, thh)
        elif entry == "multiconv":
            outs = OT.multiconv(self.p.variant, x[0], x[1], th, thh)
        else:
            outs = self.layer_ref(th, thh, *x)
        sum((o * g).sum() for o, g in zip(outs, u)).backward()
        refs = [t.grad for t in x] + [l[k].grad for l in th + thh for k in _keys(self.p.variant)]
        assert len(got) == len(refs)
        for i, (g, r) in enumerate(zip(got, refs)):
            assert bwd_err(g, r) < TOL, i


def capture(fn):
    """bench.py's pattern: a fresh side stream that waits for the current one, ``fn`` captured on it, then the current
    stream waits for it.  Returns (graph, what fn returned, the capture stream)."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            out = fn()
    torch.cuda.current_stream().wait_stream(s)
    return g, out, s


def _assert_equal(got, want):
    assert len(got) == len(want)
    for i, (a, b) in enumerate(zip(got, want)):
        assert torch.equal(a, b), i


def _forward(op, entry, ins):
    if entry == "step":
        return list(op.step(*ins))
    if entry == "step-null":
        out = op.step(*ins, want_logsd=False, want_logdet=False)
        assert out[1] is None and out[2] is None
        return [out[0]]
    if entry == "multiconv":
        return list(op.multiconv(*ins))
    return list(op.layer(*ins))


# ---------------------------------------------------------------------------------------------------------------------
# 1. graph replay of each forward entry point
# ---------------------------------------------------------------------------------------------------------------------
SUMMED = {"step": 2, "step-null": 0, "multiconv": 1, "layer": 3}  # the output the graph sums: log-dets, z', s, kl_cost


@pytest.mark.parametrize("entry", list(SUMMED))
@plans
def test_graph_replay_matches_eager_and_oracle(plan, entry):
    """Three back-to-back calls over three static input sets and a torch.sum of their log-dets, captured on a side
    stream after an eager warm-up.  Each replay is bit-equal to eager calls on the same inputs and within tolerance of
    the oracle, also after the inputs are overwritten in place."""
    c = Case(plan)
    B = 4
    base = entry.split("-")[0]
    sets = [c.inputs(base, B, seed=10 + k) for k in range(3)]
    with torch.no_grad():
        _forward(c.op, entry, sets[0])  # warm-up: plan, packed weights, scratch at B
        torch.cuda.synchronize()
        c.assert_paths((base,))
        l0 = c.op.launch_count()

        def body():
            outs = [_forward(c.op, entry, s) for s in sets]
            return outs, torch.sum(torch.cat([o[SUMMED[entry]].reshape(-1) for o in outs]))
        g, (outs, total), _ = capture(body)
        assert c.op.launch_count() - l0 == 3 * c.p.launches  # the capture went through the expected kernels
        for rnd in range(2):
            if rnd:
                for s, k in zip(sets, range(3)):
                    for t, v in zip(s, c.inputs(base, B, seed=20 + k)):
                        t.copy_(v)
            g.replay()
            torch.cuda.synchronize()
            eager = [_forward(c.op, entry, s) for s in sets]
            for o, e in zip(outs, eager):
                _assert_equal(o, e)
            assert torch.equal(total, torch.sum(torch.cat([e[SUMMED[entry]].reshape(-1) for e in eager])))
            for s, o in zip(sets, outs):
                c.check_forward(entry, s, o)


# ---------------------------------------------------------------------------------------------------------------------
# 2. captured training pairs
# ---------------------------------------------------------------------------------------------------------------------
def _training_pair(c, entry, ins, g_up):
    """What the autograd node of ``entry`` runs: the training forward (keeps the hidden activations) and the backward
    from them, with the parameter gradients.  Returns (forward outputs, gradients in Case.check_backward's order)."""
    op = c.op
    if entry == "step":
        zo, ls, ld, hidden = op._step_train_raw(*ins)
        grads = op._backward("step", ins[0], ins[1], op._layers, tuple(g_up), True, saved=(zo, ls, hidden))
        return [zo, ls, ld], _flat(grads)
    if entry == "multiconv":
        outs, hidden = op._multiconv_train_raw(*ins)
        grads = op._backward("multiconv", ins[0], ins[1], op._layers, list(g_up), True, saved=(None, None, hidden))
        return outs, _flat(grads)
    xs = [_leaf(t) for t in ins]
    outs = op.layer(*xs)
    grads = torch.autograd.grad(outs, xs + c.params, grad_outputs=list(g_up))
    return [o.detach() for o in outs], list(grads)


@pytest.mark.parametrize("entry", ["step", "multiconv", "layer"])
@plans
def test_captured_training_pair(plan, entry):
    """The forward + backward pair of each entry point's autograd node (op.layer's: the node itself) captured in one
    graph.  Replayed outputs and gradients are bit-equal to eager calls of the same operator and the gradients are within
    tolerance of fp64 autograd."""
    c = Case(plan, grad=True)
    B = 3
    ins = c.inputs(entry, B, seed=30)
    if entry == "step":
        g_up = c.step_grads(B, seed=31)
    elif entry == "multiconv":
        g_up = c.step_grads(B, seed=31)[:2]
    else:
        g_up = c.layer_grads(B, seed=31)
    _training_pair(c, entry, ins, g_up)  # warm-up: forward and backward plans and scratch at B
    torch.cuda.synchronize()
    c.assert_paths((entry,), backward=True)
    l0 = c.op.launch_count()
    g, (outs, grads), _ = capture(lambda: _training_pair(c, entry, ins, g_up))
    assert c.op.launch_count() - l0 > c.p.launches  # the training forward and a backward were captured
    for rnd in range(2):
        if rnd:
            for t, v in zip(ins, c.inputs(entry, B, seed=32)):
                t.copy_(v)
        g.replay()
        torch.cuda.synchronize()
        e_outs, e_grads = _training_pair(c, entry, ins, g_up)
        _assert_equal(outs, e_outs)
        _assert_equal(grads, e_grads)
        c.check_forward(entry, ins, outs)
        c.check_backward(entry, ins, g_up, grads)


# ---------------------------------------------------------------------------------------------------------------------
# 3. a whole training step in one graph
# ---------------------------------------------------------------------------------------------------------------------
@plans
def test_whole_training_step_in_one_graph(plan):
    """Forward through op.step's autograd node (which invalidates and re-packs the weights: captured too), backward and
    an in-place SGD update of the raw parameters, captured after a warm-up on a side stream.  Three replays leave the
    parameters bit-equal to three eager steps of a twin operator with the same history, and every masked tap of the
    weights is still exactly zero."""
    c, twin = Case(plan, grad=True, masked=True), Case(plan, grad=True, masked=True)
    B, lr = 4, 1e-4  # random upstream gradients summed over 1024 positions: a larger step diverges
    z, ctx = c.step_inputs(B, seed=40)
    g_up = c.step_grads(B, seed=41)
    c.assert_paths(("step",), backward=True)

    def train_step(case):
        for p in case.params:
            p.grad = None
        outs = case.op.step(z, ctx)
        sum((o * g).sum() for o, g in zip(outs, g_up)).backward()
        with torch.no_grad():
            for p in case.params:
                p.add_(p.grad, alpha=-lr)

    start = [p.detach().clone() for p in c.params]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            train_step(c)
    torch.cuda.current_stream().wait_stream(side)
    for _ in range(2):
        train_step(twin)
    l0 = c.op.launch_count()
    g, _, _ = capture(lambda: train_step(c))
    assert c.op.launch_count() - l0 > c.p.launches
    for _ in range(3):
        g.replay()
        train_step(twin)
    torch.cuda.synchronize()
    assert all(bool(torch.isfinite(p).all()) for p in c.params)
    _assert_equal(c.params, twin.params)
    assert not all(torch.equal(a, b) for a, b in zip(start, c.params))  # the replays did train
    for i, l in enumerate(c.dev):
        w = _np(l[0])
        assert (w[_mask(c.p.variant, w, i >= len(c.p.hidden)) == 0] == 0).all(), i


# ---------------------------------------------------------------------------------------------------------------------
# 4. side streams
# ---------------------------------------------------------------------------------------------------------------------
@plans
def test_fresh_operator_on_a_side_stream(plan):
    """Every first call of a fresh operator (plan creation, packing, forward scratch, backward plan and scratch) made on a
    new stream while the default stream is still busy, over device memory that was just filled with 0xFF bytes and
    handed back to the driver.  Scratch the kernels expect zeroed (arrival counters, the zero tile of the operand
    images) must be zero-filled on the caller's stream, or the per-sample sums come out wrong."""
    c = Case(plan, grad=True)
    B = 5
    st = c.step_inputs(B, seed=50)
    ly = c.layer_inputs(B, seed=51)
    g_up = c.step_grads(B, seed=52)
    junk = torch.empty(512 << 20, dtype=torch.uint8, device=DEV)
    junk.fill_(0xFF)
    torch.cuda.synchronize()
    del junk
    torch.cuda.empty_cache()
    s = torch.cuda.Stream()
    torch.cuda._sleep(100_000_000)  # the default stream stays busy for tens of milliseconds
    with torch.cuda.stream(s):
        with torch.no_grad():
            step = list(c.op.step(*st))
            l0 = c.op.launch_count()
            mc = list(c.op.multiconv(*st))
            launches = c.op.launch_count() - l0
            lay = list(c.op.layer(*ly))
        xs = [_leaf(t) for t in st]
        outs = c.op.step(*xs)
        sum((o * g).sum() for o, g in zip(outs, g_up)).backward()
        grads = [x.grad for x in xs] + [p.grad for p in c.params]
    s.synchronize()
    assert launches == c.p.launches
    c.assert_paths(backward=True)
    c.check_forward("step", st, step)
    c.check_forward("multiconv", st, mc)
    c.check_forward("layer", ly, lay)
    c.check_backward("step", st, g_up, grads)


@plans
def test_two_side_streams_share_one_operator(plan):
    """step, layer, multiconv and autograd backwards alternating between two side streams on one operator, with no
    synchronisation by the caller (the library orders a call after the plan's previous one).  Every result is bit-equal
    to the same sequence on the default stream."""
    B = 4

    def sequence(c, streams):
        st = [c.step_inputs(B, seed=60 + k) for k in range(6)]
        ly = [c.layer_inputs(B, seed=70 + k) for k in range(6)]
        g_st, g_ly = c.step_grads(B, seed=80), c.layer_grads(B, seed=81)
        for s in streams:
            s.wait_stream(torch.cuda.current_stream())
        res = []
        with torch.cuda.stream(streams[0 % len(streams)]), torch.no_grad():
            res += list(c.op.step(*st[0]))
        with torch.cuda.stream(streams[1 % len(streams)]), torch.no_grad():
            res += list(c.op.layer(*ly[1]))
        with torch.cuda.stream(streams[2 % len(streams)]), torch.no_grad():
            res += list(c.op.multiconv(*st[2]))
        with torch.cuda.stream(streams[3 % len(streams)]):
            xs = [_leaf(t) for t in st[3]]
            outs = c.op.step(*xs)
            res += torch.autograd.grad(outs, xs + c.params, grad_outputs=g_st)
        with torch.cuda.stream(streams[4 % len(streams)]):
            xs = [_leaf(t) for t in ly[4]]
            outs = c.op.layer(*xs)
            res += torch.autograd.grad(outs, xs + c.params, grad_outputs=g_ly)
        with torch.cuda.stream(streams[5 % len(streams)]), torch.no_grad():
            res += list(c.op.step(*st[5]))
        torch.cuda.synchronize()
        return res

    c = Case(plan, grad=True)
    got = sequence(c, [torch.cuda.Stream(), torch.cuda.Stream()])
    want = sequence(Case(plan, grad=True), [torch.cuda.current_stream()])
    _assert_equal(got, want)
    c.assert_paths(backward=True)


# ---------------------------------------------------------------------------------------------------------------------
# 5. scratch shared by the entry points across batch sizes
# ---------------------------------------------------------------------------------------------------------------------
def _entry_call(c, kind, B, seed):
    """One call of ``kind`` at batch B.  Returns (inputs, upstream gradients or None, outputs)."""
    ins = c.inputs(kind, B, seed)
    if kind == "step_backward":
        g_up = c.step_grads(B, seed + 1)
        return ins, g_up, _flat(c.op.step_backward(*ins, *g_up, need_params=True))
    if kind == "layer_backward":
        g_up = c.layer_grads(B, seed + 1)
        xs = [_leaf(t) for t in ins]
        return ins, g_up, list(torch.autograd.grad(c.op.layer(*xs), xs + c.params, grad_outputs=g_up))
    with torch.no_grad():
        return ins, None, _forward(c.op, kind, ins)


@plans
def test_scratch_reuse_across_entries_and_batch_sizes(plan):
    """One operator: step B=5, layer B=9 (growth), multiconv B=3, step_backward B=7, layer's backward B=9, step B=2.
    Arrival counters, tile partials or operand images left dirty by one entry point or batch size and read by another
    would show up against a fresh operator making the same single call.  Forward outputs are bit-equal to it; backward
    ones within 1e-5 (the weight gradient's split-K count follows the largest batch the scratch was sized for).  The
    first call of each entry point is also checked against the oracle."""
    c = Case(plan, grad=True)
    c.assert_paths(backward=True)
    seen = set()
    for k, (kind, B) in enumerate((("step", 5), ("layer", 9), ("multiconv", 3), ("step_backward", 7),
                                   ("layer_backward", 9), ("step", 2))):
        ins, g_up, got = _entry_call(c, kind, B, seed=90 + 2 * k)
        _, _, want = _entry_call(Case(plan, grad=True), kind, B, seed=90 + 2 * k)
        if g_up is None:
            _assert_equal(got, want)
        else:
            for i, (a, b) in enumerate(zip(got, want)):
                assert float((a.double() - b.double()).abs().max()) <= 1e-5 * float(b.abs().max()), (kind, i)
        if kind not in seen:
            seen.add(kind)
            if g_up is None:
                c.check_forward(kind, ins, got)
            else:
                c.check_backward(kind.split("_")[0], ins, g_up, got)


# ---------------------------------------------------------------------------------------------------------------------
# 6. capture refusals
# ---------------------------------------------------------------------------------------------------------------------
def _capture_refused(fn):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match=REFUSED):
        with torch.cuda.stream(s):
            with torch.cuda.graph(g, stream=s):
                fn()
    torch.cuda.current_stream().wait_stream(s)


@plans
def test_first_call_inside_a_capture_is_refused(plan):
    """A fresh operator's first call inside a capture would create the plan and allocate scratch (illegal while
    capturing): it raises, and the operator then works eagerly.  The same holds when the plan exists but has no
    scratch yet; the weights that capture packed were only recorded, so the eager call packs them again."""
    c = Case(plan)
    ins = c.step_inputs(4, seed=100)
    _capture_refused(lambda: c.op.step(*ins))
    assert c.op.launch_count() == 0
    with torch.no_grad():
        c.check_forward("step", ins, list(c.op.step(*ins)))
    c.assert_paths(("step",))

    c2, other = Case(plan, seed=2), Case(plan)
    c2.op.set_weights(other.dev)
    c2.assert_paths(("step",))  # the plan, with other's weights packed: no scratch yet
    c2.op.set_weights(c2.dev)   # re-bound: packed inside the refused capture, which never runs
    _capture_refused(lambda: c2.op.step(*ins))
    with torch.no_grad():
        c2.check_forward("step", ins, list(c2.op.step(*ins)))


@plans
def test_growth_after_a_capture_is_refused(plan):
    """After a capture at B = 4, an eager call at B = 8 would free scratch the graph replays into: it raises.  Only then
    is the graph replayed, and eager calls at B = 4 and B = 2 on the capture stream still match the oracle."""
    c = Case(plan)
    z4, z8, z2 = (c.step_inputs(B, seed=110 + B) for B in (4, 8, 2))
    with torch.no_grad():
        c.op.step(*z4)
        torch.cuda.synchronize()
        c.assert_paths(("step",))
        g, out, s = capture(lambda: list(c.op.step(*z4)))
        with pytest.raises(RuntimeError, match=REFUSED):
            c.op.step(*z8)
        g.replay()
        torch.cuda.synchronize()
        c.check_forward("step", z4, out)
        s.wait_stream(torch.cuda.current_stream())  # replays bypass the library: the caller orders them
        with torch.cuda.stream(s):
            o4 = list(c.op.step(*z4))
            o2 = list(c.op.step(*z2))
        s.synchronize()
    c.check_forward("step", z4, o4)
    c.check_forward("step", z2, o2)
