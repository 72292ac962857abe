"""The reference's optimisers: Adamax and the weight average that evaluation runs on, in one fused launch per step.

Neither reference uses ``torch.optim.Adamax``, and their two rules differ from it and from each other
(include/iaf_b200.h, ``iaf_adamax_step``; INTEGRATION.md §4c):

* ``rule="tf"``: ``AdamaxOptimizer`` (tf_utils/adamax.py:40-56) with ``ExponentialMovingAverage(0.999)`` over every
  trainable variable (tf_train.py:127, 147, 155-159).  Defaults: lr 0.01 (``hps.learning_rate``), beta1 0.9,
  beta2 0.999, avg_decay 0.999.
* ``rule="theano"``: ``AdaMaxAvg`` (graphy/misc/optim.py:99-123, called at models.py:566-568).  Defaults: lr 0.002,
  beta1 0.1, beta2 0.001 (train.py:65-67, models.py:384); the average is ``w_avg = beta2 w + (1 - beta2) w_avg``, i.e.
  avg_decay = 1 - beta2.

:class:`Eve` is the Theano model's other optimiser (``optim='eve'``: graphy/misc/optim.py:125-146, called at
models.py:570-572; include/iaf_b200.h, ``iaf_eve_step``).  It takes the gradient at a lookahead point
``w' = w + (1 - beta1) / beta1 * delta``, so the model runs on :meth:`Eve.lookahead`, not on the parameters.  Defaults:
lr 0.002, beta1 0.1, beta2 0.001 as ``AdaMaxAvg``, and beta3 0.01 for the average (``Eve``'s own default, which
models.py does not override).
"""
import ctypes as C

import torch

from . import _lib

DEFAULTS = {"tf": dict(lr=0.01, beta1=0.9, beta2=0.999, avg_decay=0.999),
            "theano": dict(lr=0.002, beta1=0.1, beta2=0.001, avg_decay=None)}
EVE_DEFAULTS = dict(lr=0.002, beta1=0.1, beta2=0.001, beta3=0.01)
_ALIGN = 4  # state slices start on 16-byte boundaries, so aligned parameters take the kernel's float4 loads


def _check_params(who, params):
    """-> (names, tensors, device, state offsets, state length) of the dict ``params``, or ValueError."""
    if not isinstance(params, dict) or not params:
        raise ValueError("%s: params must be a non-empty dict of tensors" % who)
    if len(params) > 2 ** 31 - 1:
        raise ValueError("%s: too many tensors" % who)
    names = list(params)
    tensors = [params[k] for k in names]
    device = None
    for k, p in zip(names, tensors):
        if not isinstance(p, torch.Tensor) or not p.is_cuda or p.dtype != torch.float32 or not p.is_contiguous():
            raise ValueError("%s: %r must be a contiguous float32 CUDA tensor" % (who, k))
        if p.numel() == 0:
            raise ValueError("%s: %r is empty" % (who, k))
        if device is None:
            device = p.device
        elif p.device != device:
            raise ValueError("%s: %r is on %s, the others on %s" % (who, k, p.device, device))
    offsets, total = [], 0
    for p in tensors:
        offsets.append(total)
        total += -(-p.numel() // _ALIGN) * _ALIGN
    return names, tensors, device, offsets, total


def _table(params, offsets):
    t = (_lib.AdamaxTensor * len(params))()
    for e, p, off in zip(t, params, offsets):
        e.param, e.numel, e.offset = p.data_ptr(), p.numel(), off
    return t


def _bind_grads(who, names, params, table, seen, device):
    """Point entry i of ``table`` at ``params[i].grad`` (NULL for None).  ``seen[i]``: the gradient tensor the entry
    points at already, whose checks are not repeated."""
    for i, p in enumerate(params):
        g = p.grad
        if g is seen[i] and (g is None or g.data_ptr() == table[i].grad):
            continue               # the same gradient as last step (zeroed in place): already checked
        if g is not None and (g.device != device or g.dtype != torch.float32 or g.shape != p.shape or
                              not g.is_contiguous()):
            raise ValueError("%s: the gradient of %r must be a contiguous float32 tensor of its shape on %s"
                             % (who, names[i], device))
        table[i].grad = None if g is None else g.data_ptr()
        seen[i] = g


def _views(buf, names, params, offsets):
    """{name: buf's slice for the parameter, shaped like it, holding a copy of its value}."""
    out = {}
    for k, p, off in zip(names, params, offsets):
        v = buf[off:off + p.numel()].view(p.shape)
        v.copy_(p.detach())
        out[k] = v
    return out


class Adamax(object):
    """Adamax over the dict ``params`` (name -> contiguous fp32 CUDA tensor, all on one device), updated in place.

    Construct it after :func:`iaf_b200.elbo.data_init` / :func:`iaf_b200.elbo_theano.data_init`: the averages start at
    the parameters' current values (tf_train.py:157, models.py:555), the first moments at 0 and the max at 0 (TF) or
    1e-8 (Theano, optim.py:116).  :meth:`step` reads each tensor's ``.grad``; a tensor whose ``.grad`` is None is
    skipped under the TF rule (its average still moves) and takes a zero gradient under the Theano rule.
    :meth:`averaged` returns the averages under the same names, for ``forward`` / ``log_likelihood`` / ``decode``.

    The optimiser holds the tensors it was given: replacing an entry of the dict afterwards is not seen."""

    def __init__(self, params, rule="tf", lr=None, beta1=None, beta2=None, avg_decay=None):
        if rule not in DEFAULTS:
            raise ValueError("Adamax: unknown rule %r (use 'tf' or 'theano')" % (rule,))
        d = DEFAULTS[rule]
        self.rule = rule
        self.lr = d["lr"] if lr is None else float(lr)
        self.beta1 = d["beta1"] if beta1 is None else float(beta1)
        self.beta2 = d["beta2"] if beta2 is None else float(beta2)
        if avg_decay is None:
            avg_decay = d["avg_decay"] if rule == "tf" else 1.0 - self.beta2
        self.avg_decay = float(avg_decay)

        self.names, self.params, self.device, offsets, total = _check_params("Adamax", params)
        device = self.device
        with torch.no_grad():
            self.mom1 = torch.zeros(total, dtype=torch.float32, device=device)
            self.mom_max = torch.full((total,), 1e-8 if rule == "theano" else 0.0, dtype=torch.float32, device=device)
            self.avg = torch.zeros(total, dtype=torch.float32, device=device)
            self._avg = _views(self.avg, self.names, self.params, offsets)

        self._table = _table(self.params, offsets)
        self._lib = _lib.lib()
        self._written = self.params + [self.mom1, self.mom_max, self.avg]
        self._grads = [None] * len(self.params)  # the gradient tensors the table points at

    def averaged(self):
        """{name: the parameter's average} (views of one buffer the optimiser updates in place)."""
        return dict(self._avg)

    def step(self, grad_scale=1.0):
        """One update of every parameter and average, one kernel launch (more only past
        ``_lib.ADAMAX_MAX_TENSORS`` tensors) on the current stream.  The gradient used is ``grad_scale * p.grad``.
        No allocation, no copy to the device and no synchronisation: it can be captured into a CUDA graph."""
        _bind_grads("Adamax", self.names, self.params, self._table, self._grads, self.device)
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream(self.device).cuda_stream
            _lib.check(self._lib.iaf_adamax_step(_lib.ADAMAX_RULES[self.rule], self._table, len(self._table),
                                                 C.c_void_p(self.mom1.data_ptr()), C.c_void_p(self.mom_max.data_ptr()),
                                                 C.c_void_p(self.avg.data_ptr()), self.lr, self.beta1, self.beta2,
                                                 self.avg_decay, float(grad_scale), C.c_void_p(stream)))
        # the kernel wrote through raw pointers: bump the version counters (the averages' views share the buffer's), so
        # caches keyed on them -- IAFOperator's packed weights -- see the new values
        torch.autograd.graph.increment_version(self._written)


class Eve(object):
    """Eve over the dict ``params`` (name -> contiguous fp32 CUDA tensor, all on one device), updated in place: the
    Theano model's ``optim='eve'`` (graphy/misc/optim.py:125-146, models.py:570-572).

    The gradient is taken at the lookahead ``w' = w + (1 - beta1) / beta1 * delta``, where delta is the last update.
    :meth:`lookahead` returns those points under the same names: leaf tensors that require grad, views of one buffer
    the optimiser owns.  Run the model's forward and backward on them, then :meth:`step`, which reads each lookahead
    tensor's ``.grad`` (None is a zero gradient), updates the parameters, moments, averages and delta, and writes the
    next step's lookahead.  The averages are ``avg = beta3 w + (1 - beta3) avg``.

    Construct it after :func:`iaf_b200.elbo_theano.data_init`: the averages and the lookahead start at the parameters'
    current values (delta = 0), the first moments at 0 and the max at 1e-8 (optim.py:131-134, models.py:555).  The
    optimiser holds the tensors it was given: replacing an entry of the dict, or writing to a parameter between steps,
    is not seen by the lookahead."""

    def __init__(self, params, lr=None, beta1=None, beta2=None, beta3=None):
        d = EVE_DEFAULTS
        self.lr = d["lr"] if lr is None else float(lr)
        self.beta1 = d["beta1"] if beta1 is None else float(beta1)
        self.beta2 = d["beta2"] if beta2 is None else float(beta2)
        self.beta3 = d["beta3"] if beta3 is None else float(beta3)
        if self.beta1 == 0.0:
            raise ValueError("Eve: beta1 must be nonzero (the lookahead is w + (1 - beta1) / beta1 * delta)")

        self.names, self.params, self.device, offsets, total = _check_params("Eve", params)
        device = self.device
        with torch.no_grad():
            self.mom1 = torch.zeros(total, dtype=torch.float32, device=device)
            self.mom_max = torch.full((total,), 1e-8, dtype=torch.float32, device=device)
            self.delta = torch.zeros(total, dtype=torch.float32, device=device)
            self.avg = torch.zeros(total, dtype=torch.float32, device=device)
            self.lookahead_buf = torch.zeros(total, dtype=torch.float32, device=device)
            self._avg = _views(self.avg, self.names, self.params, offsets)
            # detached views: leaves of their own that share the buffer's storage and version counter
            self._la = {k: v.detach().requires_grad_()
                        for k, v in _views(self.lookahead_buf, self.names, self.params, offsets).items()}
        self._la_list = [self._la[k] for k in self.names]

        self._table = _table(self.params, offsets)
        self._lib = _lib.lib()
        self._written = self.params + self._la_list + [self.mom1, self.mom_max, self.delta, self.avg,
                                                       self.lookahead_buf]
        self._grads = [None] * len(self.params)

    def lookahead(self):
        """{name: the point the next step's gradient is taken at} (leaf views of one buffer, updated by :meth:`step`)."""
        return dict(self._la)

    def averaged(self):
        """{name: the parameter's average} (views of one buffer the optimiser updates in place)."""
        return dict(self._avg)

    def step(self, grad_scale=1.0):
        """One update of every parameter, average and lookahead, one kernel launch (more only past
        ``_lib.ADAMAX_MAX_TENSORS`` tensors) on the current stream.  The gradient used is ``grad_scale * w'.grad``.
        No allocation, no copy to the device and no synchronisation: it can be captured into a CUDA graph."""
        _bind_grads("Eve", self.names, self._la_list, self._table, self._grads, self.device)
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream(self.device).cuda_stream
            ptr = lambda t: C.c_void_p(t.data_ptr())
            _lib.check(self._lib.iaf_eve_step(self._table, len(self._table), ptr(self.mom1), ptr(self.mom_max),
                                              ptr(self.delta), ptr(self.avg), ptr(self.lookahead_buf), self.lr,
                                              self.beta1, self.beta2, self.beta3, float(grad_scale),
                                              C.c_void_p(stream)))
        # as Adamax.step: the parameters, the lookahead tensors and the averages' views see the kernel's writes
        torch.autograd.graph.increment_version(self._written)
