"""The reference's optimisers: Adamax and the weight average that evaluation runs on, in one fused launch per step.

Neither reference uses ``torch.optim.Adamax``, and their two rules differ from it and from each other
(include/iaf_b200.h, ``iaf_adamax_step``; INTEGRATION.md §4c):

* ``rule="tf"``: ``AdamaxOptimizer`` (tf_utils/adamax.py:40-56) with ``ExponentialMovingAverage(0.999)`` over every
  trainable variable (tf_train.py:127, 147, 155-159).  Defaults: lr 0.01 (``hps.learning_rate``), beta1 0.9,
  beta2 0.999, avg_decay 0.999.
* ``rule="theano"``: ``AdaMaxAvg`` (graphy/misc/optim.py:99-123, called at models.py:566-568).  Defaults: lr 0.002,
  beta1 0.1, beta2 0.001 (train.py:65-67, models.py:384); the average is ``w_avg = beta2 w + (1 - beta2) w_avg``, i.e.
  avg_decay = 1 - beta2.
"""
import ctypes as C

import torch

from . import _lib

DEFAULTS = {"tf": dict(lr=0.01, beta1=0.9, beta2=0.999, avg_decay=0.999),
            "theano": dict(lr=0.002, beta1=0.1, beta2=0.001, avg_decay=None)}
_ALIGN = 4  # state slices start on 16-byte boundaries, so aligned parameters take the kernel's float4 loads


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
        if not isinstance(params, dict) or not params:
            raise ValueError("Adamax: params must be a non-empty dict of tensors")
        if len(params) > 2 ** 31 - 1:
            raise ValueError("Adamax: too many tensors")
        d = DEFAULTS[rule]
        self.rule = rule
        self.lr = d["lr"] if lr is None else float(lr)
        self.beta1 = d["beta1"] if beta1 is None else float(beta1)
        self.beta2 = d["beta2"] if beta2 is None else float(beta2)
        if avg_decay is None:
            avg_decay = d["avg_decay"] if rule == "tf" else 1.0 - self.beta2
        self.avg_decay = float(avg_decay)

        self.names = list(params)
        self.params = [params[k] for k in self.names]
        device = None
        for k, p in zip(self.names, self.params):
            if not isinstance(p, torch.Tensor) or not p.is_cuda or p.dtype != torch.float32 or not p.is_contiguous():
                raise ValueError("Adamax: %r must be a contiguous float32 CUDA tensor" % (k,))
            if p.numel() == 0:
                raise ValueError("Adamax: %r is empty" % (k,))
            if device is None:
                device = p.device
            elif p.device != device:
                raise ValueError("Adamax: %r is on %s, the others on %s" % (k, p.device, device))
        self.device = device

        offsets, total = [], 0
        for p in self.params:
            offsets.append(total)
            total += -(-p.numel() // _ALIGN) * _ALIGN
        with torch.no_grad():
            self.mom1 = torch.zeros(total, dtype=torch.float32, device=device)
            self.mom_max = torch.full((total,), 1e-8 if rule == "theano" else 0.0, dtype=torch.float32, device=device)
            self.avg = torch.zeros(total, dtype=torch.float32, device=device)
            self._avg = {}
            for k, p, off in zip(self.names, self.params, offsets):
                v = self.avg[off:off + p.numel()].view(p.shape)
                v.copy_(p.detach())
                self._avg[k] = v

        self._table = (_lib.AdamaxTensor * len(self.params))()
        for e, p, off in zip(self._table, self.params, offsets):
            e.param, e.numel, e.offset = p.data_ptr(), p.numel(), off
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
        seen = self._grads
        for i, p in enumerate(self.params):
            g = p.grad
            if g is seen[i] and (g is None or g.data_ptr() == self._table[i].grad):
                continue               # the same gradient as last step (zeroed in place): already checked
            if g is not None and (g.device != self.device or g.dtype != torch.float32 or g.shape != p.shape or
                                  not g.is_contiguous()):
                raise ValueError("Adamax: the gradient of %r must be a contiguous float32 tensor of its shape on %s"
                                 % (self.names[i], self.device))
            self._table[i].grad = None if g is None else g.data_ptr()
            seen[i] = g
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream(self.device).cuda_stream
            _lib.check(self._lib.iaf_adamax_step(_lib.ADAMAX_RULES[self.rule], self._table, len(self._table),
                                                 C.c_void_p(self.mom1.data_ptr()), C.c_void_p(self.mom_max.data_ptr()),
                                                 C.c_void_p(self.avg.data_ptr()), self.lr, self.beta1, self.beta2,
                                                 self.avg_decay, float(grad_scale), C.c_void_p(stream)))
        # the kernel wrote through raw pointers: bump the version counters (the averages' views share the buffer's), so
        # caches keyed on them -- IAFOperator's packed weights -- see the new values
        torch.autograd.graph.increment_version(self._written)
