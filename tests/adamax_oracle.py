"""Op-by-op torch restatement of the reference's two Adamax rules and their weight averages (TEST INFRASTRUCTURE: the
yardstick of iaf_b200.optim.Adamax and its kernel).  Every line is one torch operation, in the order and with the
constants include/iaf_b200.h gives for iaf_adamax_step, in the parameters' own dtype: in float32 it is what the kernel
must match bit for bit, and in float64 it is the optimiser of the fp64 oracle training loop.  tests/golden/optim.npz
(the reference's own update code) checks it."""
import torch

from iaf_b200.optim import DEFAULTS


class RestatedAdamax(object):
    """Same constructor, ``step(grad_scale)`` and ``averaged()`` as iaf_b200.optim.Adamax, on any device and dtype.
    ``grads``: an optional {name: tensor or None} that ``step`` uses instead of the tensors' ``.grad``."""

    def __init__(self, params, rule="tf", lr=None, beta1=None, beta2=None, avg_decay=None):
        d = DEFAULTS[rule]
        lr = d["lr"] if lr is None else float(lr)
        beta1 = d["beta1"] if beta1 is None else float(beta1)
        beta2 = d["beta2"] if beta2 is None else float(beta2)
        if avg_decay is None:
            avg_decay = d["avg_decay"] if rule == "tf" else 1.0 - beta2
        self.rule, self.params = rule, dict(params)
        p0 = next(iter(self.params.values()))
        c = lambda v: torch.tensor(v, dtype=p0.dtype, device=p0.device)
        if rule == "tf":   # adamax.py:41-47; 1. - beta1_t in the variable's dtype
            self.c = [c(lr), c(beta1), c(1.0) - c(beta1), c(beta2), c(1e-8), c(1.0 - avg_decay)]
        else:              # optim.py:116-122 with alpha = -lr
            self.c = [c(-lr), c(1.0 - beta1), c(beta1), c(1.0 - beta2), c(1e-8), c(1.0 - avg_decay), c(avg_decay)]
        with torch.no_grad():
            self.mom1 = {k: torch.zeros_like(p) for k, p in self.params.items()}
            self.mom_max = {k: torch.full_like(p, 1e-8 if rule == "theano" else 0.0) for k, p in self.params.items()}
            self.avg = {k: p.detach().clone() for k, p in self.params.items()}

    def averaged(self):
        return dict(self.avg)

    @torch.no_grad()
    def step(self, grad_scale=1.0, grads=None):
        c = self.c
        for k, p in self.params.items():
            g = p.grad if grads is None else grads[k]
            m1, mx, a = self.mom1[k], self.mom_max[k], self.avg[k]
            if self.rule == "tf":
                a.copy_(a - (a - p) * c[5])
                if g is None:
                    continue
                g = g * c[0].new_tensor(grad_scale)
                m1.copy_(c[1] * m1 + c[2] * g)
                mx.copy_(torch.maximum(c[3] * mx + c[4], g.abs()))
                p.copy_(p - c[0] * (m1 / mx))
            else:
                g = torch.zeros_like(p) if g is None else g * c[0].new_tensor(grad_scale)
                a.copy_(c[5] * p + c[6] * a)
                m1.copy_(c[1] * m1 + c[2] * g)
                mx.copy_(torch.maximum(c[3] * mx, g.abs() + c[4]))
                p.copy_(p + (c[0] * m1) / mx)
