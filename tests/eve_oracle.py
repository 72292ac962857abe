"""Op-by-op torch restatement of the reference's Eve update and weight average (TEST INFRASTRUCTURE: the yardstick of
iaf_b200.optim.Eve and its kernel).  Every line is one torch operation, in the order and with the constants
include/iaf_b200.h gives for iaf_eve_step, in the parameters' own dtype: in float32 it is what the kernel must match bit
for bit, and in float64 it is the optimiser of the fp64 oracle training loop.  tests/golden/eve.npz (the reference's own
Eve source) checks it."""
import torch

from iaf_b200.optim import EVE_DEFAULTS


class RestatedEve(object):
    """Same constructor, ``lookahead()``, ``step(grad_scale)`` and ``averaged()`` as iaf_b200.optim.Eve, on any device
    and dtype.  ``grads``: an optional {name: tensor or None} that ``step`` uses instead of the lookahead's ``.grad``."""

    def __init__(self, params, lr=None, beta1=None, beta2=None, beta3=None):
        d = EVE_DEFAULTS
        lr = d["lr"] if lr is None else float(lr)
        beta1 = d["beta1"] if beta1 is None else float(beta1)
        beta2 = d["beta2"] if beta2 is None else float(beta2)
        beta3 = d["beta3"] if beta3 is None else float(beta3)
        self.params = dict(params)
        p0 = next(iter(self.params.values()))
        c = lambda v: torch.tensor(v, dtype=p0.dtype, device=p0.device)
        # optim.py:125-146 with alpha = -lr: python floats, each expression in double, then cast
        self.c = [c(-lr), c(1.0 - beta1), c(beta1), c(1.0 - beta2), c(1e-8), c(beta3), c(1.0 - beta3),
                  c((1.0 - beta1) / beta1)]
        with torch.no_grad():
            self.mom1 = {k: torch.zeros_like(p) for k, p in self.params.items()}
            self.mom_max = {k: torch.full_like(p, 1e-8) for k, p in self.params.items()}
            self.delta = {k: torch.zeros_like(p) for k, p in self.params.items()}
            self.avg = {k: p.detach().clone() for k, p in self.params.items()}
            self.la = {k: (p.detach() + self.c[7] * self.delta[k]).requires_grad_() for k, p in self.params.items()}

    def lookahead(self):
        return dict(self.la)

    def averaged(self):
        return dict(self.avg)

    @torch.no_grad()
    def step(self, grad_scale=1.0, grads=None):
        c = self.c
        for k, p in self.params.items():
            g = self.la[k].grad if grads is None else grads[k]
            m1, mx, d, a, la = self.mom1[k], self.mom_max[k], self.delta[k], self.avg[k], self.la[k]
            g = torch.zeros_like(p) if g is None else g * c[0].new_tensor(grad_scale)
            a.copy_(c[5] * p + c[6] * a)
            m1.copy_(c[1] * m1 + c[2] * g)
            mx.copy_(torch.maximum(c[3] * mx, g.abs() + c[4]))
            d.copy_((c[0] * m1) / mx)
            p.copy_(p + d)
            la.copy_(p + c[7] * d)
