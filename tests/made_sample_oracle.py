"""Oracle of the inverse of the IAF step, and of sampling the autoregressive (MADE) prior (TEST INFRASTRUCTURE ONLY).

The fp64 inverse is the fixed-point iteration ``z_{k+1} = 0.1 m(z_k) + exp(0.1 s(z_k)) u`` from ``z_0 = u`` on the
forward oracles (``O.multiconv``, ``FO.multiconv``), which tests/golden/ pins against the reference.  Each iteration
makes at least one more position final in the mask's order, so the iterate stops changing after at most
n_z*H*W + 1 iterations; taking longer means the order is not the mask's, and is an error.  It needs no knowledge of
the order itself, so it checks the kernel's order logic independently.
"""
import numpy as np
import torch

from oracle import iaf_oracle as O
from tests import flipmask_oracle as FO
from tests.made_oracle import OracleIAFTheanoMade, TorchIAFTheanoMade, _prior_layers


def heads(variant, z, ctx, hidden, hd, nl):
    if variant == "theano_flipmask":
        return FO.multiconv(z, ctx, hidden, hd, nl, flipmask=True)
    return O.multiconv(variant, z, ctx, hidden, hd, nl)


def inverse(variant, u, ctx, hidden, hd, nl="elu"):
    """fp64: (z, arw_logsd, logdet, iterations) with step(z) = u."""
    f64 = lambda ls: O.cast_params(ls, np.float64)
    hidden, hd = f64(hidden), f64(hd)
    u = np.asarray(u, np.float64)
    ctx = None if ctx is None else np.asarray(ctx, np.float64)
    bound = u[0].size + 1
    z = u.copy()
    for it in range(1, bound + 1):
        m, s = heads(variant, z, ctx, hidden, hd, nl)
        zn = 0.1 * m + np.exp(0.1 * s) * u
        if np.array_equal(zn, z):
            a = 0.1 * s
            return z, a, -a.sum(axis=(1, 2, 3)), it
        z = zn
    raise AssertionError("the fixed point did not settle within n_z*H*W + 1 iterations: not the mask's order")


class OracleIAFTheanoMadeSample(OracleIAFTheanoMade):
    """The fp64 oracle iaf_layer with ``prior_sample(name, eps, context) -> z``: the MADE prior's stack inverted by the
    fixed-point iteration."""

    def prior_sample(self, name, eps, context):
        f = lambda t: t.detach().cpu().numpy().astype(np.float64)
        hidden, hd = _prior_layers(self.w, name, self.hps["depth_ar"], f)
        z = inverse("theano", f(eps), f(context), hidden, hd, self.hps["nl"])[0]
        return torch.from_numpy(z).to(eps.dtype).to(eps.device)


class TorchIAFTheanoMadeSample(TorchIAFTheanoMade):
    def prior_sample(self, name, eps, context):
        return OracleIAFTheanoMadeSample.prior_sample(self, name, eps, context)
