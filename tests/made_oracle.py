"""Oracle of the autoregressive (MADE) prior, ``cvae_layer(..., prior='made', ...)`` (TEST INFRASTRUCTURE ONLY).

numpy (fp64) and torch (autograd) restatements of models.py:36-38, 304-309: the prior's own masked stack
``prior_conv1 = multiconv2d(name+'_prior_conv1', n_z, depth_ar*[n_h2], [n_z,n_z], kernel, False, nl, w)`` at the
posterior's final sample z with the context made_context, both heads scaled by .1, and
``logps = gaussian_diag(made_mean, 2*made_logsd, z).logps`` in rand.py:83's own form.  Built on the Theano oracles of
tests/flipmask_oracle.py (unflipped mask); tests/golden/make_golden_made.py pins them against the reference's source.
It also provides ``prior_logp`` for the oracle ``iaf_layer`` callables of iaf_b200.elbo_theano.
"""
import math

import numpy as np
import torch

from tests import flipmask_oracle as FO


def logps(z, context, hidden, heads, nl="elu"):
    """fp64 numpy: per-element log-density [B,C,H,W] of z under the prior."""
    m, s = FO.multiconv(z, context, hidden, heads, nl, flipmask=False)
    mean, logvar = 0.1 * m, 2 * (0.1 * s)
    return -0.5 * (np.log(2 * np.pi) + logvar + (z - mean) ** 2 / np.exp(logvar))   # rand.py:83


def t_logps(z, context, hidden, heads, nl="elu"):
    """torch (autograd): the same."""
    m, s = FO.t_multiconv(z, context, hidden, heads, nl, flipmask=False)
    mean, logvar = 0.1 * m, 2 * (0.1 * s)
    return -0.5 * (math.log(2 * math.pi) + logvar + (z - mean) ** 2 / torch.exp(logvar))


def _prior_layers(w, name, depth_ar, f):
    pre = "%s_prior_conv1_" % name
    layer = lambda n: {k: f(w[pre + n + "_" + k]) for k in "wsb"}
    return [layer("%d" % k) for k in range(depth_ar)], [layer("out_0"), layer("out_1")]


class OracleIAFTheanoMade(FO.OracleIAFTheanoNL2):
    """numpy fp64 oracle iaf_layer with the MADE prior: ``prior_logp(name, z, context) -> (logp_bc, logp)``."""

    def prior_logp(self, name, z, context):
        f = lambda t: t.detach().cpu().numpy().astype(np.float64)
        hidden, heads = _prior_layers(self.w, name, self.hps["depth_ar"], f)
        lp = logps(f(z), f(context), hidden, heads, self.hps["nl"])
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(z.dtype).to(z.device)
        return t(lp.sum(axis=(2, 3))), t(lp.sum(axis=(1, 2, 3)))


class TorchIAFTheanoMade(FO.TorchIAFTheanoNL2):
    """Differentiable (torch autograd) counterpart of OracleIAFTheanoMade."""

    def prior_logp(self, name, z, context):
        hidden, heads = _prior_layers(self.w, name, self.hps["depth_ar"], lambda t: t)
        lp = t_logps(z, context, hidden, heads, self.hps["nl"])
        return lp.sum(dim=(2, 3)), lp.sum(dim=(1, 2, 3))
