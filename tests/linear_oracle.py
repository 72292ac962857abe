"""Oracle of the linear IAF posteriors ``down_iaf2`` / ``up_iaf2`` (TEST INFRASTRUCTURE ONLY).

numpy (fp64) and torch (autograd) restatements of models.py:55-56, 79-82, 152-161, 246-259 in the reference's own form:
ONE masked conv ``ar.conv2d(name+'_posterior_conv1', n_z, 2 n_z)`` (ar.py:241-329, zerodiagonal, mask and l2normalize of
its [2 n_z, n_z + 1, 3, 3] kernel), no context, then ``arw_mean = out[:, ::2]``, ``arw_logsd = out[:, 1::2]``, both
scaled by .1, ``z = (z - arw_mean) / exp(arw_logsd)``.  Nothing here de-interleaves weights: the product does
(iaf_b200.weights.deinterleave_heads), this oracle slices the conv's OUTPUT as the reference does.
tests/golden/make_golden_linear.py pins it against the reference's source.  The prior (diag or made) is the one of
tests/made_oracle.py.
"""
import numpy as np
import torch

from iaf_b200.elbo import stochastic_layer
from tests import flipmask_oracle as FO
from tests.made_oracle import OracleIAFTheanoMade, TorchIAFTheanoMade


def step(z, layer, scale=0.1):
    """fp64 numpy: (z', arw_logsd) of the linear step with the conv's (w, s, b) in ``layer``."""
    out = FO.ar_conv2d(z, layer, True, False)
    arw_mean, arw_logsd = scale * out[:, ::2], scale * out[:, 1::2]
    return (z - arw_mean) / np.exp(arw_logsd), arw_logsd


def t_step(z, layer, scale=0.1):
    """torch (autograd): the same."""
    out = FO.t_ar_conv2d(z, layer, True, False)
    arw_mean, arw_logsd = scale * out[:, ::2], scale * out[:, 1::2]
    return (z - arw_mean) / torch.exp(arw_logsd), arw_logsd


def _layer(w, name, f):
    return {k: f(w["%s_posterior_conv1_%s" % (name, k)]) for k in "wsb"}


class OracleIAFTheanoLinear(OracleIAFTheanoMade):
    """numpy fp64 oracle iaf_layer for the linear posteriors: ``step(name, z, context)`` ignores the context (there is
    none), ``__call__`` is the fused block around it, ``prior_logp`` the MADE prior's."""

    def step(self, name, z, context, conv=1):
        assert context is None and conv == 1
        f = lambda t: t.detach().cpu().numpy().astype(np.float64)
        z_new, arw_logsd = step(f(z), _layer(self.w, name, f))
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(z.dtype).to(z.device)
        return t(z_new), t(arw_logsd)

    def __call__(self, name, eps, post_mean, post_logsd, prior_mean, prior_logsd, context):
        return stochastic_layer(lambda z, c: self.step(name, z, c), eps, post_mean, post_logsd, prior_mean, prior_logsd,
                                context)


class TorchIAFTheanoLinear(TorchIAFTheanoMade):
    """Differentiable (torch autograd) counterpart of OracleIAFTheanoLinear."""

    def step(self, name, z, context, conv=1):
        assert context is None and conv == 1
        return t_step(z, _layer(self.w, name, lambda t: t))
