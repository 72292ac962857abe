"""Oracle of the reversed-order IAF step, ``multiconv2d(..., flipmask=True)`` (TEST INFRASTRUCTURE ONLY).

numpy (any dtype) and torch (autograd, fp64) restatements of graphy/nodes/ar.py:241-329 with flipmask, built on the
unflipped oracles of oracle/iaf_oracle.py and oracle/iaf_oracle_torch.py; tests/golden/make_golden_flipmask.py pins them
against the reference's own source.  What flipmask changes (ar.py:263-276):
  * the mask [n_out, n_in+1, 3, 3] is reversed on all four axes, pad channel included;
  * for heads (zerodiagonal), l2normalize zeroes the centre tap of rows [0, n_out/n_in) (row 0 when n_out < n_in) after
    the mask and before the norm.  Unflipped those entries are already masked; flipped they are live, so they leave the
    norm and get exactly zero gradient.  Here they are zeroed before the norm, so autograd gives the reference gradient.
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import iaf_oracle as O
from oracle import iaf_oracle_torch as OT
from oracle.elbo_oracle import OracleIAFTheano, TorchIAFTheano


def conv_ar_mask(n_in, n_out, zerodiagonal, flipmask):
    """ar.py:241-264: [n_out, n_in+1, 3, 3], pad channel last."""
    m = O.theano_conv_ar_mask(n_in, n_out, (3, 3), zerodiagonal, pad_channel=True)
    return np.ascontiguousarray(m[::-1, ::-1, ::-1, ::-1]) if flipmask else m


def zero_rows(n_in, n_out):
    """Output rows whose centre tap l2normalize zeroes for heads (ar.py:273-276)."""
    return n_out // n_in if n_out >= n_in else 1


def effective_kernel(w, s, zerodiagonal, flipmask, logscale_scale=3.0):
    """ar.py:312-317 with l2normalize 267-281 (logscale=True)."""
    n_out, n_in1 = w.shape[:2]
    kerns = conv_ar_mask(n_in1 - 1, n_out, zerodiagonal, flipmask).astype(w.dtype) * w
    if zerodiagonal:
        kerns[:zero_rows(n_in1 - 1, n_out), :, 1, 1] = 0
    norm = np.sqrt(np.sum(kerns ** 2, axis=(1, 2, 3), keepdims=True)) + 1e-8
    return kerns * (1.0 / norm) * np.exp(logscale_scale * s).reshape(-1, 1, 1, 1)


def ar_conv2d(h, layer, zerodiagonal, flipmask):
    kerns = effective_kernel(layer["w"], layer["s"], zerodiagonal, flipmask)
    return O.trueconv2d_valid(O.pad2dwithchannel(h), kerns) + layer["b"].reshape(1, -1, 1, 1)


def multiconv(z, context, hidden, heads, nl="elu", flipmask=True):
    """ar.py:396-416."""
    f = O.nonlinearity(nl)
    h = z
    for i, layer in enumerate(hidden):
        h = ar_conv2d(h, layer, False, flipmask)
        if i == 0:
            h = h + context
        h = f(h)
    return [ar_conv2d(h, layer, True, flipmask) for layer in heads]


def iaf_step(z, context, hidden, heads, nl="elu", flipmask=True, scale=0.1):
    """models.py:281-285 (or 287-291 for the flipped second step): (z', arw_logsd, logdet)."""
    m, s = multiconv(z, context, hidden, heads, nl, flipmask)
    arw_logsd = s * scale
    z_new = (z - m * scale) / np.exp(arw_logsd)
    return z_new, arw_logsd, -arw_logsd.reshape(z.shape[0], -1).sum(axis=1)


# ---------------------------------------------------------------------------------------------------------------------
# torch (autograd)
# ---------------------------------------------------------------------------------------------------------------------
def t_ar_conv2d(h, layer, zerodiagonal, flipmask):
    w, s, b = layer["w"], layer["s"], layer["b"]
    n_out, n_in1 = w.shape[:2]
    mask = torch.from_numpy(conv_ar_mask(n_in1 - 1, n_out, zerodiagonal, flipmask)).to(w.dtype)
    kerns = mask * w
    if zerodiagonal:
        keep = torch.ones_like(kerns)
        keep[:zero_rows(n_in1 - 1, n_out), :, 1, 1] = 0
        kerns = kerns * keep
    norm = torch.sqrt((kerns ** 2).sum(dim=(1, 2, 3), keepdim=True)) + 1e-8
    kerns = kerns * (1.0 / norm) * torch.exp(3.0 * s).reshape(-1, 1, 1, 1)
    B, C, H, W = h.shape
    hp = torch.zeros((B, C + 1, H + 2, W + 2), dtype=h.dtype)
    hp[:, C] = 1.0
    hp[:, C, 1:-1, 1:-1] = 0.0
    hp[:, :C, 1:-1, 1:-1] = h
    return F.conv2d(hp, torch.flip(kerns, dims=(2, 3))) + b.reshape(1, -1, 1, 1)


def t_multiconv(z, context, hidden, heads, nl="elu", flipmask=True):
    f = OT._nl(nl)
    x = z
    for i, layer in enumerate(hidden):
        x = t_ar_conv2d(x, layer, False, flipmask)
        if i == 0:
            x = x + context
        x = f(x)
    return [t_ar_conv2d(x, layer, True, flipmask) for layer in heads]


def t_iaf_step(z, context, hidden, heads, nl="elu", flipmask=True, scale=0.1):
    m, s = t_multiconv(z, context, hidden, heads, nl, flipmask)
    arw_logsd = s * scale
    z_new = (z - m * scale) / torch.exp(arw_logsd)
    return z_new, arw_logsd, -arw_logsd.flatten(1).sum(dim=1)


def t_stochastic_layer(eps, post_mean, post_logsd, prior_mean, prior_logsd, context, hidden, heads, nl="elu",
                       flipmask=True):
    """The fused layer entry's block (one step) with the given mask order: (z', kl, kl_bc, kl_cost)."""
    z = post_mean + torch.exp(post_logsd) * eps
    logqs = -0.5 * (np.log(2 * np.pi) + 2 * post_logsd + (z - post_mean) ** 2 / torch.exp(2 * post_logsd))
    z, arw_logsd, _ = t_iaf_step(z, context, hidden, heads, nl, flipmask)
    logqs = logqs + arw_logsd
    logps = -0.5 * (np.log(2 * np.pi) + 2 * prior_logsd + (z - prior_mean) ** 2 / torch.exp(2 * prior_logsd))
    kl = logqs - logps
    return z, kl, kl.sum(dim=(2, 3)), kl.sum(dim=(1, 2, 3))


# ---------------------------------------------------------------------------------------------------------------------
# iaf_layer callables for iaf_b200.elbo_theano with posterior='down_iaf2_nl2' (models.py:93-98, 273-291)
# ---------------------------------------------------------------------------------------------------------------------
def _conv_layers(w, name, conv, depth_ar, f):
    pre = "%s_posterior_conv%d_" % (name, conv)
    layer = lambda n: {k: f(w[pre + n + "_" + k]) for k in "wsb"}
    return [layer("%d" % k) for k in range(depth_ar)], [layer("out_0"), layer("out_1")]


class OracleIAFTheanoNL2(OracleIAFTheano):
    """The numpy fp64 oracle block with the bare step of either posterior conv: ``step(name, z, context, conv)``,
    conv 2 in the reversed order (flipmask=True)."""

    def step(self, name, z, context, conv=1):
        f = lambda t: t.detach().cpu().numpy().astype(np.float64)
        hidden, heads = _conv_layers(self.w, name, conv, self.hps["depth_ar"], f)
        z_new, arw_logsd, _ = iaf_step(f(z), f(context), hidden, heads, self.hps["nl"], flipmask=conv == 2)
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(z.dtype).to(z.device)
        return t(z_new), t(arw_logsd)


class TorchIAFTheanoNL2(TorchIAFTheano):
    """Differentiable (torch autograd) counterpart of OracleIAFTheanoNL2."""

    def step(self, name, z, context, conv=1):
        hidden, heads = _conv_layers(self.w, name, conv, self.hps["depth_ar"], lambda t: t)
        return t_iaf_step(z, context, hidden, heads, self.hps["nl"], flipmask=conv == 2)[:2]
