"""ELBO forward of the Theano front-end around the IAF operator (SURVEY 8f-2, configs C1 / C4):
`cvae1.f_encode_decode` (models.py:435-497) with `cvae_layer.up` / `cvae_layer.down_q` (models.py:133-328) for
``posterior='down_iaf2_nl'`` (the README configs, train.py:55-75) and ``posterior='up_iaf2_nl'`` (the bottom-up
placement of the same operator, models.py:169-178) and ``posterior='down_iaf2_nl2'`` (two steps, the second with
``flipmask=True``: models.py:93-98, 286-291), ``prior='diag'``, ``px='logistic'``, ``downsample_type='nn'``,
restated in PyTorch so that bits/dim can be compared between the CUDA operator and the oracle
operator on identical weights, inputs and noise.

As in :mod:`iaf_b200.elbo`, only the stochastic-layer block goes through a pluggable callable: for down_iaf2_nl the
fused ``iaf_layer`` (posterior sample -> IAF step -> KL against the prior, all known in the top-down pass), for
up_iaf2_nl the plain step ``iaf_layer.step(name, z, context) -> (z', arw_logsd)`` in the bottom-up pass (the prior is
only known later, so the KL is assembled top-down from the stored sample and log q); the rest is plumbing on stock
torch ops.  Parameters are a dict under the reference's Theano names (graphy/nodes/conv.py:156-173, ar.py:288-296): ``x_enc_{w,b,s}``, ``x_dec_{w,b,s}``, ``logsd_x``,
``h_top``, ``{i}_{j}_up_conv1_{ds}_*``, ``{i}_{j}_up_conv2_*``, ``{i}_{j}_down_conv1_*``, ``{i}_{j}_down_conv2_{ds}_*``,
``{i}_{j}_posterior_conv1_{k}_*`` and ``{i}_{j}_posterior_conv1_out_{k}_*`` (down_iaf2_nl2 also
``{i}_{j}_posterior_conv2_{k}_*`` and ``{i}_{j}_posterior_conv2_out_{k}_*``).  For down_iaf2_nl2 the block is
sample -> step(conv1) -> step(conv2, reversed order) -> KL with both ``arw_logsd`` in log q, assembled by
:func:`iaf_b200.elbo.stochastic_layer` around the two calls ``iaf_layer.step(name, z, context, conv)``, conv = 1, 2.
Any other posterior name raises ``ValueError``.

``prior='made'`` (the autoregressive prior, models.py:36-38, 304-309, 328) is available with all three posteriors:
down_conv1's prior channels are then ``[h_det n_h2 | made_context n_h2]``, the prior's own masked stack
``{i}_{j}_prior_conv1_{k}_*`` / ``{i}_{j}_prior_conv1_out_{k}_*`` is evaluated at the posterior's final sample, and
``kl = logqs - logps_made(z, made_context)``.  The posterior half of the down posteriors is then
:func:`iaf_b200.elbo.posterior_sample` around ``iaf_layer.step`` (the fused diagonal-prior ``layer`` entry does not
apply), and the prior's density is the pluggable ``iaf_layer.prior_logp(name, z, context) -> (logp_bc, logp)``.
:func:`decode` is the generative path, ``cvae1.f_decoder`` (models.py:499-521) over :func:`layer_down_p`; with
``prior='made'`` it samples the prior through ``iaf_layer.prior_sample(name, eps, made_context) -> z``, where the
reference uses ``z = eps`` as a placeholder (models.py:338-340).
``prior='diag'`` is the default; any other prior name (``diag2``, ``bernoulli``, ...) raises ``ValueError``.
``posterior='down_iaf2'`` and ``'up_iaf2'`` are the linear IAF (models.py:55-56, 79-82, 152-161, 246-259): one masked
conv ``{i}_{j}_posterior_conv1_{w,s,b}`` with ``w`` of shape [2 n_z, n_z + 1, 3, 3], whose even rows are the mean head
and odd rows the logsd head, and no context (up_conv1 and down_conv1 have no context channels).  The operator runs it as
a stack without hidden layers and two heads of n_z (:func:`iaf_b200.weights.deinterleave_heads`).
:func:`data_init` is cvae1's data-dependent initialisation (``w['__init']``) for every posterior and prior above.
"""
import math
import warnings

import numpy as np
import torch
import torch.nn.functional as F

from .elbo import InitPass
from .masks import theano_conv_ar_mask
from .weights import deinterleave_heads

LOGSCALE_SCALE = 3.0  # graphy/nodes/conv.py:19 (conv.py:16-22: logscale=True, bn=False, maxweight=0)
INIT_STDEV = 0.1      # graphy/nodes/conv.py:22: the std a datainit conv's output is initialised to
POSTERIORS = ("down_iaf2_nl", "up_iaf2_nl", "down_iaf2_nl2", "down_iaf2", "up_iaf2")
PRIORS = ("diag", "made")
# the paper's linear IAF (models.py:55-56, 79-82): one masked conv ``ar.conv2d(name+'_posterior_conv1', n_z, 2 n_z)``,
# no hidden layer and no context, its rows interleaving the two heads (mean = out[:, ::2], logsd = out[:, 1::2])
LINEAR = ("down_iaf2", "up_iaf2")
UP_POSTERIORS = ("up_iaf2_nl", "up_iaf2")  # the sample is drawn and transformed in the bottom-up pass


def posterior_of(hps):
    """The posterior of ``hps`` (default down_iaf2_nl); any other reference posterior is refused, not approximated."""
    p = hps.get("posterior", "down_iaf2_nl")
    if p not in POSTERIORS:
        raise ValueError("posterior %r is not implemented (available: %s)" % (p, ", ".join(POSTERIORS)))
    return p


def prior_of(hps):
    """The prior of ``hps`` (default diag); any other reference prior (diag2, bernoulli) is refused, not approximated."""
    p = hps.get("prior", "diag")
    if p not in PRIORS:
        raise ValueError("prior %r is not implemented (available: %s)" % (p, ", ".join(PRIORS)))
    return p


def pad2dwithchannel(x, k):
    """graphy/nodes/conv.py:71-83: zero-pad by (k-1)/2 and append a channel that is 1 on the border ring."""
    a = (k - 1) // 2
    B, C, H, W = x.shape
    out = x.new_zeros((B, C + 1, H + 2 * a, W + 2 * a))
    out[:, C] = 1.0
    out[:, C, a:-a, a:-a] = 0.0
    out[:, :C, a:-a, a:-a] = x
    return out


def conv2d(w, name, x, downsample=1, upsample=1):
    """graphy/nodes/conv.py:122-274, run-time branch: kernel / ||kernel|| * exp(3 s) per output map (no epsilon),
    pad channel for k > 1, TRUE convolution 'valid' with stride ``downsample``, bias, then depth-to-space.  During
    :func:`data_init` the datainit branch (conv.py:225-250) runs on the output before depth-to-space."""
    W, b, s = w[name + "_w"], w[name + "_b"], w[name + "_s"]
    k = W.shape[2]
    kern = W / torch.sqrt((W * W).sum(dim=(1, 2, 3), keepdim=True)) * torch.exp(LOGSCALE_SCALE * s).reshape(-1, 1, 1, 1)
    if k > 1:
        x = pad2dwithchannel(x, k)
    y = F.conv2d(x, kern.flip(2, 3), stride=downsample) + b.reshape(1, -1, 1, 1)   # dnn_conv default conv_mode='conv'
    if isinstance(w, InitPass):
        y = _data_init(w, name, y, 1.0 / INIT_STDEV, 1e-7)                          # conv.py:225-250 (datainit)
    if upsample > 1:
        y = F.pixel_shuffle(y, upsample)     # depool2d_split, conv.py:26-33: channel c*f*f + fy*f + fx -> (y*f+fy, x*f+fx)
    return y


def nonlinearity(h, which):
    """graphy/nodes/__init__.py:159-177 (the cases the configs use)."""
    if which == "elu":
        return torch.where(h < 0, torch.exp(torch.clamp(h, max=0.0)) - 1, h)
    if which == "softplus":
        return F.softplus(h)
    if which == "relu":
        return h * (h >= 0).to(h.dtype)
    if which == "tanh":
        return torch.tanh(h)
    if which in (None, "None"):
        return h
    raise ValueError("nonlinearity %r" % (which,))


def downsample_nn(x):
    """conv.py:36-40: mean over 2x2 blocks."""
    B, C, H, W = x.shape
    return x.reshape(B, C, H // 2, 2, W // 2, 2).mean(dim=5).mean(dim=3)


def upsample_nn(x):
    """conv.py:43-49."""
    return x.repeat_interleave(2, dim=2).repeat_interleave(2, dim=3)


def gaussian_logps(mean, logvar, x):
    """graphy/nodes/rand.py:83."""
    return -0.5 * (math.log(2 * math.pi) + logvar + (x - mean) ** 2 / torch.exp(logvar))


def _contiguous(t):
    return None if t is None else t.contiguous()


def layer_up(w, name, h_in, hps, downsample, eps=None, iaf_layer=None):
    """cvae_layer.up (models.py:133-196).  down_iaf2_nl: returns (output, (qz_mean, qz_logsd, up_context)).
    up_iaf2_nl (models.py:169-178): the posterior sample is drawn and transformed HERE, with the context taken from
    up_conv1's channels; returns (output, (z, logqs)) for the top-down pass.  The linear posteriors have no context:
    up_context is None (up_iaf2: models.py:152-161)."""
    nz, nh2, nl = hps["n_z"], hps["n_h2"], hps["nl"]
    ds = 2 if downsample else 1
    posterior = posterior_of(hps)
    h = conv2d(w, "%s_up_conv1_%d" % (name, ds), nonlinearity(h_in, nl), downsample=ds)
    if posterior in LINEAR:                                            # no up context (models.py:25, 55-56, 79-82)
        (h_det, qz_mean, qz_logsd), up_context = torch.split(h, [nh2, nz, nz], dim=1), None
    else:
        h_det, qz_mean, qz_logsd, up_context = torch.split(h, [nh2, nz, nz, nh2], dim=1)
    if downsample:
        h_in = downsample_nn(h_in)
    if posterior in UP_POSTERIORS:
        z0 = qz_mean + torch.exp(qz_logsd) * eps                       # gaussian_diag(qz_mean, 2 qz_logsd).sample
        logqs = gaussian_logps(qz_mean, 2 * qz_logsd, z0)
        z, arw_logsd = iaf_layer.step(name, z0.contiguous(), _contiguous(up_context))
        logqs = logqs + arw_logsd                                      # models.py:174
        hh = torch.cat([h_det, z], dim=1)
        return h_in + 0.1 * conv2d(w, name + "_up_conv2", nonlinearity(hh, nl)), (z, logqs)
    return h_in + 0.1 * conv2d(w, name + "_up_conv2", nonlinearity(h_det, nl)), (qz_mean, qz_logsd, up_context)


def layer_down_q(w, name, h_in, up_state, eps, iaf_layer, hps, downsample):
    """cvae_layer.down_q for down_iaf2_nl / prior diag (models.py:203-328): returns (output, kl_bc [B,C], kl_sum [B])."""
    nz, nh2, nl = hps["n_z"], hps["n_h2"], hps["nl"]
    ds = 2 if downsample else 1
    h = conv2d(w, name + "_down_conv1", nonlinearity(h_in, nl))
    posterior = posterior_of(hps)
    if prior_of(hps) == "made":
        return _layer_down_q_made(w, name, h_in, h, up_state, eps, iaf_layer, hps, downsample)
    if posterior in UP_POSTERIORS:                                     # models.py:215-217, 287-290
        h_det, pz_mean, pz_logsd = torch.split(h, [nh2, nz, nz], dim=1)
        z, logqs = up_state
        kl = logqs - gaussian_logps(pz_mean, 2 * pz_logsd, z)
        hh = torch.cat([h_det, z], dim=1)
        if downsample:
            h_in = upsample_nn(h_in)
        out = h_in + 0.1 * conv2d(w, "%s_down_conv2_%d" % (name, ds), nonlinearity(hh, nl), upsample=ds)
        return out, kl.sum(dim=(2, 3)), kl.sum(dim=(1, 2, 3))
    qz_mean, qz_logsd, up_context = up_state
    if posterior in LINEAR:
        # channel map: [h_det n_h2 | pz_mean n_z | pz_logsd n_z || rz_mean n_z | rz_logsd n_z]  (models.py:79-82, 246-259)
        h_det, pz_mean, pz_logsd, rz_mean, rz_logsd = torch.split(h, [nh2, nz, nz, nz, nz], dim=1)
        context = None
    else:
        # channel map: [h_det n_h2 | pz_mean n_z | pz_logsd n_z || rz_mean n_z | rz_logsd n_z | down_context n_h2]
        h_det, pz_mean, pz_logsd, rz_mean, rz_logsd, down_context = torch.split(h, [nh2, nz, nz, nz, nz, nh2], dim=1)
        context = (up_context + down_context).contiguous()
    # posterior N(qz.mean + rz_mean, qz.logvar + 2 rz_logsd) with qz.logvar = 2 qz_logsd (models.py:139,275)
    stats = ((qz_mean + rz_mean).contiguous(), (qz_logsd + rz_logsd).contiguous(), pz_mean.contiguous(),
             pz_logsd.contiguous(), context)
    if posterior == "down_iaf2_nl2":
        # models.py:281-291: step(conv1), then step(conv2) in the reversed order; both arw_logsd go into logqs
        from .elbo import stochastic_layer

        def two_steps(z, c):
            z, a1 = iaf_layer.step(name, z, c, 1)
            z, a2 = iaf_layer.step(name, z.contiguous(), c, 2)
            return z, a1 + a2
        z, kl_bc, kl_sum = stochastic_layer(two_steps, eps, *stats)
    else:
        z, kl_bc, kl_sum = iaf_layer(name, eps, *stats)
    hh = torch.cat([h_det, z], dim=1)
    if downsample:
        h_in = upsample_nn(h_in)
    out = h_in + 0.1 * conv2d(w, "%s_down_conv2_%d" % (name, ds), nonlinearity(hh, nl), upsample=ds)
    return out, kl_bc, kl_sum


def _layer_down_q_made(w, name, h_in, h, up_state, eps, iaf_layer, hps, downsample):
    """down_q with prior='made' (models.py:36-38, 304-309, 328): the posterior's final sample z and its logqs, then
    kl = logqs - logps_made(z, made_context) with the prior's own masked stack (``iaf_layer.prior_logp``)."""
    nz, nh2, nl = hps["n_z"], hps["n_h2"], hps["nl"]
    ds = 2 if downsample else 1
    posterior = posterior_of(hps)
    if posterior in UP_POSTERIORS:
        # channel map: [h_det n_h2 | made_context n_h2]; z and logqs come from the bottom-up pass (models.py:215-217)
        h_det, made_context = torch.split(h, [nh2, nh2], dim=1)
        z, logqs = up_state
    else:
        qz_mean, qz_logsd, up_context = up_state
        if posterior in LINEAR:
            # channel map: [h_det n_h2 | made_context n_h2 || rz_mean n_z | rz_logsd n_z]
            h_det, made_context, rz_mean, rz_logsd = torch.split(h, [nh2, nh2, nz, nz], dim=1)
            context = None
        else:
            # channel map: [h_det n_h2 | made_context n_h2 || rz_mean n_z | rz_logsd n_z | down_context n_h2]
            h_det, made_context, rz_mean, rz_logsd, down_context = torch.split(h, [nh2, nh2, nz, nz, nh2], dim=1)
            context = (up_context + down_context).contiguous()
        from .elbo import posterior_sample
        if posterior == "down_iaf2_nl2":
            def steps(z, c):
                z, a1 = iaf_layer.step(name, z, c, 1)
                z, a2 = iaf_layer.step(name, z.contiguous(), c, 2)
                return z, a1 + a2
        else:
            steps = lambda z, c: iaf_layer.step(name, z, c)
        z, logqs = posterior_sample(steps, eps, (qz_mean + rz_mean).contiguous(), (qz_logsd + rz_logsd).contiguous(),
                                    context)
    logp_bc, logp = iaf_layer.prior_logp(name, z.contiguous(), made_context.contiguous())
    kl_bc = logqs.sum(dim=(2, 3)) - logp_bc
    kl_sum = logqs.sum(dim=(1, 2, 3)) - logp
    hh = torch.cat([h_det, z], dim=1)
    if downsample:
        h_in = upsample_nn(h_in)
    out = h_in + 0.1 * conv2d(w, "%s_down_conv2_%d" % (name, ds), nonlinearity(hh, nl), upsample=ds)
    return out, kl_bc, kl_sum


def layer_down_p(w, name, h_in, eps, iaf_layer, hps, downsample):
    """cvae_layer.down_p (models.py:330-359), the generative half of the layer: the prior's sample from the noise eps,
    then down_conv2.  prior='diag': ``z = mean_prior + eps * exp(logsd_prior)`` from down_conv1's prior channels, as the
    reference.  prior='made': the sample of the autoregressive prior with ``made_context = h[:, n_h2:2 n_h2]``, through
    ``iaf_layer.prior_sample(name, eps, made_context) -> z`` (the step run backwards, z = 0.1 m(z) + exp(0.1 s(z)) eps).
    This deliberately replaces the reference's placeholder, which prints "TODO: SAMPLES FROM MADE PRIOR" and uses
    ``z = eps`` (models.py:338-340)."""
    nz, nh2, nl = hps["n_z"], hps["n_h2"], hps["nl"]
    ds = 2 if downsample else 1
    posterior_of(hps)
    h = conv2d(w, name + "_down_conv1", nonlinearity(h_in, nl))
    h_det = h[:, :nh2]
    if prior_of(hps) == "made":
        z = iaf_layer.prior_sample(name, eps.contiguous(), h[:, nh2:2 * nh2].contiguous())
    else:
        z = h[:, nh2:nh2 + nz] + eps * torch.exp(h[:, nh2 + nz:nh2 + 2 * nz])
    hh = torch.cat([h_det, z], dim=1)
    if downsample:
        h_in = upsample_nn(h_in)
    return h_in + 0.1 * conv2d(w, "%s_down_conv2_%d" % (name, ds), nonlinearity(hh, nl), upsample=ds)


def decode(w, eps, iaf_layer, hps):
    """cvae1.f_decoder (models.py:499-521) for px='logistic': noise to a uint8 image [B,3,S,S].  eps[(i, j)]: the
    N(0,1) draw of layer (i, j), the keys ``forward``'s noise uses."""
    depths, nl = hps["depths"], hps["nl"]
    prior_of(hps)
    B = eps[(0, 0)].shape[0]
    size = hps["image_size"] // 2 ** len(depths)
    h = w["h_top"].reshape(1, -1, 1, 1).expand(B, -1, size, size)
    for i in reversed(range(len(depths))):
        for j in reversed(range(depths[i])):
            h = layer_down_p(w, "%d_%d" % (i, j), h, eps[(i, j)], iaf_layer, hps, i > 0 and j == 0)
    out = 0.1 * conv2d(w, "x_dec", nonlinearity(h, nl), upsample=2)
    mean_x = torch.clamp(out + 0.5, 1 / 512.0, 1 - 1 / 512.0)
    return (256.0 * mean_x).to(torch.uint8)


def discretized_logistic_logp(mean, logscale, binsize, sample):
    """graphy/nodes/rand.py:169-178 (.logp)."""
    scale = torch.exp(logscale)
    s = (torch.floor(sample / binsize) * binsize - mean) / scale
    logps = torch.log(torch.sigmoid(s + binsize / scale) - torch.sigmoid(s) + 1e-7)
    return logps.flatten(1).sum(dim=1)


def _image(w, x_uint8):
    return torch.clamp((x_uint8.to(w["h_top"].dtype) + 0.5) / 256.0, 0.0, 1.0)     # models.py:425


def _up_pass(w, x, noise, iaf_layer, hps):
    """cvae_layer.up over all layers: {(i, j): up_state}.  noise is only read by the up posteriors."""
    depths = hps["depths"]
    h = conv2d(w, "x_enc", x - 0.5, downsample=2)
    ups = {}
    for i in range(len(depths)):
        for j in range(depths[i]):
            eps = None if noise is None else noise[(i, j)]
            h, ups[(i, j)] = layer_up(w, "%d_%d" % (i, j), h, hps, i > 0 and j == 0, eps, iaf_layer)
    return ups


def _down_pass(w, ups, noise, iaf_layer, hps, n):
    """cvae_layer.down_q over all layers and the decoder mean, for ``n`` samples per row of ``ups`` (the rows of
    ``noise`` are image-major; each up state is expanded to them layer by layer).  Returns
    ([(cost key, kl_bc, kl_sum)] top layer first, mean_x)."""
    from .elbo import expand_samples
    depths, nl = hps["depths"], hps["nl"]
    B = noise[(0, 0)].shape[0]
    size = hps["image_size"] // 2 ** len(depths)
    h = w["h_top"].reshape(1, -1, 1, 1).expand(B, -1, size, size)
    kls = []
    for i in reversed(range(len(depths))):
        for j in reversed(range(depths[i])):
            up_state = tuple(expand_samples(u, n) for u in ups[(i, j)])
            h, kl_bc, kl_sum = layer_down_q(w, "%d_%d" % (i, j), h, up_state, noise[(i, j)], iaf_layer, hps,
                                            i > 0 and j == 0)
            kls.append(("cost_z%03d_%03d" % (i, j), kl_bc, kl_sum))
    out = 0.1 * conv2d(w, "x_dec", nonlinearity(h, nl), upsample=2)
    return kls, torch.clamp(out + 0.5, 1 / 512.0, 1 - 1 / 512.0)


def forward(w, x_uint8, noise, iaf_layer, hps):
    """cvae1.f_encode_decode (models.py:435-497).  hps: n_z, n_h1, n_h2, depths (list), depth_ar, nl, kl_min,
    image_size.  noise[(i, j)]: the N(0,1) draw of layer (i, j).  Returns the reference's ``results`` entries plus
    bits_per_dim (= mean of ``cost``, what train.py reports)."""
    prior_of(hps)
    x = _image(w, x_uint8)
    results = {}
    obj_kl = torch.zeros((), dtype=x.dtype, device=x.device)
    kls, mean_x = _down_pass(w, _up_pass(w, x, noise, iaf_layer, hps), noise, iaf_layer, hps, 1)
    for key, kl_bc, kl_sum in kls:
        results[key] = kl_sum
        if hps["kl_min"] > 0:        # models.py:458-461: free bits per feature map, averaged over the minibatch
            obj_kl = obj_kl + torch.clamp(kl_bc.mean(dim=0), min=hps["kl_min"]).sum()
        else:
            obj_kl = obj_kl + kl_sum
    logpx = discretized_logistic_logp(mean_x, w["logsd_x"], 1 / 256.0, x)
    num = 3 * hps["image_size"] ** 2
    obj = (logpx - obj_kl) / (num * math.log(2.0))
    results["cost_x"] = -logpx
    results["cost"] = -obj
    results["bits_per_dim"] = (-obj).mean()
    return results


def _elems_per_sample(hps):
    """An upper bound on the elements of one posterior sample's largest tensor: a level-0 conv output or its
    pad-channel input, or an image-sized one."""
    nz, nh1, nh2, S = hps["n_z"], hps["n_h1"], hps["n_h2"], hps["image_size"]
    return max((max(nh1, 2 * nh2 + 4 * nz) + 1) * (S // 2 + 2) ** 2, 4 * (S + 4) ** 2)


def log_likelihood(w, x_uint8, iaf_layer, hps, k, chunk=None, noise=None, seed=0):
    """Importance-sampled log-likelihood with k posterior samples per image, what ``est_marglik = k`` estimates
    (train.py:187-205): ``log_px[b] = log mean_j exp(logpx - sum_layers kl_sum)[b, j]`` in nats, and
    ``bits_per_dim = -mean(log_px) / (prod(shape_x) log 2)`` (train.py:203).

    The log-weight uses the true KL sums, whatever ``kl_min`` is.  This departs from the reference, whose
    ``est_marglik`` reuses the training ``cost``: with kl_min > 0 that contains the free-bits floor (models.py:458-466),
    so its estimate is then not an estimate of log p(x).  With kl_min = 0 the two agree.

    For the down posteriors the up pass does not depend on the noise: it runs once per image and its state is expanded
    over the samples.  For up_iaf2_nl / up_iaf2 the sample is drawn in the up pass (models.py:145-176), so the up pass
    runs per sample.  Chunking, noise(start, count) and the default noise are those of ``iaf_b200.elbo.log_likelihood``;
    noise[(i, j)] is the draw ``forward`` takes.  Runs under no_grad: use the inference wrapper, CudaIAF.
    Returns dict(log_px [B] fp64 nats, bits_per_dim, elbo [B] fp64: the mean log-weight)."""
    from .elbo import LogMeanExp, _check_k_chunk, default_chunk, default_noise, expand_samples
    posterior, depths = posterior_of(hps), hps["depths"]
    prior_of(hps)
    _check_k_chunk(k, chunk)
    k = int(k)
    B, S = x_uint8.shape[0], hps["image_size"]
    dev, dt = w["h_top"].device, w["h_top"].dtype
    chunk = default_chunk(B, k, _elems_per_sample(hps)) if chunk is None else min(int(chunk), k)
    if noise is None:
        shapes = {(i, j): (B, hps["n_z"], S // 2 ** (i + 1), S // 2 ** (i + 1))
                  for i in range(len(depths)) for j in range(depths[i])}
        noise = default_noise(shapes, dev, dt, seed)
    with torch.no_grad():
        x = _image(w, x_uint8)
        shared = None if posterior in UP_POSTERIORS else _up_pass(w, x, None, iaf_layer, hps)
        acc = LogMeanExp(B, dev)
        for start in range(0, k, chunk):
            n = min(chunk, k - start)
            eps = noise(start, n)
            xs = expand_samples(x, n)
            if shared is None:
                kls, mean_x = _down_pass(w, _up_pass(w, xs, eps, iaf_layer, hps), eps, iaf_layer, hps, 1)
            else:
                kls, mean_x = _down_pass(w, shared, eps, iaf_layer, hps, n)
            logw = discretized_logistic_logp(mean_x, w["logsd_x"], 1 / 256.0, xs).double()
            for _, _, kl_sum in kls:
                logw = logw - kl_sum.double()
            acc.add(logw.reshape(B, n))
        log_px, mean_w = acc.result()
    return dict(log_px=log_px, bits_per_dim=-log_px.mean() / (3 * S * S * math.log(2.0)), elbo=mean_w)


def train_step(w, x_uint8, opt, hps, noise=None, iaf_layer=None, sharded=False, group=None):
    """One training step of the Theano model, ``f_train`` (models.py:563-573), then ``opt.step()``.  ``w``: leaf tensors
    (fp32 CUDA for :mod:`iaf_b200.optim`); ``opt`` updates them in place.  ``noise[(i, j)]``: the N(0, 1) draw of layer
    (i, j) for the global batch (default: torch.randn on the parameters' device).  ``sharded=True`` (or a ``group``):
    this rank takes its contiguous slice of the batch and the ranks' gradients are averaged before the step, as
    :func:`iaf_b200.elbo.train_step`.  Returns the step's bits/dim (a tensor).

    * ``optim='adamax'`` (:class:`iaf_b200.optim.Adamax`, ``rule="theano"``): the gradient of ``cost.sum()``
      (optim.py:102) at ``w``, which must require grad.  ``iaf_layer``: default ``CudaIAFTrain(w, hps)``, built per call
      -- pass one to keep its operators across steps.
    * ``optim='eve'`` (an ``opt`` with ``lookahead()``, :class:`iaf_b200.optim.Eve`): the gradient of the global batch's
      MEAN cost (optim.py:138) at ``opt.lookahead()``, where the forward runs; the bits/dim returned are those at the
      lookahead, what the reference's ``f_train`` returns.  Sharded, each rank's objective is its cost sum times
      world / B, so the ranks' average is the global mean for any shard sizes.  ``iaf_layer``: default
      ``CudaIAFTrain(opt.lookahead(), hps)``; a layer bound to other tensors is refused."""
    import torch.distributed as dist
    from .elbo import run_train_step
    lookahead = getattr(opt, "lookahead", None)
    wf = w if lookahead is None else lookahead()
    if iaf_layer is None:
        iaf_layer = CudaIAFTrain(wf, hps)
    elif lookahead is not None:
        bound = getattr(iaf_layer, "w", None)
        if bound is None or any(bound.get(k) is not v for k, v in wf.items()):
            raise ValueError("train_step: with Eve the iaf_layer must be bound to opt.lookahead(), where the gradient "
                             "is taken")
    S, B = hps["image_size"], x_uint8.shape[0]
    if noise is None:
        h = w["h_top"]
        noise = {(i, j): torch.randn((B, hps["n_z"], S // 2 ** (i + 1), S // 2 ** (i + 1)), device=h.device, dtype=h.dtype)
                 for i in range(len(hps["depths"])) for j in range(hps["depths"][i])}
    world = 1
    if (sharded or group is not None) and dist.is_initialized():
        world = dist.get_world_size(group)

    def objective(x, nz):
        out = forward(wf, x, nz, iaf_layer, hps)
        obj = out["cost"].sum()
        if lookahead is not None:
            obj = obj * (world / B)  # the towers' average of these is the global batch's mean cost
        return obj, out["bits_per_dim"]
    return run_train_step(wf, x_uint8, opt, noise, objective, 1.0, sharded, group)


def make_optimizer(w, hps):
    """cvae1's optimiser (models.py:563-573) over ``w``: ``hps.get("optim", "adamax")`` selects
    ``Adamax(w, rule="theano")`` or ``Eve(w)``; ``alpha``, ``beta1`` and ``beta2`` in ``hps`` (cvae1's argument names;
    alpha is the learning rate) override the defaults."""
    from .optim import Adamax, Eve
    name = hps.get("optim", "adamax")
    hp = dict(lr=hps.get("alpha"), beta1=hps.get("beta1"), beta2=hps.get("beta2"))
    if name == "adamax":
        return Adamax(w, rule="theano", **hp)
    if name == "eve":
        return Eve(w, **hp)
    raise ValueError("make_optimizer: unknown optim %r (the reference has 'adamax' and 'eve')" % (name,))


def make_params(hps, seed=0, dtype=np.float32):
    """Seeded synthetic parameters under the reference's Theano names and shapes (no checkpoint exists offline)."""
    rng = np.random.RandomState(seed)
    nz, nh1, nh2, depths = hps["n_z"], hps["n_h1"], hps["n_h2"], hps["depths"]
    posterior = posterior_of(hps)
    up_post, linear = posterior in UP_POSTERIORS, posterior in LINEAR
    made = prior_of(hps) == "made"
    n_ctx = 0 if linear else nh2                       # the context channels of up_conv1 / down_conv1
    w = {}

    def conv(name, cin, cout, k, pad_channel=True):
        w[name + "_w"] = (0.05 * rng.randn(cout, cin + (1 if pad_channel else 0), k, k)).astype(dtype)
        w[name + "_b"] = (0.05 * rng.randn(cout)).astype(dtype)
        w[name + "_s"] = rng.uniform(-0.1, 0.1, size=(cout,)).astype(dtype)

    conv("x_enc", 3, nh1, 5)
    conv("x_dec", nh1, 3 * 4, 5)                       # upsample=2: n_out * 2**2 maps before depth-to-space
    w["logsd_x"] = np.asarray(-1.0, dtype=dtype)
    w["h_top"] = (0.1 * rng.randn(nh1)).astype(dtype)
    for i in range(len(depths)):
        for j in range(depths[i]):
            n = "%d_%d" % (i, j)
            ds = 2 if (i > 0 and j == 0) else 1
            conv("%s_up_conv1_%d" % (n, ds), nh1, nh2 + 2 * nz + n_ctx, 3)
            conv(n + "_up_conv2", nh2 + nz if up_post else nh2, nh1, 3)                       # models.py:25,55-84
            conv(n + "_down_conv1", nh1, (2 * nh2 if made else nh2 + 2 * nz) + (0 if up_post else 2 * nz + n_ctx),
                 3)                                                    # models.py:27-28,36-38,79-86
            conv("%s_down_conv2_%d" % (n, ds), nh2 + nz, nh1 * ds * ds, 3)
            sizes = [nz] + hps["depth_ar"] * [nh2]
            if linear:                                                 # ar.conv2d(n_z, 2 n_z): rows interleave the heads
                conv("%s_posterior_conv1" % n, nz, 2 * nz, 3)
            else:
                for k in range(hps["depth_ar"]):
                    conv("%s_posterior_conv1_%d" % (n, k), sizes[k], sizes[k + 1], 3)
                for k in range(2):
                    conv("%s_posterior_conv1_out_%d" % (n, k), sizes[-1], nz, 3)
            if posterior == "down_iaf2_nl2":                           # models.py:98
                for k in range(hps["depth_ar"]):
                    conv("%s_posterior_conv2_%d" % (n, k), sizes[k], sizes[k + 1], 3)
                for k in range(2):
                    conv("%s_posterior_conv2_out_%d" % (n, k), sizes[-1], nz, 3)
            if made:                                                   # models.py:36-38
                for k in range(hps["depth_ar"]):
                    conv("%s_prior_conv1_%d" % (n, k), sizes[k], sizes[k + 1], 3)
                for k in range(2):
                    conv("%s_prior_conv1_out_%d" % (n, k), sizes[-1], nz, 3)
    return w


def _data_init(w, name, h, inv_stdev, eps):
    """The data-dependent branch of a conv on its output h (bias included): conv.py:225-250 with ``inv_stdev`` 1 /
    init_stdev and ``eps`` 1e-7, ar.py:331-353 with 1 and 0.  ``std = data_std inv_stdev + eps`` from the population
    std over (0, 2, 3), ``_s = -log(std) / 3``, h / std, ``_b = -mean`` of that; returns the standardised h.  When a
    channel's std is exactly 0 the conv keeps its parameters and returns h, with the reference's warning."""
    data_std = h.std(dim=(0, 2, 3), unbiased=False)
    num_zeros = int((data_std == 0).sum())
    if num_zeros > 0:
        warnings.warn("Stdev=0 for %d features in %s. Skipping data-dependent init." % (num_zeros, name))
        return h
    std = data_std * inv_stdev + eps
    w[name + "_s"] = -torch.log(std) / LOGSCALE_SCALE
    h = h / std.reshape(1, -1, 1, 1)
    mean = h.mean(dim=(0, 2, 3))
    w[name + "_b"] = -mean
    return h - mean.reshape(1, -1, 1, 1)


def _init_ar_conv2d(w, name, h, zerodiagonal, flipmask):
    """ar.conv2d (graphy/nodes/ar.py:241-353) in the init pass: the mask (masks.py), l2normalize with its zeroed centre
    rows and 1e-8 (ar.py:267-281), exp(3 s), the pad channel, TRUE convolution, bias, then the data-dependent branch."""
    W, s, b = w[name + "_w"], w[name + "_s"], w[name + "_b"]
    n_out, n_in = W.shape[0], W.shape[1] - 1
    kerns = torch.from_numpy(theano_conv_ar_mask(n_in, n_out, zerodiagonal=zerodiagonal, flipmask=flipmask)).to(W) * W
    if zerodiagonal:
        keep = torch.ones_like(kerns)
        keep[:n_out // n_in if n_out >= n_in else 1, :, 1, 1] = 0
        kerns = kerns * keep
    kerns = kerns * (1.0 / (torch.sqrt((kerns ** 2).sum(dim=(1, 2, 3), keepdim=True)) + 1e-8))
    kerns = kerns * torch.exp(LOGSCALE_SCALE * s).reshape(-1, 1, 1, 1)
    y = F.conv2d(pad2dwithchannel(h, 3), kerns.flip(2, 3)) + b.reshape(1, -1, 1, 1)
    return _data_init(w, name, y, 1.0, 0.0)


class _InitLayer(object):
    """iaf_layer of the init pass: the masked convs of every posterior and prior stack run in init mode, in the order
    ``f_encode_decode`` runs them, with the operator's formulas around them (models.py:168-176, 272-291, 304-309).
    Records each stack's input in ``stacks``."""

    def __init__(self, w, hps):
        self.w, self.hps, self.stacks = w, hps, {}

    def _stack(self, pre, z, context, flipmask=False):
        """multiconv2d (ar.py:396-416) -> [mean, logsd]; the linear IAF's one conv with its rows interleaving them."""
        self.stacks[pre] = (z, context)
        if pre.endswith("_posterior_conv1") and posterior_of(self.hps) in LINEAR:
            out = _init_ar_conv2d(self.w, pre, z, True, False)
            return out[:, ::2], out[:, 1::2]
        h = z
        for k in range(self.hps["depth_ar"]):
            h = _init_ar_conv2d(self.w, "%s_%d" % (pre, k), h, False, flipmask)
            if k == 0:
                h = h + context
            h = nonlinearity(h, self.hps["nl"])
        return [_init_ar_conv2d(self.w, "%s_out_%d" % (pre, k), h, True, flipmask) for k in range(2)]

    def step(self, name, z, context, conv=1):
        mean, logsd = self._stack("%s_posterior_conv%d" % (name, conv), z, context, flipmask=conv == 2)
        arw_logsd = 0.1 * logsd
        return (z - 0.1 * mean) / torch.exp(arw_logsd), arw_logsd

    def __call__(self, name, eps, post_mean, post_logsd, prior_mean, prior_logsd, context):
        from .elbo import stochastic_layer
        return stochastic_layer(lambda z, c: self.step(name, z, c), eps, post_mean, post_logsd, prior_mean, prior_logsd,
                                context)

    def prior_logp(self, name, z, context):
        mean, logsd = self._stack("%s_prior_conv1" % name, z, context)
        logps = gaussian_logps(0.1 * mean, 2 * (0.1 * logsd), z)
        return logps.sum(dim=(2, 3)), logps.sum(dim=(1, 2, 3))


def data_init_pass(w, x_uint8, hps, noise=None, seed=0):
    """:func:`data_init` with what the pass saw: (w, results, stacks).  ``results`` is :func:`forward`'s dict for the
    init pass; ``stacks[name] = (z, context)`` is the input the masked stack ``name`` (``{i}_{j}_posterior_conv{1,2}``,
    ``{i}_{j}_prior_conv1``) was initialised on."""
    posterior_of(hps)
    prior_of(hps)
    if noise is None:
        from .elbo import default_noise
        B, S, depths = x_uint8.shape[0], hps["image_size"], hps["depths"]
        shapes = {(i, j): (B, hps["n_z"], S // 2 ** (i + 1), S // 2 ** (i + 1))
                  for i in range(len(depths)) for j in range(depths[i])}
        noise = default_noise(shapes, w["h_top"].device, w["h_top"].dtype, seed)(0, 1)
    p = InitPass(w)
    layer = _InitLayer(p, hps)
    with torch.no_grad():
        results = forward(p, x_uint8, noise, layer, hps)
    return dict(p), results, layer.stacks


def data_init(w, x_uint8, hps, noise=None, seed=0):
    """The reference's data-dependent initialisation, ``cvae1(..., data_init={'x': x})`` (models.py:540-544: one
    ``f_encode_decode`` with ``w['__init']`` set) on the batch ``x_uint8``: returns a new dict with the ``_s`` and
    ``_b`` of every conv set from the batch's statistics.  The plain convs (x_enc, x_dec, up_conv1/2, down_conv1/2) take
    conv.py:225-250: ``std = data_std / 0.1 + 1e-7``; every masked conv (the posterior stacks, the flipped second stack
    of down_iaf2_nl2, the linear IAF's conv with its interleaved rows, the MADE prior's ``prior_conv1``), heads
    included, takes ar.py:331-353: ``std = data_std``.  Then ``_s = -log(std) / 3`` and ``_b = -mean`` of the rescaled
    output.  A conv with a channel of std exactly 0 skips its init, warning as the reference prints.  Every ``_w``,
    ``h_top`` and ``logsd_x`` is passed through.

    The pass is :func:`forward` in stock torch ops on the device and dtype of ``w`` (tensors), the posterior sampled from
    the noise as in training.  noise[(i, j)]: the N(0, 1) draw of layer (i, j) (the shapes :func:`forward` takes);
    default: torch.randn from one generator seeded with ``seed``."""
    return data_init_pass(w, x_uint8, hps, noise, seed)[0]


class CudaIAF(object):
    """iaf_layer callable backed by the fused CUDA operator, Theano variant: one IAFOperator per layer name and
    posterior conv (conv 2, down_iaf2_nl2's second step, is the flipmask operator)."""

    def __init__(self, w, hps, path="auto"):
        from .ops import IAFOperator
        self.w, self.hps, self.path, self.IAFOperator, self.ops = w, hps, path, IAFOperator, {}
        self.prior_ops = {}  # prior='made': layer name -> the prior's operator (prior_conv1, models.py:36-38)

    def _linear(self, conv):
        return conv != 0 and posterior_of(self.hps) in LINEAR

    def _new_op(self, conv):
        nz, nh2, dar = self.hps["n_z"], self.hps["n_h2"], self.hps["depth_ar"]
        hidden = [] if self._linear(conv) else dar * [nh2]             # the linear IAF: no hidden layer, no context
        return self.IAFOperator("theano", nz, hidden, [nz, nz], nl=self.hps["nl"], path=self.path,
                                flipmask=conv == 2)                    # models.py:36-38,92,97-98 (conv 0: the prior)

    def _posterior_layers(self, name, conv, convert):
        """The (w, s, b) triples of posterior conv ``conv``, each tensor passed through ``convert``: the stack's, or the
        linear IAF's one conv with its interleaved rows split into the two heads."""
        pre = "%s_posterior_conv%d" % (name, conv)
        if self._linear(conv):
            return deinterleave_heads(*(convert(self.w[pre + "_" + k]) for k in "wsb"))
        dar = self.hps["depth_ar"]
        names = ["%s_%d" % (pre, i) for i in range(dar)] + ["%s_out_%d" % (pre, k) for k in range(2)]
        return [tuple(convert(self.w[n + "_" + k]) for k in "wsb") for n in names]

    def _prior_op(self, name, device):
        op = self.prior_ops.get(name)
        if op is None:
            from .weights import theano_layers
            op = self._new_op(0)
            op.set_weights(theano_layers(self.w, "%s_prior_conv1" % name, self.hps["depth_ar"], device=device))
            self.prior_ops[name] = op
        return op

    def prior_logp(self, name, z, context):
        """prior='made': log-density of the autoregressive prior at the posterior's final sample z with the context
        made_context (models.py:304-309), summed per (sample, channel) and per sample -> (logp_bc [B,C], logp [B])."""
        _, logp_bc, logp = self._prior_op(name, z.device).ar_logp(z, context)
        return logp_bc, logp

    def prior_sample(self, name, eps, context):
        """prior='made': a sample of the autoregressive prior from the noise eps with the context made_context
        (IAFOperator.ar_sample: the step inverted, in the mask's order).  Not differentiable: runs under no_grad."""
        with torch.no_grad():
            return self._prior_op(name, eps.device).ar_sample(eps, context)[0]

    def _op(self, name, device, conv=1):
        op = self.ops.get((name, conv))
        if op is None:
            from .weights import _as_f32
            op = self._new_op(conv)
            op.set_weights(self._posterior_layers(name, conv, lambda a: _as_f32(a, device)))
            self.ops[(name, conv)] = op
        return op

    def invalidate(self):
        """The inference wrapper converts ``w`` (numpy or torch) to device tensors ONCE per layer; after changing or
        replacing entries of ``w`` call this so the next evaluation re-imports and re-packs them."""
        self.ops.clear()
        self.prior_ops.clear()
        return self

    def __call__(self, name, eps, post_mean, post_logsd, prior_mean, prior_logsd, context):
        z, _, kl_bc, kl_cost = self._op(name, eps.device).layer(eps, post_mean, post_logsd, prior_mean, prior_logsd,
                                                                context, want_kl=False)
        return z, kl_bc, kl_cost

    def step(self, name, z, context, conv=1):
        """The bare step of posterior conv ``conv`` (models.py:170-173; 281-291) -> (z', arw_logsd)."""
        z_new, arw_logsd, _ = self._op(name, z.device, conv).step(z, context)
        return z_new, arw_logsd


class CudaIAFTrain(CudaIAF):
    """Differentiable iaf_layer for training through the Theano front-end (what ``T.grad`` over cvae1's cost gives the
    reference, graphy/misc/optim.py:99-123): the posterior sample, logqs, prior logps and the KL sums are torch ops
    (models.py:273-298) around ``IAFOperator.step``, whose autograd node runs iaf_step_fwd_train / iaf_step_bwd_saved
    (SURVEY 8f-4).  The parameter tensors are re-bound on every call so gradients flow to the entries of ``w``
    (``{name}_posterior_conv{1,2}_{k}_w/_s/_b``), with masked taps at exactly zero (ar.py:369-373)."""

    def _op(self, name, device, conv=1):
        op = self.ops.get((name, conv))
        if op is None:
            op = self._new_op(conv)
            self.ops[(name, conv)] = op
        # the live tensors of w (float32, on the device): not detached, so their .grad is filled by backward().  The linear
        # IAF's rows are split on every call, inside autograd, so its gradient lands interleaved in w[...]
        op.set_weights(self._posterior_layers(name, conv, lambda t: t))
        return op

    def _prior_op(self, name, device):
        op = self.prior_ops.get(name)
        if op is None:
            op = self._new_op(0)
            self.prior_ops[name] = op
        pre, dar = "%s_prior_conv1" % name, self.hps["depth_ar"]
        names = ["%s_%d" % (pre, i) for i in range(dar)] + ["%s_out_%d" % (pre, k) for k in range(2)]
        # the live tensors of w, as for the posterior convs: IAFOperator.ar_logp records one autograd node
        op.set_weights([(self.w[n + "_w"], self.w[n + "_s"], self.w[n + "_b"]) for n in names])
        return op

    def __call__(self, name, eps, post_mean, post_logsd, prior_mean, prior_logsd, context):
        from .elbo import stochastic_layer
        op = self._op(name, eps.device)
        return stochastic_layer(lambda z, c: op.step(z, c, want_logdet=False)[:2], eps, post_mean, post_logsd, prior_mean,
                                prior_logsd, context)
