"""ELBO forward around the IAF operator (SURVEY 8f-2): the TF model's `CVAE1._forward`
(tf_train.py:161-219) with `IAFLayer.up/down` (tf_train.py:29-95), restated in PyTorch so that
bits/dim can be compared between the CUDA operator and the oracle operator on identical weights
and inputs ("bits/dim parity" in BASELINE.json's metric).

Only the stochastic-layer block (posterior sample -> IAF step -> KL) is the hot path and goes
through the pluggable ``iaf_layer`` callable; everything else here is plumbing (weight-normed
conv / deconv, elu, discretized logistic) expressed with stock torch ops on whatever device and
dtype the parameters live on.  Parameters are a dict under the reference's TF variable names:
``x_enc/{V,g,b}``, ``IAF_{i}_{j}/{up_conv1,up_conv3,down_conv1,down_conv2|down_deconv2}/{V,g,b}``,
``IAF_{i}_{j}/ar_multiconv2d/layer_{k}|layer_out_{k}/{V,g,b}``, ``h_top``, ``dec_log_stdv``, ``x_dec/{V,g,b}``.
:func:`data_init` is the reference's data-dependent initialisation of all of them (mode "init").
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from .masks import tf_conv_ar_mask


def _same_pad(n, k, s):
    out = -(-n // s)
    total = max((out - 1) * s + k - n, 0)
    return total // 2, total - total // 2


def _conv_same(x, w, stride):
    """tf.nn.conv2d, SAME padding, NCHW input, filter [kh,kw,Cin,Cout]."""
    pt, pb = _same_pad(x.shape[2], w.shape[0], stride)
    pl, pr = _same_pad(x.shape[3], w.shape[1], stride)
    return F.conv2d(F.pad(x, (pl, pr, pt, pb)), w.permute(3, 2, 0, 1), stride=stride)


def _deconv_same(x, w, stride):
    """my_deconv2d (layers.py:67-76): conv2d_transpose, SAME padding, filter [kh,kw,Cout,Cin]."""
    H, W = x.shape[2] * stride, x.shape[3] * stride
    y = F.conv_transpose2d(x, w.permute(3, 2, 0, 1), stride=stride)  # full output (H-1)*s + k
    pt, _ = _same_pad(H, w.shape[0], stride)
    pl, _ = _same_pad(W, w.shape[1], stride)
    return y[:, :, pt:pt + H, pl:pl + W]


def _l2_normalize(v):
    """tf.nn.l2_normalize(v, [0, 1, 2]) = v * rsqrt(max(sum(v^2), 1e-12))."""
    return v * torch.rsqrt(torch.clamp((v * v).sum(dim=(0, 1, 2), keepdim=True), min=1e-12))


def conv2d(params, name, x, stride=1):
    """tf_utils/layers.py:31-64 (run-time branch, mask=None): w = exp(g) * l2_normalize(V,[0,1,2]); SAME padding.
    During :func:`data_init` the init branch (layers.py:38-51) instead."""
    if isinstance(params, InitPass):
        return params.init(name, _conv_same(x, _l2_normalize(params[name + "/V"]), stride), 0.1)
    V, g, b = params[name + "/V"], params[name + "/g"], params[name + "/b"]
    w = torch.exp(g).reshape(1, 1, 1, -1) * V * torch.rsqrt(torch.clamp((V * V).sum(dim=(0, 1, 2), keepdim=True), min=1e-12))
    return _conv_same(x, w, stride) + b.reshape(1, -1, 1, 1)


def deconv2d(params, name, x, stride=2):
    """tf_utils/layers.py:67-112: conv2d_transpose, SAME, filter [kh,kw,Cout,Cin], weight norm over [0,1,2] -> per Cin.
    During :func:`data_init` the init branch (layers.py:86-100) instead."""
    if isinstance(params, InitPass):
        return params.init(name, _deconv_same(x, _l2_normalize(params[name + "/V"]), stride), 0.1)
    V, g, b = params[name + "/V"], params[name + "/g"], params[name + "/b"]
    # layers.py:108: w = reshape(exp(g), [1,1,num_filters,1]) * l2_normalize(v, [0,1,2])
    w = torch.exp(g).reshape(1, 1, -1, 1) * V * torch.rsqrt(torch.clamp((V * V).sum(dim=(0, 1, 2), keepdim=True), min=1e-12))
    return _deconv_same(x, w, stride) + b.reshape(1, -1, 1, 1)


def resize_nearest_neighbor(x, scale):
    """tf_utils/layers.py:169-175."""
    if scale == 0.5:
        return x[:, :, ::2, ::2]
    return x.repeat_interleave(int(scale), dim=2).repeat_interleave(int(scale), dim=3)


def discretized_logistic(mean, logscale, sample, binsize=1 / 256.0):
    """tf_utils/distributions.py:28-32."""
    scale = torch.exp(logscale)
    s = (torch.floor(sample / binsize) * binsize - mean) / scale
    logp = torch.log(torch.sigmoid(s + binsize / scale) - torch.sigmoid(s) + 1e-7)
    return logp.sum(dim=(1, 2, 3))


def _layers(hps):
    return [(i, j) for i in range(hps["depth"]) for j in range(hps["num_blocks"])]


def _image(params, x_uint8):
    x = x_uint8.to(params["h_top"].dtype)
    return torch.clamp((x + 0.5) / 256.0, 0.0, 1.0) - 0.5       # tf_train.py:164-165


def expand_samples(t, n):
    """[B, ...] -> [B n, ...]: every image's row repeated n times, image-major (distributions.py:41-52, ``repeat``)."""
    return t if t is None or n == 1 else t.repeat_interleave(n, dim=0)


def _up_pass(params, x, hps):
    """IAFLayer.up over all layers (tf_train.py:29-44): {(i, j): (qz_mean, qz_logsd, up_context)}.  It does not depend
    on the posterior's noise."""
    zs, hs = hps["z_size"], hps["h_size"]
    h = conv2d(params, "x_enc", x, stride=2)
    up = {}
    for (i, j) in _layers(hps):
        sc = "IAF_%d_%d" % (i, j)
        down = (i > 0) and (j == 0)
        t = conv2d(params, sc + "/up_conv1", F.elu(h), stride=2 if down else 1)
        qz_mean, qz_logsd, up_context, hh = torch.split(t, [zs, zs, hs, hs], dim=1)
        up[(i, j)] = (qz_mean, qz_logsd, up_context)
        hh = conv2d(params, sc + "/up_conv3", F.elu(hh))
        if down:
            h = resize_nearest_neighbor(h, 0.5)
        h = h + 0.1 * hh
    return up


def _down_pass(params, up, noise, iaf_layer, hps, n, free_bits=True):
    """IAFLayer.down over all layers (tf_train.py:46-95) and the decoder mean, for ``n`` posterior samples per image:
    the rows of ``noise`` are image-major, and ``up`` (one row per image) is expanded to them layer by layer.
    Returns (kl_obj, kl_cost, xd); kl_obj is kl_cost when ``free_bits`` is False."""
    zs, hs = hps["z_size"], hps["h_size"]
    B = next(iter(noise.values())).shape[0]
    size = hps["image_size"] // 2 ** hps["depth"]
    h = params["h_top"].reshape(1, -1, 1, 1).expand(B, hs, size, size)
    kl_obj = torch.zeros(B, dtype=h.dtype, device=h.device)
    kl_cost = torch.zeros(B, dtype=h.dtype, device=h.device)
    for (i, j) in reversed(_layers(hps)):
        sc = "IAF_%d_%d" % (i, j)
        down = (i > 0) and (j == 0)
        t = conv2d(params, sc + "/down_conv1", F.elu(h))
        pz_mean, pz_logsd, rz_mean, rz_logsd, down_context, h_det = torch.split(t, [zs] * 4 + [hs] * 2, dim=1)
        qz_mean, qz_logsd, up_context = (expand_samples(u, n) for u in up[(i, j)])
        z, kl_bc, cost = iaf_layer(sc, noise[(i, j)], (rz_mean + qz_mean).contiguous(), (rz_logsd + qz_logsd).contiguous(),
                                   pz_mean.contiguous(), pz_logsd.contiguous(), (up_context + down_context).contiguous())
        if free_bits and hps["kl_min"] > 0:                       # tf_train.py:77-83: free bits, batch mean is local
            obj = torch.clamp(kl_bc.mean(dim=0, keepdim=True), min=hps["kl_min"]).expand(B, -1).sum(dim=1)
        else:
            obj = cost
        kl_obj = kl_obj + obj
        kl_cost = kl_cost + cost
        hh = F.elu(torch.cat([z, h_det], dim=1))
        if down:
            h = resize_nearest_neighbor(h, 2)
            hh = deconv2d(params, sc + "/down_deconv2", hh)
        else:
            hh = conv2d(params, sc + "/down_conv2", hh)
        h = h + 0.1 * hh
    xd = deconv2d(params, "x_dec", F.elu(h))
    return kl_obj, kl_cost, torch.clamp(xd, -0.5 + 1 / 512.0, 0.5 - 1 / 512.0)


def forward(params, x_uint8, noise, iaf_layer, hps):
    """bits/dim and the per-sample pieces for one batch.

    hps: dict(z_size, h_size, depth, num_blocks, kl_min, image_size).  noise[(i, j)]: the N(0,1) draw of
    layer (i, j)'s posterior (tf_train.py:57).  iaf_layer(scope, eps, post_mean, post_logsd, prior_mean,
    prior_logsd, context) -> (z, kl_bc [B,C], kl_cost [B])."""
    orig_x = _image(params, x_uint8)
    B = orig_x.shape[0]
    kl_obj, kl_cost, xd = _down_pass(params, _up_pass(params, orig_x, hps), noise, iaf_layer, hps, 1)
    log_pxz = discretized_logistic(xd, params["dec_log_stdv"], orig_x)
    loss = (kl_cost - log_pxz).sum()                              # compute_lowerbound, k = 1 (distributions.py:55-57)
    num_pixels = 3 * hps["image_size"] ** 2
    return dict(bits_per_dim=loss / (math.log(2.0) * num_pixels * B), obj=(kl_obj - log_pxz).sum(), kl_cost=kl_cost,
                kl_obj=kl_obj, log_pxz=log_pxz)


class LogMeanExp(object):
    """Streaming per-image ``log (1/k) sum_j exp(w_j)`` in fp64: a running max and a sum scaled by it, so chunks of
    log-weights near -1e4 with a spread of 1e3 neither overflow nor underflow.  Also keeps the plain sum of the
    log-weights (their mean is the ELBO of the same samples)."""

    def __init__(self, n_images, device):
        self.max = torch.full((n_images,), -math.inf, dtype=torch.float64, device=device)
        self.scaled = torch.zeros(n_images, dtype=torch.float64, device=device)
        self.total = torch.zeros(n_images, dtype=torch.float64, device=device)
        self.count = 0

    def add(self, w):
        """w: [n_images, c] log-weights of c more samples of every image."""
        w = w.to(torch.float64)
        m = torch.maximum(self.max, w.max(dim=1).values)
        self.scaled = self.scaled * torch.exp(self.max - m) + torch.exp(w - m[:, None]).sum(dim=1)
        self.max = m
        self.total = self.total + w.sum(dim=1)
        self.count += w.shape[1]

    def result(self):
        """(log mean exp [n_images], mean [n_images]) over every sample added."""
        return self.max + torch.log(self.scaled) - math.log(self.count), self.total / self.count


# every tensor of one estimator call stays below 2^31 elements: the kernels index memory in 64 bits, but their sample and
# tensor-core slot indices are 32-bit ints, and the slot stream refuses a call past 2^31 slots (iaf_tc.cu, tc_num_tiles)
MAX_ELEMS = 2 ** 31 - 1
# and at most this many samples per call: every layer's operator keeps its own kernel scratch, sized for the largest
# call it has seen (about 0.1 MB per sample and layer at h_size 160), so memory grows with the samples per call times
# the layers.  4096 samples fill the H100 many times over; the README's TF eval model (20 layers) at 100 images and
# 119 samples each (the index bound) ran out of 80 GB.
MAX_SAMPLES = 4096


def default_chunk(n_images, k, elems_per_sample):
    """Samples per image of one call: the largest that keeps every tensor below 2^31 elements and the call at most
    MAX_SAMPLES samples, at most k, at least 1."""
    return max(1, min(k, MAX_ELEMS // (n_images * elems_per_sample), MAX_SAMPLES // n_images))


def _elems_per_sample(hps):
    """An upper bound on the elements of one posterior sample's largest tensor (down_conv1's output, the padded input
    of the encoder and the decoder's full transposed-conv output are the candidates)."""
    zs, hs, S = hps["z_size"], hps["h_size"], hps["image_size"]
    return max((4 * zs + 2 * hs + 1) * (S // 2 + 4) ** 2, 4 * (S + 4) ** 2)


def default_noise(shapes, device, dtype, seed=0):
    """noise(start, count): torch.randn from ONE seeded generator on ``device``, drawn chunk by chunk, so the draws (and
    the estimate) depend on the chunk size.  shapes: {(i, j): (B, C, H, W)}."""
    gen = torch.Generator(device=device)
    gen.manual_seed(seed)

    def noise(start, count):
        return {key: torch.randn((B * count,) + tuple(s), generator=gen, device=device, dtype=dtype)
                for key, (B, *s) in sorted(shapes.items())}
    return noise


def _noise_shapes(hps, B):
    zs, S = hps["z_size"], hps["image_size"]
    return {(i, j): (B, zs, S // 2 ** (i + 1), S // 2 ** (i + 1)) for (i, j) in _layers(hps)}


def _check_k_chunk(k, chunk):
    if int(k) < 1 or (chunk is not None and int(chunk) < 1):
        raise ValueError("k and chunk must be positive")


def log_likelihood(params, x_uint8, iaf_layer, hps, k, chunk=None, noise=None, seed=0):
    """Importance-sampled log-likelihood with k posterior samples per image (tf_train.py:167-170, 218 at ``hps.k = k``;
    ``compute_lowerbound``, distributions.py:55-62): ``log_px[b] = -log k + logsumexp_j (log_pxz - kl_cost)[b, j]``, with
    the true KL sum ``kl_cost`` (never the free-bits objective).

    The up pass does not depend on the noise: it runs once per image, and its posterior statistics and context are
    expanded over the samples.  Samples are processed ``chunk`` per image at a time (image-major, as ``repeat`` lays them
    out) and reduced into a running fp64 log-sum-exp, so memory is bounded by B * chunk samples whatever k is.  Default
    chunk: the largest that keeps every tensor of one call below 2^31 elements and the call at most MAX_SAMPLES samples
    (:func:`default_chunk`).  noise(start, count) ->
    {(i, j): [B count, z_size, s, s]}: samples [start, start + count) of every image; default: torch.randn from one
    generator seeded with ``seed`` on the parameters' device.  An evaluation: runs under no_grad and records no graph
    (use the inference wrapper, CudaIAF).

    Returns dict(log_px [B] fp64 nats, bits_per_dim (tf_train.py:142), elbo [B] fp64: the mean log-weight)."""
    _check_k_chunk(k, chunk)
    k = int(k)
    B = x_uint8.shape[0]
    dev, dt = params["h_top"].device, params["h_top"].dtype
    chunk = default_chunk(B, k, _elems_per_sample(hps)) if chunk is None else min(int(chunk), k)
    if noise is None:
        noise = default_noise(_noise_shapes(hps, B), dev, dt, seed)
    with torch.no_grad():
        x = _image(params, x_uint8)
        up = _up_pass(params, x, hps)
        acc = LogMeanExp(B, dev)
        for start in range(0, k, chunk):
            n = min(chunk, k - start)
            _, kl_cost, xd = _down_pass(params, up, noise(start, n), iaf_layer, hps, n, free_bits=False)
            log_pxz = discretized_logistic(xd, params["dec_log_stdv"], expand_samples(x, n))
            acc.add((log_pxz.double() - kl_cost.double()).reshape(B, n))
        log_px, mean_w = acc.result()
    num_pixels = 3 * hps["image_size"] ** 2
    return dict(log_px=log_px, bits_per_dim=(-log_px).sum() / (math.log(2.0) * num_pixels * B), elbo=mean_w)


def make_params(hps, seed=0, dtype=np.float32):
    """Seeded synthetic parameters under the reference's TF variable names (no checkpoint exists offline)."""
    rng = np.random.RandomState(seed)
    zs, hs = hps["z_size"], hps["h_size"]
    p = {}

    def conv(name, kh, kw, cin, cout, transpose=False):
        shape = (kh, kw, cout, cin) if transpose else (kh, kw, cin, cout)
        p[name + "/V"] = (0.05 * rng.randn(*shape)).astype(dtype)
        p[name + "/g"] = rng.uniform(-0.3, 0.3, size=(cout,)).astype(dtype)
        p[name + "/b"] = (0.05 * rng.randn(cout)).astype(dtype)

    conv("x_enc", 5, 5, 3, hs)
    conv("x_dec", 5, 5, hs, 3, transpose=True)
    for i in range(hps["depth"]):
        for j in range(hps["num_blocks"]):
            sc = "IAF_%d_%d" % (i, j)
            conv(sc + "/up_conv1", 3, 3, hs, 2 * zs + 2 * hs)
            conv(sc + "/up_conv3", 3, 3, hs, hs)
            conv(sc + "/down_conv1", 3, 3, hs, 4 * zs + 2 * hs)
            if i > 0 and j == 0:
                conv(sc + "/down_deconv2", 3, 3, zs + hs, hs, transpose=True)
            else:
                conv(sc + "/down_conv2", 3, 3, zs + hs, hs)
            conv(sc + "/ar_multiconv2d/layer_0", 3, 3, zs, hs)
            conv(sc + "/ar_multiconv2d/layer_1", 3, 3, hs, hs)
            conv(sc + "/ar_multiconv2d/layer_out_0", 3, 3, hs, zs)
            conv(sc + "/ar_multiconv2d/layer_out_1", 3, 3, hs, zs)
    p["h_top"] = (0.1 * rng.randn(hs)).astype(dtype)
    p["dec_log_stdv"] = np.asarray(-1.0, dtype=dtype)
    return p


class InitPass(dict):
    """The parameters while a data-dependent init pass runs (``tf_train.py:175`` with mode "init"; ``'__init' in w`` in
    the Theano model).  The weight-normed convs of :mod:`iaf_b200.elbo` and :mod:`iaf_b200.elbo_theano` recognise it and
    take their init branch: they write the gain and bias they derive from the batch here and return the standardised
    pre-activation, which the next layers are initialised on."""

    def init(self, name, x_init, init_scale):
        """TF, layers.py:47-51 (conv2d) and 95-99 (deconv2d): ``x_init`` is the convolution with the l2-normalised V.
        Population moments over (0, 2, 3), ``scale = init_scale / sqrt(var + 1e-10)``, ``g = log(scale) / 3`` and
        ``b = -m scale``; returns ``scale (x_init - m)``.  The run-time branch applies exp(g), not exp(3 g), so an
        initialised layer runs at gain scale^(1/3), exactly as the reference's does."""
        m = x_init.mean(dim=(0, 2, 3))
        var = x_init.var(dim=(0, 2, 3), unbiased=False)
        scale = init_scale / torch.sqrt(var + 1e-10)
        self[name + "/g"] = torch.log(scale) / 3.0
        self[name + "/b"] = -m * scale
        return scale.reshape(1, -1, 1, 1) * (x_init - m.reshape(1, -1, 1, 1))


def _init_ar_conv2d(params, name, x, zerodiagonal):
    """ar_conv2d (layers.py:144-154) in init mode: the masked, l2-normalised V, init_scale 1 (layers.py:145)."""
    V = params[name + "/V"]
    mask = torch.from_numpy(tf_conv_ar_mask(V.shape[2], V.shape[3], zerodiagonal)).to(V)
    return params.init(name, _conv_same(x, _l2_normalize(mask * V), 1), 1.0)


class _InitLayer(object):
    """iaf_layer of the init pass (IAFLayer.down in mode "init", tf_train.py:56-85): z is the PRIOR's sample
    (tf_train.py:60-61), log q the posterior's density at it, and the masked stack (tf_train.py:69) runs conv by conv
    in init mode, with ``+ context`` after the first hidden conv.  Records each stack's input in ``stacks``."""

    def __init__(self, params):
        self.params, self.stacks = params, {}

    def __call__(self, scope, eps, post_mean, post_logsd, prior_mean, prior_logsd, context):
        c = 0.5 * math.log(2.0 * math.pi)
        z = prior_mean + torch.exp(prior_logsd) * eps
        logqs = -c - post_logsd - 0.5 * (z - post_mean) ** 2 * torch.exp(-2.0 * post_logsd)
        pre = scope + "/ar_multiconv2d/"
        self.stacks[pre[:-1]] = (z, context)
        h = z
        for k in range(2):
            h = _init_ar_conv2d(self.params, pre + "layer_%d" % k, h, False)
            if k == 0:
                h = h + context
            h = F.elu(h)
        arw_mean, arw_logsd = (0.1 * _init_ar_conv2d(self.params, pre + "layer_out_%d" % k, h, True) for k in range(2))
        z = (z - arw_mean) / torch.exp(arw_logsd)
        logqs = logqs + arw_logsd
        logps = -c - prior_logsd - 0.5 * (z - prior_mean) ** 2 * torch.exp(-2.0 * prior_logsd)
        kl = logqs - logps
        return z, kl.sum(dim=(2, 3)), kl.sum(dim=(1, 2, 3))


def data_init_pass(params, x_uint8, hps, noise=None, seed=0):
    """:func:`data_init` with what the pass saw: (params, out, stacks).  ``out`` is :func:`forward`'s dict for the init
    pass (the terms ``CVAE1(hps, "init", x)`` computes); ``stacks[scope + "/ar_multiconv2d"] = (z, context)`` is the
    input each masked stack was initialised on."""
    if noise is None:
        noise = default_noise(_noise_shapes(hps, x_uint8.shape[0]), params["h_top"].device, params["h_top"].dtype,
                              seed)(0, 1)
    p = InitPass(params)
    layer = _InitLayer(p)
    with torch.no_grad():
        out = forward(p, x_uint8, noise, layer, hps)
    return dict(p), out, layer.stacks


def data_init(params, x_uint8, hps, noise=None, seed=0):
    """The reference's data-dependent initialisation (tf_train.py:222-228: ``CVAE1(hps, "init", x[:batch_size])``) on
    the batch ``x_uint8``: returns a new dict with the ``g`` and ``b`` of every conv, deconv and masked conv set from
    the batch's statistics (tf_utils/layers.py:38-51, 86-100, and 144-166 with init_scale 1).  Every other entry is
    passed through: ``V`` (the reference draws it from N(0, 0.05) as :func:`make_params` does), ``h_top`` (zero in the
    reference, tf_train.py:190) and ``dec_log_stdv``.  The pass runs in stock torch ops on the parameters' device and
    dtype, in :func:`forward`'s order, with z drawn from each layer's prior.  noise[(i, j)]: that draw's N(0, 1) noise
    (the shapes :func:`forward` takes); default: torch.randn from one generator seeded with ``seed``.

    As in the reference, ``g = log(scale) / 3`` while the run-time branch applies ``exp(g)``: an initialised layer
    runs at scale^(1/3) of the standardising scale, not at it."""
    return data_init_pass(params, x_uint8, hps, noise, seed)[0]


class CudaIAF(object):
    """iaf_layer callable backed by the fused CUDA operator (one IAFOperator per layer scope, weights cached)."""

    def __init__(self, params, hps, path="auto"):
        from .ops import IAFOperator
        self.ops = {}
        self.params, self.hps, self.path, self.IAFOperator = params, hps, path, IAFOperator

    def __call__(self, scope, eps, post_mean, post_logsd, prior_mean, prior_logsd, context):
        op = self.ops.get(scope)
        if op is None:
            zs, hs = self.hps["z_size"], self.hps["h_size"]
            op = self.IAFOperator("tf", zs, [hs, hs], [zs, zs], nl="elu", path=self.path)   # tf_train.py:69
            self.ops[scope] = op
        # re-bound on every call: replacing an entry of the params dict (checkpoint load, optimiser that rebinds) is
        # picked up; unchanged tensors keep the packed copy (key = storage + version, see IAFOperator._weights_key)
        pre = scope + "/ar_multiconv2d/"
        op.set_weights([tuple(self.params[pre + n + "/" + k] for k in "Vgb")
                        for n in ("layer_0", "layer_1", "layer_out_0", "layer_out_1")])
        z, _, kl_bc, kl_cost = op.layer(eps, post_mean, post_logsd, prior_mean, prior_logsd, context, want_kl=False)
        return z, kl_bc, kl_cost


class CudaIAFTrain(object):
    """Differentiable iaf_layer for training: the posterior sample, logqs, prior logps and the KL sums are torch ops
    (tf_train.py:56-85) around ``IAFOperator.step``, whose autograd node runs iaf_step_fwd / iaf_step_bwd
    (SURVEY 8f-4).  ``obj.backward()`` on the result of forward() then yields the gradient of the training objective
    with respect to every parameter, the masked-AR ones included (masked taps get exactly zero, ar.py:369-373)."""

    def __init__(self, params, hps, path="auto", fused=False):
        """fused=True: the whole block runs as ONE autograd node (iaf_layer_fwd / iaf_layer_bwd)."""
        from .ops import IAFOperator
        self.ops = {}
        self.params, self.hps, self.path, self.IAFOperator, self.fused = params, hps, path, IAFOperator, fused

    def __call__(self, scope, eps, post_mean, post_logsd, prior_mean, prior_logsd, context):
        op = self.ops.get(scope)
        zs, hs = self.hps["z_size"], self.hps["h_size"]
        if op is None:
            op = self.IAFOperator("tf", zs, [hs, hs], [zs, zs], nl="elu", path=self.path)
            self.ops[scope] = op
        pre = scope + "/ar_multiconv2d/"
        op.set_weights([tuple(self.params[pre + n + "/" + k] for k in "Vgb")
                        for n in ("layer_0", "layer_1", "layer_out_0", "layer_out_1")])
        if self.fused:
            z, _, kl_bc, kl_cost = op.layer(eps, post_mean, post_logsd, prior_mean, prior_logsd, context, want_kl=False)
            if not z.requires_grad:
                raise RuntimeError("CudaIAFTrain(fused=True): the fused layer node is switched off (IAF_LAYER_AUTOGRAD=0)")
            return z, kl_bc, kl_cost
        return stochastic_layer(lambda z, c: op.step(z, c, want_logdet=False)[:2], eps, post_mean, post_logsd, prior_mean,
                                prior_logsd, context)


def posterior_sample(step, eps, post_mean, post_logsd, context):
    """The posterior half of :func:`stochastic_layer`: sample, step, log q -> (z', logqs [B,C,H,W])."""
    c = 0.5 * math.log(2.0 * math.pi)
    z0 = post_mean + torch.exp(post_logsd) * eps                  # DiagonalGaussian.sample, distributions.py:20
    logqs = -c - post_logsd - 0.5 * eps * eps                     # logps of the sample itself: (z0-mean)/sd == eps
    z, arw_logsd = step(z0, context)
    return z, logqs + arw_logsd                                    # tf_train.py:72


def stochastic_layer(step, eps, post_mean, post_logsd, prior_mean, prior_logsd, context):
    """tf_train.py:56-75 around a step callable (z, context) -> (z', arw_logsd): returns (z', kl_bc [B,C], kl_cost [B])."""
    c = 0.5 * math.log(2.0 * math.pi)
    z, logqs = posterior_sample(step, eps, post_mean, post_logsd, context)
    logps = -c - prior_logsd - 0.5 * (z - prior_mean) ** 2 * torch.exp(-2.0 * prior_logsd)
    kl = logqs - logps
    return z, kl.sum(dim=(2, 3)), kl.sum(dim=(1, 2, 3))


def sharded_bits_per_dim(params, x_uint8, noise, iaf_layer, hps, group=None):
    """Batch-sharded ELBO (BASELINE config C5; tf_train.py:126-142): every rank evaluates its contiguous slice of the
    global batch, and ONE sum all-reduce of the scalar loss gives the global bits/dim.  The free-bits batch mean stays
    rank-local, exactly as it is tower-local in the reference (tf_train.py:79)."""
    import torch.distributed as dist
    from .parallel import allreduce_scalars, shard_range
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    lo, hi = shard_range(x_uint8.shape[0], rank, world)
    out = forward(params, x_uint8[lo:hi], {k: v[lo:hi] for k, v in noise.items()}, iaf_layer, hps)
    num_pixels = 3 * hps["image_size"] ** 2
    loss_local = out["bits_per_dim"] * (math.log(2.0) * num_pixels * (hi - lo))
    (loss,) = allreduce_scalars([loss_local], group)
    return loss / (math.log(2.0) * num_pixels * x_uint8.shape[0])


def run_train_step(params, x_uint8, opt, noise, objective, loss_per_bpd, sharded=False, group=None):
    """The step both models' ``train_step`` take: zero the gradients (to None, so a parameter the objective does not
    reach has no gradient: skipped by the TF rule, a zero gradient for the Theano rule), ``objective(x, noise) ->
    (obj, bits_per_dim)`` on this rank's rows, ``obj.backward()``, and when sharded the towers' average of the gradients
    (``allreduce_grads``; tf_train.py:139-147, ``average_grads``), then ``opt.step()``.  Returns the global bits/dim
    (detached): ``loss_per_bpd`` is one sample's loss at 1 bit/dim, what turns the ranks' bits/dim into a summed loss.
    ``noise`` covers the global batch; each rank takes its rows."""
    import torch.distributed as dist
    from .parallel import allreduce_grads, allreduce_scalars, shard_range
    sharded = sharded or group is not None
    B = x_uint8.shape[0]
    lo, hi = 0, B
    if sharded and dist.is_initialized():
        lo, hi = shard_range(B, dist.get_rank(group), dist.get_world_size(group))
    for p in params.values():
        p.grad = None
    obj, bpd = objective(x_uint8[lo:hi], {k: v[lo:hi] for k, v in noise.items()})
    obj.backward()
    if sharded:
        allreduce_grads(params, group)
        (loss,) = allreduce_scalars([bpd.detach() * (loss_per_bpd * (hi - lo))], group)
        bpd = loss / (loss_per_bpd * B)
    opt.step()
    return bpd.detach()


def train_step(params, x_uint8, opt, hps, noise=None, iaf_layer=None, sharded=False, group=None):
    """One training step of the TF model, as ``tf_train.run`` takes it (tf_train.py:126-147, 211): the gradient of
    ``obj = sum(kl_obj - log_pxz)`` over the batch (free bits per tower), then ``opt.step()``.  ``params``: leaf tensors
    with requires_grad (fp32 CUDA for :class:`iaf_b200.optim.Adamax`, ``rule="tf"``); ``opt`` updates them in place.
    ``iaf_layer``: default ``CudaIAFTrain(params, hps)``, built per call -- pass one to keep its operators across steps.
    ``noise[(i, j)]``: the posterior's N(0, 1) draw of the global batch (default: torch.randn on the parameters' device).
    ``sharded=True`` (or a ``group``): this rank is one tower of the reference's ``num_gpus`` and takes its contiguous
    slice of the batch; the towers' gradients are averaged before the step.  Returns the step's bits/dim (a tensor).
    An optimiser with ``lookahead()`` (Eve) is refused: the TF reference has none."""
    if hasattr(opt, "lookahead"):
        raise ValueError("elbo.train_step: the TF model trains with Adamax only (Eve is the Theano model's optim='eve')")
    if iaf_layer is None:
        iaf_layer = CudaIAFTrain(params, hps)
    if noise is None:
        h = params["h_top"]
        noise = {k: torch.randn(s, device=h.device, dtype=h.dtype) for k, s in _noise_shapes(hps, x_uint8.shape[0]).items()}

    def objective(x, nz):
        out = forward(params, x, nz, iaf_layer, hps)
        return out["obj"], out["bits_per_dim"]
    return run_train_step(params, x_uint8, opt, noise, objective, math.log(2.0) * 3 * hps["image_size"] ** 2, sharded,
                          group)


def sharded_log_likelihood(params, x_uint8, iaf_layer, hps, k, chunk=None, noise=None, seed=0, group=None,
                           estimator=None):
    """Image-sharded importance-sampled bits/dim: every rank runs all k samples of its contiguous slice of the images
    (``shard_range``), and ONE sum all-reduce of the summed -log_px gives the global bits/dim.  ``estimator``: this
    module's :func:`log_likelihood` (default) or ``elbo_theano.log_likelihood``.  A given ``noise(start, count)`` covers
    the global batch; each rank takes its images' rows.  The default noise is seeded with ``seed`` on every rank."""
    import torch.distributed as dist
    from .parallel import allreduce_scalars, shard_range
    estimator = log_likelihood if estimator is None else estimator
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    B = x_uint8.shape[0]
    lo, hi = shard_range(B, rank, world)
    local = None if noise is None else (
        lambda start, count: {key: v[lo * count:hi * count] for key, v in noise(start, count).items()})
    if hi > lo:
        nll = (-estimator(params, x_uint8[lo:hi], iaf_layer, hps, k, chunk, local, seed)["log_px"]).sum()
    else:
        nll = torch.zeros((), dtype=torch.float64, device=x_uint8.device)
    (nll,) = allreduce_scalars([nll], group)
    return nll / (math.log(2.0) * 3 * hps["image_size"] ** 2 * B)
