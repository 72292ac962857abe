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
"""
import math

import numpy as np
import torch
import torch.nn.functional as F


def _same_pad(n, k, s):
    out = -(-n // s)
    total = max((out - 1) * s + k - n, 0)
    return total // 2, total - total // 2


def conv2d(params, name, x, stride=1):
    """tf_utils/layers.py:31-64 (run-time branch, mask=None): w = exp(g) * l2_normalize(V,[0,1,2]); SAME padding."""
    V, g, b = params[name + "/V"], params[name + "/g"], params[name + "/b"]
    w = torch.exp(g).reshape(1, 1, 1, -1) * V * torch.rsqrt(torch.clamp((V * V).sum(dim=(0, 1, 2), keepdim=True), min=1e-12))
    kh, kw = V.shape[0], V.shape[1]
    pt, pb = _same_pad(x.shape[2], kh, stride)
    pl, pr = _same_pad(x.shape[3], kw, stride)
    x = F.pad(x, (pl, pr, pt, pb))
    return F.conv2d(x, w.permute(3, 2, 0, 1), stride=stride) + b.reshape(1, -1, 1, 1)


def deconv2d(params, name, x, stride=2):
    """tf_utils/layers.py:67-112: conv2d_transpose, SAME, filter [kh,kw,Cout,Cin], weight norm over [0,1,2] -> per Cin."""
    V, g, b = params[name + "/V"], params[name + "/g"], params[name + "/b"]
    # layers.py:108: w = reshape(exp(g), [1,1,num_filters,1]) * l2_normalize(v, [0,1,2])
    w = torch.exp(g).reshape(1, 1, -1, 1) * V * torch.rsqrt(torch.clamp((V * V).sum(dim=(0, 1, 2), keepdim=True), min=1e-12))
    kh, kw = V.shape[0], V.shape[1]
    H, W = x.shape[2] * stride, x.shape[3] * stride
    y = F.conv_transpose2d(x, w.permute(3, 2, 0, 1), stride=stride)  # full output (H-1)*s + k
    pt, _ = _same_pad(H, kh, stride)
    pl, _ = _same_pad(W, kw, stride)
    return y[:, :, pt:pt + H, pl:pl + W] + b.reshape(1, -1, 1, 1)


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


def forward(params, x_uint8, noise, iaf_layer, hps):
    """bits/dim and the per-sample pieces for one batch.

    hps: dict(z_size, h_size, depth, num_blocks, kl_min, image_size).  noise[(i, j)]: the N(0,1) draw of
    layer (i, j)'s posterior (tf_train.py:57).  iaf_layer(scope, eps, post_mean, post_logsd, prior_mean,
    prior_logsd, context) -> (z, kl_bc [B,C], kl_cost [B])."""
    zs, hs = hps["z_size"], hps["h_size"]
    x = x_uint8.to(params["h_top"].dtype)
    x = torch.clamp((x + 0.5) / 256.0, 0.0, 1.0) - 0.5          # tf_train.py:164-165
    orig_x = x
    B = x.shape[0]
    h = conv2d(params, "x_enc", x, stride=2)
    layers = [(i, j) for i in range(hps["depth"]) for j in range(hps["num_blocks"])]
    up = {}
    for (i, j) in layers:                                         # IAFLayer.up, tf_train.py:29-44
        sc = "IAF_%d_%d" % (i, j)
        down = (i > 0) and (j == 0)
        t = conv2d(params, sc + "/up_conv1", F.elu(h), stride=2 if down else 1)
        qz_mean, qz_logsd, up_context, hh = torch.split(t, [zs, zs, hs, hs], dim=1)
        up[(i, j)] = (qz_mean, qz_logsd, up_context)
        hh = conv2d(params, sc + "/up_conv3", F.elu(hh))
        if down:
            h = resize_nearest_neighbor(h, 0.5)
        h = h + 0.1 * hh
    size = hps["image_size"] // 2 ** hps["depth"]
    h = params["h_top"].reshape(1, -1, 1, 1).expand(B, hs, size, size)
    kl_obj = torch.zeros(B, dtype=h.dtype, device=h.device)
    kl_cost = torch.zeros(B, dtype=h.dtype, device=h.device)
    for (i, j) in reversed(layers):                               # IAFLayer.down, tf_train.py:46-95
        sc = "IAF_%d_%d" % (i, j)
        down = (i > 0) and (j == 0)
        t = conv2d(params, sc + "/down_conv1", F.elu(h))
        pz_mean, pz_logsd, rz_mean, rz_logsd, down_context, h_det = torch.split(t, [zs] * 4 + [hs] * 2, dim=1)
        qz_mean, qz_logsd, up_context = up[(i, j)]
        z, kl_bc, cost = iaf_layer(sc, noise[(i, j)], (rz_mean + qz_mean).contiguous(), (rz_logsd + qz_logsd).contiguous(),
                                   pz_mean.contiguous(), pz_logsd.contiguous(), (up_context + down_context).contiguous())
        if hps["kl_min"] > 0:                                     # tf_train.py:77-83: free bits, batch mean is local
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
    xd = torch.clamp(xd, -0.5 + 1 / 512.0, 0.5 - 1 / 512.0)
    log_pxz = discretized_logistic(xd, params["dec_log_stdv"], orig_x)
    loss = (kl_cost - log_pxz).sum()                              # compute_lowerbound, k = 1 (distributions.py:55-57)
    num_pixels = 3 * hps["image_size"] ** 2
    return dict(bits_per_dim=loss / (math.log(2.0) * num_pixels * B), obj=(kl_obj - log_pxz).sum(), kl_cost=kl_cost,
                kl_obj=kl_obj, log_pxz=log_pxz)


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
