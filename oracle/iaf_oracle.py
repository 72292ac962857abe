"""CPU oracle for the IAF masked-autoregressive transform (TEST INFRASTRUCTURE ONLY).

This file is a numpy restatement of the reference's algorithm for the hot path
(SURVEY.md section 8).  It is the *checker*: only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl
reference`` legs may import it.  Nothing under ``iaf_b200/`` imports it and the
product path never falls back to it.

PARITY PIN STATUS.  The reference (openai/iaf) ships no test,
fixture or golden vector for this path (tf_utils/distributions_test.py and
tf_utils/hparams_test.py are its only tests) and neither Theano nor TensorFlow
can be imported in the build container, so the reference cannot be *run*
unmodified.  The pin used instead (tests/golden/make_golden.py): the
reference's OWN python source for ``get_linear_ar_mask``, ``get_conv_ar_mask``,
``conv2d``, ``ar_conv2d``, ``ar_multiconv2d`` (tf_utils/layers.py),
``ar.conv2d`` / ``ar.multiconv2d`` (graphy/nodes/ar.py), ``pad2dwithchannel``
(graphy/nodes/conv.py), ``DiagonalGaussian`` / ``compute_lowerbound`` /
``logsumexp`` / ``repeat`` (tf_utils/distributions.py) and ``IAFLayer.down``
(tf_train.py) is exec'd from the reference source against small numpy stand-ins for
the handful of TF / Theano primitives it calls (conv2d, l2_normalize, elu,
dnn_conv, ...), and the resulting tensors are committed as fixtures under
tests/golden/.  The third-party primitives themselves (cuDNN conv through
TF / Theano; versions unpinned by the reference) are restated from their
published semantics; that part of parity is therefore "restated, not executed".

Every function cites the reference file:line it follows (paths relative to
the reference repository).  All arithmetic is done in the dtype of the inputs (use
float64 inputs for the truth oracle, float32 for the like-for-like CPU port).
"""
from __future__ import annotations

import math

import numpy as np

TAPS = ((1, 1), (1, 2), (2, 0), (2, 1), (2, 2))  # live (ky,kx) of the 3x3 AR mask


# ----------------------------------------------------------------------------
# masks
# ----------------------------------------------------------------------------
def get_linear_ar_mask(n_in, n_out, zerodiagonal=False):
    """MADE channel mask, [n_in, n_out].  tf_utils/layers.py:115-131
    (identical rule inline at graphy/nodes/ar.py:249-262, transposed)."""
    assert n_in % n_out == 0 or n_out % n_in == 0, "%d - %d" % (n_in, n_out)
    mask = np.ones([n_in, n_out], dtype=np.float32)
    if n_out >= n_in:
        k = n_out // n_in
        for i in range(n_in):
            mask[i + 1:, i * k:(i + 1) * k] = 0
            if zerodiagonal:
                mask[i:i + 1, i * k:(i + 1) * k] = 0
    else:
        k = n_in // n_out
        for i in range(n_out):
            mask[(i + 1) * k:, i:i + 1] = 0
            if zerodiagonal:
                mask[i * k:(i + 1) * k:, i:i + 1] = 0
    return mask


def get_conv_ar_mask(h, w, n_in, n_out, zerodiagonal=False):
    """TF-layout conv mask [h, w, n_in, n_out].  tf_utils/layers.py:134-141."""
    l = (h - 1) // 2
    m = (w - 1) // 2
    mask = np.ones([h, w, n_in, n_out], dtype=np.float32)
    mask[:l, :, :, :] = 0
    mask[l, :m, :, :] = 0
    mask[l, m, :, :] = get_linear_ar_mask(n_in, n_out, zerodiagonal)
    return mask


def theano_conv_ar_mask(n_in, n_out, size_kernel=(3, 3), zerodiagonal=True, pad_channel=True):
    """Theano-layout mask [n_out, n_in(+1), kh, kw].  graphy/nodes/ar.py:241-264
    (flipmask is always False on the down_iaf2_nl / up_iaf2_nl path, models.py:92)."""
    _n_in = n_in + (1 if pad_channel else 0)
    l = (size_kernel[0] - 1) // 2
    m = (size_kernel[1] - 1) // 2
    mask = np.ones((n_out, _n_in, size_kernel[0], size_kernel[1]), dtype=np.float32)
    mask[:, :, :l, :] = 0
    mask[:, :, l, :m] = 0
    if n_out >= n_in:
        assert n_out % n_in == 0
        k = n_out // n_in
        for i in range(n_in):
            mask[i * k:(i + 1) * k, i + 1:, l, m] = 0
            if zerodiagonal:
                mask[i * k:(i + 1) * k, i:i + 1, l, m] = 0
    else:
        assert n_in % n_out == 0
        k = n_in // n_out
        for i in range(n_out):
            mask[i:i + 1, (i + 1) * k:, l, m] = 0
            if zerodiagonal:
                mask[i:i + 1, i * k:(i + 1) * k:, l, m] = 0
    return mask


# ----------------------------------------------------------------------------
# nonlinearities
# ----------------------------------------------------------------------------
def nonlinearity(which):
    """graphy/nodes/__init__.py:158-177 (the parameter-free entries) and
    tf.nn.elu (tf_utils/layers.py:159)."""
    if which in (None, "None", "none"):
        return lambda h: h
    if which == "elu":
        return lambda h: np.where(h < 0, np.expm1(np.minimum(h, 0)), h)
    if which == "softplus":
        return lambda h: np.logaddexp(0, h)
    if which == "relu":
        return lambda h: h * (h >= 0)
    if which == "tanh":
        return np.tanh
    if which == "leakyrelu":
        return lambda h: np.where(h < 0, 0.01 * h, h)
    raise Exception("Unrecognized nonlinearity: " + str(which))


# ----------------------------------------------------------------------------
# convolution primitives (the cuDNN stand-ins)
# ----------------------------------------------------------------------------
def _shift2d(x, dy, dx):
    """y[b,c,i,j] = x[b,c,i+dy,j+dx], zero outside."""
    B, C, H, W = x.shape
    out = np.zeros_like(x)
    ys0, ys1 = max(0, -dy), min(H, H - dy)
    xs0, xs1 = max(0, -dx), min(W, W - dx)
    if ys0 < ys1 and xs0 < xs1:
        out[:, :, ys0:ys1, xs0:xs1] = x[:, :, ys0 + dy:ys1 + dy, xs0 + dx:xs1 + dx]
    return out


def xcorr2d_same(x, w_hwio):
    """tf.nn.conv2d(x, w, [1,1,1,1], "SAME", data_format="NCHW"): cross-correlation,
    zero padding; x [B,Cin,H,W], w [kh,kw,Cin,Cout].  Call site tf_utils/layers.py:64."""
    kh, kw = w_hwio.shape[:2]
    out = None
    for ky in range(kh):
        for kx in range(kw):
            wt = w_hwio[ky, kx]
            if not np.any(wt):
                continue
            xs = _shift2d(x, ky - (kh - 1) // 2, kx - (kw - 1) // 2)
            t = np.einsum("bihw,io->bohw", xs, wt)
            out = t if out is None else out + t
    if out is None:
        out = np.zeros((x.shape[0], w_hwio.shape[3]) + x.shape[2:], x.dtype)
    return out


def trueconv2d_valid(xp, k_oihw):
    """Theano dnn_conv(xp, kerns, border_mode='valid') with its default
    conv_mode='conv' (kernel flipped).  Call site graphy/nodes/ar.py:323.
    xp [B,Cin,H+2,W+2] -> [B,Cout,H,W]."""
    kh, kw = k_oihw.shape[2:]
    H = xp.shape[2] - kh + 1
    W = xp.shape[3] - kw + 1
    out = np.zeros((xp.shape[0], k_oihw.shape[0], H, W), xp.dtype)
    for ky in range(kh):
        for kx in range(kw):
            kt = k_oihw[:, :, ky, kx]
            if not np.any(kt):
                continue
            oy, ox = kh - 1 - ky, kw - 1 - kx
            out += np.einsum("bihw,oi->bohw", xp[:, :, oy:oy + H, ox:ox + W], kt)
    return out


def pad2dwithchannel(x, size_kernel=(3, 3)):
    """graphy/nodes/conv.py:71-83: zero-pad and append a channel that is 1 on the
    border ring and 0 inside."""
    a = (size_kernel[0] - 1) // 2
    b = (size_kernel[1] - 1) // 2
    B, C, H, W = x.shape
    r = np.zeros((B, C + 1, H + 2 * a, W + 2 * b), x.dtype)
    r[:, C, :, :] = 1.0
    r[:, C, a:-a, b:-b] = 0.0
    r[:, :C, a:-a, b:-b] = x
    return r


# ----------------------------------------------------------------------------
# TF variant (tf_utils/layers.py)
# ----------------------------------------------------------------------------
def tf_effective_weight(V, g, mask):
    """tf_utils/layers.py:53-60 (run-time branch): w = exp(g) * l2_normalize(mask*V, [0,1,2]);
    tf.nn.l2_normalize(x, dim, epsilon=1e-12) = x * rsqrt(max(sum(x^2, dim), epsilon))."""
    v = mask.astype(V.dtype) * V
    sq = np.sum(np.square(v), axis=(0, 1, 2), keepdims=True)
    return np.exp(g).reshape(1, 1, 1, -1) * v / np.sqrt(np.maximum(sq, 1e-12))


def tf_ar_conv2d(x, layer, zerodiagonal):
    """tf_utils/layers.py:144-154 -> 52-64.  layer = dict(V=[3,3,Cin,Cout], g=[Cout], b=[Cout])."""
    V, g, b = layer["V"], layer["g"], layer["b"]
    mask = get_conv_ar_mask(V.shape[0], V.shape[1], V.shape[2], V.shape[3], zerodiagonal)
    w = tf_effective_weight(V, g, mask)
    return xcorr2d_same(x, w) + b.reshape(1, -1, 1, 1)


def tf_ar_multiconv2d(x, context, hidden, heads, nl="elu"):
    """tf_utils/layers.py:158-166.  hidden/heads: lists of layer dicts
    (``layer_%d`` / ``layer_out_%d``)."""
    f = nonlinearity(nl)
    for i, layer in enumerate(hidden):
        x = tf_ar_conv2d(x, layer, zerodiagonal=False)
        if i == 0:
            x = x + context
        x = f(x)
    return [tf_ar_conv2d(x, layer, zerodiagonal=True) for layer in heads]


# ----------------------------------------------------------------------------
# Theano variant (graphy/nodes/ar.py)
# ----------------------------------------------------------------------------
def theano_effective_kernel(w, s, mask, logscale_scale=3.0):
    """graphy/nodes/ar.py:312-317 with l2normalize 267-281 (logscale=True, :9-10).
    The set_subtensor at :274/:276 only re-zeroes entries the mask already zeroes."""
    kerns = mask.astype(w.dtype) * w
    norm = np.sqrt(np.sum(kerns ** 2, axis=(1, 2, 3), keepdims=True)) + 1e-8
    kerns = kerns * (1.0 / norm)
    return kerns * np.exp(logscale_scale * s).reshape(-1, 1, 1, 1)


def theano_ar_conv2d(h, layer, zerodiagonal):
    """graphy/nodes/ar.py:304-329 (no '__init', bn=False).
    layer = dict(w=[Cout,Cin+1,3,3], s=[Cout], b=[Cout])."""
    w, s, b = layer["w"], layer["s"], layer["b"]
    n_out, n_in1 = w.shape[:2]
    mask = theano_conv_ar_mask(n_in1 - 1, n_out, w.shape[2:], zerodiagonal, pad_channel=True)
    hp = pad2dwithchannel(h, w.shape[2:])
    kerns = theano_effective_kernel(w, s, mask)
    return trueconv2d_valid(hp, kerns) + b.reshape(1, -1, 1, 1)


def theano_multiconv2d(h, context, hidden, heads, nl="elu"):
    """graphy/nodes/ar.py:396-416.  With no hidden layer the context is never added
    (SURVEY F8).  Returns a list (the reference returns a bare tensor when there is
    one head, ar.py:411; the host wrapper mirrors that)."""
    f = nonlinearity(nl)
    for i, layer in enumerate(hidden):
        h = theano_ar_conv2d(h, layer, zerodiagonal=False)
        if i == 0:
            h = h + context
        h = f(h)
    return [theano_ar_conv2d(h, layer, zerodiagonal=True) for layer in heads]


# ----------------------------------------------------------------------------
# the IAF step
# ----------------------------------------------------------------------------
def multiconv(variant, z, context, hidden, heads, nl="elu"):
    if variant == "tf":
        return tf_ar_multiconv2d(z, context, hidden, heads, nl)
    if variant == "theano":
        return theano_multiconv2d(z, context, hidden, heads, nl)
    raise ValueError(variant)


def iaf_step(variant, z, context, hidden, heads, nl="elu", scale=0.1):
    """models.py:281-285 / models.py:170-175 / tf_train.py:69-72:
        m *= .1; s *= .1; z' = (z - m) / exp(s); logqs += s
    Returns (z', arw_logsd_elem, logdet_per_sample) with
    logdet = log|det dz'/dz| = -sum(arw_logsd)."""
    m, s = multiconv(variant, z, context, hidden, heads, nl)
    arw_mean = m * scale
    arw_logsd = s * scale
    z_new = (z - arw_mean) / np.exp(arw_logsd)
    logdet = -arw_logsd.reshape(z.shape[0], -1).sum(axis=1)
    return z_new, arw_logsd, logdet


# ----------------------------------------------------------------------------
# neighbours of the step inside the stochastic layer
# ----------------------------------------------------------------------------
def gaussian_diag_logps(mean, logvar, sample):
    """tf_utils/distributions.py:5-10 == graphy/nodes/rand.py:83."""
    return -0.5 * (np.log(2 * np.pi) + logvar + np.square(sample - mean) / np.exp(logvar))


def gaussian_diag_sample(mean, logvar, eps):
    """tf_utils/distributions.py:19-21 / graphy/nodes/rand.py:81-82 with the noise given."""
    return mean + np.exp(0.5 * logvar) * eps


def stochastic_layer_down(variant, eps, qz_mean, qz_logsd, rz_mean, rz_logsd, pz_mean, pz_logsd,
                          up_context, down_context, hidden, heads, nl="elu", kl_min=0.0):
    """The posterior/prior block around the step: tf_train.py:56-85 and
    models.py:273-298,328 + 455-466.  Returns dict(z, logqs, logps, kl, kl_cost, kl_obj,
    arw_logsd)."""
    post_mean = rz_mean + qz_mean
    post_logvar = 2 * (rz_logsd + qz_logsd)
    context = up_context + down_context
    z0 = gaussian_diag_sample(post_mean, post_logvar, eps)
    logqs = gaussian_diag_logps(post_mean, post_logvar, z0)
    z, arw_logsd, _ = iaf_step(variant, z0, context, hidden, heads, nl)
    logqs = logqs + arw_logsd
    logps = gaussian_diag_logps(pz_mean, 2 * pz_logsd, z)
    kl = logqs - logps
    kl_cost = kl.sum(axis=(1, 2, 3))
    if kl_min > 0:
        kl_ave = kl.sum(axis=(2, 3)).mean(axis=0, keepdims=True)
        kl_ave = np.maximum(kl_ave, kl_min)
        kl_obj = np.tile(kl_ave, [z.shape[0], 1]).sum(axis=1)
    else:
        kl_obj = kl_cost
    return dict(z0=z0, z=z, logqs=logqs, logps=logps, kl=kl, kl_cost=kl_cost, kl_obj=kl_obj,
                arw_logsd=arw_logsd)


# ----------------------------------------------------------------------------
# downstream ELBO arithmetic (tf_utils/distributions.py)
# ----------------------------------------------------------------------------
def logsumexp(x):
    """tf_utils/distributions.py:36-38."""
    x_max = np.max(x, axis=1, keepdims=True)
    return x_max.reshape(-1) + np.log(np.sum(np.exp(x - x_max), axis=1))


def repeat(x, n):
    """tf_utils/distributions.py:41-52."""
    if n == 1:
        return x
    idx = np.tile(np.arange(x.shape[0]).reshape(-1, 1), [1, n]).reshape(-1)
    return x[idx]


def compute_lowerbound(log_pxz, sum_kl_costs, k=1):
    """tf_utils/distributions.py:55-62."""
    if k == 1:
        return sum_kl_costs - log_pxz
    log_pxz = log_pxz.reshape(-1, k)
    sum_kl_costs = sum_kl_costs.reshape(-1, k)
    return -(-math.log(float(k)) + logsumexp(log_pxz - sum_kl_costs))


def discretized_logistic(mean, logscale, binsize=1 / 256.0, sample=None):
    """tf_utils/distributions.py:28-32."""
    scale = np.exp(logscale)
    sample = (np.floor(sample / binsize) * binsize - mean) / scale
    sig = lambda t: 1.0 / (1.0 + np.exp(-t))
    logp = np.log(sig(sample + binsize / scale) - sig(sample) + 1e-7)
    return logp.sum(axis=(1, 2, 3))


# ----------------------------------------------------------------------------
# synthetic inputs (SURVEY 8d): the seeded workload every test and bench uses
# ----------------------------------------------------------------------------
def make_params(variant, n_z, hidden_sizes, head_sizes, seed=1, dtype=np.float32):
    """Raw (un-masked, un-normalised) parameters in the reference's own layouts:
    tf: V [3,3,Cin,Cout] ~ 0.05 N(0,1) (layers.py:40), g ~ U(-.5,.5), b ~ 0.1 N(0,1);
    theano: w [Cout,Cin+1,3,3] ~ 0.05 N(0,1) (ar.py:288), s = g/3, b."""
    rng = np.random.RandomState(seed)
    sizes = [n_z] + list(hidden_sizes)
    hidden, heads = [], []

    def one(cin, cout):
        g = rng.uniform(-0.5, 0.5, size=(cout,))
        b = 0.1 * rng.randn(cout)
        if variant == "tf":
            V = 0.05 * rng.randn(3, 3, cin, cout)
            return dict(V=V.astype(dtype), g=g.astype(dtype), b=b.astype(dtype))
        w = 0.05 * rng.randn(cout, cin + 1, 3, 3)
        return dict(w=w.astype(dtype), s=(g / 3.0).astype(dtype), b=b.astype(dtype))

    for i in range(len(hidden_sizes)):
        hidden.append(one(sizes[i], sizes[i + 1]))
    for n in head_sizes:
        heads.append(one(sizes[-1], n))
    return hidden, heads


def make_inputs(B, n_z, n_ctx, H, W, seed=0, dtype=np.float32):
    """z ~ N(0,1), context ~ 0.1 N(0,1) (SURVEY 8d)."""
    rng = np.random.RandomState(seed)
    z = rng.randn(B, n_z, H, W).astype(dtype)
    ctx = (0.1 * rng.randn(B, n_ctx, H, W)).astype(dtype)
    return z, ctx


def cast_params(layers, dtype):
    return [{k: v.astype(dtype) for k, v in l.items()} for l in layers]
