#!/usr/bin/env python
"""Generate tests/golden/cvae1_forward.npz by EXECUTING the reference's own `CVAE1._forward` (tf_train.py:161-219), with
`IAFLayer.up` / `IAFLayer.down` (tf_train.py:23-95), `conv2d` / `deconv2d` / `ar_multiconv2d` / `resize_nearest_neighbor`
(tf_utils/layers.py) and `discretized_logistic` / `compute_lowerbound` / `repeat` (tf_utils/distributions.py) all run from
the reference through the same python-2 shims and numpy-backed TensorFlow stand-in as make_golden.py (extended here
by the handful of primitives the whole forward pass needs: strided SAME convolution, conv2d_transpose, transpose,
clip_by_value, floor, sigmoid, nearest-neighbour resize).  The convolution primitives themselves are stood in for by
torch CPU float64 ops -- independent of both iaf_b200/elbo.py's restatement (which the fixture pins) and the oracle.

Needs a checkout of the reference (IAF_REFERENCE, see make_golden.py):   python tests/golden/make_golden_cvae1.py
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
sys.path.insert(0, HERE)
import make_golden as MG  # noqa: E402
from make_golden import RT, _py2div, extract, py2_compile, read  # noqa: E402


def _same_pad(n, k, s):
    out = -(-n // s)
    total = max((out - 1) * s + k - n, 0)
    return total // 2, total - total // 2


def extend_tf(tf):
    """TF <= 0.11 primitives used by CVAE1._forward beyond what IAFLayer.down needed (make_golden.TFShim)."""
    t64 = lambda a: torch.from_numpy(np.ascontiguousarray(np.asarray(a, dtype=np.float64)))

    def conv2d(x, w, strides, pad, data_format="NHWC"):
        assert data_format == "NCHW" and pad == "SAME" and strides[0] == 1 and strides[1] == 1
        w = np.asarray(w)  # [kh,kw,ci,co]
        kh, kw = w.shape[:2]
        sh, sw = int(strides[2]), int(strides[3])
        x = np.asarray(x)
        pt, pb = _same_pad(x.shape[2], kh, sh)
        pl, pr = _same_pad(x.shape[3], kw, sw)
        xp = np.pad(x, ((0, 0), (0, 0), (pt, pb), (pl, pr)))
        y = torch.nn.functional.conv2d(t64(xp), t64(w.transpose(3, 2, 0, 1)), stride=(sh, sw))
        return RT(y.numpy())
    tf.nn.conv2d = conv2d

    def conv2d_transpose(x, filters, output_shape, strides, padding="SAME"):
        """NHWC input, filter [kh, kw, out_channels, in_channels] (TF's layout), SAME padding."""
        assert padding == "SAME" and strides[0] == 1 and strides[3] == 1
        xs = np.asarray(x).transpose(0, 3, 1, 2)          # NCHW
        f = np.asarray(filters)
        kh, kw = f.shape[:2]
        sh, sw = int(strides[1]), int(strides[2])
        H, W = int(output_shape[1]), int(output_shape[2])
        # gradient of a SAME forward convolution with this filter: full transposed conv, then crop the forward padding
        y = torch.nn.functional.conv_transpose2d(t64(xs), t64(f.transpose(3, 2, 0, 1)), stride=(sh, sw)).numpy()
        pt, _ = _same_pad(H, kh, sh)
        pl, _ = _same_pad(W, kw, sw)
        y = y[:, :, pt:pt + H, pl:pl + W]
        assert y.shape[2] == H and y.shape[3] == W, (y.shape, H, W)
        return RT(y.transpose(0, 2, 3, 1))
    tf.nn.conv2d_transpose = conv2d_transpose

    tf.transpose = lambda x, perm: RT(np.asarray(x).transpose(perm))
    tf.to_float = lambda x: RT(np.asarray(x, dtype=np.float64))
    tf.clip_by_value = lambda x, lo, hi: RT(np.clip(np.asarray(x), lo, hi))
    tf.floor = lambda x: RT(np.floor(np.asarray(x)))
    tf.sigmoid = lambda x: RT(1.0 / (1.0 + np.exp(-np.asarray(x))))
    tf.zeros_initializer = None
    tf.image = types.SimpleNamespace(
        resize_nearest_neighbor=lambda x, size: RT(_resize_nn(np.asarray(x), int(size[0]), int(size[1]))))

    base_get = tf.get_variable

    def get_variable(name, shape=None, dtype=None, initializer=None):
        return base_get(name, shape)
    tf.get_variable = get_variable


import contextlib  # noqa: E402


@contextlib.contextmanager
def _arg_scope_init_false(fns, **kw):
    """arg_scope([conv2d, deconv2d], init=(mode == "init")): outside "init" mode this only sets init=False, which is
    those functions' default -- nothing to inject."""
    assert kw == {} or kw == {"init": False}, kw
    yield


def _resize_nn(x, H, W):
    """tf.image.resize_nearest_neighbor on NHWC (align_corners=False): src = floor(dst * in / out)."""
    iy = (np.arange(H) * x.shape[1] // H).astype(int)
    ix = (np.arange(W) * x.shape[2] // W).astype(int)
    return x[:, iy][:, :, ix]


def run_case(tf, layers, dist, train, kl_min, tag, out):
    import iaf_b200.elbo as E
    hps_d = dict(z_size=4, h_size=8, depth=2, num_blocks=2, kl_min=kl_min, image_size=16)
    B, seed = 3, 5
    params = E.make_params(hps_d, seed=seed, dtype=np.float32)
    rng = np.random.RandomState(seed + 1)
    x = rng.randint(0, 256, size=(B, 3, 16, 16)).astype(np.uint8)
    noise = {}
    for i in range(hps_d["depth"]):
        s = 16 // 2 ** (i + 1)
        for j in range(hps_d["num_blocks"]):
            noise[(i, j)] = rng.randn(B, hps_d["z_size"], s, s).astype(np.float32)

    # the reference's variable store: names under the "model" scope are exactly elbo.make_params' keys
    tf.store.clear()
    for k, v in params.items():
        tf.store[k] = np.asarray(v, dtype=np.float64)
    # IAFLayer.down draws prior.sample first, posterior.sample second (tf_train.py:56-57); the down pass visits the layers
    # in reverse order
    order = [(i, j) for i in range(hps_d["depth"]) for j in range(hps_d["num_blocks"])]
    tf.noise[:] = []
    for (i, j) in reversed(order):
        tf.noise.append(np.zeros_like(noise[(i, j)], dtype=np.float64))      # prior.sample (unused in "eval" mode)
        tf.noise.append(noise[(i, j)].astype(np.float64))                    # posterior.sample's noise

    hps = types.SimpleNamespace(batch_size=B, k=1, num_gpus=1, **hps_d)
    ns = {"_py2div": _py2div, "np": np, "tf": tf, "arg_scope": _arg_scope_init_false, "conv2d": layers["conv2d"],
          "deconv2d": layers["deconv2d"], "IAFLayer": train["IAFLayer"], "repeat": dist["repeat"],
          "discretized_logistic": dist["discretized_logistic"], "compute_lowerbound": dist["compute_lowerbound"]}
    src = extract(read("tf_train.py"), r"^    def _forward\(self, x, gpu\):", r"^def run\(hps\)")
    src = "\n".join(l[4:] if l.startswith("    ") else l for l in src.splitlines())   # de-indent the method
    exec(py2_compile(src, "tf_train.py:_forward"), ns)
    fake = types.SimpleNamespace(hps=hps, mode="eval", dec_log_stdv=RT(np.asarray(params["dec_log_stdv"], dtype=np.float64)))
    x_out, obj, loss = ns["_forward"](fake, RT(x.astype(np.float64)), 0)
    assert not tf.noise, "noise queue not consumed: %d left" % len(tf.noise)
    out.update({tag + "x_out": np.asarray(x_out), tag + "obj": np.float64(obj), tag + "loss": np.float64(loss),
                tag + "bits_per_dim": np.float64(loss) / (np.log(2.0) * 3 * 16 * 16 * B), tag + "kl_min": np.float64(kl_min)})
    out.update(x=x, seed=np.int64(seed), B=np.int64(B))
    for (i, j), e in noise.items():
        out["noise_%d_%d" % (i, j)] = e
    print("%s kl_min %.2f: obj %.6f loss %.6f bits/dim %.6f" % (tag, kl_min, float(obj), float(loss), out[tag + "bits_per_dim"]))


def main():
    tf, layers, dist, train = MG.load_tf_reference()
    extend_tf(tf)
    out = {}
    run_case(tf, layers, dist, train, 0.25, "", out)       # free bits not binding: objective == loss
    run_case(tf, layers, dist, train, 40.0, "kl40_", out)   # free bits binding on every channel
    np.savez_compressed(os.path.join(HERE, "cvae1_forward.npz"), **out)


if __name__ == "__main__":
    main()
