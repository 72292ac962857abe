"""Generate tests/golden/flipmask.npz: the reference's own graphy/nodes/ar.py executed with flipmask=True.

Same method as make_golden.py (whose loader this reuses): the reference's python-2 source is exec'd against numpy
stand-ins for the few Theano primitives it calls, float64 throughout.  Written:
  * ``mask_{n_in}_{n_out}_{zd}``: the flipped mask of ar.conv2d, recovered through postup() of an all-ones update
    (ar.py:369-373; the mask is built inline and visible nowhere else);
  * ``{case}_out{k}``: head k of ar.multiconv2d(..., flipmask=True) for the inputs tests/golden/cases.py's generators
    give the seeds below (n_out >= n_in and <, depth_ar 0 / 1 / 2, one and two heads, non-square maps), plus an input
    checksum.
It also writes tests/golden/cvae_layer_nl2.npz: ``cvae_layer.up`` / ``down_q`` of the reference's models.py with
posterior='down_iaf2_nl2' (two IAF steps, the second with flipmask=True; models.py:93-98, 273-291), prior 'diag', with
and without downsampling -- the same method and layout as tests/golden/make_golden_theano_layer.py (cvae_layer_down.npz).
usage: IAF_REFERENCE=<path of the reference checkout> python -m tests.golden.make_golden_flipmask
"""
import collections
import os

import numpy as np

from oracle import iaf_oracle as O
from tests.golden import make_golden as MG
from tests.golden import make_golden_theano_layer as MGL
from tests.golden.cases import checksum

HERE = os.path.dirname(os.path.abspath(__file__))

MASK_SHAPES = [(4, 8), (8, 4), (4, 4), (32, 64), (64, 32), (8, 8)]

FLIP_CASES = [
    # name, B, n_z, hidden, heads, H, W, nl
    ("d1", 3, 4, [8], [4, 4], 5, 6, "elu"),
    ("d0", 2, 4, [], [4, 4], 5, 5, "elu"),
    ("d2", 2, 4, [8, 8], [4, 4], 3, 7, "relu"),
    ("one_head_up", 2, 4, [4], [8], 4, 6, "elu"),    # heads wider than their input (n_out > n_in)
    ("narrow_hidden", 2, 8, [4], [8, 8], 6, 5, "elu"),  # hidden narrower than z (n_out < n_in), heads wider
    ("c1", 2, 32, [64], [32, 32], 8, 8, "elu"),
]


def case_inputs(ci, B, n_z, hidden, heads, H, W):
    hid, hd = O.make_params("theano", n_z, hidden, heads, seed=ci + 300)
    z, ctx = O.make_inputs(B, n_z, hidden[0] if hidden else n_z, H, W, seed=ci + 200)
    return hid, hd, z, ctx


def main():
    ar, _ = MG.load_theano_reference()
    out = {}
    for n_in, n_out in MASK_SHAPES:
        for zd in (False, True):
            w = {}
            c = ar["conv2d"]("m", n_in, n_out, (3, 3), zd, True, w=w)
            out["mask_%d_%d_%d" % (n_in, n_out, zd)] = MG._theano_mask_via_postup(c, w).astype(np.uint8)
    for ci, (name, B, n_z, hidden, heads, H, W, nl) in enumerate(FLIP_CASES):
        hid, hd, z, ctx = case_inputs(ci, B, n_z, hidden, heads, H, W)
        w = {}
        np.random.seed(0)
        op = ar["multiconv2d"]("p", n_z, list(hidden), list(heads), (3, 3), True, nl=nl, w=w)
        for pre, ls in (("p_", hid), ("p_out_", hd)):
            for i, l in enumerate(ls):
                for k in "wsb":
                    w["%s%d_%s" % (pre, i, k)] = MG.RT(l[k].astype(np.float64))
        res = op(MG.RT(z.astype(np.float64)), MG.RT(ctx.astype(np.float64)), w)
        res = [res] if len(heads) == 1 else res
        for k, r in enumerate(res):
            out["%s_out%d" % (name, k)] = np.asarray(r)
        out[name + "_insum"] = np.float64(checksum(z, ctx, *[v for l in hid + hd for v in l.values()]))
        print(name, [np.asarray(r).shape for r in res])
    np.savez_compressed(os.path.join(HERE, "flipmask.npz"), **out)
    print("written", os.path.join(HERE, "flipmask.npz"), len(out), "arrays")
    nl2_layer()


NL2_CASES = [("0_1", False, 8), ("1_0", True, 8)]   # name, downsample, H of the layer's input


def nl2_layer():
    eps_queue = collections.deque()
    models = MGL.load_theano_model(eps_queue)
    out = {}
    n_h1, n_h2, n_z, depth_ar, nl = 8, 8, 4, 1, "elu"
    for name, downsample, H in NL2_CASES:
        np.random.seed(21 if downsample else 17)                                     # conv.py:156 / ar.py:288
        w = {}
        layer = models["cvae_layer"](name, "diag", "down_iaf2_nl2", n_h1, n_h2, n_z, depth_ar, downsample, nl, (3, 3),
                                     False, "nn", w)
        assert any("_posterior_conv2_" in k for k in w)
        rng = np.random.RandomState(13 if downsample else 12)
        for k in sorted(w):                              # non-trivial scales and biases (the reference starts at 0)
            if k.endswith("_s"):
                w[k] = MGL._wrap(rng.uniform(-0.1, 0.1, size=w[k].shape))
            elif k.endswith("_b"):
                w[k] = MGL._wrap(0.05 * rng.randn(*w[k].shape))
        B = 2
        up_in = rng.randn(B, n_h1, H, H)
        Hd = H // 2 if downsample else H
        down_in = rng.randn(B, n_h1, Hd, Hd)
        eps = rng.randn(B, n_z, Hd, Hd)
        eps_queue.append(rng.randn(B, n_z, Hd, Hd))      # qz[0] in up() draws a sample that down_iaf2_nl2 never uses
        up_out = layer.up(MGL._wrap(up_in), w)
        eps_queue.append(eps)
        down_out, kl = layer.down_q(MGL._wrap(down_in), True, w)
        assert not eps_queue
        out.update({name + "/w/" + k: np.asarray(v) for k, v in w.items()})
        out.update({name + "/" + k: np.asarray(v) for k, v in dict(
            up_in=up_in, down_in=down_in, eps=eps, up_out=up_out, down_out=down_out, kl=kl,
            downsample=np.int64(downsample)).items()})
    np.savez_compressed(os.path.join(HERE, "cvae_layer_nl2.npz"), **out)
    print("written", os.path.join(HERE, "cvae_layer_nl2.npz"), len(out), "arrays")


if __name__ == "__main__":
    main()
