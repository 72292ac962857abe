"""Generate tests/golden/cvae_layer_linear.npz: the reference's own ``cvae_layer(name, prior, posterior, ...)``
(models.py:14-328) executed, ``.up`` then ``.down_q``, for the linear IAF posteriors 'down_iaf2' and 'up_iaf2'
(models.py:55-56, 79-82, 152-161, 246-259: one ``ar.conv2d(n_z, 2 n_z)`` with interleaved heads, no context), each with
prior 'diag' and 'made', each with and without downsampling, plus one 'made' case with depth_ar = 0 (the prior's stack
then has no hidden layer either).  Same method and layout as tests/golden/make_golden_made.py (the loader of
tests/golden/make_golden_theano_layer.py): keys ``{posterior}:{prior}:{depth_ar}:{name}/...``.
usage: IAF_REFERENCE=<path of the reference checkout> python -m tests.golden.make_golden_linear
"""
import collections
import os

import numpy as np

from tests.golden import make_golden_theano_layer as MGL

HERE = os.path.dirname(os.path.abspath(__file__))
# posterior, prior, depth_ar, layer name, downsample, H of the layer's input
CASES = ([(p, pr, 1, name, ds, 8) for p in ("down_iaf2", "up_iaf2") for pr in ("diag", "made")
          for name, ds in (("0_1", False), ("1_0", True))] +
         [("down_iaf2", "made", 0, "0_1", False, 8)])


def key(posterior, prior, depth_ar, name):
    return "%s:%s:%d:%s/" % (posterior, prior, depth_ar, name)


def main():
    eps_queue = collections.deque()
    models = MGL.load_theano_model(eps_queue)
    out = {}
    n_h1, n_h2, n_z, nl = 8, 8, 4, "elu"
    for ci, (posterior, prior, depth_ar, name, downsample, H) in enumerate(CASES):
        np.random.seed(61 + ci)                                                      # conv.py:156 / ar.py:288
        w = {}
        layer = models["cvae_layer"](name, prior, posterior, n_h1, n_h2, n_z, depth_ar, downsample, nl, (3, 3), False,
                                     "nn", w)
        assert w[name + "_posterior_conv1_w"].shape == (2 * n_z, n_z + 1, 3, 3)
        rng = np.random.RandomState(71 + ci)
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
        if posterior == "up_iaf2":
            eps_queue.append(eps)                        # the posterior sample is drawn (and transformed) in up()
            up_out = layer.up(MGL._wrap(up_in), w)
        else:
            eps_queue.append(rng.randn(B, n_z, Hd, Hd))  # qz[0] in up() draws a sample down_iaf2 never uses
            up_out = layer.up(MGL._wrap(up_in), w)
            eps_queue.append(eps)
        down_out, kl = layer.down_q(MGL._wrap(down_in), True, w)
        assert not eps_queue
        pre = key(posterior, prior, depth_ar, name)
        out.update({pre + "w/" + k: np.asarray(v) for k, v in w.items()})
        out.update({pre + k: np.asarray(v) for k, v in dict(
            up_in=up_in, down_in=down_in, eps=eps, up_out=up_out, down_out=down_out, kl=kl,
            downsample=np.int64(downsample)).items()})
        print(pre, np.asarray(kl).shape)
    np.savez_compressed(os.path.join(HERE, "cvae_layer_linear.npz"), **out)
    print("written", os.path.join(HERE, "cvae_layer_linear.npz"), len(out), "arrays")


if __name__ == "__main__":
    main()
