"""Generate tests/golden/cvae_layer_made.npz: the reference's own ``cvae_layer(name, 'made', posterior, ...)``
(models.py:14-328) executed, ``.up`` then ``.down_q``, with the autoregressive (MADE) prior (models.py:36-38, 304-309,
328) and posterior 'down_iaf2_nl', 'up_iaf2_nl' and 'down_iaf2_nl2', each with and without downsampling.  Same method
and layout as tests/golden/make_golden_theano_layer.py (whose loader this reuses): keys ``{posterior}:{name}/...``.
usage: IAF_REFERENCE=<path of the reference checkout> python -m tests.golden.make_golden_made
"""
import collections
import os

import numpy as np

from tests.golden import make_golden_theano_layer as MGL

HERE = os.path.dirname(os.path.abspath(__file__))
# posterior, layer name, downsample, H of the layer's input
CASES = [(p, name, ds, 8) for p in ("down_iaf2_nl", "up_iaf2_nl", "down_iaf2_nl2") for name, ds in (("0_1", False), ("1_0", True))]


def main():
    eps_queue = collections.deque()
    models = MGL.load_theano_model(eps_queue)
    out = {}
    n_h1, n_h2, n_z, depth_ar, nl = 8, 8, 4, 1, "elu"
    for ci, (posterior, name, downsample, H) in enumerate(CASES):
        np.random.seed(31 + ci)                                                      # conv.py:156 / ar.py:288
        w = {}
        layer = models["cvae_layer"](name, "made", posterior, n_h1, n_h2, n_z, depth_ar, downsample, nl, (3, 3), False,
                                     "nn", w)
        assert any("_prior_conv1_" in k for k in w)
        rng = np.random.RandomState(41 + ci)
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
        if posterior == "up_iaf2_nl":
            eps_queue.append(eps)                        # the posterior sample is drawn (and transformed) in up()
            up_out = layer.up(MGL._wrap(up_in), w)
        else:
            eps_queue.append(rng.randn(B, n_z, Hd, Hd))  # qz[0] in up() draws a sample the down posteriors never use
            up_out = layer.up(MGL._wrap(up_in), w)
            eps_queue.append(eps)
        down_out, kl = layer.down_q(MGL._wrap(down_in), True, w)
        assert not eps_queue
        pre = "%s:%s/" % (posterior, name)
        out.update({pre + "w/" + k: np.asarray(v) for k, v in w.items()})
        out.update({pre + k: np.asarray(v) for k, v in dict(
            up_in=up_in, down_in=down_in, eps=eps, up_out=up_out, down_out=down_out, kl=kl,
            downsample=np.int64(downsample)).items()})
        print(pre, np.asarray(kl).shape)
    np.savez_compressed(os.path.join(HERE, "cvae_layer_made.npz"), **out)
    print("written", os.path.join(HERE, "cvae_layer_made.npz"), len(out), "arrays")


if __name__ == "__main__":
    main()
