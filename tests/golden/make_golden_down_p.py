"""Generate tests/golden/cvae_layer_down_p.npz: the reference's own ``cvae_layer(name, 'diag', posterior, ...).down_p``
(models.py:330-359) executed, the generative half of the layer, for posterior 'down_iaf2_nl', 'up_iaf2_nl' and
'down_iaf2_nl2' (they change down_conv1's channel split), each with and without downsampling.  Same method and layout
as tests/golden/make_golden_made.py: keys ``{posterior}:{name}/...``.
usage: IAF_REFERENCE=<path of the reference checkout> python -m tests.golden.make_golden_down_p
"""
import collections
import os

import numpy as np

from tests.golden import make_golden_theano_layer as MGL

HERE = os.path.dirname(os.path.abspath(__file__))
# posterior, layer name, downsample, H of the layer's input
CASES = [(p, name, ds, 4) for p in ("down_iaf2_nl", "up_iaf2_nl", "down_iaf2_nl2") for name, ds in (("0_1", False), ("1_0", True))]


def main():
    eps_queue = collections.deque()
    models = MGL.load_theano_model(eps_queue)
    out = {}
    n_h1, n_h2, n_z, depth_ar, nl = 8, 8, 4, 1, "elu"
    for ci, (posterior, name, downsample, H) in enumerate(CASES):
        np.random.seed(51 + ci)                                                      # conv.py:156 / ar.py:288
        w = {}
        layer = models["cvae_layer"](name, "diag", posterior, n_h1, n_h2, n_z, depth_ar, downsample, nl, (3, 3), False,
                                     "nn", w)
        rng = np.random.RandomState(61 + ci)
        for k in sorted(w):                              # non-trivial scales and biases (the reference starts at 0)
            if k.endswith("_s"):
                w[k] = MGL._wrap(rng.uniform(-0.1, 0.1, size=w[k].shape))
            elif k.endswith("_b"):
                w[k] = MGL._wrap(0.05 * rng.randn(*w[k].shape))
        B = 2
        down_in = rng.randn(B, n_h1, H, H)
        eps = rng.randn(B, n_z, H, H)
        down_out = layer.down_p(MGL._wrap(down_in), MGL._wrap(eps), w)
        assert not eps_queue
        pre = "%s:%s/" % (posterior, name)
        out.update({pre + "w/" + k: np.asarray(v) for k, v in w.items() if "_down_conv" in k})   # all down_p reads
        out.update({pre + k: np.asarray(v) for k, v in dict(
            down_in=down_in, eps=eps, down_out=down_out, downsample=np.int64(downsample)).items()})
        print(pre, np.asarray(down_out).shape)
    np.savez_compressed(os.path.join(HERE, "cvae_layer_down_p.npz"), **out)
    print("written", os.path.join(HERE, "cvae_layer_down_p.npz"), len(out), "arrays")


if __name__ == "__main__":
    main()
