"""Golden vectors of the Theano front-end's stochastic layer, produced by EXECUTING the reference's own source:
`cvae_layer(...).up` / `.down_q` (models.py:14-328) with `N.conv.conv2d` (graphy/nodes/conv.py:122-274),
`N.ar.multiconv2d` (graphy/nodes/ar.py), `N.rand.gaussian_diag` (graphy/nodes/rand.py:78-87) and the
nearest-neighbour resamplers (conv.py:36-49), for posterior='down_iaf2_nl' and 'up_iaf2_nl', prior='diag'.

Needs a checkout of the reference (IAF_REFERENCE, see make_golden.py):  python tests/golden/make_golden_theano_layer.py
Writes tests/golden/cvae_layer_down.npz.  Same approach as make_golden.py: python2 -> python3 syntax shims, an
eager ndarray stand-in for Theano tensors, cuDNN replaced by torch CPU float64 convolution.
"""
import collections
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
from tests.golden import make_golden as MG  # noqa: E402

RT = MG.RT


class RTF(RT):
    """RT plus Theano's flatten(ndim) (keep the first ndim-1 axes)."""

    def flatten(self, ndim=1):
        a = np.asarray(self)
        return RTF(a.reshape(a.shape[: ndim - 1] + (-1,)))


def _wrap(a):
    return RTF(np.asarray(a, dtype=np.float64))


def load_theano_model(eps_queue):
    import torch
    T = types.ModuleType("theano.tensor")
    for nm in ("exp", "sqrt", "log", "tanh", "floor"):
        setattr(T, nm, (lambda f: (lambda x: _wrap(f(np.asarray(x, dtype=np.float64)))))(getattr(np, nm)))
    T.zeros = lambda shape, dtype=None: _wrap(np.zeros(tuple(int(s) for s in shape)))
    T.switch = lambda c, a, b: _wrap(np.where(c, a, b))
    T.maximum = lambda a, b: _wrap(np.maximum(a, b))
    T.concatenate = lambda xs, axis=0: _wrap(np.concatenate([np.asarray(x) for x in xs], axis=axis))
    T.mean = lambda x, axis=None: _wrap(np.mean(np.asarray(x), axis=axis))

    def set_subtensor(sub, val):
        base = MG._root(sub)
        sub[...] = val
        return _wrap(base)
    T.set_subtensor = set_subtensor
    T.nnet = types.SimpleNamespace(softplus=lambda x: _wrap(np.logaddexp(0, np.asarray(x))),
                                   sigmoid=lambda x: _wrap(1 / (1 + np.exp(-np.asarray(x)))))

    class Struct:  # graphy/__init__.py:35-39
        def __init__(self, **entries):
            self.__dict__.update(entries)

        def __call__(self, *a, **k):
            return self.__dict__["__call__"](*a, **k)

    class _Rng:  # G.rng_curand: the test supplies the N(0,1) draws
        def normal(self, size=None, **k):
            e = eps_queue.popleft()
            assert tuple(e.shape) == tuple(int(s) for s in size)
            return _wrap(e)

    G = types.ModuleType("graphy")
    G.floatX = "float64"
    G.sharedf = lambda x, **k: _wrap(x)
    G.Struct = Struct
    G.rng_curand = _Rng()

    theano = types.ModuleType("theano")
    theano.tensor = T
    theano.config = types.SimpleNamespace(device="gpu", floatX="float64")
    dnn = types.ModuleType("theano.sandbox.cuda.dnn")

    def dnn_conv(h, kerns, border_mode="valid", subsample=(1, 1), conv_mode="conv"):
        assert border_mode == "valid"
        w = torch.from_numpy(np.ascontiguousarray(np.asarray(kerns, dtype=np.float64)))
        if conv_mode == "conv":
            w = torch.flip(w, dims=(2, 3))
        x = torch.from_numpy(np.ascontiguousarray(np.asarray(h, dtype=np.float64)))
        return _wrap(torch.nn.functional.conv2d(x, w, stride=tuple(int(s) for s in subsample)).numpy())
    dnn.dnn_conv = dnn_conv
    dnn.dnn_pool = None

    N = types.ModuleType("graphy.nodes")
    G.nodes = N
    mods = {"theano": theano, "theano.tensor": T, "theano.sandbox": types.ModuleType("theano.sandbox"),
            "theano.sandbox.cuda": types.ModuleType("theano.sandbox.cuda"), "theano.sandbox.cuda.dnn": dnn,
            "graphy": G, "graphy.nodes": N}
    saved = {k: sys.modules.get(k) for k in list(mods) + ["graphy.nodes.conv", "graphy.nodes.rand", "graphy.nodes.ar"]}
    sys.modules.update(mods)
    try:
        init_src = MG.read("graphy/nodes/__init__.py")
        ns = {"_py2div": MG._py2div, "T": T, "G": G, "np": np}
        exec(MG.py2_compile(MG.extract(init_src, r"^def nonlinearity", r"^# n_in is an int"), "graphy/nodes/__init__.py"), ns)
        N.nonlinearity = ns["nonlinearity"]
        for sub in ("conv", "rand", "ar"):
            m = types.ModuleType("graphy.nodes." + sub)
            m.__dict__["_py2div"] = MG._py2div
            sys.modules["graphy.nodes." + sub] = m
            setattr(N, sub, m)
            exec(MG.py2_compile(MG.read("graphy/nodes/%s.py" % sub), "graphy/nodes/%s.py" % sub), m.__dict__)
        models = {"_py2div": MG._py2div}
        src = MG.extract(MG.read("models.py"), r"^import graphy as G", r"^# Conv VAE")   # imports + cvae_layer only
        exec(MG.py2_compile(src, "models.py"), models)
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    return models


def main():
    eps_queue = collections.deque()
    models = load_theano_model(eps_queue)
    out = {}
    n_h1, n_h2, n_z, depth_ar, nl = 8, 8, 4, 1, "elu"
    for name, posterior, downsample, H in (("0_1", "down_iaf2_nl", False, 8), ("1_0", "down_iaf2_nl", True, 8),
                                           ("u0_1", "up_iaf2_nl", False, 8), ("u1_0", "up_iaf2_nl", True, 8)):
        np.random.seed((11 if downsample else 7) + (100 if posterior[0] == "u" else 0))   # conv.py:156 / ar.py:288
        w = {}
        layer = models["cvae_layer"](name, "diag", posterior, n_h1, n_h2, n_z, depth_ar, downsample, nl, (3, 3),
                                     False, "nn", w)
        rng = np.random.RandomState((5 if downsample else 3) + (100 if posterior[0] == "u" else 0))
        for k in sorted(w):                              # non-trivial scales and biases (the reference starts at 0)
            if k.endswith("_s"):
                w[k] = _wrap(rng.uniform(-0.1, 0.1, size=w[k].shape))
            elif k.endswith("_b"):
                w[k] = _wrap(0.05 * rng.randn(*w[k].shape))
        B = 2
        up_in = rng.randn(B, n_h1, H, H)
        Hd = H // 2 if downsample else H                 # resolution of the stochastic layer and of the top-down input
        down_in = rng.randn(B, n_h1, Hd, Hd)
        eps = rng.randn(B, n_z, Hd, Hd)
        if posterior == "up_iaf2_nl":
            eps_queue.append(eps)                        # the posterior sample is drawn (and transformed) in up()
            up_out = layer.up(_wrap(up_in), w)
        else:
            eps_queue.append(rng.randn(B, n_z, Hd, Hd))  # qz[0] in up() draws a sample that down_iaf2_nl never uses
            up_out = layer.up(_wrap(up_in), w)
            eps_queue.append(eps)
        down_out, kl = layer.down_q(_wrap(down_in), True, w)
        assert not eps_queue
        out.update({name + "/w/" + k: np.asarray(v) for k, v in w.items()})
        out.update({name + "/" + k: np.asarray(v) for k, v in dict(
            up_in=up_in, down_in=down_in, eps=eps, up_out=up_out, down_out=down_out, kl=kl,
            downsample=np.int64(downsample)).items()})
    np.savez_compressed(os.path.join(HERE, "cvae_layer_down.npz"), **out)
    print("written", os.path.join(HERE, "cvae_layer_down.npz"), len(out), "arrays")


if __name__ == "__main__":
    main()
