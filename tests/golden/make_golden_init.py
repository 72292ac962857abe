#!/usr/bin/env python
"""Golden vectors of the data-dependent initialisation of both restated models, produced by EXECUTING the reference's
own init passes:

* TF (tests/golden/init_tf.npz): ``CVAE1._forward`` in mode "init" (tf_train.py:161-219, 222-228), i.e.
  ``arg_scope([conv2d, deconv2d], init=True)`` reaching every ``conv2d`` / ``deconv2d`` and, through ``ar_multiconv2d``
  / ``ar_conv2d``'s nested ``arg_scope``, every masked conv (tf_utils/layers.py:38-51, 86-100, 144-166).  The stand-in
  here implements ``arg_scope`` / ``add_arg_scope`` (make_golden_cvae1.py's asserts ``init=False``), and
  ``get_variable`` draws V from N(0, 0.05) (rounded to float32) and records the g and b the init branches create.
* Theano (tests/golden/init_theano.npz): ``cvae1(..., data_init={'x': x})`` (models.py:384-544): its one
  ``f_encode_decode`` with ``w['__init']`` set, through every ``N.conv.conv2d`` datainit branch (graphy/nodes/conv.py:
  225-250) and ``ar.conv2d`` init branch (graphy/nodes/ar.py:331-353), for every posterior and prior the restatement
  accepts.  The loader is make_golden_theano_layer.py's, with ``cvae1`` exec'd in the same namespace.

Both write the initial parameters, the initialised ones, the image batch, the noise and the init-mode ELBO terms.
Needs a checkout of the reference (IAF_REFERENCE, see make_golden.py):  python tests/golden/make_golden_init.py
"""
import collections
import contextlib
import functools
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
sys.path.insert(0, HERE)
import make_golden as MG  # noqa: E402
import make_golden_cvae1 as MC  # noqa: E402
import make_golden_theano_layer as MT  # noqa: E402
from iaf_b200 import elbo_theano as ET  # noqa: E402  (only for the parameter names and shapes)
from make_golden import RT, _py2div, extract, py2_compile, read  # noqa: E402

TF_HPS = dict(z_size=4, h_size=8, depth=2, num_blocks=2, kl_min=0.25, image_size=16)
TH_HPS = dict(n_z=4, n_h1=4, n_h2=8, depths=[1, 1], depth_ar=2, nl="elu", kl_min=0.25, image_size=16)
B = 4


# ---------------------------------------------------------------------------------------------------------------------
# TF
# ---------------------------------------------------------------------------------------------------------------------
class _ArgScopes(object):
    """tensorflow.contrib.framework's arg_scope / add_arg_scope: nested scopes merge, explicit kwargs win."""

    def __init__(self):
        self.stack = [{}]

    @contextlib.contextmanager
    def arg_scope(self, fns, **kw):
        cur = {k: dict(v) for k, v in self.stack[-1].items()}
        for f in fns:
            cur.setdefault(getattr(f, "_scope_key", f), {}).update(kw)
        self.stack.append(cur)
        try:
            yield
        finally:
            self.stack.pop()

    def add_arg_scope(self, f):
        @functools.wraps(f)
        def g(*a, **k):
            kw = dict(self.stack[-1].get(g, {}))
            kw.update(k)
            return f(*a, **kw)
        g._scope_key = g
        return g


class _Normal(object):
    def __init__(self, mean, stddev, dtype=None):
        self.stddev = stddev


def load_tf_init(rng):
    """tf_utils/layers.py + distributions.py + common.split + tf_train.IAFLayer, with a working arg_scope."""
    tf = MG.TFShim()
    MC.extend_tf(tf)
    scopes = _ArgScopes()
    tf.drawn, tf.created = {}, {}

    def get_variable(name, shape=None, dtype=None, initializer=None):
        key = "/".join(tf.scope + [name])
        if isinstance(initializer, _Normal):              # V: the init branch's random_normal_initializer(0, 0.05)
            if key not in tf.drawn:
                tf.drawn[key] = (initializer.stddev * rng.randn(*[int(s) for s in shape])).astype(np.float32).astype(np.float64)
            return RT(tf.drawn[key])
        if initializer is not None:                       # g and b: tf.get_variable("g", initializer=...)
            tf.created[key] = np.asarray(initializer, dtype=np.float64).copy()
            return RT(tf.created[key])
        return RT(tf.store[key])
    tf.get_variable = get_variable
    tf.random_normal_initializer = _Normal
    tf.sqrt = lambda x: RT(np.sqrt(np.asarray(x)))
    tf.nn.moments = lambda x, axes: (RT(np.mean(np.asarray(x), axis=tuple(axes))),
                                     RT(np.var(np.asarray(x), axis=tuple(axes))))
    fw = types.ModuleType("tensorflow.contrib.framework.python.ops")
    fw.arg_scope = scopes.arg_scope
    fw.add_arg_scope = scopes.add_arg_scope
    mods = {"tensorflow": tf, "tensorflow.contrib": types.ModuleType("c"),
            "tensorflow.contrib.framework": types.ModuleType("c"),
            "tensorflow.contrib.framework.python": types.ModuleType("c"),
            "tensorflow.contrib.framework.python.ops": fw}
    saved = {k: sys.modules.get(k) for k in mods}
    sys.modules.update(mods)
    try:
        layers = {"_py2div": _py2div}
        exec(py2_compile(read("tf_utils/layers.py"), "tf_utils/layers.py"), layers)
        dist = {"_py2div": _py2div}
        exec(py2_compile(read("tf_utils/distributions.py"), "tf_utils/distributions.py"), dist)
        common = {"_py2div": _py2div, "np": np, "tf": tf}
        exec(py2_compile(extract(read("tf_utils/common.py"), r"^def split\(", r"^def "), "tf_utils/common.py"), common)
        train = {"_py2div": _py2div, "np": np, "tf": tf, "arg_scope": scopes.arg_scope,
                 "conv2d": layers["conv2d"], "deconv2d": layers["deconv2d"], "ar_multiconv2d": layers["ar_multiconv2d"],
                 "resize_nearest_neighbor": layers["resize_nearest_neighbor"],
                 "DiagonalGaussian": dist["DiagonalGaussian"], "split": common["split"]}
        exec(py2_compile(extract(read("tf_train.py"), r"^class IAFLayer", r"^def get_default_hparams"), "tf_train.py"),
             train)
        src = extract(read("tf_train.py"), r"^    def _forward\(self, x, gpu\):", r"^def run\(hps\)")
        src = "\n".join(l[4:] if l.startswith("    ") else l for l in src.splitlines())   # de-indent the method
        fwd = {"_py2div": _py2div, "np": np, "tf": tf, "arg_scope": scopes.arg_scope, "conv2d": layers["conv2d"],
               "deconv2d": layers["deconv2d"], "IAFLayer": train["IAFLayer"], "repeat": dist["repeat"],
               "discretized_logistic": dist["discretized_logistic"], "compute_lowerbound": dist["compute_lowerbound"]}
        exec(py2_compile(src, "tf_train.py:_forward"), fwd)
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    return tf, fwd["_forward"]


def tf_case(out):
    rng = np.random.RandomState(21)
    tf, forward = load_tf_init(np.random.RandomState(22))
    S = TF_HPS["image_size"]
    x = rng.randint(0, 256, size=(B, 3, S, S)).astype(np.uint8)
    layers = [(i, j) for i in range(TF_HPS["depth"]) for j in range(TF_HPS["num_blocks"])]
    noise = {(i, j): rng.randn(B, TF_HPS["z_size"], S // 2 ** (i + 1), S // 2 ** (i + 1)).astype(np.float32)
             for (i, j) in layers}
    tf.store.clear()
    tf.store["h_top"] = np.zeros(TF_HPS["h_size"])                 # tf_train.py:190, zeros_initializer
    tf.noise[:] = []
    for key in reversed(layers):   # IAFLayer.down builds the prior first: its sample is z in mode "init" (:56-61)
        tf.noise.append(noise[key].astype(np.float64))
        tf.noise.append(np.zeros_like(noise[key], dtype=np.float64))   # posterior.sample, unused in mode "init"
    hps = types.SimpleNamespace(batch_size=B, k=1, num_gpus=1, **TF_HPS)
    fake = types.SimpleNamespace(hps=hps, mode="init", dec_log_stdv=RT(np.float64(0.0)))   # tf_train.py:122
    x_out, obj, loss = forward(fake, RT(x.astype(np.float64)), 0)
    assert not tf.noise, "noise queue not consumed: %d left" % len(tf.noise)
    assert len(tf.created) == 2 * len(tf.drawn), (len(tf.created), len(tf.drawn))
    out.update({"V/" + k: v.astype(np.float32) for k, v in tf.drawn.items()})
    out.update({"init/" + k: v for k, v in tf.created.items()})
    out.update({"noise_%d_%d" % k: v for k, v in noise.items()})
    out.update(x=x, x_out=np.asarray(x_out), obj=np.float64(obj), loss=np.float64(loss))
    print("tf: %d convs initialised, obj %.6f loss %.6f" % (len(tf.drawn), float(obj), float(loss)))


# ---------------------------------------------------------------------------------------------------------------------
# Theano
# ---------------------------------------------------------------------------------------------------------------------
def _functional_inplace():
    """Theano's ``a += b`` builds a new variable; the eager stand-in must not write into a (``obj_kl += kl_sum`` grows a
    scalar to [B]).  shape entries carry ``astype`` as Theano's symbolic shapes do (rand.py:181)."""
    RTF = MT.RTF
    for op in ("add", "sub", "mul", "truediv"):
        f = getattr(np.ndarray, "__%s__" % op)
        setattr(RTF, "__i%s__" % op, (lambda f: lambda self, o: MT._wrap(f(np.asarray(self), np.asarray(o))))(f))
    RTF.shape = property(lambda self: tuple(np.int64(s) for s in np.ndarray.shape.__get__(self)))
    RTF.get_value = lambda self: np.asarray(self).copy()

    def set_value(self, v):
        self[...] = v
    RTF.set_value = set_value


def theano_cases(out):
    _functional_inplace()
    S = TH_HPS["image_size"]
    depths = TH_HPS["depths"]
    layers = [(i, j) for i in range(len(depths)) for j in range(depths[i])]
    # cvae1 runs its init pass inside the constructor and drops its results (models.py:541-544); this one statement is
    # rewritten to keep them, nothing else in the source changes
    src = extract(read("models.py"), r"^def cvae1\(", r"^# Fully-connected VAE")
    init_call = "        f_encode_decode(w)\n        w.pop('__init')"
    assert src.count(init_call) == 1
    src = src.replace(init_call, "        _INIT_RESULTS.append(f_encode_decode(w))\n        w.pop('__init')")
    cases = [(p, q) for p in ("down_iaf2_nl", "up_iaf2_nl", "down_iaf2_nl2", "down_iaf2", "up_iaf2") for q in ("diag", "made")]
    for ci, (posterior, prior) in enumerate(cases):
        tag = "%s_%s/" % (posterior, prior)
        rng = np.random.RandomState(100 + ci)
        x = rng.randint(0, 256, size=(B, 3, S, S)).astype(np.uint8)
        f32 = lambda a: a.astype(np.float32).astype(np.float64)
        up_eps = {k: f32(rng.randn(B, TH_HPS["n_z"], S // 2 ** (k[0] + 1), S // 2 ** (k[0] + 1))) for k in layers}
        down_eps = {k: f32(rng.randn(*up_eps[k].shape)) for k in layers}
        queue = collections.deque()
        models = MT.load_theano_model(queue)
        T, G = models["T"], models["G"]
        T.tensor4 = lambda name, dtype=None: MT._wrap(x)            # x.tag.test_value = data_init['x'] (models.py:426)
        T.clip = lambda a, lo, hi: MT._wrap(np.clip(np.asarray(a), lo, hi))
        T.tile = lambda a, reps: MT._wrap(np.tile(np.asarray(a), tuple(int(r) for r in reps)))
        created = {}
        sharedf = G.sharedf

        def record(v, **k):        # every parameter's initial value, rounded to float16 so the fixture stores it exactly
            a = sharedf(np.asarray(v, dtype=np.float16).astype(np.float64), **k)
            created[id(a)] = np.asarray(a).copy()
            return a
        G.sharedf = record
        models["_INIT_RESULTS"] = []
        exec(py2_compile(src, "models.py:cvae1"), models)
        # draw order: every layer's up() draws qz[0].sample bottom-up (models.py:144); the down posteriors draw their
        # sample again top-down (models.py:275)
        queue.extend(up_eps[k] for k in layers)
        if posterior.startswith("down"):
            queue.extend(down_eps[k] for k in reversed(layers))
        np.random.seed(200 + ci)                                     # conv.py:172 / ar.py:288: the 0.05 randn kernels
        model = models["cvae1"]([3, S, S], list(depths), TH_HPS["depth_ar"], TH_HPS["n_h1"], TH_HPS["n_h2"],
                                 TH_HPS["n_z"], prior=prior, posterior=posterior, nl=TH_HPS["nl"],
                                 kl_min=TH_HPS["kl_min"], data_init={"x": x}, downsample_type="nn")
        assert not queue, "noise queue not consumed: %d left" % len(queue)
        (results,) = models["_INIT_RESULTS"]
        w = model.w
        assert all(np.array_equal(created[id(v)], np.asarray(v)) for k, v in w.items() if k.endswith("_w"))
        # two flat vectors per case, in sorted name order with elbo_theano.make_params' shapes: every initial value,
        # and the initialised values of every parameter but the kernels (which the pass leaves as they are)
        names = sorted(w)
        shapes = {k: v.shape for k, v in ET.make_params(dict(TH_HPS, posterior=posterior, prior=prior)).items()}
        assert names == sorted(shapes) and all(np.asarray(w[k]).shape == shapes[k] for k in names)
        out[tag + "w0"] = np.concatenate([created[id(w[k])].ravel() for k in names]).astype(np.float16)
        out[tag + "w"] = np.concatenate([np.asarray(w[k]).ravel() for k in names if not k.endswith("_w")])
        out.update({tag + "eps_%d_%d" % k: (up_eps if posterior.startswith("up") else down_eps)[k].astype(np.float32)
                    for k in layers})
        out.update({tag + "results/" + k: np.asarray(v) for k, v in results.items()})
        out[tag + "x"] = x
        changed = sum(not np.array_equal(created[id(v)], np.asarray(v)) for v in w.values())
        print("theano %s / %s: %d of %d parameters initialised, cost %s" % (
            posterior, prior, changed, len(w), np.array2string(np.asarray(results["cost"]), precision=5)))


def main():
    tf_out, th_out = {}, {}
    tf_case(tf_out)
    theano_cases(th_out)
    np.savez_compressed(os.path.join(HERE, "init_tf.npz"), **tf_out)
    np.savez_compressed(os.path.join(HERE, "init_theano.npz"), **th_out)


if __name__ == "__main__":
    main()
