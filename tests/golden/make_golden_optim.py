#!/usr/bin/env python
"""Golden trajectories of the reference's two Adamax rules and their weight averages (tests/golden/optim.npz), produced
by EXECUTING the reference's own update code on float32 numpy stand-ins:

* TF: ``AdamaxOptimizer`` (tf_utils/adamax.py), its ``_create_slots`` once and ``_apply_dense(grad, var)`` per step and
  variable, against stand-ins of ``math_ops`` / ``state_ops`` / ``ops`` / ``optimizer`` in which a tensor is a float32
  array and every operation one float32 numpy operation (python float constants are weak scalars, NEP 50, as TF
  converts them to the variable's dtype).  A variable without a gradient is skipped, as ``apply_gradients`` skips a
  None gradient.  The average is TensorFlow's ``assign_moving_average`` (library code, not the reference's):
  ``shadow -= (shadow - var) * float32(1 - 0.999)``, taken from the variable's value before the step's update.
* Theano: ``AdaMaxAvg`` (graphy/misc/optim.py:99-123) with ``alpha=-alpha`` as models.py:568 calls it, with
  ``G.ndict.T_grad`` patched to return the step's gradients (zeros for a disconnected input,
  ``disconnected_inputs='ignore'``) and ``G.sharedf`` returning the same persistent state arrays on every step.  The
  returned updates are applied together, as a Theano function applies its updates.

The gradient sequence: 30 steps over three small tensors, with all-zero steps, zero elements, sign flips, magnitudes
of 1e-30 and 1e4, and steps where tensor "c" has no gradient.
Needs a checkout of the reference (IAF_REFERENCE, see make_golden.py):  python tests/golden/make_golden_optim.py
"""
import os
import sys
import types
from collections import OrderedDict

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import extract, py2_compile, read, _py2div  # noqa: E402

SHAPES = OrderedDict([("a", (5,)), ("b", (2, 3)), ("c", (4,))])
STEPS = 30
NO_GRAD_C = (5, 6, 17)  # steps at which "c" has no gradient


def gradient_sequence():
    """{name: [STEPS, ...] float32}, and a [STEPS] bool mask of the steps at which "c" has a gradient."""
    rng = np.random.RandomState(7)
    g = {k: (rng.randn(STEPS, *s) * np.exp(rng.uniform(-3, 3, size=(STEPS,) + s))).astype(np.float32)
         for k, s in SHAPES.items()}
    for k in g:
        g[k][3] = 0.0                                   # an all-zero step
        g[k][8] = -g[k][7]                              # sign flips
        g[k][9] = -g[k][8]
        g[k][10:13] *= np.float32(1e-30) / np.maximum(np.abs(g[k][10:13]), np.float32(1e-30))  # |g| = 1e-30
        g[k][20] = np.float32(1e4) * np.sign(g[k][20])  # 1e4
        g[k][21:24] = -g[k][20]
    g["a"][:, 0] = 0.0                                  # an element that never sees a gradient
    g["b"][::4, 1, 2] = 0.0
    has_c = np.ones(STEPS, bool)
    has_c[list(NO_GRAD_C)] = False
    return g, has_c


def initial_params():
    rng = np.random.RandomState(3)
    return {k: (0.3 * rng.randn(*s)).astype(np.float32) for k, s in SHAPES.items()}


# ---------------------------------------------------------------------------------------------------------------------
class _Slot(np.ndarray):
    """A TF slot variable: a float32 array with ``assign``."""

    def assign(self, value):
        self[...] = np.asarray(value, dtype=np.float32)
        return self


class _Var(object):
    """A TF variable handed to _apply_dense: its value and the dtype the optimiser casts its constants to."""

    def __init__(self, value):
        self.value = np.array(value, dtype=np.float32)
        self.dtype = types.SimpleNamespace(base_dtype="float32")


def load_tf_adamax():
    class Optimizer(object):
        def __init__(self, use_locking, name):
            self._name, self._slots = name, {}

        def _zeros_slot(self, var, slot_name, op_name):
            self._slots[(id(var), slot_name)] = np.zeros_like(var.value).view(_Slot)

        def get_slot(self, var, name):
            return self._slots[(id(var), name)]

    def assign_sub(var, delta):
        var.value = (var.value - np.asarray(delta)).astype(np.float32)
        return var

    ns = {"_py2div": _py2div,
          "optimizer": types.SimpleNamespace(Optimizer=Optimizer),
          "ops": types.SimpleNamespace(convert_to_tensor=lambda x, name=None: np.float32(x)),
          "math_ops": types.SimpleNamespace(cast=lambda x, dtype: np.float32(x)),
          "state_ops": types.SimpleNamespace(assign_sub=assign_sub),
          "control_flow_ops": types.SimpleNamespace(group=lambda *a: None),
          "tf": types.SimpleNamespace(float16="float16", maximum=np.maximum, abs=np.abs)}
    src = extract(read("tf_utils/adamax.py"), r"^class AdamaxOptimizer", r"^\Z")
    exec(py2_compile(src, "tf_utils/adamax.py"), ns)
    return ns["AdamaxOptimizer"]


def tf_trajectory(params0, grads, has_c, lr=0.01):
    opt = load_tf_adamax()(lr)              # tf_train.py:127: AdamaxOptimizer(hps.learning_rate)
    opt._prepare()
    vars_ = OrderedDict((k, _Var(v)) for k, v in params0.items())
    opt._create_slots(list(vars_.values()))
    shadow = {k: v.value.copy() for k, v in vars_.items()}  # ema.apply: the shadow starts at the variable's value
    decay = np.float32(1.0 - 0.999)                           # assign_moving_average: convert_to_tensor(1.0 - decay)
    out = {key: [] for key in ("param", "mom1", "mom_max", "avg")}
    for t in range(STEPS):
        for k, v in vars_.items():
            shadow[k] = shadow[k] - (shadow[k] - v.value) * decay
        for k, v in vars_.items():
            if k == "c" and not has_c[t]:
                continue                                      # apply_gradients skips a None gradient
            opt._apply_dense(grads[k][t], v)
        out["param"].append(np.concatenate([v.value.ravel() for v in vars_.values()]))
        out["mom1"].append(np.concatenate([opt.get_slot(v, "v").ravel() for v in vars_.values()]))
        out["mom_max"].append(np.concatenate([opt.get_slot(v, "m").ravel() for v in vars_.values()]))
        out["avg"].append(np.concatenate([shadow[k].ravel() for k in vars_]))
    return {k: np.stack(v).astype(np.float32) for k, v in out.items()}


# ---------------------------------------------------------------------------------------------------------------------
class _Shared(np.ndarray):
    """A Theano shared variable: a float32 array that is a dict key by identity and answers get_value()."""
    __hash__ = object.__hash__

    def get_value(self):
        return np.asarray(self).copy()


def theano_trajectory(params0, grads, has_c, alpha=0.002, beta1=0.1, beta2=0.001):
    state, cursor, cur_grads = [], [0], {}

    def sharedf(x, **k):
        i = cursor[0]
        cursor[0] += 1
        if i == len(state):
            state.append(np.array(x, dtype=np.float32).view(_Shared))
        return state[i]

    G = types.SimpleNamespace(sharedf=sharedf,
                              ndict=types.SimpleNamespace(T_grad=lambda obj, ws, disconnected_inputs=None: [cur_grads]))
    ns = {"_py2div": _py2div, "G": G, "T": types.SimpleNamespace(maximum=np.maximum), "OrderedDict": OrderedDict,
          "np": np, "math": __import__("math")}
    src = extract(read("graphy/misc/optim.py"), r"^def AdaMaxAvg\(", r"^# Eve that keeps")
    exec(py2_compile(src, "graphy/misc/optim.py"), ns)

    w = OrderedDict((k, np.array(v, dtype=np.float32).view(_Shared)) for k, v in params0.items())
    w_avg = {k: np.array(v, dtype=np.float32).view(_Shared) for k, v in params0.items()}  # models.py:555
    objective = types.SimpleNamespace(sum=lambda: None)
    out = {key: [] for key in ("param", "mom1", "mom_max", "avg")}
    for t in range(STEPS):
        cursor[0] = 0
        cur_grads.clear()
        for k in w:
            g = grads[k][t] if (k != "c" or has_c[t]) else np.zeros(SHAPES[k], np.float32)
            cur_grads[k] = g
        new = ns["AdaMaxAvg"]([w], [w_avg], objective, alpha=-alpha, beta1=beta1, beta2=beta2,
                              disconnected_inputs="ignore")
        values = [(dst, np.asarray(v, dtype=np.float32)) for dst, v in new.items()]
        for dst, v in values:
            dst[...] = v
        out["param"].append(np.concatenate([np.asarray(v).ravel() for v in w.values()]))
        out["mom1"].append(np.concatenate([np.asarray(state[2 * i]).ravel() for i in range(len(w))]))
        out["mom_max"].append(np.concatenate([np.asarray(state[2 * i + 1]).ravel() for i in range(len(w))]))
        out["avg"].append(np.concatenate([np.asarray(w_avg[k]).ravel() for k in w]))
    return {k: np.stack(v).astype(np.float32) for k, v in out.items()}


def main():
    params0 = initial_params()
    grads, has_c = gradient_sequence()
    out = {"has_c": has_c}
    for k in SHAPES:
        out["param0/" + k] = params0[k]
        out["grads/" + k] = grads[k]
    for rule, traj in (("tf", tf_trajectory(params0, grads, has_c)), ("theano", theano_trajectory(params0, grads, has_c))):
        for k, v in traj.items():
            out[rule + "/" + k] = v
        print(rule, "final params", np.array2string(traj["param"][-1], precision=4))
    np.savez_compressed(os.path.join(HERE, "optim.npz"), **out)


if __name__ == "__main__":
    main()
