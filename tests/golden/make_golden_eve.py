#!/usr/bin/env python
"""Golden trajectory of the reference's Eve optimiser and its weight average (tests/golden/eve.npz), produced by
EXECUTING the reference's own ``Eve`` (graphy/misc/optim.py:125-151) on float32 numpy stand-ins, as
make_golden_optim.py runs ``AdaMaxAvg``:

* ``G.sharedf`` returns the same persistent state arrays (mom, max, delta per parameter) on every call, and ``w_avg``
  starts at the parameters' values (models.py:555);
* ``f`` is a stand-in objective that records the point ``w'`` it is called at and whose gradient depends on it:
  ``g = noise[t] + KAPPA (w' - target)`` in float32 (zero where the step's noise is zero), except on the edge steps,
  where ``g = noise[t]``.  ``G.ndict.T_grad`` returns that gradient (zeros for "c" on the steps where it is
  disconnected, ``disconnected_inputs='ignore'``), so a trajectory with the gradient taken at ``w`` instead diverges;
* ``Eve`` is called with ``alpha=-alpha`` as models.py:571 calls it, and its returned updates are applied together, as
  a Theano function applies its updates.

The noise is make_golden_optim.py's edge-case sequence: all-zero steps, sign flips, magnitudes of 1e-30 and 1e4, an
element that never sees a gradient, and steps where "c" has no gradient.  Recorded per step: the gradient used, and the
parameters, mom1, max, delta, average and the next step's lookahead (the ``w'`` of the following call).
Needs a checkout of the reference (IAF_REFERENCE, see make_golden.py):  python tests/golden/make_golden_eve.py
"""
import os
import sys
import types
from collections import OrderedDict

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import extract, py2_compile, read, _py2div  # noqa: E402
from make_golden_optim import SHAPES, STEPS, _Shared, gradient_sequence, initial_params  # noqa: E402

KAPPA = np.float32(1.5)
EDGE_STEPS = (3, 7, 8, 9, 10, 11, 12, 20, 21, 22, 23)  # the noise's edge cases, kept exactly


def targets():
    rng = np.random.RandomState(11)
    return {k: (0.5 * rng.randn(*s)).astype(np.float32) for k, s in SHAPES.items()}


def gradient_at(wp, noise_t, target, pull):
    """The stand-in objective's gradient at the point ``wp`` (float32)."""
    if not pull:
        return noise_t.copy()
    g = noise_t + KAPPA * (wp - target)
    g[noise_t == 0] = 0.0
    return g.astype(np.float32)


def eve_trajectory(params0, noise, has_c, tgt, alpha=0.002, beta1=0.1, beta2=0.001):
    state, cursor, seen = [], [0], {}

    def sharedf(x, **k):
        i = cursor[0]
        cursor[0] += 1
        if i == len(state):
            state.append(np.array(x, dtype=np.float32).view(_Shared))
        return state[i]

    def T_grad(cost, w, disconnected_inputs=None):
        return cost.grads

    G = types.SimpleNamespace(sharedf=sharedf, ndict=types.SimpleNamespace(T_grad=T_grad))
    ns = {"_py2div": _py2div, "G": G, "T": types.SimpleNamespace(maximum=np.maximum), "OrderedDict": OrderedDict,
          "np": np, "print": lambda *a, **k: None}
    src = extract(read("graphy/misc/optim.py"), r"^def Eve\(", r"^# AdaMax that keeps running average of parameter\n"
                  r"# Accumulates")
    exec(py2_compile(src, "graphy/misc/optim.py"), ns)

    w = OrderedDict((k, np.array(v, dtype=np.float32).view(_Shared)) for k, v in params0.items())
    w_avg = {k: np.array(v, dtype=np.float32).view(_Shared) for k, v in params0.items()}  # models.py:555
    out = {key: [] for key in ("grad", "param", "mom1", "mom_max", "delta", "avg", "lookahead")}
    for t in range(STEPS + 1):                      # call STEPS + 1 only records the lookahead STEPS leaves behind
        cursor[0] = 0
        seen.clear()

        def f(wp):
            seen.update({k: np.asarray(v, dtype=np.float32).copy() for k, v in wp.items()})
            grads = {}
            for k in w:
                if t == STEPS or (k == "c" and not has_c[t]):
                    grads[k] = np.zeros(SHAPES[k], np.float32)
                else:
                    grads[k] = gradient_at(seen[k], noise[k][t], tgt[k], t not in EDGE_STEPS)
            return types.SimpleNamespace(mean=lambda: types.SimpleNamespace(grads=grads))

        train_cost, new = ns["Eve"](w, w_avg, f, alpha=-alpha, beta1=beta1, beta2=beta2,
                                    disconnected_inputs="ignore")
        if t > 0:
            out["lookahead"].append(np.concatenate([seen[k].ravel() for k in w]))
        if t == STEPS:
            break
        out["grad"].append(np.concatenate([train_cost.grads[k].ravel() for k in w]))
        values = [(dst, np.asarray(v, dtype=np.float32)) for dst, v in new.items()]
        for dst, v in values:
            dst[...] = v
        out["param"].append(np.concatenate([np.asarray(v).ravel() for v in w.values()]))
        for name, j in (("mom1", 0), ("mom_max", 1), ("delta", 2)):
            out[name].append(np.concatenate([np.asarray(state[3 * i + j]).ravel() for i in range(len(w))]))
        out["avg"].append(np.concatenate([np.asarray(w_avg[k]).ravel() for k in w]))
    return {k: np.stack(v).astype(np.float32) for k, v in out.items()}


def main():
    params0, tgt = initial_params(), targets()
    noise, has_c = gradient_sequence()
    out = {"has_c": has_c, "kappa": KAPPA, "edge_steps": np.array(EDGE_STEPS)}
    for k in SHAPES:
        out["param0/" + k] = params0[k]
        out["noise/" + k] = noise[k]
        out["target/" + k] = tgt[k]
    traj = eve_trajectory(params0, noise, has_c, tgt)
    for k, v in traj.items():
        out["eve/" + k] = v
    print("eve final params", np.array2string(traj["param"][-1], precision=4))
    np.savez_compressed(os.path.join(HERE, "eve.npz"), **out)


if __name__ == "__main__":
    main()
