"""Time the MADE prior's fused log-density entry (IAFOperator.ar_logp, iaf_ar_logp_fwd) against the composition it
replaces: the IAF step (z', arw_logsd written to HBM), then torch for logps = -0.5 log 2pi - arw_logsd - 0.5 z'^2 and
its per-(sample, channel) and per-sample sums.  Also times the training pair (iaf_ar_logp_fwd_train +
iaf_ar_logp_bwd_saved through the autograd node).  Shapes: the prior of c2a (n_z 32, hidden [64]) and c2b (n_z 32,
hidden [160, 160]), Theano variant, 16x16, B = 256.  CUDA events around K calls of each, the variants alternating over
several rounds after a warm-up (eager calls: the host's launch time counts where it is not hidden behind the GPU).
Prints one JSON line with the card's name and power limit.
usage: python tools/bench_made.py [steps] [rounds]"""
import json
import math
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from iaf_b200 import IAFOperator  # noqa: E402
from oracle import iaf_oracle as O  # noqa: E402  (synthetic parameter / input generator only)

C = 0.5 * math.log(2 * math.pi)


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # the timing does not depend on it
        return "unknown (%s)" % e


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 100
    rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    n_z, H, W, B = 32, 16, 16, 256
    out = {"gpu": torch.cuda.get_device_name(0), "card": card(), "B": B, "steps": steps, "rounds": rounds}
    for shape, hidden in (("c2a", [64]), ("c2b", [160, 160])):
        hid, hd = O.make_params("theano", n_z, hidden, [n_z, n_z], seed=1)
        z, ctx = O.make_inputs(B, n_z, hidden[0], H, W, seed=0)
        dev = [tuple(torch.from_numpy(np.ascontiguousarray(l[k])).cuda() for k in "wsb") for l in hid + hd]
        op = IAFOperator("theano", n_z, hidden, [n_z, n_z], nl="elu").set_weights(dev)
        params = [tuple(t.clone().requires_grad_(True) for t in l) for l in dev]
        op_train = IAFOperator("theano", n_z, hidden, [n_z, n_z], nl="elu").set_weights(params)
        zg, cg = torch.from_numpy(z).cuda(), torch.from_numpy(ctx).cuda()

        def fused():
            return op.ar_logp(zg, cg)

        def composed():
            zo, logsd, _ = op.step(zg, cg, want_logdet=False)
            logps = -C - logsd - 0.5 * zo * zo
            bc = logps.sum(dim=(2, 3))
            return logps, bc, bc.sum(dim=1)

        def train():
            _, bc, lp = op_train.ar_logp(zg, cg)
            (bc.sum() + lp.sum()).backward()

        runs = {"fused_ar_logp": fused, "step_plus_torch": composed, "train_pair": train}
        with torch.no_grad():
            ref = composed()[2]
            got = fused()[2]
        err = float((got - ref).abs().max() / ref.abs().max())
        for f in runs.values():
            for _ in range(10):
                if f is train:
                    f()
                else:
                    with torch.no_grad():
                        f()
        torch.cuda.synchronize()
        ms = {name: [] for name in runs}
        for _ in range(rounds):
            for name, f in runs.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                with torch.set_grad_enabled(f is train):
                    e0.record()
                    for _ in range(steps):
                        f()
                    e1.record()
                torch.cuda.synchronize()
                ms[name].append(e0.elapsed_time(e1) / steps)
        med = {name: statistics.median(v) for name, v in ms.items()}
        out[shape] = {"hidden": hidden, "path": op.path_used(H, W, "cuda:0", "ar_logp"),
                      "bwd_path": op_train.backward_path(H, W, "cuda:0"), "ms_per_call": ms, "median_ms": med,
                      "fused_over_composed": med["fused_ar_logp"] / med["step_plus_torch"],
                      "logp_rel_diff_fused_vs_composed": err}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
