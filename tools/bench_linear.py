"""Time the linear IAF step (a stack without hidden layers: ``ar.conv2d(n_z, 2 n_z)``, the posteriors down_iaf2 /
up_iaf2) on the tensor cores (path="auto") against the exact-fp32 SIMT kernels (path="simt"): the inference step and the
training pair (iaf_step_fwd_train + iaf_step_bwd_saved through the autograd node).  Theano variant, n_z 32, 16x16,
B = 256.  CUDA events around K calls of each, the four arms alternating over several rounds after a warm-up (eager
calls: the host's launch time counts where it is not hidden behind the GPU).  Prints one JSON line with the card's name
and power limit, and the step's algorithmic bytes and flops (iaf_plan_algorithmic_bytes / _flops: counted from the
shapes, not measured) with the time they bound at the data sheet's 3.35 TB/s.
usage: python tools/bench_linear.py [steps] [rounds]"""
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from iaf_b200 import IAFOperator  # noqa: E402
from oracle import iaf_oracle as O  # noqa: E402  (synthetic parameter / input generator only)

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


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
    _, hd = O.make_params("theano", n_z, [], [n_z, n_z], seed=1)
    z = torch.from_numpy(O.make_inputs(B, n_z, 1, H, W, seed=0)[0]).cuda()
    dev = [tuple(torch.from_numpy(np.ascontiguousarray(l[k])).cuda() for k in "wsb") for l in hd]
    out = {"gpu": torch.cuda.get_device_name(0), "card": card(), "B": B, "n_z": n_z, "H": H, "W": W, "steps": steps,
           "rounds": rounds}
    runs, ops = {}, {}
    for path in ("auto", "simt"):
        op = IAFOperator("theano", n_z, [], [n_z, n_z], nl="elu", path=path).set_weights(dev)
        op_train = IAFOperator("theano", n_z, [], [n_z, n_z], nl="elu", path=path).set_weights(
            [tuple(t.clone().requires_grad_(True) for t in l) for l in dev])
        zt = z.clone().requires_grad_(True)   # a SIMT plan's backward is SIMT too

        def step(op=op):
            return op.step(z, None)

        def train(op=op_train, zt=zt):
            zo, ls, _ = op.step(zt, None, want_logdet=False)
            (zo.sum() + ls.sum()).backward()

        ops[path] = (op, op_train)
        runs["step_" + path], runs["train_" + path] = step, train
    with torch.no_grad():
        a, b = runs["step_auto"](), runs["step_simt"]()
    out["rel_diff_tc_vs_simt"] = {k: float((x - y).abs().max() / y.abs().max()) for k, x, y in zip(("z", "logsd", "logdet"), a, b)}
    for path, (op, op_train) in ops.items():
        out["path_" + path] = {"step": op.path_used(H, W, "cuda:0", "step"), "bwd": op_train.backward_path(H, W, "cuda:0")}
    for f in runs.values():
        for _ in range(10):
            with torch.set_grad_enabled(f.__name__ == "train"):
                f()
    torch.cuda.synchronize()
    ms = {name: [] for name in runs}
    for _ in range(rounds):
        for name, f in runs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with torch.set_grad_enabled(name.startswith("train")):
                e0.record()
                for _ in range(steps):
                    f()
                e1.record()
            torch.cuda.synchronize()
            ms[name].append(e0.elapsed_time(e1) / steps)
    med = {name: statistics.median(v) for name, v in ms.items()}
    op = ops["auto"][0]
    nbytes, flops = op.algorithmic_bytes(B, H, W, "cuda:0"), op.algorithmic_flops(B, H, W, "cuda:0")
    out.update({"ms_per_call": ms, "median_ms": med,
                "step_speedup_tc_over_simt": med["step_simt"] / med["step_auto"],
                "train_speedup_tc_over_simt": med["train_simt"] / med["train_auto"],
                "algorithmic_bytes": nbytes, "algorithmic_flops": flops,
                "hbm_bound_us": 1e6 * nbytes / HBM_BYTES_PER_S,
                "step_auto_share_of_hbm_bound": 1e6 * nbytes / HBM_BYTES_PER_S / (1e3 * med["step_auto"])})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
