"""Time sampling the autoregressive (MADE) prior, IAFOperator.ar_sample (one iaf_step_inverse kernel), against the
fixed-point baseline it replaces: z <- 0.1 m(z) + exp(0.1 s(z)) eps, one iaf_step_fwd plus torch per iteration
(with z', a = step(z): 0.1 m = z - z' exp(a), so z <- z + exp(a) (eps - z')).

The fixed point is exact after at most n_z*H*W iterations (the length of the dependency chain); the script times K of
its iterations and reports the per-iteration time, the number of iterations after which the fp32 iterate reaches the
kernel's own round-trip error on this data (measured, capped), and the products of the per-iteration time with both
counts, labelled as extrapolated.  Also reports the round-trip error max|step(ar_sample(eps)).z' - eps| on the timed data,
and the reparameterised sample's training pair: ar_rsample's forward and the backward of its logp (each call timed on
its own with CUDA events), and the adjoint kernel (iaf_step_inverse_adjoint) alone.
Shapes: the prior of c2a (n_z 32, hidden [64]) and c2b (hidden [160, 160]), Theano variant, 16x16, B = 256.  CUDA
events after a warm-up, the calls alternating over several rounds.  Prints one JSON line with the card's name and power
limit.
usage: python tools/bench_sample.py [calls] [rounds] [fixed_point_cap]"""
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


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # the timing does not depend on it
        return "unknown (%s)" % e


def main():
    calls = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    cap = int(sys.argv[3]) if len(sys.argv) > 3 else 2000
    n_z, H, W, B = 32, 16, 16, 256
    out = {"gpu": torch.cuda.get_device_name(0), "card": card(), "B": B, "calls": calls, "rounds": rounds,
           "chain_length_n_z_H_W": n_z * H * W}
    for shape, hidden in (("c2a", [64]), ("c2b", [160, 160])):
        hid, hd = O.make_params("theano", n_z, hidden, [n_z, n_z], seed=1)
        eps, ctx = O.make_inputs(B, n_z, hidden[0], H, W, seed=0)
        dev = [tuple(torch.from_numpy(np.ascontiguousarray(l[k])).cuda() for k in "wsb") for l in hid + hd]
        op = IAFOperator("theano", n_z, hidden, [n_z, n_z], nl="elu").set_weights(dev)
        e, c = torch.from_numpy(eps).cuda(), torch.from_numpy(ctx).cuda()

        def sample():
            return op.ar_sample(e, c)

        z_fp = e.clone()

        def fixed_point_iteration():
            zo, a, _ = op.step(z_fp, c, want_logdet=False)
            z_fp.add_(torch.exp(a) * (e - zo))

        runs = {"ar_sample": sample, "fixed_point_iteration": fixed_point_iteration}
        with torch.no_grad():
            z = sample()[0]
            rt = float((op.step(z, c)[0] - e).abs().max())
            # iterations of the baseline until its round trip is as good as the kernel's (measured, capped)
            z_fp.copy_(e)
            iters = None
            for k in range(1, cap + 1):
                fixed_point_iteration()
                if k % 10 == 0 and float((op.step(z_fp, c)[0] - e).abs().max()) <= rt:
                    iters = k
                    break
            for f in runs.values():
                for _ in range(5):
                    f()
            torch.cuda.synchronize()
            ms = {name: [] for name in runs}
            for _ in range(rounds):
                for name, f in runs.items():
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(calls):
                        f()
                    e1.record()
                    torch.cuda.synchronize()
                    ms[name].append(e0.elapsed_time(e1) / calls)
        # the reparameterised sample's training pair: ar_rsample with eps, context and the parameters requiring grad,
        # then the backward of its logp (hidden activations at z, the adjoint, the step's saved backward); and the
        # adjoint kernel alone on the same data
        train = [tuple(t.detach().clone().requires_grad_(True) for t in l) for l in dev]
        top = IAFOperator("theano", n_z, hidden, [n_z, n_z], nl="elu").set_weights(train)
        eg, cg = e.clone().requires_grad_(True), c.clone().requires_grad_(True)
        with torch.no_grad():
            zi, lsi, _ = top.step_inverse(e, c)
            hid_act = top._step_train_raw(zi, c)[3]
            g_z, g_ls = torch.randn_like(e), torch.randn_like(e)

        def adjoint():
            return top._step_inverse_adjoint_raw(e, lsi, hid_act, g_z, g_ls)

        pair = {"ar_rsample_fwd": [], "ar_rsample_bwd": [], "adjoint_kernel": []}
        for r in range(rounds + 1):  # round 0: warm-up
            for _ in range(calls):
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
                ev[0].record()
                lp = top.ar_rsample(eg, cg)[2]
                ev[1].record()
                lp.sum().backward()
                ev[2].record()
                torch.cuda.synchronize()
                if r:
                    pair["ar_rsample_fwd"].append(ev[0].elapsed_time(ev[1]))
                    pair["ar_rsample_bwd"].append(ev[1].elapsed_time(ev[2]))
            with torch.no_grad():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(calls):
                    adjoint()
                e1.record()
                torch.cuda.synchronize()
                if r:
                    pair["adjoint_kernel"].append(e0.elapsed_time(e1) / calls)
        med = {name: statistics.median(v) for name, v in ms.items()}
        it_ms = med["fixed_point_iteration"]
        out[shape] = {
            "hidden": hidden, "step_path": op.path_used(H, W, "cuda:0", "step"), "ms_per_call": ms,
            "ar_sample_ms": med["ar_sample"], "fixed_point_ms_per_iteration": it_ms,
            "fixed_point_iterations_to_kernel_roundtrip": iters if iters is not None else "more than %d" % cap,
            "extrapolated_fixed_point_ms_at_chain_length": it_ms * n_z * H * W,
            "extrapolated_fixed_point_ms_at_measured_iterations": (it_ms * iters) if iters is not None else None,
            "roundtrip_max_abs_err": rt,
            "ar_rsample_fwd_ms": statistics.median(pair["ar_rsample_fwd"]),
            "ar_rsample_bwd_ms": statistics.median(pair["ar_rsample_bwd"]),
            "adjoint_kernel_ms": statistics.median(pair["adjoint_kernel"])}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
