"""Time the importance-sampled log-likelihood (``elbo.log_likelihood`` / ``elbo_theano.log_likelihood``) against the
reference's method on the same weights, images, k and noise: ``forward`` on ``repeat(x, chunk)`` (the up pass recomputed
for every sample), then ``compute_lowerbound``'s -log k + logsumexp over the k log-weights of each image.  That baseline
lives only here.

Workloads (synthetic weights from ``make_params``, seeded uint8 images, B = 100 = the TF model's eval_batch_size):
* ``tf``: the README's eval configuration of tf_train.py: depth 1, num_blocks 20, h_size 160, z_size 32, 32x32;
* ``theano_c2a``: the Theano model at c2a's stack shape (README cifar10 model): n_z 32, n_h1 = n_h2 = 64, depth_ar 1,
  depths [2, 2, 2], down_iaf2_nl, prior diag.
Metric: image-samples per second, B k / (time of one whole call), CUDA events around each call after a warm-up call,
the two methods alternating over the rounds in one process.  The baseline runs chunks of half the estimator's (still
2000 samples per forward at B = 100): ``forward`` keeps every layer's up-pass output for all B * chunk samples until the
top-down pass.  The 10^4-sample time of a 10^4-image test set is an
extrapolation from it.  The two methods' log_px are compared on the last timed call (same noise).

--profile: instead of timing, one call of each method at k = chunk under torch.profiler (CUDA activities), and the
share of GPU kernel time in this library's kernels (``iaf_*``), in cuDNN / GEMM convolution kernels, and in the rest
(elementwise, reductions, copies).  Prints one JSON line with the card's name and power limit.
usage: python tools/bench_marglik.py [--k K] [--rounds R] [--workload tf|theano_c2a|all] [--profile]"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from iaf_b200 import elbo  # noqa: E402
from iaf_b200 import elbo_theano as ET  # noqa: E402

B = 100
TEST_SET = 10000     # CIFAR-10's test images, at 10^4 samples each (the README's estimate)


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # the timing does not depend on it
        return "unknown (%s)" % e


def workload(name, dev):
    rng = np.random.RandomState(1)
    x = torch.from_numpy(rng.randint(0, 256, size=(B, 3, 32, 32)).astype(np.uint8)).to(dev)
    if name == "tf":
        hps = dict(z_size=32, h_size=160, depth=1, num_blocks=20, kl_min=0.0, image_size=32)
        params = {k: torch.from_numpy(np.asarray(v)).to(dev) for k, v in elbo.make_params(hps, seed=0).items()}
        iaf = elbo.CudaIAF(params, hps)
        shapes = {(i, j): (B, 32, 32 // 2 ** (i + 1), 32 // 2 ** (i + 1)) for i in range(1) for j in range(20)}
        estimator, elems = elbo.log_likelihood, elbo._elems_per_sample(hps)

        def log_weights(noise, n):
            out = elbo.forward(params, x.repeat_interleave(n, dim=0), noise, iaf, hps)
            return out["log_pxz"].double() - out["kl_cost"].double()
    else:
        hps = dict(n_z=32, n_h1=64, n_h2=64, depths=[2, 2, 2], depth_ar=1, nl="elu", kl_min=0.0, image_size=32,
                   posterior="down_iaf2_nl", prior="diag")
        params = {k: torch.from_numpy(np.asarray(v)).to(dev) for k, v in ET.make_params(hps, seed=0).items()}
        iaf = ET.CudaIAF(params, hps)
        shapes = {(i, j): (B, 32, 32 // 2 ** (i + 1), 32 // 2 ** (i + 1)) for i in range(3) for j in range(2)}
        estimator, elems = ET.log_likelihood, ET._elems_per_sample(hps)

        def log_weights(noise, n):       # train.py:193-197: cost * correction factor = the log-weight in nats
            return ET.forward(params, x.repeat_interleave(n, dim=0), noise, iaf, hps)["cost"].double() * \
                -(3 * 32 * 32 * math.log(2.0))
    return params, x, iaf, hps, shapes, estimator, elems, log_weights


def reference_method(log_weights, noise, k, chunk):
    """forward on repeat(x, chunk) per chunk, then compute_lowerbound over the k log-weights of every image."""
    with torch.no_grad():
        ws = []
        for start in range(0, k, chunk):
            n = min(chunk, k - start)
            ws.append(log_weights(noise(start, n), n).reshape(B, n))
        return torch.logsumexp(torch.cat(ws, dim=1), dim=1) - math.log(k)


def kernel_shares(prof):
    """GPU time of the profiled region by kernel family (microseconds and shares)."""
    fam = {"iaf": 0.0, "cudnn_gemm": 0.0, "other": 0.0}
    names = {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        n, t = e.name, e.time_range.elapsed_us()
        names[n] = names.get(n, 0.0) + t
        if "iaf_" in n:                   # demangled: "void iaf_ly_kernel<...>(...)"
            fam["iaf"] += t
        elif any(s in n.lower() for s in ("cudnn", "conv", "xmma", "gemm", "cutlass", "fprop", "dgrad", "wgrad",
                                          "implicit")):
            fam["cudnn_gemm"] += t
        else:
            fam["other"] += t
    total = sum(fam.values())
    top = sorted(names.items(), key=lambda kv: -kv[1])[:8]
    return {"us": fam, "share": {k: (v / total if total else 0.0) for k, v in fam.items()},
            "top_kernels_us": [(n[:100], t) for n, t in top]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--k", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--workload", default="all", choices=["tf", "theano_c2a", "all"])
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_marglik: needs a CUDA device")
    dev = torch.device("cuda:0")
    out = {"gpu": torch.cuda.get_device_name(0), "card": card(), "B": B, "k": a.k, "rounds": a.rounds,
           "cudnn_allow_tf32": torch.backends.cudnn.allow_tf32, "mode": "profile" if a.profile else "time"}
    for name in (("tf", "theano_c2a") if a.workload == "all" else (a.workload,)):
        params, x, iaf, hps, shapes, estimator, elems, log_weights = workload(name, dev)
        chunk = elbo.default_chunk(B, a.k, elems)
        k = chunk if a.profile else a.k
        ref_chunk = max(1, chunk // 2)
        gen = torch.Generator(device=dev)

        def noise(start, count):
            """Sample j of every image is drawn from a generator seeded with j: the same draws whatever the chunking."""
            per = []
            for j in range(start, start + count):
                gen.manual_seed(j)
                per.append({key: torch.randn((B, 1) + tuple(s[1:]), generator=gen, device=dev)
                            for key, s in sorted(shapes.items())})
            return {key: torch.cat([p[key] for p in per], dim=1).reshape((-1,) + tuple(shapes[key][1:]))
                    for key in shapes}
        runs = {"log_likelihood": lambda: estimator(params, x, iaf, hps, k, chunk=chunk, noise=noise)["log_px"],
                "forward_on_repeat": lambda: reference_method(log_weights, noise, k, ref_chunk)}
        res = {"chunk": chunk, "ref_chunk": ref_chunk, "k": k, "samples_per_call": B * k}
        if a.profile:
            for f in runs.values():            # warm-up
                f()
            torch.cuda.synchronize()
            for m, f in runs.items():
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    f()
                    torch.cuda.synchronize()
                res[m] = kernel_shares(prof)
            out[name] = res
            continue
        got = {m: f() for m, f in runs.items()}  # warm-up: every shape of the timed calls
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        ms = {m: [] for m in runs}
        for _ in range(a.rounds):
            for m, f in runs.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                got[m] = f()
                e1.record()
                torch.cuda.synchronize()
                ms[m].append(e0.elapsed_time(e1))
        med = {m: statistics.median(v) for m, v in ms.items()}
        ll, ref = got["log_likelihood"], got["forward_on_repeat"]
        res.update({
            "ms_per_call": ms, "median_ms": med,
            "image_samples_per_s": {m: B * k / (t / 1e3) for m, t in med.items()},
            "speedup_over_forward_on_repeat": med["forward_on_repeat"] / med["log_likelihood"],
            "log_px_max_rel_diff": float(((ll - ref).abs() / ref.abs().clamp(min=1.0)).max()),
            "bits_per_dim": float(-ll.mean() / (3 * 32 * 32 * math.log(2.0))),
            "peak_mem_gb": torch.cuda.max_memory_allocated() / 2 ** 30,
            "extrapolated_s_test_set_1e4_samples": med["log_likelihood"] / 1e3 * (TEST_SET / B) * (1e4 / k)})
        out[name] = res
        del params, iaf, got
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
