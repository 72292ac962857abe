"""Time the fused Adamax step (``iaf_b200.optim.Adamax.step``: one ``iaf_adamax_kernel`` launch for the whole parameter
set) against the op-by-op torch restatement of the same rule (tests/adamax_oracle.py: about ten elementwise launches per
tensor), and a whole ``train_step`` of each restated model.

Workloads (synthetic weights from ``make_params``, seeded gradients and uint8 images):
* ``tf_default``: the TF model at tf_train.py's default hps (z_size 32, h_size 160, depth 2, num_blocks 2): 104 tensors,
  8.33 M fp32 elements, rule "tf";
* ``theano_c2a``: the Theano model at c2a's stack shape (the README's cifar10 model): n_z 32, n_h1 = n_h2 = 64,
  depth_ar 1, depths [2, 2, 2], rule "theano".
Optimiser step: CUDA events around ``--steps`` eager steps (host work included: each step reads every ``.grad``), the
two implementations alternating over ``--rounds`` rounds in one process, after a warm-up; the median per-step time of
each.  Then the fused step alone: captured into a CUDA graph and replayed, which times the kernel without the host.
Achieved bandwidth: 36 bytes per element (the kernel reads the parameter, gradient, both moments and the average and
writes all but the gradient) over the kernel's time, against the 3.35 TB/s of NVIDIA's data sheet for the H100 SXM.
The two implementations' results are compared bit for bit after the eager rounds (they start from the same state and
see the same gradients).
train_step: batch 16 (tf_train.py's per-GPU batch_size), CudaIAFTrain, the fused optimiser; CUDA events around each
step after two warm-up steps, median of ``--steps``.
Prints one JSON line with the card's name and power limit.
usage: python tools/bench_train.py [--steps K] [--rounds R]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from iaf_b200 import _lib  # noqa: E402
from iaf_b200 import elbo  # noqa: E402
from iaf_b200 import elbo_theano as ET  # noqa: E402
from iaf_b200.optim import Adamax  # noqa: E402
from tests.adamax_oracle import RestatedAdamax  # noqa: E402

BYTES_PER_ELEMENT = 36
HBM_PEAK = 3.35e12
WORKLOADS = {
    "tf_default": ("tf", dict(z_size=32, h_size=160, depth=2, num_blocks=2, kl_min=0.25, image_size=32)),
    "theano_c2a": ("theano", dict(n_z=32, n_h1=64, n_h2=64, depths=[2, 2, 2], depth_ar=1, nl="elu", kl_min=0.25,
                                  image_size=32)),
}


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # the timing does not depend on it
        return "unknown (%s)" % e


def params_of(rule, hps, dev):
    mp = elbo.make_params if rule == "tf" else ET.make_params
    return {k: torch.tensor(np.asarray(v), device=dev).requires_grad_() for k, v in mp(hps, seed=0).items()}


def timed(fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1e-3 / n


def bench_step(rule, hps, dev, steps, rounds):
    p = params_of(rule, hps, dev)
    q = {k: v.detach().clone().requires_grad_() for k, v in p.items()}
    gen = torch.Generator(device=dev).manual_seed(0)
    for k in p:
        p[k].grad = torch.randn(p[k].shape, generator=gen, device=dev)
        q[k].grad = p[k].grad.clone()
    fused, ref = Adamax(p, rule), RestatedAdamax(q, rule)
    numel = sum(t.numel() for t in p.values())
    before = _lib.lib().iaf_adamax_launch_count()
    fused.step()
    launches = _lib.lib().iaf_adamax_launch_count() - before
    ref.step()
    t_fused, t_ref = [], []
    for _ in range(rounds):
        t_fused.append(timed(fused.step, steps))
        t_ref.append(timed(ref.step, steps))
    torch.cuda.synchronize()
    same = all(torch.equal(p[k], q[k]) for k in p) and all(
        torch.equal(a, b) for a, b in zip(fused.averaged().values(), ref.averaged().values()))
    # the kernel alone: the fused step captured into a CUDA graph, ``steps`` replays per timing
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fused.step()
    graph.replay()
    t_kernel = [timed(graph.replay, steps) for _ in range(rounds)]
    tf, tr, tk = statistics.median(t_fused), statistics.median(t_ref), statistics.median(t_kernel)
    return dict(tensors=len(p), elements=numel, launches_per_step=launches, fused_step_us=tf * 1e6,
                restated_step_us=tr * 1e6, speedup=tr / tf, fused_step_us_rounds=[t * 1e6 for t in t_fused],
                fused_kernel_us=tk * 1e6, kernel_bytes_per_s=BYTES_PER_ELEMENT * numel / tk,
                kernel_share_of_hbm_peak=BYTES_PER_ELEMENT * numel / tk / HBM_PEAK, bit_identical=same)


def bench_train_step(rule, hps, dev, steps):
    p = params_of(rule, hps, dev)
    opt = Adamax(p, rule)
    mod = elbo if rule == "tf" else ET
    layer = elbo.CudaIAFTrain(p, hps) if rule == "tf" else ET.CudaIAFTrain(p, hps)
    rng = np.random.RandomState(1)
    x = torch.from_numpy(rng.randint(0, 256, size=(16, 3, 32, 32)).astype(np.uint8)).to(dev)
    times, bpd = [], []
    for i in range(steps + 2):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = mod.train_step(p, x, opt, hps, iaf_layer=layer)
        b.record()
        b.synchronize()
        bpd.append(float(out))
        if i >= 2:
            times.append(a.elapsed_time(b) * 1e-3)
    return dict(batch=16, train_step_ms=statistics.median(times) * 1e3, bits_per_dim_first_last=[bpd[0], bpd[-1]])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=7)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train needs a CUDA device")
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    res = {"card": card()}
    for name, (rule, hps) in WORKLOADS.items():
        r = bench_step(rule, hps, dev, a.steps, a.rounds)
        r.update(bench_train_step(rule, hps, dev, min(a.steps, 20)))
        res[name] = r
    print(json.dumps(res))


if __name__ == "__main__":
    main()
