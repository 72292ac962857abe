"""Time the fused Eve step (``iaf_b200.optim.Eve.step``: one ``iaf_eve_kernel`` launch for the whole parameter set)
against the op-by-op torch restatement of the same rule (tests/eve_oracle.py: about a dozen elementwise launches per
tensor), and a whole Eve ``train_step`` of the Theano model.  The method is tools/bench_train.py's.

Workload: the Theano model at c2a's stack shape (the README's cifar10 model: n_z 32, n_h1 = n_h2 = 64, depth_ar 1,
depths [2, 2, 2]): 134 tensors, 2.84 M fp32 elements, synthetic weights from ``make_params`` and seeded gradients.
Optimiser step: CUDA events around ``--steps`` eager steps (host work included: each step reads every ``.grad``), the
two implementations alternating over ``--rounds`` rounds in one process, after a warm-up; the median per-step time of
each.  Then the fused step alone: captured into a CUDA graph and replayed, which times the kernel without the host.
Achieved bandwidth: 44 bytes per element (the kernel reads the parameter, gradient, both moments and the average, and
writes all but the gradient plus delta and the lookahead; it does not read the previous delta) over the kernel's time,
against the 3.35 TB/s of NVIDIA's data sheet for the H100 SXM.  The two implementations' results (parameters, averages
and lookahead) are compared bit for bit after the eager rounds (they start from the same state and see the same
gradients).
train_step: batch 16, CudaIAFTrain on the lookahead, the fused Eve; CUDA events around each step after two warm-up
steps, median of ``--steps`` (at most 20).
Prints one JSON line with the card's name and power limit.
usage: python tools/bench_eve.py [--steps K] [--rounds R]"""
import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from iaf_b200 import _lib  # noqa: E402
from iaf_b200 import elbo_theano as ET  # noqa: E402
from iaf_b200.optim import Eve  # noqa: E402
from tests.eve_oracle import RestatedEve  # noqa: E402
from tools.bench_train import HBM_PEAK, card, timed  # noqa: E402

BYTES_PER_ELEMENT = 44
HPS = dict(n_z=32, n_h1=64, n_h2=64, depths=[2, 2, 2], depth_ar=1, nl="elu", kl_min=0.25, image_size=32)


def params_of(dev):
    return {k: torch.tensor(np.asarray(v), device=dev) for k, v in ET.make_params(HPS, seed=0).items()}


def same(fused, ref, p, q):
    return (all(torch.equal(p[k], q[k]) for k in p) and
            all(torch.equal(a, b) for a, b in zip(fused.averaged().values(), ref.averaged().values())) and
            all(torch.equal(a, b) for a, b in zip(fused.lookahead().values(), ref.lookahead().values())))


def bench_step(dev, steps, rounds):
    p = params_of(dev)
    q = {k: v.clone() for k, v in p.items()}
    fused, ref = Eve(p), RestatedEve(q)
    gen = torch.Generator(device=dev).manual_seed(0)
    rla = ref.lookahead()
    for k, t in fused.lookahead().items():
        t.grad = torch.randn(t.shape, generator=gen, device=dev)
        rla[k].grad = t.grad.clone()
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
    same_eager = same(fused, ref, p, q)
    # the kernel alone: the fused step captured into a CUDA graph, ``steps`` replays per timing
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fused.step()
    graph.replay()
    t_kernel = [timed(graph.replay, steps) for _ in range(rounds)]
    tf, tr, tk = (statistics.median(t) for t in (t_fused, t_ref, t_kernel))
    return dict(tensors=len(p), elements=numel, launches_per_step=launches, fused_step_us=tf * 1e6,
                restated_step_us=tr * 1e6, speedup=tr / tf, fused_step_us_rounds=[t * 1e6 for t in t_fused],
                fused_kernel_us=tk * 1e6, fused_kernel_us_rounds=[t * 1e6 for t in t_kernel],
                kernel_bytes_per_s=BYTES_PER_ELEMENT * numel / tk,
                kernel_share_of_hbm_peak=BYTES_PER_ELEMENT * numel / tk / HBM_PEAK,
                bit_identical=same_eager)


def bench_train_step(dev, steps):
    p = params_of(dev)
    opt = Eve(p)
    layer = ET.CudaIAFTrain(opt.lookahead(), HPS)
    rng = np.random.RandomState(1)
    x = torch.from_numpy(rng.randint(0, 256, size=(16, 3, 32, 32)).astype(np.uint8)).to(dev)
    times, bpd = [], []
    for i in range(steps + 2):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = ET.train_step(p, x, opt, HPS, iaf_layer=layer)
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
        raise SystemExit("bench_eve needs a CUDA device")
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    r = bench_step(dev, a.steps, a.rounds)
    r.update(bench_train_step(dev, min(a.steps, 20)))
    print(json.dumps({"card": card(), "theano_c2a_eve": r}))


if __name__ == "__main__":
    main()
