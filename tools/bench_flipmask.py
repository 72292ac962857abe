"""Time the reversed-order (flipmask) IAF step against the unflipped Theano step on one GPU: the C1 shape (n_z 32, hidden
[64], 16x16, B = 256), inputs resident in HBM, CUDA events around K forward calls of each orientation, the two
orientations alternating over several rounds after a warm-up.  Prints one JSON line: per-round milliseconds per step of
each, the medians, and flipped / unflipped.  Both run the same kernels; the flipped step differs only in its flags (no
data reflection, the pad-channel table kept).
usage: python tools/bench_flipmask.py [steps] [rounds] [path]"""
import json
import os
import statistics
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from iaf_b200 import IAFOperator  # noqa: E402
from oracle import iaf_oracle as O  # noqa: E402  (synthetic parameter / input generator only)


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 200
    rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    path = sys.argv[3] if len(sys.argv) > 3 else "auto"
    n_z, hidden, H, W, B = 32, [64], 16, 16, 256
    hid, hd = O.make_params("theano", n_z, hidden, [n_z, n_z], seed=1)
    z, ctx = O.make_inputs(B, n_z, hidden[0], H, W, seed=0)
    dev = [tuple(torch.from_numpy(np.ascontiguousarray(l[k])).cuda() for k in "wsb") for l in hid + hd]
    ops = {name: IAFOperator("theano", n_z, hidden, [n_z, n_z], nl="elu", path=path, flipmask=flip).set_weights(dev)
           for name, flip in (("unflipped", False), ("flipped", True))}
    zg, cg = torch.from_numpy(z).cuda(), torch.from_numpy(ctx).cuda()
    for op in ops.values():
        for _ in range(20):
            op.step(zg, cg)
    torch.cuda.synchronize()
    ms = {name: [] for name in ops}
    for _ in range(rounds):
        for name, op in ops.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                op.step(zg, cg)
            e1.record()
            torch.cuda.synchronize()
            ms[name].append(e0.elapsed_time(e1) / steps)
    med = {name: statistics.median(v) for name, v in ms.items()}
    print(json.dumps({"shape": "C1 n_z=32 hidden=[64] 16x16", "B": B, "steps": steps, "rounds": rounds,
                      "path": {n: op.path_used(H, W, "cuda:0", "step") for n, op in ops.items()},
                      "gpu": torch.cuda.get_device_name(0), "ms_per_step": ms, "median_ms": med,
                      "flipped_over_unflipped": med["flipped"] / med["unflipped"]}))


if __name__ == "__main__":
    main()
