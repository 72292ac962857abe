"""Two-GPU NCCL test of the batch-sharded ELBO (BASELINE config C5 structure; tf_train.py:126-142): every rank evaluates
its slice with the CUDA operator, ONE all-reduce of the scalar gives the global bits/dim, which must equal the
single-process evaluation of the whole batch with the same rank-local free-bits rule.  Skips with fewer than two GPUs (the
gloo world-2 twin in tests/test_elbo.py covers the host logic on CPU)."""
import os
import socket

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _worker(rank, world, port, q):
    import torch.distributed as dist
    from iaf_b200 import elbo
    from tests.test_elbo import _setup
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(rank)
    # the spawned worker does not inherit conftest's fixture: the torch plumbing convolutions must run in fp32 here too
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    hps = dict(z_size=32, h_size=160, depth=1, num_blocks=3, kl_min=0.1, image_size=32)
    dev = "cuda:%d" % rank
    p, x, n = _setup(hps, 8, 7, torch.float32, dev)
    with torch.no_grad():
        bpd = elbo.sharded_bits_per_dim(p, x, n, elbo.CudaIAF(p, hps), hps)
    q.put((rank, float(bpd)))
    dist.destroy_process_group()


def test_sharded_bits_per_dim_nccl_world2():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import torch.multiprocessing as mp
    from iaf_b200 import elbo
    from tests.test_elbo import _setup
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for pr in procs:
        pr.start()
    got = dict(q.get(timeout=300) for _ in procs)
    for pr in procs:
        pr.join(timeout=60)
    assert abs(got[0] - got[1]) < 1e-7, got
    # single process: the two shards evaluated one after the other with the tower-local free-bits mean (tf_train.py:79)
    hps = dict(z_size=32, h_size=160, depth=1, num_blocks=3, kl_min=0.1, image_size=32)
    p, x, n = _setup(hps, 8, 7, torch.float32, "cuda:0")
    with torch.no_grad():
        tot = 0.0
        for lo, hi in ((0, 4), (4, 8)):
            out = elbo.forward(p, x[lo:hi], {k: v[lo:hi] for k, v in n.items()}, elbo.CudaIAF(p, hps), hps)
            tot += float(out["bits_per_dim"]) * (hi - lo)
    assert abs(got[0] - tot / 8) <= 5e-6 * max(abs(tot / 8), 1.0), (got, tot / 8)
