"""CPU-side checks: the C-ABI library loads and exports everything include/iaf_b200.h
declares, argument validation happens before any device work, host masks / factories
mirror the reference, the torch-CPU baseline port equals the oracle, and the sharded
ELBO reduction works over gloo with world_size 2."""
import ctypes as C
import os
import re
import sys

import numpy as np
import pytest
import torch

import __graft_entry__
from iaf_b200 import _lib, masks, multiconv2d, IAFOperator
from oracle import iaf_oracle as O
from oracle import iaf_oracle_torch as OT

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    __graft_entry__.build()
    return _lib.lib()


def test_library_exports_every_declared_symbol(lib):
    hdr = open(os.path.join(ROOT, "include", "iaf_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = set(re.findall(r"\b(iaf_[a-z_0-9]+)\s*\(", hdr))
    assert declared == set(_lib.SYMBOLS), declared ^ set(_lib.SYMBOLS)
    for name in declared:
        assert getattr(lib, name) is not None


def test_version_and_strerror(lib):
    assert lib.iaf_version() >= 100
    for st in range(0, -8, -1):
        assert lib.iaf_strerror(st) and b"unknown" not in lib.iaf_strerror(st)
    assert b"unknown" in lib.iaf_strerror(-99)


def test_capture_refusal_raises_capture_error(lib):
    """IAF_ERR_CAPTURED reaches python as CaptureError (a RuntimeError) telling the caller how to warm up."""
    with pytest.raises(_lib.CaptureError, match="largest batch size"):
        _lib.check(_lib.ERR_CAPTURED)
    assert issubclass(_lib.CaptureError, RuntimeError)


def _desc(**kw):
    d = _lib.IafDesc()
    d.variant, d.n_z, d.n_hidden, d.n_heads, d.H, d.W, d.nl, d.path = 0, 32, 1, 2, 16, 16, 1, 0
    d.hidden[0] = 64
    d.head[0] = d.head[1] = 32
    for k, v in kw.items():
        if isinstance(v, (list, tuple)):
            for i, x in enumerate(v):
                getattr(d, k)[i] = x
        else:
            setattr(d, k, v)
    return d


def test_plan_create_validates_before_touching_the_device(lib):
    h = C.c_void_p()
    assert lib.iaf_plan_create(None, None) == _lib.ERR_BAD_ARG
    assert lib.iaf_plan_create(C.byref(h), C.byref(_desc(n_z=0))) == _lib.ERR_BAD_ARG
    assert lib.iaf_plan_create(C.byref(h), C.byref(_desc(variant=7))) == _lib.ERR_BAD_ARG
    assert lib.iaf_plan_create(C.byref(h), C.byref(_desc(head=[32, 16]))) == _lib.ERR_BAD_SHAPE
    assert lib.iaf_plan_create(C.byref(h), C.byref(_desc(hidden=[48]))) == _lib.ERR_BAD_SHAPE  # 32 vs 48: ar.py:250
    assert lib.iaf_plan_create(C.byref(h), C.byref(_desc(n_hidden=9))) == _lib.ERR_UNSUPPORTED
    assert lib.iaf_plan_create(C.byref(h), C.byref(_desc(nl=17))) == _lib.ERR_UNSUPPORTED
    if not torch.cuda.is_available():
        assert lib.iaf_plan_create(C.byref(h), C.byref(_desc())) == _lib.ERR_NO_DEVICE
        assert not h.value
    lib.iaf_plan_destroy(None)  # harmless


def test_null_plan_entry_points(lib):
    assert lib.iaf_step_fwd(None, None, None, None, None, None, 1, None) == _lib.ERR_BAD_ARG
    assert lib.iaf_multiconv_fwd(None, None, None, None, 1, None) == _lib.ERR_BAD_ARG
    assert lib.iaf_pack_weights(None, None, None, None, None) == _lib.ERR_BAD_ARG
    assert lib.iaf_plan_launch_count(None) == 0


def test_host_masks_equal_oracle_masks():
    for n_in, n_out in [(4, 8), (8, 4), (32, 64), (64, 32), (160, 160), (4, 4)]:
        for zd in (False, True):
            assert np.array_equal(masks.tf_conv_ar_mask(n_in, n_out, zd), O.get_conv_ar_mask(3, 3, n_in, n_out, zd))
            assert np.array_equal(masks.theano_conv_ar_mask(n_in, n_out, (3, 3), zd),
                                  O.theano_conv_ar_mask(n_in, n_out, (3, 3), zd))


def test_multiconv2d_factory_creates_reference_parameters_and_postup():
    w = {}
    op = multiconv2d("1_0_posterior_conv1", 4, [8], [4, 4], (3, 3), False, nl="elu", w=w, device="cpu")
    assert sorted(w) == sorted("1_0_posterior_conv1_%s_%s" % (a, b) for a in ("0", "out_0", "out_1") for b in "wbs")
    assert tuple(w["1_0_posterior_conv1_0_w"].shape) == (8, 5, 3, 3)      # [Cout, Cin+1, 3, 3]  ar.py:288
    assert tuple(w["1_0_posterior_conv1_out_1_w"].shape) == (4, 9, 3, 3)
    m = O.theano_conv_ar_mask(4, 8, (3, 3), False)
    assert np.all(w["1_0_posterior_conv1_0_w"].numpy()[m == 0] == 0)        # created masked
    upd = {"1_0_posterior_conv1_0_w": torch.ones(8, 5, 3, 3)}
    upd = op.postup(upd, w)                                                  # ar.py:369-373
    assert np.array_equal(upd["1_0_posterior_conv1_0_w"].numpy(), m)
    with pytest.raises(NotImplementedError):
        multiconv2d("x", 4, [8], [4, 4], (5, 5), False, w={}, device="cpu")
    with pytest.raises(RuntimeError):  # CPU tensors: no CPU fallback
        op(torch.zeros(1, 4, 3, 3), torch.zeros(1, 8, 3, 3), w)


def test_operator_rejects_bad_arguments():
    with pytest.raises(ValueError):
        IAFOperator("caffe", 4, [8], [4, 4])
    with pytest.raises(NotImplementedError):
        IAFOperator("tf", 4, [8], [4, 4], nl="prelu")
    op = IAFOperator("tf", 4, [8], [4, 4])
    with pytest.raises(ValueError):
        op.set_weights([])
    with pytest.raises(RuntimeError):
        op.set_weights([(torch.zeros(3, 3, 4, 8), torch.zeros(8), torch.zeros(8))] * 3)  # CPU tensors


@pytest.mark.parametrize("variant,hidden,nl", [("tf", [8, 8], "elu"), ("theano", [8], "softplus"), ("theano", [], "elu")])
def test_torch_cpu_port_equals_oracle(variant, hidden, nl):
    hid, heads = O.make_params(variant, 4, hidden, [4, 4], seed=5)
    z, ctx = O.make_inputs(3, 4, hidden[0] if hidden else 4, 6, 5, seed=6)
    a = O.iaf_step(variant, z, ctx, hid, heads, nl)
    with torch.no_grad():
        b = OT.iaf_step(variant, torch.from_numpy(z), torch.from_numpy(ctx), OT.to_torch(hid), OT.to_torch(heads), nl)
    for x, y in zip(a, b):
        np.testing.assert_allclose(x, y.numpy(), rtol=1e-4, atol=2e-5)


def _gloo_worker(rank, world, port, q):
    import torch.distributed as dist
    from iaf_b200.parallel import shard_range, allreduce_scalars
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    lo, hi = shard_range(10, rank, world)
    logdet = torch.arange(10, dtype=torch.float32)[lo:hi]
    out = allreduce_scalars([logdet.sum(), torch.tensor(float(hi - lo))])
    q.put((rank, lo, hi, [float(v) for v in out]))
    dist.destroy_process_group()


def test_sharded_elbo_reduction_gloo_world2():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + os.getpid() % 2000
    ps = [ctx.Process(target=_gloo_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in ps:
        p.start()
    res = sorted(q.get(timeout=120) for _ in ps)
    for p in ps:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert [(r[1], r[2]) for r in res] == [(0, 5), (5, 10)]
    for r in res:
        assert r[3] == [45.0, 10.0]


def test_weight_containers_roundtrip(tmp_path):
    """The reference's Theano weight container (graphy/ndict.py:209-236) and the name maps of both front-ends."""
    from iaf_b200 import weights
    hid, heads = O.make_params("theano", 4, [8], [4, 4], seed=9)
    w = {}
    for i, l in enumerate(hid):
        for k in "wsb":
            w["0_1_posterior_conv1_%d_%s" % (i, k)] = l[k]
    for i, l in enumerate(heads):
        for k in "wsb":
            w["0_1_posterior_conv1_out_%d_%s" % (i, k)] = l[k]
    w["logsd_x"] = np.zeros((), np.float32)
    f = str(tmp_path / "weights.ndict.tar.gz")
    weights.np_savez(w, f)
    back = weights.np_loadz(f)
    assert sorted(back) == sorted(w) and all(np.array_equal(back[k], w[k]) for k in w)
    layers = weights.theano_layers(back, "0_1_posterior_conv1", 1, device="cpu")
    assert len(layers) == 3 and tuple(layers[0][0].shape) == (8, 5, 3, 3) and tuple(layers[2][1].shape) == (4,)
    assert np.array_equal(layers[1][0].numpy(), heads[0]["w"])
    hid, heads = O.make_params("tf", 4, [8, 8], [4, 4], seed=9)
    v = {}
    for n, l in zip(["layer_0", "layer_1", "layer_out_0", "layer_out_1"], hid + heads):
        for k in "Vgb":
            v["model/IAF_0_3/ar_multiconv2d/%s/%s" % (n, k)] = l[k]
    layers = weights.tf_layers(v, "model/IAF_0_3/ar_multiconv2d", device="cpu")
    assert len(layers) == 4 and tuple(layers[1][0].shape) == (3, 3, 8, 8)
    assert np.array_equal(layers[3][2].numpy(), heads[1]["b"])


def test_bench_reference_arm_line_schema():
    """`bench.py --impl reference` (the CPU port of the reference path) prints ONE JSON line with the contract's keys."""
    import json
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--workload", "c1_l2",
                          "--steps", "2", "--warmup", "1"], capture_output=True, text=True, timeout=600, cwd=root)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [l for l in out.stdout.splitlines() if l.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["higher_is_better"] is True and d["gpu_launches"] == 0
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "scaling", "dtype", "data", "config",
              "cpu_baseline", "e2e"):
        assert k in d, k
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1 and d["cpu_baseline"]["value"] == d["value"]
    assert d["e2e"] == {"value": d["value"], "unit": d["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert "theano-variant" in d["config"]["workload"]


def test_development_variants_still_compile_for_sm90a(tmp_path):
    """The flag-gated development variants (IAF_TC_TIMELINE: in-kernel timeline of the tensor-core stage kernel;
    BW_FASTDIV) must keep compiling for sm_90a next to the default build (nvcc cross-compiles without a GPU)."""
    import shutil
    import subprocess
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    csrc = os.path.join(ROOT, "iaf_b200", "csrc")
    base = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-std=c++17", "-c"]
    jobs = [(["-DIAF_TC_TIMELINE"], "iaf_tc.cu"), (["-DBW_FASTDIV"], "iaf_bwd.cu")]
    procs = [subprocess.Popen(base + flags + [src, "-o", str(tmp_path / (src + ".o"))], cwd=csrc, stdout=subprocess.PIPE,
                              stderr=subprocess.STDOUT, text=True) for flags, src in jobs]
    for (flags, src), pr in zip(jobs, procs):
        out, _ = pr.communicate(timeout=600)
        assert pr.returncode == 0, "%s %s:\n%s" % (src, flags, out[-2000:])
