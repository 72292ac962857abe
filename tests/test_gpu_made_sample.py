"""The inverse of the IAF step (``IAFOperator.step_inverse`` / ``ar_sample``, iaf_step_inverse) and the Theano decoder
with prior='made' on the H100: against the fp64 fixed point at small shapes and C1, by round trip at the benchmark
shapes (c2a, c2b; B = 256), determinism and batch independence, CUDA graphs and side streams, the shared-memory
envelope, and the decoder against its host-emulated run."""
import contextlib
import ctypes as C

import numpy as np
import pytest
import torch

from iaf_b200 import IAFOperator
from iaf_b200 import elbo_theano as ET
from oracle import iaf_oracle as O
from tests import made_sample_oracle as MS

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-4
VARIANTS = ("tf", "theano", "theano_flipmask")


def _np(t):
    return t.detach().double().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t, dtype=np.float64)


def per_sample_err(a, ref):
    a, ref = _np(a), _np(ref)
    assert np.isfinite(a).all()
    d = np.abs(a - ref).reshape(a.shape[0], -1).max(axis=1)
    r = np.maximum(np.abs(ref).reshape(a.shape[0], -1).max(axis=1), 1.0)
    return float((d / r).max())


class Case(object):
    def __init__(self, variant, n_z, hidden, H, W, nl="elu", path="auto", seed=1):
        self.variant, self.n_z, self.hidden, self.H, self.W, self.nl = variant, n_z, hidden, H, W, nl
        keys = "Vgb" if variant == "tf" else "wsb"
        self.hid, self.hd = O.make_params("tf" if variant == "tf" else "theano", n_z, hidden, [n_z, n_z], seed=seed)
        self.layers = [tuple(torch.from_numpy(l[k]).to(DEV) for k in keys) for l in self.hid + self.hd]
        self.op = IAFOperator("tf" if variant == "tf" else "theano", n_z, hidden, [n_z, n_z], nl=nl, path=path,
                              flipmask=variant == "theano_flipmask").set_weights(self.layers)

    def inputs(self, B, seed=0):
        u, ctx = O.make_inputs(B, self.n_z, self.hidden[0] if self.hidden else 1, self.H, self.W, seed=seed)
        return torch.from_numpy(u).to(DEV), (torch.from_numpy(ctx).to(DEV) if self.hidden else None)


SMALL = [
    # n_z, hidden, H, W, B, nl
    (4, [8], 4, 4, 2, "elu"),
    (8, [16, 16], 5, 7, 2, "softplus"),
    (4, [], 3, 6, 2, "elu"),
    (4, [8], 12, 9, 1, "relu"),
    (8, [4], 4, 5, 2, "tanh"),
    (32, [64], 16, 16, 4, "elu"),   # C1 level 0
    (32, [64], 8, 8, 4, "elu"),     # C1 level 1
    (32, [64], 4, 4, 4, "elu"),     # C1 level 2
]


def _small():
    for v in VARIANTS:
        for s in SMALL:
            if v == "tf" and not s[1]:
                continue
            yield (v,) + s


@pytest.mark.parametrize("variant,n_z,hidden,H,W,B,nl", list(_small()))
def test_inverse_matches_the_fp64_fixed_point(variant, n_z, hidden, H, W, B, nl):
    k = Case(variant, n_z, hidden, H, W, nl, path="simt")
    u, ctx = k.inputs(B)
    with torch.no_grad():
        z, ls, ld = k.op.step_inverse(u, ctx)
    zr, ar, ldr, iters = MS.inverse(variant, u.cpu().numpy(), None if ctx is None else ctx.cpu().numpy(), k.hid, k.hd, nl)
    assert iters <= n_z * H * W + 1
    assert per_sample_err(z, zr) < TOL and per_sample_err(ls, ar) < TOL
    assert per_sample_err(ld[:, None], ldr[:, None]) < TOL
    assert k.op.path_used(H, W, DEV, "step") == "simt"


FULL = [("c2a", [64]), ("c2b", [160, 160])]


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("shape,hidden", FULL)
def test_inverse_round_trips_at_the_benchmark_shapes(variant, shape, hidden):
    simt = Case(variant, 32, hidden, 16, 16, path="simt")
    u, ctx = simt.inputs(256)
    with torch.no_grad():
        z, ls, ld = simt.op.step_inverse(u, ctx)
        zs, lss, lds = simt.op.step(z, ctx)                         # step(inverse(u)) == u
        assert per_sample_err(zs, u) < TOL and per_sample_err(lss, ls) < TOL
        assert per_sample_err(lds[:, None], ld[:, None]) < TOL
        z2 = torch.randn(u.shape, generator=torch.Generator().manual_seed(3)).to(DEV)
        u2, _, _ = simt.op.step(z2, ctx)                           # inverse(step(z)) == z
        assert per_sample_err(simt.op.step_inverse(u2, ctx)[0], z2) < TOL
        # a tensor-core operator runs the same inverse kernel on its own (SIMT) pack: the step's tc-vs-simt agreement
        tc = Case(variant, 32, hidden, 16, 16, path="auto")
        assert tc.op.path_used(16, 16, DEV) == "tc"
        zt, lst, ldt = tc.op.step_inverse(u, ctx)
        assert per_sample_err(zt, z) < TOL and per_sample_err(lst, ls) < TOL


@pytest.mark.parametrize("variant", VARIANTS)
def test_inverse_is_deterministic_and_batch_independent(variant):
    k = Case(variant, 32, [64], 16, 16)
    u, ctx = k.inputs(64)
    with torch.no_grad():
        a = k.op.step_inverse(u, ctx)
        b = k.op.step_inverse(u, ctx)
        assert all(torch.equal(x, y) for x, y in zip(a, b))
        for lo, hi in ((0, 1), (5, 6), (17, 40)):
            s = k.op.step_inverse(u[lo:hi].contiguous(), ctx[lo:hi].contiguous())
            assert all(torch.equal(x, y[lo:hi]) for x, y in zip(s, a))
        none = k.op.step_inverse(u, ctx, want_logsd=False, want_logdet=False)
        assert torch.equal(none[0], a[0]) and none[1] is None and none[2] is None


def test_inverse_in_a_cuda_graph_and_on_a_side_stream():
    k = Case("theano", 32, [64], 16, 16)
    u, ctx = k.inputs(32)
    with torch.no_grad():
        ref = k.op.step_inverse(u, ctx)
        z, ls, ld = torch.empty_like(u), torch.empty_like(u), torch.empty((32,), device=DEV)
        launches = k.op.launch_count()
        g = torch.cuda.CUDAGraph()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            with torch.cuda.graph(g, stream=s):
                out = k.op.step_inverse(u, ctx)
                z.copy_(out[0]); ls.copy_(out[1]); ld.copy_(out[2])
        torch.cuda.current_stream().wait_stream(s)
        assert k.op.launch_count() == launches + 1     # one kernel, nothing allocated
        z.zero_(); ls.zero_(); ld.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(z, ref[0]) and torch.equal(ls, ref[1]) and torch.equal(ld, ref[2])
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            got = k.op.step_inverse(u, ctx)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        assert all(torch.equal(x, y) for x, y in zip(got, ref))


def test_inverse_refuses_the_first_window_that_does_not_fit():
    """Shared memory: per stage two rows of its input (W + 2 columns), the accumulators and the per-channel sums,
    4 bytes each, at most 225 KiB.  c2b's stack (n_z 32, hidden [160, 160]) fits up to W = 79."""
    def smem(W):
        return 4 * (2 * (W + 2) * (32 + 160 + 160) + (160 + 160 + 64) + 32)
    assert smem(79) <= 225 * 1024 < smem(80)
    for W, ok in ((79, True), (80, False)):
        k = Case("theano", 32, [160, 160], 2, W, path="auto")
        assert k.op.path_used(2, W, DEV) == "tc"     # (the SIMT step's band does not fit at these widths)
        u, ctx = k.inputs(2)
        with torch.no_grad():
            if ok:
                z = k.op.step_inverse(u, ctx)[0]
                assert per_sample_err(k.op.step(z, ctx)[0], u) < TOL
            else:
                with pytest.raises(NotImplementedError):
                    k.op.step_inverse(u, ctx)


@contextlib.contextmanager
def _emulated_abi(monkeypatch):
    from iaf_b200 import _lib as L
    from iaf_b200 import ops
    from tests.emu.inverse import emu

    def check_input(t, name, shape=None):
        assert isinstance(t, torch.Tensor) and t.dtype == torch.float32
        return t.contiguous()
    monkeypatch.setattr(L, "lib", emu)
    monkeypatch.setattr(ops, "_check_input", check_input)
    monkeypatch.setattr(ops, "_stream", lambda device: C.c_void_p(0))
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    yield


class _Recording(object):
    def __init__(self, inner):
        self.inner, self.samples = inner, {}

    def prior_sample(self, name, eps, context):
        z = self.inner.prior_sample(name, eps, context)
        self.samples[name] = z
        return z


@pytest.mark.parametrize("posterior", ET.POSTERIORS)
def test_made_decoder_on_the_gpu_matches_the_emulated_decoder(posterior, monkeypatch):
    hps = dict(n_z=4, n_h1=8, n_h2=8, depths=[1, 1], depth_ar=1, nl="elu", kl_min=0.0, image_size=8,
               posterior=posterior, prior="made")
    w = {k: torch.from_numpy(np.asarray(v)) for k, v in ET.make_params(hps, seed=5).items()}
    rng = np.random.RandomState(6)
    eps = {(i, 0): torch.from_numpy(rng.randn(2, 4, 8 // 2 ** (i + 1), 8 // 2 ** (i + 1)).astype(np.float32))
           for i in range(2)}
    gpu_layer = _Recording(ET.CudaIAF({k: v.to(DEV) for k, v in w.items()}, hps))
    got = ET.decode({k: v.to(DEV) for k, v in w.items()}, {k: v.to(DEV) for k, v in eps.items()}, gpu_layer, hps)
    with monkeypatch.context() as m:
        with _emulated_abi(m):
            emu_layer = _Recording(ET.CudaIAF(w, hps, path="simt"))
            ref = ET.decode(w, eps, emu_layer, hps)
    assert got.dtype == torch.uint8 and torch.equal(got.cpu(), ref)
    for name, z in emu_layer.samples.items():
        assert per_sample_err(gpu_layer.samples[name], z) < TOL, name
