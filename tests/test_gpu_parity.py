"""GPU parity tests (H100): the CUDA path, called through the C ABI, against
 (1) the fixtures produced by executing the reference's own source (tests/golden),
 (2) the fp64 oracle on seeded inputs,
 (3) size-independent properties at BASELINE.json's full size (B=256).
Tolerance (north_star): ||delta||_inf / max(||ref||_inf, 1) <= 1e-4 for z' and logdet."""
import os

import numpy as np
import pytest
import torch

from oracle import iaf_oracle as O
from tests.golden.cases import MULTICONV_CASES, case_inputs

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")
TOL = 1e-4


def relerr(a, ref):
    a = a.detach().cpu().numpy().astype(np.float64) if isinstance(a, torch.Tensor) else a
    return float(np.abs(a - ref).max() / max(np.abs(ref).max(), 1.0))


def dev_layers(variant, hid, heads, dev="cuda"):
    keys = ("V", "g", "b") if variant == "tf" else ("w", "s", "b")
    return [tuple(torch.from_numpy(np.ascontiguousarray(l[k])).to(dev) for k in keys) for l in hid + heads]


def make_op(variant, n_z, hidden, nl, path, hid, heads, n_out=None):
    from iaf_b200 import IAFOperator
    op = IAFOperator(variant, n_z, hidden, n_out or [n_z, n_z], nl=nl, path=path)
    return op.set_weights(dev_layers(variant, hid, heads))


def paths_for(variant, n_z, hidden, H, W):
    """simt always; tc where the plan accepts it."""
    from iaf_b200 import IAFOperator
    out = ["simt"]
    try:
        op = IAFOperator(variant, n_z, hidden, [n_z, n_z], path="tc")
        hid, heads = O.make_params(variant, n_z, hidden, [n_z, n_z], seed=0)
        op.set_weights(dev_layers(variant, hid, heads))
        op.path_used(H, W, "cuda:0")
        out.append("tc")
    except NotImplementedError:
        pass
    return out


# ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("ci", range(len(MULTICONV_CASES)))
def test_multiconv_against_reference_fixtures(ci):
    """iaf_multiconv_fwd == what the reference's ar_multiconv2d / multiconv2d source produced."""
    name, variant, B, n_z, hidden, H, W, nl = MULTICONV_CASES[ci]
    g = np.load(os.path.join(G, "multiconv.npz"))
    hid, heads, z, ctx = case_inputs(variant, B, n_z, hidden, H, W, seed=ci)
    for path in (paths_for(variant, n_z, hidden, H, W) if hidden else ["simt"]):
        op = make_op(variant, n_z, hidden, nl, path, hid, heads)
        m, s = op.multiconv(torch.from_numpy(z).cuda(), torch.from_numpy(ctx).cuda())
        assert relerr(m, g[name + "_m"]) < 2e-5, path
        assert relerr(s, g[name + "_s"]) < 2e-5, path


STEP_CASES = [
    # variant, B, n_z, hidden, H, W, nl
    ("tf", 8, 32, [64], 16, 16, "elu"),           # C2a shape
    ("tf", 3, 32, [160, 160], 16, 16, "elu"),     # C2b / C3 shape
    ("theano", 4, 32, [64], 16, 16, "elu"),       # C1 level 0
    ("theano", 4, 32, [64], 8, 8, "elu"),         # C1 level 1
    ("theano", 4, 32, [64], 4, 4, "elu"),         # C1 level 2
    ("theano", 2, 32, [160, 160], 16, 16, "elu"), # C4
    ("theano", 2, 32, [160, 160], 8, 8, "softplus"),
    ("tf", 5, 4, [8, 8], 7, 5, "elu"),            # ragged, non-square, odd sizes
    ("theano", 3, 4, [8], 1, 1, "elu"),           # 1x1 feature map
    ("tf", 1, 4, [8], 3, 19, "relu"),             # wider than two x-segments
    ("theano", 2, 4, [], 5, 5, "elu"),            # depth_ar = 0: context unused (F8)
    ("tf", 2, 6, [12], 6, 6, "tanh"),             # channels not a multiple of 4/8
    ("tf", 2, 8, [4], 6, 6, "elu"),               # n_out < n_in in the hidden layer
    ("tf", 3, 16, [32], 16, 16, "elu"),           # one-launch tensor-core step, 32 columns: padded column groups
    ("theano", 2, 16, [48, 48], 8, 8, "elu"),     # per-stage tensor-core kernels, 48 columns: padded column groups
]


@pytest.mark.parametrize("case", STEP_CASES, ids=lambda c: "%s-%s-%dx%d" % (c[0], "x".join(map(str, c[3])) or "0", c[4], c[5]))
def test_step_against_fp64_oracle(case):
    variant, B, n_z, hidden, H, W, nl = case
    hid, heads = O.make_params(variant, n_z, hidden, [n_z, n_z], seed=21)
    z, ctx = O.make_inputs(B, n_z, hidden[0] if hidden else n_z, H, W, seed=22)
    f64 = lambda ls: O.cast_params(ls, np.float64)
    z_ref, logsd_ref, logdet_ref = O.iaf_step(variant, z.astype(np.float64), ctx.astype(np.float64), f64(hid), f64(heads), nl)
    for path in paths_for(variant, n_z, hidden, H, W):
        op = make_op(variant, n_z, hidden, nl, path, hid, heads)
        z1, logsd, logdet = op.step(torch.from_numpy(z).cuda(), torch.from_numpy(ctx).cuda() if hidden else None)
        assert relerr(z1, z_ref) < TOL, path
        assert relerr(logsd, logsd_ref) < TOL, path
        assert relerr(logdet, logdet_ref) < TOL, path
        # the un-fused entry feeds the same numbers
        m, s = op.multiconv(torch.from_numpy(z).cuda(), torch.from_numpy(ctx).cuda() if hidden else None)
        assert relerr(0.1 * s, logsd_ref) < TOL


def test_optional_outputs_may_be_null():
    variant, n_z, hidden, H, W = "tf", 4, [8], 5, 5
    hid, heads = O.make_params(variant, n_z, hidden, [n_z, n_z], seed=1)
    z, ctx = O.make_inputs(2, n_z, hidden[0], H, W, seed=2)
    op = make_op(variant, n_z, hidden, "elu", "simt", hid, heads)
    a = op.step(torch.from_numpy(z).cuda(), torch.from_numpy(ctx).cuda())
    b = op.step(torch.from_numpy(z).cuda(), torch.from_numpy(ctx).cuda(), want_logsd=False, want_logdet=False)
    assert b[1] is None and b[2] is None
    assert torch.equal(a[0], b[0])


def test_single_head_multiconv():
    """down_iaf1_nl style stack: one head (ar.py:411 returns the bare tensor)."""
    from iaf_b200 import multiconv2d
    n_z, hidden, H, W = 4, [8], 6, 6
    hid, heads = O.make_params("theano", n_z, hidden, [n_z], seed=3)
    z, ctx = O.make_inputs(2, n_z, hidden[0], H, W, seed=4)
    w = {}
    for i, l in enumerate(hid):
        for k in "wsb":
            w["p_%d_%s" % (i, k)] = torch.from_numpy(l[k]).cuda()
    for k in "wsb":
        w["p_out_0_" + k] = torch.from_numpy(heads[0][k]).cuda()
    op = multiconv2d("p", n_z, hidden, n_z, (3, 3), False, nl="elu", w=w, path="simt")
    out = op(torch.from_numpy(z).cuda(), torch.from_numpy(ctx).cuda(), w)
    assert isinstance(out, torch.Tensor)
    f64 = lambda ls: O.cast_params(ls, np.float64)
    ref = O.theano_multiconv2d(z.astype(np.float64), ctx.astype(np.float64), f64(hid), f64(heads), "elu")[0]
    assert relerr(out, ref) < 2e-5


def test_tf_style_entry_point_with_tf_variable_names():
    from iaf_b200 import ar_multiconv2d
    n_z, hs, H, W = 4, 8, 6, 6
    hid, heads = O.make_params("tf", n_z, [hs, hs], [n_z, n_z], seed=77)
    z, ctx = O.make_inputs(4, n_z, hs, H, W, seed=5)
    params = {}
    for i, l in enumerate(hid):
        for k in "Vgb":
            params["ar_multiconv2d/layer_%d/%s" % (i, k)] = torch.from_numpy(l[k]).cuda()
    for i, l in enumerate(heads):
        for k in "Vgb":
            params["ar_multiconv2d/layer_out_%d/%s" % (i, k)] = torch.from_numpy(l[k]).cuda()
    x = ar_multiconv2d("ar_multiconv2d", torch.from_numpy(z).cuda(), torch.from_numpy(ctx).cuda(), [hs, hs], [n_z, n_z],
                       params=params, path="simt")
    f64 = lambda ls: O.cast_params(ls, np.float64)
    m, s = O.tf_ar_multiconv2d(z.astype(np.float64), ctx.astype(np.float64), f64(hid), f64(heads))
    assert relerr(x[0], m) < 2e-5 and relerr(x[1], s) < 2e-5
    # weights are re-packed when a parameter changes in place (graph-builder vs eager, F9)
    params["ar_multiconv2d/layer_out_1/b"].add_(1.0)
    x2 = ar_multiconv2d("ar_multiconv2d", torch.from_numpy(z).cuda(), torch.from_numpy(ctx).cuda(), [hs, hs], [n_z, n_z],
                        params=params, path="simt")
    assert relerr(x2[1], s + 1.0) < 2e-5


@pytest.mark.parametrize("name", ["kl0", "kl01", "kl5"])
def test_fused_layer_against_iaflayer_down_fixture(name):
    """iaf_layer_fwd vs the tensors IAFLayer.down (tf_train.py:46-95, executed from the reference
    source) produced: z', kl_cost and -- through the rank-local free-bits rule -- kl_obj."""
    g = np.load(os.path.join(G, "iaflayer_down.npz"))
    v = lambda k: g[name + "_" + k]
    hid, heads = O.make_params("tf", 4, [8, 8], [4, 4], seed=77)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a.astype(np.float32))).cuda()
    context = v("up_context") + v("down_context")
    for path in paths_for("tf", 4, [8, 8], 6, 6):
        op = make_op("tf", 4, [8, 8], "elu", path, hid, heads)
        z1, kl, kl_bc, kl_cost = op.layer(t(v("eps")), t(v("rz_mean") + v("qz_mean")), t(v("rz_logsd") + v("qz_logsd")),
                                          t(v("pz_mean")), t(v("pz_logsd")), t(context))
        z_ref = (v("z0") - 0.1 * v("m")) / np.exp(0.1 * v("s"))
        assert relerr(z1, z_ref) < TOL
        assert relerr(kl_cost, v("kl_cost")) < TOL
        assert relerr(kl.sum(dim=(2, 3)), kl_bc.cpu().numpy().astype(np.float64)) < 1e-5
        kl_min = float(v("kl_min"))
        if kl_min > 0:   # tf_train.py:77-83
            kl_obj = torch.clamp(kl_bc.mean(dim=0, keepdim=True), min=kl_min).expand(kl_bc.shape[0], -1).sum(dim=1)
        else:
            kl_obj = kl_cost
        assert relerr(kl_obj, v("kl_obj")) < TOL


def test_error_behaviour_on_device():
    from iaf_b200 import IAFOperator
    hid, heads = O.make_params("tf", 4, [8], [4, 4], seed=1)
    op = make_op("tf", 4, [8], "elu", "simt", hid, heads)
    z = torch.zeros(2, 4, 5, 5, device="cuda")
    with pytest.raises(ValueError):
        op.step(z, torch.zeros(2, 7, 5, 5, device="cuda"))          # wrong context channels
    with pytest.raises(ValueError):
        op.step(torch.zeros(2, 5, 5, 5, device="cuda"), torch.zeros(2, 8, 5, 5, device="cuda"))
    with pytest.raises(TypeError):
        op.step(z.double(), torch.zeros(2, 8, 5, 5, device="cuda"))
    with pytest.raises(RuntimeError):
        op.step(z.cpu(), torch.zeros(2, 8, 5, 5))                    # no CPU fallback
    with pytest.raises(ValueError):                                   # 32 -> 48: ar.py:250 assert
        IAFOperator("tf", 32, [48], [32, 32]).set_weights(dev_layers("tf", *O.make_params("tf", 32, [48], [32, 32])))\
            .step(torch.zeros(1, 32, 4, 4, device="cuda"), torch.zeros(1, 48, 4, 4, device="cuda"))
    op1 = make_op("tf", 4, [8], "elu", "simt", *O.make_params("tf", 4, [8], [4], seed=1), n_out=[4])
    with pytest.raises(ValueError):                                   # the fused step needs two heads of n_z
        op1.step(z, torch.zeros(2, 8, 5, 5, device="cuda"))


# ---------------------------------------------------------------------------------------
# full-size properties (B = 256, n_z = 32, 16x16): BASELINE configs C2a / C2b
# ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("hidden", [[64], [160, 160]], ids=["c2a", "c2b"])
def test_full_size_properties(hidden):
    variant, B, n_z, H, W = "tf", 256, 32, 16, 16
    hid, heads = O.make_params(variant, n_z, hidden, [n_z, n_z], seed=1)
    z, ctx = O.make_inputs(B, n_z, hidden[0], H, W, seed=0)
    zc, cc = torch.from_numpy(z).cuda(), torch.from_numpy(ctx).cuda()
    f64 = lambda ls: O.cast_params(ls, np.float64)
    for path in paths_for(variant, n_z, hidden, H, W):
        op = make_op(variant, n_z, hidden, "elu", path, hid, heads)
        z1, logsd, logdet = op.step(zc, cc)
        # (a) checksum of checksums: per-sample logdet is minus the sum of the per-element terms
        assert relerr(logdet, -logsd.double().sum(dim=(1, 2, 3)).cpu().numpy()) < 1e-5
        # (b) samples are independent: any sub-batch gives bit-identical z' rows (the per-sample logdet is a
        #     fixed-order fp32 sum whose grouping follows the tile grid, so it may differ in the last bits
        #     when the sample sits at another batch position); run to run everything is deterministic
        z1b, logsdb, logdetb = op.step(zc[37:41].contiguous(), cc[37:41].contiguous())
        assert torch.equal(z1b, z1[37:41]) and torch.equal(logsdb, logsd[37:41])
        assert relerr(logdetb, logdet[37:41].double().cpu().numpy()) < 1e-6
        z1c, _, logdetc = op.step(zc, cc)
        assert torch.equal(z1c, z1) and torch.equal(logdetc, logdet)
        # (c) autoregressive: perturbing z at pixel (y0,x0) leaves every output at a LATER position of the
        #     TF variant's reverse-raster order (smaller raster index) untouched... and earlier ones too
        #     except through s,m of positions that can see it: outputs at positions > p0 in raster
        #     order (which the mask lets see nothing before them) are bit-identical.
        y0, x0 = 7, 9
        zp = zc.clone()
        zp[:, :, y0, x0] += 0.5
        z1p, _, _ = op.step(zp, cc)
        p0 = y0 * W + x0
        flat, flatp = z1.reshape(B, n_z, -1), z1p.reshape(B, n_z, -1)
        assert torch.equal(flat[:, :, p0 + 1:], flatp[:, :, p0 + 1:])
        assert not torch.equal(flat[:, :, :p0], flatp[:, :, :p0])
        # (d) invertibility of the affine map given (m, s): z = z' * exp(arw_logsd) + 0.1 m
        m, s = op.multiconv(zc, cc)
        assert relerr(z1 * torch.exp(logsd) + 0.1 * m, z.astype(np.float64)) < 1e-5
        # (e) spot-check a slice against the fp64 oracle at full batch position
        sl = slice(250, 252)
        z_ref, logsd_ref, logdet_ref = O.iaf_step(variant, z[sl].astype(np.float64), ctx[sl].astype(np.float64),
                                                  f64(hid), f64(heads))
        assert relerr(z1[sl], z_ref) < TOL and relerr(logdet[sl], logdet_ref) < TOL


def test_step_host_entry_matches_device_entry():
    variant, B, n_z, hidden, H, W = "tf", 16, 32, [64], 16, 16
    hid, heads = O.make_params(variant, n_z, hidden, [n_z, n_z], seed=1)
    z, ctx = O.make_inputs(B, n_z, hidden[0], H, W, seed=0)
    op = make_op(variant, n_z, hidden, "elu", "auto", hid, heads)
    a = op.step(torch.from_numpy(z).cuda(), torch.from_numpy(ctx).cuda())
    hz, hc = torch.from_numpy(z).pin_memory(), torch.from_numpy(ctx).pin_memory()
    ho, hl, hd = torch.empty_like(hz).pin_memory(), torch.empty_like(hz).pin_memory(), torch.empty(B).pin_memory()
    op.step_host(hz, hc, ho, hl, hd)
    assert torch.equal(ho, a[0].cpu()) and torch.equal(hl, a[1].cpu()) and torch.equal(hd, a[2].cpu())
    # pageable buffers work too
    ho2 = torch.empty(B, n_z, H, W)
    op.step_host(torch.from_numpy(z), torch.from_numpy(ctx), ho2, None, None)
    assert torch.equal(ho2, ho)
    # pipelined submission: 7 batches through 3 staging slots, every result equals the device entry
    outs = []
    for i in range(7):
        zi = (torch.from_numpy(z) + 0.01 * i).pin_memory()
        o = [torch.empty_like(hz).pin_memory(), torch.empty_like(hz).pin_memory(), torch.empty(B).pin_memory()]
        op.submit_host(zi, hc, o[0], o[1], o[2])
        outs.append((zi, o))
    op.wait_host()
    for zi, o in outs:
        ref = op.step(zi.cuda(), torch.from_numpy(ctx).cuda())
        assert torch.equal(o[0], ref[0].cpu()) and torch.equal(o[1], ref[1].cpu()) and torch.equal(o[2], ref[2].cpu())


@pytest.mark.parametrize("variant,B,hidden,H,W", [
    ("tf", 300, [64], 16, 16),         # 678 tiles over 132 CTAs: runs of 5 and 6 tiles
    ("theano", 97, [64], 16, 16),      # odd batch, point-reflected orientation, pad channel
    ("theano", 515, [64], 4, 4),       # 5+ samples per 128-slot tile
    ("tf", 37, [160, 160], 16, 16),    # layer-at-a-time kernels, fewer tiles than SMs
    ("theano", 150, [160, 160], 8, 8), # layered, several samples per tile
])
def test_tensor_core_paths_agree_with_fp32_path_at_odd_batches(variant, B, hidden, H, W):
    """Cross-check of the two independent CUDA implementations (exact-fp32 SIMT vs wgmma) on batch sizes that
    exercise uneven tile runs, partial last tiles and tiles spanning many samples."""
    n_z = 32
    hid, heads = O.make_params(variant, n_z, hidden, [n_z, n_z], seed=5)
    z, ctx = O.make_inputs(B, n_z, hidden[0], H, W, seed=6)
    zc, cc = torch.from_numpy(z).cuda(), torch.from_numpy(ctx).cuda()
    a = make_op(variant, n_z, hidden, "elu", "simt", hid, heads).step(zc, cc)
    b = make_op(variant, n_z, hidden, "elu", "tc", hid, heads).step(zc, cc)
    for x, y in zip(a, b):
        assert relerr(y, x.double().cpu().numpy()) < 5e-5


def test_full_size_properties_theano_c1():
    """C1 (Theano numerics, hidden [64]) at B=256: determinism, AR direction (raster order: a perturbation only
    reaches LATER raster positions), logdet consistency."""
    variant, B, n_z, hidden, H, W = "theano", 256, 32, [64], 16, 16
    hid, heads = O.make_params(variant, n_z, hidden, [n_z, n_z], seed=1)
    z, ctx = O.make_inputs(B, n_z, hidden[0], H, W, seed=0)
    zc, cc = torch.from_numpy(z).cuda(), torch.from_numpy(ctx).cuda()
    for path in paths_for(variant, n_z, hidden, H, W):
        op = make_op(variant, n_z, hidden, "elu", path, hid, heads)
        z1, logsd, logdet = op.step(zc, cc)
        assert relerr(logdet, -logsd.double().sum(dim=(1, 2, 3)).cpu().numpy()) < 1e-5
        z1c, _, logdetc = op.step(zc, cc)
        assert torch.equal(z1c, z1) and torch.equal(logdetc, logdet)
        y0, x0 = 7, 9
        zp = zc.clone()
        zp[:, :, y0, x0] += 0.5
        z1p, _, _ = op.step(zp, cc)
        p0 = y0 * W + x0
        flat, flatp = z1.reshape(B, n_z, -1), z1p.reshape(B, n_z, -1)
        assert torch.equal(flat[:, :, :p0], flatp[:, :, :p0])            # earlier raster positions untouched
        assert not torch.equal(flat[:, :, p0 + 1:], flatp[:, :, p0 + 1:])
