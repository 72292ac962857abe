"""GPU parity, the thin spots VERDICT round 1 listed:
 * EVERY sample of the full-size headline workloads (B = 256: C2a hidden [64], C2b hidden [160,160]) against the fp64
   oracle (z', per-element arw_logsd, per-sample logdet), not a two-sample spot check;
 * the operator's robustness items (plans created large-to-small keep working, parameters updated through ``.data``,
   per-entry path report, imported weights drive the operator);
 * full-depth bits/dim: C3 (tf_train.py defaults: num_blocks=20, depth=1, h=160, B=32) and C4 (README 3.28-bpd config:
   n_h=160, depths [10,10], depth_ar=2) once each against the fp64 oracle ELBO.
Tolerance (north_star): ||delta||_inf / max(||ref||_inf, 1) <= 1e-4."""
import os

import numpy as np
import pytest
import torch

from oracle import iaf_oracle as O
from oracle import iaf_oracle_torch as OT
from tests.test_gpu_parity import TOL, dev_layers, make_op, relerr

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("variant,hidden", [("tf", [64]), ("tf", [160, 160]), ("theano", [64])],
                         ids=["c2a", "c2b", "c1-theano"])
def test_every_sample_of_the_full_batch_against_fp64_oracle(variant, hidden):
    """All 256 samples.  The fp64 reference is the torch-CPU restatement (oracle/iaf_oracle_torch.py, pinned to the numpy
    oracle and through it to the reference-executed fixtures by tests/test_oracle_golden.py)."""
    B, n_z, H, W = 256, 32, 16, 16
    hid, heads = O.make_params(variant, n_z, hidden, [n_z, n_z], seed=1)
    z, ctx = O.make_inputs(B, n_z, hidden[0], H, W, seed=0)
    t64 = lambda ls: OT.to_torch(ls, torch.float64)
    with torch.no_grad():
        z_ref, logsd_ref, logdet_ref = OT.iaf_step(variant, torch.from_numpy(z).double(), torch.from_numpy(ctx).double(),
                                                   t64(hid), t64(heads), "elu")
    # the torch restatement against the numpy oracle on a slice (belt and braces at this size)
    f64 = lambda ls: O.cast_params(ls, np.float64)
    zo, _, ldo = O.iaf_step(variant, z[100:102].astype(np.float64), ctx[100:102].astype(np.float64), f64(hid), f64(heads))
    assert np.abs(z_ref[100:102].numpy() - zo).max() < 1e-10 and np.abs(logdet_ref[100:102].numpy() - ldo).max() < 1e-9
    op = make_op(variant, n_z, hidden, "elu", "tc", hid, heads)
    z1, logsd, logdet = op.step(torch.from_numpy(z).cuda(), torch.from_numpy(ctx).cuda())
    assert op.path_used(H, W, "cuda:0", entry="step") == "tc"
    # per sample, so that one bad sample cannot hide behind the batch maximum of the reference
    per = (z1.double().cpu() - z_ref).abs().flatten(1).max(dim=1).values / z_ref.abs().flatten(1).max(dim=1).values.clamp(min=1.0)
    bad = [(int(i), float(per[i])) for i in torch.nonzero(per >= TOL).flatten()[:12]]
    assert not bad, "samples with z' error above tolerance (index, rel err): %s" % bad
    per_ld = (logdet.double().cpu() - logdet_ref).abs() / logdet_ref.abs().clamp(min=1.0)
    bad = [(int(i), float(per_ld[i])) for i in torch.nonzero(per_ld >= TOL).flatten()[:12]]
    assert not bad, "samples with logdet error above tolerance (index, rel err): %s" % bad
    assert relerr(z1, z_ref.numpy()) < TOL
    assert relerr(logsd, logsd_ref.numpy()) < TOL
    assert relerr(logdet, logdet_ref.numpy()) < TOL


def test_plans_created_large_to_small_keep_working():
    """ADVICE round 1 (high): a kernel's dynamic shared-memory limit used to be set per plan, so creating a plan with a
    smaller footprint lowered it for earlier, larger plans.  16x16, then 4x4, then forward + backward on 16x16 again."""
    variant, n_z, hidden = "theano", 32, [64]
    hid, heads = O.make_params(variant, n_z, hidden, [n_z, n_z], seed=3)
    for path in ("simt", "tc"):
        op = make_op(variant, n_z, hidden, "elu", path, hid, heads)
        for layer in op._layers:
            for t in layer:
                t.requires_grad_(True)
        outs = {}
        for hw in (16, 4, 16, 8, 16):
            z, ctx = O.make_inputs(3, n_z, hidden[0], hw, hw, seed=4)
            zc = torch.from_numpy(z).cuda().requires_grad_(True)
            cc = torch.from_numpy(ctx).cuda().requires_grad_(True)
            z1, logsd, logdet = op.step(zc, cc)
            (z1.square().sum() + logdet.sum()).backward()
            torch.cuda.synchronize()
            key = (hw,)
            if key in outs:
                assert torch.equal(outs[key][0], z1.detach()) and torch.allclose(outs[key][1], zc.grad, rtol=1e-5, atol=1e-6)
            outs[key] = (z1.detach().clone(), zc.grad.clone())


def test_parameters_updated_through_data_need_invalidate():
    """ADVICE round 1 (medium): ``p.data`` updates do not bump the tensor version the packed-weight cache keys on."""
    variant, n_z, hidden, H, W = "tf", 4, [8], 5, 5
    hid, heads = O.make_params(variant, n_z, hidden, [n_z, n_z], seed=1)
    z, ctx = O.make_inputs(2, n_z, hidden[0], H, W, seed=2)
    zc, cc = torch.from_numpy(z).cuda(), torch.from_numpy(ctx).cuda()
    op = make_op(variant, n_z, hidden, "elu", "simt", hid, heads)
    a = op.step(zc, cc)[0].clone()
    op._layers[1][2].data.add_(1.0)          # head-0 bias through .data: version counter unchanged
    op.invalidate()
    b = op.step(zc, cc)[0]
    heads[0]["b"] = heads[0]["b"] + 1.0
    f64 = lambda ls: O.cast_params(ls, np.float64)
    ref = O.iaf_step(variant, z.astype(np.float64), ctx.astype(np.float64), f64(hid), f64(heads))[0]
    assert relerr(b, ref) < TOL and not torch.equal(a, b)
    # calls recorded for autograd re-pack on every call: no invalidate() needed in a training loop
    for layer in op._layers:
        for t in layer:
            t.requires_grad_(True)
    op.step(zc, cc)
    op._layers[1][2].data.add_(1.0)
    c = op.step(zc, cc)[0]
    heads[0]["b"] = heads[0]["b"] + 1.0
    ref2 = O.iaf_step(variant, z.astype(np.float64), ctx.astype(np.float64), f64(hid), f64(heads))[0]
    assert relerr(c.detach(), ref2) < TOL


def test_path_report_per_entry_and_no_silent_downgrade():
    from iaf_b200 import IAFOperator
    hid, heads = O.make_params("tf", 32, [64], [32, 32], seed=1)
    auto = IAFOperator("tf", 32, [64], [32, 32], path="auto").set_weights(dev_layers("tf", hid, heads))
    for entry in ("step", "multiconv", "layer"):
        assert auto.path_used(16, 16, "cuda:0", entry=entry) in ("tc", "simt")
    assert auto.path_used(16, 16, "cuda:0", entry="step") == "tc"
    # a shape the tensor-core kernels cannot take: auto reports simt, an explicit tc operator refuses
    hid4, heads4 = O.make_params("tf", 4, [8], [4, 4], seed=1)
    small = IAFOperator("tf", 4, [8], [4, 4], path="auto").set_weights(dev_layers("tf", hid4, heads4))
    assert small.path_used(6, 6, "cuda:0", entry="layer") == "simt"
    with pytest.raises(NotImplementedError):
        IAFOperator("tf", 4, [8], [4, 4], path="tc").set_weights(dev_layers("tf", hid4, heads4)).path_used(6, 6, "cuda:0")


def test_imported_theano_weights_drive_the_operator(tmp_path):
    """SURVEY 8f-3: graphy's ``.ndict.tar.gz`` container (ndict.py:209-236) -> np_loadz -> theano_layers -> operator."""
    from iaf_b200 import IAFOperator
    from iaf_b200.weights import np_loadz, np_savez, theano_layers
    n_z, n_h, dar, H, W = 32, 64, 1, 8, 8
    hid, heads = O.make_params("theano", n_z, dar * [n_h], [n_z, n_z], seed=11)
    name = "0_1_posterior_conv1"                                  # models.py:410: {i}_{j}_posterior_conv1
    w = {}
    for i, l in enumerate(hid):
        for k in "wsb":
            w["%s_%d_%s" % (name, i, k)] = l[k]
    for i, l in enumerate(heads):
        for k in "wsb":
            w["%s_out_%d_%s" % (name, i, k)] = l[k]
    w["unrelated_conv_w"] = np.zeros((3, 3), np.float32)
    fn = os.path.join(str(tmp_path), "weights.ndict.tar.gz")
    np_savez(w, fn)
    loaded = np_loadz(fn)
    op = IAFOperator("theano", n_z, dar * [n_h], [n_z, n_z], nl="elu").set_weights(theano_layers(loaded, name, dar))
    z, ctx = O.make_inputs(5, n_z, n_h, H, W, seed=12)
    f64 = lambda ls: O.cast_params(ls, np.float64)
    z_ref, logsd_ref, logdet_ref = O.iaf_step("theano", z.astype(np.float64), ctx.astype(np.float64), f64(hid), f64(heads))
    z1, logsd, logdet = op.step(torch.from_numpy(z).cuda(), torch.from_numpy(ctx).cuda())
    assert relerr(z1, z_ref) < TOL and relerr(logsd, logsd_ref) < TOL and relerr(logdet, logdet_ref) < TOL


def test_bits_per_dim_c3_full_depth():
    """BASELINE config C3: ResNet-VAE num_blocks=20, depth=1, z=32, h=160, kl_min=0.1, batch 32 (tf_train.py:98-112).  The
    CUDA-backed ELBO against the same ELBO with the fp64 oracle block on the host."""
    from iaf_b200 import elbo
    from oracle.elbo_oracle import TorchIAF
    from tests.test_elbo import _setup
    hps = dict(z_size=32, h_size=160, depth=1, num_blocks=20, kl_min=0.1, image_size=32)
    pg, xg, ng = _setup(hps, 32, 9, torch.float32, "cuda")
    pc, xc, nc = _setup(hps, 32, 9, torch.float64, "cpu")
    with torch.no_grad():
        got = elbo.forward(pg, xg, ng, elbo.CudaIAF(pg, hps), hps)
        ref = elbo.forward(pc, xc, nc, TorchIAF(pc, hps), hps)
    g, r = float(got["bits_per_dim"]), float(ref["bits_per_dim"])
    assert abs(g - r) <= 1e-4 * max(abs(r), 1.0), (g, r)


def test_bits_per_dim_c4_full_depth():
    """BASELINE config C4: the 3.28-bpd Theano model, n_h=160, depths [10,10], depth_ar=2, down_iaf2_nl (README.md:55-58)."""
    from iaf_b200 import elbo_theano as ET
    from oracle.elbo_oracle import TorchIAFTheano
    from tests.test_elbo_theano import _setup as theano_setup
    hps = dict(n_z=32, n_h1=160, n_h2=160, depths=[10, 10], depth_ar=2, nl="elu", kl_min=0.25, image_size=32)
    wg, xg, ng = theano_setup(hps, 4, 9, torch.float32, "cuda")
    wc, xc, nc = theano_setup(hps, 4, 9, torch.float64, "cpu")
    with torch.no_grad():
        got = ET.forward(wg, xg, ng, ET.CudaIAF(wg, hps), hps)
        ref = ET.forward(wc, xc, nc, TorchIAFTheano(wc, hps), hps)
    g, r = float(got["bits_per_dim"]), float(ref["bits_per_dim"])
    assert abs(g - r) <= 1e-4 * max(abs(r), 1.0), (g, r)


@pytest.mark.parametrize("name", ["tc_kl01", "tc_kl0"])
def test_tensor_core_fused_layer_against_iaflayer_down_fixture(name):
    """iaf_layer_fwd on the TENSOR-CORE path (z 32, h 64, 8x8: hidden [64, 64] runs the tensor-core stage kernels in
    their layer mode) against tensors IAFLayer.down (tf_train.py:46-95) produced when executed from the reference's source
    (tests/golden/make_golden.py): z', kl_cost, the per-(sample, channel) KL sums and the free-bits objective."""
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "iaflayer_down_tc.npz"))
    v = lambda k: g[name + "_" + k].astype(np.float64)
    zs, hs = 32, 64
    hid, heads = O.make_params("tf", zs, [hs, hs], [zs, zs], seed=77)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a.astype(np.float32))).cuda()
    op = make_op("tf", zs, [hs, hs], "elu", "tc", hid, heads)
    assert op.path_used(8, 8, "cuda:0", entry="layer") == "tc"
    z1, kl, kl_bc, kl_cost = op.layer(t(v("eps")), t(v("rz_mean") + v("qz_mean")), t(v("rz_logsd") + v("qz_logsd")),
                                      t(v("pz_mean")), t(v("pz_logsd")), t(v("up_context") + v("down_context")))
    z_ref = (v("z0") - 0.1 * v("m")) / np.exp(0.1 * v("s"))
    assert relerr(z1, z_ref) < TOL
    assert relerr(kl_cost, v("kl_cost")) < TOL
    assert relerr(kl.sum(dim=(2, 3)), kl_bc.cpu().numpy().astype(np.float64)) < 1e-5
    kl_min = float(g[name + "_kl_min"])
    if kl_min > 0:   # tf_train.py:77-83
        kl_obj = torch.clamp(kl_bc.mean(dim=0, keepdim=True), min=kl_min).expand(kl_bc.shape[0], -1).sum(dim=1)
    else:
        kl_obj = kl_cost
    assert relerr(kl_obj, v("kl_obj")) < TOL
