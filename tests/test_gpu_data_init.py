"""The data-dependent initialisation on the H100: elbo.data_init / elbo_theano.data_init on CUDA tensors (cuDNN convs)
against the fp64 CPU pass, the reference's post-condition of the init (standardised heads) checked through the CUDA
operator on the tensor cores, the cube-root gain of the TF model pinned there too, and training gradients at the
initialised parameters.  TF32 is switched off throughout: the pass's convs then run in full fp32."""
import numpy as np
import pytest
import torch

from iaf_b200 import elbo
from iaf_b200 import elbo_theano as ET
from iaf_b200.ops import IAFOperator
from oracle import iaf_oracle as O

pytestmark = pytest.mark.gpu

TF_HPS = dict(z_size=32, h_size=64, depth=2, num_blocks=1, kl_min=0.25, image_size=32)
# c2a's stack (n_z 32, one hidden layer of 64) at 16x16 on level 0
TH_HPS = dict(n_z=32, n_h1=64, n_h2=64, depths=[1, 1], depth_ar=1, nl="elu", kl_min=0.25, image_size=32,
              posterior="down_iaf2_nl", prior="diag")


@pytest.fixture(autouse=True)
def _no_tf32():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def _tf_setup(B, seed):
    """The reference's starting point: V from make_params, h_top and dec_log_stdv zero; g, b are overwritten."""
    p = {k: torch.from_numpy(np.asarray(v, dtype=np.float64)) for k, v in elbo.make_params(TF_HPS, seed=seed).items()}
    p["h_top"] = torch.zeros_like(p["h_top"])
    p["dec_log_stdv"] = torch.zeros_like(p["dec_log_stdv"])
    rng = np.random.RandomState(seed + 1)
    S = TF_HPS["image_size"]
    x = torch.from_numpy(rng.randint(0, 256, size=(B, 3, S, S)).astype(np.uint8))
    noise = {(i, j): torch.from_numpy(rng.randn(B, TF_HPS["z_size"], S // 2 ** (i + 1), S // 2 ** (i + 1)))
             for i in range(TF_HPS["depth"]) for j in range(TF_HPS["num_blocks"])}
    return p, x, noise


def _th_setup(B, seed):
    """The reference's starting point: kernels from make_params, every _s and _b zero (conv.py:176-182, ar.py:292-296),
    h_top and logsd_x zero."""
    w = {k: torch.from_numpy(np.asarray(v, dtype=np.float64)) for k, v in ET.make_params(TH_HPS, seed=seed).items()}
    for k in w:
        if not k.endswith("_w"):
            w[k] = torch.zeros_like(w[k])
    rng = np.random.RandomState(seed + 1)
    S = TH_HPS["image_size"]
    x = torch.from_numpy(rng.randint(0, 256, size=(B, 3, S, S)).astype(np.uint8))
    noise = {(i, 0): torch.from_numpy(rng.randn(B, TH_HPS["n_z"], S // 2 ** (i + 1), S // 2 ** (i + 1))) for i in range(2)}
    return w, x, noise


def _to(d, dtype, device="cuda"):
    return {k: v.to(dtype).to(device) for k, v in d.items()}


@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-9), (torch.float32, 2e-3)])
@pytest.mark.parametrize("model", ["tf", "theano"])
def test_data_init_on_cuda_matches_fp64_cpu(model, dtype, tol):
    """Every initialised parameter of the pass on CUDA (cuDNN convs) against the fp64 pass on the CPU: gains are logs,
    so their absolute error is the relative error of the scale; biases relative to their largest magnitude.  fp32:
    the pass standardises 20-odd convs in sequence, each on the previous one's fp32 output."""
    mod, (p, x, noise) = (elbo, _tf_setup(8, 3)) if model == "tf" else (ET, _th_setup(8, 3))
    ref = mod.data_init(p, x, TF_HPS if model == "tf" else TH_HPS, noise)
    got = mod.data_init(_to(p, dtype), x.cuda(), TF_HPS if model == "tf" else TH_HPS, _to(noise, dtype))
    for k, r in ref.items():
        assert got[k].device.type == "cuda", k
        g = got[k].double().cpu()
        if k.endswith(("/g", "_s")):
            err = float((g - r).abs().max())
        else:
            err = float((g - r).abs().max()) / max(float(r.abs().max()), 1e-30)
        assert err <= tol, (k, err)


def test_theano_heads_standardised_after_init_on_tensor_cores():
    """ar.py:331-353's post-condition: after the init pass, the stack run at the new parameters on the input the pass
    gave it returns heads with mean 0 and std 1 per channel over the batch.  Through IAFOperator.multiconv on the
    tensor cores, c2a-shaped, for the level-0 posterior stack of the pass run on CUDA."""
    w, x, noise = _th_setup(16, 5)
    w = _to(w, torch.float32)
    new, _, stacks = ET.data_init_pass(w, x.cuda(), TH_HPS, _to(noise, torch.float32))
    z, ctx = stacks["0_0_posterior_conv1"]
    assert tuple(z.shape) == (16, 32, 16, 16)
    op = IAFOperator("theano", 32, [64], [32, 32], nl="elu", path="tc")
    op.set_weights(ET.CudaIAF(new, TH_HPS)._posterior_layers("0_0", 1, lambda t: t.float().contiguous()))
    assert op.path_used(16, 16, "cuda", entry="multiconv") == "tc"
    for head in op.multiconv(z.contiguous(), ctx.contiguous()):
        h = head.double()
        mean, std = h.mean(dim=(0, 2, 3)), h.std(dim=(0, 2, 3), unbiased=False)
        assert float(mean.abs().max()) <= 1e-4, float(mean.abs().max())
        assert float((std - 1).abs().max()) <= 1e-4, float((std - 1).abs().max())


def test_tf_heads_after_init_run_at_cube_root_gain_on_tensor_cores():
    """layers.py:49, 60: the init pass stores g = log(scale) / 3 and the run-time branch applies exp(g).  The stack run
    on the tensor cores at the initialised parameters, on the input the fp64 CPU pass gave it, equals the fp64 run-time
    stack exp(g) conv(x, v_norm) + b at those parameters -- not the pass's standardised output."""
    p, x, noise = _tf_setup(8, 7)
    new, _, stacks = elbo.data_init_pass(p, x, TF_HPS, noise)
    z, ctx = stacks["IAF_0_0/ar_multiconv2d"]
    pre = "IAF_0_0/ar_multiconv2d/"
    names = ["layer_0", "layer_1", "layer_out_0", "layer_out_1"]
    layers = [{k: new[pre + n + "/" + k].numpy() for k in "Vgb"} for n in names]
    ref = O.tf_ar_multiconv2d(z.numpy(), ctx.numpy(), layers[:2], layers[2:], "elu")
    op = IAFOperator("tf", 32, [64, 64], [32, 32], nl="elu", path="tc")
    op.set_weights([tuple(new[pre + n + "/" + k].float().cuda() for k in "Vgb") for n in names])
    assert op.path_used(16, 16, "cuda", entry="multiconv") == "tc"
    got = op.multiconv(z.float().cuda().contiguous(), ctx.float().cuda().contiguous())
    for g, r in zip(got, ref):
        err = float(np.abs(g.double().cpu().numpy() - r).max()) / float(np.abs(r).max())
        assert err <= 1e-4, err
        std = r.std(axis=(0, 2, 3))
        assert float(np.abs(std - 1).max()) > 0.05       # the heads are NOT standardised: g is a cube root


def test_training_gradients_at_initialised_parameters():
    """As test_training_objective_gradient_parity, at the parameters data_init gives (head gains up to the batch's
    scale^(1/3) instead of make_params' exp(+-0.3)): CudaIAFTrain's objective and every parameter gradient against fp64
    torch autograd through the oracle block."""
    from oracle.elbo_oracle import TorchIAF
    hps = dict(z_size=32, h_size=64, depth=2, num_blocks=1, kl_min=0.25, image_size=32)
    p, x, noise = _tf_setup(3, 9)
    init = elbo.data_init(p, x, hps, noise)
    pc = {k: v.clone().requires_grad_(True) for k, v in init.items()}
    pg = {k: v.float().cuda().requires_grad_(True) for k, v in init.items()}
    ng = _to(noise, torch.float32)
    got = elbo.forward(pg, x.cuda(), ng, elbo.CudaIAFTrain(pg, hps), hps)
    ref = elbo.forward(pc, x, noise, TorchIAF(pc, hps), hps)
    np.testing.assert_allclose(float(got["obj"].detach()), float(ref["obj"].detach()), rtol=1e-4)
    got["obj"].backward()
    ref["obj"].backward()
    for k in pc:
        g, r = pg[k].grad, pc[k].grad
        if r is None:
            assert g is None, k
            continue
        assert g is not None, k
        err = float((g.double().cpu() - r).abs().max()) / max(float(r.abs().max()), 1e-12)
        assert err < 2e-3, (k, err)
        if "ar_multiconv2d" in k and k.endswith("/V"):
            mask = O.get_conv_ar_mask(3, 3, g.shape[2], g.shape[3], "layer_out" in k)
            assert bool((g.cpu().numpy()[mask == 0] == 0).all()), k
