"""CPU simulation of operand precision for the IAF step (development aid): rounds the conv operands
of an fp64 evaluation of the oracle to candidate tensor-core formats and reports the z' / logdet errors the parity tests
measure.  usage: python tools/experiments/prec_sim.py"""
import os, sys, time
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', '..'))
import numpy as np, torch
import torch.nn.functional as F
from oracle import iaf_oracle as O, iaf_oracle_torch as OT
torch.set_num_threads(8)

def quant(x, mode):
    if mode == "exact": return x
    if mode == "fp16": return x.to(torch.float16).to(x.dtype)
    if mode == "bf16": return x.to(torch.bfloat16).to(x.dtype)
    if mode == "bf16x2":  # hi+lo bf16 (what the kernel does now)
        hi = x.to(torch.bfloat16).to(x.dtype); lo = (x - hi).to(torch.bfloat16).to(x.dtype); return hi + lo
    if mode == "tf32":
        xf = x.float(); i = xf.view(torch.int32); i = (i + 0x1000) & ~0x1FFF; return i.view(torch.float32).to(x.dtype)
    raise ValueError

def step(variant, z, ctx, hid, heads, mode, wmode="exact"):
    x = z
    conv = OT.tf_ar_conv2d
    for i, l in enumerate(hid):
        x = conv(quant(x, mode), l, False)
        if i == 0: x = x + ctx
        x = F.elu(x)
    m = conv(quant(x, mode), heads[0], True); s = conv(quant(x, mode), heads[1], True)
    zn = (z - 0.1*m) / torch.exp(0.1*s)
    return zn, -(0.1*s).flatten(1).sum(1)

for name, hidden in (("c2a", [64]), ("c2b", [160, 160])):
    B = 64 if name == "c2a" else 32
    hid, hd = O.make_params("tf", 32, hidden, [32, 32], seed=1)
    z, ctx = O.make_inputs(B, 32, hidden[0], 16, 16, seed=0)
    f64 = lambda ls: OT.to_torch(O.cast_params(ls, np.float64), torch.float64)
    th, thh = f64(hid), f64(hd)
    zt, ct = torch.from_numpy(z).double(), torch.from_numpy(ctx).double()
    ref = step("tf", zt, ct, th, thh, "exact")
    print(name, "max|z'|=%.2f max|logdet|=%.2f" % (ref[0].abs().max(), ref[1].abs().max()))
    for mode in ("bf16x2", "fp16", "tf32", "bf16"):
        t = time.time()
        got = step("tf", zt, ct, th, thh, mode)
        ez = float((got[0]-ref[0]).abs().max() / max(ref[0].abs().max(), 1.0))
        el = float((got[1]-ref[1]).abs().max() / max(ref[1].abs().max(), 1.0))
        ela = float((got[1]-ref[1]).abs().max())
        print("  activations %-7s  rel err z' %.2e  logdet %.2e (abs %.2e)  [tol 1e-4]" % (mode, ez, el, ela))

print("---- weights quantised (effective, normalised weights), activations exact ----")
def eff_w(l, zd):
    V, g = l["V"], l["g"]
    mask = torch.from_numpy(O.get_conv_ar_mask(3, 3, V.shape[2], V.shape[3], zd)).to(V.dtype)
    v = mask * V
    return torch.exp(g).reshape(1,1,1,-1) * v * torch.rsqrt(torch.clamp((v*v).sum(dim=(0,1,2), keepdim=True), min=1e-12))
def conv_w(x, w, b): return F.conv2d(x, w.permute(3,2,0,1), padding=1) + b.reshape(1,-1,1,1)
def step_w(z, ctx, hid, heads, wq, aq):
    x = z
    for i, l in enumerate(hid):
        x = conv_w(quant(x, aq), quant(eff_w(l, False), wq), l["b"])
        if i == 0: x = x + ctx
        x = F.elu(x)
    m = conv_w(quant(x, aq), quant(eff_w(heads[0], True), wq), heads[0]["b"]); s = conv_w(quant(x, aq), quant(eff_w(heads[1], True), wq), heads[1]["b"])
    return (z - 0.1*m)/torch.exp(0.1*s), -(0.1*s).flatten(1).sum(1)
for name, hidden in (("c2a", [64]), ("c2b", [160, 160])):
    B = 64 if name == "c2a" else 32
    hid, hd = O.make_params("tf", 32, hidden, [32, 32], seed=1)
    z, ctx = O.make_inputs(B, 32, hidden[0], 16, 16, seed=0)
    f64 = lambda ls: OT.to_torch(O.cast_params(ls, np.float64), torch.float64)
    th, thh = f64(hid), f64(hd)
    zt, ct = torch.from_numpy(z).double(), torch.from_numpy(ctx).double()
    ref = step_w(zt, ct, th, thh, "exact", "exact")
    for wq, aq in (("fp16", "exact"), ("fp16", "bf16x2"), ("bf16", "exact"), ("bf16x2", "bf16x2")):
        got = step_w(zt, ct, th, thh, wq, aq)
        ez = float((got[0]-ref[0]).abs().max() / max(ref[0].abs().max(), 1.0))
        el = float((got[1]-ref[1]).abs().max() / max(ref[1].abs().max(), 1.0))
        print("  %s weights %-7s activations %-7s rel err z' %.2e  logdet %.2e" % (name, wq, aq, ez, el))

print("---- round 2: per-SAMPLE log-det error (|d logdet_n| / max(|logdet_n|, 1)), weights bf16+bf16 vs fp16+fp16 ----")
def quant2(x, mode):
    if mode == "fp16x2":
        hi = x.to(torch.float16).to(x.dtype); lo = (x - hi).to(torch.float16).to(x.dtype); return hi + lo
    return quant(x, mode)
for name, hidden in (("c2a", [64]), ("c2b", [160, 160])):
    B = 64 if name == "c2a" else 32
    hid, hd = O.make_params("tf", 32, hidden, [32, 32], seed=1)
    z, ctx = O.make_inputs(B, 32, hidden[0], 16, 16, seed=0)
    f64 = lambda ls: OT.to_torch(O.cast_params(ls, np.float64), torch.float64)
    th, thh = f64(hid), f64(hd)
    zt, ct = torch.from_numpy(z).double(), torch.from_numpy(ctx).double()
    ref = step_w(zt, ct, th, thh, "exact", "exact")
    for wq, aq in (("bf16x2", "bf16x2"), ("fp16x2", "bf16x2"), ("fp16x2", "exact"), ("exact", "bf16x2")):
        x = zt
        for i, l in enumerate(th):
            x = conv_w(quant2(x, aq), quant2(eff_w(l, False), wq), l["b"])
            if i == 0: x = x + ct
            x = F.elu(x)
        m = conv_w(quant2(x, aq), quant2(eff_w(thh[0], True), wq), thh[0]["b"]); s = conv_w(quant2(x, aq), quant2(eff_w(thh[1], True), wq), thh[1]["b"])
        ld = -(0.1*s).flatten(1).sum(1)
        per = ((ld - ref[1]).abs() / ref[1].abs().clamp(min=1.0))
        print("  %s weights %-7s activations %-7s  worst per-sample logdet err %.2e (abs %.2e)" % (name, wq, aq, float(per.max()), float((ld-ref[1]).abs().max())))
