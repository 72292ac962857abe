"""The one-launch step kernel's handoffs across tile boundaries: outputs bit for bit against the per-stage kernels and
across SM caps.

The one-launch kernel (``iaf_ly_kernel`` with ``FUSED``) hands its hidden activations to the heads MMAs through a
shared-memory buffer, one barrier per 16-channel chunk, so that the heads MMAs of a chunk run while the hidden
epilogue computes the later ones; two warps of their own build each tile's z window while the epilogue warps run the
previous tile's epilogues.  A wrong parity or a missing wait in that schedule shows up as a tile that reads another
tile's hidden rows or window -- most likely where a CTA moves from one tile to the next, or on a last, partial tile.

1. z' and arw_logsd of the one-launch step equal, bit for bit, those of the per-stage plan (``IAF_TC_FUSED=0``: one
   launch per stage, activations through global operand images).  The two compute every element in the same order;
   only the log-dets are summed over other tilings.
2. Every output of the step, layer and MADE-prior (logp) entries of the one-launch kernel is bit-identical across
   ``IAF_NUM_SMS`` = 1, 2, 3 and the device's count: one CTA running every tile, uneven runs of tiles, and one tile per
   CTA or close to it.

Shapes: c2a (n_z 32, hidden [64], 16x16) at the benchmark batch B = 256 and at B = 37, whose last tile is partial;
the TF, Theano and flipmask variants, elu and softplus."""
import numpy as np
import pytest
import torch

from oracle import iaf_oracle as O
from tests.test_gpu_flipmask_envelope import _pv, v_op
from tests.test_gpu_tc_envelope import DEV, layer_inputs, make_params

pytestmark = pytest.mark.gpu

N_Z, HIDDEN, H, W = 32, [64], 16, 16
VARIANTS = ["tf", "theano", "flip"]
NLS = ["elu", "softplus"]
BATCHES = [256, 37]
CAPS = [None, 1, 2, 3]


def _tiles(B):
    ts = 128 - (W + 2 + 7) // 8 * 8
    return B * (H + 1) * (W + 1) / ts


def test_partial_batch_has_a_partial_last_tile():
    t = _tiles(37)
    assert t != int(t) and _tiles(256) > 132


def _op(monkeypatch, variant, nl, fused, cap, layers):
    monkeypatch.setenv("IAF_TC_FUSED", "1" if fused else "0")  # read at plan creation
    if cap is None:
        monkeypatch.delenv("IAF_NUM_SMS", raising=False)
    else:
        monkeypatch.setenv("IAF_NUM_SMS", str(cap))
    op, _ = v_op(variant, N_Z, HIDDEN, "auto", layers, nl=nl)
    assert op.path_used(H, W, DEV, entry="step") == "tc"
    return op


def _inputs(variant, B):
    hid, hd = make_params(_pv(variant), N_Z, HIDDEN, seed=301)
    z, ctx = O.make_inputs(B, N_Z, HIDDEN[0], H, W, seed=302)
    lin = layer_inputs(B, N_Z, HIDDEN, H, W, seed=303)
    t = lambda a: torch.from_numpy(a).to(DEV)
    return hid + hd, t(z), t(ctx), [t(a) for a in lin]


def _step(op, z, ctx, launches):
    l0 = op.launch_count()
    out = op.step(z, ctx)
    torch.cuda.synchronize()
    assert op.launch_count() - l0 == launches
    return out


@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("nl", NLS)
@pytest.mark.parametrize("variant", VARIANTS)
def test_one_launch_step_equals_per_stage(variant, nl, B, monkeypatch):
    layers, z, ctx, _ = _inputs(variant, B)
    z1, ls1, _ = _step(_op(monkeypatch, variant, nl, True, None, layers), z, ctx, 1)
    z2, ls2, _ = _step(_op(monkeypatch, variant, nl, False, None, layers), z, ctx, 2)
    assert torch.isfinite(z1).all() and torch.isfinite(ls1).all()
    assert torch.equal(z1, z2)
    assert torch.equal(ls1, ls2)


@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("nl", NLS)
@pytest.mark.parametrize("variant", VARIANTS)
def test_one_launch_outputs_across_sm_caps(variant, nl, B, monkeypatch):
    layers, z, ctx, lin = _inputs(variant, B)
    base = None
    for cap in CAPS:
        op = _op(monkeypatch, variant, nl, True, cap, layers)
        got = list(_step(op, z, ctx, 1))
        got += list(op.layer(*lin))
        got += list(op.ar_logp(z, ctx, want_logps=True))
        torch.cuda.synchronize()
        assert all(torch.isfinite(g).all() for g in got), cap
        if base is None:
            base = got
            continue
        for k, (a, b) in enumerate(zip(got, base)):
            assert torch.equal(a, b), (cap, k)
