"""The one-launch step kernel's CTA pairs: every output bit for bit against the per-stage plan, at pair boundaries.

When the device holds the grid's clusters, the one-launch kernel (``iaf_ly_kernel`` with ``FUSED``) runs in clusters of
two CTAs (``fz_run`` in ``iaf_tc_gemm.cuh``).  Cluster c of G / 2 covers the tiles [T0, T2) and splits them at
T1 = T0 + floor((T2 - T0) / 2): the giver runs [T0, T1) downwards from T1 - 1, the receiver [T1, T2) upwards.  Both
first tiles need the hidden rows of slots [128 T1, +MIR); the giver computes them in its halo block and writes them into
the receiver's shared memory, and the receiver runs no halo block.  A downward tile computes its own 128 rows and
carries the MIR rows after them from the tile it ran before.  A cluster of one tile has an empty lower run, and its
receiver runs alone with a halo block of its own.  An odd grid below the SM cap gets one CTA more.

A hidden row adds the same products in the same order whichever tile computes it, and the heads' per-tile partials
keep the per-stage kernel's tiles, so every output -- z', arw_logsd, log-dets, the layer mode's and the MADE prior's
per-sample and per-channel sums, and the activations the training forward keeps -- equals the per-stage plan's
(``IAF_TC_FUSED=0``) bit for bit.  The training forward's activations go into a NaN-poisoned buffer, so a slot that no
tile keeps stays NaN.  A halo sent to the wrong rows, a carry in the wrong direction or a receiver that reads its rows
before they arrive shows up as a difference at a pair's first tiles.

The cases place pair boundaries (``IAF_NUM_SMS`` caps the grid) on a sample boundary, mid-sample and where the halo
crosses into the next sample; give pairs of equal and unequal runs, of one-tile runs and with an empty run; and cover a
map whose MIR is 64."""
import ctypes as C

import pytest
import torch

from iaf_b200 import _lib
from iaf_b200.ops import _ptr, _stream
from tests.test_gpu_one_launch_runs import C2A, EDGE, NLS, VARIANTS, _geom, _inputs, _op
from tests.test_gpu_graphs_streams import capture

# (shape, batch, SM cap; None = the device's count), and what the case places at a pair
CASES = [
    (C2A, 256, 2, "one pair of equal runs; its boundary on a sample boundary"),
    (C2A, 256, 10, "equal and unequal pairs; boundaries mid-sample and where the halo crosses into the next sample"),
    (C2A, 37, None, "pairs of one-tile runs; partial last tile"),
    (C2A, 3, None, "a pair with an empty run: the grid rounded up to even"),
    (EDGE, 5, 4, "MIR = 64; equal and unequal pairs"),
    (EDGE, 5, None, "MIR = 64; one-tile runs and an empty run"),
]
CASE_IDS = ["c2a-B256-cap2", "c2a-B256-cap10", "c2a-B37-all", "c2a-B3-all", "mir64-B5-cap4", "mir64-B5-all"]


def _fz_run(b, G, NT):
    """(first tile, tiles, downwards, halo block) of CTA b of a paired grid of G, as fz_run computes it."""
    nc, c = G // 2, b // 2
    t0, t2 = c * NT // nc, (c + 1) * NT // nc
    t1 = t0 + (t2 - t0) // 2
    if t1 == t0:
        return (t1, t2 - t1, False, True) if b & 1 else (t0, 0, False, False)
    return (t1, t2 - t1, False, False) if b & 1 else (t1 - 1, t1 - t0, True, True)


def _paired_grid(nt, cap):
    g = min(cap, nt)
    return g + (g & 1)


def test_pair_runs_cover_every_tile_once():
    """The pairs' runs partition the tiles, no run is longer than an unpaired one, and a receiver whose giver has tiles
    is never shorter than it."""
    for nt in range(1, 700):
        for cap in (2, 4, 10, 132):
            G = _paired_grid(nt, cap)
            if G > cap:
                continue
            seen = []
            for b in range(G):
                first, n, down, _ = _fz_run(b, G, nt)
                seen += [first - i for i in range(n)] if down else [first + i for i in range(n)]
                assert n <= -(-nt // G), (nt, cap, b)
                if b & 1 and _fz_run(b - 1, G, nt)[1]:
                    assert n >= _fz_run(b - 1, G, nt)[1]
            assert sorted(seen) == list(range(nt)), (nt, cap)


def test_cases_cover_the_pair_boundaries():
    """The cases place each boundary where the docstring says (132 SMs for an uncapped H100 SXM)."""
    seen = set()
    for shape, B, cap, _ in CASES:
        sps, mir, nt = _geom(shape, B)
        G = _paired_grid(nt, cap or 132)
        assert G <= (cap or 132)
        if mir == 64:
            seen.add("mir64")
        if (B * sps) % 128:
            seen.add("partial")
        for c in range(G // 2):
            giver, recv = _fz_run(2 * c, G, nt), _fz_run(2 * c + 1, G, nt)
            if giver[1] == 0:
                seen.add("empty")
                continue
            seen.add("equal" if giver[1] == recv[1] else "unequal")
            if recv[1] == 1:
                seen.add("one-tile")
            off = 128 * (giver[0] + 1) % sps
            seen.add("on sample" if off == 0 else "halo crosses" if off + mir > sps else "mid-sample")
    assert seen == {"mir64", "partial", "empty", "equal", "unequal", "one-tile", "on sample", "halo crosses",
                    "mid-sample"}


def _train_hidden(op, z, ctx):
    """The training forward's kept activations, written into a NaN-poisoned buffer."""
    B, _, H, W = z.shape
    plan = op._plan(H, W, z.device)
    z_out, logsd = torch.empty_like(z), torch.empty_like(z)
    logdet = torch.empty((B,), device=z.device, dtype=torch.float32)
    hidden = torch.full((B, op.hidden[0], H, W), float("nan"), device=z.device, dtype=torch.float32)
    harr = (C.c_void_p * 1)(hidden.data_ptr())
    with torch.cuda.device(z.device):
        _lib.check(op._lib.iaf_step_fwd_train(plan, _ptr(z), _ptr(ctx), _ptr(z_out), _ptr(logsd), _ptr(logdet), harr,
                                              B, _stream(z.device)))
    return [z_out, logsd, logdet, hidden]


def _outputs(op, z, ctx, lin, launches):
    l0 = op.launch_count()
    got = list(op.step(z, ctx))
    torch.cuda.synchronize()
    assert op.launch_count() - l0 == launches
    got += list(op.layer(*lin))
    got += list(op.ar_logp(z, ctx, want_logps=True))
    got += _train_hidden(op, z, ctx)
    torch.cuda.synchronize()
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
@pytest.mark.parametrize("nl", NLS)
@pytest.mark.parametrize("variant", VARIANTS)
def test_one_launch_pairs_equal_per_stage(variant, nl, case, monkeypatch):
    shape, B, cap, _ = case
    if cap is None:
        assert _geom(shape, B)[2] < torch.cuda.get_device_properties(0).multi_processor_count
    layers, z, ctx, lin = _inputs(variant, shape, B)
    one = _outputs(_op(monkeypatch, variant, nl, shape, True, cap, layers), z, ctx, lin, 1)
    per = _outputs(_op(monkeypatch, variant, nl, shape, False, None, layers), z, ctx, lin, 2)
    assert len(one) == len(per)
    for k, (a, b) in enumerate(zip(one, per)):
        assert torch.isfinite(a).all(), k
        assert torch.equal(a, b), k


@pytest.mark.gpu
@pytest.mark.parametrize("variant", VARIANTS)
def test_captured_paired_step_equals_per_stage(variant, monkeypatch):
    """The paired step captured in a CUDA graph (halo crossing into the next sample), replayed after its inputs
    change in place."""
    layers, z, ctx, _ = _inputs(variant, C2A, 256)
    one = _op(monkeypatch, variant, "softplus", C2A, True, 10, layers)
    per = _op(monkeypatch, variant, "softplus", C2A, False, None, layers)
    zg, cg = z.clone(), ctx.clone()
    one.step(zg, cg)  # plan scratch allocated outside the capture
    torch.cuda.synchronize()
    graph, out, _ = capture(lambda: one.step(zg, cg))
    for scale in (1.0, 0.5):
        zg.copy_(z * scale)
        cg.copy_(ctx)
        graph.replay()
        torch.cuda.synchronize()
        want = per.step(zg, cg)
        torch.cuda.synchronize()
        for k, (a, b) in enumerate(zip(out, want)):
            assert torch.equal(a, b), (scale, k)
