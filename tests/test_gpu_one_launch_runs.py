"""The one-launch step kernel's runs of tiles: every output bit for bit against the per-stage plan, at run boundaries.

The one-launch kernel (``iaf_ly_kernel`` with ``FUSED``) covers tile t with slots [128 t, +128), as the per-stage
kernel does, and CTA b of G runs the tiles [floor(b NT / G), floor((b + 1) NT / G)) in ascending order.  The heads'
taps read up to MIR hidden rows past a tile's 128, so a tile's hidden rows [0, MIR) are the previous tile's last MIR,
carried in shared memory; a run's first tile computes them in a halo block over a z window of its own.  A hidden row
adds the same products in the same order whichever tile computes it, and the heads' per-tile partials have the
per-stage kernel's tile boundaries, so every output -- z', arw_logsd, log-dets, the layer mode's and the MADE prior's
per-sample and per-channel sums, and the activations the training forward keeps -- equals the per-stage plan's
(``IAF_TC_FUSED=0``) bit for bit.  A wrong carry, a halo written over the wrong rows or a run that starts where its
halo is not computed shows up as a difference at a run's first tiles.

The cases place run boundaries (``IAF_NUM_SMS`` caps the grid) on a sample boundary, mid-sample, where a run's halo
crosses into the next sample, at runs of a single tile, at a partial last tile and at one run of every tile; and at a
map whose MIR is 64, the edge of the one-launch envelope, where the halo is one full 64-row block."""
import pytest
import torch

from oracle import iaf_oracle as O
from tests.test_gpu_flipmask_envelope import _pv, v_op
from tests.test_gpu_graphs_streams import capture
from tests.test_gpu_tc_envelope import DEV, layer_inputs, make_params

VARIANTS = ["tf", "theano", "flip"]
NLS = ["elu", "softplus"]
C2A = (32, [64], 16, 16)
EDGE = (16, [32], 5, 62)  # MIR = 64
# (shape, batch, SM cap; None = the device's count), and what the case places at a run boundary
CASES = [
    (C2A, 256, 2, "a run starts on a sample boundary"),
    (C2A, 256, 3, "runs start mid-sample"),
    (C2A, 256, 5, "a run's halo crosses into the next sample"),
    (C2A, 37, None, "runs of a single tile; partial last tile"),
    (C2A, 37, 1, "one run of every tile; partial last tile"),
    (EDGE, 5, 4, "MIR = 64; a run's halo crosses into the next sample"),
    (EDGE, 5, None, "MIR = 64; runs of a single tile"),
]
CASE_IDS = ["c2a-B256-cap2", "c2a-B256-cap3", "c2a-B256-cap5", "c2a-B37-all", "c2a-B37-cap1", "mir64-B5-cap4",
            "mir64-B5-all"]


def _geom(shape, B):
    _, _, H, W = shape
    sps = (H + 1) * (W + 1)
    mir = (W + 2 + 7) // 8 * 8
    return sps, mir, -(-B * sps // 128)


def _runs(shape, B, G):
    """(first tile, tiles) of each CTA's run."""
    nt = _geom(shape, B)[2]
    G = min(G, nt)
    return [(b * nt // G, (b + 1) * nt // G - b * nt // G) for b in range(G)]


def test_cases_cover_the_run_boundaries():
    """The cases place each boundary where the docstring says (132 SMs for an uncapped H100 SXM)."""
    seen = set()
    for shape, B, cap, _ in CASES:
        sps, mir, nt = _geom(shape, B)
        runs = _runs(shape, B, cap or 132)
        if mir == 64:
            seen.add("mir64")
        if (B * sps) % 128:
            seen.add("partial")
        if len(runs) == 1:
            seen.add("one run")
        for t0, n in runs:
            off = 128 * t0 % sps
            if n == 1:
                seen.add("single")
            if t0 and off == 0:
                seen.add("on sample")
            if off:
                seen.add("mid-sample")
            if off + mir > sps:
                seen.add("halo crosses")
    assert seen == {"mir64", "partial", "one run", "single", "on sample", "mid-sample", "halo crosses"}


def _op(monkeypatch, variant, nl, shape, fused, cap, layers):
    n_z, hidden, H, W = shape
    monkeypatch.setenv("IAF_TC_FUSED", "1" if fused else "0")  # read at plan creation
    if cap is None:
        monkeypatch.delenv("IAF_NUM_SMS", raising=False)
    else:
        monkeypatch.setenv("IAF_NUM_SMS", str(cap))
    op, _ = v_op(variant, n_z, hidden, "auto", layers, nl=nl)
    assert op.path_used(H, W, DEV, entry="step") == "tc"
    return op


def _inputs(variant, shape, B):
    n_z, hidden, H, W = shape
    hid, hd = make_params(_pv(variant), n_z, hidden, seed=311)
    z, ctx = O.make_inputs(B, n_z, hidden[0], H, W, seed=312)
    lin = layer_inputs(B, n_z, hidden, H, W, seed=313)
    t = lambda a: torch.from_numpy(a).to(DEV)
    return hid + hd, t(z), t(ctx), [t(a) for a in lin]


def _outputs(op, z, ctx, lin, launches):
    l0 = op.launch_count()
    got = list(op.step(z, ctx))
    torch.cuda.synchronize()
    assert op.launch_count() - l0 == launches
    got += list(op.layer(*lin))
    got += list(op.ar_logp(z, ctx, want_logps=True))
    got.append(op._step_train_raw(z, ctx)[3][0])  # the hidden activations the training forward keeps
    torch.cuda.synchronize()
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
@pytest.mark.parametrize("nl", NLS)
@pytest.mark.parametrize("variant", VARIANTS)
def test_one_launch_runs_equal_per_stage(variant, nl, case, monkeypatch):
    shape, B, cap, _ = case
    if cap is None:
        assert _geom(shape, B)[2] <= torch.cuda.get_device_properties(DEV).multi_processor_count
    layers, z, ctx, lin = _inputs(variant, shape, B)
    one = _outputs(_op(monkeypatch, variant, nl, shape, True, cap, layers), z, ctx, lin, 1)
    per = _outputs(_op(monkeypatch, variant, nl, shape, False, None, layers), z, ctx, lin, 2)
    assert len(one) == len(per)
    for k, (a, b) in enumerate(zip(one, per)):
        assert torch.isfinite(a).all(), k
        assert torch.equal(a, b), k


@pytest.mark.gpu
@pytest.mark.parametrize("variant", VARIANTS)
def test_captured_one_launch_step_equals_per_stage(variant, monkeypatch):
    """The step captured in a CUDA graph, replayed after its inputs change in place."""
    layers, z, ctx, _ = _inputs(variant, C2A, 256)
    one = _op(monkeypatch, variant, "elu", C2A, True, None, layers)
    per = _op(monkeypatch, variant, "elu", C2A, False, None, layers)
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
