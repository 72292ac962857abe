"""The persistent tensor-core kernels with many tiles per CTA, in every mode and every backward kernel, against fp64.

Every tensor-core kernel is persistent.  ``iaf_ly_kernel`` (the forward, and the backward's data-gradient stages) runs
min(SMs, tiles) CTAs, CTA b taking tiles b, b + grid, b + 2 grid, ...; ``iaf_wg_kernel`` (the weight gradient) splits the
slot stream over a number of groups derived from the SM count.  What a CTA carries from one tile to the next -- the
mbarrier parities of the accumulator tile, the z window and the one-launch kernel's hidden buffer, the weight ring
position (two K passes per tile for stages of 161-192 columns), the reducer warp's double-buffered partials, the
"weights already resident" skip, the next tile's window built before this tile's epilogue -- only matters from a CTA's
second tile on.  The small batches whose fp64 reference is cheap run one tile per CTA on a 132-SM H100, so here
``IAF_NUM_SMS=n`` caps the SM count a plan schedules for: at n = 1 one CTA runs every tile, at n = 2, 3, 7 the CTAs run
uneven runs of tiles and a sample's tiles land on different CTAs (the per-sample counter and the tile-partial fold).

1. The forward of every kernel family at each cap: step, multiconv, layer and the training forward's kept activations
   against fp64, and every output bit-identical across caps (a tile's work and the tile-ordered per-sample fold do not
   depend on which CTA ran the tile).
2. The backward at each cap through the step node (kept activations), ``op.step_backward`` (recompute) and the layer
   node, with the weight gradient on the tensor cores and on SIMT: every gradient against fp64 autograd, input and data
   gradients bit-identical across caps, masked taps exactly zero.
3. The headline shapes at the benchmark batch (B = 256, 16x16) on the device's own grid: c2a is 712 tiles of the
   one-launch kernel, c2b 578 tiles per stage, over 132 CTAs.

Tolerances are those of tests/test_gpu_tc_envelope.py: forward ``|d|_inf / max(|ref|_inf, 1) <= 1e-4`` per sample, the
log-det also against the size of what it sums (``logdet_err``), backward ``|d|_inf / |ref|_inf <= 1e-4`` per tensor.
Every case asserts which kernels ran (``path_used``, ``backward_path``, the launch count) and records its worst errors
with ``record_property``."""
import numpy as np
import pytest
import torch

from oracle import iaf_oracle as O
from oracle import iaf_oracle_torch as OT
from tests import flipmask_oracle as FO
from tests.test_gpu_flipmask_envelope import (BWD_ENV, _pv, bwd_launches, check_grads, counted, ref_layer, ref_step,
                                              route_grads, route_ref, v_op)
from tests.test_gpu_tc_envelope import (DEV, LOGDET_TOL, TOL, _np, bwd_err, f64_layers, layer_inputs, logdet_err,
                                        make_params, per_sample_fwd_err)

pytestmark = pytest.mark.gpu
# SM caps: None (the device's count) first, the baseline every capped run must reproduce
CAPS = [None, 1, 2, 3, 7]


# ---------------------------------------------------------------------------------------------------------------------
# helpers.  ``variant`` is "tf", "theano" or "flip" (the Theano parameterisation with flipmask=True).
# ---------------------------------------------------------------------------------------------------------------------
def set_cap(monkeypatch, cap):
    """IAF_NUM_SMS for the plans created from here on (read once, at plan creation)."""
    if cap is None:
        monkeypatch.delenv("IAF_NUM_SMS", raising=False)
    else:
        monkeypatch.setenv("IAF_NUM_SMS", str(cap))


def num_tiles(H, W, B, one_launch):
    """Tiles of a forward call: the one-launch kernel advances 128 - MIR slots per tile, the stage kernel 128."""
    mir = (W + 2 + 7) // 8 * 8
    ts = 128 - mir if one_launch else 128
    return (B * (H + 1) * (W + 1) + ts - 1) // ts


class Worst(dict):
    """The largest error recorded under each name (over caps and configurations), for record_property."""

    def __call__(self, name, err):
        self[name] = max(self.get(name, 0.0), err)

    def record(self, record_property):
        for k in sorted(self):
            record_property(k, self[k])


def ref_multiconv(variant, zt, ct, th, thh):
    if variant == "flip":
        return FO.t_multiconv(zt, ct, th, thh)
    return OT.multiconv(variant, zt, ct, th, thh, "elu")


def ref_hiddens(variant, zt, ct, th):
    """The hidden layers' activations (what the training forward keeps for the backward), fp64."""
    out, x = [], zt
    for i, l in enumerate(th):
        if variant == "flip":
            x = FO.t_ar_conv2d(x, l, False, True)
        else:
            x = (OT.tf_ar_conv2d if variant == "tf" else OT.theano_ar_conv2d)(x, l, False)
        if i == 0:
            x = x + ct
        x = torch.nn.functional.elu(x)
        out.append(x)
    return out


def check_masked_zero(variant, gws, n_hidden):
    """Weight gradients (raw layout) of the masked taps are exactly zero; flipped heads also on their zero-diagonal
    centre rows."""
    for i, gw in enumerate(gws):
        gw = _np(gw)
        zd = i >= n_hidden
        if variant == "tf":
            mask = O.get_conv_ar_mask(3, 3, gw.shape[2], gw.shape[3], zd)
        elif variant == "theano":
            mask = O.theano_conv_ar_mask(gw.shape[1] - 1, gw.shape[0], (3, 3), zd)
        else:
            mask = FO.conv_ar_mask(gw.shape[1] - 1, gw.shape[0], zd, True)
            if zd:
                assert (gw[:FO.zero_rows(gw.shape[1] - 1, gw.shape[0]), :, 1, 1] == 0).all(), i
        assert (gw[mask == 0] == 0).all(), i


def _cid(c):
    return "%s-z%d-%s-%dx%d-b%d" % (c[0], c[1], "x".join(map(str, c[2])), c[3], c[4], c[5])


# ---------------------------------------------------------------------------------------------------------------------
# 1. forward, every kernel family x cap
# ---------------------------------------------------------------------------------------------------------------------
FWD_CASES = [
    # variant, n_z, hidden, H, W, B, launches of one call                       tiles
    ("tf", 32, [64], 16, 16, 4, 1),               # one launch (c2a's kernel)        12
    ("flip", 16, [16], 2, 2, 200, 1),             # one launch, ~13 samples a tile   15
    ("theano", 32, [64], 8, 8, 16, 1),            # one launch                       12
    ("theano", 32, [64, 64], 8, 8, 16, 3),        # per stage                        11
    ("tf", 16, [80], 16, 16, 4, 2),               # NGW 3 with a padded group        10
    ("flip", 16, [112], 8, 8, 16, 2),             # NGW 4 with a padded group        11
    ("tf", 32, [160, 160], 16, 16, 4, 3),         # c2b's kernels                    10
    ("tf", 16, [176, 176], 16, 16, 4, 3),         # streamed ring, two K passes      10
    ("flip", 16, [48, 96, 48, 16], 8, 8, 16, 5),  # four hidden layers               11
    ("theano", 32, [64, 64], 1, 1, 200, 3),       # 32 samples a tile                 7
    ("tf", 32, [64, 64], 32, 32, 2, 3),           # one sample spans ~9 tiles        18
]


@pytest.mark.parametrize("case", FWD_CASES, ids=_cid)
def test_forward_many_tiles_per_cta(case, monkeypatch, record_property):
    """Step, multiconv, layer and the training forward (its kept hidden activations) of a fresh operator per SM cap,
    each through the expected kernels and per sample within the tolerance of fp64; every output bit-identical to the
    uncapped run."""
    variant, n_z, hidden, H, W, B, launches = case
    record_property("tiles", num_tiles(H, W, B, launches == 1))
    hid, hd = make_params(_pv(variant), n_z, hidden, seed=201)
    z, ctx = O.make_inputs(B, n_z, hidden[0], H, W, seed=202)
    lin = layer_inputs(B, n_z, hidden, H, W, seed=203)
    th, thh = f64_layers(hid), f64_layers(hd)
    d = lambda a: torch.from_numpy(a).double()
    ref = {}
    with torch.no_grad():
        ref["z"], ref["arw_logsd"], ref["logdet"] = ref_step(variant, d(z), d(ctx), th, thh)
        ref["m"], ref["s"] = ref_multiconv(variant, d(z), d(ctx), th, thh)
        ref["layer.z"], ref["layer.kl"], ref["layer.kl_bc"], ref["layer.kl_cost"] = ref_layer(variant, "elu", th, thh,
                                                                                             *map(d, lin))
        for j, h in enumerate(ref_hiddens(variant, d(z), d(ctx), th)):
            ref["hidden%d" % j] = h
    t = lambda a: torch.from_numpy(a).to(DEV)
    worst = Worst()
    base = None
    for cap in CAPS:
        set_cap(monkeypatch, cap)
        op, _ = v_op(variant, n_z, hidden, "auto", hid + hd)
        for entry in ("step", "multiconv", "layer"):
            assert op.path_used(H, W, DEV, entry=entry) == "tc", (cap, entry)
        got = {}
        got["z"], got["arw_logsd"], got["logdet"] = counted(op, launches, op.step, t(z), t(ctx))
        got["m"], got["s"] = counted(op, launches, op.multiconv, t(z), t(ctx))
        got["layer.z"], got["layer.kl"], got["layer.kl_bc"], got["layer.kl_cost"] = counted(op, launches, op.layer,
                                                                                            *map(t, lin))
        zt_, ls_, ld_, hs = counted(op, launches, op._step_train_raw, t(z), t(ctx))
        assert len(hs) == len(hidden)
        for j, h in enumerate(hs):
            got["hidden%d" % j] = h
        # the training forward runs the step's kernels, writing the activations besides
        for a, b in ((zt_, got["z"]), (ls_, got["arw_logsd"]), (ld_, got["logdet"])):
            assert torch.equal(a, b), cap
        for k, r in ref.items():
            a = got[k]
            err = per_sample_fwd_err(a[:, None], r[:, None]) if a.dim() == 1 else per_sample_fwd_err(a, r)
            worst("fwd." + k, err)
            assert err < TOL, (cap, k, err)
        err = logdet_err(got["logdet"], ref["logdet"], ref["arw_logsd"])
        worst("fwd.logdet_err", err)
        assert err <= LOGDET_TOL, (cap, err)
        if base is None:
            base = got
            continue
        for k, v in got.items():
            assert torch.equal(v, base[k]), (cap, k)
    worst.record(record_property)


# ---------------------------------------------------------------------------------------------------------------------
# 2. backward x cap
# ---------------------------------------------------------------------------------------------------------------------
BWD_CASES = [
    # variant, n_z, hidden, H, W, B, launches of one forward call               data-gradient tiles
    ("tf", 32, [64], 16, 16, 4, 1),               # one-launch forward               10
    ("theano", 32, [64, 64], 8, 8, 16, 3),        # per stage                        11
    ("flip", 32, [160, 160], 16, 16, 4, 3),       # c2b's kernels                    10
    ("tf", 16, [176, 176], 16, 16, 4, 3),         # 176 columns, cin 176 > 128       10
    ("flip", 16, [48, 96, 48, 16], 8, 8, 16, 5),  # four hidden layers               11
    ("theano", 32, [64], 4, 22, 12, 1),           # W = 22: Wp + 1 = WG_HALO         11
    ("tf", 32, [64], 40, 20, 2, 1),               # cp H W 4 > 160 KB: non-fused step prologue  14
]
CONFIGS = [
    # name, environment, backward path
    ("tc", {}, "tc"),
    ("tc-dgrad", {"IAF_BWD_WG_TC": "0"}, "tc-dgrad"),
]


def route_inputs(route, B, n_z, hidden, H, W, seed):
    """(inputs, upstream gradients) of a backward route: the layer node's six inputs and four outputs, or the step's
    (z, context) and three outputs."""
    r = np.random.RandomState(seed + 1)
    shp = (B, n_z, H, W)
    if route == "layer":
        ins = list(layer_inputs(B, n_z, hidden, H, W, seed=seed))
        ups = [r.randn(*shp).astype(np.float32), r.randn(*shp).astype(np.float32), r.randn(B, n_z).astype(np.float32),
               r.randn(B).astype(np.float32)]
    else:
        ins = list(O.make_inputs(B, n_z, hidden[0], H, W, seed=seed))
        ups = [r.randn(*shp).astype(np.float32), r.randn(*shp).astype(np.float32), r.randn(B).astype(np.float32)]
    return ins, ups


@pytest.mark.parametrize("route", ["step", "recompute", "layer"])
@pytest.mark.parametrize("case", BWD_CASES, ids=_cid)
def test_backward_many_tiles_per_cta(case, route, monkeypatch, record_property):
    """One backward route with the weight gradient on the tensor cores and on SIMT, on a fresh operator per SM cap:
    the expected kernels ran, every gradient is within 1e-4 of fp64 autograd (pad-channel slices at their own scale),
    masked taps get exactly zero, input and data gradients are bit-identical across caps and parameter gradients agree
    with the uncapped run."""
    variant, n_z, hidden, H, W, B, fwd_launches = case
    hid, hd = make_params(_pv(variant), n_z, hidden, seed=211)
    ins, ups = route_inputs(route, B, n_z, hidden, H, W, seed=212)
    ref = route_ref(variant, route, ins, ups, hid, hd)
    worst = Worst()
    for combo, env, bpath in CONFIGS:
        base = None
        for cap in CAPS:
            for k in BWD_ENV:
                monkeypatch.delenv(k, raising=False)
            for k, v in env.items():
                monkeypatch.setenv(k, v)
            set_cap(monkeypatch, cap)
            op, dev = v_op(variant, n_z, hidden, "auto", hid + hd, grad=True)
            for entry in ("step", "layer"):
                assert op.path_used(H, W, DEV, entry=entry) == "tc", (combo, cap, entry)
            assert op.backward_path(H, W, DEV) == bpath, (combo, cap)
            names, got, n = route_grads(op, dev, variant, route, ins, ups)
            assert n == bwd_launches(bpath, route, n_z, hidden, H, W, fwd_launches), (combo, cap, n)
            fails = check_grads(worst, variant, list(zip(names, got, ref)), tag=combo + ".")
            assert not fails, (cap, fails)
            check_masked_zero(variant, [g for nm, g in zip(names, got) if nm.endswith((".V", ".w"))], len(hidden))
            if base is None:
                base = got
                continue
            for name, a, b in zip(names, got, base):
                if not name.startswith("layer"):
                    # the data-gradient stages run tile by tile (iaf_ly_kernel), and no tile's result depends on the CTA
                    # that ran it
                    assert torch.equal(a, b), (combo, cap, name)
                    continue
                # Parameter gradients may change in the last bits with the SM count: the weight gradient splits the
                # slot stream into split-K groups whose partials are summed in a fixed order, and how many groups
                # there are follows the SM count (iaf_wg_kernel: NG = min(groups the backward plan allows, K tiles,
                # SMs / output tiles); the SIMT weight gradient of "tc-dgrad": NG[j] = ceil(2 SMs / output tiles)).
                # Fewer groups sum the same products in a different grouping of fp32 additions.
                err = bwd_err(a, b)
                worst("%s.vs-uncapped.%s" % (combo, name), err)
                assert err <= TOL, (combo, cap, name, err)
    worst.record(record_property)


# ---------------------------------------------------------------------------------------------------------------------
# 3. the production grid: the benchmark batch on every SM
# ---------------------------------------------------------------------------------------------------------------------
PROD = [("c2a", [64], 1), ("c2b", [160, 160], 3)]


@pytest.mark.parametrize("name,hidden,launches", PROD, ids=[p[0] for p in PROD])
def test_production_grid_multiconv_layer_and_kept_activations(name, hidden, launches, monkeypatch, record_property):
    """B = 256 at 16x16 without a cap: multiconv and layer entries, and (c2a) the training forward's kept activations
    and step outputs, every sample within the tolerance of fp64."""
    monkeypatch.delenv("IAF_NUM_SMS", raising=False)
    n_z, H, W, B = 32, 16, 16, 256
    hid, hd = make_params("tf", n_z, hidden, seed=221)
    op, _ = v_op("tf", n_z, hidden, "auto", hid + hd)
    for entry in ("step", "multiconv", "layer"):
        assert op.path_used(H, W, DEV, entry=entry) == "tc", entry
    z, ctx = O.make_inputs(B, n_z, hidden[0], H, W, seed=222)
    lin = layer_inputs(B, n_z, hidden, H, W, seed=223)
    th, thh = f64_layers(hid), f64_layers(hd)
    d = lambda a: torch.from_numpy(a).double()
    t = lambda a: torch.from_numpy(a).to(DEV)
    worst = Worst()

    def chk(k, a, r):
        err = per_sample_fwd_err(a[:, None], r[:, None]) if a.dim() == 1 else per_sample_fwd_err(a, r)
        worst("prod." + k, err)
        assert err < TOL, (k, err)

    m, s = counted(op, launches, op.multiconv, t(z), t(ctx))
    with torch.no_grad():
        m_ref, s_ref = ref_multiconv("tf", d(z), d(ctx), th, thh)
    chk("m", m, m_ref)
    chk("s", s, s_ref)
    outs = counted(op, launches, op.layer, *map(t, lin))
    with torch.no_grad():
        refs = ref_layer("tf", "elu", th, thh, *map(d, lin))
    for k, a, r in zip(("layer.z", "layer.kl", "layer.kl_bc", "layer.kl_cost"), outs, refs):
        chk(k, a, r)
    if name == "c2a":
        z1, logsd, logdet, hs = counted(op, launches, op._step_train_raw, t(z), t(ctx))
        with torch.no_grad():
            z_ref, logsd_ref, logdet_ref = ref_step("tf", d(z), d(ctx), th, thh)
            h_ref = ref_hiddens("tf", d(z), d(ctx), th)[0]
        chk("z", z1, z_ref)
        chk("arw_logsd", logsd, logsd_ref)
        chk("logdet", logdet, logdet_ref)
        chk("hidden0", hs[0], h_ref)
    worst.record(record_property)


def test_production_grid_c2a_backward_through_the_step_node(monkeypatch, record_property):
    """c2a at B = 256 without a cap: every gradient of the step's autograd node (kept activations) against fp64
    autograd, masked taps exactly zero."""
    monkeypatch.delenv("IAF_NUM_SMS", raising=False)
    for k in BWD_ENV:
        monkeypatch.delenv(k, raising=False)
    n_z, hidden, H, W, B = 32, [64], 16, 16, 256
    hid, hd = make_params("tf", n_z, hidden, seed=231)
    ins, ups = route_inputs("step", B, n_z, hidden, H, W, seed=232)
    op, dev = v_op("tf", n_z, hidden, "auto", hid + hd, grad=True)
    assert op.path_used(H, W, DEV, entry="step") == "tc"
    assert op.backward_path(H, W, DEV) == "tc"
    names, got, n = route_grads(op, dev, "tf", "step", ins, ups)
    assert n == bwd_launches("tc", "step", n_z, hidden, H, W, 1), n
    ref = route_ref("tf", "step", ins, ups, hid, hd)
    worst = Worst()
    fails = check_grads(worst, "tf", list(zip(names, got, ref)), tag="prod.")
    assert not fails, fails
    check_masked_zero("tf", [g for nm, g in zip(names, got) if nm.endswith(".V")], len(hidden))
    worst.record(record_property)
