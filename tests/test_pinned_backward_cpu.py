"""The pinned float64 backward harness (tests/pinned_backward.py) without a GPU.

  * The oracle at B = 2 in float64: pins taken from its own forward, written into the engine's layouts by an encoder independent
    of the harness's decoders (numpy packbits for the NHWC ReLU bitmaps, a scan over the nine window offsets for the max-pool
    codes).  Replayed through the shim, every pin is consumed, no decision differs and the gradients and running statistics
    equal plain autograd's.
  * The decoders against hand-built cases: bit order, max-pool ties, border windows, codes that point into the padding.
  * The same at B = 2 for every other replay path (BCE / CE mask heads, the pose-loss switches with Smooth-L1, L2, MSE and
    symmetric point matching, a class-aware head, the GroupNorm head, DropBlock, a frozen backbone and Patch-PnP): every pin
    kind is consumed, no decision differs, and the gradients equal plain autograd's.  For the pose switches the loss pins are
    also built the way `capture` builds them, from fp32 outputs in the engine's layouts, and must agree with the oracle's own.
  * Hand-built Smooth-L1 residuals at |d| = beta and symmetric candidates that tie.
  * The comparator flags a planted 1 % error in one row of a 512-row tensor, which a tensor-level rel-L2 would not notice.
"""
import math
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as TF

import pinned_backward as PB
from gdr_net_b200 import synth
from oracle import class_aware_oracle as CA
from oracle import dropblock_oracle as DB
from oracle import fixtures
from oracle import freeze_oracle as FO
from oracle import gdrn_oracle as O
from oracle import head_gn_oracle as HG
from oracle import mask_oracle as M
from oracle import pose_loss_oracle as P
from oracle import region_oracle as RO
import test_class_aware_cpu as TCA  # noqa: E402 (tests/ is on sys.path)
import test_pose_losses_cpu as TPL  # noqa: E402


# ------------------------------------------------------------------------------------------------ independent encoder
def encode_bitmap(x_nchw: torch.Tensor) -> torch.Tensor:
    """[x > 0] in the engine's layout: flat NHWC element e is bit e & 7 of byte e >> 3."""
    bits = (x_nchw > 0).permute(0, 2, 3, 1).reshape(-1).numpy()
    return torch.from_numpy(np.packbits(bits, bitorder="little"))


def encode_pool(x_nchw: torch.Tensor) -> torch.Tensor:
    """uint8 NHWC window codes dy * 3 + dx of max_pool2d(x, 3, 2, 1): the first strict maximum over dy, then dx."""
    x = x_nchw.numpy()
    B, C, H, W = x.shape
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    pad = np.full((B, C, H + 2, W + 2), -np.inf)
    pad[:, :, 1:-1, 1:-1] = x
    best = np.full((B, C, Ho, Wo), -np.inf)
    code = np.zeros((B, C, Ho, Wo), np.uint8)
    for dy in range(3):
        for dx in range(3):
            v = pad[:, :, dy:dy + 2 * Ho:2, dx:dx + 2 * Wo:2]
            upd = v > best
            best = np.where(upd, v, best)
            code = np.where(upd, dy * 3 + dx, code).astype(np.uint8)
    return torch.from_numpy(np.ascontiguousarray(code.transpose(0, 2, 3, 1)))


class Recorder:
    """torch.nn.functional with the arguments of the decision calls recorded in call order (calls without gradient, which
    decide nothing, are not recorded)."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        return getattr(TF, name)

    def relu(self, x, inplace=False):
        if x.requires_grad:
            self.calls.append(("relu", x.detach().clone()))
        return TF.relu(x)

    def leaky_relu(self, x, negative_slope=0.01, inplace=False):
        self.calls.append(("leaky_relu", x.detach().clone()))
        return TF.leaky_relu(x, negative_slope)

    def linear(self, x, weight, bias=None):
        y = TF.linear(x, weight, bias)
        self.calls.append(("linear", (tuple(x.shape), y.detach().clone())))
        return y

    def max_pool2d(self, x, *a, **k):
        if x.requires_grad:
            self.calls.append(("max_pool2d", x.detach().clone()))
        return TF.max_pool2d(x, *a, **k)

    def l1_loss(self, a, b, reduction="mean", **k):
        if a.requires_grad or b.requires_grad:
            self.calls.append(("l1_loss", (a - b).detach().clone()))
        return TF.l1_loss(a, b, reduction=reduction)

    def smooth_l1_loss(self, a, b, reduction="mean", beta=1.0, **k):
        self.calls.append(("smooth_l1_loss", ((a - b).detach().clone(), beta)))
        return TF.smooth_l1_loss(a, b, reduction=reduction, beta=beta)

    def closest_rot_batch(self, pred_rots, gt_rots, sym_infos):
        self.calls.append(("closest_rot_batch", PB.closest_sym_index(pred_rots, gt_rots, sym_infos)))
        return O.closest_rot_batch(pred_rots, gt_rots, sym_infos)


def pins_from_oracle(calls, n_bitmaps=40):
    """Pins in the engine's layouts from recorded oracle calls: BatchNorm / head-norm sites (the first n_bitmaps ReLUs) as
    bitmaps, the Patch-PnP GroupNorm and LeakyReLU sites from their outputs, the max-pool as codes, the L1 calls as signs, the
    Smooth-L1 calls as branch / sign codes, the symmetric search as candidate indices."""
    pins, n_relu = [], 0
    for i, (kind, x) in enumerate(calls):
        name = f"{kind}#{i}"
        if kind == "relu" and n_relu < n_bitmaps:
            B, C, H, W = x.shape
            pins.append(PB.Pin.relu_bitmap(name, encode_bitmap(x), (B, H, W, C)))
        elif kind == "relu":
            pins.append(PB.Pin.positive("relu", name, TF.relu(x).permute(0, 2, 3, 1)))
        elif kind == "leaky_relu":
            pins.append(PB.Pin.positive("leaky_relu", name, TF.leaky_relu(x, 0.1)))
        elif kind == "max_pool2d":
            B, C, H, W = x.shape
            pins.append(PB.Pin.pool(name, encode_pool(x), (B, H, W, C)))
        elif kind == "linear":  # the rotation / translation outputs (6 and 3 wide) as values, fc1 and fc2 unpinned
            pins.append(PB.Pin.linear(name, x[0], x[1] if x[1].shape[1] <= 6 else None))
        elif kind == "smooth_l1_loss":
            pins.append(PB.Pin.smooth_l1(name, x[0], x[1]))
        elif kind == "closest_rot_batch":
            pins.append(PB.Pin.sym(name, x))
        else:
            pins.append(PB.Pin.sign(name, torch.sign(x)))
        n_relu += kind == "relu"
    return pins


def record(fwd, sd, batch, modules):
    """The plain float64 step with the decision calls recorded: (calls, result, leaf state dict)."""
    rec = Recorder()
    old = [(m, m.F) for m in modules]
    for m in modules:
        m.F = rec
    try:
        out, leaf, _ = PB.replay(fwd, sd, batch, None, modules, device="cpu")
    finally:
        for m, f in old:
            m.F = f
    return rec.calls, out, leaf


def assert_replay_is_autograd(sd, batch, fwd, modules, pins, out, leaf, inert=0):
    """The pinned replay consumes every pin, decides nothing differently and gives plain autograd's losses, gradients and
    running statistics."""
    out_p, leaf_p, shim = PB.replay(fwd, sd, batch, pins, modules, device="cpu")
    assert len(shim.sites) == len(pins) and shim.inert == inert, (len(shim.sites), len(pins), shim.inert)
    assert all(s["flips"] == 0 for s in shim.sites), [s for s in shim.sites if s["flips"]]
    assert list(out_p["losses"]) == list(out["losses"])
    for k, v in out["losses"].items():
        assert abs(float(out_p["losses"][k].detach()) - float(v.detach())) <= 1e-12 * abs(float(v)), k
    worst, worst_rel = 0.0, 0.0
    for name, t in leaf.items():
        if isinstance(t, torch.Tensor) and t.requires_grad:
            assert (leaf_p[name].grad is None) == (t.grad is None), name
            if t.grad is None:
                continue
            e, rel = PB.row_errors(leaf_p[name].grad, t.grad)
            worst, worst_rel = max(worst, float(e.max())), max(worst_rel, rel)
        elif name.endswith(("running_mean", "running_var")):
            assert float((leaf_p[name] - t).abs().max()) <= 1e-12 * float(t.abs().max()), name
        elif name.endswith("num_batches_tracked"):
            assert int(leaf_p[name]) == int(t) == int(sd[name]) + 1, name
    # measured: rel-L2 <= 4e-13 per tensor; rows whose gradient is a cancelling sum (BatchNorm, GroupNorm entries) reach 5e-10
    print(f"pinned vs plain autograd, float64 B = 2: worst rel-L2 {worst_rel:.1e}, worst per-row error {worst:.1e}")
    assert worst_rel < 2e-12 and worst < 1e-8
    return shim


@pytest.fixture(scope="module")
def oracle_b2():
    sd = fixtures.calibrated_state_dict(0)
    batch = synth.make_batch(2, seed=3)
    fwd = lambda leaf, b: O.gdrn_forward(leaf, b, train=True, do_loss=True, update_stats=True)  # noqa: E731
    calls, out, leaf = record(fwd, sd, batch, (O,))
    return sd, batch, fwd, calls, out, leaf


def test_recorded_call_order_is_the_engines(oracle_b2):
    calls = oracle_b2[3]
    kinds = [k for k, _ in calls]
    assert kinds == (["relu", "max_pool2d"] + ["relu"] * 39 + ["relu"] * 3 + ["linear", "leaky_relu"] * 2 + ["linear"] * 2
                     + ["l1_loss"] * 7)
    assert [x[1].shape for k, x in calls if k == "linear"] == [(2, 1024), (2, 256), (2, 6), (2, 3)]
    calls = [c for c in calls if c[0] != "linear"]
    shapes = [tuple(x.shape) for _, x in calls]
    assert shapes[0] == (2, 64, 128, 128) and shapes[1] == (2, 64, 128, 128) and shapes[40] == (2, 256, 64, 64) and shapes[41] == (2, 128, 32, 32)
    assert shapes[-7:-3] == [(2, 1, 64, 64)] * 3 + [(2, 64, 64)] and shapes[-2:] == [(2, 2), (2,)]
    assert shapes[-3][0] == 2 and shapes[-3][2] == 3  # point matching: [B, n, 3]


def test_pinned_replay_equals_autograd(oracle_b2):
    """Pins from the oracle's own decisions: the pinned float64 step is the plain one, to rounding."""
    sd, batch, fwd, calls, out, leaf = oracle_b2
    pins = pins_from_oracle(calls)
    assert len(pins) == 57
    assert_replay_is_autograd(sd, batch, fwd, (O,), pins, out, leaf)


def test_every_pin_must_be_consumed_and_match(oracle_b2):
    sd, batch, fwd, calls, _, _ = oracle_b2
    pins = pins_from_oracle(calls)
    with pytest.raises(AssertionError, match="not consumed"):
        PB.replay(fwd, sd, batch, pins + [PB.Pin.sign("extra", torch.zeros(2))], (O,), device="cpu")
    bad = list(pins)
    bad[3] = PB.Pin.relu_bitmap("wrong", torch.zeros(2 * 64 * 64 * 64 // 8, dtype=torch.uint8), (2, 64, 64, 32))
    with pytest.raises(AssertionError, match="shape"):
        PB.replay(fwd, sd, batch, bad, (O,), device="cpu")


def test_flipped_decisions_are_counted(oracle_b2):
    """A pin that disagrees with the float64 forward is followed, and counted."""
    sd, batch, fwd, calls, _, _ = oracle_b2
    pins = pins_from_oracle(calls)
    B, C, H, W = calls[2][1].shape
    inv = encode_bitmap(calls[2][1]) ^ 0x01  # element 0 of every byte flipped
    pins[2] = PB.Pin.relu_bitmap("flipped", inv, (B, H, W, C))
    _, _, shim = PB.replay(fwd, sd, batch, pins, (O,), device="cpu", parity=False)
    assert shim.sites[2]["flips"] == B * C * H * W // 8


# ------------------------------------------------------------------------------------------------ the other replay paths
def _seeded(rot_head=None, pnp_net=None, seed=0):
    """Seeded weights (synth.seeded_state_dict) of the model build_model_optimizer makes with these switches."""
    from gdr_net_b200 import GDRN as G
    from gdr_net_b200.config import a6_config

    cfg = a6_config(device="cpu")
    for k, v in (rot_head or {}).items():
        setattr(cfg.MODEL.CDPN.ROT_HEAD, k, v)
    for k, v in (pnp_net or {}).items():
        setattr(cfg.MODEL.CDPN.PNP_NET, k, v)
    model, _ = G.build_model_optimizer(cfg)
    return synth.seeded_state_dict(model.state_dict(), seed=seed), cfg


def _sym_batch():
    """Two crops whose objects are symmetric: a four-fold and a discretised continuous axis."""
    batch = synth.make_batch(2, seed=3)
    batch["sym_info"] = [synth.discrete_symmetries("z4"), synth.discrete_symmetries("cont")]
    return batch


POSE = {k: TPL.CASES[k][0] for k in ("rt_sl1", "disz_l2", "dist_nop_sym")}
POSE["rt_l1_trans"] = dict(PM_R_ONLY=False, PM_DISENTANGLE_T=True, PM_T_USE_POINTS=True, PM_LOSS_TYPE="L1", TRANS_LW=1.0,
                           TRANS_LOSS_TYPE="L1", TRANS_LOSS_DISENTANGLE=False)  # L1 point matching with points, L1 translation


def _path(name):
    """(state dict, batch, forward, oracle modules, bitmap sites, inert calls, pose config or None) of one replay path."""
    sd0 = fixtures.calibrated_state_dict(0)
    batch = synth.make_batch(2, seed=3)
    if name in ("bce", "ce"):
        kind = name.upper()
        sd = _seeded({"MASK_LOSS_TYPE": "CE"}, seed=6)[0] if kind == "CE" else sd0
        gt = ("obj", "visib", "visib") if kind == "BCE" else ("visib", "obj", "trunc")  # test_mask_heads_cpu.CASES
        fwd = lambda leaf, b: M.gdrn_forward(leaf, b, True, True, mask_loss_type=kind, mask_gt=gt, update_stats=True)  # noqa: E731
        return sd, batch, fwd, (O, M), 40, 4, None
    if name in POSE:
        p = TPL.pose_config(**POSE[name]).MODEL.CDPN.PNP_NET
        sym = bool(POSE[name].get("PM_LOSS_SYM"))
        fwd = lambda leaf, b: P.gdrn_forward(leaf, b, p, train=True, pm_sym=sym, update_stats=True)  # noqa: E731
        return sd0, (_sym_batch() if sym else batch), fwd, (O, M, P), 40, 4, p
    if name == "all13":
        sd = _seeded(dict(NUM_CLASSES=13, ROT_CLASS_AWARE=True, MASK_CLASS_AWARE=True, REGION_CLASS_AWARE=True), seed=51)[0]
        batch["roi_cls"] = torch.tensor([3, 12])
        kw = dict(num_classes=13, rot_aware=True, mask_aware=True, region_aware=True, num_regions=64)
        fwd = lambda leaf, b: CA.gdrn_forward(leaf, b, True, True, update_stats=True, **kw)  # noqa: E731
        return sd, batch, fwd, (O, M, RO), 40, 4, None
    if name == "mr_ce21":  # CE mask head, class-aware mask and region blocks, 8 regions
        sd = TCA.seeded_weights(name)
        batch = synth.make_batch(2, seed=3, num_regions=8)
        batch["roi_cls"] = torch.tensor([5, 20])
        kw = TCA.oracle_kwargs(name)
        fwd = lambda leaf, b: CA.gdrn_forward(leaf, b, True, True, update_stats=True, **kw)  # noqa: E731
        return sd, batch, fwd, (O, M, RO), 40, 4, None
    if name == "gn":
        sd = _seeded(dict(NORM="GN", NUM_GN_GROUPS=32), seed=71)[0]
        fwd = lambda leaf, b: HG.gdrn_forward(leaf, b, True, True, G=32, update_stats=True)  # noqa: E731
        return sd, batch, fwd, (O, M, RO, HG), 40, 4, None
    if name == "dropblock":
        seeds = (torch.rand(2, 64, 64, generator=torch.Generator().manual_seed(5)) < 0.25 / 25).float()
        fwd = lambda leaf, b: DB.gdrn_forward(leaf, b, True, True, seeds=seeds, block_size=5, update_stats=True)  # noqa: E731
        return sd0, batch, fwd, (O, M, RO, DB), 40, 5, None  # + DropBlock's max-pool over the seed mask
    if name == "bb_pnp":
        fwd = lambda leaf, b: FO.gdrn_forward(leaf, b, True, True, freeze=FO.CASES["bb_pnp"], update_stats=True)  # noqa: E731
        return sd0, batch, fwd, (O,), 7, 33 + 1, None  # the frozen backbone's 33 ReLUs and its max-pool
    raise KeyError(name)


PATHS = ["bce", "ce", "rt_sl1", "disz_l2", "dist_nop_sym", "rt_l1_trans", "all13", "mr_ce21", "gn", "dropblock", "bb_pnp"]
LOSS_KINDS = {  # the decision calls of the loss terms, in order (the shipped pose terms that pose_loss_oracle drops included)
    "bce": ["l1_loss"] * 3 + ["l1_loss"] * 3,
    "ce": ["l1_loss"] * 3 + ["l1_loss"] * 3,
    "mr_ce21": ["l1_loss"] * 3 + ["l1_loss"] * 3,
    "rt_sl1": ["l1_loss"] * 7 + ["smooth_l1_loss", "l1_loss", "l1_loss", "l1_loss"],      # PM_RT, centroid, z, bind
    "disz_l2": ["l1_loss"] * 7,                                                               # all smooth
    "dist_nop_sym": ["l1_loss"] * 7 + ["closest_rot_batch", "l1_loss", "l1_loss", "l1_loss"],  # centroid, z, bind
    "rt_l1_trans": ["l1_loss"] * 7 + ["l1_loss"] * 5,                                        # PM_R, PM_T, centroid, z, LPnP
}


@pytest.mark.parametrize("name", PATHS)
def test_every_replay_path_equals_autograd(name):
    sd, batch, fwd, modules, n_bitmaps, inert, _ = _path(name)
    calls, out, leaf = record(fwd, sd, batch, modules)
    kinds = [k for k, _ in calls]
    assert kinds.count("relu") == n_bitmaps + 3 and kinds.count("max_pool2d") == (n_bitmaps == 40)
    if name in LOSS_KINDS:
        assert kinds[n_bitmaps + 10:] == LOSS_KINDS[name], kinds[n_bitmaps + 10:]
    if name == "dist_nop_sym":
        idx = [x for k, x in calls if k == "closest_rot_batch"][0]
        assert (idx >= 0).any(), idx  # a symmetric candidate is taken
    if name == "rt_sl1":
        d, beta = [x for k, x in calls if k == "smooth_l1_loss"][0]
        inner = (d.abs() < beta).float().mean()
        assert 0 < inner < 1, inner  # both branches are exercised
    shim = assert_replay_is_autograd(sd, batch, fwd, modules, pins_from_oracle(calls, n_bitmaps), out, leaf, inert)
    if name == "bb_pnp":
        for k, t in leaf.items():
            if isinstance(t, torch.Tensor) and t.requires_grad:
                assert (t.grad is not None) == FO.live(k, FO.CASES["bb_pnp"]), k
    assert {s["kind"] for s in shim.sites} >= set(kinds)


def _engine_like(out, batch, p):
    """An object with the attributes loss_sign_pins reads, holding the oracle's outputs in fp32 and the engine's layouts."""
    B = batch["roi_img"].shape[0]
    head = out["head"].detach().float()
    logits = torch.zeros(B, 64, 64, 72)
    logits[..., :head.shape[1]] = head.permute(0, 2, 3, 1)
    pred = torch.zeros(B, 16)
    pred[:, :6], pred[:, 6:9] = out["rot6d"].detach().float(), out["pred_t_"].detach().float()
    f = lambda k: batch[k].float()  # noqa: E731
    aux = dict(gt_mask_visib=f("roi_mask_visib"), gt_mask_trunc=f("roi_mask_trunc"), gt_mask_obj=f("roi_mask_obj"),
               gt_xyz=f("roi_xyz"), gt_ego_rot=f("ego_rot"), gt_points=f("roi_points"), roi_extents=f("roi_extent"),
               gt_trans=f("trans"), gt_trans_ratio=f("roi_trans_ratio"))
    table = torch.zeros(0, 3, 3)
    if p is not None and p.PM_LOSS_SYM:
        sets = batch["sym_info"]
        counts = [0 if s is None else s.shape[0] for s in sets]
        table = torch.cat([s for s in sets if s is not None])
        aux["sym_idx"] = torch.tensor([[sum(counts[:b]), counts[b]] for b in range(B)], dtype=torch.int32)
    S = dict(B=B, aux=aux, logits=logits.view(-1, 72), out_rot=out["rot"].detach().float(), out_trans=out["trans"].detach().float(),
             pred=pred)
    cfg = types.SimpleNamespace(MODEL=types.SimpleNamespace(CDPN=types.SimpleNamespace(PNP_NET=p)))
    return types.SimpleNamespace(saved=S, mask_out=1, mask_loss=0, mask_gt=M.DEFAULT_MASK_GT, live_head=True, pose_ex=p is not None,
                                 model=types.SimpleNamespace(cfg=cfg, pnp_net=types.SimpleNamespace(fc_r=types.SimpleNamespace(out_features=6))),
                                 sym_table=types.SimpleNamespace(table=table))


@pytest.mark.parametrize("name", [n for n in PATHS if n in POSE])
def test_loss_pins_from_fp32_outputs_agree_with_the_oracle(name):
    """The loss pins `capture` forms from the engine's fp32 outputs (loss_sign_pins, pose_pins, sym_choice) follow the pose
    oracle's call order and shapes and take its decisions: replayed with the network's pins from the oracle, every pin is
    consumed, nothing flips and the gradients are plain autograd's."""
    sd, batch, fwd, modules, n_bitmaps, inert, p = _path(name)
    calls, out, leaf = record(fwd, sd, batch, modules)
    n_net = sum(k in ("relu", "max_pool2d", "leaky_relu", "linear") for k, _ in calls)
    eng = _engine_like(out, batch, p)
    loss_pins = PB.loss_sign_pins(eng, eng.saved)
    assert [q.kind for q in loss_pins] == [k for k, _ in calls[n_net:]]
    assert_replay_is_autograd(sd, batch, fwd, modules, pins_from_oracle(calls, n_bitmaps)[:n_net] + loss_pins, out, leaf, inert)


def test_capture_refuses_switches_without_a_pin():
    from gdr_net_b200.config import a6_config

    cfg = a6_config(device="cpu")
    cfg.MODEL.CDPN.PNP_NET.PM_LOSS_TYPE, cfg.MODEL.CDPN.PNP_NET.PM_SMOOTH_L1_BETA = "Smooth_L1", 1e-6
    eng = types.SimpleNamespace(saved=dict(aux={}), pose_ex=True, model=types.SimpleNamespace(cfg=cfg))
    with pytest.raises(NotImplementedError, match="beta"):
        PB.capture(eng)
    eng = types.SimpleNamespace(saved=dict(aux=dict(sym_idx=torch.zeros(2, 2))), pose_ex=False, model=types.SimpleNamespace(cfg=a6_config(device="cpu")))
    with pytest.raises(NotImplementedError, match="symmetric"):
        PB.capture(eng)


# ------------------------------------------------------------------------------------------------ pin kinds, hand-built
def test_smooth_l1_branch_at_beta():
    """|d| = beta is the linear branch for the kernel and torch (|d| < beta is quadratic); both branches give the same value
    and gradient there, so a pin taking the other branch is counted but changes nothing."""
    beta = 0.5
    d = torch.tensor([0.5, -0.5, 0.25, -1.5, 0.0, 0.4999999], dtype=torch.float64)
    q = PB.Pin.smooth_l1("sl1", d, beta).decide("cpu")
    assert q.tolist() == [1.0, -1.0, 0.0, -1.0, 0.0, 0.0]
    for pin, flips in ((PB.Pin.smooth_l1("sl1", d, beta), 0), (PB.Pin.smooth_l1("wide", d, 0.6), 2)):
        a = d.clone().requires_grad_(True)
        shim = PB.PinnedF([pin])
        v = shim.smooth_l1_loss(a, torch.zeros_like(d), reduction="mean", beta=beta)
        v.backward()
        b = d.clone().requires_grad_(True)
        ref = TF.smooth_l1_loss(b, torch.zeros_like(d), reduction="mean", beta=beta)
        ref.backward()
        assert abs(float(v) - float(ref)) <= 1e-16 and torch.allclose(a.grad, b.grad, rtol=0, atol=1e-16), (pin.name, a.grad, b.grad)
        assert shim.sites[0]["flips"] == flips
        shim.finish()


def _rz(a):
    c, s = math.cos(a), math.sin(a)
    return torch.tensor([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]], dtype=torch.float64)


def test_symmetric_ties():
    """A candidate that ties the unmodified R_gt loses to it; of two equal candidates the first is taken -- in the oracle's
    float64 search, in the restatement of the pose kernel's fp32 one, and the shim follows its pin and counts a different
    (equal-valued) choice as a flip."""
    Rg = _rz(0.3) @ torch.tensor([[1.0, 0.0, 0.0], [0.0, 0.0, -1.0], [0.0, 1.0, 0.0]], dtype=torch.float64)
    quarter = _rz(math.pi / 2)
    sets = [torch.stack([torch.eye(3), _rz(math.pi)]).float(),          # crop 0: R = R_gt, identity candidate ties it
            torch.stack([_rz(math.pi), quarter, quarter]).float()]      # crop 1: R = R_gt Rz(pi/2), candidates 1 and 2 tie
    R = torch.stack([Rg, Rg @ quarter])
    Rgs = torch.stack([Rg, Rg])
    want = torch.tensor([-1, 1])
    assert torch.equal(PB.closest_sym_index(R, Rgs, sets), want)
    table = torch.cat(sets)
    sym_idx = torch.tensor([[0, 2], [2, 3]], dtype=torch.int32)
    assert torch.equal(PB.sym_choice(R.float(), Rgs.float(), table, sym_idx), want)
    assert torch.allclose(O.closest_rot_batch(R, Rgs, sets), Rgs @ torch.stack([torch.eye(3, dtype=torch.float64), quarter]), rtol=0, atol=1e-7)
    for pin_idx, flips in ((want, 0), (torch.tensor([-1, 2]), 1)):
        shim = PB.PinnedF([PB.Pin.sym("sym", pin_idx)])
        out = shim.closest_rot_batch(R, Rgs, sets)
        assert torch.allclose(out, O.closest_rot_batch(R, Rgs, sets), rtol=0, atol=1e-7) and shim.sites[0]["flips"] == flips
        shim.finish()


# ------------------------------------------------------------------------------------------------ decoders, hand-built
def test_bitmap_bit_order():
    # NHWC [1, 2, 2, 4]: flat e = ((h * 2) + w) * 4 + c; set e = 2, 9 and 15
    bits = torch.tensor([0b00000100, 0b10000010], dtype=torch.uint8)
    m = PB.unpack_bitmap(bits, (1, 2, 2, 4))
    assert m.shape == (1, 4, 2, 2)
    on = {tuple(i) for i in m.nonzero().tolist()}
    # e = 2 -> h 0 w 0 c 2;  e = 9 -> h 1 w 0 c 1;  e = 15 -> h 1 w 1 c 3
    assert on == {(0, 2, 0, 0), (0, 1, 1, 0), (0, 3, 1, 1)}
    x = torch.randn(2, 16, 5, 8, dtype=torch.float64)
    assert torch.equal(PB.unpack_bitmap(encode_bitmap(x), (2, 5, 8, 16)), x > 0)


def test_pool_codes_ties_and_borders():
    x = torch.tensor([[[[1.0, 5.0, 5.0, 0.0],
                        [5.0, 2.0, 0.0, 0.0],
                        [3.0, 3.0, 3.0, 3.0],
                        [0.0, 0.0, 7.0, 7.0]]]], dtype=torch.float64)
    # windows start at (2 oy - 1, 2 ox - 1); row dy = 0 / column dx = 0 of the top / left windows are padding
    # (0,0): rows -1..1, cols -1..1: max 5 at (0,1) and (1,0) -> first is (0,1): dy 1 dx 2 -> 5
    # (0,1): rows -1..1, cols 1..3: 5 at (0,1) and (0,2) -> (0,1): dy 1 dx 0 -> 3
    # (1,0): rows 1..3, cols -1..1: 5 at (1,0): dy 0 dx 1 -> 1
    # (1,1): rows 1..3, cols 1..3: 7 at (3,2) and (3,3) -> (3,2): dy 2 dx 1 -> 7
    want = torch.tensor([[[[5, 3], [1, 7]]]])
    arg = encode_pool(x)
    assert torch.equal(arg.permute(0, 3, 1, 2).long(), want)
    assert torch.equal(PB.first_max_codes(x), want)
    xg = x.clone().requires_grad_(True)
    y = PB.pool_gather(xg, PB.pool_codes(arg))
    assert torch.equal(y.detach(), TF.max_pool2d(x, 3, 2, 1))
    y.sum().backward()
    g = torch.zeros_like(x)
    g[0, 0, 0, 1] = 2.0  # chosen by two windows
    g[0, 0, 1, 0] = 1.0
    g[0, 0, 3, 2] = 1.0
    assert torch.equal(xg.grad, g)
    with pytest.raises(AssertionError, match="padding"):
        PB.pool_gather(x, torch.tensor([[[[0, 3], [1, 7]]]]))  # code 0 of window (0,0) is the padded corner


def test_pool_codes_random_against_torch():
    x = torch.randn(2, 8, 9, 12, dtype=torch.float64)
    x[0, 0, :4, :4] = 0.0  # ties
    codes = PB.pool_codes(encode_pool(x))
    assert torch.equal(codes, PB.first_max_codes(x))
    assert torch.equal(PB.pool_gather(x, codes), TF.max_pool2d(x, 3, 2, 1))


# ------------------------------------------------------------------------------------------------ comparator
def test_comparator_flags_one_row_at_one_percent():
    g = torch.Generator().manual_seed(0)
    ref = torch.randn(512, 256, 3, 3, generator=g, dtype=torch.float64)
    noisy = ref + 1e-4 * ref.flatten(1).norm(dim=1).view(-1, 1, 1, 1) / 48 * torch.randn(ref.shape, generator=g, dtype=torch.float64)
    fails, table = PB.compare_grads({"w": noisy}, {"w": ref}, 5e-3)
    assert not fails and table[0][2] < 2e-4
    bad = noisy.clone()
    d = torch.randn(256, 3, 3, generator=g, dtype=torch.float64)
    bad[137] += 0.01 * ref[137].norm() * d / d.norm()
    fails, table = PB.compare_grads({"w": bad}, {"w": ref}, 5e-3)
    assert [f[:2] for f in fails] == [("w", 137)] and 0.009 < fails[0][2] < 0.011
    assert table[0][3] < 1e-3  # the tensor-level rel-L2 of the same error: 0.01 / sqrt(512)
    nan = noisy.clone()
    nan[3, 0, 0, 0] = float("nan")
    assert [f[:2] for f in PB.compare_grads({"w": nan}, {"w": ref}, 5e-3)[0]] == [("w", 3)]


def test_comparator_floor_and_one_d():
    ref = torch.tensor([1.0, 1e-9, -2.0, 0.0], dtype=torch.float64)
    got = ref + torch.tensor([0.0, 1e-9, 0.0, 1e-7], dtype=torch.float64)
    e, rel = PB.row_errors(got, ref)
    floor = 1e-3 * float(ref.norm()) / 2
    assert torch.allclose(e, torch.tensor([0.0, 1e-9 / floor, 0.0, 1e-7 / floor], dtype=torch.float64))
    # with a 1-D bound the entries are measured against 0.1 of the RMS entry: a 2 % error of a typical entry is flagged, the
    # same absolute error on an entry that is 1e-3 of the RMS one is not
    g = torch.Generator().manual_seed(1)
    ref = torch.randn(128, generator=g, dtype=torch.float64)
    ref[7] = 1e-3 * ref.norm() / 128 ** 0.5
    got = ref.clone()
    got[7] += 0.002 * ref.norm() / 128 ** 0.5  # e_r 0.02 against 0.1 of the RMS entry
    assert not PB.compare_grads({"b": got}, {"b": ref}, 1e-3, 0.05)[0]
    assert PB.compare_grads({"b": got}, {"b": ref}, 1e-3)[0]  # against the row floor it would be
    ref[3] = ref.norm() / 128 ** 0.5
    got = ref.clone()
    got[3] *= 1.02
    assert [f[:2] for f in PB.compare_grads({"b": got}, {"b": ref}, 1e-3, 1e-2)[0]] == [("b", 3)]


def test_family_names():
    assert PB.family("backbone.conv1.weight") == "backbone.stem/conv.weight"
    assert PB.family("backbone.bn1.bias") == "backbone.stem/bn.bias"
    assert PB.family("backbone.layer3.1.bn2.weight") == "backbone.layer3/bn.weight"
    assert PB.family("backbone.layer2.0.downsample.1.weight") == "backbone.layer2/bn.weight"
    assert PB.family("backbone.layer2.0.downsample.0.weight") == "backbone.layer2/conv.weight"
    assert PB.family("rot_head_net.features.21.weight") == "rot_head_net/bn.weight"
    assert PB.family("rot_head_net.features.23.bias") == "rot_head_net/conv.bias"
    assert PB.family("pnp_net.features.4.bias") == "pnp_net/gn.bias"
    assert PB.family("pnp_net.fc_r.weight") == "pnp_net/fc.weight"
    assert PB.family("rot_head_net.features.21.weight", head_gn=True) == "rot_head_net/gn.weight"
    assert PB.family("rot_head_net.features.1.bias", head_gn=True) == "rot_head_net/gn.bias"
    assert PB.family("rot_head_net.features.20.weight", head_gn=True) == "rot_head_net/conv.weight"
