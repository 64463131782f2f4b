"""Every parameter gradient of a whole engine step, per output channel, against a float64 replay of the oracle that follows the
engine's own ReLU, max-pool, L1, Smooth-L1 and symmetric-candidate decisions and evaluates the pose losses at the engine's
Patch-PnP outputs (tests/pinned_backward.py), on the bench.py workload and on every head and loss switch family.

What is left after pinning is backward arithmetic, so the bounds below are set by it, per channel: a wrong saved tensor or
bitmap handed to a backward launch, a weight gradient joined from the side stream too early, a loss scale removed from the wrong
segment, a wrong `unpack_wgrad` layout or bias column sum, or an fp16 activation gradient that underflows under the static loss
scale shows up in the channels it touches.  Each case also checks every BatchNorm running mean, variance and counter (43 with a
BatchNorm head, 36 with a GroupNorm one) and a per-layer forward parity of the engine's stored activations against the pinned
float64 forward, and prints the worst channel per tensor family and the decisions the float64 forward would have taken
differently.

  mixed  B = 64   module API (`model(...)`, `.backward()`, `p.grad`): the bench.py path, fp16 backward at loss scale 1024
  fp32x3 B = 64   two-plane backward: a much tighter bound
  mixed  B = 64   `engine.deterministic = False`: epilogue statistics and atomic BatchNorm-backward sums
  mixed  B = 20   a batch that is not a power of two: other tails in every batch-sized loop
  mixed  B = 64   8 surface regions (ROT_HEAD.NUM_REGIONS = 8), replayed through oracle/region_oracle.py
  mixed  B = 64   BCE and CE mask heads with other loss masks (tests/test_mask_heads_cpu.py), oracle/mask_oracle.py
  mixed  B = 64   the pose-loss switches rt_sl1, disz_l2, dist_nop_sym (tests/test_pose_losses_cpu.py; the last also fp32x3,
                  with YCB-V-like symmetries), oracle/pose_loss_oracle.py: fp16 backward at loss scale 64
  mixed  B = 64   class-aware heads all13 and mr_ce21 (tests/test_class_aware_cpu.py; the last also fp32x3) with three classes
                  absent from the batch, whose output-conv rows and bias entries must get exactly zero,
                  oracle/class_aware_oracle.py
  mixed  B = 64   the GroupNorm head ship_g32 (tests/test_head_gn_cpu.py), oracle/head_gn_oracle.py
  mixed  B = 64   DropBlock at drop_prob 0.25 on the GroupNorm, BCE, class-aware head bce_rot_g64, fed the engine's seed mask
                  (oracle/dropblock_oracle.py)
  mixed  B = 64   frozen backbone and Patch-PnP (oracle/freeze_oracle.py): only live parameters have a gradient
"""
import gc

import pytest
import torch

import pinned_backward as PB
from gdr_net_b200 import synth
from gdr_net_b200.config import a6_config
from oracle import class_aware_oracle as CA
from oracle import dropblock_oracle as DB
from oracle import freeze_oracle as FO
from oracle import gdrn_oracle as O
from oracle import head_gn_oracle as HG
from oracle import mask_oracle as M
from oracle import pose_loss_oracle as P
from oracle import region_oracle as RO
from test_regions_cpu import CASES, oracle_kwargs, region_config  # noqa: E402 (tests/ is on sys.path)
import test_class_aware_cpu as TCA  # noqa: E402
import test_head_gn_cpu as THG  # noqa: E402
import test_mask_heads_cpu as TMH  # noqa: E402
import test_pose_losses_cpu as TPL  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

# Per-channel gradient bounds (e_r of tests/pinned_backward.py): (weight rows, entries of 1-D tensors).  Measured worst over the
# five shipped-switch cases on an H100 80GB HBM3 at 700 W (the switch cases that pass reach rows 1.6e-2 (rt_sl1:
# pnp_net.fc1.weight, at loss scale 64) and 1-D 8.6e-2 (ship_g32: backbone.bn1.bias)):
#   fp32x3  rows 2.0e-3 (backbone.conv1.weight)   1-D 5.4e-3 (backbone.layer1.0.bn2.bias)
#   mixed   rows 1.4e-2 (r8: backbone.layer1.0.conv1.weight; 7.5e-3 .. 8.2e-3 in the shipped head, pnp_net.features.3.weight)
#           1-D 7.8e-2 (small entries of BatchNorm gamma / beta gradients whose tensors agree to 2e-3 rel-L2)
# The mixed row bound was 4e-2 until mr_ce21: its pnp_net.fc1.weight row 889 is a nearly dead LeakyReLU unit whose gradient is
# 7.8e-3 of the RMS row, while the one-plane fp16 backward leaves it an absolute error of 4.1e-4 of the RMS row (the median row's
# is 1.3e-4): e_r 5.3e-2.  The same case in fp32x3 has that row at 9e-5 and every row within 6.6e-4.  A scaled row (1.1) still
# gives e_r 0.1.
BOUND = {"fp32x3": (5e-3, 1.5e-2), "mixed": (6e-2, 2e-1)}
STAT_BOUND = 1e-4    # running mean / variance, in units of the step's update (momentum * batch std / variance); measured 1.4e-5
PARITY_BOUND = 1e-3  # rel-L2 of each stored activation against the pinned float64 forward; measured 7.9e-5 (rot_head_net.features.21)
LOSS_BOUND = 1e-4    # every loss against the pinned float64 one; measured 2.0e-6 (r8: loss_coor_x).  A wrong symmetric candidate
                     # for one crop of 64 moves loss_PM_R by ~1e-2


@pytest.fixture(scope="module")
def workload():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from oracle import fixtures

    return synth.seeded_state_dict(fixtures.template_from_manifest(), 0)


class Case:
    """One configuration: the model with its weights loaded, the CPU batch, the oracle forward and the modules whose `F` the
    shim replaces, the inert calls of the replay, the BatchNorm count, whether the head is GroupNorm, the parameters that
    receive a gradient and the output-conv rows no crop of the batch uses."""

    def __init__(self, model, sd, batch, fwd, modules, inert=4, n_bn=43, head_gn=False, live=None, absent=()):
        self.model, self.sd, self.batch, self.fwd, self.modules = model, sd, batch, fwd, modules
        self.inert, self.n_bn, self.head_gn, self.live, self.absent = inert, n_bn, head_gn, live, list(absent)


def _build(cfg, precision, sd=None, seed=None):
    from gdr_net_b200 import GDRN as G

    model, _ = G.build_model_optimizer(cfg, precision=precision)
    if sd is None:
        sd = synth.seeded_state_dict({k: v.cpu() for k, v in model.state_dict().items()}, seed=seed)
    model.load_state_dict(sd)
    return model, sd


def _shipped(precision, sd, B):
    model, sd = _build(a6_config(device="cuda"), precision, sd)
    fwd = lambda leaf, b: O.gdrn_forward(leaf, b, train=True, do_loss=True, update_stats=True)  # noqa: E731
    return Case(model, sd, synth.make_batch(B, seed=100), fwd, (O,), inert=0)


def _r8():
    model, sd = _build(region_config("r8", device="cuda"), "mixed", seed=CASES["r8"][2])
    kw = oracle_kwargs("r8")
    fwd = lambda leaf, b: RO.gdrn_forward(leaf, b, train=True, do_loss=True, update_stats=True, **kw)  # noqa: E731
    return Case(model, sd, synth.make_batch(64, seed=100, num_regions=8), fwd, (O, M, RO))


def _mask(case):
    switches, wseed, _ = TMH.CASES[case]
    cfg = TMH.mask_config(device="cuda", **switches)
    model, sd = _build(cfg, "mixed", seed=wseed)
    kind, gt = cfg.MODEL.CDPN.ROT_HEAD.MASK_LOSS_TYPE, TMH.mask_gt(cfg)
    fwd = lambda leaf, b: M.gdrn_forward(leaf, b, True, True, mask_loss_type=kind, mask_gt=gt, update_stats=True)  # noqa: E731
    return Case(model, sd, synth.make_batch(64, seed=100), fwd, (O, M))


def _pose(case, precision):
    switches, wseed, _, with_sym = TPL.CASES[case]
    cfg = TPL.pose_config(device="cuda", **switches)
    model, sd = _build(cfg, precision, seed=wseed)
    p, sym = cfg.MODEL.CDPN.PNP_NET, bool(switches.get("PM_LOSS_SYM"))
    fwd = lambda leaf, b: P.gdrn_forward(leaf, b, p, train=True, pm_sym=sym, update_stats=True)  # noqa: E731
    return Case(model, sd, synth.make_batch(64, seed=100, with_sym=with_sym), fwd, (O, M, P))


def _classes(n_classes, B=64):
    """Every class but the last three, in a fixed interleaved order."""
    return (torch.arange(B) * 7) % (n_classes - 3)


def _absent(n_classes, mo, R, aware, present):
    from gdr_net_b200.engine import class_rows

    rows, n = class_rows(n_classes, mo, R, *aware)
    used = {r for c in present for r in rows[c]}
    return sorted(set(range(n)) - used)


def _class_aware(case, precision):
    rh = TCA.CASES[case][0]
    model, sd = _build(TCA.case_config(case, device="cuda"), precision, seed=TCA.CASES[case][2])
    batch = synth.make_batch(64, seed=100, num_regions=rh["NUM_REGIONS"])
    batch["roi_cls"] = _classes(rh["NUM_CLASSES"])
    kw = TCA.oracle_kwargs(case)
    aware = (kw["rot_aware"], kw["mask_aware"], kw["region_aware"])
    absent = _absent(kw["num_classes"], M.mask_channels(kw["mask_loss_type"]), kw["num_regions"], aware, set(batch["roi_cls"].tolist()))
    fwd = lambda leaf, b: CA.gdrn_forward(leaf, b, True, True, update_stats=True, **kw)  # noqa: E731
    return Case(model, sd, batch, fwd, (O, M, RO), absent=absent)


def _gn(case):
    model, sd = _build(THG.case_config(case, device="cuda"), "mixed", seed=THG.CASES[case][3])
    kw = THG.oracle_kwargs(case)
    fwd = lambda leaf, b: HG.gdrn_forward(leaf, b, True, True, update_stats=True, **kw)  # noqa: E731
    return Case(model, sd, synth.make_batch(64, seed=100), fwd, (O, M, RO, HG), n_bn=36, head_gn=True)


def _dropblock_gn():
    """test_head_gn_gpu.test_dropblock_and_class_aware_with_gn at B = 64: the GroupNorm, BCE, class-aware xyz head bce_rot_g64
    with DropBlock at drop_prob 0.25 (the schedule's last step); the oracle takes the seed mask the engine drew."""
    case = "bce_rot_g64"
    _, sd = _build(THG.case_config(case, device="cuda"), "mixed", seed=THG.CASES[case][3])  # the weights of that test
    cfg = THG.case_config(case, device="cuda")
    cfg.MODEL.CDPN.PNP_NET.PNP_HEAD_CFG.drop_prob = 0.25
    model, sd = _build(cfg, "mixed", sd)
    model.pnp_net.dropblock_step = 4999
    kw = THG.oracle_kwargs(case)
    batch = synth.make_batch(64, seed=100)
    batch["roi_cls"] = _classes(13)
    pn = model.pnp_net

    def fwd(leaf, b):
        lay = dict(mo=1, R=64, region_att=True, with_2d=True, n_in=69)
        feat = O.backbone_forward(b["roi_img"], leaf, True, True)
        head = CA.select_class_maps(HG.head_forward(feat, leaf, kw["G"]), b["roi_cls"], 13, 1, 64, True, False, False)
        coor_feat, region = RO.pnp_input(head, b, lay)
        seeds = pn.dropblock_seeds.to(head.device)  # the engine's seed mask of this step
        rot6d, pred_t_ = DB.pnp_forward(coor_feat, region, b["roi_extent"].to(head.dtype), leaf, seeds, pn.dropblock_size)
        args = [b[k].to(head.dtype) for k in ("roi_cam", "roi_center", "resize_ratio", "roi_wh")]
        rot, trans = O.pose_decode_train(O.ortho6d_to_mat(rot6d), pred_t_, *args)
        return dict(losses=M.gdrn_losses(head, rot, pred_t_, b, mask_loss_type="BCE"))

    absent = _absent(13, 1, 64, (True, False, False), set(batch["roi_cls"].tolist()))
    return Case(model, sd, batch, fwd, (O, M, RO, HG, DB), inert=4 + 1, n_bn=36, head_gn=True, absent=absent)


def _frozen(case, sd):
    freeze = FO.CASES[case]
    cfg = a6_config(device="cuda")
    cfg.MODEL.CDPN.BACKBONE.FREEZE, cfg.MODEL.CDPN.ROT_HEAD.FREEZE, cfg.MODEL.CDPN.PNP_NET.FREEZE = freeze
    model, sd = _build(cfg, "mixed", sd)
    fwd = lambda leaf, b: FO.gdrn_forward(leaf, b, True, True, freeze=freeze, update_stats=True)  # noqa: E731
    inert = (33 + 1) if freeze[0] else 0  # a frozen backbone's ReLUs and max-pool run without gradient
    return Case(model, sd, synth.make_batch(64, seed=100), fwd, (O,), inert=inert, live=lambda n: FO.live(n, freeze))


CASE_IDS = ["mixed_b64", "fp32x3_b64", "mixed_b64_atomic", "mixed_b20", "r8_mixed_b64", "bce_mixed_b64", "ce_mixed_b64",
            "rt_sl1_mixed_b64", "disz_l2_mixed_b64", "dist_nop_sym_mixed_b64", "dist_nop_sym_fp32x3_b64", "all13_mixed_b64",
            "mr_ce21_mixed_b64", "mr_ce21_fp32x3_b64", "ship_g32_mixed_b64", "dropblock_gn_mixed_b64", "bb_pnp_mixed_b64"]


def _case(case, workload) -> Case:
    precision = "fp32x3" if "fp32x3" in case else "mixed"
    name = case.split("_mixed")[0].split("_fp32x3")[0]
    if case in ("mixed_b64", "fp32x3_b64", "mixed_b64_atomic", "mixed_b20"):
        return _shipped(precision, workload, 20 if case == "mixed_b20" else 64)
    if name == "r8":
        return _r8()
    if name in TMH.CASES:
        return _mask(name)
    if name in TPL.CASES:
        return _pose(name, precision)
    if name in TCA.CASES:
        return _class_aware(name, precision)
    if name in THG.CASES:
        return _gn(name)
    if name == "dropblock_gn":
        return _dropblock_gn()
    return _frozen(name, workload)


@pytest.mark.parametrize("case", CASE_IDS)
def test_pinned_gradients(workload, case):
    c = _case(case, workload)
    model, sd, batch_cpu = c.model, c.sd, c.batch
    precision = model.precision
    model.train()
    model.engine.deterministic = case != "mixed_b64_atomic"
    batch = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in batch_cpu.items()}
    for p in model.parameters():
        p.grad = None
    # the module API step, with the decisions taken between forward and backward (backward clears engine.saved)
    _, ld = model(batch["roi_img"], **synth.forward_kwargs(batch, train=True))
    pins = PB.capture(model.engine)
    sum(ld.values()).backward()
    torch.cuda.synchronize()
    params = dict(model.named_parameters())
    live = [n for n in params if c.live is None or c.live(n)]
    frozen_grads = [n for n in params if n not in live and params[n].grad is not None]
    out, leaf, shim = PB.replay(c.fwd, sd, batch_cpu, pins, c.modules)
    del pins
    gc.collect()
    ref = {n: leaf[n].grad for n in live}
    fails, table = PB.compare_grads({n: params[n].grad for n in live}, ref, *BOUND[precision])
    stats = PB.running_stat_errors(model, sd, leaf)

    tag = f"[{case}]"
    print(f"{tag} loss scale {model.engine.grad_scale:g} ({model.engine.storage_name} planes)")
    loss_rel = {}
    for k, v in ld.items():
        r = float(out["losses"][k].detach())
        loss_rel[k] = abs(float(v.detach()) - r) / abs(r)
        print(f"{tag} {k}: engine {float(v.detach()):.6f} pinned float64 {r:.6f} rel {loss_rel[k]:.1e}")
    for fam, (name, row, e, rel) in sorted(PB.worst_by_family(table, c.head_gn).items()):
        print(f"{tag} worst e_r {fam:34s} {e:.2e}  ({name} row {row}, tensor rel-L2 {rel:.1e})")
    for one_d, what in ((False, "weight row"), (True, "1-D entry")):
        sub = [t for t in table if (ref[t[0]].dim() == 1) == one_d]
        worst = max(sub, key=lambda t: t[2] if t[2] == t[2] else float("inf"))
        print(f"{tag} WORST {what}: {worst[0]} row {worst[1]}: e_r {worst[2]:.3e} (bound {BOUND[precision][one_d]:.1e})")
    flips = {s["name"]: s["flips"] for s in shim.sites if s["flips"]}
    print(f"{tag} decision flips (float64 forward vs engine): {sum(flips.values())} of {sum(s['n'] for s in shim.sites)} "
          f"decisions, per site {flips}")
    par = max((s["parity"], s["name"]) for s in shim.sites if s["parity"] is not None)
    print(f"{tag} forward parity: worst site {par[1]} rel-L2 {par[0]:.2e}; "
          + " ".join(f"{s['name'].replace('backbone.', '')}={s['parity']:.1e}" for s in shim.sites if s["parity"] is not None))
    sm = max(stats.items(), key=lambda kv: kv[1][0])
    sv = max(stats.items(), key=lambda kv: kv[1][1])
    print(f"{tag} running stats: worst mean {sm[1][0]:.2e} ({sm[0]}), worst var {sv[1][1]:.2e} ({sv[0]}) over {len(stats)} BatchNorms")

    assert list(ld) == list(out["losses"]) and max(loss_rel.values()) < LOSS_BOUND, loss_rel
    assert shim.inert == c.inert, shim.inert  # mask_oracle's pose losses call gdrn_losses on an inert head
    assert not frozen_grads, frozen_grads  # a frozen parameter keeps .grad None
    assert len(stats) == c.n_bn and all(nbt for _, _, nbt in stats.values()), stats
    if c.absent:  # rows of the class-aware output conv that no crop selects: exactly zero, in the engine and the oracle
        for w in ("weight", "bias"):
            g = params["rot_head_net.features.23." + w].grad
            assert not g[c.absent].any() and not ref["rot_head_net.features.23." + w][c.absent].any(), w
    assert not fails, f"{len(fails)} channels above {BOUND[precision]}: {fails[:10]}"
    assert sm[1][0] < STAT_BOUND and sv[1][1] < STAT_BOUND, (sm, sv)
    assert par[0] < PARITY_BOUND, par
