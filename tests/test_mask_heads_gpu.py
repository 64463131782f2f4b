"""GPU: the BCE and CE mask heads and selectable loss masks through the whole model (ROT_HEAD.MASK_LOSS_TYPE, XYZ_LOSS_MASK_GT,
MASK_LOSS_GT, REGION_LOSS_MASK_GT; GDRN.py:339-400) and the CE head at test time (mask_mode 3 of csrc/pnp_ransac.cu).

  * the two configurations of tests/golden/train_mask_{bce,ce}_b4.npz (the unmodified reference with only those switches changed)
    at B = 4 against the golden and the oracle, and at B = 64 in "mixed" against the oracle, with the bounds of
    tests/test_parity_b64_gpu.py;
  * the captured train step replays to the eager result bit for bit, and two runs are bit-identical (deterministic mode);
  * the test-mode maps of a CE head carry a [B, 2, 64, 64] mask;
  * `process_pnp` with a CE head selects exactly the reference's points (tests/golden/pnp_ce_select_b3.npz, exact z0 == z1 ties
    included) and matches cv2 like the existing RANSAC and iterative tests."""
import os
import types

import numpy as np
import pytest
import torch

from gdr_net_b200 import synth
from oracle import gdrn_oracle as O
from oracle import mask_oracle as M

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

REL = 1e-3
CASES = {  # as oracle/make_golden_masks.py
    "bce": (dict(MASK_LOSS_TYPE="BCE", MASK_LOSS_GT="visib", XYZ_LOSS_MASK_GT="obj"), 5, 23),
    "ce": (dict(MASK_LOSS_TYPE="CE", MASK_LOSS_GT="obj", REGION_LOSS_MASK_GT="trunc"), 6, 29),
}


@pytest.fixture(scope="module", autouse=True)
def _gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _cfg(case, device="cuda", **kw):
    from gdr_net_b200.config import a6_config

    cfg = a6_config(device=device, **kw)
    for k, v in CASES[case][0].items():
        setattr(cfg.MODEL.CDPN.ROT_HEAD, k, v)
    return cfg


def _mask_gt(cfg):
    r = cfg.MODEL.CDPN.ROT_HEAD
    return (r.XYZ_LOSS_MASK_GT, r.MASK_LOSS_GT, r.REGION_LOSS_MASK_GT)


def _model(case, sd=None, precision="mixed", **kw):
    from gdr_net_b200 import GDRN as G

    model, _ = G.build_model_optimizer(_cfg(case, **kw), precision=precision)
    if sd is None:
        sd = synth.seeded_state_dict({k: v.cpu() for k, v in model.state_dict().items()}, seed=CASES[case][1])
    model.load_state_dict(sd)
    return model, sd


def _cuda(batch):
    return {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in batch.items()}


def _train_step(model, batch):
    for p in model.parameters():
        p.grad = None
    _, ld = model(batch["roi_img"], **synth.forward_kwargs(batch, train=True))
    sum(ld.values()).backward()
    torch.cuda.synchronize()
    return {k: float(v.detach()) for k, v in ld.items()}


@pytest.mark.parametrize("case", sorted(CASES))
def test_b4_matches_golden_and_oracle(case, golden_dir):
    g = np.load(os.path.join(golden_dir, f"train_mask_{case}_b4.npz"))
    model, sd = _model(case)
    mlt = CASES[case][0]["MASK_LOSS_TYPE"]
    assert model.engine.mask_out == M.mask_channels(mlt)
    batch_cpu = synth.make_batch(4, seed=CASES[case][2])
    batch = _cuda(batch_cpu)
    model.train()
    ld = _train_step(model, batch)
    leaf = O.leaf_state_dict(sd)
    o = M.gdrn_forward(leaf, batch_cpu, train=True, do_loss=True, mask_loss_type=mlt, mask_gt=_mask_gt(_cfg(case)), update_stats=True)
    sum(o["losses"].values()).backward()
    # seeded (not calibrated) weights: the bound of test_parity_b64_gpu.py::test_nin67_without_2d_coords_matches_oracle, which
    # uses the same kind of weights; measured on an H100: loss_PM_R of the BCE case 1.5e-3, every other loss <= 1.1e-5
    for k, v in ld.items():
        ref = float(g["loss/" + k])
        print(f"[{case}] B=4 {k}: {v:.6f} vs golden {ref:.6f} rel {abs(v - ref) / abs(ref):.2e}")
        assert abs(v - ref) <= 2 * REL * abs(ref), (k, v, ref)
        assert abs(v - float(o["losses"][k])) <= 2 * REL * abs(ref), k
    params = dict(model.named_parameters())
    for key in g.files:
        if key.startswith("grad/"):
            name = key[len("grad/"):]
            r_g, r_o = _rel(params[name].grad, g[key]), _rel(params[name].grad, leaf[name].grad)
            print(f"[{case}] grad {name}: rel-L2 vs golden {r_g:.2e}, vs oracle {r_o:.2e}")
            # the bound of test_parity_b64_gpu.py's gradient checks; measured: BCE <= 5.8e-2 (the forward's point-matching L1
            # decisions differ, as the 1.5e-3 of loss_PM_R shows, and move every gradient), CE <= 2.1e-2
            assert r_g < 0.06 and r_o < 0.06, (name, r_g, r_o)
    # eval mode, TEST.USE_PNP maps: the head against the golden (every 4th pixel), the mask carries MO channels
    model, _ = _model(case, sd=sd, use_pnp_test=True)
    model.eval()
    with torch.no_grad():
        out = model(batch["roi_img"], **synth.forward_kwargs(batch, train=False))
    mo = M.mask_channels(mlt)
    assert tuple(out["mask"].shape) == (4, mo, 64, 64) and tuple(out["region"].shape) == (4, 65, 64, 64)
    head = torch.cat([out["mask"], out["coor_x"], out["coor_y"], out["coor_z"], out["region"]], dim=1)[:, :, ::4, ::4].cpu()
    r = _rel(head, g["eval/head"])
    print(f"[{case}] eval head rel-L2 vs golden {r:.2e}, rot {_rel(out['rot'], g['eval/rot']):.2e}, trans {_rel(out['trans'], g['eval/trans']):.2e}")
    assert r < REL and _rel(out["rot"], g["eval/rot"]) < 2e-3 and _rel(out["trans"], g["eval/trans"]) < 2e-3  # measured 5.5e-5, 2.9e-5, 2.5e-5


@pytest.mark.parametrize("case", sorted(CASES))
def test_b64_mixed_matches_oracle(case):
    """The benchmark's batch (B = 64, seed 100) in the headline "mixed" mode: all 8 losses and the head within 1e-3 of the oracle."""
    from gdr_net_b200.engine import LOSS_NAMES

    model, sd = _model(case)
    mlt = CASES[case][0]["MASK_LOSS_TYPE"]
    batch_cpu = synth.make_batch(64, seed=100)
    with torch.no_grad():
        o = M.gdrn_forward(O.leaf_state_dict(sd, requires_grad=False), batch_cpu, train=True, do_loss=True, mask_loss_type=mlt,
                           mask_gt=_mask_gt(_cfg(case)))
    model.train()
    batch = _cuda(batch_cpu)
    ld = _train_step(model, batch)
    for k in LOSS_NAMES:
        ref = float(o["losses"][k])
        print(f"[{case}] B=64 {k}: {ld[k]:.6f} vs {ref:.6f} rel {abs(ld[k] - ref) / abs(ref):.2e}")
        assert abs(ld[k] - ref) <= REL * abs(ref), (k, ld[k], ref)  # measured <= 2.8e-5 (loss_PM_R, BCE)
    assert all(torch.isfinite(p.grad).all() for p in model.parameters())


@pytest.mark.parametrize("case", sorted(CASES))
def test_graph_replay_equals_eager_and_runs_are_bit_identical(case):
    """Deterministic mode, as tests/test_parity_b64_gpu.py::test_deterministic_mode_is_bit_reproducible_and_graph_equals_eager:
    losses and the gradients of parameters that are not atomically summed (bias and GroupNorm entries are) are bit-identical.
    The 7x7 stem's gradient is left out: with these seeded, uncalibrated weights its fp16 backward overflows in the default L1
    configuration as well (NaN, which no comparison equals)."""
    batch = _cuda(synth.make_batch(4, seed=CASES[case][2]))
    runs = []
    sd = None
    for graphs in (False, False, True):
        model, sd = _model(case, sd=sd)
        model.train()
        model.engine.deterministic = True
        model.use_cuda_graphs = graphs
        for _ in range(2):  # the second step replays when graphs are on
            ld = _train_step(model, batch)
        p = dict(model.named_parameters())
        runs.append((ld, {n: p[n].grad.clone() for n in ("rot_head_net.features.23.weight", "rot_head_net.features.20.weight",
                                                        "backbone.layer1.0.conv1.weight", "pnp_net.features.0.weight")}))
    for other in runs[1:]:
        assert other[0] == runs[0][0]
        for n, v in runs[0][1].items():
            assert torch.equal(other[1][n], v), n


# ------------------------------------------------------------------------------------------------ test time: CE mask head
def _ce_inputs(golden_dir):
    g = np.load(os.path.join(golden_dir, "pnp_ce_select_b3.npz"))
    d = {k: torch.from_numpy(g[k]) for k in ("mask", "xyz", "coord_2d", "extents", "im_wh", "cams", "R", "t")}
    return g, d


def _pnp_cfg(pnp_type):
    rh = types.SimpleNamespace(MASK_LOSS_TYPE="CE", MASK_THR_TEST=0.5)
    return types.SimpleNamespace(TEST=types.SimpleNamespace(PNP_TYPE=pnp_type), MODEL=types.SimpleNamespace(CDPN=types.SimpleNamespace(ROT_HEAD=rh)))


def test_ce_head_ransac_selects_reference_points_and_matches_cv2(golden_dir):
    import pnp_common
    from gdr_net_b200.pnp_ransac import pnp_ransac, process_pnp
    from oracle import pnp_oracle as PO

    pytest.importorskip("cv2")
    g, d = _ce_inputs(golden_dir)
    B = d["mask"].shape[0]
    c = lambda t: t.cuda()  # noqa: E731
    res = pnp_ransac(c(d["mask"]), c(d["xyz"]), c(d["coord_2d"]), c(d["extents"]), c(d["im_wh"]), c(d["cams"]), mask_loss_type="CE",
                     return_inliers=True)
    torch.cuda.synchronize()
    info = torch.stack([res["num_points"], res["num_inliers"], res["iterations"], res["ok"].int()], dim=1).cpu().numpy()
    ref = []
    for b in range(B):
        ip, mp = g[f"img_points_{b}"], g[f"model_points_{b}"]
        pose, inl = PO.pnp_ransac_cv2(mp, ip, d["cams"][b].numpy())
        ref.append((ip, mp, pose, inl))
    pnp_common.check_against_reference(d, ref, res["pose"].cpu().numpy(), info, res["inliers"].cpu().numpy())
    # process_pnp(cfg): the model's two-channel mask passes through; translation from the network
    out_dict = dict(mask=c(d["mask"]), coor_x=c(d["xyz"][:, 0:1]), coor_y=c(d["xyz"][:, 1:2]), coor_z=c(d["xyz"][:, 2:3]),
                    rot=c(d["R"]), trans=c(d["t"]) + 0.01)
    pose = process_pnp(_pnp_cfg("ransac_pnp"), out_dict, c(d["coord_2d"]), c(d["extents"]), c(d["im_wh"]), c(d["cams"]))
    assert torch.equal(pose[:, :, :3], res["pose"][:, :, :3]) and torch.equal(pose[:, :, 3], out_dict["trans"])
    with pytest.raises(ValueError):  # a one-channel mask is not a CE head's output
        pnp_ransac(c(d["mask"][:, :1]), c(d["xyz"]), c(d["coord_2d"]), c(d["extents"]), c(d["im_wh"]), c(d["cams"]), mask_loss_type="CE")


def test_ce_head_net_pnp_modes_match_reference(golden_dir):
    import pnp_net_common as NC
    from gdr_net_b200.pnp_ransac import pnp_ransac, process_pnp
    from oracle import net_pnp_oracle as N
    from oracle import pnp_oracle as PO

    pytest.importorskip("cv2")
    g, d = _ce_inputs(golden_dir)
    B = d["mask"].shape[0]
    R_net, t_net = NC.net_pose(d, seed=3)
    ref = []
    for b in range(B):
        ip, mp = g[f"img_points_{b}"], g[f"model_points_{b}"]
        K = d["cams"][b].numpy()
        r = dict(n=len(ip), inliers=PO.pnp_ransac_cv2(mp, ip, K, iters=20)[1] if len(ip) >= 5 else None)
        for mode in NC.MODES:
            r[mode] = N.net_and_pnp(mp, ip, K, R_net[b], t_net[b], mode)
        ref.append(r)
    c = lambda t: torch.as_tensor(t).cuda()  # noqa: E731
    out_dict = dict(mask=c(d["mask"]), coor_x=c(d["xyz"][:, 0:1]), coor_y=c(d["xyz"][:, 1:2]), coor_z=c(d["xyz"][:, 2:3]),
                    rot=c(R_net), trans=c(t_net))
    args = (out_dict, c(d["coord_2d"]), c(d["extents"]), c(d["im_wh"]), c(d["cams"]))
    poses = {m: process_pnp(_pnp_cfg(t), *args).cpu().numpy() for m, t in (("iter", "net_iter_pnp"), ("ransac", "net_ransac_pnp"),
                                                                          ("ransac_rot", "net_ransac_pnp_rot"))}
    xyz = torch.cat([out_dict["coor_x"], out_dict["coor_y"], out_dict["coor_z"]], dim=1)
    res = pnp_ransac(out_dict["mask"], xyz, *args[1:], mask_loss_type="CE", iters=20, return_inliers=True)
    NC.check(ref, R_net, t_net, res["num_points"].cpu().numpy(), poses, res["inliers"].cpu().numpy(), d, min_identical_frac=0.5)
