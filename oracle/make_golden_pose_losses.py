"""TEST INFRASTRUCTURE ONLY -- golden vectors for the PNP_NET pose-loss switches, produced by the UNMODIFIED reference (run in the
build container; the GPU box has no /root/reference).

The reference model (GDRN.py) is built from the a6 config with only PNP_NET switches changed, trained one step in train mode on a
seeded batch of four crops; the losses and the gradients of GRAD_KEYS after `sum(loss_dict.values()).backward()` are written to
tests/golden/train_pose_losses_b4.npz under "<case>/loss/<name>" and "<case>/grad/<param>".  Cases (CASES):

  rt_sl1       point matching on R and t together, Smooth-L1 with a beta that both branches use (asserted below), angular rot
               loss, disentangled MSE translation loss, L1 bind loss;
  disz_l2      DISENTANGLE_Z with points, L2 point matching, L2 rot loss, non-disentangled L2 translation loss, MSE centroid,
               L2 z;
  dist_nop_sym DISENTANGLE_T without points, MSE, not normalised by the extent, PM_LOSS_SYM on the YCB-V-like object set of
               synth.py, angular rot and L1 bind losses (both on the original gt rotation);
  bind_mse     BIND_LOSS_TYPE "MSE" through the CENTROID_LOSS_TYPE = "MSE" rule of GDRN.py:510, DISENTANGLE_Z without points;
  pm_off       PM_LW = 0 (no PM entry), angular rot loss, L1 translation loss.

ref_shim stubs fvcore's smooth_l1_loss with F.smooth_l1_loss.  The two agree for beta >= 1e-5 (fvcore switches to plain L1
below that), so the Smooth-L1 case uses beta = 0.5.

Usage: python -m oracle.make_golden_pose_losses"""
import copy
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gdr_net_b200 import synth  # noqa: E402
from gdr_net_b200.config import Config, postprocess_like_main_gdrn  # noqa: E402
from oracle import ref_shim  # noqa: E402
from oracle.make_golden import REF_CFG  # noqa: E402

_PM = dict(PM_R_ONLY=False)
CASES = {  # name -> (PNP_NET switches, weight seed, batch seed, batch with_sym)
    "rt_sl1": (dict(_PM, PM_LOSS_TYPE="Smooth_L1", PM_SMOOTH_L1_BETA=0.5, ROT_LW=1.0, ROT_LOSS_TYPE="angular", TRANS_LW=1.0,
                    TRANS_LOSS_TYPE="MSE", TRANS_LOSS_DISENTANGLE=True, BIND_LW=1.0, BIND_LOSS_TYPE="L1"), 7, 31, False),
    "disz_l2": (dict(_PM, PM_DISENTANGLE_Z=True, PM_T_USE_POINTS=True, PM_LOSS_TYPE="L2", ROT_LW=1.0, ROT_LOSS_TYPE="L2",
                     TRANS_LW=1.0, TRANS_LOSS_TYPE="L2", TRANS_LOSS_DISENTANGLE=False, CENTROID_LOSS_TYPE="MSE",
                     Z_LOSS_TYPE="L2"), 8, 37, False),
    "dist_nop_sym": (dict(_PM, PM_DISENTANGLE_T=True, PM_T_USE_POINTS=False, PM_LOSS_TYPE="MSE", PM_NORM_BY_EXTENT=False,
                          PM_LOSS_SYM=True, ROT_LW=1.0, ROT_LOSS_TYPE="angular", BIND_LW=1.0, BIND_LOSS_TYPE="L1"), 9, 41, "ycbv"),
    "bind_mse": (dict(_PM, PM_DISENTANGLE_Z=True, PM_T_USE_POINTS=False, BIND_LW=1.0, BIND_LOSS_TYPE="MSE",
                      CENTROID_LOSS_TYPE="MSE"), 10, 43, False),
    "pm_off": (dict(PM_LW=0.0, ROT_LW=1.0, ROT_LOSS_TYPE="angular", TRANS_LW=1.0, TRANS_LOSS_TYPE="L1"), 11, 47, False),
}
GRAD_KEYS = ("rot_head_net.features.23.weight", "rot_head_net.features.23.bias", "rot_head_net.features.21.weight",
             "pnp_net.features.1.weight", "pnp_net.fc_r.weight", "pnp_net.fc_t.weight", "backbone.bn1.weight")


def reference_config(switches):
    cfg = Config.fromfile(os.path.join(ref_shim.REFERENCE_ROOT, REF_CFG))
    cfg = postprocess_like_main_gdrn(cfg, device="cpu")
    cfg.MODEL.CDPN.BACKBONE.PRETRAINED = ""
    cfg.MODEL.CDPN.PNP_NET.update(switches)
    return cfg


def check_smooth_l1_branches(model, batch, beta):
    """Both branches of the Smooth-L1 loss occur in the rt_sl1 case: residuals below and above beta."""
    from oracle import gdrn_oracle as O
    from oracle import mask_oracle as M

    with torch.no_grad():
        o = M.gdrn_forward(O.leaf_state_dict(model.state_dict(), requires_grad=False), batch, train=True, do_loss=True)
    R, T = o["rot"], o["trans"]
    pts = batch["roi_points"]
    w = (1.0 / batch["roi_extent"].max(1, keepdim=True)[0]).view(-1, 1, 1)
    e = w * ((R[:, None] @ pts[..., None]).squeeze(-1) + T[:, None]) - w * ((batch["ego_rot"][:, None] @ pts[..., None]).squeeze(-1)
                                                                         + batch["trans"][:, None])
    below = float((e.abs() < beta).float().mean())
    print(f"rt_sl1: {below:.3f} of the residuals below beta = {beta}")
    assert 0.05 < below < 0.95, below


def train_case(ref_gdrn, name, save):
    switches, wseed, bseed, with_sym = CASES[name]
    cfg = reference_config(switches)
    torch.manual_seed(0)
    model, _ = ref_gdrn.build_model_optimizer(copy.deepcopy(cfg))
    sd = synth.seeded_state_dict(model.state_dict(), seed=wseed)
    batch = synth.make_batch(4, seed=bseed, with_sym=with_sym)
    model.load_state_dict(sd)
    model.train()
    if name == "rt_sl1":
        check_smooth_l1_branches(model, batch, switches["PM_SMOOTH_L1_BETA"])
        model.load_state_dict(sd)  # the check ran the oracle on a copy; the BatchNorm statistics are untouched
    _, loss_dict = model(batch["roi_img"].clone(), **synth.forward_kwargs(batch, train=True))
    sum(loss_dict.values()).backward()
    save.update({f"{name}/loss/{k}": np.array(float(v)) for k, v in loss_dict.items()})
    save[f"{name}/names"] = np.array(list(loss_dict))
    grads = dict(model.named_parameters())
    for k in GRAD_KEYS:
        save[f"{name}/grad/{k}"] = grads[k].grad.detach().numpy()
    print(name, {k: float(v) for k, v in loss_dict.items()})


def main():
    torch.set_num_threads(os.cpu_count())
    ref_gdrn = ref_shim.import_reference_gdrn()
    save = {}
    for name in CASES:
        train_case(ref_gdrn, name, save)
    path = os.path.join(ROOT, "tests", "golden", "train_pose_losses_b4.npz")
    np.savez_compressed(path, **save)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
