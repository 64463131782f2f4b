"""TEST INFRASTRUCTURE ONLY -- frozen sub-networks (MODEL.CDPN.BACKBONE.FREEZE, ROT_HEAD.FREEZE, PNP_NET.FREEZE) on top of the
oracle restatement (oracle/gdrn_oracle.py).

The reference (core/gdrn_modeling/models/GDRN.py:550-700, resnet_backbone.py:53-67, cdpn_rot_head_region.py:167-181):
  * a frozen backbone or head runs under torch.no_grad() and its output is detached.  Its BatchNorms stay in train mode, so
    they still normalise with batch statistics and still update running_mean / running_var / num_batches_tracked.  A frozen
    head therefore also cuts the backbone off from every loss;
  * a frozen head's per-pixel losses (loss_coor_x/y/z, loss_mask, loss_region) are absent (gdrn_loss, GDRN.py:342-400);
  * a frozen Patch-PnP changes no value: its parameters stop requiring grad (GDRN.py:684-687), so gradients still flow through
    it.  Here its parameters enter as detached constants.
Pinned to the unmodified reference by oracle/make_golden_freeze.py (tests/golden/train_freeze_<case>_b4.npz)."""
from __future__ import annotations

from typing import Dict

import torch

from oracle import gdrn_oracle as O

Tensor = torch.Tensor

PIXEL_LOSSES = ("loss_coor_x", "loss_coor_y", "loss_coor_z", "loss_mask", "loss_region")
# case -> (BACKBONE.FREEZE, ROT_HEAD.FREEZE, PNP_NET.FREEZE), as oracle/make_golden_freeze.py
CASES = {"bb": (True, False, False), "head": (False, True, False), "pnp": (False, False, True), "bb_pnp": (True, False, True),
         "head_pnp": (False, True, True), "all": (True, True, True)}
SUBNETS = ("backbone.", "rot_head_net.", "pnp_net.")


def live(name: str, freeze) -> bool:
    """Whether parameter `name` receives a gradient under freeze = (backbone, head, pnp)."""
    fb, fh, fp = freeze
    if name.startswith("pnp_net."):
        return not fp
    if name.startswith("rot_head_net."):
        return not fh
    return not (fb or fh)


def gdrn_forward(sd: Dict[str, Tensor], batch: dict, train: bool, do_loss: bool, freeze=(False, False, False),
                 update_stats: bool = False) -> dict:
    """O.gdrn_forward (a6 configuration) with frozen sub-networks; freeze = (BACKBONE, ROT_HEAD, PNP_NET) .FREEZE."""
    fb, fh, fp = freeze
    grad = torch.is_grad_enabled()
    x = batch["roi_img"]
    with torch.set_grad_enabled(grad and not fb):
        feat = O.backbone_forward(x, sd, train, update_stats)
    if fb:
        feat = feat.detach()
    with torch.set_grad_enabled(grad and not fh):
        head = O.head_forward(feat, sd, train, update_stats)
    if fh:
        head = head.detach()
    psd = {k: (v.detach() if (fp and k.startswith("pnp_net.")) else v) for k, v in sd.items()}
    coor_feat = head[:, 1:4]
    if psd["pnp_net.features.0.weight"].shape[1] == 69:
        coor_feat = torch.cat([coor_feat, batch["roi_coord_2d"].to(head.dtype)], dim=1)
    rot6d, pred_t_ = O.pnp_forward(coor_feat, torch.softmax(head[:, 5:], dim=1), batch["roi_extent"].to(head.dtype), psd)
    rot_m = O.ortho6d_to_mat(rot6d)
    args = (batch["roi_cam"].to(head.dtype), batch["roi_center"].to(head.dtype), batch["resize_ratio"].to(head.dtype),
            batch["roi_wh"].to(head.dtype))
    res = dict(head=head, rot6d=rot6d, pred_t_=pred_t_, feat=feat)
    if not do_loss:
        res["rot"], res["trans"] = O.pose_decode_test(rot_m, pred_t_, *args)
        return res
    rot, trans = O.pose_decode_train(rot_m, pred_t_, *args)
    res.update(rot=rot, trans=trans)
    losses = O.gdrn_losses(head, rot, pred_t_, batch)
    res["losses"] = {k: v for k, v in losses.items() if not (fh and k in PIXEL_LOSSES)}
    return res
