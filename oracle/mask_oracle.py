"""TEST INFRASTRUCTURE ONLY -- the mask-head switches of the geometric head on top of the oracle restatement (oracle/gdrn_oracle.py).

`gdrn_oracle` restates the shipped configuration: an L1 mask head with one channel, xyz and region losses weighted by the visible
mask, the mask loss against the truncated one.  The reference's `gdrn_loss` (core/gdrn_modeling/models/GDRN.py:339-400) has two
more switches, restated here with the same functions:

  * ROT_HEAD.MASK_LOSS_TYPE  L1 | BCE | CE (:376-385).  CE makes the head emit TWO mask channels (GDRN.py:536-541), so the
    output conv has 70 rows: mask 0..1 | xyz 2..4 | bg 5 | regions 6..69 (cdpn_rot_head_region.py:185-192);
  * the GT mask of each per-pixel loss, gt_masks[XYZ_LOSS_MASK_GT / MASK_LOSS_GT / REGION_LOSS_MASK_GT] with
    gt_masks = {"trunc", "visib", "obj"} (:339); xyz and region are normalised by the sum of their own mask.

`select_points_ce` is `get_out_mask` (engine_utils.py:108-126) of a CE head followed by the evaluator's point selection.
Pinned to the unmodified reference by oracle/make_golden_masks.py (tests/golden/train_mask_*_b4.npz, pnp_ce_select_b3.npz).
"""
from __future__ import annotations

from typing import Dict

import numpy as np
import torch
import torch.nn.functional as F

from oracle import gdrn_oracle as O
from oracle import pnp_oracle

Tensor = torch.Tensor
DEFAULT_MASK_GT = ("visib", "trunc", "visib")  # XYZ_LOSS_MASK_GT, MASK_LOSS_GT, REGION_LOSS_MASK_GT of the shipped configs


def mask_channels(mask_loss_type: str) -> int:
    """get_xyz_mask_region_out_dim (GDRN.py:536-541): 2 mask channels for CE, 1 for L1 / BCE."""
    return 2 if mask_loss_type == "CE" else 1


def pixel_losses(head_out: Tensor, batch: dict, mask_loss_type: str = "L1", mask_gt=DEFAULT_MASK_GT) -> Dict[str, Tensor]:
    """The five per-pixel losses of gdrn_loss (GDRN.py:339-400) on the head output [B, 68 + MO, H, W]."""
    mo = mask_channels(mask_loss_type)
    out_mask = head_out[:, :mo]
    out_x, out_y, out_z = head_out[:, mo:mo + 1], head_out[:, mo + 1:mo + 2], head_out[:, mo + 2:mo + 3]
    out_region = head_out[:, mo + 3:]
    dt = head_out.dtype
    gt_xyz = batch["roi_xyz"].to(dt)
    gt_masks = {"trunc": batch["roi_mask_trunc"], "visib": batch["roi_mask_visib"], "obj": batch.get("roi_mask_obj")}
    m_xyz, m_mask, m_reg = (gt_masks[k].to(dt) for k in mask_gt)  # KeyError for anything else, like the reference
    L = {}
    denom = m_xyz.sum().float().clamp(min=1.0)
    for name, o, c in (("x", out_x, 0), ("y", out_y, 1), ("z", out_z, 2)):  # :343-355
        L[f"loss_coor_{name}"] = F.l1_loss(o * m_xyz[:, None], gt_xyz[:, c:c + 1] * m_xyz[:, None], reduction="sum") / denom
    if mask_loss_type == "L1":  # :378-379
        L["loss_mask"] = F.l1_loss(out_mask[:, 0], m_mask, reduction="mean")
    elif mask_loss_type == "BCE":  # :380-381
        L["loss_mask"] = F.binary_cross_entropy_with_logits(out_mask[:, 0], m_mask, reduction="mean")
    elif mask_loss_type == "CE":  # :382-383 (.long() truncates a soft target)
        L["loss_mask"] = F.cross_entropy(out_mask, m_mask.long(), reduction="mean")
    else:
        raise NotImplementedError(mask_loss_type)
    gt_region = batch["roi_region"].long()
    L["loss_region"] = (  # :388-397 (logits AND labels multiplied by the mask, SURVEY P5)
        F.cross_entropy(out_region * m_reg[:, None], gt_region * m_reg.long(), reduction="sum") / m_reg.sum().float().clamp(min=1.0)
    )
    return L


def gdrn_losses(head_out: Tensor, pred_ego_rot: Tensor, pred_t_: Tensor, batch: dict, pm_sym: bool = False,
                mask_loss_type: str = "L1", mask_gt=DEFAULT_MASK_GT) -> Dict[str, Tensor]:
    """gdrn_oracle.gdrn_losses with the mask switches: the per-pixel losses above, the pose losses of gdrn_oracle (which do not
    depend on the head output)."""
    L = pixel_losses(head_out, batch, mask_loss_type, mask_gt)
    B, dt, dev = head_out.shape[0], head_out.dtype, head_out.device
    inert = dict(batch, roi_xyz=torch.zeros(B, 3, 1, 1, dtype=dt, device=dev), roi_mask_visib=torch.zeros(B, 1, 1, dtype=dt, device=dev),
                 roi_mask_trunc=torch.zeros(B, 1, 1, dtype=dt, device=dev), roi_region=torch.zeros(B, 1, 1, dtype=torch.long, device=dev))
    P = O.gdrn_losses(torch.zeros(B, 69, 1, 1, dtype=dt, device=dev), pred_ego_rot, pred_t_, inert, pm_sym=pm_sym)
    for k in ("loss_PM_R", "loss_centroid", "loss_z"):
        L[k] = P[k]
    return L


def gdrn_forward(sd: Dict[str, Tensor], batch: dict, train: bool, do_loss: bool, mask_loss_type: str = "L1",
                 mask_gt=DEFAULT_MASK_GT, pm_sym: bool = False, update_stats: bool = False) -> dict:
    """gdrn_oracle.gdrn_forward (GDRN.py:83-306) for a head with MO = mask_channels(mask_loss_type) mask channels: the xyz and
    region slices of the Patch-PnP input start at MO instead of 1."""
    mo = mask_channels(mask_loss_type)
    assert sd["rot_head_net.features.23.weight"].shape[0] == 68 + mo, sd["rot_head_net.features.23.weight"].shape
    x = batch["roi_img"]
    feat = O.backbone_forward(x, sd, train, update_stats)
    head = O.head_forward(feat, sd, train, update_stats)
    coor_feat = head[:, mo:mo + 3]
    if sd["pnp_net.features.0.weight"].shape[1] == 69:
        coor_feat = torch.cat([coor_feat, batch["roi_coord_2d"].to(head.dtype)], dim=1)
    region_softmax = F.softmax(head[:, mo + 4:], dim=1)  # region[:, 1:]
    rot6d, pred_t_ = O.pnp_forward(coor_feat, region_softmax, batch["roi_extent"].to(head.dtype), sd)
    rot_m = O.ortho6d_to_mat(rot6d)
    args = (batch["roi_cam"].to(head.dtype), batch["roi_center"].to(head.dtype), batch["resize_ratio"].to(head.dtype),
            batch["roi_wh"].to(head.dtype))
    res = dict(head=head, rot6d=rot6d, pred_t_=pred_t_, rot_allo=rot_m, feat=feat)
    if not do_loss:
        rot, trans = O.pose_decode_test(rot_m, pred_t_, *args)
        res.update(rot=rot, trans=trans)
        return res
    rot, trans = O.pose_decode_train(rot_m, pred_t_, *args)
    res.update(rot=rot, trans=trans)
    res["losses"] = gdrn_losses(head, rot, pred_t_, batch, pm_sym=pm_sym, mask_loss_type=mask_loss_type, mask_gt=mask_gt)
    re_, te_ = O.mean_re_te(trans, rot, batch["trans"], batch["ego_rot"])
    res["vis"] = {"vis/error_R": float(re_), "vis/error_t": float(te_) * 100}
    return res


def ce_mask(mask2) -> np.ndarray:
    """get_out_mask of a CE head (engine_utils.py:123-124): argmax over the two channels [2, H, W], the first maximum on a tie."""
    m = np.asarray(mask2, np.float32)
    return (m[1] > m[0]).astype(np.float32)


def select_points_ce(mask2, xyz, coord2d, extent, im_W, im_H, mask_thr=0.5):
    """get_out_mask (CE) + get_img_model_points_with_coords2d (gdrn_evaluator.py:89-126): (image points, model points)."""
    return pnp_oracle.select_points(ce_mask(mask2), xyz, coord2d, extent, im_W, im_H, mask_thr)
