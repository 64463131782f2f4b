"""TEST INFRASTRUCTURE ONLY -- any surface-region count and Patch-PnP without region attention, on top of the oracle restatement
(oracle/gdrn_oracle.py, oracle/mask_oracle.py).

Those two restate the shipped layout: 64 regions whose softmax is the region attention of Patch-PnP, the Patch-PnP input 69 or 67
channels.  The reference has two more switches (core/gdrn_modeling/models/GDRN.py:156-181, 524-547, conv_pnp_net.py:111-127):

  * ROT_HEAD.NUM_REGIONS = R: the output conv has MO + 3 + (R + 1) rows, mask | xyz | bg | R regions, and the region CE runs over
    R + 1 classes (mask_oracle.pixel_losses already takes every channel after xyz);
  * PNP_NET.REGION_ATTENTION: Patch-PnP sees xyz (+ coord2d) (+ softmax(region[:, 1:])), nIn = 3 (+2) (+R).  Without attention
    the region logits get their gradient from the region CE alone.

The channel layout comes from the weight shapes: R from the output conv's rows, attention and the 2-D coordinates from the
Patch-PnP input channels (explicit arguments break the one tie, R = 2 with nIn = 5).  Pinned to the unmodified reference by
oracle/make_golden_regions.py (tests/golden/train_regions_b4.npz)."""
from __future__ import annotations

from typing import Dict, Optional

import torch
import torch.nn.functional as F

from oracle import gdrn_oracle as O
from oracle import mask_oracle as M

Tensor = torch.Tensor


def layout(sd: Dict[str, Tensor], mask_loss_type: str = "L1", region_att: Optional[bool] = None,
           with_2d: Optional[bool] = None) -> dict:
    """mo, R, region_att, with_2d, n_in of the model whose state dict is sd."""
    mo = M.mask_channels(mask_loss_type)
    R = sd["rot_head_net.features.23.weight"].shape[0] - mo - 4
    n_in = sd["pnp_net.features.0.weight"].shape[1]
    if region_att is None:
        region_att = n_in - 3 - R in (0, 2)
    if with_2d is None:
        with_2d = n_in - 3 - (R if region_att else 0) == 2
    assert n_in == 3 + (2 if with_2d else 0) + (R if region_att else 0), (n_in, R, region_att, with_2d)
    return dict(mo=mo, R=R, region_att=bool(region_att), with_2d=bool(with_2d), n_in=n_in)


def pnp_input(head: Tensor, batch: dict, lay: dict):
    """(coor_feat, region attention or an empty channel block) of GDRN.py:156-176 for the layout lay."""
    mo = lay["mo"]
    coor_feat = head[:, mo:mo + 3]
    if lay["with_2d"]:
        coor_feat = torch.cat([coor_feat, batch["roi_coord_2d"].to(head.dtype)], dim=1)
    if lay["region_att"]:
        region = F.softmax(head[:, mo + 4:], dim=1)  # region[:, 1:]
    else:
        region = head.new_zeros(head.shape[0], 0, head.shape[2], head.shape[3])  # x = coor_feat (conv_pnp_net.py:124-127)
    return coor_feat, region


def gdrn_forward(sd: Dict[str, Tensor], batch: dict, train: bool, do_loss: bool, mask_loss_type: str = "L1",
                 mask_gt=M.DEFAULT_MASK_GT, pm_sym: bool = False, update_stats: bool = False, region_att: Optional[bool] = None,
                 with_2d: Optional[bool] = None) -> dict:
    """mask_oracle.gdrn_forward (GDRN.py:83-306) for any region count, with or without region attention."""
    lay = layout(sd, mask_loss_type, region_att, with_2d)
    feat = O.backbone_forward(batch["roi_img"], sd, train, update_stats)
    head = O.head_forward(feat, sd, train, update_stats)
    coor_feat, region = pnp_input(head, batch, lay)
    rot6d, pred_t_ = O.pnp_forward(coor_feat, region, batch["roi_extent"].to(head.dtype), sd)
    rot_m = O.ortho6d_to_mat(rot6d)
    args = (batch["roi_cam"].to(head.dtype), batch["roi_center"].to(head.dtype), batch["resize_ratio"].to(head.dtype),
            batch["roi_wh"].to(head.dtype))
    res = dict(head=head, rot6d=rot6d, pred_t_=pred_t_, rot_allo=rot_m, feat=feat, layout=lay)
    if not do_loss:
        rot, trans = O.pose_decode_test(rot_m, pred_t_, *args)
        res.update(rot=rot, trans=trans)
        return res
    rot, trans = O.pose_decode_train(rot_m, pred_t_, *args)
    res.update(rot=rot, trans=trans)
    res["losses"] = M.gdrn_losses(head, rot, pred_t_, batch, pm_sym=pm_sym, mask_loss_type=mask_loss_type, mask_gt=mask_gt)
    re_, te_ = O.mean_re_te(trans, rot, batch["trans"], batch["ego_rot"])
    res["vis"] = {"vis/error_R": float(re_), "vis/error_t": float(te_) * 100}
    return res
