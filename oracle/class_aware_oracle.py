"""TEST INFRASTRUCTURE ONLY -- class-aware geometry heads (ROT_HEAD.ROT_CLASS_AWARE / MASK_CLASS_AWARE / REGION_CLASS_AWARE) on top
of the oracle restatement (oracle/gdrn_oracle.py, oracle/mask_oracle.py, oracle/region_oracle.py).

The reference (core/gdrn_modeling/models/GDRN.py:134-151, cdpn_rot_head_region.py:114-135, 186-193) multiplies a block of the 1x1
output conv by NUM_CLASSES when its switch is set: the mask block (MO per class, class-major), the xyz block (viewed as
[3][C]: x of every class, then y, then z) and the region block (bg + R regions per class, class-major).  Each crop then keeps the
channels of its class (`roi_classes`), and everything after that -- Patch-PnP, losses, pose decode -- sees the usual
mask | xyz | bg | regions maps.  Here the full output conv runs on every crop and the selection is a per-crop index, so the
backward gives exact zeros to the rows of classes no crop uses.  Pinned to the unmodified reference by
oracle/make_golden_class_aware.py (tests/golden/train_class_aware_b4.npz)."""
from __future__ import annotations

from typing import Dict

import torch

from oracle import gdrn_oracle as O
from oracle import mask_oracle as M
from oracle import region_oracle as RO

Tensor = torch.Tensor


def select_class_maps(head: Tensor, classes: Tensor, num_classes: int, mo: int, R: int, rot_aware: bool, mask_aware: bool,
                      region_aware: bool) -> Tensor:
    """[B, rows, H, W] output of the class-aware conv -> [B, MO + 4 + R, H, W] maps of each crop's class (mask | xyz | bg | regions)."""
    B, _, H, W = head.shape
    cm, cr, cg = (num_classes if mask_aware else 1), (num_classes if rot_aware else 1), (num_classes if region_aware else 1)
    assert head.shape[1] == mo * cm + 3 * cr + (R + 1) * cg, (head.shape, mo, R, num_classes)
    mask = head[:, :mo * cm].reshape(B, cm, mo, H, W)
    xyz = head[:, mo * cm:mo * cm + 3 * cr].reshape(B, 3, cr, H, W)
    region = head[:, mo * cm + 3 * cr:].reshape(B, cg, R + 1, H, W)
    b = torch.arange(B, device=head.device)
    cls = classes.long().to(head.device)
    zero = torch.zeros_like(cls)
    mask = mask[b, cls if mask_aware else zero]                                     # [B, MO, H, W]
    xyz = xyz[b, :, cls if rot_aware else zero]                                     # [B, 3, H, W]
    region = region[b, cls if region_aware else zero]                               # [B, R + 1, H, W]
    return torch.cat([mask, xyz, region], dim=1)


def gdrn_forward(sd: Dict[str, Tensor], batch: dict, train: bool, do_loss: bool, *, num_classes: int, rot_aware: bool,
                 mask_aware: bool, region_aware: bool, num_regions: int, mask_loss_type: str = "L1", mask_gt=M.DEFAULT_MASK_GT,
                 region_att: bool = True, with_2d: bool = True, update_stats: bool = False) -> dict:
    """region_oracle.gdrn_forward with a class-aware output conv; the crops' classes are batch["roi_cls"]."""
    mo = M.mask_channels(mask_loss_type)
    lay = dict(mo=mo, R=num_regions, region_att=region_att, with_2d=with_2d, n_in=3 + 2 * with_2d + num_regions * region_att)
    feat = O.backbone_forward(batch["roi_img"], sd, train, update_stats)
    full = O.head_forward(feat, sd, train, update_stats)
    head = select_class_maps(full, batch["roi_cls"], num_classes, mo, num_regions, rot_aware, mask_aware, region_aware)
    coor_feat, region = RO.pnp_input(head, batch, lay)
    rot6d, pred_t_ = O.pnp_forward(coor_feat, region, batch["roi_extent"].to(head.dtype), sd)
    rot_m = O.ortho6d_to_mat(rot6d)
    args = (batch["roi_cam"].to(head.dtype), batch["roi_center"].to(head.dtype), batch["resize_ratio"].to(head.dtype),
            batch["roi_wh"].to(head.dtype))
    res = dict(head=head, full_head=full, rot6d=rot6d, pred_t_=pred_t_, rot_allo=rot_m, feat=feat, layout=lay)
    if not do_loss:
        rot, trans = O.pose_decode_test(rot_m, pred_t_, *args)
        res.update(rot=rot, trans=trans)
        return res
    rot, trans = O.pose_decode_train(rot_m, pred_t_, *args)
    res.update(rot=rot, trans=trans)
    res["losses"] = M.gdrn_losses(head, rot, pred_t_, batch, mask_loss_type=mask_loss_type, mask_gt=mask_gt)
    return res
