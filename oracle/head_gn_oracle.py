"""TEST INFRASTRUCTURE ONLY -- the GroupNorm geometry head (ROT_HEAD.NORM = "GN", NUM_GN_GROUPS) on top of the oracle restatement
(oracle/gdrn_oracle.py, oracle/mask_oracle.py, oracle/region_oracle.py, oracle/class_aware_oracle.py).

The reference builds every norm layer of RotWithRegionHead with get_norm(NORM, 256, num_gn_groups=NUM_GN_GROUPS)
(cdpn_rot_head_region.py, GDRN.py:592-593, core/utils/layer_utils.py): with "GN" the seven layers at features 1, 4, 7, 11, 14, 18
and 21 are nn.GroupNorm(G, 256, eps=1e-5), weight 1 and bias 0 at construction.  GroupNorm has no running statistics, so the
train-mode and the eval-mode head are the same function.  Everything else -- backbone BatchNorm, Patch-PnP, losses, pose decode --
is the oracle's.  Pinned to the unmodified reference by oracle/make_golden_head_gn.py (tests/golden/train_head_gn_b4.npz)."""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn.functional as F

from oracle import class_aware_oracle as CA
from oracle import gdrn_oracle as O
from oracle import mask_oracle as M
from oracle import region_oracle as RO

Tensor = torch.Tensor
NORM_AT = (1, 4, 7, 11, 14, 18, 21)  # features indices of the head's norm layers


def head_forward(feat: Tensor, sd: Dict[str, Tensor], G: int) -> Tensor:
    """gdrn_oracle.head_forward with GroupNorm(G, 256) + ReLU after the deconv and each 3x3 conv."""
    p = "rot_head_net.features."

    def gn_relu(x, i):
        return F.relu(F.group_norm(x, G, sd[f"{p}{i}.weight"], sd[f"{p}{i}.bias"], 1e-5))

    x = gn_relu(F.conv_transpose2d(feat, sd[p + "0.weight"], None, stride=2, padding=1, output_padding=1), 1)
    for ci, bi in [(3, 4), (6, 7), (10, 11), (13, 14), (17, 18), (20, 21)]:
        if ci in (10, 17):
            x = F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=True)
        x = gn_relu(F.conv2d(x, sd[f"{p}{ci}.weight"], None, stride=1, padding=1), bi)
    return F.conv2d(x, sd[p + "23.weight"], sd[p + "23.bias"])


def gdrn_forward(sd: Dict[str, Tensor], batch: dict, train: bool, do_loss: bool, *, G: int, num_regions: int = 64,
                 mask_loss_type: str = "L1", region_att: bool = True, with_2d: bool = True, num_classes: int = 1,
                 rot_aware: bool = False, mask_aware: bool = False, region_aware: bool = False, update_stats: bool = False) -> dict:
    """The GDRN forward (losses with do_loss) of a GroupNorm head; `train` only selects the backbone's BatchNorm statistics.
    A class-aware head takes the crops' classes from batch["roi_cls"] (class_aware_oracle.select_class_maps)."""
    mo = M.mask_channels(mask_loss_type)
    lay = dict(mo=mo, R=num_regions, region_att=region_att, with_2d=with_2d, n_in=3 + 2 * with_2d + num_regions * region_att)
    feat = O.backbone_forward(batch["roi_img"], sd, train, update_stats)
    full = head_forward(feat, sd, G)
    head = CA.select_class_maps(full, batch["roi_cls"], num_classes, mo, num_regions, rot_aware, mask_aware, region_aware)
    coor_feat, region = RO.pnp_input(head, batch, lay)
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
    res["losses"] = M.gdrn_losses(head, rot, pred_t_, batch, mask_loss_type=mask_loss_type)
    return res
