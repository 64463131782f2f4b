"""TEST INFRASTRUCTURE ONLY -- the geometry head's shape switches (ROT_HEAD.CONV_KERNEL_SIZE, OUT_CONV_KERNEL_SIZE) on top of the
oracle restatement (oracle/gdrn_oracle.py, oracle/head_gn_oracle.py, oracle/class_aware_oracle.py, oracle/mask_oracle.py,
oracle/region_oracle.py).

The reference's RotWithRegionHead (cdpn_rot_head_region.py:33-46, 81-91, 127-135) builds its first layer as
ConvTranspose2d(512, 256, k, stride 2, padding, output_padding) with k = 2 (pad 0, op 0), 3 (pad 1, op 1) or 4 (pad 1, op 0) --
8x8 -> 16x16 every time -- and its output conv with kernel 1 (pad 0) or 3 (pad 1), so the maps stay 64x64.  Everything else --
the norm layers (BN or GN), backbone, Patch-PnP, losses, pose decode -- is the oracle's.  Pinned to the unmodified reference by
oracle/make_golden_head_shape.py (tests/golden/train_head_shape_b4.npz)."""
from __future__ import annotations

from typing import Dict, Optional

import torch
import torch.nn.functional as F

from oracle import class_aware_oracle as CA
from oracle import gdrn_oracle as O
from oracle import mask_oracle as M
from oracle import region_oracle as RO

Tensor = torch.Tensor
DECONV_PADDING = {2: (0, 0), 3: (1, 1), 4: (1, 0)}  # CONV_KERNEL_SIZE -> (padding, output_padding)


def head_forward(feat: Tensor, sd: Dict[str, Tensor], train: bool, update_stats: bool = False, *, k: int = 3, k_out: int = 1,
                 G: Optional[int] = None) -> Tensor:
    """gdrn_oracle.head_forward (G None: BatchNorm) or head_gn_oracle.head_forward (G groups) with a k x k deconv and a
    k_out x k_out output conv."""
    p = "rot_head_net.features."

    def norm_relu(x, i):
        if G is not None:
            return F.relu(F.group_norm(x, G, sd[f"{p}{i}.weight"], sd[f"{p}{i}.bias"], 1e-5))
        return F.relu(O._bn(x, sd, f"{p}{i}", train, update_stats))

    pad, out_pad = DECONV_PADDING[k]
    x = norm_relu(F.conv_transpose2d(feat, sd[p + "0.weight"], None, stride=2, padding=pad, output_padding=out_pad), 1)
    for ci, bi in [(3, 4), (6, 7), (10, 11), (13, 14), (17, 18), (20, 21)]:
        if ci in (10, 17):
            x = F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=True)
        x = norm_relu(F.conv2d(x, sd[f"{p}{ci}.weight"], None, stride=1, padding=1), bi)
    return F.conv2d(x, sd[p + "23.weight"], sd[p + "23.bias"], padding=k_out // 2)


def gdrn_forward(sd: Dict[str, Tensor], batch: dict, train: bool, do_loss: bool, *, k: int = 3, k_out: int = 1,
                 G: Optional[int] = None, num_regions: int = 64, mask_loss_type: str = "L1", region_att: bool = True,
                 with_2d: bool = True, num_classes: int = 1, rot_aware: bool = False, mask_aware: bool = False,
                 region_aware: bool = False, update_stats: bool = False) -> dict:
    """The GDRN forward (losses with do_loss) of a head with the given shape.  A class-aware head takes the crops' classes from
    batch["roi_cls"] (class_aware_oracle.select_class_maps)."""
    mo = M.mask_channels(mask_loss_type)
    lay = dict(mo=mo, R=num_regions, region_att=region_att, with_2d=with_2d, n_in=3 + 2 * with_2d + num_regions * region_att)
    feat = O.backbone_forward(batch["roi_img"], sd, train, update_stats)
    full = head_forward(feat, sd, train, update_stats, k=k, k_out=k_out, G=G)
    if num_classes > 1 or rot_aware or mask_aware or region_aware:
        head = CA.select_class_maps(full, batch["roi_cls"], num_classes, mo, num_regions, rot_aware, mask_aware, region_aware)
    else:
        head = full
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
    res["losses"] = M.gdrn_losses(head, rot, pred_t_, batch, mask_loss_type=mask_loss_type)
    return res
