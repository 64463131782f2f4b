"""TEST INFRASTRUCTURE ONLY -- DropBlock on the Patch-PnP input (PNP_NET.PNP_HEAD_CFG.drop_prob / dropblock_size) on top of the
oracle restatement (oracle/gdrn_oracle.py, oracle/region_oracle.py).

The reference (core/gdrn_modeling/models/conv_pnp_net.py:66-72,128-142, core/utils/dropblock/{dropblock,scheduler}.py):
  * schedule: LinearScheduler(start 0, stop drop_prob, nr_steps 5000) holds np.linspace(0, drop_prob, 5000); with drop_prob > 0
    every ConvPnPNet.forward (train or eval) first calls step(), so forward k (from 0) uses values[min(k, 4999)];
  * in train mode with a non-zero probability p: seeds = torch.rand(B, H, W) < p / block_size**2 (float32 comparison),
    block_mask = 1 - max_pool2d(seeds, block_size, stride 1, padding block_size // 2) (an even size crops the last row and
    column), out = x * block_mask[:, None] * block_mask.numel() / block_mask.sum(); x is the whole Patch-PnP input, after the
    xyz de-normalisation and the concat.
The random draw is replaced by the seed mask as an input.  Pinned to the unmodified reference by oracle/make_golden_dropblock.py
(tests/golden/train_dropblock_b4.npz)."""
from __future__ import annotations

from typing import Dict

import numpy as np
import torch
import torch.nn.functional as F

from oracle import gdrn_oracle as O
from oracle import mask_oracle as M
from oracle import region_oracle as RO

Tensor = torch.Tensor
N_STEPS = 5000


def drop_values(p: float) -> np.ndarray:
    """LinearScheduler.drop_values."""
    return np.linspace(0.0, p, N_STEPS)


def prob_at(p: float, k: int) -> float:
    """The probability forward k (counted from 0) uses."""
    return float(drop_values(p)[min(k, N_STEPS - 1)])


def block_mask(seeds: Tensor, block_size: int) -> Tensor:
    """DropBlock2D._compute_block_mask of a [B, H, W] 0/1 seed mask."""
    bm = F.max_pool2d(seeds.float()[:, None], kernel_size=(block_size, block_size), stride=(1, 1), padding=block_size // 2)
    if block_size % 2 == 0:
        bm = bm[:, :, :-1, :-1]
    return 1 - bm.squeeze(1)


def dropblock(x: Tensor, seeds: Tensor, block_size: int) -> Tensor:
    """DropBlock2D.forward (train mode, p > 0) of x [B, C, H, W] with the seed mask in place of the random draw."""
    bm = block_mask(seeds, block_size).to(x.dtype)
    out = x * bm[:, None, :, :]
    return out * bm.numel() / bm.sum()


def pnp_forward(coor_feat: Tensor, region: Tensor, extents: Tensor, sd: Dict[str, Tensor], seeds=None, block_size: int = 5):
    """O.pnp_forward with DropBlock on its input (seeds None: no DropBlock, as in eval mode or at probability 0)."""
    bs, in_c = coor_feat.shape[:2]
    if in_c in (3, 5):
        xyz = (coor_feat[:, :3] - 0.5) * extents.view(bs, 3, 1, 1)
        coor_feat = torch.cat([xyz, coor_feat[:, 3:]], dim=1)
    x = torch.cat([coor_feat, region], dim=1)
    if seeds is not None:
        x = dropblock(x, seeds, block_size)
    return O.pnp_forward(x[:, :0], x, extents, sd)  # zero coordinate channels: no second de-normalisation


def gdrn_forward(sd: Dict[str, Tensor], batch: dict, train: bool, do_loss: bool, seeds=None, block_size: int = 5,
                 mask_loss_type: str = "L1", mask_gt=M.DEFAULT_MASK_GT, update_stats: bool = False, region_att=None,
                 with_2d=None) -> dict:
    """region_oracle.gdrn_forward with DropBlock on the Patch-PnP input given its seed mask [B, 64, 64]."""
    lay = RO.layout(sd, mask_loss_type, region_att, with_2d)
    feat = O.backbone_forward(batch["roi_img"], sd, train, update_stats)
    head = O.head_forward(feat, sd, train, update_stats)
    coor_feat, region = RO.pnp_input(head, batch, lay)
    rot6d, pred_t_ = pnp_forward(coor_feat, region, batch["roi_extent"].to(head.dtype), sd, seeds if train else None, block_size)
    rot_m = O.ortho6d_to_mat(rot6d)
    args = (batch["roi_cam"].to(head.dtype), batch["roi_center"].to(head.dtype), batch["resize_ratio"].to(head.dtype),
            batch["roi_wh"].to(head.dtype))
    res = dict(head=head, rot6d=rot6d, pred_t_=pred_t_)
    if not do_loss:
        res["rot"], res["trans"] = O.pose_decode_test(rot_m, pred_t_, *args)
        return res
    rot, trans = O.pose_decode_train(rot_m, pred_t_, *args)
    res.update(rot=rot, trans=trans)
    res["losses"] = M.gdrn_losses(head, rot, pred_t_, batch, mask_loss_type=mask_loss_type, mask_gt=mask_gt)
    return res
