"""TEST INFRASTRUCTURE ONLY -- the PNP_NET pose-loss switches on top of the oracle restatement (oracle/gdrn_oracle.py).

`gdrn_oracle` restates the shipped pose losses: r_only L1 point matching normalised by the extent, L1 centroid and z.  The
reference's `gdrn_loss` (core/gdrn_modeling/models/GDRN.py:402-514) has more switches, restated here with the same functions:

  * PyPMLoss (pm_loss.py:20-171): PM_LOSS_TYPE L1 | Smooth_L1 (fvcore, PM_SMOOTH_L1_BETA) | MSE | L2 (l2_loss.py: per-crop
    norm, mean over B), PM_NORM_BY_EXTENT, PM_R_ONLY, PM_DISENTANGLE_T / _Z with or without PM_T_USE_POINTS, PM_LOSS_SYM;
  * loss_rot (rot_loss.py:30-48): angular_distance_rot or rot_l2_loss against the ORIGINAL gt rotation;
  * loss_centroid / loss_z (GDRN.py:439-471), loss_trans_xy + loss_trans_z or loss_trans_LPnP (:474-500), loss_bind (:503-514,
    whose MSE branch tests CENTROID_LOSS_TYPE).

`p` is a PNP_NET config (attribute access); the returned dict is the reference's loss_dict order with the weights applied.
Pinned to the unmodified reference by oracle/make_golden_pose_losses.py (tests/golden/train_pose_losses_b4.npz).
"""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn.functional as F

from oracle import gdrn_oracle as O
from oracle import mask_oracle as M

Tensor = torch.Tensor


def smooth_l1(a: Tensor, b: Tensor, beta: float) -> Tensor:
    """fvcore.nn.smooth_l1_loss, reduction mean: plain L1 for beta < 1e-5, else torch's smooth L1."""
    if beta < 1e-5:
        return (a - b).abs().mean()
    return F.smooth_l1_loss(a, b, beta=beta, reduction="mean")


def l2_loss(a: Tensor, b: Tensor) -> Tensor:
    """l2_loss.py:5-27, reduction mean: the norm over everything but the batch dimension, then the mean over B."""
    B = a.shape[0]
    return torch.norm((a - b).view(B, -1), p=2, dim=1, keepdim=True).mean()


def loss_func(kind: str, beta: float = 1.0):
    kind = kind.lower()
    if kind == "smooth_l1":
        return lambda a, b: smooth_l1(a, b, beta)
    if kind == "l1":
        return lambda a, b: F.l1_loss(a, b, reduction="mean")
    if kind == "mse":
        return lambda a, b: F.mse_loss(a, b, reduction="mean")
    if kind == "l2":
        return l2_loss
    raise ValueError(kind)


def pm_losses(p, pred_rots, gt_rots, points, pred_transes, gt_transes, extents) -> Dict[str, Tensor]:
    """PyPMLoss.forward (pm_loss.py:82-171) after the closest symmetric gt_rots; loss_weight = PM_LW."""
    f = loss_func(p.PM_LOSS_TYPE, p.PM_SMOOTH_L1_BETA)
    lw = p.PM_LW
    dis_z = p.PM_DISENTANGLE_Z
    dis_t = p.PM_DISENTANGLE_T or dis_z  # :58-60
    use_pts = True if not dis_t else p.PM_T_USE_POINTS  # :62-66
    est = (pred_rots[:, None] @ points[..., None]).squeeze(-1)  # transform_pts_batch(points, R, t=None)
    tgt = (gt_rots[:, None] @ points[..., None]).squeeze(-1)
    w = (1.0 / extents.max(1, keepdim=True)[0]).view(-1, 1, 1) if p.PM_NORM_BY_EXTENT else 1
    gt_t = gt_transes.view(-1, 1, 3)
    if p.PM_R_ONLY:
        return {"loss_PM_R": 3 * f(w * est, w * tgt) * lw}
    if dis_z:
        if use_pts:
            tgt_RT = tgt + gt_t
            t_xy = pred_transes.clone()
            t_xy[:, 2] = gt_transes[:, 2]
            t_z = pred_transes.clone()
            t_z[:, :2] = gt_transes[:, :2]
            return {"loss_PM_R": 3 * f(w * (est + gt_t), w * tgt_RT) * lw,
                    "loss_PM_xy": 3 * f(w * (tgt + t_xy.view(-1, 1, 3)), w * tgt_RT) * lw,
                    "loss_PM_z": 3 * f(w * (tgt + t_z.view(-1, 1, 3)), w * tgt_RT) * lw}
        return {"loss_PM_R": 3 * f(w * est, w * tgt) * lw, "loss_PM_xy_noP": f(pred_transes[:, :2], gt_transes[:, :2]),
                "loss_PM_z_noP": f(pred_transes[:, 2], gt_transes[:, 2])}
    if dis_t:
        if use_pts:
            tgt_RT = tgt + gt_t
            return {"loss_PM_R": 3 * f(w * (est + gt_t), w * tgt_RT) * lw,
                    "loss_PM_T": 3 * f(w * (tgt + pred_transes.view(-1, 1, 3)), w * tgt_RT) * lw}
        return {"loss_PM_R": 3 * f(w * est, w * tgt) * lw, "loss_PM_T_noP": f(pred_transes, gt_transes)}
    return {"loss_PM_RT": 3 * f(w * (est + pred_transes.view(-1, 1, 3)), w * (tgt + gt_t)) * lw}


def _typed(kind: str):
    return {"L1": lambda a, b: F.l1_loss(a, b, reduction="mean"), "L2": l2_loss,
            "MSE": lambda a, b: F.mse_loss(a, b, reduction="mean")}[kind]


def pose_losses(p, out_rot: Tensor, out_trans: Tensor, pred_t_: Tensor, batch: dict, pm_sym: bool = False) -> Dict[str, Tensor]:
    """The pose half of gdrn_loss (GDRN.py:402-514) with the weights applied, in the reference's loss_dict order."""
    dt = out_rot.dtype
    gt_rot = batch["ego_rot"].to(dt)
    gt_trans = batch["trans"].to(dt)
    ratio = batch["roi_trans_ratio"].to(dt)
    L = {}
    if p.PM_LW > 0:
        closest = getattr(F, "closest_rot_batch", O.closest_rot_batch)  # a stand-in for F may answer it (tests/pinned_backward.py)
        gt_pm = closest(out_rot, gt_rot, batch["sym_info"]).to(dt) if pm_sym else gt_rot
        L.update(pm_losses(p, out_rot, gt_pm, batch["roi_points"].to(dt), out_trans, gt_trans, batch["roi_extent"].to(dt)))
    if p.ROT_LW > 0:
        if p.ROT_LOSS_TYPE == "angular":  # angular_distance_rot
            m = torch.bmm(out_rot, gt_rot.transpose(1, 2))
            cos = (torch.einsum("bii->b", m) - 1) / 2
            L["loss_rot"] = ((1 - cos) / 2).mean()
        else:  # rot_l2_loss
            L["loss_rot"] = torch.pow(out_rot - gt_rot, 2).mean()
        L["loss_rot"] = L["loss_rot"] * p.ROT_LW
    if p.CENTROID_LW > 0:
        L["loss_centroid"] = _typed(p.CENTROID_LOSS_TYPE)(pred_t_[:, :2], ratio[:, :2]) * p.CENTROID_LW
    if p.Z_LW > 0:
        L["loss_z"] = _typed(p.Z_LOSS_TYPE)(pred_t_[:, 2], ratio[:, 2]) * p.Z_LW
    if p.TRANS_LW > 0:
        f = _typed(p.TRANS_LOSS_TYPE)
        if p.TRANS_LOSS_DISENTANGLE:
            L["loss_trans_xy"] = f(out_trans[:, :2], gt_trans[:, :2]) * p.TRANS_LW
            L["loss_trans_z"] = f(out_trans[:, 2], gt_trans[:, 2]) * p.TRANS_LW
        else:
            L["loss_trans_LPnP"] = f(out_trans, gt_trans) * p.TRANS_LW
    if p.get("BIND_LW", 0.0) > 0:
        pred_bind = torch.bmm(out_rot.permute(0, 2, 1), out_trans.view(-1, 3, 1)).view(-1, 3)
        gt_bind = torch.bmm(gt_rot.permute(0, 2, 1), gt_trans.view(-1, 3, 1)).view(-1, 3)
        bt = p.BIND_LOSS_TYPE
        kind = bt if bt in ("L1", "L2") else ("MSE" if p.CENTROID_LOSS_TYPE == "MSE" else None)  # GDRN.py:510 tests CENTROID
        if kind is None:
            raise ValueError(f"Unknown bind loss (R^T@t) type: {bt}")
        L["loss_bind"] = _typed(kind)(pred_bind, gt_bind) * p.BIND_LW
    return L


def gdrn_forward(sd: Dict[str, Tensor], batch: dict, p, train: bool = True, pm_sym: bool = False,
                 update_stats: bool = False) -> dict:
    """mask_oracle.gdrn_forward (L1 mask head) with the pose losses of `p`: the pixel losses, then pose_losses."""
    res = M.gdrn_forward(sd, batch, train=train, do_loss=True, update_stats=update_stats)
    pix = {k: res["losses"][k] for k in ("loss_coor_x", "loss_coor_y", "loss_coor_z", "loss_mask", "loss_region")}
    pix.update(pose_losses(p, res["rot"], res["trans"], res["pred_t_"], batch, pm_sym=pm_sym))
    res["losses"] = pix
    return res
