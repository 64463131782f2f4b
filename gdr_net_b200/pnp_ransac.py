"""Test-time RANSAC-PnP on the device (SURVEY.md 8f row f-4, the `TEST.USE_PNP` branch of the evaluator).

Reference: `GDRN_Evaluator.process_pnp_ransac` (`core/gdrn_modeling/gdrn_evaluator.py:316-436`) loops over the instances on the
host: `get_out_coor` / `get_out_mask` (`engine_utils.py:92-126`), D2H copies, `get_img_model_points_with_coords2d` (:89-126) and
`misc.pnp_v2(..., cv2.SOLVEPNP_EPNP, ransac=True, ransac_reprojErr=3, ransac_iter=100)` (`lib/pysixd/misc.py:145-194`), then
replaces the translation by the one decoded from the network's (cx, cy, z) head (:398-421).

Here the whole batch is solved by three kernel launches (`csrc/pnp_ransac.cu`), following OpenCV's algorithm closely enough that
the inlier sets and poses agree with cv2 up to round-off (tests/test_pnp_ransac_gpu.py).  No host synchronisation.

The network-initialised modes of the evaluator (`process_net_and_pnp`, gdrn_evaluator.py:187-314: TEST.PNP_TYPE net_iter_pnp,
net_ransac_pnp, net_ransac_pnp_rot) are `process_net_and_pnp` below: the iterative one is OpenCV's Levenberg-Marquardt
(`pnp_iterative`, two launches), the RANSAC ones reuse `pnp_ransac` with 20 iterations.  `process_pnp` dispatches on the
config like the evaluator does."""
from __future__ import annotations

import torch

from .capi import C

_MASK_MODES = {"none": 0, "L1": 1, "BCE": 2, "CE": 3}


def _mask_planes(mask: torch.Tensor, mask_loss_type: str, B: int, h: int, w: int) -> torch.Tensor:
    """The mask head output as the kernels read it: [B, h*w], or [B, 2*h*w] (two planes per ROI) for the CE head."""
    n = 2 if mask_loss_type == "CE" else 1
    if mask.numel() != B * n * h * w:
        raise ValueError(f"mask: expected {n} channel(s) of {h}x{w} per ROI for mask_loss_type {mask_loss_type!r}, got {tuple(mask.shape)}")
    return mask.reshape(B, n * h * w)


def pnp_ransac(mask: torch.Tensor, xyz: torch.Tensor, coord_2d: torch.Tensor, extents: torch.Tensor, im_wh, cams: torch.Tensor,
               mask_loss_type: str = "L1", mask_thr: float = 0.5, reproj_err: float = 3.0, iters: int = 100,
               confidence: float = 0.99, return_inliers: bool = False) -> dict:
    """mask [B,1,h,w] raw head output (normalised here like `get_out_mask` for `mask_loss_type` "L1" / "BCE"; "none": used as is)
    or [B,2,h,w] for the CE mask head (`mask_loss_type` "CE": argmax over the two channels, a tie selecting class 0),
    xyz [B,3,h,w] in [0,1] (`get_out_coor` of the regression head = cat(coor_x, coor_y, coor_z)), coord_2d [B,2,h,w] in [0,1],
    extents [B,3], im_wh [B,2] or (W, H), cams [B,3,3] or [3,3].
    Returns dict(pose [B,3,4], num_points [B], num_inliers [B], iterations [B], ok [B] (bool)[, inliers [B,h*w] uint8 flags over
    the row-major list of selected points]).  Instances with fewer than 5 selected points get ok = False and an identity pose
    (the reference writes -100 there, gdrn_evaluator.py:388-390; `process_pnp_ransac` below does the same)."""
    if not mask.is_cuda:
        raise RuntimeError("gdr_net_b200.pnp_ransac runs on CUDA only; there is no CPU fallback")
    if mask_loss_type not in _MASK_MODES:
        raise NotImplementedError(f"unknown mask loss type: {mask_loss_type}")
    dev = mask.device
    B, _, h, w = xyz.shape
    f = lambda t: t.detach().to(dev).float().contiguous()  # noqa: E731
    mask, xyz, coord_2d, extents = _mask_planes(f(mask), mask_loss_type, B, h, w), f(xyz), f(coord_2d), f(extents).reshape(B, 3)
    if coord_2d.shape != (B, 2, h, w):
        raise ValueError(f"pnp_ransac: coord_2d {tuple(coord_2d.shape)} does not match xyz {tuple(xyz.shape)}")
    if not torch.is_tensor(im_wh):
        im_wh = torch.tensor(im_wh, dtype=torch.float32)
    im_wh = f(im_wh)
    im_wh = (im_wh.reshape(1, 2).expand(B, 2) if im_wh.numel() == 2 else im_wh.reshape(B, 2)).contiguous()
    cams = f(cams)
    cams = (cams.reshape(1, 3, 3).expand(B, 3, 3) if cams.dim() == 2 else cams.reshape(B, 3, 3)).contiguous()
    nbytes = int(C.load().gdrn_pnp_ransac_workspace_bytes(B, h * w, iters))
    ws = torch.empty((nbytes + 7) // 8, dtype=torch.float64, device=dev)
    pose = torch.empty(B, 3, 4, device=dev)
    info = torch.empty(B, 4, dtype=torch.int32, device=dev)
    inl = torch.empty(B, h * w, dtype=torch.uint8, device=dev) if return_inliers else None
    C.gdrn_pnp_ransac(mask.data_ptr(), xyz.data_ptr(), coord_2d.data_ptr(), extents.data_ptr(), im_wh.data_ptr(), cams.data_ptr(),
                      B, h, w, _MASK_MODES[mask_loss_type], float(mask_thr), float(reproj_err), int(iters), float(confidence),
                      ws.data_ptr(), ws.numel() * 8, pose.data_ptr(), info.data_ptr(), inl.data_ptr() if inl is not None else None,
                      torch.cuda.current_stream().cuda_stream)
    out = dict(pose=pose, num_points=info[:, 0], num_inliers=info[:, 1], iterations=info[:, 2], ok=info[:, 3] != 0)
    if inl is not None:
        out["inliers"] = inl
    return out


def process_pnp_ransac(out_dict: dict, roi_coord_2d: torch.Tensor, roi_extents: torch.Tensor, im_wh, cams: torch.Tensor,
                       mask_loss_type: str = "L1", mask_thr: float = 0.5, use_net_trans: bool = True) -> torch.Tensor:
    """Batched equivalent of the pose part of `process_pnp_ransac` (gdrn_evaluator.py:316-421): rotation from RANSAC-PnP on the
    predicted coordinate maps, translation from the network (`out_dict["trans"]`, already decoded on the device by the model's
    test branch) when `use_net_trans`.  out_dict: the model's test-mode output with `TEST.USE_PNP` keys (mask, coor_x/y/z, trans).
    Returns [B,3,4]; instances without enough points get the reference's -100 marker."""
    xyz = torch.cat([out_dict["coor_x"], out_dict["coor_y"], out_dict["coor_z"]], dim=1)
    res = pnp_ransac(out_dict["mask"], xyz, roi_coord_2d, roi_extents, im_wh, cams, mask_loss_type=mask_loss_type, mask_thr=mask_thr)
    pose = res["pose"].clone()
    pose = torch.where(res["ok"].view(-1, 1, 1), pose, torch.full_like(pose, -100.0))
    if use_net_trans:
        pose[:, :, 3] = out_dict["trans"].to(pose.dtype)
    return pose


def _net_pose(out_dict: dict) -> tuple:
    R = out_dict["rot"].detach().float().reshape(-1, 3, 3).contiguous()
    t = out_dict["trans"].detach().float().reshape(-1, 3).contiguous()
    return R, t


def pnp_iterative(mask: torch.Tensor, xyz: torch.Tensor, coord_2d: torch.Tensor, extents: torch.Tensor, im_wh, cams: torch.Tensor,
                  R_init: torch.Tensor, t_init: torch.Tensor, mask_loss_type: str = "L1", mask_thr: float = 0.5,
                  max_iters: int = 20) -> dict:
    """cv2.solvePnP(SOLVEPNP_ITERATIVE, useExtrinsicGuess=True) for the whole batch on the device: OpenCV's Levenberg-Marquardt
    refinement of the reprojection error, started at (R_init [B,3,3], t_init [B,3]).  Points are selected like `pnp_ransac`, whose
    argument conventions this follows.  Like the evaluator's call, whose guess arrays are float32, the start rotation vector and
    the solution are rounded to float32 before R is formed.
    Returns dict(pose [B,3,4], num_points [B], iterations [B] (accepted LM steps), ok [B] (bool)).  Instances with fewer than 4
    selected points get ok = False and the initial pose."""
    if not mask.is_cuda:
        raise RuntimeError("gdr_net_b200.pnp_iterative runs on CUDA only; there is no CPU fallback")
    if mask_loss_type not in _MASK_MODES:
        raise NotImplementedError(f"unknown mask loss type: {mask_loss_type}")
    dev = mask.device
    B, _, h, w = xyz.shape
    f = lambda t: t.detach().to(dev).float().contiguous()  # noqa: E731
    mask, xyz, coord_2d, extents = _mask_planes(f(mask), mask_loss_type, B, h, w), f(xyz), f(coord_2d), f(extents).reshape(B, 3)
    if coord_2d.shape != (B, 2, h, w):
        raise ValueError(f"pnp_iterative: coord_2d {tuple(coord_2d.shape)} does not match xyz {tuple(xyz.shape)}")
    R_init, t_init = f(R_init).reshape(B, 3, 3), f(t_init).reshape(B, 3)
    if not torch.is_tensor(im_wh):
        im_wh = torch.tensor(im_wh, dtype=torch.float32)
    im_wh = f(im_wh)
    im_wh = (im_wh.reshape(1, 2).expand(B, 2) if im_wh.numel() == 2 else im_wh.reshape(B, 2)).contiguous()
    cams = f(cams)
    cams = (cams.reshape(1, 3, 3).expand(B, 3, 3) if cams.dim() == 2 else cams.reshape(B, 3, 3)).contiguous()
    nbytes = int(C.load().gdrn_pnp_iterative_workspace_bytes(B, h * w))
    ws = torch.empty((nbytes + 7) // 8, dtype=torch.float64, device=dev)
    pose = torch.empty(B, 3, 4, device=dev)
    info = torch.empty(B, 4, dtype=torch.int32, device=dev)
    C.gdrn_pnp_iterative(mask.data_ptr(), xyz.data_ptr(), coord_2d.data_ptr(), extents.data_ptr(), im_wh.data_ptr(), cams.data_ptr(),
                         R_init.data_ptr(), t_init.data_ptr(), B, h, w, _MASK_MODES[mask_loss_type], float(mask_thr), int(max_iters),
                         ws.data_ptr(), ws.numel() * 8, pose.data_ptr(), info.data_ptr(), torch.cuda.current_stream().cuda_stream)
    return dict(pose=pose, num_points=info[:, 0], iterations=info[:, 1], ok=info[:, 2] != 0)


def process_net_and_pnp(out_dict: dict, roi_coord_2d: torch.Tensor, roi_extents: torch.Tensor, im_wh, cams: torch.Tensor,
                        pnp_type: str = "iter", mask_loss_type: str = "L1", mask_thr: float = 0.5) -> torch.Tensor:
    """Batched equivalent of the pose part of `process_net_and_pnp` (gdrn_custom_evaluator.py:207-335, gdrn_evaluator.py:187-314):
    PnP on the predicted coordinate maps, initialised with the network pose (out_dict["rot"] [B,3,3], out_dict["trans"] [B,3]).

      * "iter":       cv2.solvePnP(ITERATIVE, useExtrinsicGuess) -> `pnp_iterative`; R and t from PnP;
      * "ransac":     cv2.solvePnPRansac(EPNP, 3 px, 20 iterations) -> `pnp_ransac(iters=20)` (EPnP ignores the guess); R and
                      t from PnP, but the network's t where |t_pnp - t_net| > 1 m;
      * "ransac_rot": as "ransac", t always from the network.

    Fewer than 4 selected points, or a failed RANSAC: the network pose.  The reference's `te > 1` fallback is not applied in
    "iter" mode because it never fires there: cv2 writes the solution into the float32 guess array that the reference then
    compares it with.  Deviation: with exactly 4 points OpenCV's RANSAC switches to P3P, which has no device kernel here; those
    instances keep the network pose in the two RANSAC modes ("iter" runs the LM on 4 points like cv2).
    Returns [B,3,4] float32, computed on the device without host synchronisation (capturable in a CUDA graph)."""
    R_net, t_net = _net_pose(out_dict)
    xyz = torch.cat([out_dict["coor_x"], out_dict["coor_y"], out_dict["coor_z"]], dim=1)
    if pnp_type == "iter":
        res = pnp_iterative(out_dict["mask"], xyz, roi_coord_2d, roi_extents, im_wh, cams, R_net, t_net, mask_loss_type=mask_loss_type,
                            mask_thr=mask_thr)
    elif pnp_type in ("ransac", "ransac_rot"):
        res = pnp_ransac(out_dict["mask"], xyz, roi_coord_2d, roi_extents, im_wh, cams, mask_loss_type=mask_loss_type,
                         mask_thr=mask_thr, iters=20)
    else:
        raise NotImplementedError(f"unknown net + PnP type: {pnp_type}")
    return combine_net_and_pnp(pnp_type, R_net, t_net, res["pose"], res["ok"])


def combine_net_and_pnp(pnp_type: str, R_net: torch.Tensor, t_net: torch.Tensor, pnp_pose: torch.Tensor, pnp_ok: torch.Tensor):
    """The per-ROI rules of `process_net_and_pnp` as tensor operations (any device, no host reads): R_net [B,3,3], t_net [B,3],
    pnp_pose [B,3,4], pnp_ok [B] bool -> [B,3,4]."""
    ok = pnp_ok.view(-1)
    R = torch.where(ok.view(-1, 1, 1), pnp_pose[:, :, :3], R_net)
    t_pnp = pnp_pose[:, :, 3]
    if pnp_type == "iter":
        use_t = ok
    elif pnp_type == "ransac":
        use_t = ok & ((t_pnp.double() - t_net.double()).norm(dim=1) <= 1.0)
    else:
        use_t = torch.zeros_like(ok)
    t = torch.where(use_t.view(-1, 1), t_pnp, t_net)
    return torch.cat([R, t.unsqueeze(-1)], dim=-1)


_NET_PNP_TYPES = {"net_iter_pnp": "iter", "net_ransac_pnp": "ransac", "net_ransac_pnp_rot": "ransac_rot"}


def process_pnp(cfg, out_dict: dict, roi_coord_2d: torch.Tensor, roi_extents: torch.Tensor, im_wh, cams: torch.Tensor) -> torch.Tensor:
    """The evaluator's `TEST.USE_PNP` dispatch (gdrn_custom_evaluator.py:160-171) on `cfg.TEST.PNP_TYPE` (case-insensitive):
    "ransac_pnp" -> `process_pnp_ransac`; "net_iter_pnp" / "net_ransac_pnp" / "net_ransac_pnp_rot" -> `process_net_and_pnp`
    with "iter" / "ransac" / "ransac_rot"; anything else raises NotImplementedError.  The mask head type and threshold come
    from cfg.MODEL.CDPN.ROT_HEAD (MASK_LOSS_TYPE, MASK_THR_TEST).  Returns the [B,3,4] poses."""
    pnp_type = cfg.TEST.PNP_TYPE.lower()
    r = cfg.MODEL.CDPN.ROT_HEAD
    kw = dict(mask_loss_type=r.MASK_LOSS_TYPE, mask_thr=r.MASK_THR_TEST)
    if pnp_type == "ransac_pnp":
        return process_pnp_ransac(out_dict, roi_coord_2d, roi_extents, im_wh, cams, **kw)
    if pnp_type in _NET_PNP_TYPES:
        return process_net_and_pnp(out_dict, roi_coord_2d, roi_extents, im_wh, cams, pnp_type=_NET_PNP_TYPES[pnp_type], **kw)
    raise NotImplementedError(f"unknown TEST.PNP_TYPE: {cfg.TEST.PNP_TYPE}")
