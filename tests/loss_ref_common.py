"""Float64 references for the op tests of csrc/losses.cu and of the BatchNorm / small backward kernels.

Every reference is built from the kernel's exact inputs (the fp32 logits as passed, `PT.float()` of planar operands) and run
in float64 through the oracle's own functions (oracle/gdrn_oracle.py, pinned to the unmodified reference by
tests/test_oracle_golden.py), so it differs from a kernel only by the kernel's fp32 rounding and, for a single-plane
output, by the rounding to the 16-bit storage format.  Results are compared per channel group, each group scaled by its
own magnitude: a whole-tensor max-normalised error hides a wrong factor in a group that is orders of magnitude smaller
than the largest one (the mask-channel gradient is ~1e-5 of the region gradient)."""
import torch
import torch.nn.functional as F

from oracle import gdrn_oracle as O

HW = 4096  # 64 x 64 head output per crop
NCH = {1: 69, 0: 67}  # Patch-PnP input channels with / without the 2-D coordinates (GDRN.py:171-173)

REPORT = {}  # name -> worst error seen in this session (printed by `check`, recorded next to each bound)


def unit_roundoff() -> float:
    """Unit roundoff of the 16-bit storage format: a single-plane output is the fp32 value rounded to it."""
    from gdr_net_b200 import ops

    return float(torch.finfo(ops.storage_format()[0]).eps) / 2


def grad_scale() -> float:
    """The engine carries fp16 gradients with a static loss scale of 1024 (Engine.grad_scale); the tests do the same so that
    the smallest gradients (the mask channel, ~gw / (B * 4096)) stay out of the fp16 subnormal range."""
    from gdr_net_b200 import ops

    return 1024.0 if ops.storage_format()[2] == "fp16" else 1.0


def rel_err(got, ref) -> float:
    """max |got - ref| / max |ref|; a reference that is exactly zero must be matched exactly (returns inf otherwise)."""
    got, ref = got.double(), ref.double()
    den = float(ref.abs().max()) if ref.numel() else 0.0
    num = float((got - ref).abs().max()) if ref.numel() else 0.0
    if den == 0.0:
        return 0.0 if num == 0.0 else float("inf")
    return num / den


def check(name: str, got, ref, tol: float, err: float = None):
    e = rel_err(got, ref) if err is None else err
    key = name.split("[")[0]
    last = name.rstrip("]").split(",")[-1].split("[")[-1] if name.endswith("]") else ""
    if last in ("1", "2"):
        key += f" planes{last}"
    REPORT[key] = max(REPORT.get(key, 0.0), e)
    print(f"{name}: {e:.3e} (bound {tol:.1e})")
    assert e <= tol, (name, e, tol)


def nan_planes(shape, planes, device="cuda"):
    """A planar output pre-filled with NaN, so that an element the kernel does not write fails every comparison."""
    from gdr_net_b200 import ops

    return ops.PT(shape, planes, device=device, buf=torch.full((planes,) + tuple(shape), float("nan"),
                                                                 dtype=ops.storage_format()[0], device=device))


# ------------------------------------------------------------------------------------------------ head: glue + pixel losses
def head_nchw(z: torch.Tensor, B: int) -> torch.Tensor:
    """[B * 4096, 72] pixel-major logits (the 1x1 conv's fp32 output) -> the reference's NCHW head [B, 69, 64, 64]."""
    return z[:, :69].reshape(B, 64, 64, 69).permute(0, 3, 1, 2)


def pixel_losses64(z: torch.Tensor, gt_xyz, m_vis, m_trunc, labels, B: int) -> dict:
    """The five per-pixel losses of oracle.gdrn_losses (GDRN.py:341-400) on the float64 logits z [B * 4096, 72]; the pose
    part of the oracle call gets inert placeholders and is dropped."""
    head = head_nchw(z, B)
    dt, dev = z.dtype, z.device
    batch = dict(roi_xyz=gt_xyz.view(B, 3, 64, 64).to(dt), roi_mask_visib=m_vis.view(B, 64, 64).to(dt),
                 roi_mask_trunc=m_trunc.view(B, 64, 64).to(dt), roi_region=labels.view(B, 64, 64),
                 ego_rot=torch.eye(3, dtype=dt, device=dev).expand(B, 3, 3), roi_points=torch.zeros(B, 1, 3, dtype=dt, device=dev),
                 roi_extent=torch.ones(B, 3, dtype=dt, device=dev), roi_trans_ratio=torch.zeros(B, 3, dtype=dt, device=dev))
    L = O.gdrn_losses(head, torch.eye(3, dtype=dt, device=dev).expand(B, 3, 3), torch.zeros(B, 3, dtype=dt, device=dev), batch)
    return {k: L[k] for k in ("loss_coor_x", "loss_coor_y", "loss_coor_z", "loss_mask", "loss_region")}


PIXEL_LOSSES = ("loss_coor_x", "loss_coor_y", "loss_coor_z", "loss_mask", "loss_region")


def glue64(z: torch.Tensor, coord2d, extents, with_2d: int, B: int) -> torch.Tensor:
    """The Patch-PnP input of GDRN.py:156-173 + conv_pnp_net.py:120-125 in pixel-major layout [B * 4096, 69 | 67]:
    (xyz - 0.5) * extent | coord2d | softmax(region[:, 1:]) -- the oracle's gdrn_forward / pnp_forward steps."""
    head = head_nchw(z, B)
    xyz = (head[:, 1:4] - 0.5) * extents.to(z.dtype).view(B, 3, 1, 1)
    parts = [xyz]
    if with_2d:
        parts.append(coord2d.view(B, 2, 64, 64).to(z.dtype))
    parts.append(F.softmax(head[:, 5:], dim=1))
    return torch.cat(parts, 1).permute(0, 2, 3, 1).reshape(B * HW, -1)


# ------------------------------------------------------------------------------------------------ pose decode + pose losses
def pose_train64(pred9: torch.Tensor, a: dict):
    """(R_ego, T) of the differentiable train decode (rot_reps.py:34-49, pose_from_pred_centroid_z.py:144-227 with
    eps = 1e-4) on the float64 network outputs pred9 [B, 9] = rot6d | centroid dx, dy | z."""
    dt = pred9.dtype
    rot_allo = O.ortho6d_to_mat(pred9[:, :6])
    return O.pose_decode_train(rot_allo, pred9[:, 6:9], a["cams"].to(dt), a["centers"].to(dt), a["ratios"].to(dt),
                               a["whs"].to(dt))


def pose_losses64(pred9: torch.Tensor, a: dict, sym_infos=None):
    """loss_PM_R, loss_centroid, loss_z of oracle.gdrn_losses (pm_loss.py:82-114, GDRN.py:439-471) on the float64 decode;
    the closest symmetric ground truth is oracle.closest_rot_batch when sym_infos is given."""
    dt, dev = pred9.dtype, pred9.device
    B = pred9.shape[0]
    R, T = pose_train64(pred9, a)
    batch = dict(roi_xyz=torch.zeros(B, 3, 1, 1, dtype=dt, device=dev), roi_mask_visib=torch.zeros(B, 1, 1, dtype=dt, device=dev),
                 roi_mask_trunc=torch.zeros(B, 1, 1, dtype=dt, device=dev), roi_region=torch.zeros(B, 1, 1, dtype=torch.long, device=dev),
                 ego_rot=a["gt_rot"].to(dt), roi_points=a["points"].to(dt), roi_extent=a["extents"].to(dt),
                 roi_trans_ratio=a["gt_ratio"].to(dt), sym_info=sym_infos)
    L = O.gdrn_losses(torch.zeros(B, 69, 1, 1, dtype=dt, device=dev), R, pred9[:, 6:9], batch, pm_sym=sym_infos is not None)
    return R, T, (L["loss_PM_R"], L["loss_centroid"], L["loss_z"])
