"""GPU: csrc/losses.cu against float64 autograd of the oracle's own functions (tests/loss_ref_common.py).

Covered: gdrn_head_glue_fwd, gdrn_pnp_pack_input, gdrn_pixel_loss_fwd + gdrn_loss_finalize, gdrn_head_bwd and gdrn_pose_loss
(train decode with its forward-mode Jacobian, the symmetric point-matching loss through the device table, the test-time
decode).  Every kernel is a deterministic function of its inputs, so the bounds are fp32 rounding (about 1e-5 of each
channel group) for two-plane outputs and the 16-bit storage rounding for single-plane outputs; each bound is derived at its
definition and the worst error measured on an H100 (80 GB HBM3) is recorded next to it."""
import math

import numpy as np
import pytest
import torch

from loss_ref_common import (HW, NCH, PIXEL_LOSSES, REPORT, check, glue64, grad_scale, nan_planes,  # noqa: E402 (tests/ is on
                             pixel_losses64, pose_losses64, pose_train64, rel_err, unit_roundoff)  # sys.path: rootdir conftest)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]

# Two-plane outputs: the value is hi + lo of the fp32 result (representation error ~2^-22), and each kernel output is a
# handful of fp32 operations on fp32 inputs (a few 6e-8 roundings; expf / logf are within 2 ulp).  1e-5 of the group maximum
# leaves a 10x margin over that budget and is three orders of magnitude below any dropped or mis-scaled term.
TOL2 = 1e-5


def tol_for(planes: int, fp32: float = TOL2) -> float:
    """Single-plane outputs are the fp32 result rounded to the storage format: at most one unit roundoff of the element
    (values in the fp16 subnormal range round to 2^-25 absolute, far below u of any group maximum), plus the fp32 error."""
    return fp32 if planes == 2 else unit_roundoff() + fp32


@pytest.fixture(scope="module", autouse=True)
def _setup():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    print("worst errors:", {k: f"{v:.2e}" for k, v in sorted(REPORT.items())})


def _C():
    from gdr_net_b200.capi import C

    return C


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ------------------------------------------------------------------------------------------------ per-pixel inputs
# (case, B): "edges" adds, in every crop, pixels whose masked residual is exactly 0 (xyz logit == gt, mask logit == trunc),
# labels 0 and 64, region logits of +-80 (exp overflows without the max shift), exact ties and near one-hot rows.
HEAD_CASES = [("base", 4), ("edges", 3), ("empty_crop", 3), ("empty_batch", 2), ("soft_mask", 3), ("b80", 80)]


def _head_inputs(case: str, B: int, seed: int = 0) -> dict:
    g = torch.Generator(device="cuda").manual_seed(1000 + seed + 17 * B + len(case))
    dev = "cuda"
    P = B * HW
    z = torch.randn(P, 72, device=dev, generator=g) * 2.0
    z[:, 69:] = float("nan")  # the three padding floats of a logit row are never read
    gt_xyz = torch.rand(B, 3, HW, device=dev, generator=g)
    m_vis = (torch.rand(B, HW, device=dev, generator=g) < 0.6).float()
    flip = torch.rand(B, HW, device=dev, generator=g) < 0.15
    m_trunc = torch.where(flip, 1.0 - m_vis, m_vis)  # m_trunc != m_visib on ~15 % of the pixels
    labels = torch.randint(0, 65, (B, HW), device=dev, generator=g)
    coord2d = torch.rand(B, 2, HW, device=dev, generator=g) * 2 - 1
    extents = torch.rand(B, 3, device=dev, generator=g) * 0.25 + 0.05
    if case in ("edges", "empty_crop", "b80", "soft_mask"):
        zv = z.view(B, HW, 72)
        for j in range(3):
            zv[:, 0:400:4, 1 + j] = gt_xyz[:, j, 0:400:4]  # |z*m - gt*m| == 0 exactly
        zv[:, 1:400:4, 0] = m_trunc[:, 1:400:4]  # |mask - trunc| == 0 exactly
        labels[:, :50] = 0
        labels[:, 50:100] = 64
        sgn = torch.where(torch.rand(B, 100, 65, device=dev, generator=g) < 0.5, -80.0, 80.0)
        zv[:, 400:500, 4:69] = sgn
        zv[:, 500:600, 4:69] = 0.7  # exact ties
        hot = torch.full((B, 100, 65), -30.0, device=dev)
        hot.scatter_(2, torch.randint(0, 65, (B, 100, 1), device=dev, generator=g), 30.0)
        zv[:, 600:700, 4:69] = hot  # near one-hot
    if case == "empty_crop":
        m_vis[0] = 0.0
    if case == "empty_batch":
        m_vis.zero_()
    if case == "soft_mask":
        # the formulas hold for any weight; a 0/1 mask hides a lost factor of m (every term it multiplies is 0 where m is 0)
        # and makes z * m exact, so |z m - gt m| is 0 where z == gt however it is evaluated.  With m = 0.3 or 0.7 it is 0
        # only if both products are rounded before the subtraction, as in the reference (an fma leaves z m's rounding error).
        m_vis = torch.tensor([0.0, 0.3, 0.7, 1.0], device=dev)[torch.randint(0, 4, (B, HW), device=dev, generator=g)]
    return dict(B=B, z=z.contiguous(), gt_xyz=gt_xyz, m_vis=m_vis.contiguous(), m_trunc=m_trunc.contiguous(),
                labels=labels.contiguous(), coord2d=coord2d, extents=extents)


def _glue(d, with_2d, planes):
    B = d["B"]
    out = nan_planes((B * HW, 128), planes)
    _C().gdrn_head_glue_fwd(d["z"].data_ptr(), d["coord2d"].data_ptr() if with_2d else None, d["extents"].data_ptr(), out.hi_ptr,
                            out.lo_ptr, B, HW, with_2d, _stream())
    return out


def _assert_zero_cols(out, c0: int, name: str):
    pad = out.buf[:, :, c0:]
    assert bool((pad == 0).all()), (name, "padding columns not exactly zero", int((pad != 0).sum()))


# ------------------------------------------------------------------------------------------------ A.1 glue
@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("with_2d", [1, 0])
@pytest.mark.parametrize("case,B", HEAD_CASES)
def test_head_glue_fwd(case, B, with_2d, planes):
    d = _head_inputs(case, B)
    out = _glue(d, with_2d, planes)
    torch.cuda.synchronize()
    got = out.float()
    ref = glue64(d["z"].double(), d["coord2d"].double(), d["extents"].double(), with_2d, B)
    nch, ro = NCH[with_2d], 5 if with_2d else 3
    tol = tol_for(planes)  # measured: planes 2 <= 7.4e-7 (softmax64), planes 1 <= 4.1e-4 (u of fp16 = 4.9e-4)
    for j, nm in enumerate("xyz"):
        check(f"glue {nm}[{case},{with_2d},{planes}]", got[:, j], ref[:, j], tol)
    if with_2d:
        check(f"glue coord2d[{case},{planes}]", got[:, 3:5], ref[:, 3:5], tol)
    check(f"glue softmax64[{case},{with_2d},{planes}]", got[:, ro:nch], ref[:, ro:nch], tol)
    _assert_zero_cols(out, nch, "glue")


# ------------------------------------------------------------------------------------------------ A.2 stand-alone Patch-PnP input
@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("c_feat,c_reg,with_ext", [(3, 64, True), (5, 64, True), (5, 64, False), (3, 0, True), (5, 0, True)])
def test_pnp_pack_input(c_feat, c_reg, with_ext, planes):
    """conv_pnp_net.py:111-125: xyz de-normalised by the extents when c_feat is 3 or 5 and extents are given, then
    cat(coor_feat, region) in NHWC, channels c_feat + c_reg .. 127 zero."""
    B = 3
    g = torch.Generator(device="cuda").manual_seed(c_feat * 100 + c_reg + with_ext)
    coor = torch.rand(B, c_feat, HW, device="cuda", generator=g)
    region = torch.softmax(torch.randn(B, 64, HW, device="cuda", generator=g), 1)[:, :c_reg].contiguous() if c_reg else None
    ext = torch.rand(B, 3, device="cuda", generator=g) * 0.25 + 0.05
    out = nan_planes((B * HW, 128), planes)
    _C().gdrn_pnp_pack_input(coor.data_ptr(), c_feat, region.data_ptr() if region is not None else None, c_reg,
                             ext.data_ptr() if with_ext else None, out.hi_ptr, out.lo_ptr, B, HW, _stream())
    torch.cuda.synchronize()
    c64 = coor.double()
    if with_ext:
        c64 = torch.cat([(c64[:, :3] - 0.5) * ext.double().view(B, 3, 1), c64[:, 3:]], 1)
    parts = [c64] + ([region.double()] if c_reg else [])
    ref = torch.cat(parts, 1).permute(0, 2, 1).reshape(B * HW, c_feat + c_reg)
    got = out.float()
    tol = tol_for(planes)  # measured: planes 2 <= 1.8e-7, planes 1 <= 4.7e-4
    for j in range(c_feat):
        check(f"pack coor{j}[{c_feat},{with_ext},{planes}]", got[:, j], ref[:, j], tol)
    if c_reg:
        check(f"pack region[{c_feat},{planes}]", got[:, c_feat:c_feat + c_reg], ref[:, c_feat:], tol)
    _assert_zero_cols(out, c_feat + c_reg, "pack")


# ------------------------------------------------------------------------------------------------ A.3 pixel losses
def _pixel_sums(d):
    sums = torch.full((6,), float("nan"), dtype=torch.float64, device="cuda")
    _C().gdrn_pixel_loss_fwd(d["z"].data_ptr(), d["gt_xyz"].data_ptr(), d["m_vis"].data_ptr(), d["m_trunc"].data_ptr(),
                             d["labels"].data_ptr(), sums.data_ptr(), d["B"], HW, _stream())
    return sums


@pytest.mark.parametrize("case,B", HEAD_CASES)
def test_pixel_loss_fwd_and_finalize(case, B):
    """B = 80: 80 * 4096 pixels exceed px_grid's cap (SMs * 16 CTAs of 128 threads on a 132-SM H100), so the grid-stride
    loop takes a second turn; B = 64 fits in one."""
    d = _head_inputs(case, B)
    sums = _pixel_sums(d)
    losses = torch.full((8,), float("nan"), device="cuda")
    vis_out = torch.full((2,), float("nan"), device="cuda")
    pose_sums = torch.zeros(4, dtype=torch.float64, device="cuda")
    vis = torch.zeros(B, 2, device="cuda")
    _C().gdrn_loss_finalize(sums.data_ptr(), pose_sums.data_ptr(), vis.data_ptr(), losses.data_ptr(), vis_out.data_ptr(), B, HW, 1,
                            _stream())
    torch.cuda.synchronize()
    L = pixel_losses64(d["z"].double(), d["gt_xyz"].double(), d["m_vis"].double(), d["m_trunc"].double(), d["labels"], B)
    # sum(m_visib): fp32 partials of 0 / 1 masks are exact integers; the 0.3 / 0.7 masks round (measured 3.0e-9)
    check(f"pixel sum_m_visib[{case}]", sums[5:6], d["m_vis"].double().sum().view(1), 1e-7)
    # Per pixel, fp32 rounding of |z m - gt m| and of logsumexp - z_label (at most ~|max logit| * 6e-8 = 5e-6 absolute for
    # the +-80 rows); per CTA an fp32 sum of <= 384 pixels (<= 9 roundings deep in the shuffle tree), across CTAs fp64
    # atomics.  Relative to the loss this is <= 1e-6 with random signs; the bound leaves 2x.  Measured: <= 6.5e-8.
    for i, k in enumerate(PIXEL_LOSSES):
        check(f"pixel {k}[{case}]", losses[i:i + 1], L[k].view(1), 2e-6)


# ------------------------------------------------------------------------------------------------ A.4 head backward
def _din(B, planes, seed):
    """Gradient of the Patch-PnP input as the dgrad of its first conv delivers it; all 128 columns carry values, so a kernel
    that read a column it must ignore (the 2-D coordinates, the padding) would disagree with the reference."""
    from gdr_net_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B * HW, 128, device="cuda", generator=g) * (5e-4 * grad_scale())
    return ops.PT.from_float(x, planes)


@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("with_2d", [1, 0])
@pytest.mark.parametrize("case,B", HEAD_CASES)
def test_head_bwd(case, B, with_2d, planes):
    """d/d logits of sum_i gw_i L_i + <din, glue(logits)>: the five pixel losses and the glue's backward in one pass."""
    d = _head_inputs(case, B)
    sums = _pixel_sums(d)
    gw = torch.tensor([0.7, -1.3, 2.1, 0.4, 1.7, 1.0, 1.0, 1.0], device="cuda") * grad_scale()
    nch = NCH[with_2d]
    for dmode in (None, 1, 2):
        din = _din(B, dmode, 7 + B) if dmode else None
        out = nan_planes((B * HW, 128), planes)
        _C().gdrn_head_bwd(d["z"].data_ptr(), d["gt_xyz"].data_ptr(), d["m_vis"].data_ptr(), d["m_trunc"].data_ptr(),
                           d["labels"].data_ptr(), sums.data_ptr(), gw.data_ptr(), din.hi_ptr if din else None,
                           din.lo_ptr if din else None, d["extents"].data_ptr(), out.hi_ptr, out.lo_ptr, B, HW, with_2d, _stream())
        torch.cuda.synchronize()
        z = d["z"].double().requires_grad_(True)
        L = pixel_losses64(z, d["gt_xyz"].double(), d["m_vis"].double(), d["m_trunc"].double(), d["labels"], B)
        tot = sum(float(gw[i]) * L[k] for i, k in enumerate(PIXEL_LOSSES))
        if din is not None:
            tot = tot + (din.float().double()[:, :nch] * glue64(z, d["coord2d"].double(), d["extents"].double(), with_2d, B)).sum()
        (ref,) = torch.autograd.grad(tot, z)
        got = out.float()
        tag = f"[{case},{with_2d},{planes},din{dmode}]"
        # the mask channel (gw/(B*HW) per pixel) is ~1e-5 of the region gradient: compared on its own scale.
        # Measured: planes 2 <= 1.4e-6 (region channels, where the softmax backward subtracts), <= 1.5e-7 for mask and
        # xyz; planes 1 <= 4.8e-4.
        tol = tol_for(planes)
        check(f"head_bwd mask{tag}", got[:, 0], ref[:, 0], tol)
        for j, nm in enumerate("xyz"):
            check(f"head_bwd {nm}{tag}", got[:, 1 + j], ref[:, 1 + j], tol)
        check(f"head_bwd bg{tag}", got[:, 4], ref[:, 4], tol)
        check(f"head_bwd regions{tag}", got[:, 5:69], ref[:, 5:69], tol)
        _assert_zero_cols(out, 69, "head_bwd")


# ------------------------------------------------------------------------------------------------ A.5-A.7 pose decode and losses
def _rotations(n, g):
    q = torch.randn(n, 4, generator=g, dtype=torch.float64)
    q = q / q.norm(dim=1, keepdim=True)
    from oracle import gdrn_oracle as O

    return O.quat2mat(q)


def _pose_inputs(B: int, seed: int, on_axis=(), degenerate=()) -> dict:
    """Network outputs and crop geometry in the ranges of the B = 64 benchmark batch (LM-like intrinsics, crops of 80-250
    px, z ratios around 1).  on_axis: crops whose SITE centroid lands on the principal point (translation on the optical
    axis); degenerate: crops whose first rot6d column has norm 5e-13 (< 1e-12, the F.normalize clamp)."""
    g = torch.Generator().manual_seed(seed)
    K = torch.tensor([[572.4114, 0.0, 325.2611], [0.0, 573.57043, 242.04899], [0.0, 0.0, 1.0]])
    cams = K.expand(B, 3, 3).clone()
    centers = torch.stack([325.26 + (torch.rand(B, generator=g) - 0.5) * 300, 242.05 + (torch.rand(B, generator=g) - 0.5) * 200], 1)
    whs = 80 + torch.rand(B, 2, generator=g) * 170
    ratios = 0.4 + torch.rand(B, generator=g) * 1.2
    pred = torch.full((B, 16), float("nan"))  # cols 9..15 are never read
    pred[:, :6] = torch.randn(B, 6, generator=g)
    pred[:, 6:8] = torch.randn(B, 2, generator=g) * 0.05
    pred[:, 8] = 0.8 + torch.rand(B, generator=g) * 0.4
    for b in on_axis:
        pred[b, 6:8] = 0.0
        centers[b] = torch.tensor([cams[b, 0, 2], cams[b, 1, 2]])
    for b in degenerate:
        pred[b, :3] = torch.tensor([3e-13, 4e-13, 0.0])
    gt_ratio = pred[:, 6:9] + torch.randn(B, 3, generator=g) * 0.02
    extents = 0.05 + torch.rand(B, 3, generator=g) * 0.25
    gt_rot = _rotations(B, g).float()
    gt_trans = torch.randn(B, 3, generator=g) * 0.05 + torch.tensor([0.0, 0.0, 0.9])
    a = dict(pred=pred, cams=cams, centers=centers, whs=whs, ratios=ratios.contiguous(), extents=extents, gt_rot=gt_rot,
             gt_trans=gt_trans, gt_ratio=gt_ratio.contiguous())
    return {k: v.float().contiguous().cuda() for k, v in a.items()}


def _add_points(a: dict, n: int, seed: int, sym_infos=None):
    """n model points per crop, uniform in the extent box, drawn so that every component of w (R - R_gt) p is at least 2e-5 |p|
    away from 0 in float64.  The L1 point-matching gradient is sign(e) p: where |e| is within the fp32 error of R (~1e-6) its
    sign is a coin flip and one flipped term moves the gradient by 2/n of itself, which is a property of the loss and not
    of the kernel.  Components whose row of R - R_gt is exactly zero (constructed crops) are exactly zero in both."""
    from oracle import gdrn_oracle as O

    B = a["pred"].shape[0]
    R64, _ = pose_train64(a["pred"][:, :9].double(), a)
    Rgt = a["gt_rot"].double()
    if sym_infos is not None:
        Rgt = O.closest_rot_batch(R64, Rgt, sym_infos).to(R64)
    D = R64 - Rgt
    g = torch.Generator(device="cuda").manual_seed(seed)
    cand = ((torch.rand(B, 8 * n, 3, device="cuda", generator=g) - 0.5) * a["extents"][:, None, :]).float()
    e = torch.einsum("bij,bkj->bki", D, cand.double())
    pn = cand.double().norm(dim=2, keepdim=True)
    rowzero = (D.abs().amax(2) == 0)[:, None, :]
    ok = ((e.abs() >= 2e-5 * pn) | rowzero).all(2)
    order = torch.sort((~ok).to(torch.int8), dim=1, stable=True).indices[:, :n]
    assert bool(torch.gather(ok, 1, order).all()), "not enough well-separated points"
    a["points"] = torch.gather(cand, 1, order[..., None].expand(B, n, 3)).contiguous()
    return a


def _pose_kernel(a: dict, gw3, planes: int, syms=None, sym_idx=None):
    from gdr_net_b200 import ops

    B, n = a["pred"].shape[0], a["points"].shape[1]
    out = dict(rot=torch.full((B, 3, 3), float("nan"), device="cuda"), trans=torch.full((B, 3), float("nan"), device="cuda"),
               sums=torch.full((4,), float("nan"), dtype=torch.float64, device="cuda"), vis=torch.full((B, 2), float("nan"), device="cuda"),
               dy=nan_planes((B, 64), planes))
    _C().gdrn_pose_loss(a["pred"].data_ptr(), 16, a["cams"].data_ptr(), a["centers"].data_ptr(), a["whs"].data_ptr(),
                        a["ratios"].data_ptr(), a["extents"].data_ptr(), a["points"].data_ptr(), a["gt_rot"].data_ptr(),
                        a["gt_trans"].data_ptr(), a["gt_ratio"].data_ptr(), ops.ptr(syms), ops.ptr(sym_idx), gw3.data_ptr(),
                        out["rot"].data_ptr(), out["trans"].data_ptr(), out["sums"].data_ptr(), out["vis"].data_ptr(), out["dy"].hi_ptr,
                        out["dy"].lo_ptr, B, n, 1, 1e-4, _stream())  # as Engine._pose (engine.py:572-577)
    losses = torch.full((8,), float("nan"), device="cuda")
    out["vis_out"] = torch.full((2,), float("nan"), device="cuda")
    pix = torch.zeros(6, dtype=torch.float64, device="cuda")
    _C().gdrn_loss_finalize(pix.data_ptr(), out["sums"].data_ptr(), out["vis"].data_ptr(), losses.data_ptr(), out["vis_out"].data_ptr(),
                            B, HW, n, _stream())
    torch.cuda.synchronize()
    out["losses"] = losses
    return out


# dY = cpm J^T G: each entry is a 9-term fp32 dot product of G (sums of n sign(e) w p terms) with the forward-mode Jacobian,
# whose terms cancel to a few percent of their magnitude for the centroid entries: 5e-5.  Measured, planes 2: centroid
# 1.1e-5, rot6d 1.2e-6, z 2.2e-6; planes 1: <= 4.4e-4.
TOL_DY = 5e-5


def _check_pose(tag, a, out, gw3, planes, sym_infos=None, tol_rot=TOL2, tol_dy=TOL_DY, groups=("rot6d", "centroid", "z")):
    from oracle import gdrn_oracle as O

    pred9 = a["pred"][:, :9].double().requires_grad_(True)
    R, T, L = pose_losses64(pred9, a, sym_infos)
    (ref,) = torch.autograd.grad(sum(float(gw3[i]) * L[i] for i in range(3)), pred9)
    check(f"pose out_rot{tag}", out["rot"], R.detach(), tol_rot)
    check(f"pose out_trans{tag}", out["trans"], T.detach(), 1e-6)  # 3-4 fp32 operations: measured <= 5.3e-8
    # loss_PM_R: fp32 sums of |w (R p - R_gt p)| over <= 24 points per thread, then shuffles: measured <= 1.1e-7
    for i, nm in enumerate(("PM_R", "centroid", "z")):
        check(f"pose loss_{nm}{tag}", out["losses"][5 + i:6 + i], L[i].detach().view(1), 1e-5)
    # vis: re (deg) and te per crop, from the kernel's own R and T in fp64 (ill-conditioned acos near re = 0 is not the
    # kernel's), then the fp32 batch mean of model_utils.py:40-52
    R_k, T_k = out["rot"].double().cpu().numpy(), out["trans"].double().cpu()
    re = torch.tensor([O._re_deg(R_k[b], a["gt_rot"][b].double().cpu().numpy()) for b in range(R_k.shape[0])])
    te = (a["gt_trans"].double().cpu() - T_k).norm(dim=1)
    check(f"pose vis re{tag}", out["vis"][:, 0].cpu(), re, 1e-6)  # measured 0 (te 5.3e-8, mean 1.2e-7)
    check(f"pose vis te{tag}", out["vis"][:, 1].cpu(), te, 1e-6)
    mre, mte = O.mean_re_te(out["trans"], out["rot"], a["gt_trans"], a["gt_rot"])
    check(f"pose vis mean{tag}", out["vis_out"].cpu().double(), torch.tensor([float(mre), float(mte)], dtype=torch.float64), 1e-5)
    got = out["dy"].float()
    sl = dict(rot6d=slice(0, 6), centroid=slice(6, 8), z=slice(8, 9))
    for gname in groups:
        check(f"pose dY {gname}{tag}", got[:, sl[gname]], ref[:, sl[gname]], tol_for(planes, tol_dy))
    assert bool((out["dy"].buf[:, :, 9:] == 0).all()), "dY columns 9..63 not exactly zero"


# Rotation entries go through ~30 fp32 operations of the dual-number decode (normalise, cross, normalise, quaternion, 3x3
# product) with O(1) condition numbers away from the optical axis: measured <= 2.0e-6; bound 1e-5.  dY: TOL_DY above.
@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("n_pts", [1, 100, 128, 129, 3000])
@pytest.mark.parametrize("B", [1, 7, 64])
def test_pose_loss_train(B, n_pts, planes):
    a = _add_points(_pose_inputs(B, seed=B * 7 + n_pts), n_pts, seed=n_pts)
    gw3 = torch.tensor([1.3, -0.6, 0.9], device="cuda") * grad_scale()
    out = _pose_kernel(a, gw3, planes)
    _check_pose(f"[B{B},n{n_pts},{planes}]", a, out, gw3, planes)


@pytest.mark.parametrize("planes", [1, 2])
def test_pose_loss_on_optical_axis(planes):
    """Both crops' translations lie on the optical axis: the axis (-ray_y, ray_x, 0) is exactly zero and the 1e-4 in its norm
    keeps the decode differentiable.  The centroid gradient then carries d(axis)/dt ~ 1/1e-4 times sin(angle / 2), where
    angle = acos(z / (z + 1e-4)) ~ 0.014: ray_z is 1 - 1e-4 to one fp32 ulp (6e-8), so 1 - ray_z and the angle carry a
    relative error of up to 6e-4 / 2 = 3e-4 that no fp32 evaluation avoids.  That group is bounded by 1e-3 (measured
    1.6e-4 with two planes, 4.4e-4 with one); rotation and the other groups keep their fp32 bounds (the rotation is exactly the allocentric one)."""
    a = _add_points(_pose_inputs(2, seed=5, on_axis=(0, 1)), 100, seed=3)
    gw3 = torch.tensor([0.8, 1.4, -0.7], device="cuda") * grad_scale()
    out = _pose_kernel(a, gw3, planes)
    _check_pose(f"[axis,{planes}]", a, out, gw3, planes, groups=("rot6d", "z"))
    pred9 = a["pred"][:, :9].double().requires_grad_(True)
    _, _, L = pose_losses64(pred9, a)
    (ref,) = torch.autograd.grad(sum(float(gw3[i]) * L[i] for i in range(3)), pred9)
    check(f"pose dY centroid on-axis[{planes}]", out["dy"].float()[:, 6:8], ref[:, 6:8], tol_for(planes, 1e-3))


@pytest.mark.parametrize("planes", [1, 2])
def test_pose_loss_degenerate_rot6d(planes):
    """Crop 0's first rot6d column has norm 5e-13 < 1e-12: F.normalize divides by the clamp 1e-12 (a constant, so the norm
    contributes no derivative) and the derivative of that column is 1e12 times larger.  The point-matching weight is scaled
    by 1e-12 so that the 16-bit dY stays in range; crop 1 is regular."""
    a = _add_points(_pose_inputs(2, seed=9, degenerate=(0,)), 64, seed=4)
    gw3 = torch.tensor([1e-12, 0.8, -1.1], device="cuda") * grad_scale()
    out = _pose_kernel(a, gw3, planes)
    _check_pose(f"[degenerate,{planes}]", a, out, gw3, planes)


def _cube_rotations():
    """The 24 rotations of the cube: signed permutation matrices with determinant +1 (exact in any precision)."""
    import itertools

    out = []
    for perm in itertools.permutations(range(3)):
        for signs in itertools.product((1.0, -1.0), repeat=3):
            m = np.zeros((3, 3))
            for i, j in enumerate(perm):
                m[i, j] = signs[i]
            if round(np.linalg.det(m)) == 1:
                out.append(m)
    return out


def _rz(t):
    c, s = math.cos(t), math.sin(t)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])


@pytest.mark.parametrize("planes", [1, 2])
def test_pose_loss_symmetric(planes):
    """Closest symmetric ground truth through the device table (pose_utils.py:430-482 restated on the device):
    crops 0, 2: asymmetric (count 0) between symmetric ones;
    crop 1: 628 rotations about z (more than the CTA's 128 threads, identity first), random prediction;
    crop 3: a 4-element table with the identity, random prediction;
    crop 4: an exact tie.  The prediction is exactly I (rot6d (1,0,0,0,1,0) on the optical axis) and R_gt = Rz(180).  In a
    628-entry table of cube rotations that are all worse, Rz(90) sits at index 5 and Rz(-90) at index 133 (the same thread
    of the 128-thread scan): both give geodesic error exactly pi/2, so the first (5) must win like the reference's strict
    `<` scan, and the two choices give different point-matching gradients;
    crop 5: 628 rotations about z again, another random prediction."""
    B, n = 6, 200
    a = _pose_inputs(B, seed=21, on_axis=(4,))
    a["pred"][4, :6] = torch.tensor([1.0, 0.0, 0.0, 0.0, 1.0, 0.0], device="cuda")
    a["gt_rot"][4] = torch.tensor(np.diag([-1.0, -1.0, 1.0]), dtype=torch.float32, device="cuda")
    cont = np.stack([_rz(2 * math.pi * k / 628) for k in range(628)]).astype(np.float32)
    four = np.stack([np.eye(3), np.diag([-1.0, -1.0, 1.0]), np.diag([1.0, -1.0, -1.0]), np.diag([-1.0, 1.0, -1.0])]).astype(np.float32)
    M = np.diag([-1.0, -1.0, 1.0])  # R_gt^T R of crop 4
    worse = [c for c in _cube_rotations() if np.sum(M * c) < 1]  # trace(R^T R_gt S) < 1: error > pi/2
    tie = np.stack([worse[k % len(worse)] for k in range(628)])
    tie[5], tie[133] = _rz(math.pi / 2).round(), _rz(-math.pi / 2).round()
    tie = tie.astype(np.float32)
    sym_infos = [None, cont, None, four, tie, cont]
    rows, idx = [], []
    for s in sym_infos:
        idx.append((sum(len(r) for r in rows), 0 if s is None else len(s)))
        if s is not None:
            rows.append(s)
    syms = torch.from_numpy(np.concatenate(rows)).cuda().contiguous()
    sym_idx = torch.tensor(idx, dtype=torch.int32, device="cuda")
    _add_points(a, n, seed=6, sym_infos=[None if s is None else torch.from_numpy(s) for s in sym_infos])
    gw3 = torch.tensor([1.1, 0.5, -0.9], device="cuda") * grad_scale()
    out = _pose_kernel(a, gw3, planes, syms, sym_idx)
    assert bool((out["rot"][4] == torch.eye(3, device="cuda")).all()), out["rot"][4]  # the tie needs R == I exactly
    sym_t = [None if s is None else torch.from_numpy(s) for s in sym_infos]
    _check_pose(f"[sym,{planes}]", a, out, gw3, planes, sym_infos=sym_t, groups=("rot6d", "z"))
    pred9 = a["pred"][:, :9].double().requires_grad_(True)
    _, _, L = pose_losses64(pred9, a, sym_t)
    (ref,) = torch.autograd.grad(sum(float(gw3[i]) * L[i] for i in range(3)), pred9)
    # crop 4 lies on the optical axis: the centroid group carries the acos conditioning of test_pose_loss_on_optical_axis
    check(f"pose dY centroid on-axis[sym,{planes}]", out["dy"].float()[:, 6:8], ref[:, 6:8], tol_for(planes, 1e-3))
    # crop 4 alone, so that its dY is not compared on the scale of another crop's
    check(f"pose dY tie crop[{planes}]", out["dy"].float()[4, :6], ref[4, :6], tol_for(planes, TOL_DY))


def test_pose_decode_test_time():
    """do_loss = 0, eps = 0, every loss pointer null, exactly as Engine._tail_inference calls it (engine.py:353-356), against
    the reference's numpy test-time decode (pose_from_pred_centroid_z.py:52-141, utils.py:39-94).  Crop 0 lies on the optical
    axis (angle 0: the allocentric rotation is returned unchanged).  Measured: rotation <= 5.5e-7, translation <= 3.3e-8."""
    from oracle import gdrn_oracle as O

    B = 7
    a = _pose_inputs(B, seed=33, on_axis=(0,))
    out_rot = torch.full((B, 3, 3), float("nan"), device="cuda")
    out_trans = torch.full((B, 3), float("nan"), device="cuda")
    _C().gdrn_pose_loss(a["pred"].data_ptr(), 16, a["cams"].data_ptr(), a["centers"].data_ptr(), a["whs"].data_ptr(),
                        a["ratios"].data_ptr(), a["extents"].data_ptr(), None, None, None, None, None, None, None,
                        out_rot.data_ptr(), out_trans.data_ptr(), None, None, None, None, B, 0, 0, 0.0, _stream())
    torch.cuda.synchronize()
    p64 = a["pred"][:, :9].double().cpu()
    rot_allo = O.ortho6d_to_mat(p64[:, :6])
    R, T = O.pose_decode_test(rot_allo, p64[:, 6:9], a["cams"].double().cpu(), a["centers"].double().cpu(),
                              a["ratios"].double().cpu(), a["whs"].double().cpu())
    check("decode_test rot", out_rot.cpu(), R, 1e-5)
    check("decode_test trans", out_trans.cpu(), T, 1e-6)
    assert rel_err(out_rot[0].cpu(), rot_allo[0]) < 1e-6  # on the axis: the allocentric rotation itself
