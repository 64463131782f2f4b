"""Deterministic synthetic crops / targets / weights for parity tests and bench.

Follows the input contract of the reference hot path (SURVEY.md 8a row a0, 8d):
reference `core/gdrn_modeling/engine_utils.py:6-60` (batch_data) and
`core/gdrn_modeling/data_loader.py:617-632` (SITE translation targets).

All randomness comes from CPU `torch.Generator`s so that the same tensors are
produced in the build container, on the GPU box, by the oracle and by the
product path.
"""
from __future__ import annotations

import math
import zlib

import torch

LM_K = [[572.4114, 0.0, 325.2611], [0.0, 573.57043, 242.04899], [0.0, 0.0, 1.0]]  # reference ref/lm_full.py:106


def _gen(seed: int, tag: str) -> torch.Generator:
    g = torch.Generator(device="cpu")
    g.manual_seed((seed * 1000003 + zlib.crc32(tag.encode())) % (2**63 - 1))
    return g


def random_rotations(n: int, g: torch.Generator) -> torch.Tensor:
    a = torch.randn(n, 3, 3, generator=g, dtype=torch.float64)
    q, r = torch.linalg.qr(a)
    d = torch.diagonal(r, dim1=-2, dim2=-1).sign()
    q = q * d[:, None, :]
    det = torch.linalg.det(q)
    q[:, :, 0] *= det[:, None]
    return q.float()


def discrete_symmetries(kind: str) -> torch.Tensor | None:
    """Model-to-model symmetry rotation sets like `sym_info` (reference misc.py:233)."""
    if kind == "none":
        return None

    def rz(a):
        c, s = math.cos(a), math.sin(a)
        return [[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]]

    if kind == "z2":
        return torch.tensor([rz(0.0), rz(math.pi)], dtype=torch.float32)
    if kind == "z4":
        return torch.tensor([rz(i * math.pi / 2) for i in range(4)], dtype=torch.float32)
    if kind == "cont":  # continuous axis discretised (reference uses up to 314·n steps; 64 keeps tests quick)
        return torch.tensor([rz(i * 2 * math.pi / 64) for i in range(64)], dtype=torch.float32)
    raise ValueError(kind)


_YCBV_SYMS: list = []


def ycbv_like_symmetries() -> list:
    """21 entries: None (asymmetric) or a [K,3,3] float32 tensor of model-to-model symmetry rotations; built once."""
    if not _YCBV_SYMS:
        def rot(axis, a):
            c, s = math.cos(a), math.sin(a)
            if axis == "z":
                return [[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]]
            if axis == "x":
                return [[1.0, 0.0, 0.0], [0.0, c, -s], [0.0, s, c]]
            return [[c, 0.0, s], [0.0, 1.0, 0.0], [-s, 0.0, c]]

        def cyc(axis, n):
            return torch.tensor([rot(axis, 2 * math.pi * i / n) for i in range(n)], dtype=torch.float32)

        table = {0: cyc("z", 628), 12: cyc("z", 628), 15: cyc("x", 2), 17: cyc("y", 2), 18: cyc("z", 4), 19: cyc("y", 2), 20: cyc("x", 4)}
        _YCBV_SYMS.extend(table.get(i) for i in range(21))
    return _YCBV_SYMS


def make_batch(bs: int, seed: int = 0, n_points: int = 3000, with_sym: bool = False, dtype=torch.float32,
               num_regions: int = 64) -> dict:
    """Synthetic batch with the reference field names (CPU tensors); region labels 1..num_regions on the object, 0 off it
    (ROT_HEAD.NUM_REGIONS; the default draws the same random stream as before the parameter existed)."""
    g = _gen(seed, "batch")
    H = W = 64
    roi_img = torch.rand(bs, 3, 256, 256, generator=g, dtype=dtype)

    # 2D coords of the crop window in [0,1] (any affine sub-window of the unit meshgrid)
    lin = torch.linspace(0, 1, W, dtype=dtype)
    gy, gx = torch.meshgrid(lin, lin, indexing="ij")
    sc = 0.5 + 0.5 * torch.rand(bs, 1, 1, generator=g, dtype=dtype)
    ox = (1 - sc) * torch.rand(bs, 1, 1, generator=g, dtype=dtype)
    oy = (1 - sc) * torch.rand(bs, 1, 1, generator=g, dtype=dtype)
    roi_coord_2d = torch.stack([ox + sc * gx[None], oy + sc * gy[None]], dim=1)

    # masks: ellipse object, blob occlusion, half-plane truncation
    cx = 32 + 6 * torch.randn(bs, 1, 1, generator=g)
    cy = 32 + 6 * torch.randn(bs, 1, 1, generator=g)
    ax = 14 + 10 * torch.rand(bs, 1, 1, generator=g)
    ay = 14 + 10 * torch.rand(bs, 1, 1, generator=g)
    px = torch.arange(W, dtype=torch.float32)[None, None, :]
    py = torch.arange(H, dtype=torch.float32)[None, :, None]
    mask_obj = ((((px - cx) / ax) ** 2 + ((py - cy) / ay) ** 2) <= 1.0).float()
    bx = 64 * torch.rand(bs, 1, 1, generator=g)
    by = 64 * torch.rand(bs, 1, 1, generator=g)
    br = 6 + 8 * torch.rand(bs, 1, 1, generator=g)
    occl = (((px - bx) ** 2 + (py - by) ** 2) <= br**2).float()
    mask_visib = mask_obj * (1 - occl)
    cut = 44 + 20 * torch.rand(bs, 1, 1, generator=g)
    mask_trunc = mask_visib * (px < cut).float()

    roi_xyz = torch.rand(bs, 3, H, W, generator=g, dtype=dtype) * mask_obj[:, None]
    roi_region = (torch.randint(1, num_regions + 1, (bs, H, W), generator=g) * mask_obj.long()).long()

    roi_extent = 0.05 + 0.25 * torch.rand(bs, 3, generator=g, dtype=dtype)
    roi_points = (torch.rand(bs, n_points, 3, generator=g, dtype=dtype) - 0.5) * roi_extent[:, None, :]
    ego_rot = random_rotations(bs, g).to(dtype)
    trans = torch.stack(
        [
            -0.2 + 0.4 * torch.rand(bs, generator=g),
            -0.2 + 0.4 * torch.rand(bs, generator=g),
            0.4 + 1.1 * torch.rand(bs, generator=g),
        ],
        dim=1,
    ).to(dtype)
    roi_cam = torch.tensor(LM_K, dtype=dtype)[None].repeat(bs, 1, 1)
    roi_center = torch.stack(
        [160 + 320 * torch.rand(bs, generator=g), 120 + 240 * torch.rand(bs, generator=g)], dim=1
    ).to(dtype)
    roi_wh = (40 + 160 * torch.rand(bs, 2, generator=g)).to(dtype)
    scale = 1.5 * roi_wh.max(dim=1)[0]
    resize_ratio = (64.0 / scale).to(dtype)
    # SITE targets (reference data_loader.py:628-632): centroid offset / bbox size, z scaled by resize ratio
    proj = (roi_cam @ trans[:, :, None])[:, :, 0]
    obj_center = proj[:, :2] / proj[:, 2:3]
    delta_c = obj_center - roi_center
    trans_ratio = torch.stack(
        [delta_c[:, 0] / roi_wh[:, 0], delta_c[:, 1] / roi_wh[:, 1], trans[:, 2] / resize_ratio], dim=1
    ).to(dtype)

    sym_infos = None
    if with_sym == "ycbv":
        # a YCB-V-like object set (reference configs/gdrn/ycbv/*: 21 objects, PM_LOSS_SYM; ref/ycbv.py lists 5 symmetric
        # ones): per crop one of 21 objects, the arrays SHARED per object like the per-dataset `sym_infos` dict of the
        # reference data loader (so the device table is filled once); K up to 628 (continuous axis at 0.01 rad steps)
        objs = ycbv_like_symmetries()
        ids = torch.randint(0, len(objs), (bs,), generator=g).tolist()
        sym_infos = [objs[i] for i in ids]
    elif with_sym:
        kinds = ["none", "z2", "cont", "z4"]
        sym_infos = [discrete_symmetries(kinds[i % len(kinds)]) for i in range(bs)]

    return dict(
        roi_img=roi_img, roi_coord_2d=roi_coord_2d, roi_xyz=roi_xyz, roi_mask_trunc=mask_trunc,
        roi_mask_visib=mask_visib, roi_mask_obj=mask_obj, roi_region=roi_region,
        roi_cls=torch.zeros(bs, dtype=torch.long), roi_cam=roi_cam, roi_center=roi_center, roi_wh=roi_wh,
        resize_ratio=resize_ratio, roi_extent=roi_extent, roi_points=roi_points, ego_rot=ego_rot, trans=trans,
        roi_trans_ratio=trans_ratio, sym_info=sym_infos,
    )


def forward_kwargs(batch: dict, train: bool) -> dict:
    """Maps batch fields to `GDRN.forward` kwargs exactly like reference `engine.py:244-269` /
    `gdrn_evaluator.py:569-578`."""
    kw = dict(
        roi_classes=batch["roi_cls"], roi_coord_2d=batch["roi_coord_2d"], roi_cams=batch["roi_cam"],
        roi_centers=batch["roi_center"], roi_whs=batch["roi_wh"], roi_extents=batch["roi_extent"],
        resize_ratios=batch["resize_ratio"],
    )
    if train:
        kw.update(
            gt_xyz=batch["roi_xyz"], gt_xyz_bin=None, gt_mask_trunc=batch["roi_mask_trunc"],
            gt_mask_visib=batch["roi_mask_visib"], gt_mask_obj=batch["roi_mask_obj"], gt_region=batch["roi_region"],
            gt_ego_rot=batch["ego_rot"], gt_points=batch["roi_points"], sym_infos=batch["sym_info"],
            gt_trans=batch["trans"], gt_trans_ratio=batch["roi_trans_ratio"], do_loss=True,
        )
    return kw


def seeded_state_dict(template: dict, seed: int = 0) -> dict:
    """Non-degenerate weights for every entry of `template` (a state_dict giving names/shapes).

    SURVEY.md pitfall P1: the reference init (normal std=1e-3) collapses eval-mode activations,
    so parity fixtures use Kaiming-scale weights and randomised BN statistics instead.
    Each tensor is seeded by its own name => independent of iteration order.
    """
    out = {}
    for name, t in template.items():
        g = _gen(seed, name)
        shape = tuple(t.shape)
        if name.endswith("num_batches_tracked"):
            out[name] = torch.zeros((), dtype=torch.long)
        elif name.endswith("running_mean"):
            out[name] = 0.1 * torch.randn(shape, generator=g)
        elif name.endswith("running_var"):
            out[name] = 0.5 + torch.rand(shape, generator=g)
        elif len(shape) == 1 and name.endswith("weight"):  # BN / GN gamma
            out[name] = 0.5 + torch.rand(shape, generator=g)
        elif len(shape) == 1 and name.endswith("bias"):
            out[name] = 0.1 * torch.randn(shape, generator=g)
        elif len(shape) >= 2:
            if "rot_head_net.features.0." in name:  # ConvTranspose2d weight is [Cin, Cout, k, k]
                fan_in = shape[0] * shape[2] * shape[3] / 4.0  # each output sees ~k*k/s^2 taps
            else:
                fan_in = 1
                for s in shape[1:]:
                    fan_in *= s
            std = math.sqrt(2.0 / fan_in)
            if name.startswith("pnp_net.fc_"):
                std = math.sqrt(1.0 / fan_in)
            out[name] = std * torch.randn(shape, generator=g)
        else:
            out[name] = torch.zeros(shape)
        out[name] = out[name].to(t.dtype) if t.dtype.is_floating_point else out[name]
    return out


def make_pnp_maps(bs: int, seed: int = 0, res: int = 64, noise: float = 0.004, outlier_frac: float = 0.15, im_wh=(640, 480)) -> dict:
    """Geometrically consistent test-time head outputs for the RANSAC-PnP path (gdrn_evaluator.py:316-436): an ellipsoid with the
    object's extent is placed at a random pose, every pixel of the `res` x `res` ROI grid whose viewing ray hits it gets the
    normalised object coordinate of the hit point (+ Gaussian noise; a fraction of the pixels gets a random coordinate = outlier),
    the raw mask output is high on the object and low elsewhere (with a few wrong pixels).  Returns CPU tensors:
    mask [B,1,res,res] (raw, L1-head style), xyz [B,3,res,res] in [0,1], coord_2d [B,2,res,res] in [0,1], extents [B,3], cams
    [B,3,3], im_wh [B,2], R [B,3,3], t [B,3] (the true pose)."""
    g = _gen(seed, "pnp_maps")
    W, H = im_wh
    K = torch.tensor(LM_K, dtype=torch.float64)
    R = random_rotations(bs, g).double()
    ext = (torch.rand(bs, 3, generator=g, dtype=torch.float64) * 0.2 + 0.06)
    tz = torch.rand(bs, generator=g, dtype=torch.float64) * 0.8 + 0.5
    cx = torch.rand(bs, generator=g, dtype=torch.float64) * 0.4 * W + 0.3 * W
    cy = torch.rand(bs, generator=g, dtype=torch.float64) * 0.4 * H + 0.3 * H
    t = torch.stack([(cx - K[0, 2]) * tz / K[0, 0], (cy - K[1, 2]) * tz / K[1, 1], tz], dim=1)
    scale = 1.5 * ext.max(dim=1).values / tz * K[0, 0]  # ROI side in pixels
    lin = (torch.arange(res, dtype=torch.float64) + 0.5) / res - 0.5
    mask = torch.zeros(bs, 1, res, res)
    xyz = torch.zeros(bs, 3, res, res)
    c2d = torch.zeros(bs, 2, res, res)
    for b in range(bs):
        u = cx[b] + lin.view(1, res) * scale[b]
        v = cy[b] + lin.view(res, 1) * scale[b]
        u, v = u.expand(res, res), v.expand(res, res)
        c2d[b, 0], c2d[b, 1] = (u / W).float(), (v / H).float()
        # ray d through the pixel, in the object frame: o = -R^T t, dir = R^T d; unit sphere after scaling by 2 / extent
        d = torch.stack([(u - K[0, 2]) / K[0, 0], (v - K[1, 2]) / K[1, 1], torch.ones_like(u)], dim=-1)
        s = 2.0 / ext[b]
        o = (-(R[b].T @ t[b])) * s
        dd = (d @ R[b]) * s  # R^T d for row vectors
        A = (dd * dd).sum(-1)
        Bq = 2 * (dd * o).sum(-1)
        Cq = (o * o).sum() - 1.0
        disc = Bq * Bq - 4 * A * Cq
        hit = disc > 0
        lam = (-Bq - torch.sqrt(disc.clamp_min(0))) / (2 * A)
        p = (o + lam.unsqueeze(-1) * dd) / s  # object-frame point, metres
        xn = p / ext[b] + 0.5
        xn = xn + torch.randn(res, res, 3, generator=g, dtype=torch.float64) * noise
        outl = torch.rand(res, res, generator=g) < outlier_frac
        xn = torch.where(outl.unsqueeze(-1), torch.rand(res, res, 3, generator=g, dtype=torch.float64), xn)
        xyz[b] = torch.where(hit.unsqueeze(-1), xn, torch.zeros_like(xn)).permute(2, 0, 1).float()
        m = torch.where(hit, torch.full_like(A, 0.9), torch.full_like(A, 0.05)) + torch.randn(res, res, generator=g, dtype=torch.float64) * 0.03
        flip = torch.rand(res, res, generator=g) < 0.01
        m = torch.where(flip, 0.95 - m, m)
        mask[b, 0] = m.float()
    return dict(mask=mask, xyz=xyz, coord_2d=c2d, extents=ext.float(), cams=K.float().expand(bs, 3, 3).contiguous(),
                im_wh=torch.tensor([[W, H]] * bs, dtype=torch.float32), R=R.float(), t=t.float())
