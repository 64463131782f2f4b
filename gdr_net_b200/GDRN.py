"""Drop-in replacement for the reference module `core/gdrn_modeling/models/GDRN.py`.

Same plugin seam (`build_model_optimizer(cfg) -> (model, optimizer)`, selected by
`eval(cfg.MODEL.CDPN.NAME)`, reference main_gdrn.py:31,108), same `GDRN.forward` signature and
return values (GDRN.py:83-109, 233-306), same sub-module attribute names and state_dict keys
(`backbone.*`, `rot_head_net.features.{0,1,3,...,23}.*`, `pnp_net.*`; SURVEY.md 8b) so reference
checkpoints load unchanged, same `get_event_storage().put_scalars(**vis_dict)` side effect.

The `nn.Module`s below only OWN the parameters / buffers (ordinary `nn.Parameter`s, so optimizers,
DDP and checkpointers see the usual thing).  All compute is done by `engine.Engine` through the C ABI
of libgdrn_b200.so (hand-written sm_90a kernels); there is no PyTorch / CPU fallback path.
"""
from __future__ import annotations

import logging
from typing import Optional

import torch
import torch.nn as nn

from .engine import Engine, LOSS_NAMES, check_roi_classes, pose_loss_switches  # noqa: F401  (LOSS_NAMES: the default list, re-exported)

logger = logging.getLogger(__name__)

resnet_spec = {  # reference resnet_backbone.py:8-14 (BasicBlock variants are the supported ones)
    18: ("basic", [2, 2, 2, 2], [64, 64, 128, 256, 512], "resnet18"),
    34: ("basic", [3, 4, 6, 3], [64, 64, 128, 256, 512], "resnet34"),
}


def _normal_init(m, std, bias=0.0):
    nn.init.normal_(m.weight, 0.0, std)
    if getattr(m, "bias", None) is not None:
        nn.init.constant_(m.bias, bias)


class _ParamsOnly(nn.Module):
    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError(
            f"{type(self).__name__} only owns parameters; the forward/backward math runs in "
            "gdr_net_b200.engine.Engine (libgdrn_b200.so). There is no PyTorch fallback."
        )


class BasicBlock(_ParamsOnly):
    """Parameter container with torchvision BasicBlock's names (conv1, bn1, conv2, bn2, downsample.{0,1})."""

    expansion = 1

    def __init__(self, inplanes, planes, stride=1, downsample=None):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, 3, stride, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = nn.Conv2d(planes, planes, 3, 1, 1, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.downsample = downsample
        self.stride = stride


class ResNetBackboneNet(_ParamsOnly):
    """reference models/resnet_backbone.py:17-51"""

    def __init__(self, layers, in_channel=3, freeze=False):
        super().__init__()
        self.freeze = freeze
        self.inplanes = 64
        self.conv1 = nn.Conv2d(in_channel, 64, kernel_size=7, stride=2, padding=3, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        self.layer1 = self._make_layer(64, layers[0])
        self.layer2 = self._make_layer(128, layers[1], stride=2)
        self.layer3 = self._make_layer(256, layers[2], stride=2)
        self.layer4 = self._make_layer(512, layers[3], stride=2)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                _normal_init(m, 0.001)
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.constant_(m.weight, 1.0)
                nn.init.constant_(m.bias, 0.0)

    def _make_layer(self, planes, blocks, stride=1):
        downsample = None
        if stride != 1 or self.inplanes != planes:
            downsample = nn.Sequential(nn.Conv2d(self.inplanes, planes, 1, stride, bias=False), nn.BatchNorm2d(planes))
        layers = [BasicBlock(self.inplanes, planes, stride, downsample)]
        self.inplanes = planes
        for _ in range(1, blocks):
            layers.append(BasicBlock(planes, planes))
        return nn.Sequential(*layers)


class RotWithRegionHead(_ParamsOnly):
    """reference models/cdpn_rot_head_region.py:10-143 (ROT_CONCAT=False branch; concat mode is broken
    upstream, SURVEY P8).  `features` keeps the reference indices: ReLU / upsample placeholders included.
    With rot / mask / region_class_aware the output conv carries that block once per class (engine.class_rows).
    norm = "BN" (nn.BatchNorm2d) or "GN" (nn.GroupNorm(num_gn_groups, 256), layer_utils.get_norm) at 1, 4, 7, 11, 14, 18, 21."""

    def __init__(self, in_channels=512, num_layers=3, num_filters=256, kernel_size=3, output_kernel_size=1,
                 rot_output_dim=3, mask_output_dim=1, num_regions=64, norm="BN", num_gn_groups=32, freeze=False, num_classes=1,
                 rot_class_aware=False, mask_class_aware=False, region_class_aware=False):
        super().__init__()
        check_head_norm(norm, num_gn_groups)
        if kernel_size != 3 or output_kernel_size != 1 or num_layers != 3:
            raise NotImplementedError("only the a6 head (k3 deconv, 1x1 output conv, BN, 3 stages) is implemented")
        self.freeze = freeze
        f = nn.ModuleList()
        def norm_layer():
            return nn.GroupNorm(num_gn_groups, num_filters) if norm == "GN" else nn.BatchNorm2d(num_filters)

        f.append(nn.ConvTranspose2d(in_channels, num_filters, 3, stride=2, padding=1, output_padding=1, bias=False))
        f.append(norm_layer())
        f.append(nn.ReLU(inplace=True))
        for i in range(num_layers):
            if i >= 1:
                f.append(nn.UpsamplingBilinear2d(scale_factor=2))
            for _ in range(2):
                f.append(nn.Conv2d(num_filters, num_filters, 3, 1, 1, bias=False))
                f.append(norm_layer())
                f.append(nn.ReLU(inplace=True))
        self.rot_output_dim = rot_output_dim * (num_classes if rot_class_aware else 1)
        self.mask_output_dim = mask_output_dim * (num_classes if mask_class_aware else 1)
        self.region_output_dim = (num_regions + 1) * (num_classes if region_class_aware else 1)
        f.append(nn.Conv2d(num_filters, self.mask_output_dim + self.rot_output_dim + self.region_output_dim, 1, padding=0, bias=True))
        self.features = f
        for m in self.modules():
            if isinstance(m, (nn.Conv2d, nn.ConvTranspose2d)):
                _normal_init(m, 0.001)
            elif isinstance(m, (nn.BatchNorm2d, nn.GroupNorm)):
                nn.init.constant_(m.weight, 1.0)
                nn.init.constant_(m.bias, 0.0)


def check_head_norm(norm, num_gn_groups):
    """ROT_HEAD.NORM / NUM_GN_GROUPS: BatchNorm, or GroupNorm with a group count that divides 256 and is at most 64 (the
    gdrn_head_gn_* kernels); anything else raises NotImplementedError naming the key."""
    if norm not in ("BN", "GN"):
        raise NotImplementedError(f"ROT_HEAD.NORM = {norm!r} (BN or GN)")
    if norm == "GN" and (int(num_gn_groups) != num_gn_groups or not 1 <= num_gn_groups <= 64 or 256 % int(num_gn_groups)):
        raise NotImplementedError(f"ROT_HEAD.NUM_GN_GROUPS = {num_gn_groups!r} (a divisor of 256, at most 64)")


class ConvPnPNet(_ParamsOnly):
    """reference models/conv_pnp_net.py:41-109 (mask_attention 'none').

    DropBlock (PNP_HEAD_CFG.drop_prob > 0, conv_pnp_net.py:66-72,128-142): every forward, in train and in eval mode, advances
    the LinearScheduler counter (np.linspace(0, drop_prob, 5000)[min(k, 4999)] at forward k); in train mode the Patch-PnP input
    is multiplied by a block mask and numel / sum(mask).  The counter lives on the device (`dropblock_step` reads and sets it),
    is not part of the state_dict and starts at 0 with every new module, like the reference's plain attribute.
    `dropblock_seed` (default: derived from torch.initial_seed() at construction) keys the Philox generator of the mask
    together with the data-parallel rank.  After a train forward, `dropblock_seeds`, `dropblock_keep` ([B, 64, 64] uint8) and
    `dropblock_scale` ([1] fp32) are the device tensors of the mask it used."""

    def __init__(self, nIn, featdim=128, rot_dim=6, num_layers=3, norm="GN", num_gn_groups=32, num_regions=64,
                 drop_prob=0.0, dropblock_size=5, mask_attention_type="none"):
        super().__init__()
        if norm != "GN" or num_layers != 3 or featdim != 128 or mask_attention_type != "none":
            raise NotImplementedError("only the a6 Patch-PnP (3 stride-2 convs, GN, featdim 128) is implemented")
        if not 0.0 <= float(drop_prob) <= 1.0:
            raise NotImplementedError(f"PNP_HEAD_CFG.drop_prob = {drop_prob!r} (0 <= drop_prob <= 1)")
        if int(dropblock_size) != dropblock_size or not 1 <= dropblock_size <= 15:
            raise NotImplementedError(f"PNP_HEAD_CFG.dropblock_size = {dropblock_size!r} (1..15)")
        self.featdim, self.num_regions, self.nIn, self.rot_dim = featdim, num_regions, nIn, rot_dim
        self.drop_prob, self.dropblock_size = float(drop_prob), int(dropblock_size)
        self.dropblock_seed = torch.initial_seed()
        self._db_step = None  # int64 [1] on the device, created by dropblock_counter
        self._db_bufs = {}    # batch size -> (keep, seeds, counts, scale), patch_pnp.dropblock_step
        self.dropblock_seeds = self.dropblock_keep = self.dropblock_scale = None
        f = nn.ModuleList()
        for i in range(3):
            f.append(nn.Conv2d(nIn if i == 0 else featdim, featdim, 3, 2, 1, bias=False))
            f.append(nn.GroupNorm(num_gn_groups, featdim))
            f.append(nn.ReLU(inplace=True))
        self.features = f
        self.fc1 = nn.Linear(featdim * 8 * 8, 1024)
        self.fc2 = nn.Linear(1024, 256)
        self.fc_r = nn.Linear(256, rot_dim)
        self.fc_t = nn.Linear(256, 3)
        for m in self.modules():
            if isinstance(m, (nn.Conv2d, nn.Linear)):
                _normal_init(m, 0.001)
            elif isinstance(m, nn.GroupNorm):
                nn.init.constant_(m.weight, 1.0)
                nn.init.constant_(m.bias, 0.0)
        _normal_init(self.fc_r, 0.01)
        _normal_init(self.fc_t, 0.01)
        self.precision = "fp32x3"  # stand-alone forward: "fp32x3" (1e-3 parity) | "half"
        self._runner = None

    def dropblock_counter(self, device) -> torch.Tensor:
        """The device-resident DropBlock step counter (int64 [1]) on `device`."""
        if self._db_step is None:
            self._db_step = torch.zeros(1, dtype=torch.int64, device=device)
        elif self._db_step.device != torch.device(device):
            self._db_step = self._db_step.to(device)
        return self._db_step

    @property
    def dropblock_step(self) -> int:
        """Forwards counted by the DropBlock schedule so far (the reference's `dropblock.i`); settable, e.g. to resume."""
        return 0 if self._db_step is None else int(self._db_step.item())

    @dropblock_step.setter
    def dropblock_step(self, k: int):
        self.dropblock_counter(self.fc1.weight.device).fill_(int(k))

    def forward(self, coor_feat, region=None, extents=None, mask_attention=None):
        """Stand-alone Patch-PnP inference with the reference signature (conv_pnp_net.py:111): xyz(+2-D coords) maps
        [B, 3|5, 64, 64], region attention [B, R, 64, 64] or None, extents [B, 3] -> (rot [B, rot_dim], t [B, 3]).
        Runs patch_pnp.PatchPnP (libgdrn_b200.so kernels, one CUDA graph); no autograd, no CPU fallback.  Inside
        `GDRN.forward` the engine runs the same kernels with the hand-written backward instead."""
        if mask_attention is not None:
            raise NotImplementedError("mask attention is 'none' in the a6 configuration")
        from .patch_pnp import PatchPnP

        if self._runner is None or self._runner.precision != {"mixed": "fp32x3"}.get(self.precision, self.precision):
            self._runner = PatchPnP(self, self.precision)
        return self._runner(coor_feat, region, extents, train=self.training)


def get_xyz_mask_region_out_dim(cfg):
    """reference GDRN.py:524-547"""
    r = cfg.MODEL.CDPN.ROT_HEAD
    if r.XYZ_LOSS_TYPE in ["MSE", "L1", "L2", "SmoothL1"]:
        r_out_dim = 3
    elif r.XYZ_LOSS_TYPE in ["CE_coor", "CE"]:
        r_out_dim = 3 * (r.XYZ_BIN + 1)
    else:
        raise NotImplementedError(f"unknown xyz loss type: {r.XYZ_LOSS_TYPE}")
    if r.MASK_LOSS_TYPE in ["L1", "BCE"]:
        mask_out_dim = 1
    elif r.MASK_LOSS_TYPE in ["CE"]:
        mask_out_dim = 2
    else:
        raise NotImplementedError(f"unknown mask loss type: {r.MASK_LOSS_TYPE}")
    region_out_dim = r.NUM_REGIONS + 1
    assert region_out_dim > 2, region_out_dim
    return r_out_dim, mask_out_dim, region_out_dim


def _check_supported(cfg):
    """The hot path implements the configuration used by all 41 shipped experiment configs (SURVEY 0)."""
    c = cfg.MODEL.CDPN
    r, p = c.ROT_HEAD, c.PNP_NET
    problems = []
    if c.BACKBONE.NUM_LAYERS not in resnet_spec or c.BACKBONE.INPUT_RES != 256 or c.BACKBONE.OUTPUT_RES != 64:
        problems.append("backbone must be resnet18/34 at 256 -> 64")
    if r.ROT_CONCAT:
        problems.append("concat heads (ROT_HEAD.ROT_CONCAT)")
    try:
        check_head_norm(r.NORM, r.get("NUM_GN_GROUPS", 32))
    except NotImplementedError as e:
        problems.append(str(e))
    if (r.ROT_CLASS_AWARE or r.MASK_CLASS_AWARE or r.REGION_CLASS_AWARE) and not int(r.NUM_CLASSES) >= 1:
        problems.append(f"ROT_HEAD.NUM_CLASSES = {r.NUM_CLASSES!r} with a class-aware head (>= 1)")
    if r.XYZ_LOSS_TYPE != "L1" or r.MASK_LOSS_TYPE not in ("L1", "BCE", "CE") or r.REGION_LOSS_TYPE != "CE":
        problems.append("losses other than xyz L1 / mask L1, BCE or CE / region CE")
    # the per-pixel kernels hold a logit row of 72 floats: MO + 3 + (R + 1) <= 70 for R <= 64; R < 2 fails the reference's own
    # region_out_dim > 2 assert (GDRN.py:546)
    if not 2 <= r.NUM_REGIONS <= 64:
        problems.append(f"ROT_HEAD.NUM_REGIONS = {r.NUM_REGIONS!r} (2..64)")
    # gdrn_loss builds gt_masks = {"trunc", "visib", "obj"} (GDRN.py:339); any other key (the config comment's "gt") is a KeyError there
    for key in ("XYZ_LOSS_MASK_GT", "MASK_LOSS_GT", "REGION_LOSS_MASK_GT"):
        if getattr(r, key) not in ("trunc", "visib", "obj"):
            problems.append(f"ROT_HEAD.{key} = {getattr(r, key)!r} (trunc, visib or obj)")
    if p.MASK_ATTENTION != "none" or p.R_ONLY:
        problems.append("Patch-PnP input other than xyz (+ 2D coords) (+ region attention) (PNP_NET.MASK_ATTENTION, R_ONLY)")
    if p.ROT_TYPE != "allo_rot6d" or p.TRANS_TYPE != "centroid_z" or p.Z_TYPE != "REL":
        problems.append(f"pose parametrisation other than allo_rot6d + centroid_z(REL) (PNP_NET.ROT_TYPE = {p.ROT_TYPE!r}, "
                        f"TRANS_TYPE = {p.TRANS_TYPE!r}, Z_TYPE = {p.Z_TYPE!r})")
    # the PNP_NET loss switches (PM_*, ROT_*, CENTROID_*, Z_*, TRANS_*, BIND_*): engine.pose_loss_switches names a bad one
    try:
        pose_loss_switches(p)
    except ValueError as e:
        problems.append(str(e))
    # BACKBONE / ROT_HEAD / PNP_NET .FREEZE are supported in every combination (Engine.live_*); with all three frozen the
    # optimizer gets no parameters and fails to build, as the reference's does
    if c.TRANS_HEAD.ENABLED or c.USE_MTL:
        problems.append("trans head / MTL weighting (TRANS_HEAD.ENABLED, USE_MTL)")
    if problems:
        raise NotImplementedError("gdr_net_b200 implements the a6_cPnP hot path only; unsupported: " + "; ".join(problems))


class GDRN(nn.Module):
    def __init__(self, cfg, backbone, rot_head_net, trans_head_net=None, pnp_net=None, precision: str = "mixed"):
        super().__init__()
        assert cfg.MODEL.CDPN.NAME == "GDRN", cfg.MODEL.CDPN.NAME
        _check_supported(cfg)
        self.backbone = backbone
        self.rot_head_net = rot_head_net
        self.pnp_net = pnp_net
        self.trans_head_net = trans_head_net
        self.cfg = cfg
        self.concat = cfg.MODEL.CDPN.ROT_HEAD.ROT_CONCAT
        self.r_out_dim, self.mask_out_dim, self.region_out_dim = get_xyz_mask_region_out_dim(cfg)
        self._engine: Optional[Engine] = None
        self._vis_dev, self._vis_host = None, None
        self.use_cuda_graphs = False  # set True for fixed-shape training loops: forward/backward replay CUDA graphs
        # "mixed" (default): fp32-faithful 3-pass forward (1e-3 parity on every output / loss) + single-pass fp16 backward;
        # "fp32x3": 3-pass forward and backward; "half": single-pass everywhere (throughput mode, TF32-class arithmetic)
        self.precision = {"bf16": "half", "fp16": "half"}.get(precision, precision)

    @property
    def last_vis_dict(self) -> dict:
        """The `vis/*` scalars of the most recent do_loss forward (synchronises on first access)."""
        if self._vis_host is None:
            if self._vis_dev is None:
                return {}
            v = self._vis_dev.tolist()
            self._vis_host = {
                "vis/error_R": v[0], "vis/error_t": v[1] * 100,
                "vis/error_tx": abs(v[2] - v[8]) * 100, "vis/error_ty": abs(v[3] - v[9]) * 100,
                "vis/error_tz": abs(v[4] - v[10]) * 100,
                "vis/tx_pred": v[2], "vis/ty_pred": v[3], "vis/tz_pred": v[4],
                "vis/tx_net": v[5], "vis/ty_net": v[6], "vis/tz_net": v[7],
                "vis/tx_gt": v[8], "vis/ty_gt": v[9], "vis/tz_gt": v[10],
                "vis/tx_rel_gt": v[11], "vis/ty_rel_gt": v[12], "vis/tz_rel_gt": v[13],
            }
        return self._vis_host

    @property
    def engine(self) -> Engine:
        if self._engine is None or self._engine.precision != self.precision:
            self._engine = Engine(self, precision=self.precision)
        self._engine.use_cuda_graphs = self.use_cuda_graphs
        return self._engine

    def forward(self, x, gt_xyz=None, gt_xyz_bin=None, gt_mask_trunc=None, gt_mask_visib=None, gt_mask_obj=None,
                gt_region=None, gt_allo_quat=None, gt_ego_quat=None, gt_allo_rot6d=None, gt_ego_rot6d=None, gt_ego_rot=None,
                gt_points=None, sym_infos=None, gt_trans=None, gt_trans_ratio=None, roi_classes=None, roi_coord_2d=None,
                roi_cams=None, roi_centers=None, roi_whs=None, roi_extents=None, resize_ratios=None, do_loss=False):
        cfg = self.cfg
        r_cfg = cfg.MODEL.CDPN.ROT_HEAD
        if r_cfg.ROT_CLASS_AWARE or r_cfg.MASK_CLASS_AWARE or r_cfg.REGION_CLASS_AWARE:
            check_roi_classes(roi_classes, x.shape[0], int(r_cfg.NUM_CLASSES))
        if not x.is_cuda:
            raise RuntimeError("gdr_net_b200.GDRN runs on CUDA (sm_90a) only; there is no CPU fallback")
        pnp_cfg = cfg.MODEL.CDPN.PNP_NET
        res = self.engine.run(
            x, roi_classes=roi_classes, roi_coord_2d=roi_coord_2d, roi_cams=roi_cams, roi_centers=roi_centers,
            roi_whs=roi_whs, roi_extents=roi_extents, resize_ratios=resize_ratios, gt_xyz=gt_xyz, gt_mask_trunc=gt_mask_trunc,
            gt_mask_visib=gt_mask_visib, gt_mask_obj=gt_mask_obj, gt_region=gt_region, gt_ego_rot=gt_ego_rot, gt_points=gt_points,
            sym_infos=sym_infos if pnp_cfg.PM_LOSS_SYM else None, gt_trans=gt_trans, gt_trans_ratio=gt_trans_ratio,
            do_loss=do_loss, train_bn=self.training, want_maps=(not do_loss) and bool(cfg.TEST.USE_PNP),
        )
        if not do_loss:
            # NOTE: the reference returns `rot` on the CPU in test mode (numpy loop, pose_from_pred_centroid_z.py:141);
            # we keep it on the device -- `.cpu()` is a no-op for consumers that need host data.  With a class-aware head the
            # maps are those of each crop's class (GDRN.py:134-151).
            out_dict = {"rot": res["rot"], "trans": res["trans"]}
            if cfg.TEST.USE_PNP:
                out_dict.update({k: res[k] for k in ("mask", "coor_x", "coor_y", "coor_z", "region")})
            return out_dict
        assert (gt_xyz is not None) and (gt_trans is not None) and (gt_trans_ratio is not None) and (gt_region is not None)
        lw = dict(loss_coor_x=r_cfg.XYZ_LW, loss_coor_y=r_cfg.XYZ_LW, loss_coor_z=r_cfg.XYZ_LW, loss_mask=r_cfg.MASK_LW,
                  loss_region=r_cfg.REGION_LW, loss_rot=pnp_cfg.ROT_LW, loss_centroid=pnp_cfg.CENTROID_LW, loss_z=pnp_cfg.Z_LW,
                  loss_trans_xy=pnp_cfg.TRANS_LW, loss_trans_z=pnp_cfg.TRANS_LW, loss_trans_LPnP=pnp_cfg.TRANS_LW,
                  loss_bind=pnp_cfg.get("BIND_LW", 0.0))
        for name in ("loss_PM_R", "loss_PM_RT", "loss_PM_T", "loss_PM_xy", "loss_PM_z"):
            lw[name] = pnp_cfg.PM_LW
        for name in ("loss_PM_T_noP", "loss_PM_xy_noP", "loss_PM_z_noP"):  # pm_loss.py:146-164: neither PM_LW nor 3
            lw[name] = 1.0
        losses = res["losses"]  # [len(engine.loss_names)] tensor attached to the autograd graph through _GDRNFunction
        loss_dict = {}
        for i, name in enumerate(self.engine.loss_names):
            if name in ("loss_centroid", "loss_z") and lw[name] <= 0:
                continue
            loss_dict[name] = losses[i] * lw[name]
        # logging side effect (GDRN.py:246-303): ONE device->host copy of 14 scalars instead of 18 .item() syncs -- and only
        # when somebody consumes them: with an active detectron2 EventStorage now (reference behaviour), otherwise lazily
        # through `last_vis_dict`, so a training loop without a logger never stalls the GPU between forward and backward.
        self._vis_dev, self._vis_host = res["vis"], None
        storage = _get_event_storage()
        if storage is not None:
            storage.put_scalars(**self.last_vis_dict)
        return {}, loss_dict


def _get_event_storage():
    """detectron2's EventStorage when detectron2 is present and a storage is active (reference GDRN.py:302)."""
    try:
        from detectron2.utils.events import get_event_storage  # type: ignore

        return get_event_storage()
    except Exception:
        return None


def _load_backbone_pretrained(backbone, spec: str):
    """reference GDRN.py:713-721: `load_checkpoint(model.backbone, PRETRAINED, strict=False)` (mmcv).  `torchvision://name`
    resolves through torchvision's model-zoo table (torch hub cache, downloads if absent); anything else is a checkpoint
    file whose tensors may sit under `state_dict` / `model`.  Fails loudly: a reference config must never silently train a
    randomly initialised backbone."""
    if spec.startswith("torchvision://"):
        name = spec[len("torchvision://"):]
        try:
            import torchvision

            weights = torchvision.models.get_model_weights(name).DEFAULT
            sd = weights.get_state_dict(progress=False)
        except Exception as e:
            raise RuntimeError(
                f"cfg.MODEL.CDPN.BACKBONE.PRETRAINED={spec!r}: could not obtain the torchvision weights ({type(e).__name__}: {e}). "
                "Put the checkpoint in the torch hub cache, point PRETRAINED at a local file, or set it to '' explicitly.") from e
    else:
        sd = torch.load(spec, map_location="cpu")
        for k in ("state_dict", "model"):
            if isinstance(sd, dict) and k in sd and isinstance(sd[k], dict):
                sd = sd[k]
        sd = {(k[len("module."):] if k.startswith("module.") else k): v for k, v in sd.items()}
        if any(k.startswith("backbone.") for k in sd):
            sd = {k[len("backbone."):]: v for k, v in sd.items() if k.startswith("backbone.")}
    missing, unexpected = backbone.load_state_dict(sd, strict=False)
    logger.info(f"backbone weights from {spec}: {len(missing)} missing, {len(unexpected)} unexpected keys (strict=False)")
    return missing, unexpected


def _freeze_or_add(net, freeze, params_lr_list, lr):
    """reference GDRN.py:563-571, 595-603, 684-692: a frozen sub-network's parameters stop requiring grad and get no
    optimizer group; any other one gets a group of its trainable parameters."""
    if freeze:
        for p in net.parameters():
            p.requires_grad_(False)
    else:
        params_lr_list.append({"params": [p for p in net.parameters() if p.requires_grad], "lr": lr})


def build_model_optimizer(cfg, precision: str = "mixed"):
    """reference GDRN.py:550-724"""
    backbone_cfg = cfg.MODEL.CDPN.BACKBONE
    r_head_cfg = cfg.MODEL.CDPN.ROT_HEAD
    pnp_net_cfg = cfg.MODEL.CDPN.PNP_NET
    _check_supported(cfg)
    params_lr_list = []
    _block, layers, channels, _name = resnet_spec[backbone_cfg.NUM_LAYERS]
    backbone_net = ResNetBackboneNet(layers, backbone_cfg.INPUT_CHANNEL, freeze=backbone_cfg.FREEZE)
    _freeze_or_add(backbone_net, backbone_cfg.FREEZE, params_lr_list, float(cfg.SOLVER.BASE_LR))

    r_out_dim, mask_out_dim, region_out_dim = get_xyz_mask_region_out_dim(cfg)
    rot_head_net = RotWithRegionHead(
        channels[-1], r_head_cfg.NUM_LAYERS, r_head_cfg.NUM_FILTERS, r_head_cfg.CONV_KERNEL_SIZE,
        r_head_cfg.OUT_CONV_KERNEL_SIZE, rot_output_dim=r_out_dim, mask_output_dim=mask_out_dim,
        num_regions=r_head_cfg.NUM_REGIONS, norm=r_head_cfg.NORM, num_gn_groups=r_head_cfg.NUM_GN_GROUPS, freeze=r_head_cfg.FREEZE,
        num_classes=r_head_cfg.NUM_CLASSES, rot_class_aware=r_head_cfg.ROT_CLASS_AWARE,
        mask_class_aware=r_head_cfg.MASK_CLASS_AWARE, region_class_aware=r_head_cfg.REGION_CLASS_AWARE,
    )
    _freeze_or_add(rot_head_net, r_head_cfg.FREEZE, params_lr_list, float(cfg.SOLVER.BASE_LR))

    pnp_net_in_channel = r_out_dim
    if pnp_net_cfg.WITH_2D_COORD:
        pnp_net_in_channel += 2
    if pnp_net_cfg.REGION_ATTENTION:
        pnp_net_in_channel += r_head_cfg.NUM_REGIONS
    rot_dim = 6  # allo_rot6d / ego_rot6d
    pnp_head_cfg = pnp_net_cfg.PNP_HEAD_CFG
    pnp_head_type = pnp_head_cfg.pop("type")  # mutates cfg like the reference (GDRN.py:658-659)
    if pnp_head_type != "ConvPnPNet":
        raise NotImplementedError(f"pnp head type {pnp_head_type}: only ConvPnPNet (Patch-PnP) is implemented")
    pnp_head_cfg.update(nIn=pnp_net_in_channel, rot_dim=rot_dim, num_regions=r_head_cfg.NUM_REGIONS, featdim=128,
                        num_layers=3, mask_attention_type=pnp_net_cfg.MASK_ATTENTION)
    pnp_net = ConvPnPNet(**pnp_head_cfg)
    _freeze_or_add(pnp_net, pnp_net_cfg.FREEZE, params_lr_list, float(cfg.SOLVER.BASE_LR) * pnp_net_cfg.LR_MULT)

    model = GDRN(cfg, backbone_net, rot_head_net, trans_head_net=None, pnp_net=pnp_net, precision=precision)
    from .solver import build_optimizer_with_params

    optimizer = build_optimizer_with_params(cfg, params_lr_list)
    if cfg.MODEL.WEIGHTS == "":
        backbone_pretrained = cfg.MODEL.CDPN.BACKBONE.get("PRETRAINED", "")
        if backbone_pretrained == "":
            logger.warning("Randomly initialize weights for backbone!")
        else:
            logger.info(f"load backbone weights from: {backbone_pretrained}")
            _load_backbone_pretrained(model.backbone, backbone_pretrained)
    model.to(torch.device(cfg.MODEL.DEVICE))
    return model, optimizer
