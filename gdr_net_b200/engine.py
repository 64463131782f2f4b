"""Forward / backward orchestration of the GDR-Net hot path over the C ABI (libgdrn_b200.so).

Mirrors reference `GDRN.forward` (core/gdrn_modeling/models/GDRN.py:83-306), `gdrn_loss` (:308-521) and the
autograd backward of both, but every tensor op is one of our sm_90a kernels (gdr_net_b200/csrc).  PyTorch is
used for device memory, streams and the autograd/DDP boundary only.

precision = "half"   : activations / gradients are 16-bit NHWC tensors (fp16 by default, bf16 if the library is built with
                       GDRN_STORE_F16=0), one wgmma pass per k-step.  "fp16" / "bf16" are accepted as aliases.
precision = "fp32x3" : (hi, lo) 16-bit planes (22-bit operands with fp16), three wgmma passes in forward AND backward
precision = "mixed"  : the fp32x3 forward (every output / loss inside the 1e-3 parity bound, identical ReLU / max-pool / L1
                       decisions) with the single-plane backward of "half": the backward is linear given the forward's
                       masks, so 11-bit operands there cost ~1e-3 on the gradients (what cuDNN's TF32 backward gives the
                       reference) instead of flipping decisions.  Saved activations are read through their hi plane.
"""
from __future__ import annotations

import os
from typing import Dict, Optional

import torch

from . import ops
from .capi import C
from .ops import PT, _stream
from .patch_pnp import dropblock_step, pnp_net_forward

LOSS_NAMES = ["loss_coor_x", "loss_coor_y", "loss_coor_z", "loss_mask", "loss_region", "loss_PM_R", "loss_centroid", "loss_z"]
MASK_LOSSES = {"L1": 0, "BCE": 1, "CE": 2}  # ROT_HEAD.MASK_LOSS_TYPE -> the mask_loss argument of the gdrn_*_ex loss kernels
HEAD_CONVS = [(3, 4, False), (6, 7, False), (10, 11, True), (13, 14, False), (17, 18, True), (20, 21, False)]

# PNP_NET pose-loss switches -> gdrn_pose_switches (include/gdrn_b200.h)
POSE_LOSS_KINDS = {"l1": 0, "smooth_l1": 1, "mse": 2, "l2": 3}  # PM_LOSS_TYPE, lower-cased like PyPMLoss (pm_loss.py:70)
POSE_LOSS_KINDS3 = {"L1": 0, "MSE": 2, "L2": 3}  # CENTROID / Z / TRANS / BIND_LOSS_TYPE (GDRN.py:439-514)
PM_MODES = {"off": -1, "R": 0, "RT": 1, "T": 2, "Z": 3, "T_noP": 4, "Z_noP": 5}
DEFAULT_POSE_SWITCHES = dict(pm_mode=0, pm_type=0, pm_norm_extent=1, rot_type=-1, centroid_type=0, z_type=0, trans_type=-1,
                             trans_disentangle=1, bind_type=-1)


def pose_loss_switches(pnp_cfg) -> tuple:
    """(switches dict, the pose-side loss names in loss_dict order) of a PNP_NET config; raises ValueError naming the offending key.
    PyPMLoss (pm_loss.py:58-171): R_ONLY wins, DISENTANGLE_Z implies DISENTANGLE_T, without either t joins the points.  The
    centroid and z losses are always computed (GDRN.forward drops them when their weight is 0)."""
    p = pnp_cfg
    sw = dict(DEFAULT_POSE_SWITCHES, pm_beta=float(p.get("PM_SMOOTH_L1_BETA", 1.0)), pm_norm_extent=int(bool(p.PM_NORM_BY_EXTENT)))
    names = []
    pm_type = str(p.PM_LOSS_TYPE).lower()
    if pm_type not in POSE_LOSS_KINDS:
        raise ValueError(f"PNP_NET.PM_LOSS_TYPE = {p.PM_LOSS_TYPE!r} (L1, Smooth_L1, MSE or L2)")
    sw["pm_type"] = POSE_LOSS_KINDS[pm_type]
    if p.PM_LW <= 0:
        mode = "off"
    elif p.PM_R_ONLY:
        mode, names = "R", ["loss_PM_R"]
    elif p.PM_DISENTANGLE_Z:
        mode = "Z" if p.PM_T_USE_POINTS else "Z_noP"
        names = ["loss_PM_R", "loss_PM_xy", "loss_PM_z"] if p.PM_T_USE_POINTS else ["loss_PM_R", "loss_PM_xy_noP", "loss_PM_z_noP"]
    elif p.PM_DISENTANGLE_T:
        mode = "T" if p.PM_T_USE_POINTS else "T_noP"
        names = ["loss_PM_R", "loss_PM_T"] if p.PM_T_USE_POINTS else ["loss_PM_R", "loss_PM_T_noP"]
    else:
        mode, names = "RT", ["loss_PM_RT"]
    sw["pm_mode"] = PM_MODES[mode]

    def kind3(key):
        v = p.get(key, "L1")
        if v not in POSE_LOSS_KINDS3:
            raise ValueError(f"PNP_NET.{key} = {v!r} (L1, L2 or MSE)")
        return POSE_LOSS_KINDS3[v]

    if p.ROT_LW > 0:
        if p.ROT_LOSS_TYPE not in ("angular", "L2"):
            raise ValueError(f"PNP_NET.ROT_LOSS_TYPE = {p.ROT_LOSS_TYPE!r} (angular or L2)")
        sw["rot_type"] = 0 if p.ROT_LOSS_TYPE == "angular" else 1
        names.append("loss_rot")
    sw["centroid_type"] = kind3("CENTROID_LOSS_TYPE") if p.CENTROID_LW > 0 else 0
    sw["z_type"] = kind3("Z_LOSS_TYPE") if p.Z_LW > 0 else 0
    names += ["loss_centroid", "loss_z"]
    if p.TRANS_LW > 0:
        sw["trans_type"] = kind3("TRANS_LOSS_TYPE")
        sw["trans_disentangle"] = int(bool(p.TRANS_LOSS_DISENTANGLE))
        names += ["loss_trans_xy", "loss_trans_z"] if p.TRANS_LOSS_DISENTANGLE else ["loss_trans_LPnP"]
    if p.get("BIND_LW", 0.0) > 0:
        # GDRN.py:505-512: L1, L2, else MSE when CENTROID_LOSS_TYPE (sic) is "MSE", else a ValueError
        bt = p.get("BIND_LOSS_TYPE", "L1")
        if bt in ("L1", "L2"):
            sw["bind_type"] = POSE_LOSS_KINDS3[bt]
        elif p.CENTROID_LOSS_TYPE == "MSE":
            sw["bind_type"] = POSE_LOSS_KINDS3["MSE"]
        else:
            raise ValueError(f"PNP_NET.BIND_LOSS_TYPE = {bt!r} (L1 or L2, or anything with CENTROID_LOSS_TYPE = 'MSE', which then "
                             "selects MSE)")
        names.append("loss_bind")
    return sw, names


def check_roi_classes(roi_classes, B: int, num_classes: int):
    """ValueError unless roi_classes holds B integer class indices in [0, num_classes) (reference GDRN.py:134-151 asserts that
    they are given and indexes with them).  Costs one small device-to-host copy when they live on the device."""
    if roi_classes is None:
        raise ValueError("roi_classes is required: the geometry head is class-aware (ROT_HEAD.*_CLASS_AWARE)")
    c = torch.as_tensor(roi_classes)
    if c.dtype.is_floating_point or c.dtype.is_complex or c.dtype == torch.bool:
        raise ValueError(f"roi_classes: expected integer class indices, got {c.dtype}")
    if c.numel() != B:
        raise ValueError(f"roi_classes: expected {B} class indices, got shape {tuple(c.shape)}")
    lo, hi = torch.stack([c.min(), c.max()]).tolist()
    if lo < 0 or hi >= num_classes:
        raise ValueError(f"roi_classes: class indices must lie in [0, NUM_CLASSES = {num_classes}), got [{lo}, {hi}]")
    return c


def class_rows(num_classes: int, mo: int, num_regions: int, rot_aware: bool, mask_aware: bool, region_aware: bool):
    """(rows, n_rows): rows[c] lists the output-conv rows of class c in the engine's logit order (mask | x y z | bg | R regions),
    n_rows the output conv's row count.  The reference's layout (cdpn_rot_head_region.py:114-135, 186-193; GDRN.py:134-151):
    [mask, MO per class if MASK_CLASS_AWARE] [x_0..x_{C-1} | y_0.. | z_0.. if ROT_CLASS_AWARE, else x y z] [bg + R regions, per
    class if REGION_CLASS_AWARE]; a block that is not class-aware is shared by every class."""
    cm, cr, cg = (num_classes if mask_aware else 1), (num_classes if rot_aware else 1), (num_classes if region_aware else 1)
    xyz0 = mo * cm
    reg0 = xyz0 + 3 * cr
    rows = []
    for c in range(num_classes):
        r = [(c if mask_aware else 0) * mo + j for j in range(mo)]
        r += [xyz0 + a * cr + (c if rot_aware else 0) for a in range(3)]
        r += [reg0 + (c if region_aware else 0) * (num_regions + 1) + j for j in range(num_regions + 1)]
        rows.append(r)
    return rows, reg0 + (num_regions + 1) * cg


class _BN:
    """Per-BatchNorm scratch: scale/shift (forward), mean/invstd (backward), statistic slices."""

    def __init__(self, C_, dev):
        self.scale = torch.empty(C_, device=dev)
        self.shift = torch.empty(C_, device=dev)
        self.mean = torch.empty(C_, device=dev)
        self.invstd = torch.empty(C_, device=dev)
        self.sums = torch.empty(2, C_, device=dev)
        self.stats = None  # view into Engine.stats_all
        self.stats64 = None  # view into Engine.stats64_all: the epilogue statistics of the atomic path


class SymTable:
    """Device-resident table of symmetry rotations (reference `sym_infos`: per-object [K,3,3] model-to-model transforms,
    core/utils/pose_utils.py:457-482, built per dataset by misc.get_symmetry_transformations).  Each distinct object is
    uploaded ONCE; a step only sends B (first row, count) pairs, so the symmetric PM loss needs no per-step packing of
    the matrices, no host loop over candidates and is CUDA-graph capturable (fixed table address, fixed capacity)."""

    CAPACITY = 16384  # rows (YCB-V: 21 objects x <= 628 discretised transforms fits several times over)

    def __init__(self, dev):
        self.dev = dev
        self.table = torch.zeros(self.CAPACITY, 3, 3, device=dev)
        self.rows = 0
        self._by_id = {}     # id(obj) -> (obj, first, count): fast path for the per-dataset arrays reused every step
        self._by_bytes = {}  # content -> (first, count)

    def _register(self, s):
        import numpy as np

        arr = s.detach().cpu().numpy() if isinstance(s, torch.Tensor) else np.asarray(s)
        arr = np.ascontiguousarray(arr, dtype=np.float32).reshape(-1, 3, 3)
        key = arr.tobytes()
        ent = self._by_bytes.get(key)
        if ent is None:
            k = arr.shape[0]
            if self.rows + k > self.CAPACITY:
                raise RuntimeError(f"symmetry table full ({self.rows} + {k} > {self.CAPACITY} rows)")
            self.table[self.rows:self.rows + k].copy_(torch.from_numpy(arr))
            ent = (self.rows, k)
            self.rows += k
            self._by_bytes[key] = ent
        return ent

    def indices(self, sym_infos) -> torch.Tensor:
        """list[B] of None | [K,3,3] -> int32 [B,2] (first row, count) on the device (one small async H2D copy)."""
        out = torch.zeros(len(sym_infos), 2, dtype=torch.int32).pin_memory()
        for b, s in enumerate(sym_infos):
            if s is None:
                continue
            hit = self._by_id.get(id(s))
            if hit is None or hit[0] is not s:
                first, count = self._register(s)
                if len(self._by_id) > 4096:
                    self._by_id.clear()
                self._by_id[id(s)] = (s, first, count)
            else:
                first, count = hit[1], hit[2]
            out[b, 0], out[b, 1] = first, count
        return out.to(self.dev, non_blocking=True)


class Engine:
    def __init__(self, model, precision: str = "half"):
        precision = {"bf16": "half", "fp16": "half"}.get(precision, precision)
        assert precision in ("half", "fp32x3", "mixed"), precision
        C.load()  # fail loudly if the CUDA library is missing
        self.model = model
        self.precision = precision
        self.planes = 1 if precision == "half" else 2      # forward activations / forward weight operands
        self.bplanes = 2 if precision == "fp32x3" else 1   # activation gradients / dgrad weight operands
        self.dev = next(model.parameters()).device
        if self.dev.type != "cuda":
            raise RuntimeError("gdr_net_b200 engine needs CUDA parameters (model.to('cuda')); no CPU fallback exists")
        self.ws = ops.Workspace(self.dev)
        self.sym_table = SymTable(self.dev)
        self.wgrad_side_stream = True  # weight gradients and the weight pack on a second stream (_on_side)
        self._side_stream, self._side_keep = None, []
        # BatchNorm batch statistics and backward sums in two ordered stages (default) instead of fp32 atomics in the GEMM
        # epilogue: the same inputs give the same step every run.  With atomics the ~1e-7 jitter of the statistics flips
        # ReLU / L1 decisions and moves gradients by up to ~5e-2; the ordered statistics cost one extra read of every pre-BN
        # tensor in forward (3 % of the B = 64 step on an H100).  GDRN_DETERMINISTIC=0 selects the atomics.
        self.deterministic = os.environ.get("GDRN_DETERMINISTIC", "1") == "1"
        self._det_ws = None
        self.fold_eval = True  # inference by forward_eval_folded; False runs it through the unfused train-path kernels
        # surface regions (ROT_HEAD.NUM_REGIONS = R) and the Patch-PnP input (GDRN.py:156-181): xyz | coord2d (WITH_2D_COORD) |
        # softmax over the R region logits (REGION_ATTENTION), nIn channels in rows of pnp_ld = round_up(nIn, 64)
        rh = model.cfg.MODEL.CDPN.ROT_HEAD
        self.num_regions = int(rh.NUM_REGIONS)
        self.region_att = int(bool(model.cfg.MODEL.CDPN.PNP_NET.REGION_ATTENTION))
        n_in = model.pnp_net.features[0].in_channels
        self.with_2d = int(n_in - 3 - self.region_att * self.num_regions == 2)
        assert n_in == 3 + 2 * self.with_2d + self.region_att * self.num_regions, (n_in, self.num_regions, self.region_att)
        self.pnp_ld = -(-n_in // 64) * 64
        # the shipped head (64 regions with attention) runs the gdrn_*_ex loss kernels, every other one the gdrn_*_ex2 ones
        self.regions_ex2 = not (self.num_regions == 64 and self.region_att)
        # DropBlock on the Patch-PnP input (PNP_HEAD_CFG.drop_prob, dropblock_size; ConvPnPNet): with drop_prob > 0 every forward
        # advances the device-resident schedule counter and a train-mode one runs the gdrn_*_db glue and head backward
        self.drop_prob = float(model.pnp_net.drop_prob)
        if self.drop_prob > 0:
            model.pnp_net.dropblock_counter(self.dev)
        # mask head (GDRN.py:339-400): MASK_LOSS_TYPE, the mask logits per pixel (1, or 2 for CE) and the GT mask of the xyz, mask
        # and region losses (XYZ_LOSS_MASK_GT, MASK_LOSS_GT, REGION_LOSS_MASK_GT)
        self.mask_loss = MASK_LOSSES[rh.MASK_LOSS_TYPE]
        self.mask_out = 2 if self.mask_loss == MASK_LOSSES["CE"] else 1
        self.n_logits = self.mask_out + 4 + self.num_regions  # per crop: mask | xyz | bg | R regions
        # head shape (ROT_HEAD.CONV_KERNEL_SIZE, OUT_CONV_KERNEL_SIZE; GDRN.check_head_shape): the deconv's kernel k and padding
        # (k3 p1 op1, k4 p1, k2 p0: 8x8 -> 16x16 every time) and the output conv's kernel (1 or 3, pad k // 2: 64x64 logits)
        hf = model.rot_head_net.features
        self.deconv_k, self.deconv_pad, self.out_k = hf[0].kernel_size[0], hf[0].padding[0], hf[23].kernel_size[0]
        # class-aware head (ROT_HEAD.*_CLASS_AWARE): the output conv holds per-class rows (class_rows) and every crop's logits come
        # from its class's rows, selected per 128-row tile by the grouped GEMMs -- the logit row layout stays the one above
        aware = (bool(rh.ROT_CLASS_AWARE), bool(rh.MASK_CLASS_AWARE), bool(rh.REGION_CLASS_AWARE))
        self.class_aware = any(aware)
        self.num_classes = int(rh.NUM_CLASSES) if self.class_aware else 1
        rows, n_rows = class_rows(self.num_classes, self.mask_out, self.num_regions, *aware)
        assert model.rot_head_net.features[23].out_channels == n_rows, (model.rot_head_net.features[23].out_channels, n_rows)
        if self.class_aware:
            self._init_class_tables(rows, n_rows)
        self.mask_gt = (rh.XYZ_LOSS_MASK_GT, rh.MASK_LOSS_GT, rh.REGION_LOSS_MASK_GT)
        # pose losses (PNP_NET switches): the shipped set runs gdrn_pose_loss (8 losses, LOSS_NAMES), any other gdrn_pose_loss_ex
        sw, pose_names = pose_loss_switches(model.cfg.MODEL.CDPN.PNP_NET)
        self.loss_names = LOSS_NAMES[:5] + pose_names
        self.pose_ex = any(sw[k] != v for k, v in DEFAULT_POSE_SWITCHES.items())
        from .capi import PoseSwitches

        self.pose_sw = PoseSwitches(**sw)
        assert self.pose_ex or self.loss_names == LOSS_NAMES, self.loss_names
        # frozen sub-networks (BACKBONE / ROT_HEAD / PNP_NET .FREEZE, GDRN.py:550-700): the reference runs a frozen backbone or
        # head under no_grad and detaches its output, so a frozen head also cuts the backbone off; a frozen Patch-PnP only
        # stops its own parameters.  live_* = that sub-network's parameters receive gradients; a frozen head's per-pixel
        # losses are not computed (gdrn_loss, GDRN.py:342-400)
        cd = model.cfg.MODEL.CDPN
        self.freeze = (bool(cd.BACKBONE.FREEZE), bool(rh.FREEZE), bool(cd.PNP_NET.FREEZE))
        self.live_head = not self.freeze[1]
        self.live_bb = self.live_head and not self.freeze[0]
        self.live_pnp = not self.freeze[2]
        self.live_any = self.live_head or self.live_pnp
        self.n_pix = 5 if self.live_head else 0  # per-pixel losses at the head of the loss vector
        if not self.live_head:
            self.loss_names = self.loss_names[5:]
        assert int(C.load().gdrn_pose_loss_count(self.pose_sw)) == len(pose_names), (sw, pose_names)
        self.named_params = list(model.named_parameters())
        # geometry-head normalisation (ROT_HEAD.NORM): "GN" takes the head's seven norm layers out of the BatchNorm tables, the
        # statistic slices and the fold jobs; they run the gdrn_head_gn_* kernels (no running statistics: train = eval)
        self.head_gn = rh.NORM == "GN"
        self._gn_mods = {n: m for n, m in model.rot_head_net.named_modules(prefix="rot_head_net")
                         if isinstance(m, torch.nn.GroupNorm)} if self.head_gn else {}
        self._last_gstats = None
        self.bn: Dict[str, _BN] = {}
        total = 0
        self._bn_mods = {}
        for name, m in model.named_modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                self.bn[name] = _BN(m.num_features, self.dev)
                self._bn_mods[name] = m
                total += 2 * m.num_features
        self.stats_all = torch.zeros(total, device=self.dev)
        # GEMM-epilogue statistics (deterministic = False): the CTAs' partial sums are added in double, so the result does not
        # move with the order of the atomics beyond the fp32 rounding of each partial
        self.stats64_all = torch.zeros(total, dtype=torch.float64, device=self.dev)
        self.bwd_sums_all = torch.zeros(total, device=self.dev)  # BN-backward accumulators: one memset per backward
        off = 0
        for name, m in self._bn_mods.items():
            n = 2 * m.num_features
            self.bn[name].stats = self.stats_all[off:off + n]
            self.bn[name].stats64 = self.stats64_all[off:off + n]
            self.bn[name].sums = self.bwd_sums_all[off:off + n].view(2, m.num_features)
            off += n
        # flat gradient buffer (one NCCL-friendly allocation); per-parameter views
        self.flat_grad = torch.zeros(sum(p.numel() for _, p in self.named_params), device=self.dev)
        self.grads: Dict[str, torch.Tensor] = {}
        off = 0
        for name, p in self.named_params:
            self.grads[name] = self.flat_grad[off:off + p.numel()].view_as(p)
            off += p.numel()
        self.saved = None
        self.wf: Dict[str, PT] = {}
        self.wd: Dict[str, PT] = {}
        self.grad_hook = None  # optional callable(engine) invoked at bucket boundaries during backward (DDP overlap)
        self.use_cuda_graphs = False  # module API: replay forward / backward CUDA graphs (fixed shapes, no symmetric PM)
        self._graphed = None
        # fp16 planes: activation gradients are carried with a static power-of-two loss scale (exactly removed from the
        # fp32 parameter gradients at the end of backward), like the GradScaler of the reference's AMP configs
        self.storage_name = ops.storage_format()[2]
        # The pose-loss switches bring gradients up to ~sqrt(n) w / B per unit loss (L2 point matching: 2e2 at n = 3000, B = 4),
        # which overflow fp16 at 1024; 64 keeps them in range and the smallest (mask channel, 1 / (B 4096) at B = 64) normal.
        self.grad_scale = (64.0 if self.pose_ex else 1024.0) if self.storage_name == "fp16" else 1.0
        from .dist import SEGMENTS, segment_bounds

        self._seg = segment_bounds(self.named_params, SEGMENTS)
        # (parameter, flat_grad offset) of every parameter that can receive a gradient: only these enter _GDRNFunction, so
        # every other parameter keeps .grad None
        live = lambda n: self.live_pnp if n.startswith("pnp_net.") else self.live_head if n.startswith("rot_head_net.") else self.live_bb  # noqa: E731
        self.live_params, off = [], 0
        for name, p in self.named_params:
            if live(name):
                self.live_params.append((p, off))
            off += p.numel()

    def _init_class_tables(self, rows, n_rows):
        """Device tables of the class-aware head: cls_idx [C * cls_npad] = the output-conv row behind each slot of the class-major
        weight table (-1: zero padding), cls_slot [C][n_rows] = the logit slot of each row for each class (-1: not used by it),
        and the persistent class-major fp32 tables w_cls [C * cls_npad][256] / b_cls that every step gathers and packs."""
        import numpy as np

        C_, npad = self.num_classes, -(-self.n_logits // 64) * 64
        idx = np.full(C_ * npad, -1, dtype=np.int32)
        slot = np.full((C_, n_rows), -1, dtype=np.int32)
        for c, r in enumerate(rows):
            idx[c * npad:c * npad + len(r)] = r
            slot[c, r] = np.arange(len(r))
        self.cls_npad, self.cls_rows = npad, n_rows
        self.cls_idx = torch.from_numpy(idx).to(self.dev)
        self.cls_slot = torch.from_numpy(slot).to(self.dev)
        self.w_cls = torch.zeros(C_ * npad, 256 * self.out_k * self.out_k, device=self.dev)
        self.b_cls = torch.zeros(C_ * npad, device=self.dev)

    def _classes(self, roi_classes, B: int) -> torch.Tensor:
        """roi_classes [B] (any integer dtype, host or device; GDRN.forward checked the range) -> int32 [B] on the device.  The
        kernels clamp a class outside [0, NUM_CLASSES) to the nearest table entry instead of reading outside the tables."""
        if roi_classes is None:
            raise ValueError("roi_classes is required: the geometry head is class-aware (ROT_HEAD.*_CLASS_AWARE)")
        c = torch.as_tensor(roi_classes)
        if c.numel() != B:
            raise ValueError(f"roi_classes: expected {B} class indices, got shape {tuple(c.shape)}")
        return c.reshape(B).to(self.dev, torch.int32).contiguous()

    # ------------------------------------------------------------------------------------------ weights
    def _conv_modules(self):
        """(key, module) of every conv packed by pack_conv_fwd; the 7x7 stem is a GEMM over its im2col matrix (pack_stem)."""
        m = self.model
        out = []
        for li in range(1, 5):
            for bi, blk in enumerate(getattr(m.backbone, f"layer{li}")):
                p = f"backbone.layer{li}.{bi}"
                out.append((p + ".conv1", blk.conv1))
                out.append((p + ".conv2", blk.conv2))
                if blk.downsample is not None:
                    out.append((p + ".downsample.0", blk.downsample[0]))
        for ci, _bi, _u in HEAD_CONVS:
            out.append((f"rot_head_net.features.{ci}", m.rot_head_net.features[ci]))
        out.append(("rot_head_net.features.23", m.rot_head_net.features[23]))
        for ci in (0, 3, 6):
            out.append((f"pnp_net.features.{ci}", m.pnp_net.features[ci]))
        return out

    def prepare_weights(self, need_dgrad: bool):
        """fp32 parameters -> K-major bf16 (hi, lo) GEMM operands, re-done every step (weights change) by ONE batched
        launch over a device-resident job table (rebuilt only if a parameter / buffer pointer moved)."""
        key = (need_dgrad, tuple(p.data_ptr() for _, p in self.named_params))
        tables = self.__dict__.setdefault("_pack_tables", {})
        tab = tables.get(key)
        if tab is None:
            # One persistent job table per (need_dgrad, parameter addresses).  Tables are NEVER freed or overwritten: a
            # captured CUDA graph holds the raw device pointer of the table it was captured with, and an eager call with
            # the other need_dgrad value (train -> eval -> train) must not invalidate it (ADVICE r1).
            tab = tables[key] = self._pack_table(lambda: self._prepare_weights_calls(need_dgrad))
        with torch.no_grad():
            torch.cat([self.model.pnp_net.fc_r.weight, self.model.pnp_net.fc_t.weight], 0, out=self.w_rt)
            torch.cat([self.model.pnp_net.fc_r.bias, self.model.pnp_net.fc_t.bias], 0, out=self.b_rt)
        if self.class_aware:  # the class-major tables the pack jobs of the output conv read
            w23 = self.model.rot_head_net.features[23]
            n = self.num_classes * self.cls_npad
            C.gdrn_class_gather(w23.weight.data_ptr(), self.cls_idx.data_ptr(), self.w_cls.data_ptr(), n, self.w_cls.shape[1],
                                self.cls_rows, _stream())
            C.gdrn_class_gather(w23.bias.data_ptr(), self.cls_idx.data_ptr(), self.b_cls.data_ptr(), n, 1, self.cls_rows, _stream())
        C.gdrn_pack_weight_batched(tab["jobs"].data_ptr(), tab["njobs"], tab["blocks"], _stream())

    def _pack_table(self, pack, row_scales=None) -> dict:
        """Runs pack() with its ops.pack_* calls recorded instead of launched and returns them as the device job table of
        gdrn_pack_weight_batched (jobs, njobs, blocks).  row_scales[n], if given, multiplies every output row of job n.
        The table keeps the jobs' sources and destinations alive."""
        import numpy as np

        ops._pack_recorder = []
        try:
            pack()
            jobs = ops._pack_recorder
        finally:
            ops._pack_recorder = None
        assert row_scales is None or len(row_scales) == len(jobs)
        dt = np.dtype([("src", "<u8"), ("hi", "<u8"), ("lo", "<u8"), ("so", "<i8"), ("si", "<i8"), ("sr", "<i8"), ("ss", "<i8"),
                       ("begin", "<i8"), ("O", "<i4"), ("I", "<i4"), ("KH", "<i4"), ("KW", "<i4"), ("opad", "<i4"),
                       ("ipad", "<i4"), ("krow", "<i4"), ("flip", "<i4"), ("row_scale", "<u8")])  # struct PackJob (pack.cu)
        assert dt.itemsize == 104
        arr = np.zeros(len(jobs), dtype=dt)
        begin = 0
        for n, (src, out, O, I, KH, KW, opad, ipad, krow, so, si, sr, ss, flip) in enumerate(jobs):
            scale = 0 if row_scales is None else row_scales[n].data_ptr()
            arr[n] = (src.data_ptr(), out.hi_ptr, out.lo_ptr or 0, so, si, sr, ss, begin, O, I, KH, KW, opad, ipad, krow, flip, scale)
            begin += -(-opad // 16) * -(-ipad // 64) * -(-(KH * KW) // 9)  # tiles of 16 rows x 64 channels x 9 taps (pack.cu)
        return dict(jobs=torch.from_numpy(arr.view(np.uint8).copy()).to(self.dev), njobs=len(jobs), blocks=begin,
                    keep=[j[0] for j in jobs] + [j[1] for j in jobs])

    # ------------------------------------------------------------------------------------------ eval: folded conv+BN+ReLU
    # (conv key, BatchNorm key) of every conv that is followed by a BatchNorm, in forward order
    def _conv_bn_pairs(self):
        m = self.model
        out = [("stem", "backbone.bn1")]
        for li in range(1, 5):
            for bi, blk in enumerate(getattr(m.backbone, f"layer{li}")):
                p = f"backbone.layer{li}.{bi}"
                out += [(p + ".conv1", p + ".bn1"), (p + ".conv2", p + ".bn2")]
                if blk.downsample is not None:
                    out.append((p + ".downsample.0", p + ".downsample.1"))
        if not self.head_gn:  # GroupNorm has no running statistics to fold
            out.append(("deconv", "rot_head_net.features.1"))
            out += [(f"rot_head_net.features.{ci}", f"rot_head_net.features.{bi}") for ci, bi, _u in HEAD_CONVS]
        return out

    def prepare_weights_folded(self):
        """Inference operands: eval-mode BatchNorm folded into the conv weights (scale, at pack time) and the conv epilogue
        (shift as bias), so conv + BN (+ identity) + ReLU is ONE kernel per layer.  Two launches per forward:
        gdrn_bn_fold_batched (all layers' scale / shift from the running statistics) and one batched weight pack."""
        import numpy as np

        key = tuple(p.data_ptr() for _, p in self.named_params)
        fold = getattr(self, "_fold", None)
        if fold is None or fold["key"] != key:
            m, pl = self.model, self.planes
            pairs = self._conv_bn_pairs()
            convs = dict(self._conv_modules())
            wfe, sc, sh = {}, {}, {}
            fdt = np.dtype([("gamma", "<u8"), ("beta", "<u8"), ("mean", "<u8"), ("var", "<u8"), ("scale", "<u8"), ("shift", "<u8"),
                            ("C", "<i4"), ("eps", "<f4"), ("pad", "<i8")])
            assert fdt.itemsize == 64
            farr = np.zeros(len(pairs), dtype=fdt)
            for n, (ck, bk) in enumerate(pairs):
                mod = self._bn_mods[bk]
                sc[bk] = torch.empty(mod.num_features, device=self.dev)
                sh[bk] = torch.empty(mod.num_features, device=self.dev)
                farr[n] = (mod.weight.data_ptr(), mod.bias.data_ptr(), mod.running_mean.data_ptr(), mod.running_var.data_ptr(),
                           sc[bk].data_ptr(), sh[bk].data_ptr(), mod.num_features, float(mod.eps), 0)

            def pack():  # one job per (conv, BatchNorm) pair, its rows scaled by that BatchNorm's scale
                for ck, _bk in pairs:
                    if ck == "stem":
                        wfe[ck] = ops.pack_stem(m.backbone.conv1.weight, pl)
                    elif ck == "deconv":
                        wfe[ck] = ops.pack_conv_dgrad(m.rot_head_net.features[0].weight, pl)  # see _prepare_weights_calls
                    else:
                        wfe[ck] = ops.pack_conv_fwd(convs[ck].weight, pl)

            fold = self._fold = dict(key=key, wf=wfe, scale=sc, shift=sh, nfold=len(pairs),
                                     fjobs=torch.from_numpy(farr.view(np.uint8).copy()).to(self.dev),
                                     **self._pack_table(pack, row_scales=[sc[bk] for _ck, bk in pairs]))
        C.gdrn_bn_fold_batched(fold["fjobs"].data_ptr(), fold["nfold"], _stream())
        C.gdrn_pack_weight_batched(fold["jobs"].data_ptr(), fold["njobs"], fold["blocks"], _stream())
        return fold

    def forward_eval_folded(self, x: torch.Tensor, aux: dict, want_maps: bool = False) -> dict:
        """Inference forward (reference caller gdrn_evaluator.py:568-580) with every conv + BatchNorm (+ residual) + ReLU
        fused into the GEMM epilogue: no BatchNorm pass, no pre-activation tensor in HBM."""
        m, pl, dev = self.model, self.planes, self.dev
        B = x.shape[0]
        assert x.shape[1:] == (3, 256, 256), x.shape
        fold_box = {}

        def packs():  # weight operands are input-independent: packed on the side stream while the main stream builds the im2col matrix
            self.prepare_weights(need_dgrad=False)  # head 1x1 / Patch-PnP / FC operands (no BatchNorm behind them)
            fold_box["F"] = self.prepare_weights_folded()

        self._on_side(packs)

        def cbr(xin, ck, bk, conv, relu=True, res=None):
            gn = self._gn_mods.get(bk)
            if gn is not None:  # GroupNorm head: the unfolded conv, then GroupNorm + ReLU
                u = (ops.conv_dgrad_s2(xin, self.wf[ck], conv.out_channels, self.deconv_k, self.deconv_pad) if ck == "deconv"
                     else ops.conv_fwd(xin, self.wf[ck], conv.out_channels, 3, 3, 1, 1))
                return ops.head_gn_relu_fwd(u, gn.weight, gn.bias, gn.num_groups, gn.eps)[0]
            if ck == "deconv":
                return ops.conv_dgrad_s2(xin, wfe[ck], conv.out_channels, self.deconv_k, self.deconv_pad, bias=shift[bk],
                                         act=2 if relu else 0)
            k, stride, pad = conv.kernel_size[0], conv.stride[0], conv.padding[0]
            return ops.conv_fwd(xin, wfe[ck], conv.out_channels, k, k, stride, pad, bias=shift[bk], act=2 if relu else 0, res=res)

        a_col = PT((B * 128 * 128, 192), pl, device=dev)
        C.gdrn_stem_im2col(x.data_ptr(), a_col.hi_ptr, a_col.lo_ptr, B, 256, 256, _stream())
        self._join_side(force=True)
        wfe, shift = fold_box["F"]["wf"], fold_box["F"]["shift"]
        a0 = ops.gemm_fwd(a_col, wfe["stem"], 64, bias=shift["backbone.bn1"], act=2).view(B, 128, 128, 64)
        cur = ops.maxpool_fwd(a0)
        for li in range(1, 5):
            for bi, blk in enumerate(getattr(m.backbone, f"layer{li}")):
                p = f"backbone.layer{li}.{bi}"
                a1 = cbr(cur, p + ".conv1", p + ".bn1", blk.conv1)
                idn = cur
                if blk.downsample is not None:
                    idn = cbr(cur, p + ".downsample.0", p + ".downsample.1", blk.downsample[0], relu=False)
                cur = cbr(a1, p + ".conv2", p + ".bn2", blk.conv2, res=idn)
        hf = m.rot_head_net.features
        cur = cbr(cur, "deconv", "rot_head_net.features.1", hf[0])
        for ci, bi, up in HEAD_CONVS:
            if up:
                cur = ops.upsample2x_fwd(cur)
            cur = cbr(cur, f"rot_head_net.features.{ci}", f"rot_head_net.features.{bi}", hf[ci])
        return self._tail_inference(cur, aux, want_maps, train=False)

    def _eval_graphed(self, x: torch.Tensor, aux: dict, want_maps: bool) -> dict:
        """Inference forward replayed as ONE CUDA graph per input signature (`use_cuda_graphs`): ~230 launches incl. the
        BatchNorm folding and the weight pack (so updated weights / running statistics are picked up at every replay)."""
        tens = {k: v for k, v in aux.items() if isinstance(v, torch.Tensor)}
        key = (tuple(x.shape), want_maps, tuple(sorted((k, tuple(v.shape)) for k, v in tens.items())),
               tuple(p.data_ptr() for _, p in self.named_params))
        cache = self.__dict__.setdefault("_eval_graphs", {})
        if key not in cache:
            inputs = _clone_inputs(x, aux)
            [(graph, res)] = _capture(self, [lambda: self.forward_eval_folded(*inputs, want_maps=want_maps)], warmup=1)
            if len(cache) > 8:
                cache.clear()
            cache[key] = (inputs, graph, res)
        inputs, graph, res = cache[key]
        _copy_inputs(*inputs, x, aux)
        graph.replay()
        return {k: (v.clone() if isinstance(v, torch.Tensor) else v) for k, v in res.items()}

    def _head_pnp(self, head_in: PT, aux: dict, pnp_saved: Optional[list] = None, train: bool = False):
        """output conv (1x1 or 3x3) -> glue -> Patch-PnP (GDRN.py:156-181, conv_pnp_net.py:111-157).  Returns the fp32 logits
        [B*4096, 72] (n_logits valid), the Patch-PnP input planes [B, 64, 64, pnp_ld], pred [B, 16] (cols 0..5 rot6d, 6..8 centroid dx, dy and z), the inputs
        of the three FC layers and the DropBlock (keep, scale) of a train-mode forward with drop_prob > 0, else None; pnp_saved
        receives the Patch-PnP conv activations (pnp_net_forward)."""
        m, B, dev = self.model, head_in.shape[0], self.dev
        logits = torch.empty(B * 4096, 72, device=dev)
        if self.class_aware:  # crop b (4096 rows) reads the weight / bias block of class roi_classes[b]
            ops.conv_fwd_grouped(head_in, self.wf["rot_head_net.features.23"], self.n_logits, self.cls_npad, aux["roi_classes"], 4096,
                                 out_f32=logits, bias=self.b_cls, bias_stride=self.cls_npad, ldc=72, k=self.out_k)
        else:
            k = self.out_k
            ops.conv_fwd(head_in, self.wf["rot_head_net.features.23"], self.n_logits, k, k, 1, k // 2, out_f32=logits,
                         bias=m.rot_head_net.features[23].bias, ldc=72, want_planes=False)
        pnp_in = PT((B, 64, 64, self.pnp_ld), self.planes, device=dev)
        glue = (logits.data_ptr(), ops.ptr(aux.get("roi_coord_2d")), aux["roi_extents"].data_ptr(), pnp_in.hi_ptr, pnp_in.lo_ptr, B, 4096,
                self.with_2d, self.mask_out)
        db = dropblock_step(m.pnp_net, B, train, dev) if self.drop_prob > 0 else None
        if db is not None:
            C.gdrn_head_glue_fwd_db(*glue, self.num_regions, self.region_att, self.pnp_ld, db[0].data_ptr(), db[1].data_ptr(), _stream())
        elif self.regions_ex2:
            C.gdrn_head_glue_fwd_ex2(*glue, self.num_regions, self.region_att, self.pnp_ld, _stream())
        else:
            C.gdrn_head_glue_fwd_ex(*glue, _stream())
        pred = torch.zeros(B, 16, device=dev)
        fc_in = pnp_net_forward(pnp_in, m.pnp_net, self.wf, self.b_rt, pred, pnp_saved)
        return logits, pnp_in, pred, fc_in, db

    def _tail_inference(self, head_in: PT, aux: dict, want_maps: bool, train: bool) -> dict:
        """output conv -> glue -> Patch-PnP -> test-time pose decode (shared by the folded and the plain eval forward);
        train: DropBlock applies (a train-mode forward without losses)."""
        B = head_in.shape[0]
        logits, _, pred, _, _ = self._head_pnp(head_in, aux, train=train)
        out_rot = torch.empty(B, 3, 3, device=self.dev)
        out_trans = torch.empty(B, 3, device=self.dev)
        C.gdrn_pose_loss(pred.data_ptr(), 16, aux["roi_cams"].data_ptr(), aux["roi_centers"].data_ptr(),
                         aux["roi_whs"].data_ptr(), aux["resize_ratios"].data_ptr(), aux["roi_extents"].data_ptr(), None,
                         None, None, None, None, None, None, out_rot.data_ptr(), out_trans.data_ptr(), None, None, None,
                         None, B, 0, 0, 0.0, _stream())
        res = dict(rot=out_rot, trans=out_trans, pred=pred, logits=logits)
        if want_maps:
            maps = logits.view(B, 64, 64, 72).permute(0, 3, 1, 2)
            mo = self.mask_out
            res.update(mask=maps[:, 0:mo], coor_x=maps[:, mo:mo + 1], coor_y=maps[:, mo + 1:mo + 2], coor_z=maps[:, mo + 2:mo + 3],
                       region=maps[:, mo + 3:self.n_logits])
        return res

    def _runs_dgrad(self, key: str) -> bool:
        """Whether backward runs the data gradient of the layer `key` (_conv_modules keys, "deconv", "fc*"): only where a
        gradient still has to flow to a live parameter below it."""
        if key.startswith("backbone.") or key == "deconv":
            return self.live_bb
        if key.startswith("rot_head_net.") or key == "pnp_net.features.0":
            return self.live_head
        return self.live_any  # Patch-PnP convs 3 and 6 and the FC stack

    def _prepare_weights_calls(self, need_dgrad: bool):
        m, pl, bpl = self.model, self.planes, self.bplanes
        wf, wd = self.wf, self.wd
        for key, conv in self._conv_modules():
            if key == "rot_head_net.features.23" and self.class_aware:
                self._class_head_pack_calls(need_dgrad and self._runs_dgrad(key))
                continue
            wf[key] = ops.pack_conv_fwd(conv.weight, pl, out=wf.get(key))
            if need_dgrad and self._runs_dgrad(key):
                # the logit gradient of head_bwd is 128 columns wide whatever the output conv's row count (MO + 4 + R)
                ipad = 128 if key == "rot_head_net.features.23" else None
                wd[key] = ops.pack_conv_dgrad(conv.weight, bpl, out=wd.get(key), ipad=ipad)
        dc = m.rot_head_net.features[0]
        # the ConvTranspose2d forward IS the data gradient of the stride-2 conv whose OIHW weight its IOHW weight is:
        # gdrn_conv_dgrad_s2 evaluates it by output parity over the un-dilated input (no zero-inserted tensor, 1/4 of the MACs)
        wf["deconv"] = ops.pack_conv_dgrad(dc.weight, pl, out=wf.get("deconv"))
        if need_dgrad and self._runs_dgrad("deconv"):
            wd["deconv"] = ops.pack_deconv_dgrad(dc.weight, bpl, out=wd.get("deconv"))
        pn = m.pnp_net
        wf["fc1"] = ops.pack_linear(pn.fc1.weight, pl, out=wf.get("fc1"), nhwc_from=(128, 8, 8))
        wf["fc2"] = ops.pack_linear(pn.fc2.weight, pl, out=wf.get("fc2"))
        if not hasattr(self, "w_rt"):
            self.w_rt = torch.empty(pn.fc_r.out_features + 3, pn.fc_r.in_features, device=self.dev)
            self.b_rt = torch.empty(pn.fc_r.out_features + 3, device=self.dev)
        wf["fc_rt"] = ops.pack_linear(self.w_rt, pl, out=wf.get("fc_rt"))
        if need_dgrad and self._runs_dgrad("fc_rt"):
            wd["fc1"] = ops.pack_linear(pn.fc1.weight, bpl, out=wd.get("fc1"), nhwc_from=(128, 8, 8), transpose=True)
            wd["fc2"] = ops.pack_linear(pn.fc2.weight, bpl, out=wd.get("fc2"), transpose=True)
            wd["fc_rt"] = ops.pack_linear(self.w_rt, bpl, out=wd.get("fc_rt"), transpose=True)
        wf["stem"] = ops.pack_stem(m.backbone.conv1.weight, pl, out=wf.get("stem"))

    def _class_head_pack_calls(self, need_dgrad: bool):
        """Class-aware output conv: forward operand [C * cls_npad][k * k * 256] and dgrad operand [C][256][k * k * 128] from the
        class-major table."""
        key, C_, npad, k = "rot_head_net.features.23", self.num_classes, self.cls_npad, self.out_k
        src = self.w_cls.view(C_ * npad, 256, k, k)
        self.wf[key] = ops.pack_conv_fwd(src, self.planes, out=self.wf.get(key))
        if need_dgrad:
            wd = self.wd.get(key) or PT((C_ * 256, k * k * 128), self.bplanes, device=self.dev)
            self.wd[key] = wd
            for c in range(C_):
                ops.pack_conv_dgrad(src[c * npad:(c + 1) * npad], self.bplanes, out=_PlaneRows(wd, c * 256), ipad=128)

    # ------------------------------------------------------------------------------------------ building blocks
    def _bn_fwd(self, key: str, u: PT, relu: bool, train_bn: bool, res: Optional[PT] = None) -> PT:
        """y = [relu](bn(u) [+ res]).  When the step keeps activations for backward (`self._want_masks`) and relu is set, the
        kernel also emits the ReLU mask as one BIT per element (self._last_mask): BatchNorm backward then reads 1/8 byte
        instead of the 2-byte activation per element in both of its passes."""
        mod, st = self._bn_mods[key], self.bn[key]
        Cc = mod.num_features
        count = u.numel() // Cc
        mom = mod.momentum if mod.momentum is not None else 0.1
        if train_bn and mod.num_batches_tracked is not None:
            self._nbt.append(mod.num_batches_tracked)
        if train_bn and self.deterministic:
            C.gdrn_bn_stats(u.hi_ptr, u.lo_ptr, self._det_workspace().data_ptr(), st.stats.data_ptr(), count, Cc, _stream())
        y = ops.like(u)
        mask = None
        if relu and self._want_masks:
            mask = torch.empty(u.numel() // 8, dtype=torch.uint8, device=self.dev)
        self._last_mask = mask
        C.gdrn_bn_fwd(u.hi_ptr, u.lo_ptr, res.hi_ptr if res else None, res.lo_ptr if res else None, y.hi_ptr, y.lo_ptr,
                      ops.ptr(st.stats if self.deterministic else st.stats64) if train_bn else None, mod.weight.data_ptr(),
                      mod.bias.data_ptr(), mod.running_mean.data_ptr(), mod.running_var.data_ptr(), st.mean.data_ptr(),
                      st.invstd.data_ptr(), ops.ptr(mask), count, Cc, float(mod.eps), float(mom),
                      int(train_bn) | (2 if train_bn and not self.deterministic else 0), int(relu), _stream())
        return y

    def _det_workspace(self):
        if self._det_ws is None:
            self._det_ws = torch.empty(2 * 512 * int(C.load().gdrn_det_parts()), device=self.dev)
        return self._det_ws

    def _conv_bn(self, x: PT, ckey: str, conv, bkey: str, relu: bool, train_bn: bool, res: Optional[PT] = None):
        """conv -> BatchNorm or, in a GroupNorm head, GroupNorm (+ ReLU); a GroupNorm leaves its statistics in _last_gstats."""
        gn = self._gn_mods.get(bkey)
        # deterministic: from gdrn_bn_stats
        stats = self.bn[bkey].stats64 if (gn is None and train_bn and not self.deterministic) else None
        k, stride, pad = conv.kernel_size[0], conv.stride[0], conv.padding[0]
        if ckey == "deconv":
            u = ops.conv_dgrad_s2(x, self.wf["deconv"], conv.out_channels, self.deconv_k, self.deconv_pad, stats=stats)
        else:
            u = ops.conv_fwd(x, self.wf[ckey], conv.out_channels, k, k, stride, pad, stats=stats)
        if gn is not None:
            y, self._last_gstats, self._last_mask = ops.head_gn_relu_fwd(u, gn.weight, gn.bias, gn.num_groups, gn.eps,
                                                                         want_mask=self._want_masks)
            return u, y
        return u, self._bn_fwd(bkey, u, relu, train_bn, res)

    # ------------------------------------------------------------------------------------------ forward
    def run(self, x, *, roi_coord_2d, roi_cams, roi_centers, roi_whs, roi_extents, resize_ratios, roi_classes=None, gt_xyz=None,
            gt_mask_trunc=None, gt_mask_visib=None, gt_mask_obj=None, gt_region=None, gt_ego_rot=None, gt_points=None,
            sym_infos=None, gt_trans=None, gt_trans_ratio=None, do_loss=False, train_bn=False, want_maps=False):
        aux = dict(roi_coord_2d=roi_coord_2d, roi_cams=roi_cams, roi_centers=roi_centers, roi_whs=roi_whs,
                   roi_extents=roi_extents, resize_ratios=resize_ratios, gt_xyz=gt_xyz, gt_mask_trunc=gt_mask_trunc,
                   gt_mask_visib=gt_mask_visib, gt_mask_obj=gt_mask_obj, gt_region=gt_region, gt_ego_rot=gt_ego_rot,
                   gt_points=gt_points, sym_infos=sym_infos, gt_trans=gt_trans, gt_trans_ratio=gt_trans_ratio)
        B = x.shape[0]
        for k_, v in aux.items():
            if isinstance(v, torch.Tensor):
                v = v.to(self.dev)
                # gt_region is handed to the kernels as `const long long*` (the reference calls .long() itself, GDRN.py:393,
                # and its dataset emits int32): convert ANY label dtype explicitly; everything else is fp32
                aux[k_] = (v.long() if k_ == "gt_region" else v.float()).contiguous()
        if roi_cams is not None and aux["roi_cams"].dim() == 2:  # one shared K: broadcast like the reference does
            aux["roi_cams"] = aux["roi_cams"].unsqueeze(0).expand(B, 3, 3).contiguous()
        want = dict(roi_coord_2d=(B, 2, 64, 64), roi_cams=(B, 3, 3), roi_centers=(B, 2), roi_whs=(B, 2), roi_extents=(B, 3),
                    resize_ratios=(B,), gt_xyz=(B, 3, 64, 64), gt_mask_trunc=(B, 64, 64), gt_mask_visib=(B, 64, 64),
                    gt_mask_obj=(B, 64, 64), gt_region=(B, 64, 64), gt_ego_rot=(B, 3, 3), gt_trans=(B, 3), gt_trans_ratio=(B, 3))
        for k_, shp in want.items():
            v = aux.get(k_)
            if isinstance(v, torch.Tensor):
                if v.numel() != int(torch.Size(shp).numel()):
                    raise ValueError(f"{k_}: expected shape {shp} for a batch of {B}, got {tuple(v.shape)}")
                aux[k_] = v.view(shp)
        if isinstance(aux.get("gt_points"), torch.Tensor) and (aux["gt_points"].dim() != 3 or aux["gt_points"].shape[0] != B
                                                               or aux["gt_points"].shape[2] != 3):
            raise ValueError(f"gt_points: expected [B={B}, n, 3], got {tuple(aux['gt_points'].shape)}")
        if aux.get("sym_infos") is not None:
            if len(aux["sym_infos"]) != B:
                raise ValueError(f"sym_infos: expected a list of {B} entries, got {len(aux['sym_infos'])}")
            aux["sym_idx"] = self.sym_table.indices(aux["sym_infos"])  # the matrices themselves are already on the device
        aux.pop("sym_infos", None)
        if self.class_aware:  # device data: a captured graph reads the classes of each replay from its static copy
            aux["roi_classes"] = self._classes(roi_classes, B)
        x = x.to(self.dev).float().contiguous()
        if not do_loss:
            with torch.no_grad():
                if not train_bn and self.fold_eval:  # inference: conv + BN (+ identity) + ReLU fused per layer
                    if self.use_cuda_graphs:
                        return self._eval_graphed(x, aux, want_maps)
                    return self.forward_eval_folded(x, aux, want_maps=want_maps)
                return self.forward(x, aux, train_bn=train_bn, do_loss=False, want_maps=want_maps)
        if not self.live_any:  # frozen head and Patch-PnP: nothing to differentiate, the losses do not require grad
            with torch.no_grad():
                res = self.forward(x, aux, train_bn=train_bn, do_loss=True)
            self.saved = None
            return dict(losses=res["losses"], vis=res["vis"])
        losses, vis = _GDRNFunction.apply(self, x, aux, train_bn, *[p for p, _ in self.live_params])
        return dict(losses=losses, vis=vis)

    def forward(self, x: torch.Tensor, aux: dict, train_bn: bool, do_loss: bool, want_maps: bool = False) -> dict:
        m, pl, dev = self.model, self.planes, self.dev
        B = x.shape[0]
        assert x.shape[1:] == (3, 256, 256), x.shape
        # the per-step weight re-pack (0.24 ms) does not depend on the input: it runs on the side stream while the main
        # stream builds the stem's im2col matrix, and is joined right before the first GEMM
        self._on_side(lambda: self.prepare_weights(need_dgrad=do_loss))
        self._nbt = []
        if train_bn:
            (self.stats_all if self.deterministic else self.stats64_all).zero_()
        S = dict(B=B, train_bn=train_bn) if do_loss else None
        # a sub-network nothing differentiates through (frozen, or below a frozen head) runs the non-saving path of inference
        keep_bb, keep_head = do_loss and self.live_bb, do_loss and self.live_head
        self._want_masks = keep_bb

        # ---- a1: backbone (resnet_backbone.py:69-76)
        a_col = PT((B * 128 * 128, 192), pl, device=dev)
        C.gdrn_stem_im2col(x.data_ptr(), a_col.hi_ptr, a_col.lo_ptr, B, 256, 256, _stream())
        self._join_side(force=True)
        st0 = self.bn["backbone.bn1"]
        u0 = ops.gemm_fwd(a_col, self.wf["stem"], 64, stats=st0.stats64 if (train_bn and not self.deterministic) else None).view(B, 128, 128, 64)
        a0 = self._bn_fwd("backbone.bn1", u0, True, train_bn)
        if keep_bb:
            cur, pool_arg = ops.maxpool_fwd(a0, want_arg=True)
            S["stem"] = dict(a_col=a_col, u0=u0, a0=a0, pool_arg=pool_arg, m0=self._last_mask)
            S["blocks"] = []
        else:
            cur = ops.maxpool_fwd(a0)
        for li in range(1, 5):
            for bi, blk in enumerate(getattr(m.backbone, f"layer{li}")):
                p = f"backbone.layer{li}.{bi}"
                u1, a1 = self._conv_bn(cur, p + ".conv1", blk.conv1, p + ".bn1", True, train_bn)
                m1 = self._last_mask
                ud = None
                if blk.downsample is not None:
                    ud, idn = self._conv_bn(cur, p + ".downsample.0", blk.downsample[0], p + ".downsample.1", False, train_bn)
                else:
                    idn = cur
                u2, out = self._conv_bn(a1, p + ".conv2", blk.conv2, p + ".bn2", True, train_bn, res=idn)
                if keep_bb:
                    S["blocks"].append(dict(p=p, blk=blk, x_in=cur, u1=u1, a1=a1, u2=u2, out=out, ud=ud, m1=m1, m2=self._last_mask))
                cur = out
        feat = cur  # [B,8,8,512]

        # ---- a2: geometry head (cdpn_rot_head_region.py:80-135)
        hf = m.rot_head_net.features
        self._want_masks = keep_head
        u, y = self._conv_bn(feat, "deconv", hf[0], "rot_head_net.features.1", True, train_bn)
        if keep_head:
            S["deconv"] = dict(z=feat, u=u, y=y, m=self._last_mask, gs=self._last_gstats)
            S["head"] = []
        cur = y
        for ci, bi, up in HEAD_CONVS:
            if up:
                cur = ops.upsample2x_fwd(cur)
            u, y = self._conv_bn(cur, f"rot_head_net.features.{ci}", hf[ci], f"rot_head_net.features.{bi}", True, train_bn)
            if keep_head:
                S["head"].append(dict(ci=ci, bi=bi, up=up, x_in=cur, u=u, y=y, m=self._last_mask, gs=self._last_gstats))
            cur = y
        head_in = cur  # [B,64,64,256]
        if self._nbt:
            torch._foreach_add_(self._nbt, 1)  # all BatchNorm num_batches_tracked counters in one launch
        if not do_loss:
            return self._tail_inference(head_in, aux, want_maps, train=train_bn)

        # ---- a3 + a4: glue and Patch-PnP
        pnp_saved = []
        logits, pnp_in, pred, (flat, h1, h2), db = self._head_pnp(head_in, aux, pnp_saved, train=train_bn)

        # ---- a5/a6 pose decode + a7..a10 losses
        if self.live_head:
            pix_sums = torch.empty(7, dtype=torch.float64, device=dev)
            m_xyz, m_mask, m_region = self._loss_masks(aux)
            pix = (logits.data_ptr(), aux["gt_xyz"].data_ptr(), m_xyz, m_mask, m_region, aux["gt_region"].data_ptr(), pix_sums.data_ptr(),
                   B, 4096, self.mask_loss, self.mask_out)
            if self.regions_ex2:
                C.gdrn_pixel_loss_fwd_ex2(*pix, self.num_regions, self.region_att, self.pnp_ld, _stream())
            else:
                C.gdrn_pixel_loss_fwd_ex(*pix, _stream())
        else:  # frozen head: no per-pixel losses; the finalize kernel's first five outputs are dropped below
            pix_sums = torch.zeros(7, dtype=torch.float64, device=dev)
        S.update(logits=logits, pnp_in=pnp_in, pnp=pnp_saved, flat=flat, h1=h1, h2=h2, pred=pred, head_in=head_in if keep_head else None,
                 pix_sums=pix_sums, aux=aux, db=db)
        self.saved = S
        # the pose kernel needs the upstream loss gradients to emit dY9; forward calls it with unit weights and
        # backward re-runs it (cheap: B CTAs) with the actual ones.
        self._pose(S, gw=None)
        losses = torch.empty(5 - self.n_pix + len(self.loss_names), device=dev)  # the five per-pixel slots always
        vis2 = torch.empty(2, device=dev)
        n_pts = aux["gt_points"].shape[1]
        if self.pose_ex:
            C.gdrn_loss_finalize_ex2(pix_sums.data_ptr(), S["pose_part"].data_ptr(), S["vis_ps"].data_ptr(), losses.data_ptr(),
                                     vis2.data_ptr(), B, 4096, n_pts, self.pose_sw, _stream())
        else:
            C.gdrn_loss_finalize_ex(pix_sums.data_ptr(), S["pose_sums"].data_ptr(), S["vis_ps"].data_ptr(), losses.data_ptr(),
                                    vis2.data_ptr(), B, 4096, n_pts, _stream())
        vis = torch.cat([vis2, S["out_trans"][0], pred[0, 6:9], aux["gt_trans"][0], aux["gt_trans_ratio"][0]])
        if not self.live_head:
            losses = losses[5:]
        return dict(rot=S["out_rot"], trans=S["out_trans"], pred=pred, losses=losses, vis=vis, logits=logits)

    def _loss_masks(self, aux) -> tuple:
        """Device pointers of the GT masks that weight the xyz loss, are the mask loss's target and weight the region loss
        (gt_masks[XYZ_LOSS_MASK_GT], [MASK_LOSS_GT], [REGION_LOSS_MASK_GT], GDRN.py:339-395); the same mask gives the same pointer."""
        out = []
        for sel in self.mask_gt:
            m = aux.get("gt_mask_" + sel)
            if not isinstance(m, torch.Tensor):
                raise ValueError(f"the loss configuration selects gt_mask_{sel}, which was not given")
            out.append(m.data_ptr())
        return tuple(out)

    def _pose(self, S, gw):
        aux, B, dev = S["aux"], S["B"], self.dev
        if "out_rot" not in S:
            S["out_rot"] = torch.empty(B, 3, 3, device=dev)
            S["out_trans"] = torch.empty(B, 3, device=dev)
            if self.pose_ex:
                S["pose_part"] = torch.empty(B, 11, device=dev)  # [B][GDRN_POSE_SLOTS] per-crop partials
            else:
                S["pose_sums"] = torch.empty(4, dtype=torch.float64, device=dev)
            S["vis_ps"] = torch.empty(B, 2, device=dev)
            S["dy9"] = PT((B, 64), self.bplanes, device=dev)
        sym_idx = aux.get("sym_idx")
        if sym_idx is None and aux.get("sym_infos") is not None:  # direct engine.forward callers may pass the raw list
            sym_idx = aux["sym_idx"] = self.sym_table.indices(aux["sym_infos"])
        syms = self.sym_table.table if sym_idx is not None else None
        if gw is None:
            gw = torch.ones(len(self.loss_names) - self.n_pix, device=dev)
        n_pts = aux["gt_points"].shape[1]
        if self.pose_ex:
            C.gdrn_pose_loss_ex(S["pred"].data_ptr(), 16, aux["roi_cams"].data_ptr(), aux["roi_centers"].data_ptr(),
                                aux["roi_whs"].data_ptr(), aux["resize_ratios"].data_ptr(), aux["roi_extents"].data_ptr(),
                                aux["gt_points"].data_ptr(), aux["gt_ego_rot"].data_ptr(), aux["gt_trans"].data_ptr(),
                                aux["gt_trans_ratio"].data_ptr(), ops.ptr(syms), ops.ptr(sym_idx), gw.data_ptr(),
                                S["out_rot"].data_ptr(), S["out_trans"].data_ptr(), S["pose_part"].data_ptr(), S["vis_ps"].data_ptr(),
                                S["dy9"].hi_ptr, S["dy9"].lo_ptr, B, n_pts, self.pose_sw, _stream())
            return
        C.gdrn_pose_loss(S["pred"].data_ptr(), 16, aux["roi_cams"].data_ptr(), aux["roi_centers"].data_ptr(),
                         aux["roi_whs"].data_ptr(), aux["resize_ratios"].data_ptr(), aux["roi_extents"].data_ptr(),
                         aux["gt_points"].data_ptr(), aux["gt_ego_rot"].data_ptr(), aux["gt_trans"].data_ptr(),
                         aux["gt_trans_ratio"].data_ptr(), ops.ptr(syms), ops.ptr(sym_idx), gw.data_ptr(),
                         S["out_rot"].data_ptr(), S["out_trans"].data_ptr(), S["pose_sums"].data_ptr(), S["vis_ps"].data_ptr(),
                         S["dy9"].hi_ptr, S["dy9"].lo_ptr, B, n_pts, 1, 1e-4, _stream())

    # ------------------------------------------------------------------------------------------ backward
    # ---- weight gradients on a SIDE STREAM.  In backward the chain  BN-bwd(L) -> dgrad(L) -> BN-bwd(L-1) -> ...  alternates
    # tensor-bound GEMMs with HBM-bound BatchNorm passes, while wgrad(L) (+ its split-K unpack) only needs du(L) and feeds
    # nothing but the flat gradient buffer.  Issued on a second stream it runs concurrently with dgrad(L) and -- the point --
    # with the HBM-bound BN-bwd(L-1): tensor-bound and bandwidth-bound work overlap instead of serialising.  The streams join
    # at every gradient-bucket boundary (before the loss-scale removal / all-reduce of that bucket) and at the end of backward;
    # inside a CUDA graph the fork / join become graph edges.  wgrad_side_stream = False keeps everything on one stream.
    def _on_side(self, fn, keep=()):
        if not self.wgrad_side_stream:
            return fn()
        if self._side_stream is None:
            self._side_stream = torch.cuda.Stream()
        side = self._side_stream
        side.wait_stream(torch.cuda.current_stream())  # du(L) is ready
        with torch.cuda.stream(side):
            fn()
        self._side_keep.extend(keep)  # operands allocated on the main stream stay referenced until the join

    def _join_side(self, force: bool = False):
        if self._side_stream is not None and (self._side_keep or force):
            torch.cuda.current_stream().wait_stream(self._side_stream)
        self._side_keep.clear()

    def _wgrad_conv(self, du: PT, x_in: PT, conv, wname: str, ipad: Optional[int] = None):
        O, I, k = conv.out_channels, conv.in_channels, conv.kernel_size[0]

        def work():
            buf, ks, kss = ops.conv_wgrad(du, x_in, self.ws, O, k, k, conv.stride[0], conv.padding[0])
            ops.unpack_wgrad(buf, self.grads[wname], O, I, k, k, ipad or x_in.shape[-1], ks, kss, I * k * k, k * k, k, 1)

        self._on_side(work, keep=(du, x_in))

    def _dgrad_conv(self, du: PT, conv, wkey: str) -> PT:
        k, stride, pad = conv.kernel_size[0], conv.stride[0], conv.padding[0]
        if stride == 2:
            # four output-parity phases over the un-dilated dY (no zero-inserted tensor, 1/4 of its MACs)
            return ops.conv_dgrad_s2(du, self.wd[wkey], conv.in_channels, k, pad)
        return ops.conv_fwd(du, self.wd[wkey], conv.in_channels, k, k, 1, k - 1 - pad)

    def _bn_bwd(self, bkey: str, ga: PT, gb: Optional[PT], u: PT, want_gout=False, mask=None):
        """mask: the forward's ReLU bitmap (_bn_fwd), None for a BatchNorm without ReLU."""
        mod, st = self._bn_mods[bkey], self.bn[bkey]
        return ops.bn_bwd(ga, gb, None, u, st.mean, st.invstd, mod.weight, st.sums,
                          self.grads[bkey + ".weight"], self.grads[bkey + ".bias"], self.saved["train_bn"], want_gout=want_gout,
                          beta=mod.bias, sums_zeroed=True, relu_mask=mask,
                          det_ws=self._det_workspace() if self.deterministic else None)

    def _head_norm_bwd(self, bkey: str, g: PT, u: PT, L: dict) -> PT:
        """Backward of a head norm layer + ReLU (L: its saved forward entry) -> the gradient of its conv output."""
        gn = self._gn_mods.get(bkey)
        if gn is None:
            return self._bn_bwd(bkey, g, None, u, mask=L["m"])[0]
        return ops.head_gn_relu_bwd(g, u, L["m"], gn.weight, L["gs"], self.grads[bkey + ".weight"], self.grads[bkey + ".bias"])

    def backward(self, grad_losses: torch.Tensor):
        """grad_losses: upstream gradients of self.loss_names ([8], LOSS_NAMES, by default).  Fills self.grads (views of
        self.flat_grad)."""
        S, m, dev = self.saved, self.model, self.dev
        assert S is not None, "backward called without a do_loss forward"
        if not self.live_any:  # frozen head and Patch-PnP: no parameter receives a gradient
            return self._backward_done()
        B, aux, pn = S["B"], S["aux"], m.pnp_net
        bp = self.bplanes

        def h(t: PT) -> PT:  # a saved forward tensor as a backward operand
            return t.as_planes(bp)

        self.flat_grad.zero_()
        self.bwd_sums_all.zero_()
        gw = grad_losses.float().contiguous()
        if self.grad_scale != 1.0:
            gw = gw * self.grad_scale  # the whole backward is linear in the loss gradients
        self._pose(S, gw=gw[self.n_pix:].contiguous())
        dy9 = S["dy9"]
        tmp = torch.empty(1024, device=dev)
        wg = self.live_pnp  # a frozen Patch-PnP passes the gradient through but computes no weight or bias gradient

        # ---- FC stack (conv_pnp_net.py:152-156)
        if wg:
            buf, ks, kss = ops.gemm_wgrad(dy9, h(S["h2"]), self.ws)
            ops.unpack_wgrad(buf, self.grads["pnp_net.fc_r.weight"], 6, 256, 1, 1, 256, ks, kss, 256, 1, 0, 0)
            ops.unpack_wgrad(buf[6 * 256:], self.grads["pnp_net.fc_t.weight"], 3, 256, 1, 1, 256, ks, kss, 256, 1, 0, 0)
            C.gdrn_colsum(dy9.hi_ptr, dy9.lo_ptr, tmp.data_ptr(), B, 64, _stream())
            self.grads["pnp_net.fc_r.bias"].copy_(tmp[0:6])
            self.grads["pnp_net.fc_t.bias"].copy_(tmp[6:9])
        dh2 = ops.gemm_fwd(dy9, self.wd["fc_rt"], 256)
        dz2 = self._leaky_bwd(dh2, h(S["h2"]))
        if wg:
            buf, ks, kss = ops.gemm_wgrad(dz2, h(S["h1"]), self.ws)
            ops.unpack_wgrad(buf, self.grads["pnp_net.fc2.weight"], 256, 1024, 1, 1, 1024, ks, kss, 1024, 1, 0, 0)
            C.gdrn_colsum(dz2.hi_ptr, dz2.lo_ptr, self.grads["pnp_net.fc2.bias"].data_ptr(), B, 256, _stream())
        dh1 = ops.gemm_fwd(dz2, self.wd["fc2"], 1024)
        dz1 = self._leaky_bwd(dh1, h(S["h1"]))
        if wg:
            buf, ks, kss = ops.gemm_wgrad(dz1, h(S["flat"]), self.ws)
            ops.unpack_wgrad(buf, self.grads["pnp_net.fc1.weight"], 1024, 128, 8, 8, 128, ks, kss, 8192, 64, 8, 1)
            C.gdrn_colsum(dz1.hi_ptr, dz1.lo_ptr, self.grads["pnp_net.fc1.bias"].data_ptr(), B, 1024, _stream())
        g = ops.gemm_fwd(dz1, self.wd["fc1"], 8192).view(B, 8, 8, 128)

        # ---- Patch-PnP convs (conv_pnp_net.py:76-80)
        pf = pn.features
        for L in reversed(S["pnp"]):
            ci, gi = L["ci"], L["gi"]
            # a frozen Patch-PnP's GroupNorm parameter sums land in its slice of flat_grad, which is never read
            du = ops.gn_relu_bwd(g, h(L["y"]), h(L["u"]), pf[gi].weight, L["gstats"], self.grads[f"pnp_net.features.{gi}.weight"],
                                 self.grads[f"pnp_net.features.{gi}.bias"], G=pf[gi].num_groups)
            if wg:
                self._wgrad_conv(du, h(L["x_in"]), pf[ci], f"pnp_net.features.{ci}.weight")
            if ci == 0 and not self.live_head:  # a frozen head needs no Patch-PnP input gradient
                break
            g = self._dgrad_conv(du, pf[ci], f"pnp_net.features.{ci}")
        if wg:
            self._segment_done("pnp_net")
        if not self.live_head:
            return self._backward_done()
        d_pnp_in = g  # [B,64,64,pnp_ld]

        # ---- glue + per-pixel losses backward (one fused pass over the logits)
        dlog = PT((B * 4096, 128), bp, device=dev)
        m_xyz, m_mask, m_region = self._loss_masks(aux)
        hb = (S["logits"].data_ptr(), aux["gt_xyz"].data_ptr(), m_xyz, m_mask, m_region, aux["gt_region"].data_ptr(),
              S["pix_sums"].data_ptr(), gw.data_ptr(), d_pnp_in.hi_ptr, d_pnp_in.lo_ptr, aux["roi_extents"].data_ptr(), dlog.hi_ptr,
              dlog.lo_ptr, B, 4096, self.with_2d, self.mask_loss, self.mask_out)
        if S["db"] is not None:
            C.gdrn_head_bwd_db(*hb, self.num_regions, self.region_att, self.pnp_ld, S["db"][0].data_ptr(), S["db"][1].data_ptr(),
                               _stream())
        elif self.regions_ex2:
            C.gdrn_head_bwd_ex2(*hb, self.num_regions, self.region_att, self.pnp_ld, _stream())
        else:
            C.gdrn_head_bwd_ex(*hb, _stream())
        hf = m.rot_head_net.features
        head_in = h(S["head_in"])
        n_out = self.n_logits  # rows of the output conv
        if self.class_aware:
            g = self._class_head_bwd(dlog, head_in, aux["roi_classes"], B)
        elif self.out_k == 3:  # the 3x3 output conv over dlog viewed as [B, 64, 64, 128]: conv wgrad and dgrad, bias as below
            dlog4 = dlog.view(B, 64, 64, 128)
            self._wgrad_conv(dlog4, head_in, hf[23], "rot_head_net.features.23.weight")
            tmp128 = torch.empty(128, device=dev)
            C.gdrn_colsum(dlog.hi_ptr, dlog.lo_ptr, tmp128.data_ptr(), B * 4096, 128, _stream())
            self.grads["rot_head_net.features.23.bias"].copy_(tmp128[:n_out])
            g = self._dgrad_conv(dlog4, hf[23], "rot_head_net.features.23")
        else:
            def head_out_wgrad():
                buf, ks, kss = ops.gemm_wgrad(dlog, head_in.view(B * 4096, 256), self.ws)
                ops.unpack_wgrad(buf, self.grads["rot_head_net.features.23.weight"], n_out, 256, 1, 1, 256, ks, kss, 256, 1, 0, 0)

            self._on_side(head_out_wgrad, keep=(dlog,))
            tmp128 = torch.empty(128, device=dev)
            C.gdrn_colsum(dlog.hi_ptr, dlog.lo_ptr, tmp128.data_ptr(), B * 4096, 128, _stream())
            self.grads["rot_head_net.features.23.bias"].copy_(tmp128[:n_out])
            g = ops.gemm_fwd(dlog, self.wd["rot_head_net.features.23"], 256).view(B, 64, 64, 256)

        # ---- head convs (cdpn_rot_head_region.py:95-125)
        for L in reversed(S["head"]):
            ci, bi = L["ci"], L["bi"]
            du = self._head_norm_bwd(f"rot_head_net.features.{bi}", g, h(L["u"]), L)
            self._wgrad_conv(du, h(L["x_in"]), hf[ci], f"rot_head_net.features.{ci}.weight")
            g = self._dgrad_conv(du, hf[ci], f"rot_head_net.features.{ci}")
            if L["up"]:
                g = ops.upsample2x_bwd(g)
        D = S["deconv"]
        du = self._head_norm_bwd("rot_head_net.features.1", g, h(D["u"]), D)
        k, pad = self.deconv_k, self.deconv_pad

        def deconv_wgrad(du=du):
            # d wt[ci][co][r][s] = sum_q x[ci][q] * du[co][2q + (r, s) - pad]: the weight gradient of the stride-2 conv du -> x
            # with x in the role of dY; its [O = 512][I = 256][k][k] layout IS the ConvTranspose2d IOHW layout (no flip)
            buf, ks, kss = ops.conv_wgrad(h(D["z"]), du, self.ws, 512, k, k, 2, pad)
            ops.unpack_wgrad(buf, self.grads["rot_head_net.features.0.weight"], 512, 256, k, k, 256, ks, kss, 256 * k * k, k * k, k, 1)

        self._on_side(deconv_wgrad, keep=(du,))
        if not self.live_bb:  # frozen backbone: the head's gradients end the step
            self._segment_done("rot_head_net")
            return self._backward_done()
        g = ops.conv_fwd(du, self.wd["deconv"], 512, k, k, 2, pad)  # [B,8,8,512]
        self._segment_done("rot_head_net")

        # ---- backbone (torchvision BasicBlock backward)
        ga, gb = g, None
        for Lb in reversed(S["blocks"]):
            p, blk = Lb["p"], Lb["blk"]
            du2, gout = self._bn_bwd(p + ".bn2", ga, gb, h(Lb["u2"]), want_gout=True, mask=Lb["m2"])
            self._wgrad_conv(du2, h(Lb["a1"]), blk.conv2, p + ".conv2.weight")
            da1 = self._dgrad_conv(du2, blk.conv2, p + ".conv2")
            du1, _ = self._bn_bwd(p + ".bn1", da1, None, h(Lb["u1"]), mask=Lb["m1"])
            self._wgrad_conv(du1, h(Lb["x_in"]), blk.conv1, p + ".conv1.weight")
            dx_main = self._dgrad_conv(du1, blk.conv1, p + ".conv1")
            if blk.downsample is not None:
                dud, _ = self._bn_bwd(p + ".downsample.1", gout, None, h(Lb["ud"]))
                self._wgrad_conv(dud, h(Lb["x_in"]), blk.downsample[0], p + ".downsample.0.weight")
                dx_ds = self._dgrad_conv(dud, blk.downsample[0], p + ".downsample.0")
                ga, gb = dx_main, dx_ds
            else:
                ga, gb = dx_main, gout
            if p.endswith(".0") and not p.startswith("backbone.layer1"):
                self._segment_done(p[:-2])  # all gradients of backbone.layerN are final
        g_pool = ops.add2(ga, gb)
        St = S["stem"]
        g_a0 = ops.maxpool_bwd(St["pool_arg"], g_pool)
        du0, _ = self._bn_bwd("backbone.bn1", g_a0, None, h(St["u0"]), mask=St["m0"])
        def stem_wgrad():  # on the side stream like every conv wgrad: the split-K workspace is owned by that stream by now
            buf, ks, kss = ops.gemm_wgrad(du0.view(B * 128 * 128, 64), h(St["a_col"]), self.ws)
            # ws rows [64][192] with k = (r*7+s)*3 + c  ->  OIHW [64][3][7][7]
            ops.unpack_wgrad(buf, self.grads["backbone.conv1.weight"], 64, 3, 7, 7, 3, ks, kss, 147, 49, 7, 1, krow=192)

        self._on_side(stem_wgrad, keep=(du0,))
        self._segment_done("backbone.stem")  # layer1 + bn1 + conv1 (joins the wgrad side stream)
        self.saved = None
        return self.grads

    def _backward_done(self):
        """End of a backward that stops above the backbone: join the side stream (a no-op after _segment_done) and free S."""
        self._join_side()
        self.saved = None
        return self.grads

    def _class_head_bwd(self, dlog: PT, head_in: PT, classes: torch.Tensor, B: int) -> PT:
        """Backward of the class-aware output conv: the grouped dgrad on the main stream; on the side stream the per-crop weight
        partials (the wgrad GEMM split at crop boundaries, ksplit = B) and per-crop bias partials, reduced in crop order into the
        reference layout (rows of classes absent from the batch get exactly 0).  A 3x3 output conv runs the conv wgrad, split the
        same way (4096 pixels = 64 k-blocks per crop), and the grouped 3x3 dgrad; its partials are tap-major ([row][tap][ci]), so
        they are reduced into a scratch table that is then unpacked into the OIHW gradient."""
        k, key = self.out_k, "rot_head_net.features.23"

        def work():
            if k == 1:
                buf, ks, kss = ops.gemm_wgrad(dlog, head_in.view(B * 4096, 256), self.ws, ksplit=B)
            else:
                buf, ks, kss = ops.conv_wgrad(dlog.view(B, 64, 64, 128), head_in, self.ws, self.n_logits, k, k, 1, k // 2, ksplit=B)
            assert ks == B, (ks, B)  # 4096 rows = 64 k-blocks per split: split b is crop b
            bias_part = torch.empty(B, 128, device=self.dev)
            C.gdrn_crop_colsum(dlog.hi_ptr, dlog.lo_ptr, bias_part.data_ptr(), B, 4096, 128, _stream())
            K = k * k * 256
            gw = self.grads[key + ".weight"] if k == 1 else torch.empty(self.cls_rows, K, device=self.dev)
            C.gdrn_class_wgrad_reduce(buf.data_ptr(), kss, K, bias_part.data_ptr(), 128, classes.data_ptr(), B,
                                      self.cls_slot.data_ptr(), self.num_classes, self.cls_rows, self.n_logits, K,
                                      gw.data_ptr(), self.grads[key + ".bias"].data_ptr(), _stream())
            if k != 1:
                ops.unpack_wgrad(gw, self.grads[key + ".weight"], self.cls_rows, 256, k, k, 256, 1, 0, K, k * k, k, 1)

        self._on_side(work, keep=(dlog, classes))
        if k == 1:
            return ops.gemm_fwd_grouped(dlog, self.wd[key], 256, classes, 4096).view(B, 64, 64, 256)
        return ops.conv_fwd_grouped(dlog.view(B, 64, 64, 128), self.wd[key], 256, 256, classes, 4096, k=k)

    def materialize_aliased_grads(self):
        """A p.grad that still aliases flat_grad (adopted by autograd in an earlier step and not reset by zero_grad) would be
        overwritten by the next backward: give such gradients their own storage first (gradient accumulation stays exact)."""
        lo = self.flat_grad.data_ptr()
        hi = lo + self.flat_grad.numel() * self.flat_grad.element_size()
        for _, p in self.named_params:
            g = p.grad
            if g is not None and lo <= g.data_ptr() < hi:
                p.grad = g.clone()

    def _segment_done(self, stage: str):
        self._join_side()
        self._segment_done_joined(stage)

    def _segment_done_joined(self, stage: str):
        """All gradients of a sub-network are final: remove the loss scale from its slice of the flat buffer, then hand
        it to the data-parallel hook (bucketed all-reduce on a side stream)."""
        if self.grad_scale != 1.0:
            names = ("backbone.conv1", "backbone.bn1", "backbone.layer1") if stage == "backbone.stem" else (stage,)
            lo = min(self._seg[n][0] for n in names)
            hi = max(self._seg[n][1] for n in names)
            C.gdrn_scale_f32(self.flat_grad.data_ptr() + 4 * lo, hi - lo, 1.0 / self.grad_scale, _stream())
        if self.grad_hook:
            self.grad_hook(self, stage)

    def _leaky_bwd(self, g: PT, y: PT) -> PT:
        out = ops.like(g)
        C.gdrn_leaky_bwd(g.hi_ptr, g.lo_ptr, y.hi_ptr, out.hi_ptr, out.lo_ptr, g.numel(), _stream())
        return out


class _PlaneRows:
    """Rows [r0, ...) of a PT as a pack destination (the per-class blocks of the class-aware dgrad operand)."""

    def __init__(self, pt: PT, r0: int):
        self.pt = pt
        self.hi_ptr = pt.buf[0, r0].data_ptr()
        self.lo_ptr = pt.buf[1, r0].data_ptr() if pt.planes == 2 else None


def _capture_mode():
    # with a process group alive, NCCL's watchdog thread polls CUDA events while we capture: "thread_local" keeps its
    # calls legal (the collectives themselves are captured into the graph on their side stream)
    import torch.distributed as dist

    return "thread_local" if (dist.is_available() and dist.is_initialized()) else "global"


def _capture(engine: "Engine", steps, warmup: int, restore_bn: bool = False, pool=None):
    """Runs `warmup` rounds of the callables `steps` on a side stream (this also sizes the split-K workspace and uploads the
    pack job tables), then captures each step into its own CUDA graph, all in `pool` if one is given.  Returns
    [(graph, what the step returned)].  restore_bn: the warm-up leaves the BatchNorm running statistics and counters as
    they were.  The DropBlock step counter is always restored: a replayed run sees the same mask sequence as an eager one."""
    bn_bufs = [t for m in engine._bn_mods.values() for t in m.buffers()] if restore_bn else []
    if engine.drop_prob > 0:
        bn_bufs.append(engine.model.pnp_net.dropblock_counter(engine.dev))
    snap = [t.clone() for t in bn_bufs]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(warmup):
            for step in steps:
                step()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    for t, s in zip(bn_bufs, snap):
        t.copy_(s)
    out = []
    for step in steps:
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, pool=pool, capture_error_mode=_capture_mode()):
            out.append((graph, step()))
    return out


def _clone_inputs(x: torch.Tensor, aux: dict):
    """Static input buffers of a captured graph: clones of x and of the tensors in aux (other entries are shared)."""
    return x.clone(), {k: (v.clone() if isinstance(v, torch.Tensor) else v) for k, v in aux.items()}


def _copy_inputs(static_x: torch.Tensor, static_aux: dict, x: Optional[torch.Tensor], aux: dict):
    """Copies new inputs into the static buffers (device-side, ordered before the next replay); x = None keeps the old x."""
    if x is not None:
        static_x.copy_(x, non_blocking=True)
    for k, v in aux.items():
        if isinstance(v, torch.Tensor):
            static_aux[k].copy_(v, non_blocking=True)


def _finish_hook(engine: "Engine"):
    hook = engine.grad_hook
    if hook is not None and hasattr(hook, "finish"):
        hook.finish()


class GraphedTrainStep:
    """One CUDA graph for the whole train step (forward + losses + backward + bucketed gradient all-reduce): ~370 kernel
    launches AND the NCCL collectives of `engine.grad_hook` (issued on its side stream at bucket boundaries, i.e. overlapped
    with the rest of backward) are replayed with a single cudaGraphLaunch, removing the per-launch host cost of the
    Python/ctypes orchestration at every world size.  Inputs live in static buffers; call with new tensors to copy
    them in (device-side copies)."""

    def __init__(self, engine: "Engine", x: torch.Tensor, aux: dict, train_bn: bool = True, warmup: int = 2, after_backward=None):
        self.engine = engine
        self.x, self.aux = _clone_inputs(x, aux)
        if self.aux.get("sym_infos") is not None:  # symmetric PM: only the (first row, count) pairs are a per-step input
            self.aux["sym_idx"] = engine.sym_table.indices(self.aux["sym_infos"])
        self.aux.pop("sym_infos", None)
        self.gw = torch.ones(len(engine.loss_names), device=x.device)

        def one_step():
            res = engine.forward(self.x, self.aux, train_bn=train_bn, do_loss=True)
            engine.backward(self.gw)
            _finish_hook(engine)
            if after_backward is not None:
                after_backward()
            return res

        [(self.graph, res)] = _capture(engine, [one_step], warmup, restore_bn=True)
        self.losses, self.vis, self.rot, self.trans = res["losses"], res["vis"], res["rot"], res["trans"]
        self.logits = res["logits"]

    def __call__(self, x: Optional[torch.Tensor] = None, aux: Optional[dict] = None, grad_losses: Optional[torch.Tensor] = None):
        if aux is not None and aux.get("sym_infos") is not None:
            self.aux["sym_idx"].copy_(self.engine.sym_table.indices(aux["sym_infos"]), non_blocking=True)
        _copy_inputs(self.x, self.aux, x, aux or {})
        if grad_losses is not None:
            self.gw.copy_(grad_losses)
        self.graph.replay()
        return self.losses


class GraphedFwdBwd:
    """Forward and backward captured as TWO CUDA graphs sharing one memory pool, for the public module API
    (`GDRN.forward(..., do_loss=True)` then `.backward()`): the autograd Function replays them around static buffers.
    The data-parallel all-reduces of `engine.grad_hook` are captured INSIDE the backward graph (side stream, overlapped)."""

    def __init__(self, engine: "Engine", x: torch.Tensor, aux: dict, train_bn: bool):
        self.engine, self.train_bn = engine, train_bn
        self.x, self.aux = _clone_inputs(x, aux)
        self.gw = torch.ones(len(engine.loss_names), device=x.device)
        self.key = self.signature(x, aux, train_bn)

        def bwd():
            engine.backward(self.gw)
            _finish_hook(engine)

        with torch.no_grad():
            (self.g_fwd, res), (self.g_bwd, _) = _capture(
                engine, [lambda: engine.forward(self.x, self.aux, train_bn=train_bn, do_loss=True), bwd], warmup=2,
                restore_bn=True, pool=torch.cuda.graph_pool_handle())
        self.losses, self.vis = res["losses"], res["vis"]

    @staticmethod
    def signature(x, aux, train_bn):
        return (tuple(x.shape), train_bn, tuple(sorted((k, tuple(v.shape)) for k, v in aux.items() if isinstance(v, torch.Tensor))))

    def forward(self, x, aux):
        _copy_inputs(self.x, self.aux, x, aux)
        self.g_fwd.replay()
        return self.losses.clone(), self.vis.clone()

    def backward(self, g_losses):
        self.gw.copy_(g_losses)
        self.g_bwd.replay()  # includes the bucketed all-reduces and the join of their side stream
        return self.engine.grads


class _GDRNFunction(torch.autograd.Function):
    """Autograd boundary: forward + losses and the hand-written backward are both ours; autograd only routes the
    8 loss gradients in and the 148 parameter gradients out (so optimizers / DDP / GradScaler keep working)."""

    @staticmethod
    def forward(ctx, engine: Engine, x, aux, train_bn, *params):
        ctx.engine = engine
        ctx.graphed = None
        if engine.use_cuda_graphs:
            g = engine._graphed
            if g is None or g.key != GraphedFwdBwd.signature(x, aux, train_bn):
                g = engine._graphed = GraphedFwdBwd(engine, x, aux, train_bn)
            losses, vis = g.forward(x, aux)
            ctx.graphed = g
        else:
            res = engine.forward(x, aux, train_bn=train_bn, do_loss=True)
            losses, vis = res["losses"], res["vis"]
        ctx.mark_non_differentiable(vis)
        return losses, vis

    @staticmethod
    def backward(ctx, g_losses, _g_vis):
        engine = ctx.engine
        engine.materialize_aliased_grads()
        if ctx.graphed is not None:
            ctx.graphed.backward(g_losses)
        else:
            engine.backward(g_losses)
        _finish_hook(engine)  # the gradients handed to autograd are the all-reduced ones (stream-ordered wait, no host sync)
        # FRESH views of the flat gradient buffer: autograd's AccumulateGrad adopts a uniquely-referenced contiguous gradient
        # without copying, so after `zero_grad(set_to_none=True)` p.grad aliases Engine.flat_grad and the 148 per-parameter
        # clone kernels (0.4 ms per step) disappear.  materialize_aliased_grads() protects gradient accumulation.  Only the
        # live parameters are inputs of the function (Engine.live_params): frozen and unreachable ones keep .grad None.
        flat = engine.flat_grad
        outs = [flat[off:off + p.numel()].view_as(p) for p, off in engine.live_params]
        return (None, None, None, None) + tuple(outs)
