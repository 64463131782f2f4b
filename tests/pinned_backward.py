"""Pinned float64 backward: the parameter gradients of a whole engine step against a float64 replay of the oracle that follows
the engine's own non-smooth decisions.

The engine's forward differs from a float64 forward by ~1e-4 (DESIGN §8, tools/noise_floor.py).  That flips a few ReLU, max-pool
and L1-sign decisions, and every flip moves the gradients downstream of it, which is why a plain gradient comparison needs 6e-2
per tensor.  Given the decisions, the backward is linear.  So this module

  * `capture(engine)`: after a `do_loss` forward and BEFORE backward (which clears `engine.saved`), takes the decisions out of
    `engine.saved` in the oracle's call order: the 40 BatchNorm + ReLU bitmaps, the max-pool window codes, the 3 GroupNorm + ReLU
    and 2 LeakyReLU masks (`y > 0` of the stored output, as the backward kernels read them) and the decisions of the loss terms
    (the signs of the 7 L1 residuals of the shipped configuration), recomputed in fp32 from the engine's own outputs exactly as
    the loss kernels form them;
  * `pinned(pins, modules)`: swaps the oracle modules' `F` for a shim whose relu / max_pool2d / leaky_relu / linear / l1_loss /
    smooth_l1_loss / closest_rot_batch consume the next pin (a pinned ReLU is x * mask, a pinned max-pool gathers the coded
    window element, a pinned linear layer returns the engine's value, a pinned L1 is sum s (a - b), a pinned Smooth-L1 takes the pinned branch, a pinned symmetric search returns
    the pinned candidate); everything else is torch.nn.functional.  The shim counts, per site, the elements the float64
    forward would have decided differently and the rel-L2 of its output against the engine's stored activation (a per-layer forward parity);
  * `row_errors` / `compare_grads`: per output channel e_r = |g_r - ref_r| / max(|ref_r|, floor |ref| / sqrt(rows)), floor
    1e-3 for the rows of a weight.  An entry of a 1-D tensor (BatchNorm / GroupNorm gamma and beta, a bias) is one sum over
    B H W terms that largely cancel: its absolute error follows the size of the terms, not of the sum, and on the B = 64
    step the small entries' errors are ~1e-3 of the tensor's RMS entry in "mixed" (3e-4 in "fp32x3"), so those entries are
    measured against a floor of 0.1 of the RMS entry and a bound of their own;
  * `running_stat_errors`: every BatchNorm running mean / variance / counter after the step against the replay's.

The layouts decoded here (csrc/elementwise.cu): a ReLU bitmap holds flat NHWC element e as bit e & 7 of byte e >> 3, set when
the fp32 pre-activation (+ residual) is > 0 (bn_fwd); a max-pool code is dy * 3 + dx of the 3x3 / stride 2 / pad 1 window, the
first strict maximum in row-major order (maxpool_fwd_kernel).  The GroupNorm head writes the same ReLU bitmaps as the BatchNorm one.

Each switch family replays through the oracle module that restates it, and `capture` emits the pins in that module's call order:
  * BCE / CE mask losses (oracle/mask_oracle.py) decide nothing: no `loss_mask` pin, the xyz pins read the logits at MO;
  * the PNP_NET pose switches (oracle/pose_loss_oracle.py, which first runs the shipped pose terms through mask_oracle and drops
    them: those get `unused.*` pins): a sign per element of every L1 term, a Smooth-L1 pin (branch |d| < beta and sign) per
    element of Smooth-L1 point matching; MSE, L2 and the rotation losses are smooth.  Symmetric point matching pins the
    candidate the pose kernel chose, restated from its fp32 argmin (`sym_choice`);
  * the Patch-PnP rotation and translation outputs (fc_r, fc_t) enter the pose decode and the losses at the engine's fp32
    values, with the float64 gradient.  The allo-to-ego decode normalises T / (|T| + 1e-4): for a crop whose predicted depth is
    within the forward's ~1e-5 error of zero, its gradient depends on that error at first order (one crop of an untrained
    B = 64 batch moved the whole translation gradient by 30 %), like a decision would;
  * a frozen backbone or head keeps no decisions: the oracle runs it without gradient and the shim lets such calls (and
    DropBlock's max-pool over its seed mask) through as `inert`.
Switches without a pin route raise NotImplementedError: Smooth-L1 below beta = 1e-5 (the oracle's plain |a - b| bypasses F) and
symmetric point matching with the shipped pose losses.  A new pin kind is one more shim method and one more constructor below.
"""
from __future__ import annotations

import contextlib
import math
import re
from typing import Callable, Dict, List, Optional

import torch
import torch.nn.functional as TF

Tensor = torch.Tensor


# --------------------------------------------------------------------------------------------------------------- decoders
def unpack_bitmap(bits: Tensor, nhwc) -> Tensor:
    """Engine ReLU bitmap (flat NHWC element e = bit e & 7 of byte e >> 3) -> bool NCHW."""
    n = math.prod(nhwc)
    assert bits.dtype == torch.uint8 and bits.numel() * 8 == n, (bits.dtype, bits.numel(), nhwc)
    shifts = torch.arange(8, device=bits.device, dtype=torch.uint8)
    flat = ((bits.reshape(-1, 1) >> shifts) & 1).bool().reshape(-1)
    return flat.view(*nhwc).permute(0, 3, 1, 2)


def pool_codes(arg: Tensor) -> Tensor:
    """Engine max-pool window codes uint8 NHWC [B, Ho, Wo, C] -> int64 NCHW."""
    assert arg.dtype == torch.uint8 and arg.dim() == 4
    return arg.permute(0, 3, 1, 2).long()


def pool_windows(x: Tensor):
    """The 3x3 / stride 2 / pad 1 windows of x [B, C, H, W] as [B, C, 9, Ho * Wo] (row-major window order dy * 3 + dx) and
    whether each window element lies inside the image."""
    B, C, H, W = x.shape
    cols = TF.unfold(x, 3, padding=1, stride=2).view(B, C, 9, -1)
    inside = TF.unfold(torch.ones(1, 1, H, W, dtype=x.dtype, device=x.device), 3, padding=1, stride=2).view(1, 1, 9, -1) > 0
    return cols, inside


def pool_gather(x: Tensor, codes: Tensor) -> Tensor:
    """max_pool2d(x, 3, 2, 1) with the maximum taken where `codes` say (differentiable in x)."""
    B, C, H, W = x.shape
    Ho, Wo = codes.shape[2], codes.shape[3]
    cols, inside = pool_windows(x)
    idx = codes.reshape(B, C, 1, Ho * Wo)
    assert int(codes.min()) >= 0 and int(codes.max()) <= 8, "max-pool code outside the 3x3 window"
    ok = inside.expand(B, C, 9, Ho * Wo).gather(2, idx)
    assert bool(ok.all()), f"{int((~ok).sum())} max-pool codes point into the padding"
    return cols.gather(2, idx).view(B, C, Ho, Wo)


def first_max_codes(x: Tensor) -> Tensor:
    """The window codes x itself gives: the first maximum of each window, padding never chosen."""
    cols, inside = pool_windows(x)
    cols = cols.masked_fill(~inside, float("-inf"))
    B, C = x.shape[:2]
    return cols.argmax(2).view(B, C, (x.shape[2] + 1) // 2, (x.shape[3] + 1) // 2)  # argmax: the first maximal index


def _nchw(t: Tensor) -> Tensor:
    return t.permute(0, 3, 1, 2) if t.dim() == 4 else t


# --------------------------------------------------------------------------------------------------------------- pins
class Pin:
    """One decision site.  kind: the torch.nn.functional call it answers; shape: that call's first argument's shape;
    decide(device): the decision tensor in the oracle's layout; act: None or a callable giving the engine's stored output at
    this site (NCHW / [B, N] fp32) for the forward parity."""

    __slots__ = ("kind", "name", "shape", "decide", "act")

    def __init__(self, kind: str, name: str, shape, decide: Callable, act: Optional[Callable] = None):
        self.kind, self.name, self.shape, self.decide, self.act = kind, name, tuple(shape), decide, act

    @staticmethod
    def relu_bitmap(name, bits: Tensor, nhwc, act=None) -> "Pin":
        bits = bits.detach().clone()
        B, H, W, C = nhwc
        return Pin("relu", name, (B, C, H, W), lambda dev: unpack_bitmap(bits.to(dev), nhwc), act)

    @staticmethod
    def positive(kind: str, name, y: Tensor, act=None) -> "Pin":
        """mask = y > 0 of a stored output y (NHWC or [B, N]): the GroupNorm + ReLU and LeakyReLU backward kernels' decision."""
        m = _nchw(y > 0).clone()
        return Pin(kind, name, m.shape, lambda dev: m.to(dev), act)

    @staticmethod
    def pool(name, arg: Tensor, in_nhwc, act=None) -> "Pin":
        arg = arg.detach().clone()
        B, H, W, C = in_nhwc
        return Pin("max_pool2d", name, (B, C, H, W), lambda dev: pool_codes(arg.to(dev)), act)

    @staticmethod
    def sign(name, s: Tensor) -> "Pin":
        s = s.detach().double().clone()
        return Pin("l1_loss", name, s.shape, lambda dev: s.to(dev))

    @staticmethod
    def smooth_l1(name, e: Tensor, beta: float) -> "Pin":
        """Smooth-L1 of residuals e: q = 0 where |e| < beta (the quadratic branch), else sign(e)."""
        q = torch.where(e.abs() < beta, torch.zeros_like(e), torch.sign(e)).detach().double().clone()
        return Pin("smooth_l1_loss", name, q.shape, lambda dev: q.to(dev))

    @staticmethod
    def linear(name, in_shape, value: Optional[Tensor] = None) -> "Pin":
        """A Patch-PnP linear layer: with `value` (the engine's fp32 output) the replay continues from that value, its gradient
        still the float64 one; without, nothing is pinned."""
        v = None if value is None else value.detach().clone()
        return Pin("linear", name, in_shape, lambda dev: None if v is None else v.to(dev), None if v is None else (lambda: v))

    @staticmethod
    def sym(name, idx: Tensor) -> "Pin":
        """Closest symmetric ground truth: per crop the chosen candidate k of its symmetry set, -1 for the unmodified R_gt."""
        idx = idx.detach().long().cpu().clone()
        return Pin("closest_rot_batch", name, (idx.numel(), 3, 3), lambda dev: idx)


def _pt_act(pt) -> Callable:
    return lambda: _nchw(pt.float())


def capture(engine) -> List[Pin]:
    """The decisions of the engine's last do_loss forward, in the oracle's call order.  Call before engine.backward.  The
    activations of the parity check stay referenced (no copy) until the pins are dropped."""
    S = engine.saved
    assert S is not None, "capture() needs a do_loss forward whose backward has not run yet"
    if S["aux"].get("sym_idx") is not None and not engine.pose_ex:
        raise NotImplementedError("symmetric point matching is pinned with the PNP_NET pose switches only (pose_loss_oracle)")
    p = engine.model.cfg.MODEL.CDPN.PNP_NET
    if engine.pose_ex and p.PM_LW > 0 and p.PM_LOSS_TYPE.lower() == "smooth_l1" and p.PM_SMOOTH_L1_BETA < 1e-5:
        raise NotImplementedError("Smooth-L1 below beta = 1e-5 is a plain |a - b| in the oracle, which no pin can answer")

    def bitmap(name, mask, pt):
        return Pin.relu_bitmap(name, mask, pt.shape, _pt_act(pt))

    pins = []
    if engine.live_bb:  # a frozen backbone (or one below a frozen head) keeps no decisions: the oracle runs it without gradient
        St = S["stem"]
        pins += [bitmap("backbone.bn1", St["m0"], St["a0"]),
                 Pin.pool("backbone.maxpool", St["pool_arg"], St["a0"].shape, _pt_act(S["blocks"][0]["x_in"]))]
        for L in S["blocks"]:
            pins += [bitmap(L["p"] + ".bn1", L["m1"], L["a1"]), bitmap(L["p"] + ".bn2", L["m2"], L["out"])]
    if engine.live_head:  # BatchNorm + ReLU or GroupNorm + ReLU: the same bitmap layout
        pins.append(bitmap("rot_head_net.features.1", S["deconv"]["m"], S["deconv"]["y"]))
        pins += [bitmap(f"rot_head_net.features.{L['bi']}", L["m"], L["y"]) for L in S["head"]]
    pins += [Pin.positive("relu", f"pnp_net.features.{L['gi']}", L["y"].hi, _pt_act(L["y"])) for L in S["pnp"]]
    B, pn = S["B"], engine.model.pnp_net
    for k, h in (("fc1", "h1"), ("fc2", "h2")):
        pins += [Pin.linear(f"pnp_net.{k}", (B, getattr(pn, k).in_features)),
                 Pin.positive("leaky_relu", f"pnp_net.{k}", S[h].hi, _pt_act(S[h]))]
    nr = pn.fc_r.out_features
    pins += [Pin.linear("pnp_net.fc_r", (B, pn.fc_r.in_features), S["pred"][:, :nr]),
             Pin.linear("pnp_net.fc_t", (B, pn.fc_t.in_features), S["pred"][:, nr:nr + 3])]
    return pins + loss_sign_pins(engine, S)


def _rot_points(M: Tensor, P: Tensor) -> Tensor:
    """[B, n, 3]: row i of M [B, 3, 3] dotted with each point of P [B, n, 3], summed left to right in fp32."""
    return M[:, None, :, 0] * P[:, :, None, 0] + M[:, None, :, 1] * P[:, :, None, 1] + M[:, None, :, 2] * P[:, :, None, 2]


def loss_sign_pins(engine, S) -> List[Pin]:
    """The decisions of the loss terms, formed in fp32 from the engine's outputs like csrc/losses.cu forms them.  Per-pixel
    (live head): xyz masked_diff(logit, gt, m) = fl(logit m) - fl(gt m) at logit column MO; with an L1 mask head, logit - target.
    Shipped pose losses: point matching fl(w est) - fl(w tgt) with est = R p summed left to right, R the decoded ego rotation;
    centroid and z pred - ratio.  sign(0) = 0.  With the PNP_NET pose switches the shipped terms are pinned as `unused.*` (the
    oracle computes and drops them), then `pose_pins`."""
    B, aux, mo = S["B"], S["aux"], engine.mask_out
    pins = []
    if engine.live_head:
        lg = S["logits"].view(B, 64, 64, 72)
        m_xyz, m_mask = aux["gt_mask_" + engine.mask_gt[0]], aux["gt_mask_" + engine.mask_gt[1]]
        for j, c in enumerate("xyz"):
            e = lg[..., mo + j] * m_xyz - aux["gt_xyz"][:, j] * m_xyz
            pins.append(Pin.sign(f"loss_coor_{c}", torch.sign(e)[:, None]))
        if engine.mask_loss == 0:  # BCE and CE are smooth
            pins.append(Pin.sign("loss_mask", torch.sign(lg[..., 0] - m_mask)))
    R, Rg, P = S["out_rot"], aux["gt_ego_rot"], aux["gt_points"]
    w = (1.0 / aux["roi_extents"].max(1).values).view(B, 1, 1)
    pre = "unused." if engine.pose_ex else ""
    pins.append(Pin.sign(pre + "loss_PM_R", torch.sign(_rot_points(R, P) * w - _rot_points(Rg, P) * w)))
    nr = engine.model.pnp_net.fc_r.out_features
    t, ratio = S["pred"][:, nr:nr + 3], aux["gt_trans_ratio"]
    pins.append(Pin.sign(pre + "loss_centroid", torch.sign(t[:, :2] - ratio[:, :2])))
    pins.append(Pin.sign(pre + "loss_z", torch.sign(t[:, 2] - ratio[:, 2])))
    return (pins + pose_pins(engine, S)) if engine.pose_ex else pins


def _term_pins(name: str, kind: str, e: Tensor, beta: float) -> List[Pin]:
    kind = kind.lower()
    if kind == "l1":
        return [Pin.sign(name, torch.sign(e))]
    if kind == "smooth_l1":
        return [Pin.smooth_l1(name, e, beta)]
    assert kind in ("mse", "l2"), kind  # smooth: nothing to decide
    return []


def pose_pins(engine, S) -> List[Pin]:
    """The non-smooth decisions of the PNP_NET pose switches in pose_loss_oracle.pose_losses' order, with the residuals of
    pose_loss_ex_tail (csrc/losses.cu): point matching masked_diff(a, b, w) = fl(a w) - fl(b w) (w exactly 1 without
    PM_NORM_BY_EXTENT) of est + t | est + t_gt | R_gt p + t against R_gt p + t_gt, the components a disentangled term keeps at the
    ground truth exactly 0; without points t - t_gt; centroid and z pred - ratio; translation t - t_gt; bind R^T t - R_gt^T t_gt
    (the original R_gt).  With PM_LOSS_SYM the candidate of `sym_choice` comes first and is the point-matching target."""
    p = engine.model.cfg.MODEL.CDPN.PNP_NET
    B, aux = S["B"], S["aux"]
    R, T = S["out_rot"], S["out_trans"]
    Rg0, Tg, P = aux["gt_ego_rot"], aux["gt_trans"], aux["gt_points"]
    beta = float(p.PM_SMOOTH_L1_BETA)
    pins = []
    if p.PM_LW > 0:
        Rg = Rg0
        if aux.get("sym_idx") is not None:
            idx = sym_choice(R, Rg0, engine.sym_table.table, aux["sym_idx"])
            pins.append(Pin.sym("loss_PM_sym", idx))
            Rg = sym_target(Rg0, engine.sym_table.table, aux["sym_idx"], idx)
        w = (1.0 / aux["roi_extents"].max(1).values).view(B, 1, 1) if p.PM_NORM_BY_EXTENT else 1.0

        def md(a, b):
            return a * w - b * w

        est, tgt = _rot_points(R, P), _rot_points(Rg, P)
        Tp, Tq = T[:, None], Tg[:, None]
        dis_z = p.PM_DISENTANGLE_Z
        dis_t = p.PM_DISENTANGLE_T or dis_z
        use_pts = p.PM_T_USE_POINTS if dis_t else True
        if p.PM_R_ONLY:
            terms = [("loss_PM_R", md(est, tgt))]
        elif dis_z and use_pts:
            e1 = md(tgt + Tp, tgt + Tq)
            z = torch.zeros_like(e1[..., :1])
            terms = [("loss_PM_R", md(est + Tq, tgt + Tq)), ("loss_PM_xy", torch.cat([e1[..., :2], z], -1)),
                     ("loss_PM_z", torch.cat([z, z, e1[..., 2:]], -1))]
        elif dis_z:
            terms = [("loss_PM_R", md(est, tgt)), ("loss_PM_xy_noP", T[:, :2] - Tg[:, :2]), ("loss_PM_z_noP", T[:, 2] - Tg[:, 2])]
        elif dis_t and use_pts:
            terms = [("loss_PM_R", md(est + Tq, tgt + Tq)), ("loss_PM_T", md(tgt + Tp, tgt + Tq))]
        elif dis_t:
            terms = [("loss_PM_R", md(est, tgt)), ("loss_PM_T_noP", T - Tg)]
        else:
            terms = [("loss_PM_RT", md(est + Tp, tgt + Tq))]
        for name, e in terms:
            pins += _term_pins(name, p.PM_LOSS_TYPE, e, beta)
    nr = engine.model.pnp_net.fc_r.out_features
    t, ratio = S["pred"][:, nr:nr + 3], aux["gt_trans_ratio"]
    if p.CENTROID_LW > 0:
        pins += _term_pins("loss_centroid", p.CENTROID_LOSS_TYPE, t[:, :2] - ratio[:, :2], 0.0)
    if p.Z_LW > 0:
        pins += _term_pins("loss_z", p.Z_LOSS_TYPE, t[:, 2] - ratio[:, 2], 0.0)
    if p.TRANS_LW > 0:
        e = T - Tg
        if p.TRANS_LOSS_DISENTANGLE:
            pins += _term_pins("loss_trans_xy", p.TRANS_LOSS_TYPE, e[:, :2], 0.0)
            pins += _term_pins("loss_trans_z", p.TRANS_LOSS_TYPE, e[:, 2], 0.0)
        else:
            pins += _term_pins("loss_trans_LPnP", p.TRANS_LOSS_TYPE, e, 0.0)
    if p.get("BIND_LW", 0.0) > 0 and p.BIND_LOSS_TYPE == "L1":
        pb = R[:, 0] * T[:, 0:1] + R[:, 1] * T[:, 1:2] + R[:, 2] * T[:, 2:3]  # (R^T t)_j = R0j t0 + R1j t1 + R2j t2
        gb = Rg0[:, 0] * Tg[:, 0:1] + Rg0[:, 1] * Tg[:, 1:2] + Rg0[:, 2] * Tg[:, 2:3]
        pins += _term_pins("loss_bind", "L1", pb - gb, 0.0)
    return pins


def sym_choice(R: Tensor, Rg: Tensor, table: Tensor, sym_idx: Tensor) -> Tensor:
    """The pose kernel's closest symmetric candidate per crop (csrc/losses.cu, pose_loss_kernel): M = R_gt^T R in fp32, the
    geodesic error acos(clamp((tr - 1) / 2)) in double of the unmodified R_gt (trace of M) and of each candidate S_k
    (<M, S_k> summed in row-major order), the first strict minimum, the unmodified R_gt winning every tie.  Returns int64 [B]:
    the candidate index in the crop's symmetry set, or -1."""
    R, Rg = R.detach().float().cpu(), Rg.detach().float().cpu()
    table, sym_idx = table.detach().float().cpu(), sym_idx.detach().long().cpu()
    # nvcc contracts the kernel's sum of three products into fma(g2, r2, fma(g1, r1, g0 r0))
    M = _fma32(Rg[:, 2, :, None], R[:, 2, None, :], _fma32(Rg[:, 1, :, None], R[:, 1, None, :], Rg[:, 0, :, None] * R[:, 0, None, :]))
    M = M.double().reshape(-1, 9)

    def err(tr):
        return torch.acos((0.5 * (tr.clamp(max=3.0) - 1.0)).clamp(-1.0, 1.0))

    out = torch.full((R.shape[0],), -1, dtype=torch.long)
    for b in range(R.shape[0]):
        first, K = int(sym_idx[b, 0]), int(sym_idx[b, 1])
        if K == 0:
            continue
        best = err(M[b, 0] + M[b, 4] + M[b, 8])
        Sk = table[first:first + K].double().reshape(K, 9)
        tr = torch.zeros(K, dtype=torch.float64)
        for i in range(9):
            tr = tr + M[b, i] * Sk[:, i]
        e = err(tr)
        k = int(torch.argmin(e))  # the first minimum
        if bool(e[k] < best):
            out[b] = k
    return out


def _fma32(a: Tensor, b: Tensor, c: Tensor) -> Tensor:
    """fp32 fma(a, b, c): the product is exact in float64, the sum rounded once more to fp32."""
    return (a.double() * b.double() + c.double()).float()


def sym_target(Rg: Tensor, table: Tensor, sym_idx: Tensor, idx: Tensor) -> Tensor:
    """The point-matching target of the chosen candidates, R_gt S_k in fp32 with the kernel's contraction (R_gt where idx = -1)."""
    out = Rg.clone()
    first = sym_idx[:, 0].long().cpu()
    for b in (idx >= 0).nonzero().flatten().tolist():
        S = table[int(first[b]) + int(idx[b])]
        out[b] = _fma32(Rg[b, :, 2:3], S[2], _fma32(Rg[b, :, 1:2], S[1], Rg[b, :, 0:1] * S[0]))
    return out


def closest_sym_index(pred_rots: Tensor, gt_rots: Tensor, sym_infos) -> Tensor:
    """The candidate gdrn_oracle.closest_rot_batch chooses per crop (-1: the unmodified R_gt), from the same float64 errors."""
    from oracle import gdrn_oracle as O

    out = torch.full((pred_rots.shape[0],), -1, dtype=torch.long)
    for b in range(pred_rots.shape[0]):
        if sym_infos[b] is None:
            continue
        sym = torch.as_tensor(sym_infos[b]).detach().cpu().numpy().reshape(-1, 3, 3)
        est, gt = pred_rots[b].detach().cpu().numpy(), gt_rots[b].detach().cpu().numpy()
        best = O._re_deg(est, gt)
        for k in range(sym.shape[0]):
            e = O._re_deg(est, gt.dot(sym[k]))
            if e < best:
                best, out[b] = e, k
    return out


# --------------------------------------------------------------------------------------------------------------- the shim
class PinnedF:
    """Stands in for torch.nn.functional inside the oracle modules (see `pinned`)."""

    def __init__(self, pins: List[Pin], parity: bool = True):
        self._pins, self._next_i, self._parity = pins, 0, parity
        self.sites: List[dict] = []  # per consumed pin: name, kind, n, flips, parity (rel-L2 vs the engine, or None)
        self.inert = 0  # relu / max_pool2d / l1_loss calls whose operands carry no gradient (nothing to decide)

    def __getattr__(self, name):
        return getattr(TF, name)

    def _take(self, kind: str, x: Tensor) -> Pin:
        i = self._next_i
        assert i < len(self._pins), f"{kind} call #{i}: no pin left"
        pin = self._pins[i]
        assert pin.kind == kind, f"call #{i} is {kind}, pin {pin.name} is {pin.kind}"
        assert tuple(x.shape) == pin.shape, f"pin {pin.name}: call shape {tuple(x.shape)} != pin shape {pin.shape}"
        self._next_i += 1
        return pin

    @torch.no_grad()
    def _record(self, pin: Pin, flips: int, n: int, y: Tensor):
        par = None
        if self._parity and pin.act is not None:
            a = pin.act().to(y.device, torch.float64)
            par = float((a - y).norm() / y.norm().clamp_min(1e-300))
        self.sites.append(dict(name=pin.name, kind=pin.kind, n=n, flips=flips, parity=par))

    def relu(self, x: Tensor, inplace: bool = False) -> Tensor:
        if not x.requires_grad:  # a frozen sub-network: no gradient passes, nothing to pin
            self.inert += 1
            return TF.relu(x)
        pin = self._take("relu", x)
        m = pin.decide(x.device)
        y = torch.where(m, x, x.new_zeros(()))
        self._record(pin, int(((x > 0) != m).sum()), m.numel(), y)
        return y

    def leaky_relu(self, x: Tensor, negative_slope: float = 0.01, inplace: bool = False) -> Tensor:
        pin = self._take("leaky_relu", x)
        m = pin.decide(x.device)
        y = torch.where(m, x, x * negative_slope)
        self._record(pin, int(((x > 0) != m).sum()), m.numel(), y)
        return y

    def linear(self, x: Tensor, weight: Tensor, bias: Optional[Tensor] = None) -> Tensor:
        pin = self._take("linear", x)
        y = TF.linear(x, weight, bias)
        v = pin.decide(y.device)
        if v is None:
            self.sites.append(dict(name=pin.name, kind="linear", n=0, flips=0, parity=None))
            return y
        assert v.shape == y.shape, f"pin {pin.name}: value {tuple(v.shape)} != output {tuple(y.shape)}"
        self._record(pin, 0, 0, y)
        return y + (v.to(y.dtype) - y).detach()  # the engine's value, the float64 gradient

    def max_pool2d(self, x: Tensor, kernel_size, stride=None, padding=0, dilation=1, ceil_mode=False, return_indices=False):
        if not x.requires_grad:  # a frozen backbone, or DropBlock's block mask of its seed mask
            self.inert += 1
            return TF.max_pool2d(x, kernel_size, stride, padding, dilation, ceil_mode, return_indices)
        assert (kernel_size, stride, padding, dilation, ceil_mode, return_indices) == (3, 2, 1, 1, False, False)
        pin = self._take("max_pool2d", x)
        codes = pin.decide(x.device)
        y = pool_gather(x, codes)
        with torch.no_grad():
            flips = int((first_max_codes(x) != codes).sum())
        self._record(pin, flips, codes.numel(), y)
        return y

    def l1_loss(self, a: Tensor, b: Tensor, size_average=None, reduce=None, reduction: str = "mean") -> Tensor:
        if not (a.requires_grad or b.requires_grad):
            self.inert += 1
            return TF.l1_loss(a, b, reduction=reduction)
        pin = self._take("l1_loss", a)
        assert a.shape == b.shape and reduction in ("mean", "sum"), (a.shape, b.shape, reduction)
        s = pin.decide(a.device).to(a.dtype)
        d = a - b
        with torch.no_grad():
            flips = int((torch.sign(d) != s).sum())
        v = (s * d).sum() if reduction == "sum" else (s * d).mean()
        self.sites.append(dict(name=pin.name, kind="l1_loss", n=s.numel(), flips=flips, parity=None))
        return v

    def smooth_l1_loss(self, a: Tensor, b: Tensor, size_average=None, reduce=None, reduction: str = "mean",
                       beta: float = 1.0) -> Tensor:
        """torch's smooth L1 (0.5 d^2 / beta for |d| < beta, |d| - 0.5 beta otherwise) in the pinned branch."""
        pin = self._take("smooth_l1_loss", a)
        assert a.shape == b.shape and reduction == "mean" and beta > 0, (a.shape, b.shape, reduction, beta)
        q = pin.decide(a.device).to(a.dtype)
        d = a - b
        with torch.no_grad():
            inner = d.abs() < beta
            flips = int((inner != (q == 0)).sum() + (~inner & (q != 0) & (torch.sign(d) != q)).sum())
        v = torch.where(q == 0, 0.5 * d * d / beta, q * d - 0.5 * beta).mean()
        self.sites.append(dict(name=pin.name, kind="smooth_l1_loss", n=q.numel(), flips=flips, parity=None))
        return v

    def closest_rot_batch(self, pred_rots: Tensor, gt_rots: Tensor, sym_infos) -> Tensor:
        """gdrn_oracle.closest_rot_batch with the pinned candidate per crop (a detached R_gt S_k, like the oracle's)."""
        pin = self._take("closest_rot_batch", pred_rots)
        idx = pin.decide(None)
        out = gt_rots.detach().clone()
        for b, k in enumerate(idx.tolist()):
            if k >= 0:
                assert sym_infos[b] is not None, f"pin {pin.name}: crop {b} has no symmetry set"
                out[b] = gt_rots[b].detach() @ torch.as_tensor(sym_infos[b]).reshape(-1, 3, 3)[k].to(out)
        flips = int((closest_sym_index(pred_rots, gt_rots, sym_infos) != idx).sum())
        self.sites.append(dict(name=pin.name, kind="closest_rot_batch", n=idx.numel(), flips=flips, parity=None))
        return out

    def finish(self):
        left = [p.name for p in self._pins[self._next_i:]]
        assert not left, f"{len(left)} pins were not consumed: {left[:5]}"


@contextlib.contextmanager
def pinned(pins: List[Pin], modules, parity: bool = True):
    """Inside: the modules' `F` is a PinnedF over pins.  On a normal exit every pin must have been consumed."""
    shim = PinnedF(pins, parity)
    old = [(m, m.F) for m in modules]
    for m in modules:
        m.F = shim
    try:
        yield shim
    finally:
        for m, f in old:
            m.F = f
    shim.finish()


def replay(forward: Callable, sd: Dict[str, Tensor], batch: dict, pins: Optional[List[Pin]], modules, device="cuda",
           parity: bool = True):
    """forward(leaf_sd, batch) -> oracle result dict, run in float64 on `device` (pinned unless pins is None), then autograd of
    the summed losses.  Returns (result, leaf state dict with .grad and updated running statistics, shim or None)."""
    from oracle import gdrn_oracle as O

    leaf = O.leaf_state_dict({k: v.to(device) for k, v in sd.items()}, dtype=torch.float64)
    b = {k: (v.to(device) if isinstance(v, Tensor) else v) for k, v in batch.items()}
    b["roi_img"] = b["roi_img"].double()
    shim = None
    if pins is None:
        out = forward(leaf, b)
    else:
        with pinned(pins, modules, parity) as shim:
            out = forward(leaf, b)
    sum(out["losses"].values()).backward()
    return out, leaf, shim


# --------------------------------------------------------------------------------------------------------------- comparison
FLOOR = 1e-3     # rows that are vectors (conv / linear weights): e_r's floor, a fraction of the RMS row norm
FLOOR_1D = 0.1   # entries of 1-D tensors (norm gamma / beta, biases): each is ONE reduction over B H W terms that cancel


def row_errors(g: Tensor, ref: Tensor, floor: float = FLOOR):
    """Per output channel (row; the entries of a 1-D tensor) e_r = |g_r - ref_r| / max(|ref_r|, floor |ref| / sqrt(rows)), and
    the tensor's rel-L2.  Non-finite gradients give NaN rows."""
    ref = ref.detach().double()
    g = g.detach().double().to(ref.device)
    rows = ref.shape[0] if ref.dim() > 1 else ref.numel()
    g2, r2 = g.reshape(rows, -1), ref.reshape(rows, -1)
    fl = max(floor * float(ref.norm()) / math.sqrt(rows), 1e-300)
    e = (g2 - r2).norm(dim=1) / r2.norm(dim=1).clamp_min(fl)
    rel = float((g - ref).norm() / ref.norm().clamp_min(1e-300))
    return e, rel


def family(name: str, head_gn: bool = False) -> str:
    """Report group of a parameter: its sub-network and the kind of tensor (head_gn: the head's norm layers are GroupNorm)."""
    top = name.split(".")[0]
    m = re.match(r"backbone\.(layer\d)", name)
    part = m.group(1) if m else ("stem" if top == "backbone" else top)
    leaf = name.rsplit(".", 1)[1]
    if re.search(r"\.bn\d\.|downsample\.1\.|backbone\.bn1\.", name) or (top == "rot_head_net" and _head_bn(name) and not head_gn):
        kind = "bn." + leaf
    elif (top == "pnp_net" and re.search(r"features\.(1|4|7)\.", name)) or (top == "rot_head_net" and _head_bn(name)):
        kind = "gn." + leaf
    elif ".fc" in name:
        kind = "fc." + leaf
    else:
        kind = "conv." + leaf
    return f"{top}.{part}/{kind}" if top == "backbone" else f"{top}/{kind}"


def _head_bn(name: str) -> bool:
    m = re.match(r"rot_head_net\.features\.(\d+)\.", name)
    return bool(m) and int(m.group(1)) in (1, 4, 7, 11, 14, 18, 21)


def compare_grads(got: Dict[str, Tensor], ref: Dict[str, Tensor], bound: float, bound_1d: Optional[float] = None):
    """Per-row comparison of every tensor in ref: rows of a tensor with two or more dimensions against `bound` (floor FLOOR),
    entries of a 1-D tensor against `bound_1d` (floor FLOOR_1D; default: the same as rows).  Returns (failures
    [(name, row, e_r)], per-tensor rows [(name, worst row, worst e_r, rel-L2)])."""
    fails, table = [], []
    for name, r in ref.items():
        one_d = r.dim() == 1 and bound_1d is not None
        e, rel = row_errors(got[name], r, FLOOR_1D if one_d else FLOOR)
        bad = ~(e <= (bound_1d if one_d else bound))
        k = int(torch.nan_to_num(e, nan=float("inf")).argmax())
        table.append((name, k, float(e[k]), rel))
        for row in bad.nonzero().flatten().tolist()[:3]:
            fails.append((name, row, float(e[row])))
    return fails, table


def worst_by_family(table, head_gn: bool = False) -> Dict[str, tuple]:
    out = {}
    for name, row, e, rel in table:
        f = family(name, head_gn)
        if f not in out or not (out[f][2] >= e):
            out[f] = (name, row, e, rel)
    return out


def running_stat_errors(model, sd0: Dict[str, Tensor], leaf: Dict[str, Tensor], momentum: float = 0.1):
    """Every BatchNorm's running mean / variance after the step against the replay's, in units of the step's own update:
    mean |rm - rm_ref| / (momentum * batch std), var |rv - rv_ref| / (momentum * batch var) (worst channel), and whether
    num_batches_tracked agrees.  Returns {module name: (mean err, var err, counters equal)}."""
    out = {}
    for name, mod in model.named_modules():
        if not isinstance(mod, torch.nn.BatchNorm2d):
            continue
        rm, rv = mod.running_mean.detach().double().cpu(), mod.running_var.detach().double().cpu()
        rm_ref, rv_ref = leaf[name + ".running_mean"].detach().double().cpu(), leaf[name + ".running_var"].detach().double().cpu()
        rv0 = sd0[name + ".running_var"].double().cpu()
        bvar = ((rv_ref - (1 - momentum) * rv0) / momentum).clamp_min(1e-300)  # the unbiased batch variance of the step
        em = float(((rm - rm_ref).abs() / (momentum * bvar.sqrt())).max())
        ev = float(((rv - rv_ref).abs() / (momentum * bvar)).max())
        nbt = int(mod.num_batches_tracked) == int(leaf[name + ".num_batches_tracked"])
        out[name] = (em, ev, nbt)
    return out
