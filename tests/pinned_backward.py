"""Pinned float64 backward: the parameter gradients of a whole engine step against a float64 replay of the oracle that follows
the engine's own non-smooth decisions.

The engine's forward differs from a float64 forward by ~1e-4 (DESIGN §8, tools/noise_floor.py).  That flips a few ReLU, max-pool
and L1-sign decisions, and every flip moves the gradients downstream of it, which is why a plain gradient comparison needs 6e-2
per tensor.  Given the decisions, the backward is linear.  So this module

  * `capture(engine)`: after a `do_loss` forward and BEFORE backward (which clears `engine.saved`), takes the decisions out of
    `engine.saved` in the oracle's call order: the 40 BatchNorm + ReLU bitmaps, the max-pool window codes, the 3 GroupNorm + ReLU
    and 2 LeakyReLU masks (`y > 0` of the stored output, as the backward kernels read them) and the signs of the 7 L1 residuals,
    recomputed in fp32 from the engine's own outputs exactly as the loss kernels form them;
  * `pinned(pins, modules)`: swaps the oracle modules' `F` for a shim whose relu / max_pool2d / leaky_relu / l1_loss consume
    the next pin (a pinned ReLU is x * mask, a pinned max-pool gathers the coded window element, a pinned L1 is sum s (a - b));
    everything else is torch.nn.functional.  The shim counts, per site, the elements the float64 forward would have decided
    differently and the rel-L2 of its output against the engine's stored activation (a per-layer forward parity);
  * `row_errors` / `compare_grads`: per output channel e_r = |g_r - ref_r| / max(|ref_r|, floor |ref| / sqrt(rows)), floor
    1e-3 for the rows of a weight.  An entry of a 1-D tensor (BatchNorm / GroupNorm gamma and beta, a bias) is one sum over
    B H W terms that largely cancel: its absolute error follows the size of the terms, not of the sum, and on the B = 64
    step the small entries' errors are ~1e-3 of the tensor's RMS entry in "mixed" (3e-4 in "fp32x3"), so those entries are
    measured against a floor of 0.1 of the RMS entry and a bound of their own;
  * `running_stat_errors`: every BatchNorm running mean / variance / counter after the step against the replay's.

The layouts decoded here (csrc/elementwise.cu): a ReLU bitmap holds flat NHWC element e as bit e & 7 of byte e >> 3, set when
the fp32 pre-activation (+ residual) is > 0 (bn_fwd); a max-pool code is dy * 3 + dx of the 3x3 / stride 2 / pad 1 window, the
first strict maximum in row-major order (maxpool_fwd_kernel).  Only the shipped loss switches are pinned: L1 mask head, L1 point
matching on R, no symmetric candidates (`capture` rejects anything else).  A new pin kind is one more shim method and one more
constructor below.
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


def _pt_act(pt) -> Callable:
    return lambda: _nchw(pt.float())


def capture(engine) -> List[Pin]:
    """The decisions of the engine's last do_loss forward, in the oracle's call order.  Call before engine.backward.  The
    activations of the parity check stay referenced (no copy) until the pins are dropped."""
    S = engine.saved
    assert S is not None, "capture() needs a do_loss forward whose backward has not run yet"
    aux = S["aux"]
    if engine.mask_loss != 0 or engine.pose_ex or aux.get("sym_idx") is not None:
        raise NotImplementedError("pins exist for the L1 mask head and the shipped pose losses without symmetry only")

    def bitmap(name, mask, pt):
        return Pin.relu_bitmap(name, mask, pt.shape, _pt_act(pt))

    St = S["stem"]
    pins = [bitmap("backbone.bn1", St["m0"], St["a0"]),
            Pin.pool("backbone.maxpool", St["pool_arg"], St["a0"].shape, _pt_act(S["blocks"][0]["x_in"]))]
    for L in S["blocks"]:
        pins += [bitmap(L["p"] + ".bn1", L["m1"], L["a1"]), bitmap(L["p"] + ".bn2", L["m2"], L["out"])]
    pins.append(bitmap("rot_head_net.features.1", S["deconv"]["m"], S["deconv"]["y"]))
    pins += [bitmap(f"rot_head_net.features.{L['bi']}", L["m"], L["y"]) for L in S["head"]]
    pins += [Pin.positive("relu", f"pnp_net.features.{L['gi']}", L["y"].hi, _pt_act(L["y"])) for L in S["pnp"]]
    pins += [Pin.positive("leaky_relu", f"pnp_net.{k}", S[h].hi, _pt_act(S[h])) for k, h in (("fc1", "h1"), ("fc2", "h2"))]
    return pins + loss_sign_pins(engine, S)


def loss_sign_pins(engine, S) -> List[Pin]:
    """The signs of the 7 L1 residuals, formed in fp32 from the engine's outputs like csrc/losses.cu forms them: xyz
    masked_diff(logit, gt, m) = fl(logit m) - fl(gt m); mask logit - target; point matching fl(w est) - fl(w tgt) with
    est = (R p) summed left to right, R the decoded ego rotation; centroid and z pred - ratio.  sign(0) = 0."""
    B, aux, mo = S["B"], S["aux"], engine.mask_out
    lg = S["logits"].view(B, 64, 64, 72)
    m_xyz, m_mask = aux["gt_mask_" + engine.mask_gt[0]], aux["gt_mask_" + engine.mask_gt[1]]
    pins = []
    for j, c in enumerate("xyz"):
        e = lg[..., mo + j] * m_xyz - aux["gt_xyz"][:, j] * m_xyz
        pins.append(Pin.sign(f"loss_coor_{c}", torch.sign(e)[:, None]))
    pins.append(Pin.sign("loss_mask", torch.sign(lg[..., 0] - m_mask)))
    R, Rg, P = S["out_rot"], aux["gt_ego_rot"], aux["gt_points"]
    w = (1.0 / aux["roi_extents"].max(1).values).view(B, 1, 1)

    def rot(M):  # [B, n, 3]: row i of M dotted with each point, summed left to right in fp32
        return M[:, None, :, 0] * P[:, :, None, 0] + M[:, None, :, 1] * P[:, :, None, 1] + M[:, None, :, 2] * P[:, :, None, 2]

    pins.append(Pin.sign("loss_PM_R", torch.sign(rot(R) * w - rot(Rg) * w)))
    nr = engine.model.pnp_net.fc_r.out_features
    t, ratio = S["pred"][:, nr:nr + 3], aux["gt_trans_ratio"]
    pins.append(Pin.sign("loss_centroid", torch.sign(t[:, :2] - ratio[:, :2])))
    pins.append(Pin.sign("loss_z", torch.sign(t[:, 2] - ratio[:, 2])))
    return pins


# --------------------------------------------------------------------------------------------------------------- the shim
class PinnedF:
    """Stands in for torch.nn.functional inside the oracle modules (see `pinned`)."""

    def __init__(self, pins: List[Pin], parity: bool = True):
        self._pins, self._next_i, self._parity = pins, 0, parity
        self.sites: List[dict] = []  # per consumed pin: name, kind, n, flips, parity (rel-L2 vs the engine, or None)
        self.inert = 0  # l1_loss calls whose operands carry no gradient (nothing to decide)

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

    def max_pool2d(self, x: Tensor, kernel_size, stride=None, padding=0, dilation=1, ceil_mode=False, return_indices=False):
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


def family(name: str) -> str:
    """Report group of a parameter: its sub-network and the kind of tensor."""
    top = name.split(".")[0]
    m = re.match(r"backbone\.(layer\d)", name)
    part = m.group(1) if m else ("stem" if top == "backbone" else top)
    leaf = name.rsplit(".", 1)[1]
    if re.search(r"\.bn\d\.|downsample\.1\.|backbone\.bn1\.", name) or (top == "rot_head_net" and _head_bn(name)):
        kind = "bn." + leaf
    elif top == "pnp_net" and re.search(r"features\.(1|4|7)\.", name):
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


def worst_by_family(table) -> Dict[str, tuple]:
    out = {}
    for name, row, e, rel in table:
        f = family(name)
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
