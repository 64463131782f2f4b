"""Thin Python wrappers over the C ABI (device memory and streams come from PyTorch: plumbing only).

`PT` is the planar bf16 pair used for every activation / gradient: value = hi (+ lo).
`planes` = 1 -> bf16 tensor-core mode (nsplit = 1), 2 -> fp32-faithful mode (nsplit = 3).
"""
from __future__ import annotations

import ctypes

import torch

from .capi import C


def _stream():
    return torch.cuda.current_stream().cuda_stream


_FMT = {}


def storage_format():
    """(torch dtype, lo-plane scale, name) of the library's compile-time 16-bit storage format (csrc/ptx.cuh)."""
    if not _FMT:
        dll = C.load()
        dll.gdrn_lo_scale.restype = ctypes.c_float
        f16 = bool(dll.gdrn_storage_format())
        _FMT.update(dtype=torch.float16 if f16 else torch.bfloat16, lo_scale=float(dll.gdrn_lo_scale()), name="fp16" if f16 else "bf16")
    return _FMT["dtype"], _FMT["lo_scale"], _FMT["name"]


def round_storage(x: torch.Tensor) -> torch.Tensor:
    """x rounded to the single-plane storage format, as fp32 (what a planes=1 operand effectively is)."""
    return x.to(storage_format()[0]).float()


def ptr(t):
    return None if t is None else t.data_ptr()


class PT:
    """Planar (hi[, lo]) bf16 tensor of logical shape `shape` stored as [planes, *shape]."""

    __slots__ = ("buf", "shape", "planes")

    def __init__(self, shape, planes: int, device="cuda", buf=None, zero=False):
        self.shape = tuple(int(s) for s in shape)
        self.planes = planes
        if buf is None:
            alloc = torch.zeros if zero else torch.empty
            buf = alloc((planes,) + self.shape, dtype=storage_format()[0], device=device)
        self.buf = buf

    @property
    def hi(self):
        return self.buf[0]

    @property
    def lo(self):
        return self.buf[1] if self.planes == 2 else None

    @property
    def hi_ptr(self):
        return self.buf.data_ptr()

    @property
    def lo_ptr(self):
        return (self.buf.data_ptr() + self.buf[0].numel() * 2) if self.planes == 2 else None

    @property
    def nsplit(self):
        return 1 if self.planes == 1 else 3

    def numel(self):
        return self.buf[0].numel()

    def float(self):
        x = self.buf[0].float()
        if self.planes == 2:
            x = x + self.buf[1].float() * (1.0 / storage_format()[1])
        return x

    def as_planes(self, planes: int) -> "PT":
        """This tensor as a `planes`-plane operand: 2 -> 1 keeps the hi plane (= the value rounded to the 16-bit format)."""
        if planes == self.planes:
            return self
        assert planes == 1 and self.planes == 2, (planes, self.planes)
        return PT(self.shape, 1, buf=self.buf[0:1])

    def view(self, *shape):
        return PT(shape, self.planes, buf=self.buf.view((self.planes,) + tuple(shape)))

    @staticmethod
    def from_float(x: torch.Tensor, planes: int) -> "PT":
        x = x.contiguous().float()
        out = PT(x.shape, planes, device=x.device)
        assert x.numel() % 8 == 0
        C.gdrn_f32_to_planes(x.data_ptr(), out.hi_ptr, out.lo_ptr, x.numel(), _stream())
        return out

    def to_float(self) -> torch.Tensor:
        y = torch.empty(self.shape, dtype=torch.float32, device=self.buf.device)
        C.gdrn_planes_to_f32(self.hi_ptr, self.lo_ptr, y.data_ptr(), y.numel(), _stream())
        return y


ACT_STATS_F64 = 16  # act flag bit of the GEMM entry points: the epilogue statistics buffer is double (include/gdrn_b200.h)


def _act(act: int, stats) -> int:
    """act with ACT_STATS_F64 set when the statistics buffer is float64."""
    return act | ACT_STATS_F64 if stats is not None and stats.dtype == torch.float64 else act


def _round_up(x, m):
    return (x + m - 1) // m * m


_pack_recorder = None  # when a list: pack calls are recorded as job tuples instead of launched (Engine batches them)


def _pack(src: torch.Tensor, out: "PT", O, I, KH, KW, opad, ipad, krow, so, si, sr, ss, flip):
    if _pack_recorder is not None:
        _pack_recorder.append((src, out, O, I, KH, KW, opad, ipad, krow, so, si, sr, ss, flip))
        return
    C.gdrn_pack_weight(src.data_ptr(), out.hi_ptr, out.lo_ptr, O, I, KH, KW, opad, ipad, krow, so, si, sr, ss, flip, _stream())


# ---------------------------------------------------------------------------------------------
# weight packing
# ---------------------------------------------------------------------------------------------
def pack_conv_fwd(w: torch.Tensor, planes: int, out: PT | None = None, ipad: int | None = None) -> PT:
    """Conv2d OIHW fp32 -> [Cout_pad][KH*KW*Cin_pad] (forward operand)."""
    O, I, KH, KW = w.shape
    ipad = ipad or _round_up(I, 64)
    opad = _round_up(O, 64)
    krow = KH * KW * ipad
    out = out or PT((opad, krow), planes, device=w.device)
    _pack(w, out, O, I, KH, KW, opad, ipad, krow, I * KH * KW, KH * KW, KW, 1, 0)
    return out


def pack_conv_dgrad(w: torch.Tensor, planes: int, out: PT | None = None, ipad: int | None = None) -> PT:
    """Conv2d OIHW fp32 -> [Cin_pad][KH*KW*Cout_pad], taps flipped: dX = conv(dY (zero-inserted if s2), this).  ipad: Cout_pad,
    the row width of dY (default round_up(Cout, 64))."""
    O, I, KH, KW = w.shape
    opad, ipad = _round_up(I, 64), ipad or _round_up(O, 64)
    krow = KH * KW * ipad
    out = out or PT((opad, krow), planes, device=w.device)
    # rows = input channels (stride KH*KW), cols = output channels (stride I*KH*KW)
    _pack(w, out, I, O, KH, KW, opad, ipad, krow, KH * KW, I * KH * KW, KW, 1, 1)
    return out


def pack_stem(w: torch.Tensor, planes: int, out: PT | None = None) -> PT:
    """7x7 stem weight [64][3][7][7] -> [64][192] with k = (r*7+s)*3 + c (matches gdrn_stem_im2col); cols 147..191 stay zero."""
    out = out or PT((64, 192), planes, device=w.device, zero=True)
    _pack(w, out, 64, 3, 7, 7, 64, 3, 192, 147, 49, 7, 1, 0)
    return out


def pack_deconv_fwd(wt: torch.Tensor, planes: int, out: PT | None = None) -> PT:
    """ConvTranspose2d IOHW [Cin][Cout][k][k] -> equivalent stride-1 conv over the zero-inserted input
    (taps flipped): rows = Cout, cols = Cin.  (First formulation, kept for the op tests.)"""
    I, O, KH, KW = wt.shape
    opad, ipad = _round_up(O, 64), _round_up(I, 64)
    krow = KH * KW * ipad
    out = out or PT((opad, krow), planes, device=wt.device)
    _pack(wt, out, O, I, KH, KW, opad, ipad, krow, KH * KW, O * KH * KW, KW, 1, 1)
    return out


def pack_deconv_dgrad(wt: torch.Tensor, planes: int, out: PT | None = None) -> PT:
    """ConvTranspose2d IOHW -> plain stride-2 conv weight with rows = Cin, cols = Cout (dX = conv_s2(dY, this))."""
    I, O, KH, KW = wt.shape
    opad, ipad = _round_up(I, 64), _round_up(O, 64)
    krow = KH * KW * ipad
    out = out or PT((opad, krow), planes, device=wt.device)
    _pack(wt, out, I, O, KH, KW, opad, ipad, krow, O * KH * KW, KH * KW, KW, 1, 0)
    return out


def pack_linear(w: torch.Tensor, planes: int, out: PT | None = None, nhwc_from: tuple | None = None,
                transpose: bool = False) -> PT:
    """Linear [N][K] fp32 -> [N_pad][K] (forward) or [K_pad][N_pad] (transpose=True, dgrad operand).
    nhwc_from=(C,H,W): the K axis is an NCHW flatten that must become an NHWC flatten (fc1)."""
    N, K = w.shape
    if nhwc_from is not None:
        Cc, H, W = nhwc_from
        assert Cc * H * W == K
        if not transpose:
            # view as OIHW [N][C][H][W] -> rows N, cols (h, w, c)
            opad = _round_up(N, 64)
            out = out or PT((opad, K), planes, device=w.device)
            _pack(w, out, N, Cc, H, W, opad, Cc, K, K, H * W, W, 1, 0)
            return out
        # dgrad operand [K' = (h, w, c)][N]: dst viewed as [tap = h*W+w][c][n] == pack with O = taps, "taps" = C, I = N
        taps = H * W
        npad = _round_up(N, 64)
        assert npad == N
        out = out or PT((K, N), planes, device=w.device)
        _pack(w, out, taps, N, Cc, 1, taps, N, Cc * N, 1, K, taps, 0, 0)
        return out
    if not transpose:
        opad = _round_up(N, 64)
        out = out or PT((opad, K), planes, device=w.device)
        _pack(w, out, N, K, 1, 1, opad, K, K, K, 1, 0, 0, 0)
    else:
        opad, ipad = _round_up(K, 64), _round_up(N, 64)
        out = out or PT((opad, ipad), planes, device=w.device)
        _pack(w, out, K, N, 1, 1, opad, ipad, ipad, 1, K, 0, 0, 0)
    return out


# ---------------------------------------------------------------------------------------------
# GEMM / conv
# ---------------------------------------------------------------------------------------------
def conv_fwd(x: PT, wp: PT, Cout: int, KH: int, KW: int, stride: int, pad: int, *, out: PT | None = None,
             out_f32: torch.Tensor | None = None, bias=None, stats=None, act: int = 0, ldc: int | None = None,
             want_planes: bool = True, algo_scale: float = 1.0, res: PT | None = None) -> PT | None:
    """algo_scale: fraction of the launched MACs that are algorithmic (0.25 for zero-inserted inputs); bookkeeping only.
    res: residual planes added in the epilogue before the activation (act 2 = ReLU): the folded eval-mode conv+BN+add+ReLU."""
    N, H, W, Cin = x.shape
    Ho, Wo = H // stride, W // stride
    ldc = ldc or _round_up(Cout, 64)
    if want_planes and out is None:
        out = PT((N, Ho, Wo, ldc), x.planes, device=x.buf.device, zero=(ldc != Cout))
    C.gdrn_conv_fwd(x.hi_ptr, x.lo_ptr, wp.hi_ptr, wp.lo_ptr, out.hi_ptr if out is not None else None,
                    out.lo_ptr if out is not None else None, ptr(out_f32), ptr(bias), res.hi_ptr if res is not None else None,
                    res.lo_ptr if res is not None else None, ptr(stats), N, H, W, Cin, Cout, wp.shape[0], KH, KW, stride, pad,
                    ldc, _act(act, stats), x.nsplit, _stream())
    return out


def conv_dgrad_s2(du: PT, wd: PT, Cx: int, K: int, pad: int, *, out: PT | None = None, bias=None, stats=None, act: int = 0) -> PT:
    """dX of a stride-2 conv (k3 p1 / k1 p0) from the UN-dilated dY, decomposed by output parity (gdrn_conv_dgrad_s2);
    wd = pack_conv_dgrad(weight).  Replaces zero_insert + stride-1 conv (4x the MACs, plus the dilated tensor in HBM)."""
    N, Ho, Wo, Cy = du.shape
    ldc = _round_up(Cx, 64)
    if out is None:
        out = PT((N, 2 * Ho, 2 * Wo, ldc), du.planes, device=du.buf.device, zero=(K == 1 or ldc != Cx))
    C.gdrn_conv_dgrad_s2(du.hi_ptr, du.lo_ptr, wd.hi_ptr, wd.lo_ptr, out.hi_ptr, out.lo_ptr, ptr(bias), ptr(stats), N, Ho, Wo, Cy, Cx,
                         wd.shape[0], K, pad, ldc, _act(act, stats), du.nsplit, _stream())
    return out


def gemm_fwd(a: PT, wp: PT, N: int, *, out: PT | None = None, out_f32: torch.Tensor | None = None, bias=None, stats=None,
             act: int = 0, ldc: int | None = None, want_planes: bool = True) -> PT | None:
    M, K = a.shape
    ldc = ldc or _round_up(N, 64)
    if want_planes and out is None:
        out = PT((M, ldc), a.planes, device=a.buf.device, zero=(ldc != N))
    C.gdrn_gemm_fwd(a.hi_ptr, a.lo_ptr, wp.hi_ptr, wp.lo_ptr, out.hi_ptr if out is not None else None,
                    out.lo_ptr if out is not None else None, ptr(out_f32), ptr(bias), ptr(stats), M, N, wp.shape[0], K, ldc,
                    _act(act, stats), a.nsplit, _stream())
    return out


def conv_fwd_grouped(x: PT, wp: PT, Cout: int, Cout_pad: int, group: torch.Tensor, rows_per_group: int, *, out_f32: torch.Tensor,
                     bias=None, bias_stride: int = 0, ldc: int | None = None):
    """1x1 / k x k stride-1 conv whose output rows [g * rows_per_group, ...) use weight block group[g] of wp ([G * Cout_pad][K]) and
    bias[group[g] * bias_stride:]; group: int32 device tensor.  fp32 output only (the class-aware output conv's logits)."""
    N, H, W, Cin = x.shape
    G = wp.shape[0] // Cout_pad
    C.gdrn_conv_fwd_grouped(x.hi_ptr, x.lo_ptr, wp.hi_ptr, wp.lo_ptr, None, None, out_f32.data_ptr(), ptr(bias), N, H, W, Cin, Cout,
                            Cout_pad, 1, 1, 1, 0, ldc or _round_up(Cout, 64), 0, x.nsplit, group.data_ptr(), rows_per_group, G,
                            bias_stride, _stream())


def gemm_fwd_grouped(a: PT, wp: PT, N: int, group: torch.Tensor, rows_per_group: int) -> PT:
    """y = a w_g^T with w_g = block group[row // rows_per_group] of wp ([G * N][K], N % 64 == 0): the class-aware dgrad."""
    M, K = a.shape
    G = wp.shape[0] // N
    out = PT((M, N), a.planes, device=a.buf.device)
    C.gdrn_gemm_fwd_grouped(a.hi_ptr, a.lo_ptr, wp.hi_ptr, wp.lo_ptr, out.hi_ptr, out.lo_ptr, None, None, M, N, N, K, N, 0, a.nsplit,
                            group.data_ptr(), rows_per_group, G, 0, _stream())
    return out


class Workspace:
    """Grow-only fp32 scratch for split-K weight-gradient partials."""

    def __init__(self, device="cuda"):
        self.device = device
        self.buf = None

    def get(self, nfloats: int) -> torch.Tensor:
        if self.buf is None or self.buf.numel() < nfloats:
            self.buf = torch.empty(int(nfloats), dtype=torch.float32, device=self.device)
        return self.buf


def conv_wgrad(dy: PT, x: PT, ws: Workspace, Cout: int, KH: int, KW: int, stride: int, pad: int, ksplit: int = 0):
    """Returns (workspace tensor, ksplit, ks_stride).  dy [N,Ho,Wo,Cout_pad], x [N,H,W,Cin]."""
    N, H, W, Cin = x.shape
    need = ctypes.c_long(0)
    ks = ctypes.c_int(0)
    cout_ld = dy.shape[-1]
    args = (N, H, W, Cin, cout_ld, KH, KW, stride, pad, ksplit, x.nsplit, _stream())
    C.gdrn_conv_wgrad(None, None, None, None, None, 0, ctypes.addressof(need), ctypes.addressof(ks), *args)
    buf = ws.get(need.value)
    C.gdrn_conv_wgrad(dy.hi_ptr, dy.lo_ptr, x.hi_ptr, x.lo_ptr, buf.data_ptr(), buf.numel(), None, None, *args)
    mpad = _round_up(cout_ld, 128)
    return buf, ks.value, mpad * KH * KW * Cin


def gemm_wgrad(dy: PT, x: PT, ws: Workspace, ksplit: int = 0):
    """dW[M][Ntot] = dy[P][M]^T x[P][Ntot]."""
    P, M = dy.shape
    P2, Ntot = x.shape
    assert P == P2
    need = ctypes.c_long(0)
    ks = ctypes.c_int(0)
    args = (P, M, Ntot, ksplit, x.nsplit, _stream())
    C.gdrn_gemm_wgrad(None, None, None, None, None, 0, ctypes.addressof(need), ctypes.addressof(ks), *args)
    buf = ws.get(need.value)
    C.gdrn_gemm_wgrad(dy.hi_ptr, dy.lo_ptr, x.hi_ptr, x.lo_ptr, buf.data_ptr(), buf.numel(), None, None, *args)
    return buf, ks.value, _round_up(M, 128) * Ntot


def unpack_wgrad(buf, grad: torch.Tensor, O, I, KH, KW, ipad, ksplit, ks_stride, so, si, sr, ss, flip=0, accumulate=0, krow=None):
    """krow: row length of the workspace (defaults to KH*KW*ipad)."""
    C.gdrn_unpack_wgrad(buf.data_ptr(), grad.data_ptr(), O, I, KH, KW, ipad, krow or KH * KW * ipad, ksplit, ks_stride, so, si, sr,
                        ss, flip, accumulate, _stream())


# ---------------------------------------------------------------------------------------------
# elementwise
# ---------------------------------------------------------------------------------------------
def like(x: PT, shape=None) -> PT:
    return PT(shape or x.shape, x.planes, device=x.buf.device)


def bn_finalize(stats, gamma, beta, rm, rv, scale, shift, mean, invstd, C_, count, eps, momentum, train):
    C.gdrn_bn_finalize(ptr(stats), gamma.data_ptr(), beta.data_ptr(), ptr(rm), ptr(rv), scale.data_ptr(), shift.data_ptr(),
                       ptr(mean), ptr(invstd), C_, float(count), float(eps), float(momentum), int(train), _stream())


def bn_act(x: PT, scale, shift, relu: bool, res: PT | None = None, out: PT | None = None) -> PT:
    out = out or like(x)
    Cc = x.shape[-1]
    rows = x.numel() // Cc
    C.gdrn_bn_act(x.hi_ptr, x.lo_ptr, res.hi_ptr if res else None, res.lo_ptr if res else None, out.hi_ptr, out.lo_ptr,
                  scale.data_ptr(), shift.data_ptr(), rows, Cc, int(relu), _stream())
    return out


def bn_bwd(ga: PT, gb: PT | None, y: PT | None, u: PT, mean, invstd, gamma, sums, dgamma, dbeta, train: bool,
           want_gout: bool = False, beta=None, relu_from_u: bool = False, sums_zeroed: bool = False, relu_mask=None, det_ws=None):
    """y: activation whose sign gives the ReLU mask (needed when a residual was added before the ReLU); relu_from_u: plain
    conv-BN-ReLU, the mask is recomputed from u and beta and y is not read."""
    du = like(u)
    gout = like(u) if want_gout else None
    Cc = u.shape[-1]
    rows = u.numel() // Cc
    assert not (relu_from_u and y is not None)
    C.gdrn_bn_bwd(ga.hi_ptr, ga.lo_ptr, gb.hi_ptr if gb else None, gb.lo_ptr if gb else None, y.hi_ptr if y else None,
                  u.hi_ptr, u.lo_ptr, mean.data_ptr(), invstd.data_ptr(), gamma.data_ptr(), ptr(beta), sums.data_ptr(), du.hi_ptr,
                  du.lo_ptr, gout.hi_ptr if gout else None, gout.lo_ptr if gout else None, ptr(dgamma), ptr(dbeta), ptr(relu_mask),
                  ptr(det_ws), rows, Cc, int(train),
                  (1 if relu_from_u else 0) | (2 if sums_zeroed else 0) | (4 if det_ws is not None else 0), _stream())
    return du, gout


def maxpool_fwd(x: PT, want_arg: bool = False):
    B, H, W, Cc = x.shape
    out = like(x, (B, H // 2, W // 2, Cc))
    arg = torch.empty((B, H // 2, W // 2, Cc), dtype=torch.uint8, device=x.buf.device) if want_arg else None
    C.gdrn_maxpool_fwd(x.hi_ptr, x.lo_ptr, out.hi_ptr, out.lo_ptr, ptr(arg), B, H, W, Cc, _stream())
    return (out, arg) if want_arg else out


def maxpool_bwd(arg: torch.Tensor, g: PT) -> PT:
    B, Ho, Wo, Cc = g.shape
    out = like(g, (B, 2 * Ho, 2 * Wo, Cc))
    C.gdrn_maxpool_bwd(arg.data_ptr(), g.hi_ptr, g.lo_ptr, out.hi_ptr, out.lo_ptr, B, 2 * Ho, 2 * Wo, Cc, _stream())
    return out


def upsample2x_fwd(x: PT) -> PT:
    B, H, W, Cc = x.shape
    out = like(x, (B, 2 * H, 2 * W, Cc))
    C.gdrn_upsample2x_fwd(x.hi_ptr, x.lo_ptr, out.hi_ptr, out.lo_ptr, B, H, W, Cc, _stream())
    return out


def upsample2x_bwd(g: PT) -> PT:
    B, Ho, Wo, Cc = g.shape
    out = like(g, (B, Ho // 2, Wo // 2, Cc))
    C.gdrn_upsample2x_bwd(g.hi_ptr, g.lo_ptr, out.hi_ptr, out.lo_ptr, B, Ho // 2, Wo // 2, Cc, _stream())
    return out


def zero_insert(x: PT) -> PT:
    B, H, W, Cc = x.shape
    out = like(x, (B, 2 * H, 2 * W, Cc))
    C.gdrn_zero_insert(x.hi_ptr, x.lo_ptr, out.hi_ptr, out.lo_ptr, B, H, W, Cc, 0, _stream())
    return out


def extract_even(x: PT) -> PT:
    B, H2, W2, Cc = x.shape
    out = like(x, (B, H2 // 2, W2 // 2, Cc))
    C.gdrn_zero_insert(x.hi_ptr, x.lo_ptr, out.hi_ptr, out.lo_ptr, B, H2 // 2, W2 // 2, Cc, 1, _stream())
    return out


def gn_relu_fwd(u: PT, gamma, beta, stats, G=32, eps=1e-5) -> PT:
    B, H, W, Cc = u.shape
    out = like(u)
    C.gdrn_gn_relu_fwd(u.hi_ptr, u.lo_ptr, out.hi_ptr, out.lo_ptr, gamma.data_ptr(), beta.data_ptr(), stats.data_ptr(), B, H * W,
                       Cc, G, float(eps), _stream())
    return out


def gn_relu_bwd(g: PT, y: PT, u: PT, gamma, stats, dgamma, dbeta, G=32) -> PT:
    B, H, W, Cc = u.shape
    du = like(u)
    C.gdrn_gn_relu_bwd(g.hi_ptr, g.lo_ptr, y.hi_ptr, u.hi_ptr, u.lo_ptr, gamma.data_ptr(), stats.data_ptr(), du.hi_ptr, du.lo_ptr,
                       dgamma.data_ptr(), dbeta.data_ptr(), B, H * W, Cc, G, _stream())
    return du


def head_gn_workspace(B: int, HW: int, dev) -> torch.Tensor:
    """Scratch of gdrn_head_gn_fwd / _bwd (float64): the partial sums of their two-stage reductions."""
    return torch.empty(int(C.load().gdrn_head_gn_workspace(B, HW)), dtype=torch.float64, device=dev)


def head_gn_relu_fwd(u: PT, gamma, beta, G: int, eps: float = 1e-5, want_mask: bool = False):
    """Geometry-head GroupNorm(G, 256) + ReLU: (y, stats [B, G, 2] = (mean, invstd), ReLU bitmap or None)."""
    B, H, W, Cc = u.shape
    out = like(u)
    stats = torch.empty(B, G, 2, device=u.buf.device)
    mask = torch.empty(u.numel() // 8, dtype=torch.uint8, device=u.buf.device) if want_mask else None
    ws = head_gn_workspace(B, H * W, u.buf.device)
    C.gdrn_head_gn_fwd(u.hi_ptr, u.lo_ptr, out.hi_ptr, out.lo_ptr, ptr(mask), gamma.data_ptr(), beta.data_ptr(), stats.data_ptr(),
                       ws.data_ptr(), B, H * W, Cc, G, float(eps), _stream())
    return out, stats, mask


def head_gn_relu_bwd(g: PT, u: PT, mask, gamma, stats, dgamma, dbeta) -> PT:
    """Backward of head_gn_relu_fwd: dL/du in g's planes; dgamma / dbeta are written, not accumulated."""
    B, H, W, Cc = u.shape
    du = like(g)
    ws = head_gn_workspace(B, H * W, g.buf.device)
    C.gdrn_head_gn_bwd(g.hi_ptr, g.lo_ptr, u.hi_ptr, u.lo_ptr, mask.data_ptr(), gamma.data_ptr(), stats.data_ptr(), du.hi_ptr, du.lo_ptr,
                       dgamma.data_ptr(), dbeta.data_ptr(), ws.data_ptr(), B, H * W, Cc, stats.shape[1], _stream())
    return du


def add2(a: PT, b: PT) -> PT:
    out = like(a)
    C.gdrn_add2(a.hi_ptr, a.lo_ptr, b.hi_ptr, b.lo_ptr, out.hi_ptr, out.lo_ptr, a.numel(), _stream())
    return out
