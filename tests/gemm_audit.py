"""Per-launch audit of the wgmma GEMM kernels (csrc/gemm_fwd.cu, csrc/gemm_wgrad.cu) against float64.

`Audit` is a context manager that replaces ops.conv_fwd, gemm_fwd, conv_dgrad_s2, conv_wgrad, gemm_wgrad and unpack_wgrad by
wrappers.  Each wrapper runs the real op and then rebuilds the result in float64 FROM THAT LAUNCH'S EXACT OPERANDS: the
planar activation / gradient (hi + lo / lo_scale), the packed weight operand decoded from its K-major layout, and the bias,
residual, activation, statistics, ldc and fp32-output arguments as passed.  So a launch differs from its reference only by
the kernel's own arithmetic, and the comparison can be made per element:

    |got - ref| <= c * absref + u * |ref| + tiny          absref = conv(|x|, |w|) (+ |bias| + |res|)

c is one constant per kernel family and operand kind (BOUNDS below, each derived and with the worst value measured), u the
unit roundoff of a single-plane 16-bit output (0 for fp32 and two-plane outputs), tiny half the smallest subnormal of the
output format (the 1024-scaled backward reaches fp16 subnormals, where rounding is absolute).  A whole-tensor
max-normalised error hides a wrong small channel (tests/loss_ref_common.py); absref scales every element by what was
actually summed into it, so a dropped cross term of the 3-pass mode (~2^-12 of absref) stands out by two decades.

A failure names the layer, the kernel variant, the tile height, the (m_tile, n_tile, phase) of the worst element, the
128-row A box and the MMA warpgroup's 64-row half that wrote it, and how many tiles the persistent CTA that produced it had
processed before: first-tile and later-tile faults of the tile loop read differently.

The tile / grid arithmetic at the top mirrors the host code of the two kernels and runs without a GPU
(tests/test_gemm_audit_cpu.py checks it, the layout decoders and the references on CPU tensors)."""
import contextlib
import math

import torch
import torch.nn.functional as F

PHASE_ORDER = ((1, 1), (1, 0), (0, 1), (0, 0))  # gdrn_conv_dgrad_s2 walks the output-parity phases in this order (gemm_fwd.cu:686)

# ------------------------------------------------------------------------------------------------ bounds
# c of the error measure, per kernel family and operand planes.  K is the reduction length of one output element.
#   fwd, planes 1: products of two 11-bit values are exact in fp32; the tensor core adds each 16-deep MMA into the fp32
#     accumulator, K / 16 sequential additions of at most 2^-23 of the running sum (<= absref) each.  The longest forward
#     reduction is K = 8192 (fc1): worst case 512 * 2^-23 = 6e-5 if every rounding went the same way.
#   fwd, planes 2: the same, plus the dropped lo x lo products (2^-22 absref), the hi x lo + lo x hi sums folded in with one
#     fp32 fma, and the split of the output into two planes (2^-22 |ref|).
#   wgrad: as forward with K = the pixels of one K-split: n = 4 MMAs per 64-pixel k-block, up to 1366 k-blocks per split (the
#     64 x 64 x 256 head layers at B = 64 in the 3-pass mode: 5464 additions).  The errors of so long a sum do not align, and
#     the flat bound below is what the deepest launches need; a SHORT reduction gets the worst case of its own depth,
#     WGRAD_C0 + n * 2^-18 (wgrad_bound), the tighter of the two below n = 16.  2^-18 per MMA and not 2^-23: the tensor core
#     aligns the 16 products of an MMA and the accumulator to the largest of them and truncates each, so one MMA can lose
#     17 * 2^-23 of its LARGEST term, and the engine's gradients span many binades.  Measured at n = 4 (fc1 at B = 64, 3-pass,
#     the engine's operands): 1.09e-5, bound 1.7e-5; Gaussian operands of the same depth stay below 5e-7.  A wrong cross
#     term shows as ~1e-4 / sqrt(K) of absref, so it is the short reductions (K = 64 in the FC stack) that expose it.
#     The unpack kernel then sums the ksplit partials in fp32: + ksplit * 2^-24.
#   A 256-row tile sums the same k16 MMAs in the same order as a 128-row one: fwd1 holds for both tile heights.
# Measured worst c over every audited launch (NVIDIA H100 80GB HBM3, 700 W power limit) and bound / measured:
#   fwd1 5.2e-7 (conv_fwd <128,1> 128-row; 3.8x)   fwd2 1.36e-6 (conv_fwd <128,3>; 4.4x)
#   wgrad1 8.4e-6 (conv_wgrad <128,1>; 4.8x)   wgrad2 1.47e-5 (conv_wgrad <128,3>; 4.1x)
# per (op, variant, tile height, planes), with the single-pass "half" runs (train, epilogue statistics, folded eval at B = 64;
# Patch-PnP at B = 512):
#   conv_fwd       <128,1> 128-row 1: 5.19e-7 (fp32 out 3.89e-7)   <128,1> 256-row 1: 3.47e-7   <64,1> 1: 3.57e-7
#                  <128,3> 2: 1.36e-6 (fp32 out 4.07e-7)   <64,3> 2: 1.09e-6
#   gemm_fwd       <128,1> 128-row 1: 1.97e-8   <128,1> 256-row 1: 8.07e-8   <64,1> 1: 3.85e-7 (fp32 out 2.88e-7)
#                  <128,3> 2: 6.30e-7   <64,3> 2: 9.75e-7 (fp32 out 1.98e-7)
#   conv_dgrad_s2  <128,1> 1: 2.22e-7   <64,1> 1: 1.52e-7   <128,3> 2: 1.07e-6   <64,3> 2: 5.58e-7
# Audit wall time of the half runs on that card: train 1.0 s, epilogue statistics 0.4 s, folded eval 0.3 s, Patch-PnP 0.1 s.
BOUNDS = {"fwd1": 2e-6, "fwd2": 6e-6, "wgrad1": 4e-5, "wgrad2": 6e-5}
WGRAD_C0 = 2e-6  # the terms that do not grow with depth: dropped lo x lo (2^-22), the cross-term fma, 8x margin


def wgrad_bound(planes: int, blocks_per_split: int, bounds=None) -> float:
    return min((bounds or BOUNDS)[f"wgrad{planes}"], WGRAD_C0 + 4 * blocks_per_split * 2.0 ** -18)


# Epilogue BatchNorm statistics against float64 sums of the launch's OWN stored result (so the check isolates the reduction:
# fp32 sums over a warp's 16 rows, shared-memory atomics per tile, global atomics per CTA), relative to sum |y| and sum y^2
# of the channel.  When only a single-plane output exists, the epilogue sums the fp32 values that the store then rounds:
# each stored y differs by an unbiased error of at most u |y| (standard deviation <= u |y| / sqrt(3)), so the stored sums
# differ from the kernel's by noise of standard deviation u sqrt(sum y^2 / 3) and 2 u sqrt(sum y^4 / 3).  STATS_SIGMAS of
# it are taken off each channel's difference before it is compared with STATS_BOUND (stats_err).  A flat 4 u / sqrt(rows)
# is only 2 sigma of the sum of squares of a Gaussian channel, and the maximum over every channel of the half B = 64 forward
# exceeded it (2.03e-5 against 1.93e-5 on layer3.1.conv1).  A lost tile, warp or row of a channel moves its sums by more.
# Measured over the B = 64 atomic-statistics forwards and the synthetic column tails (NVIDIA H100 80GB HBM3, 700 W): <= 5.9e-7;
# the single-plane half forward leaves nothing beyond the rounding noise (0 on every channel).
STATS_BOUND = 4e-6
STATS_SIGMAS = 6.0
REPORT = {}  # key -> worst ratio seen in this session


# ------------------------------------------------------------------------------------------------ grid arithmetic (no GPU)
def pick_block_n(n_pad: int, num_m_tiles: int, sms: int) -> int:
    """Tile width of a forward / dgrad launch: pick_block_n, gemm_fwd.cu:493-498."""
    if n_pad % 64 != 0:
        return -1
    if n_pad % 128 == 0 and num_m_tiles * (n_pad // 128) >= (sms * 3) // 4:
        return 128
    if num_m_tiles * (n_pad // 128) < sms // 2:
        return 64
    return 128 if n_pad % 128 == 0 else 64


def pick_block_m(m_rows: int, n_pad: int, nsplit: int, plain: bool, sms: int) -> int:
    """Tile height of a forward launch: pick_block_m, gemm_fwd.cu:503-508.  256 rows (gemm_fwd_tall_kernel) for a single-pass
    launch that keeps the 128-wide tile (chosen from the 128-row tile count) and has a plain epilogue -- one TMA-stored 16-bit
    output plane; no fp32 output, BatchNorm statistics, residual, output-parity phases or weight groups -- while the 256-row
    tiles still fill 0.75 of a wave.  The phase dgrad (gdrn_conv_dgrad_s2) always runs 128-row tiles."""
    block_n = pick_block_n(n_pad, (m_rows + 127) // 128, sms)
    tall_tiles = (m_rows + 255) // 256 * (n_pad // block_n) if block_n > 0 else 0
    return 256 if nsplit == 1 and block_n == 128 and plain and tall_tiles >= (sms * 3) // 4 else 128


def fwd_grid(m_rows: int, n_pad: int, nphase: int, sms: int, block_m: int = 128) -> dict:
    """Tiles, groups and persistent CTAs of a forward / dgrad launch (launch_gemm, gemm_fwd.cu:412-415).  The width is
    picked from the 128-row tile count (the phase dgrad hands num_m_tiles * nphase to pick_block_n, :645), the tile list is
    then built from block_m-row tiles (set_block_m, :511-515).  max_per_cta tiles go to the first `remainder` CTAs (all, if 0)."""
    block_n = pick_block_n(n_pad, (m_rows + 127) // 128 * max(nphase, 1), sms)
    num_m = (m_rows + block_m - 1) // block_m
    num_n = n_pad // block_n
    groups = max(nphase, 1) * num_m * num_n
    ctas = min(groups, sms)
    ctas -= ctas % num_n
    if ctas <= 0:
        ctas = num_n
    return dict(block_n=block_n, block_m=block_m, num_m=num_m, num_n=num_n, groups=groups, ctas=ctas,
                max_per_cta=-(-groups // ctas), remainder=groups % ctas, nphase=nphase)


def a_box_images(Ho: int, Wo: int) -> int:
    """TN of a convolution's 128-row A box {64 ch, Wo, TH, TN} (conv_fwd_impl, gemm_fwd.cu:538-540): the images one box holds."""
    return 128 // (Wo * min(128 // Wo, Ho))


def tile_of(grid: dict, m_row: int, col: int, phase: int = 0) -> dict:
    """The tile that holds element (row m_row of the M axis, column col), its place in its CTA's walk over the tile list
    (group = phase * tiles + m_tile * num_n + n_tile, CTA = group % ctas, gemm_fwd.cu:256-264), and who wrote it inside the
    tile.  A 128-row tile is one A box; MMA warpgroup w owns its rows [64 w, 64 w + 64) (gemm_fwd.cu:237, :309).  A 256-row
    tile is two 128-row A boxes (the producer loads box b from image / row (n0[b], h0[b]), :153-164); warpgroup w multiplies
    box w (its A descriptor starts w * 16 KB in, :269) as two 64-row halves h (+ 8 KB each, :283-284)."""
    block_m = grid.get("block_m", 128)
    m_tile, n_tile = m_row // block_m, col // grid["block_n"]
    in_tile = m_row % block_m
    box, in_box = divmod(in_tile, 128)
    wg, half = (box, in_box // 64) if block_m == 256 else (in_box // 64, 0)
    grp = phase * grid["num_m"] * grid["num_n"] + m_tile * grid["num_n"] + n_tile
    return dict(m_tile=m_tile, n_tile=n_tile, phase=phase, box=box, warpgroup=wg, half=half, cta=grp % grid["ctas"],
                tiles_before=grp // grid["ctas"])


def wgrad_tile(ntot: int, nsplit: int, conv=None) -> int:
    """Column-tile width of a weight-gradient launch: pick_n_tile (gemm_wgrad.cu:292-297) and, for a convolution
    conv = (Cin, stride, KW), the tap-packed 192-wide tile of the 64-channel 3x3 layers (:334-335)."""
    if conv is not None and nsplit == 1 and conv[0] == 64 and conv[1] == 1 and conv[2] == 3:
        return 192
    if nsplit == 1 and ntot % 256 == 0:
        return 256
    if ntot % 128 == 0:
        return 128
    return 64 if ntot % 64 == 0 else -1


def choose_ksplit(base_items: int, kb_total: int, requested: int, sms: int) -> int:
    """choose_ksplit, gemm_wgrad.cu:304-314."""
    if requested > 0:
        return min(requested, kb_total)
    return max(1, min(sms // base_items, max(kb_total // 8, 1)))


def split_blocks(kb_total: int, ksplit: int) -> list:
    """k-blocks of each K-split (gemm_wgrad.cu:86-89); <= 0: an empty split, whose workspace rows are zeros."""
    kb_per = -(-kb_total // ksplit)
    return [min(kb_total, (s + 1) * kb_per) - s * kb_per for s in range(ksplit)]


def wgrad_shape(P: int, M: int, ntot: int, nsplit: int, requested: int, sms: int, conv=None, taps: int = 1) -> dict:
    """Tile width, base work items, K-split and per-split k-blocks of a weight-gradient launch (gdrn_conv_wgrad :334-348,
    gdrn_gemm_wgrad :389-401).  conv = (Cin, stride, KW), taps = KH * KW."""
    width = wgrad_tile(ntot, nsplit, conv)
    packed = width == 192
    items = (taps // conv[2] if packed else taps) if conv is not None else 1
    base = -(-M // 128) * (1 if packed else ntot // width) * items
    kb_total = -(-P // 64)
    ks = choose_ksplit(base, kb_total, requested, sms)
    return dict(width=width, base=base, kb_total=kb_total, ksplit=ks, blocks=split_blocks(kb_total, ks))


# ------------------------------------------------------------------------------------------------ packed layouts
# A packed operand is a [rows_pad][taps * ch_pad] K-major matrix (ops.pack_*, csrc/pack.cu).  Each decoder takes the matrix as
# a float tensor and returns the parameter it was packed from, in the parameter's own layout.
def decode_conv_fwd(p, O, I, KH, KW):
    """pack_conv_fwd: [Cout_pad][(r, s, ci)] -> OIHW."""
    return p.view(p.shape[0], KH, KW, -1).permute(0, 3, 1, 2)[:O, :I]


def decode_conv_dgrad(p, O, I, KH, KW):
    """pack_conv_dgrad: [Cin_pad][(flipped r, s, co)] -> OIHW."""
    return p.view(p.shape[0], KH, KW, -1).flip(1, 2).permute(3, 0, 1, 2)[:O, :I]


def decode_deconv_dgrad(p, I, O, KH, KW):
    """pack_deconv_dgrad: [Cin_pad][(r, s, co)] -> the ConvTranspose2d IOHW weight."""
    return p.view(p.shape[0], KH, KW, -1).permute(0, 3, 1, 2)[:I, :O]


def decode_stem(p):
    """pack_stem: [64][k = (r * 7 + s) * 3 + c, 147 of 192] -> [64][3][7][7]."""
    return p[:, :147].view(64, 7, 7, 3).permute(0, 3, 1, 2)


def decode_linear(p, N, K, nhwc_from=None, transpose=False):
    """pack_linear -> [N][K]; nhwc_from = (C, H, W): the packed K axis is (h, w, c), the parameter's (c, h, w)."""
    if nhwc_from is not None:
        Cc, H, W = nhwc_from
        if not transpose:
            return p[:N].view(N, H, W, Cc).permute(0, 3, 1, 2).reshape(N, K)
        return p.view(H, W, Cc, -1)[..., :N].permute(3, 2, 0, 1).reshape(N, K)
    return p.t()[:N, :K] if transpose else p[:N, :K]


def pt64(t) -> torch.Tensor:
    """The value a planar operand holds, in float64: hi + lo / lo_scale."""
    from gdr_net_b200 import ops

    x = t.buf[0].double()
    if t.planes == 2:
        x = x + t.buf[1].double() / ops.storage_format()[1]
    return x


# ------------------------------------------------------------------------------------------------ float64 references
def _nchw(x):
    return x.permute(0, 3, 1, 2)


def _finish(pre, absref, bias, res, act):
    """Epilogue of gemm_epilogue.cuh on the float64 accumulator: + bias, + residual, activation (1 LeakyReLU 0.1, 2 ReLU).
    Both activations are 1-Lipschitz, so absref bounds the propagated error unchanged."""
    if bias is not None:
        pre = pre + bias.detach().double()
        absref = absref + bias.detach().double().abs()
    if res is not None:
        pre = pre + res
        absref = absref + res.abs()
    if act == 1:
        pre = F.leaky_relu(pre, 0.1)
    elif act == 2:
        pre = torch.relu(pre)
    return pre, absref


def conv_ref(x, w, stride, pad, bias=None, res=None, act=0):
    """x NHWC, w OIHW (float64) -> (ref, absref) NHWC."""
    ref = F.conv2d(_nchw(x), w, None, stride=stride, padding=pad).permute(0, 2, 3, 1)
    absref = F.conv2d(_nchw(x.abs()), w.abs(), None, stride=stride, padding=pad).permute(0, 2, 3, 1)
    return _finish(ref, absref, bias, res, act)


def dgrad_s2_ref(du, w, K, pad, bias=None, act=0):
    """Data gradient of the stride-2 convolution with OIHW weight w from dY = du (NHWC): conv_transpose2d, output 2x."""
    kw = dict(stride=2, padding=pad, output_padding=1)
    ref = F.conv_transpose2d(_nchw(du), w, None, **kw).permute(0, 2, 3, 1)
    absref = F.conv_transpose2d(_nchw(du.abs()), w.abs(), None, **kw).permute(0, 2, 3, 1)
    return _finish(ref, absref, bias, None, act)


def gemm_ref(a, w, bias=None, act=0):
    """a [M][K], w [N][K] -> (ref, absref) [M][N]."""
    return _finish(a @ w.t(), a.abs() @ w.abs().t(), bias, None, act)


def conv_wgrad_ref(dy, x, KH, KW, stride, pad):
    """dy [N,Ho,Wo,Cout], x [N,H,W,Cin] (NHWC) -> (R, absR) in the workspace layout [Cout][(r, s, ci)]."""
    size = (dy.shape[-1], x.shape[-1], KH, KW)

    def one(d, xx):
        g = torch.nn.grad.conv2d_weight(_nchw(xx).contiguous(), size, _nchw(d).contiguous(), stride=stride, padding=pad)
        return g.permute(0, 2, 3, 1).reshape(size[0], -1)

    return one(dy, x), one(dy.abs(), x.abs())


def gemm_wgrad_ref(dy, x):
    return dy.t() @ x, dy.abs().t() @ x.abs()


def excess(got, ref, absref, u=0.0, tiny=0.0):
    """(worst c, flat index of it): the smallest c with |got - ref| <= c * absref + u * |ref| + tiny everywhere.  An element
    whose absref is zero (nothing was summed into it) must be matched exactly."""
    err = ((got.double() - ref).abs() - u * ref.abs() - tiny).clamp_min_(0.0)
    ratio = torch.where(absref > 0, err / absref.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
    ratio = torch.nan_to_num(ratio, nan=math.inf, posinf=math.inf)  # a NaN output (an element the kernel did not write) is infinitely wrong
    flat = ratio.reshape(-1)
    i = int(flat.argmax()) if flat.numel() else 0
    return (float(flat[i]) if flat.numel() else 0.0), i


def stats_err(stats, y, u: float = 0.0) -> float:
    """Epilogue statistics [2][C] against float64 sums of y [rows][C], relative to sum |y| and sum y^2, after STATS_SIGMAS
    standard deviations of the rounding noise of a stored single-plane y (unit roundoff u) are taken off each difference."""
    y2 = y * y
    noise0 = STATS_SIGMAS * u * (y2.sum(0) / 3).sqrt()
    noise1 = STATS_SIGMAS * 2 * u * ((y2 * y2).sum(0) / 3).sqrt()
    s0 = (((stats[0].double() - y.sum(0)).abs() - noise0).clamp_min(0) / y.abs().sum(0).clamp_min(1e-300)).max()
    s1 = (((stats[1].double() - y2.sum(0)).abs() - noise1).clamp_min(0) / y2.sum(0).clamp_min(1e-300)).max()
    return float(torch.maximum(s0, s1))


def out_tolerances(planes_out: int):
    """(u, tiny) of an output: single 16-bit plane, or two planes / fp32 (planes_out 0)."""
    from gdr_net_b200 import ops

    fi = torch.finfo(ops.storage_format()[0])
    sub = fi.smallest_normal * fi.eps  # smallest subnormal
    if planes_out == 1:
        return fi.eps / 2, sub / 2
    if planes_out == 2:
        return 0.0, sub / 2 / ops.storage_format()[1]
    return 0.0, 0.0


# ------------------------------------------------------------------------------------------------ the audit
class AuditFailure(AssertionError):
    pass


class Audit(contextlib.AbstractContextManager):
    """with Audit(label=...) as au: run the engine eagerly on ONE stream.  au.records holds one dict per audited launch;
    au.c_launches counts the launches of the five GEMM entry points seen at the C ABI (a call that reached the library
    without passing a wrapper shows as a difference).  nan_prefilled: the caller filled its outputs with NaN, so columns
    beyond the last written 32-column chunk must still be NaN."""

    OPS = ("conv_fwd", "gemm_fwd", "conv_dgrad_s2", "conv_wgrad", "gemm_wgrad", "unpack_wgrad")
    C_FNS = ("gdrn_conv_fwd", "gdrn_gemm_fwd", "gdrn_conv_dgrad_s2", "gdrn_conv_wgrad", "gdrn_gemm_wgrad")

    def __init__(self, label=None, nan_prefilled=False, bounds=None, guard_rows=0):
        from gdr_net_b200 import ops
        from gdr_net_b200.capi import C

        self.ops, self.C = ops, C
        self.sms = torch.cuda.get_device_properties(0).multi_processor_count
        self.label = label or (lambda wp: "?")
        self.nan_prefilled = nan_prefilled
        self.guard_rows = guard_rows
        self.bounds = dict(BOUNDS, **(bounds or {}))
        self.records, self.c_launches, self.pending = [], 0, None

    # -------------------------------------------------------------------------------------------- plumbing
    def __enter__(self):
        self._orig = {n: getattr(self.ops, n) for n in self.OPS}
        for n in self.OPS:
            setattr(self.ops, n, getattr(self, "_" + n))
        self._c_orig = {n: getattr(self.C, n) for n in self.C_FNS}
        for n, fn in self._c_orig.items():
            setattr(self.C, n, self._counted(n, fn))
        return self

    def __exit__(self, *exc):
        for n, fn in self._orig.items():
            setattr(self.ops, n, fn)
        for n, fn in self._c_orig.items():
            setattr(self.C, n, fn)
        self.pending = None
        return False

    def _counted(self, name, fn):
        ws_arg = 4 if name.endswith("wgrad") else None  # the weight-gradient entry points are also called as a size query

        def call(*a):
            if ws_arg is None or a[ws_arg] is not None:
                self.c_launches += 1
            return fn(*a)

        return call

    def n_audited(self):
        return sum(1 for r in self.records if r["op"] != "unpack_wgrad")

    def _note(self, key, value, bound, where):
        REPORT[key] = max(REPORT.get(key, 0.0), value)
        if not value <= bound:
            raise AuditFailure(f"{key}: {value:.3e} > bound {bound:.1e} at {where}")

    # -------------------------------------------------------------------------------------------- forward family
    def _grid(self, m_rows, n_pad, nphase, nsplit, out, out_f32, stats, res):
        """fwd_grid of a launch, on the tile height its own arguments select: a plain epilogue is one 16-bit output plane
        and no fp32 output, statistics, residual or phases (the audited entry points are never grouped)."""
        plain = out is not None and out.planes == 1 and out_f32 is None and stats is None and res is None and nphase == 0
        return fwd_grid(m_rows, n_pad, nphase, self.sms, pick_block_m(m_rows, n_pad, nsplit, plain, self.sms))

    def _fwd_common(self, op, x, wp, N, out, out_f32, ldc, stats, stats0, ref, absref, grid, locate, desc, nphase=0, geom=None,
                    bias=None):
        """ref / absref: [rows][N] float64 in the output's row order.  locate(row) -> (m_row, phase) of an output row.
        geom: (stride, KH, TN) of a convolution's A boxes."""
        dll = self.C.load()
        variant, block_m = int(dll.gdrn_last_gemm_variant()), int(dll.gdrn_last_gemm_block_m())
        planes = x.planes
        name = f"{op} {self.label(wp)} {desc} <{variant // 10},{variant % 10}> {block_m}-row tiles"
        assert variant == grid["block_n"] * 10 + x.nsplit, (name, grid)
        assert block_m == grid["block_m"], (name, grid)
        rows = ref.shape[0]
        stride, KH, TN = geom or (None, None, None)
        rec = dict(op=op, variant=variant, block_m=block_m, planes=planes, stats=stats is not None, nphase=nphase, name=name,
                   stride=stride, KH=KH, TN=TN, bias=bias is not None, **{k: grid[k] for k in ("groups", "ctas", "max_per_cta", "remainder")})
        self.records.append(rec)
        written = min(ldc, -(-N // 32) * 32)  # the epilogue writes whole 32-column chunks that start below N, up to ldc

        def where(i):
            r, c = divmod(i, N)
            m_row, ph = locate(r)
            t = tile_of(grid, m_row, c, ph)
            return (f"{name}: output row {r} col {c} = tile (m {t['m_tile']}, n {t['n_tile']}, phase {t['phase']}), 128-row box "
                    f"{t['box']}, warpgroup {t['warpgroup']}'s 64-row half {t['half']}, the CTA's tile #{t['tiles_before']} "
                    f"(CTA {t['cta']} of {grid['ctas']}, {grid['groups']} tiles)")

        key = f"{op} <{variant // 10},{variant % 10}> {block_m}-row planes{planes}"
        outs = []
        if out is not None:
            outs.append(("16-bit", pt64(out).reshape(-1, ldc), out.planes, out.buf.reshape(out.planes, -1, ldc)))
        if out_f32 is not None:
            o32 = out_f32.reshape(-1, ldc)
            outs.append(("fp32", o32.double(), 0, o32.unsqueeze(0)))
        assert outs, name
        basis, basis_u = None, 0.0  # the stored result the epilogue statistics are compared with: fp32 if there is one
        for kind, got, planes_out, raw in outs:
            u, tiny = out_tolerances(planes_out)
            basis, basis_u = got[:rows, :N], (u if planes_out == 1 else 0.0)
            c, i = excess(got[:rows, :N], ref, absref, u, tiny)
            self._note(key + (" fp32 out" if kind == "fp32" else ""), c, self.bounds[f"fwd{planes}"], where(i))
            if kind == "16-bit":
                assert bool(torch.isfinite(raw[:, :rows, :N]).all()), f"{name}: inf / NaN in the 16-bit output"
            assert bool((raw[:, :rows, N:written] == 0).all()), f"{name}: padding columns [{N}, {written}) of the {kind} output are not zero"
            if self.nan_prefilled:
                assert bool(torch.isnan(raw[:, :rows, written:]).all()), f"{name}: columns beyond {written} of the {kind} output were written"
                assert bool(torch.isnan(raw[:, rows:]).all()), f"{name}: rows beyond M = {rows} of the {kind} output were written"
        if stats is not None:
            got = (stats.reshape(-1)[:2 * N] - stats0.reshape(-1)[:2 * N]).view(2, N)
            self._note(f"{op} stats <{variant // 10},{variant % 10}> {block_m}-row planes{planes}", stats_err(got, basis, basis_u),
                       STATS_BOUND, name)
        return rec

    def _conv_fwd(self, x, wp, Cout, KH, KW, stride, pad, *, out=None, out_f32=None, bias=None, stats=None, act=0, ldc=None,
                  want_planes=True, algo_scale=1.0, res=None):
        stats0 = stats.clone() if stats is not None else None
        r = self._orig["conv_fwd"](x, wp, Cout, KH, KW, stride, pad, out=out, out_f32=out_f32, bias=bias, stats=stats, act=act,
                                   ldc=ldc, want_planes=want_planes, algo_scale=algo_scale, res=res)
        Nb, H, W, Cin = x.shape
        ldc = ldc or self.ops._round_up(Cout, 64)
        w = decode_conv_fwd(pt64(wp), Cout, Cin, KH, KW)
        ref, absref = conv_ref(pt64(x), w, stride, pad, bias, pt64(res)[..., :Cout] if res is not None else None, act)
        Ho, Wo = H // stride, W // stride
        grid = self._grid(Nb * Ho * Wo, wp.shape[0], 0, x.nsplit, r, out_f32, stats, res)
        desc = f"[{Nb}x{H}x{W}x{Cin} -> {Cout}, k{KH} s{stride} p{pad}, act {act}{', res' if res is not None else ''}]"
        self._fwd_common("conv_fwd", x, wp, Cout, r, out_f32, ldc, stats, stats0, ref.reshape(-1, Cout), absref.reshape(-1, Cout),
                         grid, lambda row: (row, 0), desc, geom=(stride, KH, a_box_images(Ho, Wo)), bias=bias)
        return r

    def _gemm_fwd(self, a, wp, N, *, out=None, out_f32=None, bias=None, stats=None, act=0, ldc=None, want_planes=True):
        stats0 = stats.clone() if stats is not None else None
        r = self._orig["gemm_fwd"](a, wp, N, out=out, out_f32=out_f32, bias=bias, stats=stats, act=act, ldc=ldc,
                                   want_planes=want_planes)
        M, K = a.shape
        ldc = ldc or self.ops._round_up(N, 64)
        ref, absref = gemm_ref(pt64(a), pt64(wp)[:N], bias, act)
        grid = self._grid(M, wp.shape[0], 0, a.nsplit, r, out_f32, stats, None)
        self._fwd_common("gemm_fwd", a, wp, N, r, out_f32, ldc, stats, stats0, ref, absref, grid, lambda row: (row, 0),
                         f"[{M}x{K} -> {N}, act {act}]", bias=bias)
        return r

    def _conv_dgrad_s2(self, du, wd, Cx, K, pad, *, out=None, bias=None, stats=None, act=0):
        stats0 = stats.clone() if stats is not None else None
        r = self._orig["conv_dgrad_s2"](du, wd, Cx, K, pad, out=out, bias=bias, stats=stats, act=act)
        Nb, Ho, Wo, Cy = du.shape
        ldc = self.ops._round_up(Cx, 64)
        w = decode_conv_dgrad(pt64(wd), Cy, Cx, K, K)  # [Cy][Cx][K][K]: the stride-2 conv's OIHW weight
        ref, absref = dgrad_s2_ref(pt64(du), w, K, pad, bias, act)
        nphase = 4 if K == 3 else 1
        grid = self._grid(Nb * Ho * Wo, wd.shape[0], nphase, du.nsplit, r, None, stats, None)

        def locate(row):  # output pixel (n, y, x) of the 2x larger dX -> row of the dY lattice and output-parity phase
            n, rem = divmod(row, 4 * Ho * Wo)
            y, xx = divmod(rem, 2 * Wo)
            ph = PHASE_ORDER.index((y & 1, xx & 1)) if K == 3 else 0
            return (n * Ho + (y >> 1)) * Wo + (xx >> 1), ph

        self._fwd_common("conv_dgrad_s2", du, wd, Cx, r, None, ldc, stats, stats0, ref.reshape(-1, Cx), absref.reshape(-1, Cx), grid,
                         locate, f"[{Nb}x{Ho}x{Wo}x{Cy} -> {Cx}, k{K}, act {act}]", nphase=nphase, geom=(1, K, a_box_images(Ho, Wo)),
                         bias=bias)
        return r

    # -------------------------------------------------------------------------------------------- weight gradients
    def _wgrad_common(self, op, dy, x, ret, ksplit_req, R, absR, shape, desc):
        buf, ks, kss = ret
        rows, krow = R.shape
        mpad = self.ops._round_up(rows, 128)
        assert kss == mpad * krow and ks == shape["ksplit"], (op, desc, ks, kss, shape)
        planes = x.planes
        width = shape["width"]
        name = f"{op} {desc} <{width},{x.nsplit}> ksplit {ks} of {shape['kb_total']} k-blocks"
        W = buf[:ks * kss].view(ks, mpad, krow)
        empty = [s for s, n in enumerate(shape["blocks"]) if n <= 0]
        for s in empty:
            assert bool((W[s] == 0).all()), f"{name}: the workspace of the empty split {s} is not zero"
        assert bool((W[:, rows:] == 0).all()), f"{name}: workspace rows beyond Cout = {rows} are not zero"
        total = W[:, :rows].double().sum(0)
        c, i = excess(total, R, absR)
        key = f"{op} <{width},{x.nsplit}> planes{planes}"
        bound = wgrad_bound(planes, max(shape["blocks"]), self.bounds)
        self._note(key + " split sum", c, bound, f"{name}: row {i // krow} col {i % krow}")
        self.records.append(dict(op=op, planes=planes, width=width, nsplit=x.nsplit, ksplit=ks, empty=len(empty),
                                 ragged=len(set(n for n in shape["blocks"] if n > 0)) > 1, blocks=shape["blocks"], name=name))
        self.pending = dict(ptr=buf.data_ptr(), ks=ks, kss=kss, R=R, absR=absR, key=key, name=name, bound=bound + ks * 2.0 ** -24)
        return ret

    def _conv_wgrad(self, dy, x, ws, Cout, KH, KW, stride, pad, ksplit=0):
        ret = self._orig["conv_wgrad"](dy, x, ws, Cout, KH, KW, stride, pad, ksplit)
        Nb, H, W, Cin = x.shape
        R, absR = conv_wgrad_ref(pt64(dy), pt64(x), KH, KW, stride, pad)
        shape = wgrad_shape(Nb * (H // stride) * (W // stride), dy.shape[-1], Cin, x.nsplit, ksplit, self.sms, (Cin, stride, KW), KH * KW)
        return self._wgrad_common("conv_wgrad", dy, x, ret, ksplit, R, absR, shape,
                                  f"[{Nb}x{H}x{W}x{Cin}, dY {dy.shape[-1]} ch, k{KH} s{stride} p{pad}]")

    def _gemm_wgrad(self, dy, x, ws, ksplit=0):
        ret = self._orig["gemm_wgrad"](dy, x, ws, ksplit)
        R, absR = gemm_wgrad_ref(pt64(dy), pt64(x))
        shape = wgrad_shape(dy.shape[0], dy.shape[1], x.shape[1], x.nsplit, ksplit, self.sms)
        return self._wgrad_common("gemm_wgrad", dy, x, ret, ksplit, R, absR, shape, f"[{dy.shape[0]} rows, {dy.shape[1]} x {x.shape[1]}]")

    def _unpack_wgrad(self, buf, grad, O, I, KH, KW, ipad, ksplit, ks_stride, so, si, sr, ss, flip=0, accumulate=0, krow=None):
        before = grad.clone() if accumulate else None
        self._orig["unpack_wgrad"](buf, grad, O, I, KH, KW, ipad, ksplit, ks_stride, so, si, sr, ss, flip, accumulate, krow)
        p = self.pending
        assert p is not None and ksplit == p["ks"] and ks_stride == p["kss"], "unpack_wgrad without the weight-gradient launch it reads"
        ws_krow = p["R"].shape[1]
        assert (krow or KH * KW * ipad) == ws_krow, (krow, KH, KW, ipad, ws_krow)
        row0, rem = divmod((buf.data_ptr() - p["ptr"]) // 4, ws_krow)  # fc_r | fc_t: two unpacks of one workspace
        assert rem == 0
        got = unpack_view(grad, O, I, KH, KW, so, si, sr, ss).double()
        if accumulate:
            got = got - unpack_view(before, O, I, KH, KW, so, si, sr, ss).double()
        exp, aexp = (workspace_as_param(m[row0:row0 + O], O, I, KH, KW, ipad, flip) for m in (p["R"], p["absR"]))
        c, i = excess(got, exp, aexp)
        self._note(p["key"] + " unpacked", c, p["bound"], f"{p['name']} -> unpack rows {row0}..{row0 + O}: element {i}")
        self.records.append(dict(op="unpack_wgrad", name=p["name"]))


def unpack_view(grad, O, I, KH, KW, so, si, sr, ss):
    """The gradient tensor as gdrn_unpack_wgrad addresses it: element (o, r, s, i) at o * so + i * si + r * sr + s * ss."""
    return torch.as_strided(grad, (O, KH, KW, I), (so, sr, ss, si), grad.storage_offset())


def workspace_as_param(rows, O, I, KH, KW, ipad, flip):
    """Workspace rows [O][(tap, ipad channels)...] -> [O][KH][KW][I], taps reversed when flip (pack.cu:152, :239)."""
    m = rows[:, :KH * KW * ipad].reshape(O, KH, KW, ipad)[..., :I]
    return m.flip(1, 2) if flip else m


# ------------------------------------------------------------------------------------------------ operands like the engine's
def relu_like(shape, gen, planes, scale=1.0):
    """A post-ReLU activation: half zeros, the rest half-normal."""
    from gdr_net_b200 import ops

    return ops.PT.from_float(torch.relu(torch.randn(shape, device="cuda", generator=gen)) * scale, planes)


def grad_like(shape, gen, planes, scale=1.0):
    from gdr_net_b200 import ops

    return ops.PT.from_float(torch.randn(shape, device="cuda", generator=gen) * scale, planes)


def row_scaled(shape, gen):
    """A weight whose output rows differ in scale over two decades (as BatchNorm-folded rows do)."""
    w = torch.randn(shape, device="cuda", generator=gen) / math.sqrt(math.prod(shape[1:]))
    s = 10.0 ** (torch.rand(shape[0], device="cuda", generator=gen) * 2 - 1)
    return w * s.view(-1, *([1] * (len(shape) - 1)))


def print_report():
    print("gemm audit, worst c per (op, variant, tile height, planes):")
    for k, v in sorted(REPORT.items()):
        print(f"  {k}: {v:.3e}")
