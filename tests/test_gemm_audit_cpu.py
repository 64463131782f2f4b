"""CPU: the pieces of the GEMM launch audit (tests/gemm_audit.py) on their own, so that a failure of the GPU audit points at a
kernel and not at the harness: the packed-layout decoders against a plain restatement of the pack formula, the float64
references and their absref against independent formulations, the unpack addressing, and the tile / K-split arithmetic
against cases worked out by hand for 132 SMs."""
import math

import pytest
import torch
import torch.nn.functional as F

import gemm_audit as GA  # noqa: E402 (tests/ is on sys.path: rootdir conftest)


def _pack_ref(src, O, I, KH, KW, opad, ipad, krow, so, si, sr, ss, flip):
    """dst[o][tap * ipad + i] = src[o * so + i * si + r * sr + s * ss], (r, s) the tap, reversed when flip; zero elsewhere
    (the formula at the head of pack_weight_kernel, csrc/pack.cu:16)."""
    flat = src.reshape(-1)
    dst = torch.zeros(opad, krow, dtype=src.dtype)
    for tap in range(KH * KW):
        r, s = divmod(tap, KW)
        if flip:
            r, s = KH - 1 - r, KW - 1 - s
        idx = (torch.arange(O).view(-1, 1) * so + torch.arange(I).view(1, -1) * si + r * sr + s * ss)
        dst[:O, tap * ipad:tap * ipad + I] = flat[idx]
    return dst


def _recorded(fn):
    """The argument tuple an ops.pack_* call hands to the pack kernel, and that layout built by _pack_ref."""
    from gdr_net_b200 import ops

    ops._pack_recorder = []
    try:
        fn(ops)
        (job,) = ops._pack_recorder
    finally:
        ops._pack_recorder = None
    return _pack_ref(job[0].double(), *job[2:])


def _w(*shape):
    return torch.arange(1, math.prod(shape) + 1, dtype=torch.float32).view(shape)  # every element distinct


def test_decode_conv_layouts():
    w = _w(70, 69, 3, 3)
    assert torch.equal(GA.decode_conv_fwd(_recorded(lambda o: o.pack_conv_fwd(w, 1)), 70, 69, 3, 3), w.double())
    assert torch.equal(GA.decode_conv_dgrad(_recorded(lambda o: o.pack_conv_dgrad(w, 1)), 70, 69, 3, 3), w.double())
    # the head output conv's dgrad operand is packed 128 columns wide whatever its row count
    w1 = _w(69, 256, 1, 1)
    p = _recorded(lambda o: o.pack_conv_dgrad(w1, 1, ipad=128))
    assert p.shape == (256, 128) and torch.equal(GA.decode_conv_dgrad(p, 69, 256, 1, 1), w1.double())
    wt = _w(128, 70, 3, 3)  # ConvTranspose2d IOHW
    assert torch.equal(GA.decode_deconv_dgrad(_recorded(lambda o: o.pack_deconv_dgrad(wt, 1)), 128, 70, 3, 3), wt.double())
    # the ConvTranspose2d forward operand is pack_conv_dgrad of the IOHW weight read as OIHW
    assert torch.equal(GA.decode_conv_dgrad(_recorded(lambda o: o.pack_conv_dgrad(wt, 1)), 128, 70, 3, 3), wt.double())
    ws = _w(64, 3, 7, 7)
    ps = _recorded(lambda o: o.pack_stem(ws, 1))
    assert ps.shape == (64, 192) and bool((ps[:, 147:] == 0).all())
    assert torch.equal(GA.decode_stem(ps), ws.double())


def test_decode_linear_layouts():
    w = _w(9, 256)
    assert torch.equal(GA.decode_linear(_recorded(lambda o: o.pack_linear(w, 1)), 9, 256), w.double())
    assert torch.equal(GA.decode_linear(_recorded(lambda o: o.pack_linear(w, 1, transpose=True)), 9, 256, transpose=True), w.double())
    w1 = _w(64, 8192)
    nf = (128, 8, 8)
    assert torch.equal(GA.decode_linear(_recorded(lambda o: o.pack_linear(w1, 1, nhwc_from=nf)), 64, 8192, nhwc_from=nf), w1.double())
    pt = _recorded(lambda o: o.pack_linear(w1, 1, nhwc_from=nf, transpose=True))
    assert torch.equal(GA.decode_linear(pt, 64, 8192, nhwc_from=nf, transpose=True), w1.double())
    # the packed K axis really is the NHWC flatten: column (h, w, c) of row n is w1[n][c][h][w]
    assert float(_recorded(lambda o: o.pack_linear(w1, 1, nhwc_from=nf))[5, (3 * 8 + 2) * 128 + 7]) == float(w1.view(64, 128, 8, 8)[5, 7, 3, 2])


@pytest.mark.parametrize("stride,pad,k", [(1, 1, 3), (2, 1, 3), (2, 0, 1)])
def test_conv_ref_and_absref(stride, pad, k):
    g = torch.Generator().manual_seed(k + stride)
    x = torch.randn(2, 8, 8, 5, dtype=torch.float64, generator=g)
    w = torch.randn(7, 5, k, k, dtype=torch.float64, generator=g)
    bias = torch.randn(7, generator=g)
    res = torch.randn(2, 8 // stride, 8 // stride, 7, dtype=torch.float64, generator=g)
    ref, absref = GA.conv_ref(x, w, stride, pad, bias, res, act=2)
    # independent formulation: im2col (F.unfold) and one matrix product
    cols = F.unfold(x.permute(0, 3, 1, 2), k, padding=pad, stride=stride)  # [N][Cin * k * k][L]
    pre = (w.view(7, -1) @ cols).permute(0, 2, 1).reshape(ref.shape) + bias.double() + res
    assert torch.allclose(ref, torch.relu(pre), rtol=0, atol=1e-12)
    ab = (w.abs().view(7, -1) @ cols.abs()).permute(0, 2, 1).reshape(ref.shape) + bias.double().abs() + res.abs()
    assert torch.allclose(absref, ab, rtol=0, atol=1e-12)
    assert bool((absref + 1e-12 >= ref.abs()).all())
    lk, _ = GA.conv_ref(x, w, stride, pad, None, None, act=1)
    p0, _ = GA.conv_ref(x, w, stride, pad, None, None, act=0)
    assert torch.equal(lk, torch.where(p0 > 0, p0, 0.1 * p0))


@pytest.mark.parametrize("k,pad", [(3, 1), (1, 0)])
def test_dgrad_and_wgrad_refs_are_the_conv_gradients(k, pad):
    g = torch.Generator().manual_seed(k)
    x = torch.randn(2, 8, 8, 6, dtype=torch.float64, generator=g, requires_grad=True)
    w = torch.randn(4, 6, k, k, dtype=torch.float64, generator=g, requires_grad=True)
    dy = torch.randn(2, 4, 4, 4, dtype=torch.float64, generator=g)
    y = F.conv2d(x.permute(0, 3, 1, 2), w, None, stride=2, padding=pad)
    gx, gw = torch.autograd.grad(y, (x, w), dy.permute(0, 3, 1, 2))
    ref, absref = GA.dgrad_s2_ref(dy, w.detach(), k, pad)
    assert torch.allclose(ref, gx, rtol=0, atol=1e-12) and bool((absref + 1e-12 >= ref.abs()).all())
    if k == 1:  # only the even pixels receive anything: the other three parities are exact zeros with absref 0
        assert bool((absref[:, 1::2] == 0).all()) and bool((absref[:, :, 1::2] == 0).all())
    R, absR = GA.conv_wgrad_ref(dy, x.detach(), k, k, 2, pad)
    assert torch.allclose(R, gw.permute(0, 2, 3, 1).reshape(4, -1), rtol=0, atol=1e-12)
    assert bool((absR + 1e-12 >= R.abs()).all())
    a, b = torch.randn(10, 4, dtype=torch.float64, generator=g), torch.randn(10, 6, dtype=torch.float64, generator=g)
    assert torch.allclose(GA.gemm_wgrad_ref(a, b)[0], a.t() @ b)


def test_unpack_addressing():
    """The (so, si, sr, ss) the engine passes to unpack_wgrad, as views of the parameter layouts."""
    R = _w(8, 9 * 64).double()  # a conv workspace [Cout 8][(r, s, ci 64)], 40 of 64 channels valid
    grad = torch.zeros(8, 40, 3, 3)
    view = GA.unpack_view(grad, 8, 40, 3, 3, 40 * 9, 9, 3, 1)
    view.copy_(GA.workspace_as_param(R, 8, 40, 3, 3, 64, 0))
    assert float(grad[5, 7, 2, 1]) == float(R[5, (2 * 3 + 1) * 64 + 7])
    view.copy_(GA.workspace_as_param(R, 8, 40, 3, 3, 64, 1))
    assert float(grad[5, 7, 2, 1]) == float(R[5, (0 * 3 + 1) * 64 + 7])
    Rs = _w(64, 192).double()  # stem: k = (r * 7 + s) * 3 + c, row length 192
    gs = torch.zeros(64, 3, 7, 7)
    GA.unpack_view(gs, 64, 3, 7, 7, 147, 49, 7, 1).copy_(GA.workspace_as_param(Rs, 64, 3, 7, 7, 3, 0))
    assert float(gs[9, 2, 4, 6]) == float(Rs[9, (4 * 7 + 6) * 3 + 2])
    Rf = _w(4, 8192).double()  # fc1: workspace columns (h, w, c), parameter columns (c, h, w)
    gf = torch.zeros(4, 8192)
    GA.unpack_view(gf, 4, 128, 8, 8, 8192, 64, 8, 1).copy_(GA.workspace_as_param(Rf, 4, 128, 8, 8, 128, 0))
    assert float(gf.view(4, 128, 8, 8)[3, 77, 5, 2]) == float(Rf[3, (5 * 8 + 2) * 128 + 77])


def test_excess_measure():
    ref = torch.tensor([1.0, -2.0, 0.0, 4.0], dtype=torch.float64)
    absref = torch.tensor([2.0, 2.0, 0.0, 8.0], dtype=torch.float64)
    assert GA.excess(ref.float(), ref, absref) == (0.0, 0)
    c, i = GA.excess(torch.tensor([1.0, -2.0, 0.0, 4.5]), ref, absref)
    assert i == 3 and c == pytest.approx(0.5 / 8.0)
    c, i = GA.excess(torch.tensor([1.0, -2.0, 0.0, 4.5]), ref, absref, u=0.125)  # the storage rounding is not charged to c
    assert c == 0.0
    assert GA.excess(torch.tensor([1.0, -2.0, 1e-30, 4.0]), ref, absref) == (math.inf, 2)  # nothing was summed: exact zero
    assert GA.excess(torch.tensor([1.0, float("nan"), 0.0, 4.0]), ref, absref) == (math.inf, 1)  # an unwritten element


def test_stats_err_takes_off_the_storage_rounding_only():
    """Sums of fp32 values against the fp16-stored values: the rounding noise of the store is not charged, a row missing
    from one channel's sums still is."""
    g = torch.Generator().manual_seed(3)
    f = torch.randn(16384, 256, generator=g) * torch.linspace(0.01, 10.0, 256)  # a pre-BatchNorm output, channel scales apart
    f[:, 7] = torch.relu(f[:, 7]) ** 3  # a heavy-tailed channel
    stats = torch.stack([f.double().sum(0), (f.double() ** 2).sum(0)]).float()  # what the epilogue sums (fp32 here)
    y = f.half().double()  # what the store kept
    u = torch.finfo(torch.float16).eps / 2
    assert GA.stats_err(stats, y) > GA.STATS_BOUND  # the rounding alone exceeds the bound when it is charged
    assert GA.stats_err(stats, y, u) < GA.STATS_BOUND / 4
    # one row of median magnitude of a Gaussian channel; of the heavy-tailed channel one of its top 3 %, whose sums of squares
    # are dominated, and their rounding noise set, by a few rows
    for col, rank in ((100, 8192), (7, 16000)):
        row = int(f[:, col].abs().argsort()[rank])
        bad = stats.clone()
        bad[0, col] -= f[row, col]
        bad[1, col] -= f[row, col] ** 2
        assert GA.stats_err(bad, y, u) > GA.STATS_BOUND, col


def test_tile_width_choice():
    assert GA.pick_block_n(128, 64, 132) == 64     # 2 x 64 x 64 pixels, 128 channels: 64 tiles, below half a wave
    assert GA.pick_block_n(256, 2048, 132) == 128  # the 64 x 64 x 256 head layers at B = 64
    assert GA.pick_block_n(128, 99, 132) == 128 and GA.pick_block_n(128, 98, 132) == 128  # >= 0.75 waves / the middle branch
    assert GA.pick_block_n(256, 40, 132) == 128    # layer3 at B = 20: 80 wide tiles, between half and 0.75 waves
    assert GA.pick_block_n(128, 65, 132) == 64 and GA.pick_block_n(128, 66, 132) == 128
    assert GA.pick_block_n(64, 8192, 132) == 64 and GA.pick_block_n(192, 100, 132) == 64 and GA.pick_block_n(96, 1, 132) == -1


def test_persistent_grid():
    g = GA.fwd_grid(64 * 128 * 128, 64, 0, 132)  # the stem at B = 64
    assert (g["block_n"], g["groups"], g["ctas"], g["max_per_cta"], g["remainder"]) == (64, 8192, 132, 63, 8)
    g = GA.fwd_grid(3 * 128, 256, 0, 132)  # 3 m-tiles x 4 narrow n-tiles: one CTA each
    assert (g["block_n"], g["groups"], g["ctas"], g["max_per_cta"], g["remainder"]) == (64, 12, 12, 1, 0)
    g = GA.fwd_grid(25 * 128, 1024, 0, 132)  # 8 n-tiles: 132 -> 128 CTAs so that every CTA keeps one n-tile
    assert (g["block_n"], g["num_n"], g["groups"], g["ctas"], g["remainder"]) == (128, 8, 200, 128, 72)
    g = GA.fwd_grid(64 * 32 * 32, 64, 4, 132)  # layer2.0.conv1's stride-2 dgrad at B = 64: 4 phases x 512 tiles
    assert (g["block_n"], g["groups"], g["ctas"], g["max_per_cta"], g["remainder"]) == (64, 2048, 132, 16, 68)
    t = GA.tile_of(g, 130, 5, phase=2)  # group 2 * 512 + 1 = 1025 -> CTA 1025 % 132 = 101, its 8th tile
    assert t == dict(m_tile=1, n_tile=0, phase=2, box=0, warpgroup=0, half=0, cta=101, tiles_before=7)
    g = GA.fwd_grid(512 * 128, 128, 0, 132)
    assert GA.tile_of(g, 128 * 200 + 3, 100) == dict(m_tile=200, n_tile=0, phase=0, box=0, warpgroup=0, half=0, cta=68, tiles_before=1)
    assert GA.tile_of(g, 128 * 3 + 70, 0) == dict(m_tile=3, n_tile=0, phase=0, box=0, warpgroup=1, half=0, cta=3, tiles_before=0)


def test_tile_height_choice():
    """pick_block_m at 132 SMs: 256-row tiles need nsplit 1, the 128-wide tile, a plain epilogue and ceil(M / 256) * n-tiles
    >= 99."""
    l2c1 = 64 * 32 * 32  # layer2.0.conv1 at B = 64 (3x3 s2, 64 -> 128): 512 128-row tiles, 256 tall ones
    assert GA.pick_block_m(l2c1, 128, 1, True, 132) == 256
    assert GA.pick_block_m(l2c1, 128, 1, False, 132) == 128  # the same launch with epilogue statistics (or a residual, ...)
    assert GA.pick_block_m(l2c1, 128, 3, True, 132) == 128   # 3-pass
    assert GA.pick_block_m(64 * 8 * 8, 512, 1, True, 132) == 128  # layer4: 32 x 4 128-wide tiles, only 16 x 4 = 64 tall ones
    assert GA.pick_block_m(64 * 16 * 16, 256, 1, True, 132) == 256  # layer3.0.conv1: 64 x 2 = 128 tall tiles
    assert GA.pick_block_m(99 * 256, 128, 1, True, 132) == 256 and GA.pick_block_m(98 * 256, 128, 1, True, 132) == 128
    assert GA.pick_block_m(98 * 256 + 1, 128, 1, True, 132) == 256  # a partial last tall tile counts
    assert GA.pick_block_m(64 * 64 * 64, 64, 1, True, 132) == 128  # layer1: 64 wide
    g = GA.fwd_grid(l2c1, 128, 0, 132, block_m=256)
    assert (g["block_n"], g["num_m"], g["groups"], g["ctas"], g["max_per_cta"], g["remainder"]) == (128, 256, 256, 132, 2, 124)
    g = GA.fwd_grid(l2c1, 128, 0, 132)
    assert (g["block_m"], g["num_m"], g["groups"], g["max_per_cta"], g["remainder"]) == (128, 512, 512, 4, 116)


def test_tall_tiles_with_two_images_per_box():
    """Patch-PnP features.6 at B = 512 (3x3 s2, 16^2 -> 8^2, 128 -> 128): one 128-row A box holds TN = 2 images of 8 x 8 rows, a
    tall tile 4 images; 128 tall tiles, one per CTA."""
    M = 512 * 8 * 8
    assert GA.a_box_images(8, 8) == 2 and GA.a_box_images(16, 16) == 1 and GA.a_box_images(32, 32) == 1 and GA.a_box_images(4, 4) == 8
    assert GA.pick_block_m(M, 128, 1, True, 132) == 256
    g = GA.fwd_grid(M, 128, 0, 132, block_m=256)
    assert (g["block_n"], g["num_m"], g["groups"], g["ctas"], g["max_per_cta"], g["remainder"]) == (128, 128, 128, 128, 1, 0)
    # image 22 = row 1408 + 3 * 8 + 1: tall tile 5 (images 20..23), box 1 (images 22, 23) of warpgroup 1, its first 64-row half
    assert GA.tile_of(g, 22 * 64 + 3 * 8 + 1, 7) == dict(m_tile=5, n_tile=0, phase=0, box=1, warpgroup=1, half=0, cta=5, tiles_before=0)
    # image 21, last row: box 0, second half of warpgroup 0
    assert GA.tile_of(g, 22 * 64 - 1, 7) == dict(m_tile=5, n_tile=0, phase=0, box=0, warpgroup=0, half=1, cta=5, tiles_before=0)
    # layer2.0.conv1's tall grid: row 200 of tall tile 200 = box 1, half 1; group 200 is CTA 68's second tile
    g = GA.fwd_grid(64 * 32 * 32, 128, 0, 132, block_m=256)
    assert GA.tile_of(g, 256 * 200 + 200, 127) == dict(m_tile=200, n_tile=0, phase=0, box=1, warpgroup=1, half=1, cta=68, tiles_before=1)


def test_wgrad_tiles_and_ksplit():
    assert GA.wgrad_tile(64, 1, (64, 1, 3)) == 192 and GA.wgrad_tile(64, 3, (64, 1, 3)) == 64 and GA.wgrad_tile(64, 1, (64, 2, 1)) == 64
    assert GA.wgrad_tile(512, 1) == 256 and GA.wgrad_tile(512, 3) == 128 and GA.wgrad_tile(128, 1) == 128 and GA.wgrad_tile(192, 1) == 64
    assert GA.split_blocks(20, 8) == [3, 3, 3, 3, 3, 3, 2, -1] and GA.split_blocks(20, 3) == [7, 7, 6]
    assert GA.choose_ksplit(2, 560, 0, 132) == 66  # 9 k-blocks per split: 62 full, one of 2, splits 63..65 empty
    b = GA.split_blocks(560, 66)
    assert b[61:] == [9, 2, -7, -16, -25] and sum(n for n in b if n > 0) == 560
    assert GA.choose_ksplit(72, 64, 0, 132) == 1 and GA.choose_ksplit(3, 16384, 0, 132) == 44 and GA.choose_ksplit(1, 20, 8, 132) == 8
    s = GA.wgrad_shape(35840, 128, 512, 1, 0, 132)
    assert (s["width"], s["base"], s["kb_total"], s["ksplit"]) == (256, 2, 560, 66)
    s = GA.wgrad_shape(64 * 64 * 64, 64, 64, 1, 0, 132, conv=(64, 1, 3), taps=9)  # layer1 3x3 at B = 64: three filter rows
    assert (s["width"], s["base"], s["kb_total"], s["ksplit"]) == (192, 3, 4096, 44)
