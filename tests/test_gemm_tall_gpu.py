"""GPU: the 256-row forward GEMM tile (gemm_fwd_tall_kernel, pick_block_m in gemm_fwd.cu).

A large single-pass launch with a plain epilogue runs on 256-row tiles; recomputing its rows in slices small enough that the
same rule picks 128-row tiles must give the same bits, since every output element sums the same k16 MMAs in the same order.
The convolutions cover what the engine's launches do not isolate: stride 1 and 2 (the parity sub-lattice maps), 64..256
input channels and 32^2 / 16^2 / 8^2 outputs, the last with two images per 128-row A box (TN = 2).  The row tails of the
tall tile (rows of either warpgroup or of a 64-row half beyond M, several tiles per persistent CTA) are checked against
float64, as is every tall convolution."""
import pytest
import torch

import gemm_audit as GA  # noqa: E402 (tests/ is on sys.path: rootdir conftest)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

GUARD = 8  # NaN rows behind the last output row


@pytest.fixture(scope="module", autouse=True)
def _setup():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")


def _ops():
    from gdr_net_b200 import ops

    return ops


def _last():
    """(BLOCK_N * 10 + NSPLIT, tile height) of the last forward GEMM launch."""
    from gdr_net_b200.capi import C

    dll = C.load()
    return dll.gdrn_last_gemm_variant(), dll.gdrn_last_gemm_block_m()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _tiles_ok_for_128(rows, n_tiles):
    """True when a launch of `rows` rows and n_tiles 128-wide column tiles keeps the 128-wide tile and gets 128-row tiles."""
    thr = _sms() * 3 // 4
    return -(-rows // 128) * n_tiles >= thr and -(-rows // 256) * n_tiles < thr


def _nan_out(rows, ldc):
    ops = _ops()
    buf = torch.full((1, rows + GUARD, ldc), float("nan"), dtype=ops.storage_format()[0], device="cuda")
    return ops.PT((rows + GUARD, ldc), 1, buf=buf)


def _bits(pt):
    return pt.buf.view(torch.int16)


@pytest.mark.parametrize("N,ldc", [(256, 256), (128, 128), (200, 256)])
def test_gemm_tall_matches_128_row_tiles_bit_for_bit(N, ldc):
    """Plain GEMM (the head output-conv dgrad's kind of launch: K = 128) with bias and LeakyReLU; row slices of A on 128-row
    tiles.  N = 200 with ldc = 256: the zero-filled columns [200, 224) and the unwritten [224, 256) of both launches agree."""
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(100 + N)
    n_tiles = ops._round_up(N, 128) // 128
    step = next(r for r in range(128, 1 << 20, 128) if _tiles_ok_for_128(r, n_tiles))
    M, K = -(-64 * 1024 // step) * step, 128  # whole slices: a short last slice would change the tile width
    a = GA.grad_like((M, K), g, 1)
    wp = ops.pack_linear(GA.row_scaled((N, K), g), 1)
    bias = torch.randn(N, device="cuda", generator=g)
    big = _nan_out(M, ldc)
    ops.gemm_fwd(a, wp, N, out=big, bias=bias, act=1, ldc=ldc)
    assert _last() == (1281, 256)
    small = _nan_out(M, ldc)
    for r0 in range(0, M, step):
        r1 = min(M, r0 + step)
        a_s = ops.PT((r1 - r0, K), 1, buf=a.buf[:, r0:r1])
        o_s = ops.PT((r1 - r0, ldc), 1, buf=small.buf[:, r0:r1])
        ops.gemm_fwd(a_s, wp, N, out=o_s, bias=bias, act=1, ldc=ldc)
        assert _last() == (1281, 128)
    torch.cuda.synchronize()
    assert torch.equal(_bits(big), _bits(small))
    assert bool(torch.isnan(big.buf[:, M:]).all())


def _conv_close(x, wp, N, k, stride, bias, out, i0, i1):
    """Images [i0, i1) of a ReLU conv's output against the float64 reference, per element (tests/gemm_audit.py); returns the
    worst c and its (output row, column)."""
    Nb, H, W, cin = x.shape
    xs = _images(x, i0, i1)
    ref, absref = GA.conv_ref(GA.pt64(xs), GA.decode_conv_fwd(GA.pt64(wp), N, cin, k, k), stride, k // 2, bias, None, 2)
    per_img = ref[0].numel() // N
    got = GA.pt64(out).reshape(-1, out.shape[-1])[i0 * per_img:i1 * per_img, :N]
    u, tiny = GA.out_tolerances(1)
    c, i = GA.excess(got, ref.reshape(-1, N), absref.reshape(-1, N), u, tiny)
    return c, (i0 * per_img + i // N, i % N)


def _images(x, i0, i1):
    """Images [i0, i1) of an NHWC planar tensor, as a view."""
    return _ops().PT((i1 - i0,) + x.shape[1:], x.planes, buf=x.buf[:, i0:i1])


# (output side, Cout, k, stride, Cin): the head / layer2 dgrad kinds of launch (stride 1, Cin 128, 64^2 and 32^2), and every
# stride / Cin / output size the engine's tall forwards use, at Cout 128; layer3.0.conv1 / downsample (16^2, Cout 256)
CONV_CASES = ([(hw, N, k, 1, 128) for hw, N in ((64, 256), (64, 128), (32, 256), (32, 128)) for k in (1, 3)]
              + [(hw, 128, k, s, cin) for s in (1, 2) for cin in (64, 128, 256) for hw in (32, 16, 8) for k in (1, 3)
                 if (s, cin, hw) != (1, 128, 32)]
              + [(16, 256, k, 2, 128) for k in (1, 3)])


def _conv_id(case):
    hw, N, k, s, cin = case
    return f"{hw}-{N}-{k}" if (s, cin) == (1, 128) else f"{hw}-{N}-{k}-s{s}-cin{cin}"


@pytest.mark.parametrize("hw,N,k,stride,cin", CONV_CASES, ids=[_conv_id(c) for c in CONV_CASES])
def test_conv_tall_matches_128_row_tiles_bit_for_bit(hw, N, k, stride, cin):
    """Single-pass 1x1 / 3x3 convs with bias and ReLU on hw^2 outputs; batch slices on 128-row tiles, and the tall launch
    against float64.  8^2 outputs put two images in each 128-row A box."""
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(200 + hw + N + k + 7 * stride + cin)
    n_tiles = N // 128
    per_img = hw * hw
    bs = next(b for b in range(1, 1025) if _tiles_ok_for_128(b * per_img, n_tiles))
    B = next(b for b in range(bs, 1 << 14, bs) if b * per_img // 256 * n_tiles >= 2 * _sms())  # whole slices, >= 2 tall tiles per CTA
    H = hw * stride
    x = GA.relu_like((B, H, H, cin), g, 1)
    wp = ops.pack_conv_fwd(GA.row_scaled((N, cin, k, k), g), 1)
    bias = torch.randn(N, device="cuda", generator=g)
    big = ops.conv_fwd(x, wp, N, k, k, stride, k // 2, bias=bias, act=2)
    assert _last() == (1281, 256)
    small = ops.PT(big.shape, 1, zero=True)
    for i in range(0, B, bs):
        j = min(B, i + bs)
        ops.conv_fwd(_images(x, i, j), wp, N, k, k, stride, k // 2, out=_images(small, i, j), bias=bias, act=2)
        assert _last() == (1281, 128)
    torch.cuda.synchronize()
    assert torch.equal(_bits(big), _bits(small))
    for i0 in (0, B - bs):  # float64 on the first and the last slice (the bits above tie the rest to the 128-row tiles)
        c, where = _conv_close(x, wp, N, k, stride, bias, big, i0, i0 + bs)
        assert c <= GA.BOUNDS["fwd1"], (c, where)


# rows in the last 256-row tile: several full tiles per CTA plus a partial one; a tail inside warpgroup 1's first and second
# 64-row halves; warpgroup 1 without rows (and warpgroup 0's second half without rows); exactly 128 rows
TAILS = [("several_tiles_per_cta_and_remainder", None, 0), ("tail_in_wg1_first_half", 120, 150),
         ("tail_in_wg1_second_half", 120, 200), ("wg1_beyond_M", 120, 77), ("wg0_second_half_beyond_M", 120, 40),
         ("last_tile_exactly_128_rows", 120, 128)]


@pytest.mark.parametrize("name,full,last", TAILS, ids=[t[0] for t in TAILS])
def test_gemm_tall_row_tails_against_float64(name, full, last):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(300 + last)
    if full is None:
        full = 2 * _sms() + 37
    M, N, K, ldc = 256 * full + last, 128, 192, 128
    a = GA.grad_like((M, K), g, 1)
    wp = ops.pack_linear(GA.row_scaled((N, K), g), 1)
    bias = torch.randn(N, device="cuda", generator=g)
    out = _nan_out(M, ldc)
    ops.gemm_fwd(a, wp, N, out=out, bias=bias, act=1, ldc=ldc)
    assert _last() == (1281, 256)
    tall_tiles = -(-M // 256)
    if name.startswith("several"):
        assert tall_tiles > _sms() and tall_tiles % _sms() != 0
    torch.cuda.synchronize()
    ref, absref = GA.gemm_ref(GA.pt64(a), GA.pt64(wp)[:N], bias, 1)
    got = GA.pt64(out)[:M]
    u, tiny = GA.out_tolerances(1)
    c, i = GA.excess(got, ref, absref, u, tiny)
    assert c <= GA.BOUNDS["fwd1"], (name, c, divmod(i, N))
    assert bool(torch.isnan(out.buf[:, M:]).all()), "rows beyond M were written"


# 3x3 s2 over 16^2 -> 8^2 (Patch-PnP features.6): 64 rows per image, TN = 2 images per 128-row box, 4 per tall tile.  B % 4
# images in the last tall tile: 1 = it ends inside box 0's first half, 2 = box 1 wholly beyond M (its A boxes start at an
# image >= B and are zero-filled), 3 = box 1's second half beyond M
@pytest.mark.parametrize("last_images", [1, 2, 3])
def test_conv_s2_two_images_per_box_row_tails_against_float64(last_images):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(400 + last_images)
    B, N, cin = 4 * (2 * _sms() + 9) + last_images, 128, 128
    x = GA.relu_like((B, 16, 16, cin), g, 1)
    wp = ops.pack_conv_fwd(GA.row_scaled((N, cin, 3, 3), g), 1)
    bias = torch.randn(N, device="cuda", generator=g)
    M = B * 64
    out = _nan_out(M, N)
    ops.conv_fwd(x, wp, N, 3, 3, 2, 1, out=out, bias=bias, act=2)
    assert _last() == (1281, 256)
    assert -(-M // 256) % _sms() != 0
    torch.cuda.synchronize()
    c, where = _conv_close(x, wp, N, 3, 2, bias, out, 0, B)
    assert c <= GA.BOUNDS["fwd1"], (c, where)
    assert bool(torch.isnan(out.buf[:, M:]).all()), "rows beyond M were written"
