"""GPU: the 16-bit output planes of the TMA-store forward GEMM kernel (every launch with a 16-bit output but the phase dgrads,
gemm_fwd.cu make_out_maps) are exactly the split of the fp32 output of the same launch: hi = round(y),
lo = round((y - hi) * lo_scale), bit for bit.  Every output is pre-filled with NaN and carries guard rows and guard columns, so an
element written twice with different values, a skipped element or a write outside the rows / 32-column chunks of the output
fails."""
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


def _outputs(rows, ldc, planes):
    ops = _ops()
    dtype = ops.storage_format()[0]
    planes_buf = torch.full((planes, rows + GUARD, ldc), float("nan"), dtype=dtype, device="cuda")
    out = ops.PT((rows + GUARD, ldc), planes, buf=planes_buf)
    return out, torch.full((rows + GUARD, ldc), float("nan"), device="cuda")


def _check(out, o32, rows, N, planes):
    """The planes equal the split of the fp32 output on [rows][round_up(N, 32)] (zeros in [N, ...)); guards stay NaN."""
    ops = _ops()
    dtype, lo_scale, _ = ops.storage_format()
    width = min(o32.shape[1], (N + 31) // 32 * 32)
    y = o32[:rows, :width]
    assert bool(torch.isfinite(y).all())
    assert bool((y[:, N:] == 0).all())
    hi = y.to(dtype)
    got = out.buf[:, :rows, :width]
    assert torch.equal(got[0].view(torch.int16), hi.view(torch.int16))
    if planes == 2:
        lo = ((y - hi.float()) * lo_scale).to(dtype)
        assert torch.equal(got[1].view(torch.int16), lo.view(torch.int16))
    assert bool(torch.isnan(out.buf[:, rows:]).all()) and bool(torch.isnan(o32[rows:]).all())
    assert bool(torch.isnan(out.buf[:, :, width:]).all()) and bool(torch.isnan(o32[:, width:]).all())


def _last_variant():
    from gdr_net_b200.capi import C

    return C.load().gdrn_last_gemm_variant()


@pytest.mark.parametrize("planes", [1, 2])
def test_layer1_conv_planes_are_split_of_f32(planes):
    """A layer1 3x3 conv, 64 -> 64 channels at 64 x 64 (the <64, NSPLIT> tiles), with bias, ReLU and BatchNorm statistics;
    ldc = 128 leaves 64 guard columns behind the output."""
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(1 + planes)
    B = 16
    x = GA.relu_like((B, 64, 64, 64), g, planes)
    wp = ops.pack_conv_fwd(GA.row_scaled((64, 64, 3, 3), g), planes)
    bias = torch.randn(64, device="cuda", generator=g)
    stats = torch.zeros(2 * 64, device="cuda")
    M = B * 64 * 64
    out, o32 = _outputs(M, 128, planes)
    ops.conv_fwd(x, wp, 64, 3, 3, 1, 1, out=out, out_f32=o32, bias=bias, stats=stats, act=2, ldc=128)
    torch.cuda.synchronize()
    assert _last_variant() == 64 * 10 + (3 if planes == 2 else 1)
    _check(out, o32, M, 64, planes)


@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("k", [1, 3])
def test_head_conv_planes_are_split_of_f32(k, planes):
    """A 1x1 / 3x3 head conv, 256 -> 256 channels at 64 x 64 (the <128, NSPLIT> tiles, 4 / 36 k-blocks, several tiles per CTA;
    the 3-pass tile is staged in two 64-column halves), with bias and LeakyReLU."""
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(10 + planes)
    B = 8
    x = GA.relu_like((B, 64, 64, 256), g, planes)
    wp = ops.pack_conv_fwd(GA.row_scaled((256, 256, k, k), g), planes)
    bias = torch.randn(256, device="cuda", generator=g)
    M = B * 64 * 64
    out, o32 = _outputs(M, 256, planes)
    ops.conv_fwd(x, wp, 256, k, k, 1, k // 2, out=out, out_f32=o32, bias=bias, act=1)
    torch.cuda.synchronize()
    assert _last_variant() == 128 * 10 + (3 if planes == 2 else 1)
    _check(out, o32, M, 256, planes)


@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("N", [69, 128])
def test_gemm_row_and_column_tails(N, planes):
    """A plain GEMM whose last tile holds 127 rows and whose N ends inside a 32-column chunk (69): the TMA store clips both.
    K = 192 like the stem's im2col GEMM."""
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(20 + N + planes)
    M, K = 300 * 128 + 127, 192
    a = GA.relu_like((M, K), g, planes)
    wp = ops.pack_linear(GA.row_scaled((N, K), g), planes)
    out, o32 = _outputs(M, 128, planes)
    ops.gemm_fwd(a, wp, N, out=out, out_f32=o32, ldc=128)
    torch.cuda.synchronize()
    _check(out, o32, M, N, planes)
