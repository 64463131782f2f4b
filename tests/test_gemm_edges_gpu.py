"""GPU: edge cases of the GEMM kernels that the engine's own shapes do not reach, with the references and the per-element error
measure of tests/gemm_audit.py.  Operands imitate the engine's (post-ReLU activations, weight rows spread over two decades);
every output the test allocates is pre-filled with NaN and carries guard rows, so an element the kernel skips or a write
outside its rows / 32-column chunks fails."""
import ctypes

import pytest
import torch

import gemm_audit as GA  # noqa: E402 (tests/ is on sys.path: rootdir conftest)
from loss_ref_common import nan_planes  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

GUARD = 8  # NaN rows behind the last output row


@pytest.fixture(scope="module", autouse=True)
def _setup():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    GA.print_report()


def _ops():
    from gdr_net_b200 import ops

    return ops


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------ weight gradients
# (planes, Ntot or None for the tap-packed conv) -> the six instantiated <N_TILE, NSPLIT>
WG_WIDTHS = {(256, 1): (1, 256), (192, 1): (1, None), (128, 1): (1, 128), (64, 1): (1, 192), (128, 3): (2, 256), (64, 3): (2, 64)}


def _wgrad_case(width, M, P, ksplit, seed):
    """One weight-gradient launch + unpack through the audit; returns the launch's record."""
    ops = _ops()
    planes, ntot = WG_WIDTHS[width]
    g = _gen(seed)
    with GA.Audit(label=lambda wp: "synthetic") as au:
        if ntot is None:  # 3x3 stride-1 conv over 64 channels: N x 16 x 16 pixels, 4 k-blocks per image
            assert P % 256 == 0
            x = GA.relu_like((P // 256, 16, 16, 64), g, planes)
            dy = GA.grad_like((P // 256, 16, 16, M), g, planes, scale=0.05)
            buf, ks, kss = ops.conv_wgrad(dy, x, ops.Workspace(), M, 3, 3, 1, 1, ksplit=ksplit)
            grad = torch.full((M, 64, 3, 3), float("nan"), device="cuda")
            ops.unpack_wgrad(buf, grad, M, 64, 3, 3, 64, ks, kss, 64 * 9, 9, 3, 1)
        else:
            x = GA.relu_like((P, ntot), g, planes)
            dy = GA.grad_like((P, M), g, planes, scale=0.05)
            buf, ks, kss = ops.gemm_wgrad(dy, x, ops.Workspace(), ksplit=ksplit)
            grad = torch.full((M, ntot), float("nan"), device="cuda")
            ops.unpack_wgrad(buf, grad, M, ntot, 1, 1, ntot, ks, kss, ntot, 1, 0, 0)
        torch.cuda.synchronize()
    rec = au.records[0]
    assert (rec["width"], rec["nsplit"]) == width, rec
    assert au.c_launches == 1 and bool(torch.isfinite(grad).all())
    return rec


@pytest.mark.parametrize("ksplit", [3, 8])
@pytest.mark.parametrize("width", list(WG_WIDTHS))
def test_wgrad_ragged_and_empty_splits(width, ksplit):
    """20 k-blocks over 3 splits (7, 7, 6: ragged) and over 8 (six of 3, one of 2, one EMPTY): the empty split's workspace
    rows are exact zeros (checked by the audit) and the unpacked gradient is right."""
    rec = _wgrad_case(width, 128, 1280, ksplit, seed=width[0] + ksplit)
    assert rec["ksplit"] == ksplit and rec["ragged"] and rec["empty"] == (1 if ksplit == 8 else 0), rec


def test_wgrad_chosen_ksplit_leaves_empty_splits():
    """2 base work items and 560 k-blocks: choose_ksplit takes 132 / 2 = 66 splits of 9 k-blocks, of which the last three
    get nothing."""
    rec = _wgrad_case((128, 3), 128, 560 * 64, 0, seed=5)  # Ntot 256 in two 128-wide tiles
    if _sms() == 132:
        assert rec["ksplit"] == 66 and rec["empty"] == 3 and rec["ragged"], rec


@pytest.mark.parametrize("P", [128, 256, 384, 1280, 1288])
@pytest.mark.parametrize("width", list(WG_WIDTHS))
def test_wgrad_pipeline_depths(width, P):
    """One split of 2, 4, 6 or 20 k-blocks: fewer than, as many as (4 stages at 256 wide, 6 at 64 wide) and more than the
    stages of the ring.  1288 rows: the last k-block is zero-filled beyond row 1288 (GEMM form only)."""
    if width == (192, 1) and P % 256:
        pytest.skip("the conv form reduces whole 64-pixel blocks")
    _wgrad_case(width, 128, P, 1, seed=P + width[0])


@pytest.mark.parametrize("M", [16, 64, 192])
@pytest.mark.parametrize("width", [(256, 1), (192, 1), (64, 3)])
def test_wgrad_row_tails(width, M):
    """Output rows that do not fill the 128-row tile: 64 and 192 channels, and the 9-row fc_r | fc_t gradient padded to 16
    (GEMM form; a convolution's dY has at least 64 channels)."""
    if width == (192, 1) and M == 16:
        pytest.skip("conv_wgrad needs Cout % 64 == 0")
    _wgrad_case(width, M, 1280, 4, seed=M + width[0])


# ------------------------------------------------------------------------------------------------ forward
def _guarded(rows, ldc, planes):
    return nan_planes((rows + GUARD, ldc), planes)


@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("tail", [1, 127, 129])
@pytest.mark.parametrize("N", [64, 128])
def test_gemm_fwd_row_tails_multi_tile(N, tail, planes):
    """140 full tiles + a last tile of 1 / 127 / (128 + 1) rows on 132 CTAs: the tail tile is some CTA's SECOND tile.
    K = 640: ten k-blocks, more than the ring has stages."""
    ops = _ops()
    M, K = 140 * 128 + tail, 640
    g = _gen(N + tail)
    a = GA.relu_like((M, K), g, planes)
    wp = ops.pack_linear(GA.row_scaled((N, K), g), planes)
    with GA.Audit(label=lambda w: "synthetic", nan_prefilled=True) as au:
        ops.gemm_fwd(a, wp, N, out=_guarded(M, N, planes))
        torch.cuda.synchronize()
    rec = au.records[0]
    assert rec["variant"] // 10 == N and (_sms() != 132 or (rec["max_per_cta"] == 2 and rec["remainder"] != 0)), rec


@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("N", [69, 96, 97])
def test_gemm_fwd_column_tails_all_outputs(N, planes):
    """N inside a 32-column chunk (69), at a chunk boundary (96) and one past it (97) on a 128-wide multi-tile launch with
    bias, LeakyReLU, epilogue statistics, the fp32 and the 16-bit output together."""
    ops = _ops()
    M, K = 140 * 128 + 127, 192
    g = _gen(N)
    a = GA.relu_like((M, K), g, planes)
    wp = ops.pack_linear(GA.row_scaled((N, K), g), planes)
    assert wp.shape[0] == 128
    bias = torch.randn(N, device="cuda", generator=g)
    stats = torch.zeros(2 * N, device="cuda")
    o32 = torch.full((M + GUARD, 128), float("nan"), device="cuda")
    with GA.Audit(label=lambda w: "synthetic", nan_prefilled=True) as au:
        ops.gemm_fwd(a, wp, N, out=_guarded(M, 128, planes), out_f32=o32, bias=bias, stats=stats, act=1, ldc=128)
        torch.cuda.synchronize()
    assert au.records[0]["variant"] // 10 == 128 and au.records[0]["stats"]


@pytest.mark.parametrize("planes", [1, 2])
def test_conv_fwd_residual_multi_tile(planes):
    """bias + residual (one and two planes) + ReLU on 128-wide tiles, 320 tiles on 132 CTAs."""
    ops = _ops()
    g = _gen(40 + planes)
    x = GA.relu_like((40, 32, 32, 128), g, planes)
    wp = ops.pack_conv_fwd(GA.row_scaled((128, 128, 3, 3), g), planes)
    bias = torch.randn(128, device="cuda", generator=g)
    res = GA.grad_like((40, 32, 32, 128), g, planes)
    out = nan_planes((40, 32, 32, 128), planes)
    with GA.Audit(label=lambda w: "synthetic", nan_prefilled=True) as au:
        ops.conv_fwd(x, wp, 128, 3, 3, 1, 1, out=out, bias=bias, act=2, res=res)
        torch.cuda.synchronize()
    rec = au.records[0]
    assert rec["variant"] // 10 == 128 and rec["groups"] == 320 and rec["max_per_cta"] > 1, rec


@pytest.mark.parametrize("planes", [1, 2])
def test_dgrad_s2_k1_multi_tile(planes):
    """The 1x1 stride-2 data gradient: ONE phase writes the even pixels of a caller-zeroed output, several tiles per CTA; the
    other three parities must stay exact zeros (their absref is zero)."""
    ops = _ops()
    g = _gen(50 + planes)
    du = GA.grad_like((40, 32, 32, 128), g, planes, scale=0.05)
    wd = ops.pack_conv_dgrad(GA.row_scaled((128, 64, 1, 1), g), planes)
    with GA.Audit(label=lambda w: "synthetic") as au:
        out = ops.conv_dgrad_s2(du, wd, 64, 1, 0)
        torch.cuda.synchronize()
    rec = au.records[0]
    assert rec["nphase"] == 1 and rec["groups"] == 320 and rec["max_per_cta"] > 1, rec
    assert bool((out.buf[:, :, 1::2] == 0).all()) and bool((out.buf[:, :, :, 1::2] == 0).all())


# ------------------------------------------------------------------------------------------------ argument rejection
def _rejected(fn, *args):
    from gdr_net_b200.capi import C, launch_count

    dll = C.load()
    n0 = launch_count()
    rc = getattr(dll, fn)(*args)
    assert launch_count() == n0, f"{fn} launched a kernel"
    return rc, dll.gdrn_last_error().decode()


def test_rejected_arguments():
    """Shapes the 32-bit epilogue offsets or the tiling cannot take are refused before anything is launched, with
    GDRN_ERR_ARG (-1) and a message that names the entry point and the argument.  The buffers are small dummies: a call that
    got past its checks would be caught by the launch counter, not by a fault."""
    d = torch.zeros(1 << 16, dtype=torch.float16, device="cuda")
    p = ctypes.c_void_p(d.data_ptr())
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    Z = None

    def conv(N=2, H=64, W=64, Cin=64, Cout=64, stride=1, ldc=64, nsplit=1, x_lo=None):
        return _rejected("gdrn_conv_fwd", p, x_lo, p, Z, p, Z, Z, Z, Z, Z, Z, N, H, W, Cin, Cout, 64, 3, 3, stride, 1, ldc, 0, nsplit, s)

    for rc_msg, want in ((conv(N=4096, Cout=256, ldc=256), "conv_fwd: output too large"),  # 4096 * 64 * 64 * 256 = 2^32 elements
                         (conv(W=48, H=48), "conv_fwd: unsupported output width 48"),
                         (conv(ldc=68), "conv_fwd: bad ldc=68"),
                         (conv(ldc=56), "conv_fwd: bad ldc=56"),
                         (conv(nsplit=3), "conv_fwd: lo planes missing"),
                         (conv(Cin=96), "conv_fwd: Cin=96")):
        assert rc_msg[0] == -1 and want in rc_msg[1], (rc_msg, want)

    def gemm(M=256, N=64, K=64, ldc=64, nsplit=1):
        return _rejected("gdrn_gemm_fwd", p, Z, p, Z, p, Z, Z, Z, Z, M, N, 64, K, ldc, 0, nsplit, s)

    for rc_msg, want in ((gemm(M=1 << 24, N=256, ldc=256), "gemm_fwd: output too large"), (gemm(ldc=68), "gemm_fwd: bad ldc=68"),
                         (gemm(nsplit=3), "gemm_fwd: lo planes missing"), (gemm(K=96), "gemm_fwd: K=96")):
        assert rc_msg[0] == -1 and want in rc_msg[1], (rc_msg, want)

    def dgrad(N=2, Ho=32, Wo=32, Cx=64, ldc=64, nsplit=1):
        return _rejected("gdrn_conv_dgrad_s2", p, Z, p, Z, p, Z, Z, Z, N, Ho, Wo, 64, Cx, 64, 3, 1, ldc, 0, nsplit, s)

    for rc_msg, want in ((dgrad(N=4096, Cx=256, ldc=256), "conv_dgrad_s2: output too large"),  # 4096 * 4 * 32 * 32 * 256 = 2^32
                         (dgrad(Wo=48, Ho=32), "conv_dgrad_s2: unsupported dY size 32x48"), (dgrad(ldc=68), "conv_dgrad_s2: bad ldc=68"),
                         (dgrad(nsplit=3), "conv_dgrad_s2: lo planes missing")):
        assert rc_msg[0] == -1 and want in rc_msg[1], (rc_msg, want)
    need, ks = ctypes.c_long(0), ctypes.c_int(0)
    rc, msg = _rejected("gdrn_gemm_wgrad", p, Z, p, Z, p, 1 << 30, ctypes.addressof(need), ctypes.addressof(ks), 256, 64, 64, 0, 3, s)
    assert rc == -1 and "gemm_wgrad: lo planes missing" in msg
    rc, msg = _rejected("gdrn_gemm_wgrad", p, Z, p, Z, p, 16, ctypes.addressof(need), ctypes.addressof(ks), 256, 64, 64, 0, 1, s)
    assert rc == -1 and "gemm_wgrad: workspace too small" in msg
    rc, msg = _rejected("gdrn_conv_wgrad", p, Z, p, Z, p, 1 << 30, ctypes.addressof(need), ctypes.addressof(ks), 2, 48, 48, 64, 64, 3, 3, 1, 1, 0, 1, s)
    assert rc == -1 and "conv_wgrad: unsupported output width 48" in msg
