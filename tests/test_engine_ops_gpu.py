"""GPU: the BatchNorm kernels (csrc/elementwise.cu), the small backward kernels, the weight-gradient layouts and the forward
epilogue variants exactly as Engine calls them, against float64 references built from the kernels' exact inputs.

Each engine call is copied with its argument list and the engine.py line it comes from.  Bounds: fp32 rounding for
two-plane outputs, plus one unit roundoff of the 16-bit storage format for single-plane outputs; each bound is derived at
its definition and the worst error measured on an H100 (80 GB HBM3) is recorded next to it."""
import pytest
import torch
import torch.nn.functional as F

from loss_ref_common import REPORT, check, nan_planes, rel_err, unit_roundoff  # noqa: E402 (tests/ is on sys.path: rootdir conftest)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]


@pytest.fixture(scope="module", autouse=True)
def _setup():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    print("worst errors:", {k: f"{v:.2e}" for k, v in sorted(REPORT.items())})


def _ops():
    from gdr_net_b200 import ops

    return ops


def _C():
    from gdr_net_b200.capi import C

    return C


def _s():
    return torch.cuda.current_stream().cuda_stream


def tol_for(planes: int, fp32: float) -> float:
    return fp32 if planes == 2 else unit_roundoff() + fp32


def _operand(x, planes):
    """What a packed weight / planar operand holds: the value rounded to the storage format (planes 1), or hi + lo, which is the
    fp32 value to ~2^-22 (planes 2)."""
    return _ops().round_storage(x) if planes == 1 else x


def _det_ws():
    return torch.empty(2 * 512 * int(_C().load().gdrn_det_parts()), device="cuda")  # Engine._det_workspace (engine.py:415)


def _bits(mask, rows, C_):
    return ((mask.view(-1, 1) >> torch.arange(8, device="cuda", dtype=torch.uint8)) & 1).view(rows, C_)


# ------------------------------------------------------------------------------------------------ B. BatchNorm
def _bn_inputs(rows, C_, seed, ratio=1.0):
    """Pre-BN tensor with per-channel std in [0.5, 2] and |mean| / std up to `ratio`."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    sd = torch.rand(C_, device="cuda", generator=g) * 1.5 + 0.5
    mu = (torch.rand(C_, device="cuda", generator=g) * 2 - 1) * ratio * sd
    u = torch.randn(rows, C_, device="cuda", generator=g) * sd + mu
    res = torch.randn(rows, C_, device="cuda", generator=g)
    gamma = torch.rand(C_, device="cuda", generator=g) + 0.5
    beta = torch.randn(C_, device="cuda", generator=g) * 0.3
    rm = torch.randn(C_, device="cuda", generator=g) * 0.1
    rv = torch.rand(C_, device="cuda", generator=g) + 0.5
    return u, res, gamma, beta, rm, rv


def _bn_stats(U, rows, C_, ws=None):
    stats = torch.full((2, C_), float("nan"), device="cuda")
    _C().gdrn_bn_stats(U.hi_ptr, U.lo_ptr, (ws if ws is not None else _det_ws()).data_ptr(), stats.data_ptr(), rows, C_, _s())  # :401
    return stats


def _bn_fwd(U, R, stats, gamma, beta, rm, rv, rows, C_, train, relu, planes):
    Y = nan_planes((rows, C_), planes)
    mean = torch.full((C_,), float("nan"), device="cuda")
    invstd = torch.full((C_,), float("nan"), device="cuda")
    mask = torch.zeros(rows * C_ // 8, dtype=torch.uint8, device="cuda") if relu else None
    _C().gdrn_bn_fwd(U.hi_ptr, U.lo_ptr, R.hi_ptr if R else None, R.lo_ptr if R else None, Y.hi_ptr, Y.lo_ptr,  # engine.py:407-410
                     stats.data_ptr() if train else None, gamma.data_ptr(), beta.data_ptr(), rm.data_ptr(), rv.data_ptr(),
                     mean.data_ptr(), invstd.data_ptr(), mask.data_ptr() if mask is not None else None, rows, C_, 1e-5, 0.1,
                     int(train), int(relu), _s())
    return Y, mean, invstd, mask


# rows: 192 is not a multiple of any block tiling; 65536 = 4 * 128 * 128 is the stem's BatchNorm at B = 4
BN_SHAPES = [(192, 64), (192, 512), (1024, 256), (2048, 128), (65536, 64)]


@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("train", [1, 0])
@pytest.mark.parametrize("rows,C_", BN_SHAPES)
def test_bn_fwd(rows, C_, train, planes):
    """gdrn_bn_fwd fed by gdrn_bn_stats (the engine's default, deterministic statistics) against float64 F.batch_norm."""
    ops = _ops()
    u, res, gamma, beta, rm, rv = _bn_inputs(rows, C_, seed=rows + C_ + train)
    U, R = ops.PT.from_float(u, planes), ops.PT.from_float(res, planes)
    uf, rf = U.float().double(), R.float().double()
    stats = _bn_stats(U, rows, C_) if train else None
    if train:
        m64, v64 = uf.mean(0), uf.var(0, unbiased=False)
    else:
        m64, v64 = rm.double(), rv.double()
    is64 = 1.0 / torch.sqrt(v64 + 1e-5)
    for relu, with_res in ((1, 0), (1, 1), (0, 0), (0, 1)):
        rm_k, rv_k = rm.clone(), rv.clone()
        Y, mean, invstd, mask = _bn_fwd(U, R if with_res else None, stats, gamma, beta, rm_k, rv_k, rows, C_, train, relu, planes)
        torch.cuda.synchronize()
        tag = f"[{rows}x{C_},t{train},r{relu},res{with_res},{planes}]"
        pre = (uf - m64) * is64 * gamma.double() + beta.double() + (rf if with_res else 0.0)
        ref = torch.relu(pre) if relu else pre
        if train:
            # mean = fp32 sum / count (fp32 partial sums, fp64 across blocks): measured <= 2.0e-7 of the channel's std.
            check(f"bn_fwd mean{tag}", None, None, 2e-6, err=float(((mean.double() - m64) / v64.sqrt()).abs().max()))
            # invstd from the one-pass E[x^2] - m^2: relative error ~ (1 + (m/std)^2) * (sum error ~1e-7): measured <= 3.6e-7.
            check(f"bn_fwd invstd{tag}", None, None, 1e-5, err=float(((invstd.double() - is64) / is64).abs().max()))
            # running statistics, momentum 0.1, unbiased variance: measured <= 1.1e-7
            check(f"bn_fwd running_mean{tag}", rm_k, 0.9 * rm.double() + 0.1 * m64, 1e-5)
            check(f"bn_fwd running_var{tag}", rv_k, 0.9 * rv.double() + 0.1 * v64 * rows / (rows - 1), 1e-5)
        else:
            assert torch.equal(mean, rm) and torch.equal(rm_k, rm) and torch.equal(rv_k, rv)  # eval: running stats read, not updated
            check(f"bn_fwd invstd eval{tag}", None, None, 1e-6, err=float(((invstd.double() - is64) / is64).abs().max()))
        # y: from the mean / invstd errors above plus one fp32 fma: measured planes 2 <= 1.9e-7, planes 1 <= 4.2e-4
        check(f"bn_fwd y{tag}", Y.float(), ref, tol_for(planes, 2e-5))
        if relu:
            # the bitmap is the sign of the fp32 pre-activation: it must equal the float64 sign wherever |pre| is above the
            # fp32 error of pre (~1e-5 of its range); measured mismatches there: 0
            bits = _bits(mask, rows, C_).bool()
            clear = pre.abs() > 1e-5 * float(pre.abs().max())
            assert int((bits != (pre > 0))[clear].sum()) == 0, tag


@pytest.mark.parametrize("ratio", [0.0, 1.0, 8.0])
@pytest.mark.parametrize("rows,C_", [(192, 64), (65536, 64), (2048, 512)])
def test_bn_stats(rows, C_, ratio):
    """gdrn_bn_stats against float64 sums; bit-identical on a second call; the one-pass variance of bn_fwd_kernel keeps
    invstd within 2e-6 * (1 + (mean/std)^2): E[x^2] = std^2 (1 + r^2) carries the sum's relative error (~1e-7 from fp32
    partials of <= 16 rows each, 32-lane fp32 block sums, fp64 across blocks) and the subtraction of m^2 multiplies it by
    1 + r^2.  Measured at r = 8: invstd 9.3e-6 (bound 1.3e-4); sums <= 2.9e-7."""
    ops = _ops()
    u, _res, gamma, beta, rm, rv = _bn_inputs(rows, C_, seed=3 * rows + C_, ratio=ratio)
    U = ops.PT.from_float(u, 2)
    ws = _det_ws()
    s1 = _bn_stats(U, rows, C_, ws)
    s2 = _bn_stats(U, rows, C_, ws)
    torch.cuda.synchronize()
    assert torch.equal(s1, s2)
    uf = U.float().double()
    tag = f"[{rows}x{C_},r{ratio}]"
    check(f"bn_stats sum{tag}", None, None, 1e-6, err=float(((s1[0].double() - uf.sum(0)) / uf.abs().sum(0)).abs().max()))
    check(f"bn_stats sumsq{tag}", None, None, 1e-6,
          err=float(((s1[1].double() - (uf * uf).sum(0)) / (uf * uf).sum(0)).abs().max()))
    _Y, mean, invstd, _m = _bn_fwd(U, None, s1, gamma, beta, rm.clone(), rv.clone(), rows, C_, 1, 0, 2)
    torch.cuda.synchronize()
    is64 = 1.0 / torch.sqrt(uf.var(0, unbiased=False) + 1e-5)
    check(f"bn_stats->invstd{tag}", None, None, 2e-6 * (1 + ratio ** 2), err=float(((invstd.double() - is64) / is64).abs().max()))


def _bn_bwd(GA, GB, U, mean, invstd, gamma, beta, sums, train, mask, det_ws):
    dgamma = torch.full_like(gamma, float("nan"))
    dbeta = torch.full_like(gamma, float("nan"))
    sums.zero_()  # Engine.backward zeroes every BatchNorm's sums once (engine.py:637): sums_zeroed=True
    du, gout = _ops().bn_bwd(GA, GB, None, U, mean, invstd, gamma, sums, dgamma, dbeta, train, want_gout=True,  # engine.py:621-624
                             beta=beta, sums_zeroed=True, relu_mask=mask, det_ws=det_ws)
    torch.cuda.synchronize()
    return du.float(), gout.float(), dgamma, dbeta


@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("det", [1, 0])
@pytest.mark.parametrize("train", [1, 0])
@pytest.mark.parametrize("rows,C_", [(192, 64), (1024, 256), (128, 512), (65536, 64)])
def test_bn_bwd(rows, C_, train, det, planes):
    """gdrn_bn_bwd with the engine's arguments (y = None, the ReLU bitmap of gdrn_bn_fwd, beta, sums_zeroed) against float64
    autograd of mask * (bn(u) + res) under the upstream ga + gb.  The mask is the bitmap the kernel is given: it is an input
    of the backward, and its agreement with the float64 sign is test_bn_fwd's.  Cases: gb present (the residual block's
    second upstream gradient, engine.py:717) and absent, ReLU off (the downsample BatchNorm, :724), train 0 (do_loss under
    model.eval()), the ordered (det) and the atomic reductions."""
    ops = _ops()
    u, res, gamma, beta, rm, rv = _bn_inputs(rows, C_, seed=rows * 3 + C_ + 7 * train)
    U, R = ops.PT.from_float(u, planes), ops.PT.from_float(res, planes)
    stats = _bn_stats(U, rows, C_) if train else None
    g = torch.Generator(device="cuda").manual_seed(rows + C_)
    GA = ops.PT.from_float(torch.randn(rows, C_, device="cuda", generator=g), planes)
    GBt = ops.PT.from_float(torch.randn(rows, C_, device="cuda", generator=g), planes)
    sums = torch.zeros(2, C_, device="cuda")
    ws = _det_ws() if det else None
    for relu, with_gb in ((1, 1), (1, 0), (0, 0), (0, 1)):
        tag = f"[{rows}x{C_},t{train},det{det},r{relu},gb{with_gb},{planes}]"
        _Y, mean, invstd, mask = _bn_fwd(U, R if with_gb else None, stats, gamma, beta, rm.clone(), rv.clone(), rows, C_, train,
                                         relu, planes)
        GB = GBt if with_gb else None
        du, gout, dgamma, dbeta = _bn_bwd(GA, GB, U, mean, invstd, gamma, beta, sums, train, mask, ws)
        u64 = U.float().double().requires_grad_(True)
        g64, b64 = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
        if train:
            pre = F.batch_norm(u64, None, None, g64, b64, True, 0.0, 1e-5)
        else:
            pre = F.batch_norm(u64, rm.double(), rv.double(), g64, b64, False, 0.0, 1e-5)
        maskf = _bits(mask, rows, C_).double() if relu else torch.ones_like(u64)
        up = GA.float().double() + (GB.float().double() if GB is not None else 0.0)
        gu, gg, gb_ = torch.autograd.grad(pre * maskf, (u64, g64, b64), up)
        # du = k1 g + k2 u + k3 with per-channel constants from fp32 sums (measured planes 2 <= 2.2e-7, planes 1 <= 4.2e-4;
        # the k2 u + k3 pair cancels to (u - mean) * k2 with |mean| / std <= 1); dgamma / dbeta are fp32 sums of <= 16 rows
        # per thread: measured <= 4.9e-7; gout <= 1.1e-7 (planes 2); ordered vs atomic du <= 1.4e-7 (planes 2).
        check(f"bn_bwd du{tag}", du, gu, tol_for(planes, 2e-5))
        check(f"bn_bwd gout{tag}", gout, up * maskf, tol_for(planes, 1e-6))
        check(f"bn_bwd dgamma{tag}", dgamma, gg, 1e-5)
        check(f"bn_bwd dbeta{tag}", dbeta, gb_, 1e-5)
        if det:
            du2, gout2, dgamma2, dbeta2 = _bn_bwd(GA, GB, U, mean, invstd, gamma, beta, sums, train, mask, ws)
            assert torch.equal(du, du2) and torch.equal(dgamma, dgamma2) and torch.equal(dbeta, dbeta2), tag  # bit-identical
            dua, _, dga, dba = _bn_bwd(GA, GB, U, mean, invstd, gamma, beta, sums, train, mask, None)
            check(f"bn_bwd det-vs-atomic du{tag}", du, dua, tol_for(planes, 2e-5))
            check(f"bn_bwd det-vs-atomic dgamma{tag}", dgamma, dga, 1e-5)
            check(f"bn_bwd det-vs-atomic dbeta{tag}", dbeta, dba, 1e-5)


# ------------------------------------------------------------------------------------------------ C. small backward kernels
@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("rows", [1, 3, 64, 262144])
@pytest.mark.parametrize("ld", [64, 128, 256, 1024])
def test_colsum(ld, rows, planes):
    """gdrn_colsum: every bias gradient of the FC stack (engine.py:649, :656, :661) and of the head output conv (:689, 262144
    rows = B 64 x 4096 pixels).  The output is pre-filled with NaN.  Error relative to sum |x| of the column: fp32 partials of
    at most 16 rows per thread, an fp32 sum over the <= 32 row lanes, fp32 atomics over <= 4 * 132 blocks: worst case
    (16 + 32 + 528) * 6e-8 = 3.4e-5, the bound; measured <= 9.0e-8."""
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(ld + rows)
    X = ops.PT.from_float(torch.randn(rows, ld, device="cuda", generator=g), planes)
    out = torch.full((ld,), float("nan"), device="cuda")
    _C().gdrn_colsum(X.hi_ptr, X.lo_ptr, out.data_ptr(), rows, ld, _s())
    torch.cuda.synchronize()
    xf = X.float().double()
    err = float(((out.double() - xf.sum(0)) / xf.abs().sum(0).clamp_min(1e-30)).abs().max())
    check(f"colsum[{ld},{rows},{planes}]", None, None, 3.4e-5, err=err)


@pytest.mark.parametrize("planes", [1, 2])
def test_leaky_bwd(planes):
    """gdrn_leaky_bwd (Engine._leaky_bwd, engine.py:771-774) against torch's leaky_relu backward: y > 0, y < 0, y = +0 and
    y = -0.0 (both are 'not positive': slope 0.1, like torch at an input of 0)."""
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(11)
    n = 64 * 1024
    y = torch.randn(n, device="cuda", generator=g)
    y[0::7] = 0.0
    y[3::7] = -0.0
    Y = ops.PT((n,), 1, buf=y.to(ops.storage_format()[0]).view(1, n))
    assert bool(torch.signbit(Y.hi[3::7]).all()) and not bool(torch.signbit(Y.hi[0::7]).any())
    G = ops.PT.from_float(torch.randn(n, device="cuda", generator=g), planes)
    out = nan_planes((n,), planes)
    _C().gdrn_leaky_bwd(G.hi_ptr, G.lo_ptr, Y.hi_ptr, out.hi_ptr, out.lo_ptr, n, _s())
    torch.cuda.synchronize()
    yh = Y.hi.double()
    x = torch.where(yh > 0, yh, 10.0 * yh).requires_grad_(True)  # an input with the sign of y
    (ref,) = torch.autograd.grad(F.leaky_relu(x, 0.1), x, G.float().double())
    check(f"leaky_bwd[{planes}]", out.float(), ref, tol_for(planes, 1e-6))  # one fp32 multiply: measured planes 2 <= 1.2e-8
    for sl, nm in ((slice(0, None, 7), "+0"), (slice(3, None, 7), "-0")):
        assert torch.equal(out.float()[sl], ref[sl].float()) or rel_err(out.float()[sl], ref[sl]) <= tol_for(planes, 1e-6), nm


def _wgrad_ref(fn, w_shape, x, up):
    w = torch.zeros(w_shape, dtype=torch.float64, device="cuda", requires_grad=True)
    (gw,) = torch.autograd.grad(fn(x, w), w, up)
    return gw


# Weight gradients: fp32 accumulation of exact fp16 x fp16 (planes 1) or of the three hi/lo cross products (planes 2, the
# dropped lo x lo term is ~2^-22) over K = B (fc) up to B * 16384 (stem) rows, split-K partials summed in fp32: measured
# <= 9.0e-7; bound 2e-5 (the op tests of tests/test_ops_gpu.py use 5e-5 for the plain layouts).
WG_TOL = 2e-5


@pytest.mark.parametrize("planes", [1, 2])
def test_wgrad_fc_rt_split(planes):
    """fc_r and fc_t weight gradients from ONE workspace of the concatenated [9][256] FC (engine.py:646-648)."""
    ops = _ops()
    B = 64
    g = torch.Generator(device="cuda").manual_seed(1)
    dy = torch.zeros(B, 64, device="cuda")
    dy[:, :9] = torch.randn(B, 9, device="cuda", generator=g)
    dy9, h2 = ops.PT.from_float(dy, planes), ops.PT.from_float(torch.randn(B, 256, device="cuda", generator=g), planes)
    buf, ks, kss = ops.gemm_wgrad(dy9, h2, ops.Workspace())
    gr = torch.full((6, 256), float("nan"), device="cuda")
    gt = torch.full((3, 256), float("nan"), device="cuda")
    ops.unpack_wgrad(buf, gr, 6, 256, 1, 1, 256, ks, kss, 256, 1, 0, 0)
    ops.unpack_wgrad(buf[6 * 256:], gt, 3, 256, 1, 1, 256, ks, kss, 256, 1, 0, 0)
    torch.cuda.synchronize()
    ref = dy9.float().double()[:, :9].t() @ h2.float().double()
    check(f"wgrad fc_r[{planes}]", gr, ref[:6], WG_TOL)
    check(f"wgrad fc_t[{planes}]", gt, ref[6:9], WG_TOL)


@pytest.mark.parametrize("planes", [1, 2])
def test_wgrad_fc1_nchw_flatten(planes):
    """fc1: F.linear on the NCHW flatten of the [B, 8, 8, 128] NHWC activation; the workspace columns are (h, w, c) and the
    unpack writes the (c, h, w) weight layout (engine.py:659-660)."""
    ops = _ops()
    B = 64
    g = torch.Generator(device="cuda").manual_seed(2)
    dz1 = ops.PT.from_float(torch.randn(B, 1024, device="cuda", generator=g), planes)
    flat = ops.PT.from_float(torch.randn(B, 8192, device="cuda", generator=g), planes)  # NHWC flatten (h, w, c)
    buf, ks, kss = ops.gemm_wgrad(dz1, flat, ops.Workspace())
    grad = torch.full((1024, 8192), float("nan"), device="cuda")
    ops.unpack_wgrad(buf, grad, 1024, 128, 8, 8, 128, ks, kss, 8192, 64, 8, 1)
    torch.cuda.synchronize()
    x_nchw = flat.float().double().view(B, 8, 8, 128).permute(0, 3, 1, 2).reshape(B, 8192)
    ref = _wgrad_ref(lambda x, w: F.linear(x, w), (1024, 8192), x_nchw, dz1.float().double())
    check(f"wgrad fc1[{planes}]", grad, ref, WG_TOL)


def _stem_im2col(x, planes):
    ops = _ops()
    B = x.shape[0]
    a_col = ops.PT((B * 128 * 128, 192), planes, device="cuda")
    _C().gdrn_stem_im2col(x.data_ptr(), a_col.hi_ptr, a_col.lo_ptr, B, 256, 256, _s())  # engine.py:487-488
    return a_col


@pytest.mark.parametrize("planes", [1, 2])
def test_wgrad_stem(planes):
    """The 7x7/2/3 stem: gdrn_stem_im2col, the GEMM weight gradient over its [B*16384][192] matrix and the krow-192 unpack to
    OIHW (engine.py:737-739), against float64 autograd of F.conv2d."""
    ops = _ops()
    B = 2
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(B, 3, 256, 256, device="cuda", generator=g)
    a_col = _stem_im2col(x, planes)
    du0 = ops.PT.from_float(torch.randn(B * 16384, 64, device="cuda", generator=g), planes)
    buf, ks, kss = ops.gemm_wgrad(du0, a_col, ops.Workspace())
    grad = torch.full((64, 3, 7, 7), float("nan"), device="cuda")
    ops.unpack_wgrad(buf, grad, 64, 3, 7, 7, 3, ks, kss, 147, 49, 7, 1, krow=192)
    torch.cuda.synchronize()
    assert bool((a_col.buf[:, :, 147:] == 0).all())  # the 45 padding columns of the im2col rows
    up = du0.float().double().view(B, 128, 128, 64).permute(0, 3, 1, 2)
    ref = _wgrad_ref(lambda xx, w: F.conv2d(xx, w, None, stride=2, padding=3), (64, 3, 7, 7), _operand(x, planes).double(), up)
    check(f"wgrad stem[{planes}]", grad, ref, WG_TOL)


@pytest.mark.parametrize("planes", [1, 2])
def test_wgrad_deconv_roles_swapped(planes):
    """The ConvTranspose2d (512 -> 256, k3 s2 p1 op1) weight gradient: conv_wgrad of the stride-2 conv du -> z with z in the
    role of dY, unpacked to the IOHW layout without a flip (engine.py:703-707)."""
    ops = _ops()
    B = 2
    g = torch.Generator(device="cuda").manual_seed(4)
    z = ops.PT.from_float(torch.randn(B, 8, 8, 512, device="cuda", generator=g), planes)
    du = ops.PT.from_float(torch.randn(B, 16, 16, 256, device="cuda", generator=g), planes)
    buf, ks, kss = ops.conv_wgrad(z, du, ops.Workspace(), 512, 3, 3, 2, 1)
    grad = torch.full((512, 256, 3, 3), float("nan"), device="cuda")
    ops.unpack_wgrad(buf, grad, 512, 256, 3, 3, 256, ks, kss, 256 * 9, 9, 3, 1)
    torch.cuda.synchronize()
    ref = _wgrad_ref(lambda x, w: F.conv_transpose2d(x, w, None, stride=2, padding=1, output_padding=1), (512, 256, 3, 3),
                     z.float().double().permute(0, 3, 1, 2), du.float().double().permute(0, 3, 1, 2))
    check(f"wgrad deconv[{planes}]", grad, ref, WG_TOL)


@pytest.mark.parametrize("planes", [1, 2])
def test_fc_dgrad_operands(planes):
    """dX of the FC stack through pack_linear(..., transpose=True) operands: fc_rt (engine.py:386, :652), fc2 (:385, :657) and
    fc1 with nhwc_from (:384, :662, the gradient comes out in the NHWC order of the Patch-PnP activation).  Output rounded to
    the storage format for planes 1; fp32 accumulation otherwise (measured <= 1.7e-6, planes 1 <= 2.8e-4)."""
    ops = _ops()
    B = 64
    g = torch.Generator(device="cuda").manual_seed(5)
    w_rt = torch.randn(9, 256, device="cuda", generator=g) / 16
    w2 = torch.randn(256, 1024, device="cuda", generator=g) / 32
    w1 = torch.randn(1024, 8192, device="cuda", generator=g) / 90
    dy = torch.zeros(B, 64, device="cuda")
    dy[:, :9] = torch.randn(B, 9, device="cuda", generator=g)
    dy9 = ops.PT.from_float(dy, planes)
    dz2 = ops.PT.from_float(torch.randn(B, 256, device="cuda", generator=g), planes)
    dz1 = ops.PT.from_float(torch.randn(B, 1024, device="cuda", generator=g), planes)
    dh2 = ops.gemm_fwd(dy9, ops.pack_linear(w_rt, planes, transpose=True), 256)
    dh1 = ops.gemm_fwd(dz2, ops.pack_linear(w2, planes, transpose=True), 1024)
    dfl = ops.gemm_fwd(dz1, ops.pack_linear(w1, planes, nhwc_from=(128, 8, 8), transpose=True), 8192).view(B, 8, 8, 128)
    torch.cuda.synchronize()
    tol = tol_for(planes, 1e-5)
    check(f"dgrad fc_rt[{planes}]", dh2.float(), dy9.float().double()[:, :9] @ _operand(w_rt, planes).double(), tol)
    check(f"dgrad fc2[{planes}]", dh1.float(), dz2.float().double() @ _operand(w2, planes).double(), tol)
    ref1 = (dz1.float().double() @ _operand(w1, planes).double()).view(B, 128, 8, 8).permute(0, 2, 3, 1)
    check(f"dgrad fc1 nhwc[{planes}]", dfl.float(), ref1, tol)


# ------------------------------------------------------------------------------------------------ D. forward epilogue variants
# GEMM outputs: fp32 accumulation as for the weight gradients, then bias / residual / ReLU in fp32 and the storage rounding
# (planes 1).  Bound 2e-5 (fp32) + u; measured <= 2.7e-6 (planes 2), <= 4.2e-4 (planes 1).  Epilogue statistics: fp32
# atomics of per-tile sums, error relative to sum |y| (sum) and to sum y^2: measured <= 3.2e-6; bound 1e-5.  The stem's
# epilogue statistics and gdrn_bn_stats of the same tensor: measured 5.4e-7.
EP_TOL = 2e-5


def _stats_err(stats, ref):
    s0 = float(((stats[0].double() - ref.sum(0)) / ref.abs().sum(0)).abs().max())
    s1 = float(((stats[1].double() - (ref * ref).sum(0)) / (ref * ref).sum(0)).abs().max())
    return max(s0, s1)


@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("case", [(16, 256, 256, 3, 1, 1, True, 2), (32, 128, 256, 3, 2, 1, False, 2), (32, 128, 256, 1, 2, 0, False, 0)])
def test_conv_fwd_folded_eval(case, planes):
    """Folded eval conv + BN shift + residual + ReLU (engine.py:290): conv2 of a residual block with res and act 2, conv1 of a
    downsampling block (act 2) and the downsample conv (relu False: act 0)."""
    ops = _ops()
    H, Cin, Cout, k, stride, pad, with_res, act = case
    g = torch.Generator(device="cuda").manual_seed(sum(case[:6]))
    x = ops.PT.from_float(torch.randn(2, H, H, Cin, device="cuda", generator=g), planes)
    w = torch.randn(Cout, Cin, k, k, device="cuda", generator=g) / (k * Cin ** 0.5)
    bias = torch.randn(Cout, device="cuda", generator=g)
    Ho = H // stride
    res = ops.PT.from_float(torch.randn(2, Ho, Ho, Cout, device="cuda", generator=g), planes) if with_res else None
    out = ops.conv_fwd(x, ops.pack_conv_fwd(w, planes), Cout, k, k, stride, pad, bias=bias, act=act, res=res)
    torch.cuda.synchronize()
    ref = F.conv2d(x.float().double().permute(0, 3, 1, 2), _operand(w, planes).double(), bias.double(), stride=stride, padding=pad)
    ref = ref.permute(0, 2, 3, 1) + (res.float().double() if with_res else 0.0)
    ref = torch.relu(ref) if act == 2 else ref
    check(f"conv_fwd folded{list(case)}[{planes}]", out.float(), ref, tol_for(planes, EP_TOL))


@pytest.mark.parametrize("planes", [1, 2])
def test_deconv_fwd_as_dgrad_s2(planes):
    """The ConvTranspose2d forward (512 -> 256, 8x8 -> 16x16, k3 s2 p1 op1) as gdrn_conv_dgrad_s2 over pack_conv_dgrad of its
    IOHW weight (engine.py:373): train with the BatchNorm statistics in the epilogue (:422) and folded eval with bias and
    ReLU (:288)."""
    ops = _ops()
    B = 2
    g = torch.Generator(device="cuda").manual_seed(8)
    x = ops.PT.from_float(torch.randn(B, 8, 8, 512, device="cuda", generator=g), planes)
    wt = torch.randn(512, 256, 3, 3, device="cuda", generator=g) / 40
    bias = torch.randn(256, device="cuda", generator=g)
    wp = ops.pack_conv_dgrad(wt, planes)
    ref = F.conv_transpose2d(x.float().double().permute(0, 3, 1, 2), _operand(wt, planes).double(), None, stride=2, padding=1,
                             output_padding=1).permute(0, 2, 3, 1)
    stats = torch.zeros(2, 256, device="cuda")
    u = ops.conv_dgrad_s2(x, wp, 256, 3, 1, out=nan_planes((B, 16, 16, 256), planes), stats=stats)
    y = ops.conv_dgrad_s2(x, wp, 256, 3, 1, out=nan_planes((B, 16, 16, 256), planes), bias=bias, act=2)
    torch.cuda.synchronize()
    tol = tol_for(planes, EP_TOL)
    check(f"deconv fwd[{planes}]", u.float(), ref, tol)
    check(f"deconv fwd stats[{planes}]", None, None, 1e-5, err=_stats_err(stats, ref.reshape(-1, 256)))
    check(f"deconv fwd bias+relu[{planes}]", y.float(), torch.relu(ref + bias.double()), tol)


@pytest.mark.parametrize("planes", [1, 2])
def test_dgrad_s2_padding_channels(planes):
    """The Patch-PnP first conv's dgrad (Cx = 69 of a 128-wide output, Engine._dgrad_conv, engine.py:615): channels 69..127
    are exact zeros.  The epilogue zero-fills only the partial 32-column chunk after Cx; ops.conv_dgrad_s2 allocates the
    output zeroed when ldc != Cx, which covers the whole chunks, so the check runs through the wrapper as the engine calls
    it.  The valid channels are compared on an output pre-filled with NaN."""
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(12)
    w = torch.randn(128, 69, 3, 3, device="cuda", generator=g) / 25
    dy = torch.randn(2, 128, 32, 32, device="cuda", generator=g)
    DY = ops.PT.from_float(dy.permute(0, 2, 3, 1).contiguous(), planes)
    wd = ops.pack_conv_dgrad(w, planes)
    out = ops.conv_dgrad_s2(DY, wd, 69, 3, 1)
    out_nan = ops.conv_dgrad_s2(DY, wd, 69, 3, 1, out=nan_planes((2, 64, 64, 128), planes))
    torch.cuda.synchronize()
    x = torch.zeros(2, 69, 64, 64, dtype=torch.float64, device="cuda", requires_grad=True)
    y = F.conv2d(x, _operand(w, planes).double(), None, stride=2, padding=1)
    (gx,) = torch.autograd.grad(y, x, DY.float().double().permute(0, 3, 1, 2))
    check(f"dgrad_s2 Cx69[{planes}]", out_nan.float()[..., :69], gx.permute(0, 2, 3, 1), tol_for(planes, EP_TOL))
    assert torch.equal(out.buf[..., :69], out_nan.buf[..., :69])
    assert bool((out.buf[..., 69:] == 0).all())


@pytest.mark.parametrize("planes", [1, 2])
def test_stem_gemm_fwd_stats(planes):
    """The stem forward: gdrn_stem_im2col + pack_stem + gemm_fwd with the BatchNorm statistics in the epilogue (engine.py:487-491),
    against float64 F.conv2d 7x7/2/3; the output pixels whose taps reach over the image border are also compared on their
    own.  The epilogue statistics agree with gdrn_bn_stats of the same (two-plane) tensor to fp32 rounding."""
    ops = _ops()
    B = 2
    g = torch.Generator(device="cuda").manual_seed(13)
    x = torch.randn(B, 3, 256, 256, device="cuda", generator=g)
    w = torch.randn(64, 3, 7, 7, device="cuda", generator=g) / 12
    a_col = _stem_im2col(x, planes)
    stats = torch.zeros(2, 64, device="cuda")
    u0 = ops.gemm_fwd(a_col, ops.pack_stem(w, planes), 64, stats=stats)
    torch.cuda.synchronize()
    ref = F.conv2d(_operand(x, planes).double(), _operand(w, planes).double(), None, stride=2, padding=3).permute(0, 2, 3, 1)
    got = u0.float().view(B, 128, 128, 64)
    tol = tol_for(planes, EP_TOL)
    check(f"stem fwd[{planes}]", got, ref, tol)
    border = torch.zeros(128, 128, dtype=torch.bool, device="cuda")
    border[:2], border[-2:], border[:, :2], border[:, -2:] = True, True, True, True  # taps at rows / cols < 0 or >= 256
    check(f"stem fwd border[{planes}]", got[:, border], ref[:, border], tol)
    check(f"stem fwd stats[{planes}]", None, None, 1e-5, err=_stats_err(stats, ref.reshape(-1, 64)))
    if planes == 2:
        s_bn = _bn_stats(u0, B * 16384, 64)
        torch.cuda.synchronize()
        uf = u0.float().double()
        e = max(float(((stats[0] - s_bn[0]).double().abs() / uf.abs().sum(0)).max()),
                float(((stats[1] - s_bn[1]).double().abs() / (uf * uf).sum(0)).max()))
        check("stem epilogue stats vs bn_stats", None, None, 1e-5, err=e)
