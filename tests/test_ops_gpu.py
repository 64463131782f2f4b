"""GPU: every C-ABI op against a plain PyTorch fp32 reference of the same op (TF32 disabled).
nsplit = 1 (one 16-bit plane, fp16 unless the library is built for bf16): the reference is evaluated on operands rounded to
the storage format, so only fp32 accumulation order differs.  nsplit = 3 (hi/lo planes): the reference is full fp32.
Per-launch float64 checks of the GEMM kernels at the engine's own shapes: tests/test_gemm_audit_gpu.py."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]


@pytest.fixture(scope="module", autouse=True)
def _setup():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield


def _ops():
    from gdr_net_b200 import ops

    return ops


def _rel(a, b):
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def _operand(x, planes):
    """What the kernel effectively multiplies: bf16-rounded for planes=1, ~fp32 for planes=2."""
    return _ops().round_storage(x) if planes == 1 else x


def _nhwc(x_nchw, planes):
    ops = _ops()
    return ops.PT.from_float(x_nchw.permute(0, 2, 3, 1).contiguous(), planes)


TOL = {1: 5e-5, 2: 5e-5}


@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("M,N,K", [(128, 64, 64), (256, 128, 192), (300, 256, 512), (64, 1024, 8192), (2, 9, 256), (1000, 69, 256)])
def test_gemm_fwd(planes, M, N, K):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N * 3 + K)
    a = torch.randn(M, K, device="cuda", generator=g)
    w = torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)
    bias = torch.randn(N, device="cuda", generator=g)
    A = ops.PT.from_float(a, planes)
    Wp = ops.pack_linear(w, planes)
    ldc = (N + 7) // 8 * 8
    out32 = torch.full((M, ldc), float("nan"), device="cuda")
    out = ops.gemm_fwd(A, Wp, N, out_f32=out32, bias=bias, act=1, ldc=ldc)
    torch.cuda.synchronize()
    ref = F.leaky_relu(_operand(a, planes) @ _operand(w, planes).t() + bias, 0.1)
    assert _rel(out32[:, :N], ref) < TOL[planes]
    got = out.float()[:, :N]
    assert _rel(got, ref) < (5e-3 if planes == 1 else 3e-5)  # planes=1: output rounded to the 16-bit storage format


CONV_CASES = [
    # N, H, W, Cin, Cout, k, stride, pad
    (2, 64, 64, 64, 64, 3, 1, 1),
    (2, 32, 32, 128, 128, 3, 1, 1),
    (2, 16, 16, 256, 256, 3, 1, 1),
    (4, 8, 8, 512, 512, 3, 1, 1),
    (3, 8, 8, 128, 128, 3, 1, 1),     # odd batch: half-empty last tile
    (2, 64, 64, 64, 128, 3, 2, 1),
    (2, 64, 64, 64, 128, 1, 2, 0),
    (2, 16, 16, 256, 512, 3, 2, 1),
    (2, 64, 64, 128, 128, 3, 2, 1),   # Patch-PnP first conv shape (Cin padded 69 -> 128)
    (2, 64, 64, 256, 69, 1, 1, 0),    # head output conv (N tail, bias)
]


@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("case", CONV_CASES)
def test_conv_fwd(planes, case):
    ops = _ops()
    N, H, W, Cin, Cout, k, stride, pad = case
    g = torch.Generator(device="cuda").manual_seed(sum(case))
    x = torch.randn(N, Cin, H, W, device="cuda", generator=g)
    w = torch.randn(Cout, Cin, k, k, device="cuda", generator=g) / math.sqrt(Cin * k * k)
    X = _nhwc(x, planes)
    Wp = ops.pack_conv_fwd(w, planes)
    ldc = (Cout + 7) // 8 * 8
    Ho, Wo = H // stride, W // stride
    out32 = torch.zeros(N, Ho, Wo, ldc, device="cuda")
    stats = torch.zeros(2, Cout, device="cuda")
    bias = torch.randn(Cout, device="cuda", generator=g) if Cout == 69 else None
    ops.conv_fwd(X, Wp, Cout, k, k, stride, pad, out_f32=out32, stats=stats if bias is None else None, bias=bias, ldc=ldc,
                 want_planes=False)
    torch.cuda.synchronize()
    ref = F.conv2d(_operand(x, planes), _operand(w, planes), bias, stride=stride, padding=pad).permute(0, 2, 3, 1)
    assert _rel(out32[..., :Cout], ref) < TOL[planes]
    if bias is None:
        s1 = ref.reshape(-1, Cout).sum(0)
        s2 = (ref.reshape(-1, Cout) ** 2).sum(0)
        assert float((stats[0] - s1).abs().max()) < 1e-3 * float(s2.max().sqrt()) + 1e-3
        assert _rel(stats[1], s2) < 1e-4


@pytest.mark.parametrize("planes", [1, 2])
def test_conv_dgrad_as_conv(planes):
    """dX of a 3x3 s1 conv = conv(dY, flipped/transposed weights); of a s2 conv = same over zero-inserted dY."""
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(5)
    for (N, H, Cin, Cout, stride) in [(2, 32, 64, 128, 1), (2, 32, 64, 128, 2)]:
        x = torch.randn(N, Cin, H, H, device="cuda", generator=g, requires_grad=True)
        w = torch.randn(Cout, Cin, 3, 3, device="cuda", generator=g) / 24
        w_eff = _operand(w, planes)
        y = F.conv2d(x, w_eff, None, stride=stride, padding=1)
        dy = torch.randn_like(y)
        (gx,) = torch.autograd.grad(y, x, _operand(dy, planes))
        DY = _nhwc(dy, planes)
        if stride == 2:
            DY = ops.zero_insert(DY)
        Wd = ops.pack_conv_dgrad(w, planes)
        out32 = torch.zeros(N, H, H, Cin, device="cuda")
        ops.conv_fwd(DY, Wd, Cin, 3, 3, 1, 1, out_f32=out32, want_planes=False)
        torch.cuda.synchronize()
        assert _rel(out32, gx.permute(0, 2, 3, 1)) < TOL[planes]


@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("case", [(2, 64, 64, 128, 3, 1), (3, 32, 128, 256, 3, 1), (4, 16, 256, 512, 3, 1), (2, 64, 69, 128, 3, 1),
                                  (2, 64, 64, 128, 1, 0), (4, 16, 256, 512, 1, 0)])
def test_conv_dgrad_s2_phases(planes, case):
    """dX of a stride-2 conv through the output-parity decomposition == torch's conv backward-data."""
    ops = _ops()
    N, H, Cin, Cout, k, pad = case
    g = torch.Generator(device="cuda").manual_seed(sum(case))
    x = torch.randn(N, Cin, H, H, device="cuda", generator=g, requires_grad=True)
    w = torch.randn(Cout, Cin, k, k, device="cuda", generator=g) / (3 * k * Cin ** 0.5)
    y = F.conv2d(x, _operand(w, planes), None, stride=2, padding=pad)
    dy = torch.randn_like(y)
    (gx,) = torch.autograd.grad(y, x, _operand(dy, planes))
    out = ops.conv_dgrad_s2(_nhwc(dy, planes), ops.pack_conv_dgrad(w, planes), Cin, k, pad)
    torch.cuda.synchronize()
    got = out.float()
    assert got.shape[:3] == (N, H, H)
    assert _rel(got[..., :Cin], gx.permute(0, 2, 3, 1)) < (TOL[planes] if planes == 2 else 2e-3)
    if got.shape[-1] > Cin:
        assert float(got[..., Cin:].abs().max()) == 0.0


@pytest.mark.parametrize("planes", [1, 2])
def test_deconv_fwd_and_dgrad(planes):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(9)
    N, Cin, Cout = 2, 512, 256
    x = torch.randn(N, Cin, 8, 8, device="cuda", generator=g, requires_grad=True)
    wt = torch.randn(Cin, Cout, 3, 3, device="cuda", generator=g) / 34
    y = F.conv_transpose2d(_operand(x, planes), _operand(wt, planes), None, stride=2, padding=1, output_padding=1)
    Z = ops.zero_insert(_nhwc(x.detach(), planes))
    out32 = torch.zeros(N, 16, 16, Cout, device="cuda")
    ops.conv_fwd(Z, ops.pack_deconv_fwd(wt, planes), Cout, 3, 3, 1, 1, out_f32=out32, want_planes=False)
    torch.cuda.synchronize()
    assert _rel(out32, y.permute(0, 2, 3, 1)) < TOL[planes]
    dy = torch.randn_like(y)
    y2 = F.conv_transpose2d(x, _operand(wt, planes), None, stride=2, padding=1, output_padding=1)
    (gx,) = torch.autograd.grad(y2, x, _operand(dy, planes))
    dx32 = torch.zeros(N, 8, 8, Cin, device="cuda")
    ops.conv_fwd(_nhwc(dy, planes), ops.pack_deconv_dgrad(wt, planes), Cin, 3, 3, 2, 1, out_f32=dx32, want_planes=False)
    torch.cuda.synchronize()
    assert _rel(dx32, gx.permute(0, 2, 3, 1)) < TOL[planes]


def test_pdl_chain_bit_equal():
    """Programmatic dependent launch: every GEMM kernel may start under the tail of its predecessor and waits (griddepcontrol.wait)
    before its first global read.  A chain conv -> conv -> conv (each consuming the previous output, different shapes so the
    tails differ) repeated many times must give bit-identical results with the attribute on and off."""
    ops = _ops()
    from gdr_net_b200.capi import C

    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(16, 64, 32, 32, device="cuda", generator=g)
    ws = [torch.randn(co, ci, 3, 3, device="cuda", generator=g) / math.sqrt(9 * ci) for ci, co in ((64, 128), (128, 256), (256, 64))]
    X = _nhwc(x, 1)
    Wp = [ops.pack_conv_fwd(w, 1) for w in ws]

    def chain():
        t = X
        for w, wp in zip(ws, Wp):
            t = ops.conv_fwd(t, wp, w.shape[0], 3, 3, 1, 1)
        return t.float()

    try:
        C.gdrn_set_pdl(0)
        ref = chain()
        torch.cuda.synchronize()
        C.gdrn_set_pdl(1)
        for _ in range(30):
            out = chain()
        torch.cuda.synchronize()
        assert torch.equal(out, ref)
    finally:
        C.gdrn_set_pdl(1)


WGRAD_CASES = [(2, 64, 64, 64, 64, 3, 1, 1), (2, 32, 32, 128, 128, 3, 1, 1), (4, 16, 16, 256, 256, 3, 1, 1),
               (8, 8, 8, 512, 512, 3, 1, 1), (2, 64, 64, 64, 128, 3, 2, 1), (2, 64, 64, 64, 128, 1, 2, 0),
               (2, 64, 64, 256, 128, 1, 1, 0)]


@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("case", WGRAD_CASES)
def test_conv_wgrad(planes, case):
    ops = _ops()
    N, H, W, Cin, Cout, k, stride, pad = case
    g = torch.Generator(device="cuda").manual_seed(sum(case) + 1)
    x = torch.randn(N, Cin, H, W, device="cuda", generator=g)
    w = torch.zeros(Cout, Cin, k, k, device="cuda", requires_grad=True)
    y = F.conv2d(_operand(x, planes), w, None, stride=stride, padding=pad)
    dy = torch.randn_like(y) / 8
    (gw,) = torch.autograd.grad(y, w, _operand(dy, planes))
    ws = ops.Workspace()
    buf, ks, ks_stride = ops.conv_wgrad(_nhwc(dy, planes), _nhwc(x, planes), ws, Cout, k, k, stride, pad)
    grad = torch.zeros_like(w)
    ops.unpack_wgrad(buf, grad, Cout, Cin, k, k, Cin, ks, ks_stride, Cin * k * k, k * k, k, 1)
    torch.cuda.synchronize()
    assert _rel(grad, gw) < 5e-5


@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("P,M,N", [(64, 1024, 8192), (2, 64, 256), (4096, 64, 192), (300, 256, 1024)])
def test_gemm_wgrad(planes, P, M, N):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(P + M + N)
    dy = torch.randn(P, M, device="cuda", generator=g)
    x = torch.randn(P, N, device="cuda", generator=g)
    ws = ops.Workspace()
    buf, ks, ks_stride = ops.gemm_wgrad(ops.PT.from_float(dy, planes), ops.PT.from_float(x, planes), ws)
    grad = torch.zeros(M, N, device="cuda")
    ops.unpack_wgrad(buf, grad, M, N, 1, 1, N, ks, ks_stride, N, 1, 0, 0)
    torch.cuda.synchronize()
    ref = _operand(dy, planes).t() @ _operand(x, planes)
    assert _rel(grad, ref) < 5e-5


# ------------------------------------------------------------------------------------------------ elementwise
@pytest.mark.parametrize("planes", [1, 2])
def test_pack_roundtrip_and_planes(planes):
    ops = _ops()
    x = torch.randn(4, 64, 64, device="cuda")
    P = ops.PT.from_float(x, planes)
    tol = 4e-3 if planes == 1 else 2e-5
    assert _rel(P.to_float(), x) < tol and _rel(P.float(), x) < tol


@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("C_", [64, 256])
def test_bn_train_fwd_bwd(planes, C_):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(C_)
    N, H = 3, 16
    u = torch.randn(N, C_, H, H, device="cuda", generator=g) * 2 + 0.5
    res = torch.randn(N, C_, H, H, device="cuda", generator=g)
    gamma = torch.rand(C_, device="cuda", generator=g) + 0.5
    beta = torch.randn(C_, device="cuda", generator=g) * 0.1
    rm, rv = torch.zeros(C_, device="cuda"), torch.ones(C_, device="cuda")
    U, R = _nhwc(u, planes), _nhwc(res, planes)
    uf, rf = U.float().permute(0, 3, 1, 2).clone().requires_grad_(True), R.float().permute(0, 3, 1, 2)
    gam = gamma.clone().requires_grad_(True)
    bet = beta.clone().requires_grad_(True)
    rm_ref, rv_ref = rm.clone(), rv.clone()
    y_ref = F.relu(F.batch_norm(uf, rm_ref, rv_ref, gam, bet, True, 0.1, 1e-5) + rf)
    # our path: stats straight from the tensor (the conv epilogue normally provides them)
    flat = U.float().reshape(-1, C_)
    stats = torch.stack([flat.sum(0), (flat * flat).sum(0)]).contiguous()
    scale, shift, mean, invstd = (torch.empty(C_, device="cuda") for _ in range(4))
    ops.bn_finalize(stats, gamma, beta, rm, rv, scale, shift, mean, invstd, C_, flat.shape[0], 1e-5, 0.1, True)
    Y = ops.bn_act(U, scale, shift, True, res=R)
    torch.cuda.synchronize()
    tol = 8e-3 if planes == 1 else 3e-5
    assert _rel(Y.float().permute(0, 3, 1, 2), y_ref) < tol
    assert _rel(rm, rm_ref) < 1e-5 and _rel(rv, rv_ref) < 1e-5
    gy = torch.randn_like(y_ref)
    GY = _nhwc(gy, planes)
    gu_ref, gg_ref, gb_ref = torch.autograd.grad(y_ref, (uf, gam, bet), GY.float().permute(0, 3, 1, 2))
    sums = torch.zeros(2, C_, device="cuda")
    dgamma, dbeta = torch.zeros(C_, device="cuda"), torch.zeros(C_, device="cuda")
    DU, GOUT = ops.bn_bwd(GY, None, Y, U, mean, invstd, gamma, sums, dgamma, dbeta, True, want_gout=True)
    torch.cuda.synchronize()
    tolb = 2e-2 if planes == 1 else 1e-4
    assert _rel(DU.float().permute(0, 3, 1, 2), gu_ref) < tolb
    assert _rel(dgamma, gg_ref) < tolb and _rel(dbeta, gb_ref) < tolb
    mask = (Y.float() > 0).float()
    assert _rel(GOUT.float(), GY.float() * mask) < (8e-3 if planes == 1 else 3e-5)


@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("C_", [64, 256])
def test_bn_bwd_relu_mask_from_u(planes, C_):
    """Plain conv-BN-ReLU: the ReLU mask recomputed from u (flags bit 0, y not read) gives the same result as reading y."""
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(100 + C_)
    N, H = 4, 16
    U = _nhwc(torch.randn(N, C_, H, H, device="cuda", generator=g) * 2 + 0.3, planes)
    gamma = torch.rand(C_, device="cuda", generator=g) + 0.5
    beta = torch.randn(C_, device="cuda", generator=g) * 0.3
    rm, rv = torch.zeros(C_, device="cuda"), torch.ones(C_, device="cuda")
    flat = U.float().reshape(-1, C_)
    stats = torch.stack([flat.sum(0), (flat * flat).sum(0)]).contiguous()
    scale, shift, mean, invstd = (torch.empty(C_, device="cuda") for _ in range(4))
    ops.bn_finalize(stats, gamma, beta, rm, rv, scale, shift, mean, invstd, C_, flat.shape[0], 1e-5, 0.1, True)
    Y = ops.bn_act(U, scale, shift, True)
    GY = _nhwc(torch.randn(N, C_, H, H, device="cuda", generator=g), planes)
    outs = []
    for from_u in (False, True):
        sums = torch.zeros(2, C_, device="cuda")
        dgamma, dbeta = torch.zeros(C_, device="cuda"), torch.zeros(C_, device="cuda")
        DU, _ = ops.bn_bwd(GY, None, None if from_u else Y, U, mean, invstd, gamma, sums, dgamma, dbeta, True, beta=beta,
                           relu_from_u=from_u, sums_zeroed=True)
        torch.cuda.synchronize()
        outs.append((DU.float(), dgamma, dbeta))
    # elements with 0 < bn(u) < 3e-8 round to y == 0 in the 16-bit activation: their mask (hence du) may differ
    assert int(((outs[0][0] - outs[1][0]).abs() > 1e-4).sum()) <= 4
    # (a single flipped element moves one channel's dgamma / dbeta by |g| ~ 1-4 out of ~100)
    assert _rel(outs[1][1], outs[0][1]) < 5e-2 and _rel(outs[1][2], outs[0][2]) < 5e-2


@pytest.mark.parametrize("planes", [1, 2])
def test_maxpool_upsample_zero_insert(planes):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(2, 64, 32, 32, device="cuda", generator=g)
    X = _nhwc(x, planes)
    xf = X.float().permute(0, 3, 1, 2).clone().requires_grad_(True)
    tol = 8e-3 if planes == 1 else 3e-5
    # maxpool
    y_ref = F.max_pool2d(xf, 3, 2, 1)
    Y, ARG = ops.maxpool_fwd(X, want_arg=True)
    assert _rel(Y.float().permute(0, 3, 1, 2), y_ref) < tol
    gy = torch.randn_like(y_ref)
    GY = _nhwc(gy, planes)
    (gx_ref,) = torch.autograd.grad(y_ref, xf, GY.float().permute(0, 3, 1, 2))
    GX = ops.maxpool_bwd(ARG, GY)
    assert _rel(GX.float().permute(0, 3, 1, 2), gx_ref) < tol
    # bilinear x2, align_corners=True
    xf2 = X.float().permute(0, 3, 1, 2).clone().requires_grad_(True)
    y_ref = F.interpolate(xf2, scale_factor=2, mode="bilinear", align_corners=True)
    Y = ops.upsample2x_fwd(X)
    assert _rel(Y.float().permute(0, 3, 1, 2), y_ref) < tol
    gy = torch.randn_like(y_ref)
    GY = _nhwc(gy, planes)
    (gx_ref,) = torch.autograd.grad(y_ref, xf2, GY.float().permute(0, 3, 1, 2))
    GX = ops.upsample2x_bwd(GY)
    assert _rel(GX.float().permute(0, 3, 1, 2), gx_ref) < tol
    # zero insertion and its transpose
    Z = ops.zero_insert(X)
    zf = Z.float()
    assert torch.equal(zf[:, ::2, ::2], X.float()) and float(zf[:, 1::2].abs().max()) == 0 and float(zf[:, :, 1::2].abs().max()) == 0
    assert torch.equal(ops.extract_even(Z).float(), X.float())
    torch.cuda.synchronize()


@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("H", [6, 8, 16, 32])  # 8 / 16 / 32: a sample split over a 4-CTA cluster (DSMEM), 6: single-CTA fallback
def test_groupnorm_relu(planes, H):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(11 + H)
    B = 3
    u = torch.randn(B, 128, H, H, device="cuda", generator=g) * 1.5 + 0.3
    gamma = (torch.rand(128, device="cuda", generator=g) + 0.5).requires_grad_(True)
    beta = (torch.randn(128, device="cuda", generator=g) * 0.1).requires_grad_(True)
    U = _nhwc(u, planes)
    uf = U.float().permute(0, 3, 1, 2).clone().requires_grad_(True)
    y_ref = F.relu(F.group_norm(uf, 32, gamma, beta, 1e-5))
    stats = torch.zeros(B, 32, 2, device="cuda")
    Y = ops.gn_relu_fwd(U, gamma.detach(), beta.detach(), stats)
    tol = 8e-3 if planes == 1 else 3e-5
    assert _rel(Y.float().permute(0, 3, 1, 2), y_ref) < tol
    gy = torch.randn_like(y_ref)
    GY = _nhwc(gy, planes)
    gu_ref, gg_ref, gb_ref = torch.autograd.grad(y_ref, (uf, gamma, beta), GY.float().permute(0, 3, 1, 2))
    dgamma, dbeta = torch.zeros(128, device="cuda"), torch.zeros(128, device="cuda")
    DU = ops.gn_relu_bwd(GY, Y, U, gamma.detach(), stats, dgamma, dbeta)
    torch.cuda.synchronize()
    tolb = 2e-2 if planes == 1 else 1e-4
    assert _rel(DU.float().permute(0, 3, 1, 2), gu_ref) < tolb
    assert _rel(dgamma, gg_ref) < tolb and _rel(dbeta, gb_ref) < tolb


def test_fused_ranger_matches_foreach_reference():
    """csrc/optim.cu gdrn_ranger_step (gradient centralisation + RAdam + lookahead in one launch per param group) against the
    torch._foreach restatement of lib/torch_utils/solver/ranger.py:100-200 (itself pinned to a literal per-parameter
    restatement in tests/test_module_api_cpu.py), over 14 steps (crosses the N_sma threshold and two lookahead syncs)."""
    from gdr_net_b200.solver import Ranger

    torch.manual_seed(0)
    shapes = [(64, 3, 7, 7), (128, 64, 3, 3), (16, 4608), (9, 8192), (512,), (69,), (3, 256), (3,), (1024, 128, 1, 1)]
    ps = [torch.randn(s, device="cuda") * 0.1 for s in shapes]
    a = [p.clone().requires_grad_(True) for p in ps]
    b = [p.clone().requires_grad_(True) for p in ps]
    oa = Ranger([{"params": a[:4], "lr": 1e-2}, {"params": a[4:], "lr": 3e-3, "weight_decay": 1e-2}], fused=True)
    ob = Ranger([{"params": b[:4], "lr": 1e-2}, {"params": b[4:], "lr": 3e-3, "weight_decay": 1e-2}], fused=False)
    flat = torch.zeros(sum(p.numel() for p in ps) + 3, device="cuda")[3:]  # deliberately 12-byte misaligned views
    for it in range(14):
        off = 0
        for x, y in zip(a, b):
            g = torch.randn_like(x)
            flat[off:off + x.numel()].copy_(g.flatten())
            x.grad = flat[off:off + x.numel()].view_as(x)
            y.grad = g.clone()
            off += x.numel()
        oa.step()
        ob.step()
    torch.cuda.synchronize()
    for x, y, s in zip(a, b, shapes):
        assert torch.allclose(x.detach(), y.detach(), rtol=2e-5, atol=2e-6), (s, float((x - y).abs().max()))
    for x, y in zip(a, b):
        for k in ("exp_avg", "exp_avg_sq", "slow_buffer"):
            assert torch.allclose(oa.state[x][k], ob.state[y][k], rtol=2e-5, atol=2e-7), k
        assert oa.state[x]["step"] == ob.state[y]["step"] == 14


def test_scale_f32_unaligned_slices():
    from gdr_net_b200.capi import C

    buf = torch.arange(1, 10001, device="cuda", dtype=torch.float32)
    ref = buf.clone()
    for lo, hi in ((0, 10000), (1, 9999), (3, 7), (5, 6), (2, 4099)):
        C.gdrn_scale_f32(buf.data_ptr() + 4 * lo, hi - lo, 0.5, torch.cuda.current_stream().cuda_stream)
        ref[lo:hi] *= 0.5
    torch.cuda.synchronize()
    assert torch.equal(buf, ref)


@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("with_res", [False, True])
def test_bn_relu_bitmask_roundtrip(planes, with_res):
    """bn_fwd emits the ReLU mask as one bit per element; bn_bwd fed with the bitmap (no activation read) gives the same du /
    dgamma / dbeta as the path that re-derives the mask from the stored activation."""
    from gdr_net_b200.capi import C

    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(77)
    N, H, C_ = 4, 16, 128
    U = _nhwc(torch.randn(N, C_, H, H, device="cuda", generator=g) * 2 + 0.3, planes)
    R = _nhwc(torch.randn(N, C_, H, H, device="cuda", generator=g), planes) if with_res else None
    gamma = torch.rand(C_, device="cuda", generator=g) + 0.5
    beta = torch.randn(C_, device="cuda", generator=g) * 0.3
    rm, rv = torch.zeros(C_, device="cuda"), torch.ones(C_, device="cuda")
    flat = U.float().reshape(-1, C_)
    stats = torch.stack([flat.sum(0), (flat * flat).sum(0)]).contiguous()
    mean, invstd = torch.empty(C_, device="cuda"), torch.empty(C_, device="cuda")
    Y = ops.like(U)
    mask = torch.zeros(U.numel() // 8, dtype=torch.uint8, device="cuda")
    C.gdrn_bn_fwd(U.hi_ptr, U.lo_ptr, R.hi_ptr if R else None, R.lo_ptr if R else None, Y.hi_ptr, Y.lo_ptr, stats.data_ptr(),
                  gamma.data_ptr(), beta.data_ptr(), rm.data_ptr(), rv.data_ptr(), mean.data_ptr(), invstd.data_ptr(),
                  mask.data_ptr(), flat.shape[0], C_, 1e-5, 0.1, 1, 1, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    bits = ((mask.view(-1, 1) >> torch.arange(8, device="cuda", dtype=torch.uint8)) & 1).reshape(-1)
    pos = (Y.float().reshape(-1) > 0)
    # the bitmap is taken from the fp32 pre-activation: it can only differ where a tiny positive value rounds to a 16-bit zero
    assert int((bits.bool() != pos).sum()) <= 2
    GY = _nhwc(torch.randn(N, C_, H, H, device="cuda", generator=g), planes)
    outs = []
    for use_bits in (False, True):
        sums = torch.zeros(2, C_, device="cuda")
        dgamma, dbeta = torch.zeros(C_, device="cuda"), torch.zeros(C_, device="cuda")
        DU, GOUT = ops.bn_bwd(GY, None, None if use_bits else Y, U, mean, invstd, gamma, sums, dgamma, dbeta, True, want_gout=True,
                              sums_zeroed=True, relu_mask=mask if use_bits else None)
        torch.cuda.synchronize()
        outs.append((DU.float(), GOUT.float(), dgamma.clone(), dbeta.clone()))
    assert int(((outs[0][0] - outs[1][0]).abs() > 1e-4).sum()) <= 4
    assert _rel(outs[1][1], outs[0][1]) < 1e-3 and _rel(outs[1][2], outs[0][2]) < 5e-2 and _rel(outs[1][3], outs[0][3]) < 5e-2


def test_pose_errors_match_pysixd_restatement():
    """gdrn_pose_errors (ADD / ADD-S / re / te on the device, one launch per batch) against the oracle's restatement of
    lib/pysixd/pose_error.py:297-337, 400-436 (numpy + scipy cKDTree per instance)."""
    import numpy as np

    from gdr_net_b200 import synth
    from gdr_net_b200.evaluator import pose_errors
    from oracle import gdrn_oracle as O

    g = synth._gen(9, "pose_errors")
    B, n = 6, 3000
    pts = (torch.rand(B, n, 3, generator=g) - 0.5) * 0.2
    R_gt = synth.random_rotations(B, g)
    R_est = torch.linalg.qr(R_gt + 0.05 * torch.randn(B, 3, 3, generator=g))[0]
    R_est = R_est * torch.sign(torch.linalg.det(R_est))[:, None, None]
    t_gt = torch.stack([torch.rand(B, generator=g) * 0.4 - 0.2, torch.rand(B, generator=g) * 0.4 - 0.2, 0.4 + torch.rand(B, generator=g)], 1)
    t_est = t_gt + 0.01 * torch.randn(B, 3, generator=g)
    out = pose_errors(R_est.cuda(), t_est.cuda(), R_gt.cuda(), t_gt.cuda(), pts.cuda())
    torch.cuda.synchronize()
    for i in range(B):
        args = (R_est[i].numpy(), t_est[i].numpy(), R_gt[i].numpy(), t_gt[i].numpy(), pts[i].numpy())
        add, adi = O.add_metric(*args), O.adi_metric(*args)
        assert abs(float(out["add"][i]) - add) <= 1e-5 * add + 1e-8, (i, float(out["add"][i]), add)
        assert abs(float(out["adi"][i]) - adi) <= 1e-5 * adi + 1e-8, (i, float(out["adi"][i]), adi)
        assert abs(float(out["re"][i]) - O._re_deg(R_est[i].numpy(), R_gt[i].numpy())) < 1e-3
        assert abs(float(out["te"][i]) - float(np.linalg.norm(t_gt[i].numpy() - t_est[i].numpy()))) < 1e-6


def test_roi_crop_and_targets_match_cv2_restatement():
    """f-3: gdr_net_b200.roi_targets (cv2.warpAffine's fixed-point sampling restated in two kernels) against the reference's own
    procedure run with cv2 / scipy (oracle/roi_oracle.py): nearest-sampled targets, region labels and the float crops exact (up to
    fp32 rounding), the uint8 image within one grey level on < 2 % of the values."""
    import numpy as np

    from gdr_net_b200.roi_targets import make_roi_batch
    from oracle import roi_oracle as RO

    rng = np.random.default_rng(3)
    B, H, W, F_ = 5, 480, 640, 64
    img = rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8)
    xyz = np.zeros((B, H, W, 3), np.float32)
    seg = np.zeros((B, H, W), np.float32)
    trunc = (rng.random((B, H, W)) > 0.2).astype(np.float32)
    centers = np.stack([rng.uniform(200, 440, B), rng.uniform(150, 330, B)], 1)  # float64, like the reference's aug_bbox output
    centers[4] = [30.3, 20.7]  # crop hanging over the image border
    scales = rng.uniform(90, 300, B)
    ext = rng.uniform(0.05, 0.3, (B, 3)).astype(np.float32)
    fps = ((rng.random((B, F_, 3)) - 0.5) * ext[:, None, :]).astype(np.float32)
    yy, xx = np.mgrid[0:H, 0:W]
    for b in range(B):
        blob = ((xx - centers[b, 0]) ** 2 + (yy - centers[b, 1]) ** 2) < (0.35 * scales[b]) ** 2  # noqa: E501
        xyz[b][blob] = ((rng.random((int(blob.sum()), 3)) - 0.5) * ext[b]).astype(np.float32)
        seg[b] = (blob & (rng.random((H, W)) > 0.1)).astype(np.float32)
    out = make_roi_batch(torch.from_numpy(img).cuda(), torch.from_numpy(xyz).cuda(), torch.from_numpy(seg).cuda(), torch.from_numpy(trunc).cuda(),
                         torch.from_numpy(centers).cuda(), torch.from_numpy(scales).cuda(), torch.from_numpy(ext).cuda(), torch.from_numpy(fps).cuda())
    torch.cuda.synchronize()
    for b in range(B):
        ref = RO.roi_instance(img[b], xyz[b], seg[b], trunc[b], centers[b], float(scales[b]), ext[b], fps[b])
        # The sampling positions are evaluated like cv2 (10-bit fixed point) from an inverse affine map obtained with the reference's
        # own operation sequence (float32 points, OpenCV's 6x6 LU, warpAffine's inversion -- bit-identical to cv2.getAffineTransform
        # on the host), so the nearest-sampled targets and labels are expected to be EXACT; the thresholds only leave room for a
        # stray pixel.
        for k in ("roi_mask_trunc", "roi_mask_visib", "roi_mask_obj"):
            assert (out[k][b].cpu().numpy() != ref[k]).mean() < 5e-4, (b, k)
        region_bad = out["roi_region"][b].cpu().numpy() != ref["roi_region"]
        assert region_bad.mean() < 5e-4, (b, region_bad.mean())
        dx = np.abs(out["roi_xyz"][b].cpu().numpy() - ref["roi_xyz"])
        assert (dx > 1e-6).mean() < 5e-4, (b, (dx > 1e-6).mean())
        dc = np.abs(out["roi_coord_2d"][b].cpu().numpy() - ref["roi_coord_2d"])
        assert dc.max() < 1.01 / (32.0 * (W - 1)) + 1e-6 and (dc > 1e-6).mean() < 5e-4, (b, dc.max(), (dc > 1e-6).mean())
        print(f"roi {b}: mask/region mismatches {int(region_bad.sum())}, coord max diff {dc.max():.1e}")
        d = np.abs(out["roi_img"][b].cpu().numpy() - ref["roi_img"]) * 255.0
        assert d.max() <= 1.0 + 1e-3 and (d > 0.5).mean() < 0.02, (b, d.max(), (d > 0.5).mean())
        assert abs(float(out["resize_ratio"][b]) - ref["resize_ratio"]) < 1e-6
    assert int(out["roi_region"].max()) > 1 and float(out["roi_mask_visib"].sum()) > 100
