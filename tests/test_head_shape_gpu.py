"""GPU: the geometry head's shape switches (ROT_HEAD.CONV_KERNEL_SIZE = 2 | 3 | 4, OUT_CONV_KERNEL_SIZE = 1 | 3).

  * ops against float64 on the operands' exact values, each run twice and compared bit for bit:
      - gdrn_conv_dgrad_s2 as the k2 / k4 ConvTranspose2d forward, one and two planes, B in {4, 64}, plain, with the BatchNorm
        statistics epilogue and with the folded bias + ReLU epilogue;
      - the stride-2 conv dgrad and wgrad of the k2 / k4 deconv's backward;
      - the 3x3 output conv forward (fp32 logits, ldc 72), dgrad and wgrad, plain and grouped per crop class (the wgrad split at
        crop boundaries);
  * model ("mixed"): the four cases of tests/golden/train_head_shape_b4.npz at B = 4 against the fixture and the oracle with the
    bounds of tests/test_head_gn_gpu.py, one B = 64 step of k4 / 3x3 against the oracle, a second step bit-identical;
  * paths: folded inference against unfolded and its graph against eager, GraphedTrainStep and the module API's graphs against
    eager, frozen backbone / head, DropBlock."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import gemm_audit as GA  # noqa: E402 (tests/ is on sys.path)
from gdr_net_b200 import synth
from oracle import gdrn_oracle as O
from oracle import head_shape_oracle as HS
from oracle.make_golden_head_shape import EVAL_STRIDE, grad_sample_index
from test_head_shape_cpu import CASES, golden, make_batch, oracle_kwargs  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

REL = 1e-3
B64 = 64
# the class-agnostic output-conv bias gradient is a column sum with float atomics (gdrn_colsum): it may move in the last bits
NONDET = ("rot_head_net.features.23.bias",)
# the B = 64 / path cases: k4 deconv with a 3x3 output conv on the shipped head otherwise, and the k2 / 3x3 head
EXTRA = {"k4_o3": ("k4_o1", dict(OUT_CONV_KERNEL_SIZE=3)), "k2_o3": ("k2_o3_r8", {})}


@pytest.fixture(scope="module", autouse=True)
def _gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _cuda(batch):
    return {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in batch.items()}


# ------------------------------------------------------------------------------------------------ ops
def _pt(x, planes):
    from gdr_net_b200 import ops

    return ops.PT.from_float(x.contiguous(), planes)


def _w64(w, planes):
    """The value a packed weight operand holds: the 16-bit rounding with one plane, fp32 (to 2^-22) with two."""
    from gdr_net_b200 import ops

    return (ops.round_storage(w) if planes == 1 else w).double()


def _tol(planes):
    return 1e-3 if planes == 1 else 1e-5  # one plane: the 16-bit output rounding; two planes: 22-bit operands and output


def _nchw(t):
    return t.permute(0, 3, 1, 2)


@pytest.mark.parametrize("epi", ["plain", "stats", "bias_relu"])
@pytest.mark.parametrize("B", [4, B64])
@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("k", [2, 4])
def test_deconv_forward_matches_float64(k, planes, B, epi):
    from gdr_net_b200 import ops

    pad, op = HS.DECONV_PADDING[k]
    gen = torch.Generator(device="cuda").manual_seed(1000 * k + 10 * planes + B)
    z = torch.randn(B, 8, 8, 512, device="cuda", generator=gen)
    w = torch.randn(512, 256, k, k, device="cuda", generator=gen) * (2.0 / (512 * k * k / 4)) ** 0.5
    bias = 0.1 * torch.randn(256, device="cuda", generator=gen)
    Z = _pt(z, planes)

    def run():
        stats = torch.zeros(2, 256, dtype=torch.float64, device="cuda") if epi == "stats" else None
        out = ops.conv_dgrad_s2(Z, ops.pack_conv_dgrad(w, planes), 256, k, pad, stats=stats,
                                bias=bias if epi == "bias_relu" else None, act=2 if epi == "bias_relu" else 0)
        torch.cuda.synchronize()
        return out, stats

    out, stats = run()
    ref = F.conv_transpose2d(_nchw(GA.pt64(Z)), _w64(w, planes), None, stride=2, padding=pad, output_padding=op)
    if epi == "bias_relu":
        ref = F.relu(ref + bias.double().view(1, -1, 1, 1))
    got = _nchw(GA.pt64(out))
    assert got.shape == ref.shape == (B, 256, 16, 16)
    r = _rel(got, ref)
    print(f"k={k} planes={planes} B={B} {epi}: rel-L2 {r:.2e}")
    assert r <= _tol(planes), r
    if epi == "stats":  # sum and sum of squares per channel of the output the kernel wrote, in every phase
        for ph_a in (0, 1):
            for ph_b in (0, 1):
                assert _rel(got[:, :, ph_a::2, ph_b::2], ref[:, :, ph_a::2, ph_b::2]) <= _tol(planes)
        # from the fp32 accumulators, before the output is rounded to its planes
        assert _rel(stats[0], ref.sum((0, 2, 3))) <= 1e-4 and _rel(stats[1], (ref * ref).sum((0, 2, 3))) <= 1e-4
    again, _ = run()
    assert torch.equal(out.buf, again.buf)


@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("k", [2, 4])
def test_deconv_backward_matches_float64(k, planes):
    """The deconv's input gradient (the stride-2 conv over du) and weight gradient (the stride-2 conv wgrad, du as the input)."""
    from gdr_net_b200 import ops

    pad, op = HS.DECONV_PADDING[k]
    B = B64
    gen = torch.Generator(device="cuda").manual_seed(2000 * k + planes)
    z = torch.randn(B, 8, 8, 512, device="cuda", generator=gen)
    du = torch.randn(B, 16, 16, 256, device="cuda", generator=gen)
    w = torch.randn(512, 256, k, k, device="cuda", generator=gen) * 0.05
    Z, DU = _pt(z, planes), _pt(du, planes)
    ws = ops.Workspace("cuda")

    def run():
        g = ops.conv_fwd(DU, ops.pack_deconv_dgrad(w, planes), 512, k, k, 2, pad)
        dw = torch.full_like(w, float("nan"))
        buf, ks, kss = ops.conv_wgrad(Z, DU, ws, 512, k, k, 2, pad)
        ops.unpack_wgrad(buf, dw, 512, 256, k, k, 256, ks, kss, 256 * k * k, k * k, k, 1)
        torch.cuda.synchronize()
        return g, dw

    g, dw = run()
    z64, w64 = _nchw(GA.pt64(Z)).requires_grad_(True), _w64(w, planes).requires_grad_(True)
    out = F.conv_transpose2d(z64, w64, None, stride=2, padding=pad, output_padding=op)
    dz_ref, dw_ref = torch.autograd.grad(out, (z64, w64), _nchw(GA.pt64(DU)))
    r_g, r_w = _rel(_nchw(GA.pt64(g)), dz_ref), _rel(dw, dw_ref)
    print(f"k={k} planes={planes}: dgrad {r_g:.2e} wgrad {r_w:.2e}")
    assert r_g <= _tol(planes) and r_w <= 1e-5, (r_g, r_w)
    g2, dw2 = run()
    assert torch.equal(g.buf, g2.buf) and torch.equal(dw, dw2)


def _out_conv_case(planes, C_, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    B, n, npad = 4, 69, 128
    x = torch.relu(torch.randn(B, 64, 64, 256, device="cuda", generator=gen))
    w = torch.randn(C_ * npad, 256, 3, 3, device="cuda", generator=gen) * 0.02
    bias = 0.1 * torch.randn(C_ * npad, device="cuda", generator=gen)
    for c in range(C_):  # rows beyond n of every class block are padding
        w[c * npad + n:(c + 1) * npad] = 0
        bias[c * npad + n:(c + 1) * npad] = 0
    dlog = torch.zeros(B * 4096, 128, device="cuda")
    dlog[:, :n] = 1e-2 * torch.randn(B * 4096, n, device="cuda", generator=gen)
    return B, n, npad, _pt(x, planes), w, bias, _pt(dlog, planes)


@pytest.mark.parametrize("planes", [1, 2])
def test_output_conv_3x3_matches_float64(planes):
    from gdr_net_b200 import ops

    B, n, npad, X, w, bias, DL = _out_conv_case(planes, 1, 3000 + planes)
    w, bias = w[:n], bias[:n]
    ws = ops.Workspace("cuda")

    def run():
        logits = torch.full((B * 4096, 72), float("nan"), device="cuda")
        ops.conv_fwd(X, ops.pack_conv_fwd(w, planes), n, 3, 3, 1, 1, out_f32=logits, bias=bias, ldc=72, want_planes=False)
        g = ops.conv_fwd(DL.view(B, 64, 64, 128), ops.pack_conv_dgrad(w, planes, ipad=128), 256, 3, 3, 1, 1)
        dw = torch.full_like(w, float("nan"))
        buf, ks, kss = ops.conv_wgrad(DL.view(B, 64, 64, 128), X, ws, n, 3, 3, 1, 1)
        ops.unpack_wgrad(buf, dw, n, 256, 3, 3, 256, ks, kss, 256 * 9, 9, 3, 1)
        torch.cuda.synchronize()
        return logits, g, dw

    logits, g, dw = run()
    x64, w64 = _nchw(GA.pt64(X)).requires_grad_(True), _w64(w, planes).requires_grad_(True)
    y = F.conv2d(x64, w64, bias.double(), padding=1)
    d64 = _nchw(GA.pt64(DL).view(B, 64, 64, 128)[..., :n])
    dx_ref, dw_ref = torch.autograd.grad(y, (x64, w64), d64)
    r_y = _rel(_nchw(logits.view(B, 64, 64, 72)[..., :n]), y.detach())
    r_g, r_w = _rel(_nchw(GA.pt64(g)), dx_ref), _rel(dw, dw_ref)
    print(f"3x3 output conv planes={planes}: fwd {r_y:.2e} dgrad {r_g:.2e} wgrad {r_w:.2e}")
    assert r_y <= (1e-5 if planes == 2 else 1e-4) and r_g <= _tol(planes) and r_w <= 1e-5, (r_y, r_g, r_w)
    again = run()
    assert torch.equal(logits.nan_to_num(), again[0].nan_to_num()) and torch.equal(g.buf, again[1].buf) and torch.equal(dw, again[2])


@pytest.mark.parametrize("planes", [1, 2])
def test_grouped_output_conv_3x3_matches_float64(planes):
    from gdr_net_b200 import ops
    from gdr_net_b200.engine import _PlaneRows

    C_ = 3
    B, n, npad, X, w, bias, DL = _out_conv_case(planes, C_, 4000 + planes)
    cls = torch.tensor([2, 0, 2, 1], dtype=torch.int32, device="cuda")
    ws = ops.Workspace("cuda")

    def run():
        logits = torch.full((B * 4096, 72), float("nan"), device="cuda")
        ops.conv_fwd_grouped(X, ops.pack_conv_fwd(w, planes), n, npad, cls, 4096, out_f32=logits, bias=bias, bias_stride=npad, ldc=72,
                             k=3)
        wd = ops.PT((C_ * 256, 9 * 128), planes, device="cuda")
        for c in range(C_):
            ops.pack_conv_dgrad(w[c * npad:(c + 1) * npad], planes, out=_PlaneRows(wd, c * 256), ipad=128)
        g = ops.conv_fwd_grouped(DL.view(B, 64, 64, 128), wd, 256, 256, cls, 4096, k=3)
        buf, ks, kss = ops.conv_wgrad(DL.view(B, 64, 64, 128), X, ws, n, 3, 3, 1, 1, ksplit=B)
        torch.cuda.synchronize()
        return logits, g, buf[:ks * kss].clone(), ks, kss

    logits, g, part, ks, kss = run()
    assert ks == B
    x64, d64 = _nchw(GA.pt64(X)), _nchw(GA.pt64(DL).view(B, 64, 64, 128))
    for b in range(B):  # crop b: its class's block of the weights, its own wgrad partial
        c = int(cls[b])
        wb = _w64(w[c * npad:c * npad + n], planes).requires_grad_(True)
        xb = x64[b:b + 1].clone().requires_grad_(True)
        y = F.conv2d(xb, wb, bias[c * npad:c * npad + n].double(), padding=1)
        dx_ref, dw_ref = torch.autograd.grad(y, (xb, wb), d64[b:b + 1, :n])
        r_y = _rel(_nchw(logits.view(B, 64, 64, 72)[b:b + 1, ..., :n]), y.detach())
        r_g = _rel(_nchw(GA.pt64(g)[b:b + 1]), dx_ref)
        # the partial of crop b is [row][tap][ci] (tap-major), rows padded to 128
        pw = part[b * kss:(b + 1) * kss].view(128, 9, 256)[:n]
        r_w = _rel(pw, dw_ref.permute(0, 2, 3, 1).reshape(n, 9, 256))
        print(f"grouped 3x3 planes={planes} crop {b} class {c}: fwd {r_y:.2e} dgrad {r_g:.2e} wgrad partial {r_w:.2e}")
        assert r_y <= (1e-5 if planes == 2 else 1e-4) and r_g <= _tol(planes) and r_w <= 1e-5, (b, r_y, r_g, r_w)
    again = run()
    assert torch.equal(logits.nan_to_num(), again[0].nan_to_num()) and torch.equal(g.buf, again[1].buf) and torch.equal(part, again[2])


# ------------------------------------------------------------------------------------------------ model level
def _config(case, device="cuda", **kw):
    from test_head_shape_cpu import case_config

    base, over = EXTRA.get(case, (case, {}))
    cfg = case_config(base, device=device, **kw)
    for k, v in over.items():
        setattr(cfg.MODEL.CDPN.ROT_HEAD, k, v)
    return cfg


def _oracle_kwargs(case):
    base, over = EXTRA.get(case, (case, {}))
    kw = oracle_kwargs(base)
    if "OUT_CONV_KERNEL_SIZE" in over:
        kw["k_out"] = over["OUT_CONV_KERNEL_SIZE"]
    return kw


def _model(case, sd=None, precision="mixed", freeze=(), drop_prob=0.0, **kw):
    from gdr_net_b200 import GDRN as G

    cfg = _config(case, **kw)
    for part in freeze:
        getattr(cfg.MODEL.CDPN, part).FREEZE = True
    if drop_prob:
        cfg.MODEL.CDPN.PNP_NET.PNP_HEAD_CFG.drop_prob = drop_prob
    model, _ = G.build_model_optimizer(cfg, precision=precision)
    if sd is None:
        sd = synth.seeded_state_dict({k: v.cpu() for k, v in model.state_dict().items()}, seed=CASES[EXTRA.get(case, (case,))[0]][3])
    model.load_state_dict(sd)
    return model, sd


def _train_step(model, batch):
    for p in model.parameters():
        p.grad = None
    _, ld = model(batch["roi_img"], **synth.forward_kwargs(batch, train=True))
    sum(ld.values()).backward()
    torch.cuda.synchronize()
    return {k: float(v.detach()) for k, v in ld.items()}


def _oracle_train(case, sd, batch_cpu):
    """The oracle's losses and gradients in float64 on the GPU."""
    leaf = O.leaf_state_dict({k: v.cuda() for k, v in sd.items()}, dtype=torch.float64)
    b = {k: (v.cuda().double() if isinstance(v, torch.Tensor) and v.dtype.is_floating_point else
             v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in batch_cpu.items()}
    o = HS.gdrn_forward(leaf, b, train=True, do_loss=True, update_stats=True, **_oracle_kwargs(case))
    sum(o["losses"].values()).backward()
    return {k: float(v.detach()) for k, v in o["losses"].items()}, leaf


def _eval(model, batch):
    with torch.no_grad():
        out = model(batch["roi_img"], **synth.forward_kwargs(batch, train=False))
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("case", list(CASES))
def test_b4_matches_golden_and_oracle(case, golden_dir):
    g = golden(golden_dir, case)
    model, sd = _model(case)
    batch_cpu = make_batch(case)
    batch = _cuda(batch_cpu)
    model.train()
    ld = _train_step(model, batch)
    o_losses, leaf = _oracle_train(case, sd, batch_cpu)
    for k, v in ld.items():
        ref = float(g["loss/" + k])
        print(f"[{case}] B=4 {k}: {v:.6f} vs golden {ref:.6f} rel {abs(v - ref) / abs(ref):.2e}")
        assert abs(v - ref) <= 2 * REL * abs(ref), (k, v, ref)
        assert abs(v - o_losses[k]) <= 2 * REL * abs(ref), k
    for name, p in model.named_parameters():
        mine = p.grad.reshape(-1)
        r_g = _rel(mine[torch.as_tensor(grad_sample_index(mine.numel()), device="cuda")], g["grad/" + name])
        r_o = _rel(p.grad, leaf[name].grad)
        assert r_g < 0.06 and r_o < 0.06, (name, r_g, r_o)  # the bound of tests/test_head_gn_gpu.py
    for name in ("rot_head_net.features.0.weight", "rot_head_net.features.23.weight", "rot_head_net.features.23.bias"):
        print(f"[{case}] grad {name}: rel-L2 vs oracle {_rel(dict(model.named_parameters())[name].grad, leaf[name].grad):.2e}")
    model, _ = _model(case, sd=sd, use_pnp_test=True)
    model.eval()
    for fold in (True, False):
        model.engine.fold_eval = fold
        out = _eval(model, batch)
        head = torch.cat([out["mask"], out["coor_x"], out["coor_y"], out["coor_z"], out["region"]], dim=1)[:, :, ::EVAL_STRIDE, ::EVAL_STRIDE].cpu()
        r, rr, rt = _rel(head, g["eval/head"]), _rel(out["rot"], g["eval/rot"]), _rel(out["trans"], g["eval/trans"])
        print(f"[{case}] eval fold={fold} head rel-L2 vs golden {r:.2e}, rot {rr:.2e}, trans {rt:.2e}")
        assert r < REL and rr < 2e-3 and rt < 2e-3


def test_b64_step_matches_oracle_and_repeats_bit_identically():
    case = "k4_o3"
    model, sd = _model(case)
    batch_cpu = synth.make_batch(B64, seed=100)
    o_losses, leaf = _oracle_train(case, sd, batch_cpu)
    model.train()
    batch = _cuda(batch_cpu)
    ld = _train_step(model, batch)
    g1 = {n: p.grad.clone() for n, p in model.named_parameters()}
    for k, v in ld.items():
        ref = o_losses[k]
        print(f"[{case}] B=64 {k}: {v:.6f} vs {ref:.6f} rel {abs(v - ref) / abs(ref):.2e}")
        assert abs(v - ref) <= REL * abs(ref), (k, v, ref)
    for name, p in model.named_parameters():
        assert _rel(p.grad, leaf[name].grad) < 0.06, name
    ld2 = _train_step(model, batch)
    assert ld2 == ld
    for n, p in model.named_parameters():
        if n.startswith(("rot_head_net.", "backbone.")) and n not in NONDET:
            assert torch.equal(p.grad, g1[n]), n


@pytest.mark.parametrize("case", ["k4_o3", "k3_o3_ca"])
def test_folded_inference_matches_unfolded_and_its_graph_matches_eager(case):
    model, _ = _model(case, use_pnp_test=True)
    model.eval()
    batch = _cuda(make_batch(case) if case in CASES else synth.make_batch(B64, seed=5))
    model.engine.fold_eval = False
    ref = _eval(model, batch)
    model.engine.fold_eval = True
    eager = _eval(model, batch)
    for k in ("rot", "trans", "mask", "coor_x", "region"):
        assert _rel(eager[k], ref[k]) < REL, k
    model.use_cuda_graphs = True
    for _ in range(2):
        out = _eval(model, batch)
        for k in ("rot", "trans", "mask", "coor_x", "region"):
            assert torch.equal(out[k], eager[k]), k
    assert len(model.engine._eval_graphs) == 1


# ------------------------------------------------------------------------------------------------ CUDA graphs
@pytest.mark.parametrize("case", ["k2_o3_r8", "k3_o3_ca"])
def test_graphs_replay_eager_bit_for_bit(case):
    from gdr_net_b200.engine import GraphedTrainStep

    batch = _cuda(make_batch(case))
    nondet = NONDET if case != "k3_o3_ca" else ()  # the class-aware bias gradient is reduced in crop order
    results, sd = {}, None
    for graphs in (False, True):
        model, sd = _model(case, sd=sd)
        model.train()
        model.use_cuda_graphs = graphs
        for _ in range(2):
            ld = _train_step(model, batch)
        results[graphs] = (ld, {n: p.grad.clone() for n, p in model.named_parameters()})
    assert results[True][0] == results[False][0]
    for n, v in results[False][1].items():
        if n.startswith(("rot_head_net.", "backbone.")) and n not in nondet:
            assert torch.equal(results[True][1][n], v), n
    # GraphedTrainStep: one graph for forward + backward
    model, _ = _model(case, sd=sd)
    model.train()
    eng = model.engine
    kw = synth.forward_kwargs(batch, train=True)
    names = ["roi_coord_2d", "roi_cams", "roi_centers", "roi_whs", "roi_extents", "resize_ratios", "gt_xyz", "gt_mask_trunc",
             "gt_mask_visib", "gt_mask_obj", "gt_region", "gt_ego_rot", "gt_points", "gt_trans", "gt_trans_ratio"]
    aux = {k: (kw[k].float().contiguous() if kw[k].dtype != torch.long else kw[k]) for k in names}
    aux["sym_infos"] = None
    if eng.class_aware:
        aux["roi_classes"] = eng._classes(kw["roi_classes"], batch["roi_img"].shape[0])
    x = batch["roi_img"].float().contiguous()
    step = GraphedTrainStep(eng, x, aux, train_bn=True)
    losses = step().clone()
    g_graph = {n: eng.grads[n].clone() for n, _ in eng.named_params if n.startswith("rot_head_net.") and n not in nondet}
    res = eng.forward(x, aux, train_bn=True, do_loss=True)
    eng.backward(torch.ones(len(eng.loss_names), device="cuda"))
    torch.cuda.synchronize()
    assert torch.equal(res["losses"], losses)
    for n, v in g_graph.items():
        assert torch.equal(eng.grads[n], v), n


# ------------------------------------------------------------------------------------------------ combinations
def test_frozen_backbone_and_frozen_head():
    case = "k4_o3"
    batch_cpu = synth.make_batch(4, seed=7)
    batch = _cuda(batch_cpu)
    _, sd = _model(case)
    _o, leaf = _oracle_train(case, sd, batch_cpu)
    # frozen backbone: the head and Patch-PnP gradients are those of the unfrozen model (the backbone still uses batch statistics)
    model, _ = _model(case, sd, freeze=("BACKBONE",))
    model.train()
    _train_step(model, batch)
    for n, p in model.named_parameters():
        if n.startswith("backbone."):
            assert p.grad is None, n
        else:
            assert _rel(p.grad, leaf[n].grad) < 0.06, n
    # frozen head: forward only, no head gradient, Patch-PnP gradients match the oracle's
    model, _ = _model(case, sd, freeze=("ROT_HEAD",))
    model.train()
    ld = _train_step(model, batch)
    assert "loss_coor_x" not in ld and all(np.isfinite(list(ld.values())))
    for n, p in model.named_parameters():
        if n.startswith(("backbone.", "rot_head_net.")):
            assert p.grad is None, n
        else:
            assert p.grad is not None and torch.isfinite(p.grad).all(), n


def test_dropblock_with_k2_and_3x3_output_conv():
    model, _ = _model("k2_o3", drop_prob=0.25)
    model.pnp_net.dropblock_step = 4999
    model.train()
    batch = _cuda(make_batch("k2_o3_r8"))
    ld = _train_step(model, batch)
    assert all(np.isfinite(list(ld.values())))
    assert model.pnp_net.dropblock_keep is not None and not bool(model.pnp_net.dropblock_keep.all())
    for i in (0, 23):
        gr = model.rot_head_net.features[i].weight.grad
        assert torch.isfinite(gr).all() and gr.abs().sum() > 0, i
