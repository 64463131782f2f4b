"""GPU: the GroupNorm geometry head (ROT_HEAD.NORM = "GN", NUM_GN_GROUPS).

  * kernels: gdrn_head_gn_fwd / _bwd against float64 GroupNorm for HW in {256, 1024, 4096}, G in {1, 32, 64}, B in {4, 64}, one and
    two planes (output, statistics, dx, dgamma, dbeta), bit-identical over two runs;
  * model ("mixed"): the three cases of tests/golden/train_head_gn_b4.npz at B = 4 against the fixture and the oracle with the
    bounds of tests/test_regions_gpu.py, one B = 64 step against the oracle, a second identical step bit-identical;
  * inference: folded inference against the unfolded eval forward, its cached graph against eager;
  * CUDA graphs: GraphedTrainStep and the module API's graphs replay the eager losses and gradients bit for bit;
  * combinations: frozen backbone, frozen head, DropBlock, and the BatchNorm head calling none of the GroupNorm kernels."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import gemm_audit as GA  # noqa: E402 (tests/ is on sys.path)
from gdr_net_b200 import synth
from oracle import gdrn_oracle as O
from oracle import head_gn_oracle as HG
from oracle.make_golden_head_gn import EVAL_STRIDE, grad_sample_index
from test_head_gn_cpu import CASES, case_config, golden, make_batch, oracle_kwargs  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

REL = 1e-3
B64 = 64
# the output-conv bias gradient is a column sum with float atomics (gdrn_colsum): it may move in the last bits between runs
NONDET = ("rot_head_net.features.23.bias",)


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


# ------------------------------------------------------------------------------------------------ kernels
def _bits(mask, shape):
    """The ReLU bitmap as a bool tensor of `shape`."""
    m = mask.view(-1, 1).bitwise_right_shift(torch.arange(8, device=mask.device, dtype=torch.uint8)).bitwise_and(1)
    return m.view(shape).bool()


def _gn_case(B, HW, G, planes, seed):
    from gdr_net_b200 import ops

    H = int(HW ** 0.5)
    gen = torch.Generator(device="cuda").manual_seed(seed)
    # per-channel offsets: the variance is not the plain mean of squares
    u = torch.randn(B, H, H, 256, device="cuda", generator=gen) + 0.5 * torch.randn(256, device="cuda", generator=gen)
    g = torch.randn(B, H, H, 256, device="cuda", generator=gen) * 1e-2
    gamma = 0.5 + torch.rand(256, device="cuda", generator=gen)
    beta = 0.1 * torch.randn(256, device="cuda", generator=gen)
    return ops.PT.from_float(u, planes), ops.PT.from_float(g, planes), gamma, beta


def _run(U, Gd, gamma, beta, G):
    from gdr_net_b200 import ops

    y, stats, mask = ops.head_gn_relu_fwd(U, gamma, beta, G, want_mask=True)
    dgamma, dbeta = torch.full((256,), float("nan"), device="cuda"), torch.full((256,), float("nan"), device="cuda")
    du = ops.head_gn_relu_bwd(Gd, U, mask, gamma, stats, dgamma, dbeta)
    torch.cuda.synchronize()
    return y, stats, mask, du, dgamma, dbeta


@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("B", [4, B64])
@pytest.mark.parametrize("G", [1, 32, 64])
@pytest.mark.parametrize("HW", [256, 1024, 4096])
def test_head_gn_kernels_match_float64(HW, G, B, planes):
    U, Gd, gamma, beta = _gn_case(B, HW, G, planes, seed=HW + G + B + planes)
    y, stats, mask, du, dgamma, dbeta = _run(U, Gd, gamma, beta, G)
    H = U.shape[1]
    u64 = GA.pt64(U).view(B, HW, 256).permute(0, 2, 1).reshape(B, 256, H, H).requires_grad_(True)
    g64, ga64, be64 = GA.pt64(Gd).view(B, HW, 256).permute(0, 2, 1).reshape(B, 256, H, H), gamma.double(), beta.double()
    grp = u64.detach().reshape(B, G, -1)
    mean, var = grp.mean(-1), grp.var(-1, unbiased=False)
    assert (stats[..., 0].double() - mean).abs().max() <= 1e-5 * var.sqrt().max(), "mean"
    assert ((stats[..., 1].double() * (var + 1e-5).sqrt()) - 1).abs().max() <= 1e-5, "invstd"
    ga64.requires_grad_(True)
    be64.requires_grad_(True)
    z = F.group_norm(u64, G, ga64, be64, 1e-5)
    ref_y = F.relu(z).permute(0, 2, 3, 1).reshape(B, H, H, 256)
    r_y = _rel(GA.pt64(y), ref_y.detach())
    # dy through the kernel's own ReLU decisions (a value within rounding of 0 may go either way)
    m = _bits(mask, (B, H, H, 256))
    on = (ref_y.detach() > 0)
    assert (m != on).float().mean() <= 1e-5
    dz = (g64.permute(0, 2, 3, 1) * m).permute(0, 3, 1, 2)
    du64, dga, dbe = torch.autograd.grad(z, (u64, ga64, be64), dz)
    r_du = _rel(GA.pt64(du).view(B, H, H, 256), du64.permute(0, 2, 3, 1))
    r_dg, r_db = _rel(dgamma, dga), _rel(dbeta, dbe)
    print(f"HW={HW} G={G} B={B} planes={planes}: y {r_y:.2e} du {r_du:.2e} dgamma {r_dg:.2e} dbeta {r_db:.2e}")
    tol = 2e-3 if planes == 1 else 1e-5
    assert r_y <= tol and r_du <= tol, (r_y, r_du)
    assert r_dg <= 1e-5 and r_db <= 1e-5, (r_dg, r_db)
    again = _run(U, Gd, gamma, beta, G)
    for a, b in zip((y.buf, stats, mask, du.buf, dgamma, dbeta), (again[0].buf, *again[1:3], again[3].buf, *again[4:])):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------ model level
def _model(case, sd=None, precision="mixed", **kw):
    from gdr_net_b200 import GDRN as G

    model, _ = G.build_model_optimizer(case_config(case, device="cuda", **kw), precision=precision)
    if sd is None:
        sd = synth.seeded_state_dict({k: v.cpu() for k, v in model.state_dict().items()}, seed=CASES[case][3])
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
    o = HG.gdrn_forward(leaf, b, train=True, do_loss=True, update_stats=True, **oracle_kwargs(case))
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
        assert r_g < 0.06 and r_o < 0.06, (name, r_g, r_o)  # the bound of tests/test_regions_gpu.py
    for name in [f"rot_head_net.features.{i}.{w}" for i in HG.NORM_AT for w in ("weight", "bias")]:
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
    case = "ship_g32"
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


def test_folded_inference_matches_unfolded_and_its_graph_matches_eager():
    model, _ = _model("ship_g32", use_pnp_test=True)
    model.eval()
    batch = _cuda(synth.make_batch(B64, seed=5))
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
def test_graphs_replay_eager_bit_for_bit():
    from gdr_net_b200.engine import GraphedTrainStep

    batch = _cuda(make_batch("r8_noatt_g1"))
    results, sd = {}, None
    for graphs in (False, True):
        model, sd = _model("r8_noatt_g1", sd=sd)
        model.train()
        model.use_cuda_graphs = graphs
        for _ in range(2):
            ld = _train_step(model, batch)
        results[graphs] = (ld, {n: p.grad.clone() for n, p in model.named_parameters()})
    assert results[True][0] == results[False][0]
    for n, v in results[False][1].items():
        if n.startswith(("rot_head_net.", "backbone.")) and n not in NONDET:
            assert torch.equal(results[True][1][n], v), n
    # GraphedTrainStep: one graph for forward + backward
    model, _ = _model("r8_noatt_g1", sd=sd)
    model.train()
    eng = model.engine
    kw = synth.forward_kwargs(batch, train=True)
    names = ["roi_coord_2d", "roi_cams", "roi_centers", "roi_whs", "roi_extents", "resize_ratios", "gt_xyz", "gt_mask_trunc",
             "gt_mask_visib", "gt_mask_obj", "gt_region", "gt_ego_rot", "gt_points", "gt_trans", "gt_trans_ratio"]
    aux = {k: (kw[k].float().contiguous() if kw[k].dtype != torch.long else kw[k]) for k in names}
    aux["sym_infos"] = None
    x = batch["roi_img"].float().contiguous()
    step = GraphedTrainStep(eng, x, aux, train_bn=True)
    losses = step().clone()
    g_graph = {n: eng.grads[n].clone() for n, _ in eng.named_params if n.startswith("rot_head_net.") and n not in NONDET}
    res = eng.forward(x, aux, train_bn=True, do_loss=True)
    eng.backward(torch.ones(len(eng.loss_names), device="cuda"))
    torch.cuda.synchronize()
    assert torch.equal(res["losses"], losses)
    for n, v in g_graph.items():
        assert torch.equal(eng.grads[n], v), n


# ------------------------------------------------------------------------------------------------ combinations
def test_frozen_backbone_and_frozen_head():
    case = "ship_g32"
    batch_cpu = make_batch(case)
    batch = _cuda(batch_cpu)
    _, sd = _model(case)
    _o, leaf = _oracle_train(case, sd, batch_cpu)
    # frozen backbone: the head and Patch-PnP gradients are those of the unfrozen model (the backbone still uses batch statistics)
    model, _ = _model_frozen(case, sd, backbone=True)
    model.train()
    _train_step(model, batch)
    for n, p in model.named_parameters():
        if n.startswith("backbone."):
            assert p.grad is None, n
        else:
            assert _rel(p.grad, leaf[n].grad) < 0.06, n
    # frozen head: forward only, no head gradient, Patch-PnP gradients still flow
    model = _model_frozen(case, sd, head=True)[0]
    model.train()
    ld = _train_step(model, batch)
    assert "loss_coor_x" not in ld and all(np.isfinite(list(ld.values())))
    for n, p in model.named_parameters():
        if n.startswith(("backbone.", "rot_head_net.")):
            assert p.grad is None, n
        else:
            assert p.grad is not None and torch.isfinite(p.grad).all(), n


def _model_frozen(case, sd, backbone=False, head=False):
    from gdr_net_b200 import GDRN as G

    cfg = case_config(case, device="cuda")
    cfg.MODEL.CDPN.BACKBONE.FREEZE = backbone
    cfg.MODEL.CDPN.ROT_HEAD.FREEZE = head
    model, _ = G.build_model_optimizer(cfg, precision="mixed")
    model.load_state_dict(sd)
    return model, sd


def test_dropblock_and_class_aware_with_gn():
    from gdr_net_b200 import GDRN as G

    cfg = case_config("bce_rot_g64", device="cuda")
    cfg.MODEL.CDPN.PNP_NET.PNP_HEAD_CFG.drop_prob = 0.25
    model, _ = G.build_model_optimizer(cfg, precision="mixed")
    model.load_state_dict(_model("bce_rot_g64")[1])
    model.pnp_net.dropblock_step = 4999
    model.train()
    batch = _cuda(make_batch("bce_rot_g64"))
    ld = _train_step(model, batch)
    assert all(np.isfinite(list(ld.values())))
    assert model.pnp_net.dropblock_keep is not None and not bool(model.pnp_net.dropblock_keep.all())
    for i in HG.NORM_AT:
        for w in ("weight", "bias"):
            gr = model.rot_head_net.features[i].get_parameter(w).grad
            assert torch.isfinite(gr).all() and gr.abs().sum() > 0, (i, w)


def test_bn_head_runs_no_groupnorm_kernel(monkeypatch):
    from gdr_net_b200 import GDRN as G
    from gdr_net_b200 import ops
    from gdr_net_b200.config import a6_config

    calls = []
    for name in ("head_gn_relu_fwd", "head_gn_relu_bwd"):
        fn = getattr(ops, name)
        monkeypatch.setattr(ops, name, lambda *a, _fn=fn, _n=name, **k: (calls.append(_n), _fn(*a, **k))[1])
    batch = _cuda(synth.make_batch(4, seed=3))
    counts = {}
    for norm in ("BN", "GN"):
        cfg = a6_config(device="cuda")
        cfg.MODEL.CDPN.ROT_HEAD.NORM = norm
        model, _ = G.build_model_optimizer(cfg, precision="mixed")
        model.train()
        del calls[:]
        _train_step(model, batch)
        counts[norm] = len(calls)
        eng = model.engine
        assert len(eng._bn_mods) == (43 if norm == "BN" else 36)
        assert all(not k.startswith("rot_head_net.") for k, _ in eng._conv_bn_pairs()) == (norm == "GN")
    assert counts == {"BN": 0, "GN": 14}
