"""GPU: class-aware geometry heads (ROT_HEAD.*_CLASS_AWARE).

  * op level: the grouped output conv and its grouped dgrad against float64 per-crop products with each crop's class block (B = 64,
    13 classes present and 3 absent, both forward tile widths, one and two planes), with the bounds of tests/gemm_audit.py; the
    per-crop weight / bias gradient reduction against a float64 segmented sum, bit-identical over two runs, 0 for absent classes;
  * exactness: per crop, the class-aware logits (the TEST.USE_PNP maps), rot and trans are bit-identical to those of a
    class-agnostic model whose output conv holds that crop's class rows;
  * model level ("mixed"): the three cases of tests/golden/train_class_aware_b4.npz at B = 4 with the bounds of
    tests/test_regions_gpu.py, one B = 64 step against the oracle within 1e-3, and a second identical step bit-identical;
  * CUDA graphs: train-step and folded-inference replays follow a change of roi_classes without a new capture."""
import math

import numpy as np
import pytest
import torch

import gemm_audit as GA  # noqa: E402 (tests/ is on sys.path)
from gdr_net_b200 import synth
from oracle import class_aware_oracle as CA
from oracle import gdrn_oracle as O
from test_class_aware_cpu import CASES, absent_rows, case_config, golden, make_batch, oracle_kwargs  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

REL = 1e-3
B64 = 64
# Gradients compared bit for bit between runs: the class-aware output conv's (summed in crop order) and those of
# tests/test_regions_gpu.py.  The GroupNorm and Patch-PnP FC bias gradients are added with float atomics (gdrn_gn_relu_bwd,
# gdrn_colsum) and may move in the last bits from run to run.
DET_GRADS = ("rot_head_net.features.23.weight", "rot_head_net.features.23.bias", "rot_head_net.features.20.weight",
             "backbone.layer1.0.conv1.weight", "pnp_net.features.0.weight")


@pytest.fixture(scope="module", autouse=True)
def _gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    torch.backends.cuda.matmul.allow_tf32 = False


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _cuda(batch):
    return {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in batch.items()}


def _classes64():
    """B = 64 crops over classes 0..12 in mixed order (13..15 exist in the tables but no crop uses them)."""
    return ((torch.arange(B64) * 5) % 13).to(torch.int32).cuda()


# ------------------------------------------------------------------------------------------------ op level
@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("n_out", [69, 13])  # Cout_pad 128 (128-wide tiles) and 64 (64-wide tiles)
def test_grouped_output_conv_matches_float64(planes, n_out):
    from gdr_net_b200 import ops

    G, npad = 16, -(-n_out // 64) * 64
    gen = torch.Generator(device="cuda").manual_seed(11 + n_out + planes)
    x = GA.relu_like((B64, 64, 64, 256), gen, planes)
    w = GA.row_scaled((G * npad, 256), gen)
    bias = torch.randn(G * npad, device="cuda", generator=gen)
    wp = ops.pack_conv_fwd(w.view(G * npad, 256, 1, 1), planes)
    cls = _classes64()
    out = torch.full((B64 * 4096 + 8, 72), math.nan, device="cuda")
    ops.conv_fwd_grouped(x, wp, n_out, npad, cls, 4096, out_f32=out[:B64 * 4096], bias=bias, bias_stride=npad, ldc=72)
    torch.cuda.synchronize()
    assert torch.isnan(out[B64 * 4096:]).all()  # guard rows
    wq = GA.pt64(wp).view(G, npad, 256)[cls.long(), :n_out]  # [B, n_out, 256]: each crop's class block
    x64 = GA.pt64(x).view(B64, 4096, 256)
    ref = torch.bmm(x64, wq.transpose(1, 2)) + bias.double().view(G, npad)[cls.long(), None, :n_out]
    absref = torch.bmm(x64.abs(), wq.abs().transpose(1, 2)) + bias.double().abs().view(G, npad)[cls.long(), None, :n_out]
    c, i = GA.excess(out[:B64 * 4096, :n_out].reshape(B64, 4096, n_out), ref, absref)
    print(f"grouped fwd planes={planes} n={n_out}: c = {c:.3e}")
    assert c <= GA.BOUNDS[f"fwd{planes}"], (c, i)
    if n_out % 32:
        assert not out[:B64 * 4096, n_out:-(-n_out // 32) * 32].any()  # the rest of the last 32-column chunk is zero-filled


@pytest.mark.parametrize("bplanes", [1, 2])
def test_grouped_dgrad_matches_float64(bplanes):
    from gdr_net_b200 import ops

    G = 16
    gen = torch.Generator(device="cuda").manual_seed(21 + bplanes)
    dlog = GA.grad_like((B64 * 4096, 128), gen, bplanes)
    wd = ops.PT.from_float(GA.row_scaled((G * 256, 128), gen), bplanes)
    cls = _classes64()
    out = ops.gemm_fwd_grouped(dlog, wd, 256, cls, 4096)
    torch.cuda.synchronize()
    w64 = GA.pt64(wd).view(G, 256, 128)[cls.long()]
    d64 = GA.pt64(dlog).view(B64, 4096, 128)
    ref = torch.bmm(d64, w64.transpose(1, 2))
    absref = torch.bmm(d64.abs(), w64.abs().transpose(1, 2))
    u, tiny = GA.out_tolerances(bplanes)
    c, i = GA.excess(GA.pt64(out).view(B64, 4096, 256), ref, absref, u, tiny)
    print(f"grouped dgrad planes={bplanes}: c = {c:.3e}")
    assert c <= GA.BOUNDS[f"fwd{bplanes}"], (c, i)


@pytest.mark.parametrize("layout", ["all13", "rot13"])  # every row per class / mask and region rows shared by all classes
@pytest.mark.parametrize("bplanes", [1, 2])
def test_class_wgrad_reduce_matches_float64_segmented_sum(layout, bplanes):
    from gdr_net_b200 import ops
    from gdr_net_b200.capi import C
    from gdr_net_b200.engine import class_rows

    kw = oracle_kwargs(layout)
    C_ = kw["num_classes"]
    rows, n_rows = class_rows(C_, 1, 64, kw["rot_aware"], kw["mask_aware"], kw["region_aware"])
    n_slots = len(rows[0])
    slot = torch.full((C_, n_rows), -1, dtype=torch.int32)
    for c, r in enumerate(rows):
        slot[c, r] = torch.arange(n_slots, dtype=torch.int32)
    slot = slot.cuda()
    gen = torch.Generator(device="cuda").manual_seed(31 + bplanes)
    dlog = GA.grad_like((B64 * 4096, 128), gen, bplanes, scale=1e-3)
    head = GA.relu_like((B64 * 4096, 256), gen, bplanes)
    cls = ((torch.arange(B64) * 7) % 10).to(torch.int32).cuda()  # classes 10..12 absent
    ws = ops.Workspace("cuda")

    def run():
        buf, ks, kss = ops.gemm_wgrad(dlog, head, ws, ksplit=B64)
        assert ks == B64
        part = torch.empty(B64, 128, device="cuda")
        C.gdrn_crop_colsum(dlog.hi_ptr, dlog.lo_ptr, part.data_ptr(), B64, 4096, 128, ops._stream())
        gw = torch.full((n_rows, 256), math.nan, device="cuda")
        gb = torch.full((n_rows,), math.nan, device="cuda")
        C.gdrn_class_wgrad_reduce(buf.data_ptr(), kss, 256, part.data_ptr(), 128, cls.data_ptr(), B64, slot.data_ptr(), C_, n_rows,
                                  n_slots, 256, gw.data_ptr(), gb.data_ptr(), ops._stream())
        torch.cuda.synchronize()
        return gw, gb

    gw, gb = run()
    gw2, gb2 = run()
    assert torch.equal(gw, gw2) and torch.equal(gb, gb2)  # fixed summation order
    d64, h64 = GA.pt64(dlog).view(B64, 4096, 128), GA.pt64(head).view(B64, 4096, 256)
    P, Pa = torch.bmm(d64.transpose(1, 2), h64), torch.bmm(d64.abs().transpose(1, 2), h64.abs())  # [B, 128, 256] per crop
    Bs, Ba = d64.sum(1), d64.abs().sum(1)
    ref, absref = torch.zeros(n_rows, 256, dtype=torch.float64, device="cuda"), torch.zeros(n_rows, 256, dtype=torch.float64, device="cuda")
    bref, babs = torch.zeros(n_rows, dtype=torch.float64, device="cuda"), torch.zeros(n_rows, dtype=torch.float64, device="cuda")
    for b in range(B64):
        r = torch.tensor(rows[int(cls[b])], device="cuda")
        ref.index_add_(0, r, P[b, :n_slots])
        absref.index_add_(0, r, Pa[b, :n_slots])
        bref.index_add_(0, r, Bs[b, :n_slots])
        babs.index_add_(0, r, Ba[b, :n_slots])
    used = sorted({r for c in cls.tolist() for r in rows[c]})
    absent = sorted(set(range(n_rows)) - set(used))
    assert absent and not gw[absent].any() and not gb[absent].any()  # exactly 0, not merely small
    bound = GA.wgrad_bound(bplanes, 64) + B64 * 2.0 ** -24
    c, i = GA.excess(gw, ref, absref)
    cb, ib = GA.excess(gb, bref, babs)
    print(f"class wgrad {layout} planes={bplanes}: weight c = {c:.3e} (bound {bound:.1e}), bias c = {cb:.3e}")
    assert c <= bound, (c, i)
    assert cb <= (4096 // 32 + 32 + B64) * 2.0 ** -24, (cb, ib)  # fp32 sums: 128 rows per lane, 32 lanes, 64 crops


# ------------------------------------------------------------------------------------------------ exactness
def _model(case, sd=None, precision="mixed", **kw):
    from gdr_net_b200 import GDRN as G

    model, _ = G.build_model_optimizer(case_config(case, device="cuda", **kw), precision=precision)
    if sd is None:
        sd = synth.seeded_state_dict({k: v.cpu() for k, v in model.state_dict().items()}, seed=CASES[case][2])
    model.load_state_dict(sd)
    return model, sd


def test_logits_bit_identical_to_class_agnostic_heads_per_crop():
    from gdr_net_b200 import GDRN as G
    from gdr_net_b200.config import a6_config
    from gdr_net_b200.engine import class_rows

    model, sd = _model("all13", use_pnp_test=True)
    model.eval()
    batch = _cuda(synth.make_batch(B64, seed=7))
    cls = _classes64().long()
    keys = ("mask", "coor_x", "coor_y", "coor_z", "region", "rot", "trans")
    with torch.no_grad():
        out = model(batch["roi_img"], **dict(synth.forward_kwargs(batch, train=False), roi_classes=cls))
    rows, _ = class_rows(13, 1, 64, True, True, True)
    agn, _ = G.build_model_optimizer(a6_config(device="cuda", use_pnp_test=True), precision="mixed")
    agn.eval()
    for c in sorted(set(cls.tolist())):
        r = torch.tensor(rows[c])
        sd_c = dict(sd)
        sd_c["rot_head_net.features.23.weight"] = sd["rot_head_net.features.23.weight"][r].clone()
        sd_c["rot_head_net.features.23.bias"] = sd["rot_head_net.features.23.bias"][r].clone()
        agn.load_state_dict(sd_c)
        with torch.no_grad():
            ref = agn(batch["roi_img"], **synth.forward_kwargs(batch, train=False))
        crops = (cls == c).nonzero().flatten()
        for k in keys:
            assert torch.equal(out[k][crops], ref[k][crops]), (c, k)


# ------------------------------------------------------------------------------------------------ model level
def _train_step(model, batch):
    for p in model.parameters():
        p.grad = None
    _, ld = model(batch["roi_img"], **synth.forward_kwargs(batch, train=True))
    sum(ld.values()).backward()
    torch.cuda.synchronize()
    return {k: float(v.detach()) for k, v in ld.items()}


@pytest.mark.parametrize("case", list(CASES))
def test_b4_matches_golden_and_oracle(case, golden_dir):
    g = golden(golden_dir, case)
    model, sd = _model(case)
    batch_cpu = make_batch(case)
    batch = _cuda(batch_cpu)
    model.train()
    ld = _train_step(model, batch)
    leaf = O.leaf_state_dict(sd)
    o = CA.gdrn_forward(leaf, batch_cpu, train=True, do_loss=True, update_stats=True, **oracle_kwargs(case))
    sum(o["losses"].values()).backward()
    for k, v in ld.items():
        ref = float(g["loss/" + k])
        print(f"[{case}] B=4 {k}: {v:.6f} vs golden {ref:.6f} rel {abs(v - ref) / abs(ref):.2e}")
        assert abs(v - ref) <= 2 * REL * abs(ref), (k, v, ref)
        assert abs(v - float(o["losses"][k])) <= 2 * REL * abs(ref), k
    params = dict(model.named_parameters())
    absent, _ = absent_rows(case)
    for key in g:
        if key.startswith("grad/"):
            name = key[len("grad/"):]
            r_g, r_o = _rel(params[name].grad, g[key]), _rel(params[name].grad, leaf[name].grad)
            print(f"[{case}] grad {name}: rel-L2 vs golden {r_g:.2e}, vs oracle {r_o:.2e}")
            assert r_g < 0.06 and r_o < 0.06, (name, r_g, r_o)  # the bound of tests/test_regions_gpu.py
            if name.startswith("rot_head_net.features.23."):
                assert not params[name].grad[absent].any(), name  # rows of absent classes: exactly 0
    model, _ = _model(case, sd=sd, use_pnp_test=True)
    model.eval()
    with torch.no_grad():
        out = model(batch["roi_img"], **synth.forward_kwargs(batch, train=False))
    head = torch.cat([out["mask"], out["coor_x"], out["coor_y"], out["coor_z"], out["region"]], dim=1)[:, :, ::4, ::4].cpu()
    r, rr, rt = _rel(head, g["eval/head"]), _rel(out["rot"], g["eval/rot"]), _rel(out["trans"], g["eval/trans"])
    print(f"[{case}] eval head rel-L2 vs golden {r:.2e}, rot {rr:.2e}, trans {rt:.2e}")
    assert r < REL and rr < 2e-3 and rt < 2e-3


def test_b64_step_matches_oracle_and_repeats_bit_identically():
    model, sd = _model("all13")
    batch_cpu = synth.make_batch(B64, seed=100)
    batch_cpu["roi_cls"] = _classes64().long().cpu()
    with torch.no_grad():
        o = CA.gdrn_forward(O.leaf_state_dict(sd, requires_grad=False), batch_cpu, train=True, do_loss=True, **oracle_kwargs("all13"))
    model.train()
    batch = _cuda(batch_cpu)
    ld = _train_step(model, batch)
    g1 = {n: p.grad.clone() for n, p in model.named_parameters()}
    for k, v in ld.items():
        ref = float(o["losses"][k])
        print(f"[all13] B=64 {k}: {v:.6f} vs {ref:.6f} rel {abs(v - ref) / abs(ref):.2e}")
        assert abs(v - ref) <= REL * abs(ref), (k, v, ref)
    assert all(torch.isfinite(p.grad).all() for p in model.parameters())
    ld2 = _train_step(model, batch)
    assert ld2 == ld
    p = dict(model.named_parameters())
    for n in DET_GRADS:
        assert torch.equal(p[n].grad, g1[n]), n


# ------------------------------------------------------------------------------------------------ CUDA graphs
def test_graphs_follow_roi_classes_without_recapture():
    batch = _cuda(synth.make_batch(4, seed=61))
    cls_a = torch.tensor([3, 0, 3, 12], device="cuda")
    cls_b = torch.tensor([7, 7, 1, 5], device="cuda")
    # train step: the graphed forward / backward against eager, classes changed between replays
    results = {}
    sd = None
    for graphs in (False, True):
        model, sd = _model("all13", sd=sd)
        model.train()
        model.use_cuda_graphs = graphs
        for cls in (cls_a, cls_b):
            b = dict(batch, roi_cls=cls)
            ld = _train_step(model, b)
            if graphs and cls is cls_a:
                captured = model.engine._graphed
        results[graphs] = (ld, {n: p.grad.clone() for n, p in model.named_parameters()})
        if graphs:
            assert model.engine._graphed is captured  # the second class set replayed the same graphs
    assert results[True][0] == results[False][0]
    for n in DET_GRADS:
        assert torch.equal(results[True][1][n], results[False][1][n]), n
    # folded inference: one cached graph per input signature
    model, _ = _model("all13", sd=sd, use_pnp_test=True)
    model.eval()
    eager = {}
    for cls in (cls_a, cls_b):
        with torch.no_grad():
            eager[int(cls[0])] = model(batch["roi_img"], **dict(synth.forward_kwargs(batch, train=False), roi_classes=cls))
    model.use_cuda_graphs = True
    for cls in (cls_a, cls_b, cls_a):
        with torch.no_grad():
            out = model(batch["roi_img"], **dict(synth.forward_kwargs(batch, train=False), roi_classes=cls))
        for k in ("rot", "trans", "region", "coor_x", "mask"):
            assert torch.equal(out[k], eager[int(cls[0])][k]), (int(cls[0]), k)
    assert len(model.engine._eval_graphs) == 1
    assert np.isfinite(out["rot"].cpu().numpy()).all()
