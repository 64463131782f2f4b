"""GPU: other surface-region counts (ROT_HEAD.NUM_REGIONS) and Patch-PnP without region attention (PNP_NET.REGION_ATTENTION)
through the whole model, the stand-alone Patch-PnP and the device target generator.

  * the five configurations of tests/golden/train_regions_b4.npz (the unmodified reference with only those switches changed) at
    B = 4 against the golden and the oracle (oracle/region_oracle.py), with the bounds of tests/test_mask_heads_gpu.py; the
    TEST.USE_PNP maps carry R + 1 region channels;
  * r8 and r32_noatt at B = 64 in "mixed" within 1e-3 of the oracle;
  * the captured train step equals the eager one bit for bit, and folded eval equals the unfused eval forward;
  * `ConvPnPNet.forward` with nIn 13 (a 64-wide input) and 5 (no region attention) against the oracle;
  * `make_roi_batch` with 8 FPS anchors feeding a NUM_REGIONS = 8 train step."""
import math

import numpy as np
import pytest
import torch

from gdr_net_b200 import synth
from oracle import gdrn_oracle as O
from oracle import region_oracle as RO
from test_regions_cpu import CASES, N_IN, _golden, mask_gt, oracle_kwargs, region_config  # noqa: E402 (tests/ is on sys.path)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

REL = 1e-3


@pytest.fixture(scope="module", autouse=True)
def _gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _model(case, sd=None, precision="mixed", **kw):
    from gdr_net_b200 import GDRN as G

    model, _ = G.build_model_optimizer(region_config(case, device="cuda", **kw), precision=precision)
    if sd is None:
        sd = synth.seeded_state_dict({k: v.cpu() for k, v in model.state_dict().items()}, seed=CASES[case][2])
    model.load_state_dict(sd)
    return model, sd


def _cuda(batch):
    return {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in batch.items()}


def _train_step(model, batch):
    for p in model.parameters():
        p.grad = None
    _, ld = model(batch["roi_img"], **synth.forward_kwargs(batch, train=True))
    sum(ld.values()).backward()
    torch.cuda.synchronize()
    return {k: float(v.detach()) for k, v in ld.items()}


def _batch(case, B=4, seed=None):
    return synth.make_batch(B, seed=CASES[case][3] if seed is None else seed, num_regions=CASES[case][0]["NUM_REGIONS"])


@pytest.mark.parametrize("case", list(CASES))
def test_b4_matches_golden_and_oracle(case, golden_dir):
    g = _golden(golden_dir, case)
    model, sd = _model(case)
    R = CASES[case][0]["NUM_REGIONS"]
    eng = model.engine
    assert (eng.num_regions, eng.pnp_ld) == (R, 64 if N_IN[case] <= 64 else 128)
    batch_cpu = _batch(case)
    batch = _cuda(batch_cpu)
    model.train()
    ld = _train_step(model, batch)
    leaf = O.leaf_state_dict(sd)
    o = RO.gdrn_forward(leaf, batch_cpu, train=True, do_loss=True, update_stats=True, **oracle_kwargs(case))
    sum(o["losses"].values()).backward()
    for k, v in ld.items():
        ref = float(g["loss/" + k])
        print(f"[{case}] B=4 {k}: {v:.6f} vs golden {ref:.6f} rel {abs(v - ref) / abs(ref):.2e}")
        assert abs(v - ref) <= 2 * REL * abs(ref), (k, v, ref)
        assert abs(v - float(o["losses"][k])) <= 2 * REL * abs(ref), k
    params = dict(model.named_parameters())
    for key in g:
        if key.startswith("grad/"):
            name = key[len("grad/"):]
            r_g, r_o = _rel(params[name].grad, g[key]), _rel(params[name].grad, leaf[name].grad)
            print(f"[{case}] grad {name}: rel-L2 vs golden {r_g:.2e}, vs oracle {r_o:.2e}")
            assert r_g < 0.06 and r_o < 0.06, (name, r_g, r_o)  # the bound of tests/test_mask_heads_gpu.py
    # eval mode, TEST.USE_PNP maps: R + 1 region channels; the head against the golden where it has one
    model, _ = _model(case, sd=sd, use_pnp_test=True)
    model.eval()
    with torch.no_grad():
        out = model(batch["roi_img"], **synth.forward_kwargs(batch, train=False))
    assert tuple(out["region"].shape) == (4, R + 1, 64, 64)
    if "eval/head" in g:
        head = torch.cat([out["mask"], out["coor_x"], out["coor_y"], out["coor_z"], out["region"]], dim=1)[:, :, ::4, ::4].cpu()
        r = _rel(head, g["eval/head"])
        rr, rt = _rel(out["rot"], g["eval/rot"]), _rel(out["trans"], g["eval/trans"])
        print(f"[{case}] eval head rel-L2 vs golden {r:.2e}, rot {rr:.2e}, trans {rt:.2e}")
        assert r < REL and rr < 2e-3 and rt < 2e-3


@pytest.mark.parametrize("case", ["r8", "r32_noatt"])
def test_b64_mixed_matches_oracle(case):
    model, sd = _model(case)
    batch_cpu = _batch(case, B=64, seed=100)
    with torch.no_grad():
        o = RO.gdrn_forward(O.leaf_state_dict(sd, requires_grad=False), batch_cpu, train=True, do_loss=True, **oracle_kwargs(case))
    model.train()
    ld = _train_step(model, _cuda(batch_cpu))
    for k, v in ld.items():
        ref = float(o["losses"][k])
        print(f"[{case}] B=64 {k}: {v:.6f} vs {ref:.6f} rel {abs(v - ref) / abs(ref):.2e}")
        assert abs(v - ref) <= REL * abs(ref), (k, v, ref)
    assert all(torch.isfinite(p.grad).all() for p in model.parameters())


@pytest.mark.parametrize("case", ["r8", "r32_noatt", "r60"])
def test_graph_replay_equals_eager(case):
    """Deterministic mode: losses and the gradients named below are bit-identical eager, eager again and graphed (see
    tests/test_mask_heads_gpu.py for why the stem is left out)."""
    batch = _cuda(_batch(case))
    runs = []
    sd = None
    for graphs in (False, False, True):
        model, sd = _model(case, sd=sd)
        model.train()
        model.engine.deterministic = True
        model.use_cuda_graphs = graphs
        for _ in range(2):
            ld = _train_step(model, batch)
        p = dict(model.named_parameters())
        runs.append((ld, {n: p[n].grad.clone() for n in ("rot_head_net.features.23.weight", "rot_head_net.features.20.weight",
                                                        "backbone.layer1.0.conv1.weight", "pnp_net.features.0.weight")}))
    for other in runs[1:]:
        assert other[0] == runs[0][0]
        for n, v in runs[0][1].items():
            assert torch.equal(other[1][n], v), n


@pytest.mark.parametrize("case", ["r8", "r32_noatt", "r60"])
def test_folded_eval_equals_unfused_eval(case):
    model, _ = _model(case, use_pnp_test=True)
    model.eval()
    batch = _cuda(_batch(case))
    outs = []
    for fold in (True, False):
        model.engine.fold_eval = fold
        with torch.no_grad():
            outs.append(model(batch["roi_img"], **synth.forward_kwargs(batch, train=False)))
    R = CASES[case][0]["NUM_REGIONS"]
    assert tuple(outs[0]["region"].shape) == (4, R + 1, 64, 64)
    for k in ("rot", "trans", "coor_x", "region"):
        r = _rel(outs[0][k], outs[1][k])
        print(f"[{case}] folded vs unfused {k}: {r:.2e}")
        assert r < REL, (k, r)


@pytest.mark.parametrize("c_feat,c_reg", [(5, 8), (5, 0), (3, 0)])
def test_standalone_patch_pnp_matches_oracle(c_feat, c_reg):
    from gdr_net_b200.GDRN import ConvPnPNet

    B = 16
    net = ConvPnPNet(nIn=c_feat + c_reg, num_regions=max(c_reg, 2)).cuda()
    sd = synth.seeded_state_dict({"pnp_net." + k: v for k, v in net.state_dict().items()}, seed=12)
    net.load_state_dict({k[len("pnp_net."):]: v for k, v in sd.items()})
    g = synth._gen(7 + c_feat + c_reg, "pnp_maps")
    coor = torch.rand(B, c_feat, 64, 64, generator=g)
    region = torch.softmax(2.0 * torch.randn(B, c_reg, 64, 64, generator=g), dim=1) if c_reg else None
    ext = 0.05 + 0.25 * torch.rand(B, 3, generator=g)
    with torch.no_grad():
        rot_ref, t_ref = O.pnp_forward(coor, region if c_reg else torch.zeros(B, 0, 64, 64), ext, sd)
    for it in range(2):  # the second call replays the CUDA graph
        rot, t = net(coor.cuda(), None if region is None else region.cuda(), ext.cuda())
    torch.cuda.synchronize()
    r1, r2 = _rel(rot, rot_ref), _rel(t, t_ref)
    print(f"Patch-PnP nIn={c_feat + c_reg}: rot {r1:.2e}, t {r2:.2e}")
    assert net._runner.pnp_ld == 64
    assert r1 < REL and r2 < REL, (r1, r2)


def test_roi_targets_with_8_anchors_feed_an_8_region_train_step():
    """The device target generator with 8 farthest-point anchors labels pixels 1..8; a NUM_REGIONS = 8 model trains on them."""
    from gdr_net_b200.roi_targets import make_roi_batch

    B, H, W = 4, 240, 320
    g = torch.Generator().manual_seed(3)
    img = (torch.rand(B, H, W, 3, generator=g) * 255).to(torch.uint8)
    yy, xx = torch.meshgrid(torch.arange(H).float(), torch.arange(W).float(), indexing="ij")
    mask = (((xx - 160) / 70) ** 2 + ((yy - 120) / 50) ** 2 <= 1).float().expand(B, H, W).contiguous()
    ext = 0.1 + 0.1 * torch.rand(B, 3, generator=g)
    xyz = ((torch.rand(B, H, W, 3, generator=g) - 0.5) * ext[:, None, None, :]) * mask[..., None]
    fps = (torch.rand(B, 8, 3, generator=g) - 0.5) * ext[:, None, :]
    centers = torch.tensor([[160.0, 120.0]] * B, dtype=torch.float64)
    scale = torch.full((B,), 180.0, dtype=torch.float64)
    roi = make_roi_batch(img.cuda(), xyz.cuda(), mask.cuda(), mask.cuda(), centers, scale, ext, fps)
    lab = roi["roi_region"]
    assert int(lab.max()) <= 8 and int(lab[roi["roi_mask_obj"] > 0].min()) >= 1
    batch = _cuda(synth.make_batch(B, seed=9, num_regions=8))
    batch.update({k: v for k, v in roi.items() if k != "resize_ratio"})
    model, _ = _model("r8")
    model.train()
    ld = _train_step(model, batch)
    print("chained r8 losses", ld)
    assert all(math.isfinite(v) for v in ld.values())
    assert ld["loss_region"] > 0
    assert all(torch.isfinite(p.grad).all() for p in model.parameters())
    assert np.isfinite(model.rot_head_net.features[23].weight.grad.cpu().numpy()).all()
