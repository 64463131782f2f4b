"""GPU parity of the full hot path (through the reference-compatible GDRN module -> C ABI) against
  (a) the committed golden outputs of the unmodified reference (tests/golden/*.npz), and
  (b) the CPU oracle (oracle/gdrn_oracle.py) on the same seeded inputs.

Tolerances (BASELINE.json north_star): outputs within 1e-3 relative fp32, region argmax bit-exact -- asserted in
the fp32-faithful "fp32x3" mode (three wgmma passes over hi/lo fp16 planes = 22-bit operands).  The single-pass
"half" mode (fp16 operands: 11-bit mantissa, the same as the TF32 convolutions cuDNN runs for the reference) is the
throughput mode; its deviation is bounded by operand rounding (2^-12 per tensor per layer, accumulating over ~130
roundings) and is asserted at the looser, documented bound below.
"""
import os

import numpy as np
import pytest
import torch

from gdr_net_b200 import synth
from gdr_net_b200.config import a6_config

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

REL_FP32 = 1e-3          # north-star tolerance (dense maps, losses), fp32x3 mode
REL_POSE = 1e-3          # rot / trans / ADD in fp32x3 mode (measured 1e-4 .. 2.5e-4)
REL_HALF = 0.15          # sanity bound for the single-pass fp16 mode on this RANDOM-weight 50-layer net: 2^-12 operand
                         # rounding accumulates ~linearly (measured 0.02 relative at layer4, 0.056 at the logits, 0.08 on the
                         # pose); a bf16 build (GDRN_STORE_F16=0) measures 0.13 / 0.34 here


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _relmax(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


@pytest.fixture(scope="module")
def sd():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from oracle import fixtures

    return fixtures.calibrated_state_dict(0)


def _model(sd, precision, sym=False):
    from gdr_net_b200 import GDRN as G

    cfg = a6_config(device="cuda", pm_loss_sym=sym, use_pnp_test=True)
    model, opt = G.build_model_optimizer(cfg, precision=precision)
    model.load_state_dict(sd)
    return model, opt


def _cuda_batch(batch):
    return {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in batch.items()}


@pytest.mark.parametrize("precision,tol", [("fp32x3", REL_FP32), ("half", REL_HALF)])
def test_eval_forward_b2_vs_golden(sd, golden_dir, precision, tol):
    g = np.load(os.path.join(golden_dir, "eval_b2.npz"))
    model, _ = _model(sd, precision)
    model.eval()
    batch = _cuda_batch(synth.make_batch(2, seed=0))
    with torch.no_grad():
        out = model(batch["roi_img"], **synth.forward_kwargs(batch, train=False))
    torch.cuda.synchronize()
    head = torch.cat([out["mask"], out["coor_x"], out["coor_y"], out["coor_z"], out["region"]], dim=1).cpu()
    ref = torch.from_numpy(g["head"])
    assert head.shape == ref.shape
    print(f"[{precision}] eval b2: head rel-L2 {_rel(head, ref):.2e} rel-max {_relmax(head, ref):.2e} rot {_rel(out['rot'], g['rot']):.2e} "
          f"trans {_rel(out['trans'], g['trans']):.2e}")
    assert _rel(head, ref) < tol, _rel(head, ref)
    assert _relmax(head, ref) < 2 * tol, _relmax(head, ref)
    ptol = REL_POSE if precision == "fp32x3" else 0.5
    assert _rel(out["rot"], g["rot"]) < ptol and _rel(out["trans"], g["trans"]) < ptol
    agree = (head[:, 4:].argmax(1).numpy().astype(np.uint8) == g["region_argmax"]).mean()
    if precision == "fp32x3":
        # bit-exact region argmax, except pixels whose top-2 logits are closer than the fp32 parity tolerance itself
        top2 = ref[:, 4:].topk(2, dim=1).values
        margin_ok = ((top2[:, 0] - top2[:, 1]) > 2 * REL_FP32 * ref.abs().max()).numpy()
        mism = head[:, 4:].argmax(1).numpy().astype(np.uint8) != g["region_argmax"]
        assert not (mism & margin_ok).any()
        assert agree > 0.995  # random-weight logits have many near-ties; every mismatch is inside the tie margin (above)
    else:
        print(f"[half] region argmax agreement {agree:.4f}")
        assert agree > 0.85


# Gradient tolerance: the network is non-smooth (ReLU, L1 losses, max-pool), so gradients are discontinuous in the
# forward values.  The reference's OWN fp32 gradients differ from its fp64 evaluation by 1.5e-2 relative L2 at the
# stem (tools/noise_floor.py; forward difference only 4e-5).  We require <= 0.06 per tensor and cosine > 0.995 overall
# in fp32x3 mode; per-op backward kernels are tested to ~1e-4 in tests/test_ops_gpu.py.
@pytest.mark.parametrize("precision,tol,gtol", [("fp32x3", REL_FP32, 0.06), ("mixed", REL_FP32, 0.06), ("half", REL_HALF, 1.0)])
@pytest.mark.parametrize("case,seed,sym", [("train_b4", 1, False), ("train_sym_b4", 2, True)])
def test_train_fwd_bwd_b4(sd, golden_dir, precision, tol, gtol, case, seed, sym):
    from oracle import gdrn_oracle as O

    g = np.load(os.path.join(golden_dir, case + ".npz"))
    model, _ = _model(sd, precision, sym=sym)
    model.train()
    batch_cpu = synth.make_batch(4, seed=seed, with_sym=sym)
    batch = _cuda_batch(batch_cpu)
    out_dict, loss_dict = model(batch["roi_img"], **synth.forward_kwargs(batch, train=True))
    assert out_dict == {}
    assert sorted(loss_dict) == sorted(["loss_coor_x", "loss_coor_y", "loss_coor_z", "loss_mask", "loss_region", "loss_PM_R",
                                        "loss_centroid", "loss_z"])
    total = sum(loss_dict.values())
    total.backward()
    torch.cuda.synchronize()
    for k, v in loss_dict.items():
        ref = float(g["loss/" + k])
        assert abs(float(v) - ref) <= tol * abs(ref), (k, float(v), ref)
    # logging side effect values (vis/*) against the reference's EventStorage scalars
    if "vis/error_R" in g.files:
        assert abs(model.last_vis_dict["vis/error_R"] - float(g["vis/error_R"])) < (0.05 if precision != "half" else 30.0)
        assert abs(model.last_vis_dict["vis/tz_gt"] - float(g["vis/tz_gt"])) < 1e-6
    # gradients: against the oracle's autograd (full tensors) and the reference's stored norms
    leaf = O.leaf_state_dict(sd)
    o = O.gdrn_forward(leaf, batch_cpu, train=True, do_loss=True, pm_sym=sym, update_stats=True)
    sum(o["losses"].values()).backward()
    worst = ("", 0.0)
    dot = na = nb = 0.0
    for name, p in model.named_parameters():
        assert p.grad is not None, name
        a_, b_ = p.grad.double().cpu().flatten(), leaf[name].grad.double().flatten()
        dot += float(a_ @ b_)
        na += float(a_ @ a_)
        nb += float(b_ @ b_)
        r = _rel(p.grad, leaf[name].grad)
        if r > worst[1]:
            worst = (name, r)
        assert abs(float(p.grad.double().norm()) - float(g["gnorm/" + name])) <= 2 * gtol * float(g["gnorm/" + name]) + 1e-12, name
    cos = dot / (na * nb) ** 0.5
    tail = {n: _rel(dict(model.named_parameters())[n].grad, leaf[n].grad) for n in ("pnp_net.fc_t.weight", "pnp_net.fc2.weight")}
    print(f"[{precision}] {case}: worst grad rel-L2 {worst}, cosine {cos:.6f}, tail {tail}")
    assert worst[1] < gtol, worst
    if precision in ("fp32x3", "mixed"):  # mixed = the fp32x3 forward + a single-pass backward: same bounds (measured 0.9996 / 0.9997)
        assert cos > 0.999, cos
        assert tail["pnp_net.fc_t.weight"] < 5e-3 and tail["pnp_net.fc2.weight"] < 5e-2, tail
    else:  # half: the 5e-2 forward deviation flips ReLU / L1 decisions; measured global cosine 0.82 (ADVICE r1: bound it)
        assert cos > 0.7, cos
    # BatchNorm running statistics were updated like nn.BatchNorm2d(momentum=0.1)
    msd = model.state_dict()
    for k in ("backbone.bn1.running_mean", "backbone.layer4.2.bn2.running_var", "rot_head_net.features.21.running_mean"):
        assert _relmax(msd[k], leaf[k]) < (2e-3 if precision != "half" else 0.2), k
    assert int(msd["backbone.bn1.num_batches_tracked"]) == 1


def test_add_metric_parity(sd):
    """ADD(-S) of the predicted poses (lib/pysixd/pose_error.py:297-337) within 1e-3 of the oracle's (fp32x3)."""
    from oracle import gdrn_oracle as O

    model, _ = _model(sd, "fp32x3")
    model.eval()
    batch_cpu = synth.make_batch(4, seed=7)
    batch = _cuda_batch(batch_cpu)
    with torch.no_grad():
        out = model(batch["roi_img"], **synth.forward_kwargs(batch, train=False))
        o = O.gdrn_forward(O.leaf_state_dict(sd, requires_grad=False), batch_cpu, train=False, do_loss=False)
    for i in range(4):
        pts = batch_cpu["roi_points"][i].numpy()
        args = (batch_cpu["ego_rot"][i].numpy(), batch_cpu["trans"][i].numpy(), pts)
        a = O.add_metric(out["rot"][i].cpu().numpy(), out["trans"][i].cpu().numpy(), *args)
        b = O.add_metric(o["rot"][i].numpy(), o["trans"][i].numpy(), *args)
        print(f"ADD {a:.6f} vs {b:.6f} rel {abs(a - b) / b:.2e}")
        assert abs(a - b) <= 1e-3 * max(b, 1e-6)  # north star: ADD(-S) parity within 1e-3
        a = O.adi_metric(out["rot"][i].cpu().numpy(), out["trans"][i].cpu().numpy(), *args)
        b = O.adi_metric(o["rot"][i].numpy(), o["trans"][i].numpy(), *args)
        assert abs(a - b) <= REL_POSE * max(b, 1e-6)


def test_optimizer_step_runs(sd):
    model, opt = _model(sd, "half")
    model.train()
    batch = _cuda_batch(synth.make_batch(4, seed=3))
    before = model.pnp_net.fc_r.weight.detach().clone()
    for _ in range(2):
        opt.zero_grad(set_to_none=True)
        _, loss_dict = model(batch["roi_img"], **synth.forward_kwargs(batch, train=True))
        losses = sum(loss_dict.values())
        assert torch.isfinite(losses).all()
        losses.backward()
        opt.step()
    assert not torch.equal(before, model.pnp_net.fc_r.weight)


@pytest.mark.parametrize("B", [1, 3])
def test_ragged_batch_sizes(sd, B):
    """Inference batches are 'detections per image' (any size, reference gdrn_evaluator.py:561-578); train batches may be odd."""
    from oracle import gdrn_oracle as O

    model, _ = _model(sd, "fp32x3")
    batch_cpu = synth.make_batch(B, seed=11 + B)
    batch = _cuda_batch(batch_cpu)
    model.eval()
    with torch.no_grad():
        out = model(batch["roi_img"], **synth.forward_kwargs(batch, train=False))
        o = O.gdrn_forward(O.leaf_state_dict(sd, requires_grad=False), batch_cpu, train=False, do_loss=False)
    head = torch.cat([out["mask"], out["coor_x"], out["coor_y"], out["coor_z"], out["region"]], dim=1)
    assert _rel(head, o["head"]) < REL_FP32 and _rel(out["rot"], o["rot"]) < 2e-3 and _rel(out["trans"], o["trans"]) < 2e-3
    model.train()
    _, loss_dict = model(batch["roi_img"], **synth.forward_kwargs(batch, train=True))
    sum(loss_dict.values()).backward()
    o = O.gdrn_forward(O.leaf_state_dict(sd, requires_grad=False), batch_cpu, train=True, do_loss=True)
    for k, v in loss_dict.items():
        assert abs(float(v) - float(o["losses"][k])) <= 2e-3 * abs(float(o["losses"][k])), (B, k, float(v), float(o["losses"][k]))
    assert all(torch.isfinite(p.grad).all() for p in model.parameters())


def test_module_api_cuda_graphs_match_eager(sd):
    """`model.use_cuda_graphs = True` (forward/backward replayed as CUDA graphs) gives the eager path's losses and gradients."""
    batch = _cuda_batch(synth.make_batch(4, seed=21))
    res = []
    for graphs in (False, True):
        model, _ = _model(sd, "fp32x3")  # the 3-MMA mode: run-to-run noise (BN-stat atomics order) stays ~1e-5, so a real replay bug shows
        model.train()
        model.use_cuda_graphs = graphs
        for it in range(2):  # second iteration replays
            for p in model.parameters():
                p.grad = None
            _, loss_dict = model(batch["roi_img"], **synth.forward_kwargs(batch, train=True))
            sum(loss_dict.values()).backward()
        torch.cuda.synchronize()
        res.append(({k: float(v) for k, v in loss_dict.items()}, {n: p.grad.clone() for n, p in model.named_parameters()}))
    for k in res[0][0]:
        assert abs(res[0][0][k] - res[1][0][k]) <= 2e-3 * abs(res[0][0][k]), k
    # run-to-run noise of this non-smooth net reaches ~2e-2 at the stem; a replay bug (stale buffer, missing kernel) is O(1)
    for n in ("pnp_net.fc_t.weight", "rot_head_net.features.23.weight", "backbone.conv1.weight"):
        assert _rel(res[1][1][n], res[0][1][n]) < (0.15 if n.startswith("backbone") else 5e-2), n


def test_module_api_grad_accumulation_and_aliasing(sd):
    """p.grad may alias Engine.flat_grad after a step (autograd adopts the fresh views without a copy); a second backward
    without zero_grad must still ACCUMULATE (g1 + g2), and zero_grad(set_to_none) + backward must give the plain gradient."""
    model, _ = _model(sd, "fp32x3")
    model.train()
    b1, b2 = _cuda_batch(synth.make_batch(2, seed=31)), _cuda_batch(synth.make_batch(2, seed=32))
    names = ("pnp_net.fc_t.weight", "rot_head_net.features.23.weight", "backbone.conv1.weight", "backbone.layer3.1.bn2.weight")
    params = dict(model.named_parameters())

    def run(batch):
        _, loss_dict = model(batch["roi_img"], **synth.forward_kwargs(batch, train=True))
        sum(loss_dict.values()).backward()

    single = []
    for b in (b1, b2):
        for p in model.parameters():
            p.grad = None
        run(b)
        torch.cuda.synchronize()
        single.append({n: params[n].grad.clone() for n in names})
    for p in model.parameters():
        p.grad = None
    run(b1)
    run(b2)  # no zero_grad in between
    torch.cuda.synchronize()
    for n in names:
        want = single[0][n] + single[1][n]
        # run-to-run noise (atomics order -> ReLU / max-pool flips) reaches 4e-3 (head) .. 2e-2 (stem) on this non-smooth net (DESIGN 3.3);
        # a lost or doubled gradient would be an error of 0.5-1.0
        assert _rel(params[n].grad, want) < (0.25 if n.startswith("backbone") else 5e-2), n


def test_train_harness_steps_and_async_losses(sd):
    """f-1: batch_data + TrainStep (graphs + fused Ranger, no per-iteration .item()): losses of a step match a plain eager step on
    the same batch, parameters move, and the asynchronous loss read-back returns the previous step's values."""
    from gdr_net_b200.train_harness import TrainStep, batch_data

    b = synth.make_batch(4, seed=71)
    data = [dict(roi_img=b["roi_img"][i], roi_cls=0, roi_coord_2d=b["roi_coord_2d"][i], cam=b["roi_cam"][i], bbox_center=b["roi_center"][i],
                 roi_wh=b["roi_wh"][i], resize_ratio=float(b["resize_ratio"][i]), roi_extent=b["roi_extent"][i],
                 trans_ratio=b["roi_trans_ratio"][i], roi_xyz=b["roi_xyz"][i], roi_mask_trunc=b["roi_mask_trunc"][i],
                 roi_mask_visib=b["roi_mask_visib"][i], roi_mask_obj=b["roi_mask_obj"][i], roi_region=b["roi_region"][i].int(),
                 ego_rot=b["ego_rot"][i], trans=b["trans"][i], roi_points=b["roi_points"][i]) for i in range(4)]
    batch = batch_data(None, data, device="cuda")
    model, opt = _model(sd, "mixed")
    model.train()
    ref_model, _ = _model(sd, "mixed")
    ref_model.train()
    _, ref_ld = ref_model(batch["roi_img"], **synth.forward_kwargs(_cuda_batch(b), train=True))
    step = TrainStep(model, opt, use_cuda_graphs=True)
    before = model.rot_head_net.features[23].weight.detach().clone()
    ld0 = step(batch)
    assert step.losses_async() is None
    for k, v in ld0.items():
        assert abs(float(v) - float(ref_ld[k])) <= 1e-4 * abs(float(ref_ld[k])) + 1e-7, k
    step(batch)
    prev = step.losses_async()
    assert abs(prev["total_loss"] - float(sum(ld0.values()))) <= 1e-5 * abs(prev["total_loss"])
    cur = step.losses_async(wait_current=True)
    assert cur["total_loss"] == cur["total_loss"] and cur["total_loss"] != prev["total_loss"]  # the weights moved
    assert not torch.equal(before, model.rot_head_net.features[23].weight)
