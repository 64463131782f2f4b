"""GPU: the PNP_NET pose-loss switches through the whole model (GDRN.forward(do_loss=True) + backward, the captured steps and the
train harness).

  * every case of tests/golden/train_pose_losses_b4.npz (the unmodified reference with only PNP_NET switches changed) at B = 4
    against the golden and the oracle (oracle/pose_loss_oracle.py);
  * the switch-heavy case at B = 64 in "mixed" against the oracle, with the 1e-3 bound of tests/test_parity_b64_gpu.py;
  * GraphedTrainStep and GraphedFwdBwd replay to the eager losses and gradients with a non-default loss count;
  * train_harness.TrainStep runs two steps and losses_async returns the new keys."""
import os

import numpy as np
import pytest
import torch

from gdr_net_b200 import synth
from oracle import gdrn_oracle as O
from oracle import pose_loss_oracle as P
from test_pose_losses_cpu import CASES  # noqa: E402 (tests/ is on sys.path)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

REL = 1e-3
GRAD_NAMES = ("rot_head_net.features.23.weight", "rot_head_net.features.20.weight", "pnp_net.fc_r.weight", "pnp_net.fc_t.weight",
              "pnp_net.features.0.weight")


@pytest.fixture(scope="module", autouse=True)
def _gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _cfg(case, device="cuda"):
    from gdr_net_b200.config import a6_config

    cfg = a6_config(device=device)
    for k, v in CASES[case][0].items():
        setattr(cfg.MODEL.CDPN.PNP_NET, k, v)
    return cfg


def _model(case, sd=None, precision="mixed"):
    from gdr_net_b200 import GDRN as G

    model, opt = G.build_model_optimizer(_cfg(case), precision=precision)
    if sd is None:
        sd = synth.seeded_state_dict({k: v.cpu() for k, v in model.state_dict().items()}, seed=CASES[case][1])
    model.load_state_dict(sd)
    return model, sd, opt


def _cuda(batch):
    return {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in batch.items()}


def _train_step(model, batch):
    for p in model.parameters():
        p.grad = None
    _, ld = model(batch["roi_img"], **synth.forward_kwargs(batch, train=True))
    sum(ld.values()).backward()
    torch.cuda.synchronize()
    return {k: float(v.detach()) for k, v in ld.items()}


def _sym(case):
    return bool(CASES[case][0].get("PM_LOSS_SYM"))


@pytest.mark.parametrize("case", sorted(CASES))
def test_b4_matches_golden_and_oracle(case, golden_dir):
    g = np.load(os.path.join(golden_dir, "train_pose_losses_b4.npz"))
    model, sd, _ = _model(case)
    batch_cpu = synth.make_batch(4, seed=CASES[case][2], with_sym=CASES[case][3])
    model.train()
    ld = _train_step(model, _cuda(batch_cpu))
    assert list(ld) == list(g[f"{case}/names"])
    assert model.engine.loss_names == list(g[f"{case}/names"])
    leaf = O.leaf_state_dict(sd)
    o = P.gdrn_forward(leaf, batch_cpu, _cfg(case, "cpu").MODEL.CDPN.PNP_NET, pm_sym=_sym(case), update_stats=True)
    sum(o["losses"].values()).backward()
    # seeded (not calibrated) weights: the bound of tests/test_mask_heads_gpu.py (2e-3 of each loss)
    for k, v in ld.items():
        ref = float(g[f"{case}/loss/{k}"])
        print(f"[{case}] B=4 {k}: {v:.6f} vs golden {ref:.6f} rel {abs(v - ref) / abs(ref):.2e}")
        assert abs(v - ref) <= 2 * REL * abs(ref), (k, v, ref)
        assert abs(v - float(o["losses"][k])) <= 2 * REL * abs(ref), k
    params = dict(model.named_parameters())
    prefix = f"{case}/grad/"
    for key in g.files:
        if key.startswith(prefix):
            name = key[len(prefix):]
            r_g, r_o = _rel(params[name].grad, g[key]), _rel(params[name].grad, leaf[name].grad)
            print(f"[{case}] grad {name}: rel-L2 vs golden {r_g:.2e}, vs oracle {r_o:.2e}")
            assert r_g < 0.06 and r_o < 0.06, (name, r_g, r_o)  # the bound of test_parity_b64_gpu.py's gradient checks


def test_b64_mixed_switch_heavy_matches_oracle():
    """The benchmark's batch (B = 64, seed 100) in "mixed" with the rt_sl1 switches: every loss within 1e-3 of the oracle."""
    case = "rt_sl1"
    model, sd, _ = _model(case)
    batch_cpu = synth.make_batch(64, seed=100)
    with torch.no_grad():
        o = P.gdrn_forward(O.leaf_state_dict(sd, requires_grad=False), batch_cpu, _cfg(case, "cpu").MODEL.CDPN.PNP_NET)
    model.train()
    ld = _train_step(model, _cuda(batch_cpu))
    assert list(ld) == list(o["losses"])
    for k, ref in o["losses"].items():
        ref = float(ref)
        print(f"[{case}] B=64 {k}: {ld[k]:.6f} vs {ref:.6f} rel {abs(ld[k] - ref) / abs(ref):.2e}")
        assert abs(ld[k] - ref) <= REL * abs(ref), (k, ld[k], ref)
    assert all(torch.isfinite(p.grad).all() for p in model.parameters())


@pytest.mark.parametrize("case", ["rt_sl1", "pm_off"])
def test_graph_replay_equals_eager(case):
    """Deterministic mode: eager, GraphedFwdBwd (model.use_cuda_graphs) and GraphedTrainStep give bit-identical losses and
    gradients with a loss count other than 8."""
    from gdr_net_b200.engine import GraphedTrainStep

    batch = _cuda(synth.make_batch(4, seed=CASES[case][2]))
    runs, sd = [], None
    for graphs in (False, True):
        model, sd, _ = _model(case, sd=sd)
        model.train()
        model.engine.deterministic = True
        model.use_cuda_graphs = graphs
        for _ in range(2):  # the second step replays when graphs are on
            ld = _train_step(model, batch)
        assert len(model.engine.loss_names) != 8
        p = dict(model.named_parameters())
        runs.append((ld, {n: p[n].grad.clone() for n in GRAD_NAMES}))
    assert runs[1][0] == runs[0][0]
    for n, v in runs[0][1].items():
        assert torch.equal(runs[1][1][n], v), n
    # GraphedTrainStep: one graph for forward + backward, its gradient vector sized from the loss list
    model, _, _ = _model(case, sd=sd)
    model.train()
    eng = model.engine
    eng.deterministic = True
    kw = synth.forward_kwargs(batch, train=True)
    names = ["roi_coord_2d", "roi_cams", "roi_centers", "roi_whs", "roi_extents", "resize_ratios", "gt_xyz", "gt_mask_trunc",
             "gt_mask_visib", "gt_region", "gt_ego_rot", "gt_points", "gt_trans", "gt_trans_ratio"]
    aux = {k: (kw[k].float().contiguous() if kw[k].dtype != torch.long else kw[k]) for k in names}
    aux["sym_infos"] = None
    x = batch["roi_img"].float().contiguous()
    step = GraphedTrainStep(eng, x, aux, train_bn=True)
    assert step.gw.numel() == len(eng.loss_names)
    gl = torch.linspace(0.5, 1.5, len(eng.loss_names), device="cuda")
    losses = step(grad_losses=gl).clone()
    g_graph = {n: eng.grads[n].clone() for n in GRAD_NAMES}  # not atomically summed: bit-reproducible
    res = eng.forward(x, aux, train_bn=True, do_loss=True)
    eng.backward(gl)
    torch.cuda.synchronize()
    assert torch.equal(res["losses"], losses)
    for n, v in g_graph.items():
        assert torch.equal(eng.grads[n], v), n


def test_train_harness_reports_the_new_losses():
    from gdr_net_b200.train_harness import TrainStep

    case = "disz_l2"
    model, _, opt = _model(case)
    model.train()
    step = TrainStep(model, opt, use_cuda_graphs=True)
    batch = _cuda(synth.make_batch(4, seed=CASES[case][2]))
    batch = dict(batch, roi_cls=torch.zeros(4, dtype=torch.long, device="cuda"), roi_cam=batch["roi_cam"])
    for _ in range(2):
        step(batch)
    d = step.losses_async(wait_current=True)
    assert set(d) == set(model.engine.loss_names) | {"total_loss"}
    assert {"loss_PM_xy", "loss_PM_z", "loss_rot", "loss_trans_LPnP"} <= set(d)
    assert all(np.isfinite(v) for v in d.values())
