"""GPU: DropBlock on the Patch-PnP input (PNP_NET.PNP_HEAD_CFG.drop_prob / dropblock_size) through the whole model, the
device sampler and the stand-alone Patch-PnP.

  * each golden case of tests/golden/train_dropblock_b4.npz at B = 4, with the engine's counter set to the case's step: the
    engine's keep mask is the max-pool formula of its own seed mask, its scale is numel / sum, and the losses and gradients
    match the oracle fed those seeds within the bounds of tests/test_regions_gpu.py; the same at B = 64 in "mixed";
  * the seed counts stay within 5 sigma of Binomial(B 4096, float32 gamma); masks differ between steps, crops and seeds, and
    the same seed repeats the sequence;
  * the first train forward equals the drop_prob = 0 model, eval forwards advance the counter, and p stays fixed after 5000;
  * the captured train step replays the eager sequence of masks, losses and gradients bit for bit;
  * DropBlock still applies with PNP_NET.FREEZE; the stand-alone ConvPnPNet.forward matches the oracle in train mode;
  * with drop_prob = 0 a train step launches nothing new."""
import math

import numpy as np
import pytest
import torch

from gdr_net_b200 import synth
from oracle import dropblock_oracle as DB
from oracle import gdrn_oracle as O
from test_dropblock_cpu import CASES, db_config, golden, oracle_kwargs  # noqa: E402 (tests/ is on sys.path)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

REL = 1e-3
GRAD_KEYS = ("pnp_net.features.0.weight", "pnp_net.fc_r.weight", "rot_head_net.features.23.weight", "backbone.layer1.0.conv1.weight")


@pytest.fixture(scope="module", autouse=True)
def _gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _model(case, sd=None, precision="mixed", drop_prob=None, freeze_pnp=False):
    from gdr_net_b200 import GDRN as G

    cfg = db_config(case, device="cuda", drop_prob=drop_prob)
    cfg.MODEL.CDPN.PNP_NET.FREEZE = freeze_pnp
    model, _ = G.build_model_optimizer(cfg, precision=precision)
    if sd is None:
        sd = synth.seeded_state_dict({k: v.cpu() for k, v in model.state_dict().items()}, seed=CASES[case][5])
    model.load_state_dict(sd)
    model.pnp_net.dropblock_seed = 1234
    return model, sd


def _cuda(batch):
    return {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in batch.items()}


def _batch(case, B=4, seed=None):
    return synth.make_batch(B, seed=CASES[case][6] if seed is None else seed, num_regions=CASES[case][0]["NUM_REGIONS"])


def _train_step(model, batch):
    for p in model.parameters():
        p.grad = None
    _, ld = model(batch["roi_img"], **synth.forward_kwargs(batch, train=True))
    sum(ld.values()).backward()
    torch.cuda.synchronize()
    return {k: float(v.detach()) for k, v in ld.items()}


def _check_mask(model, case):
    """The engine's keep mask against the max-pool formula of its own seeds; the scale against numel / sum."""
    pn = model.pnp_net
    seeds, keep, scale = pn.dropblock_seeds.cpu(), pn.dropblock_keep.cpu(), float(pn.dropblock_scale.cpu())
    bm = DB.block_mask(seeds, CASES[case][3])
    assert torch.equal(keep.float(), bm)
    assert scale == float(np.float32(bm.numel()) / np.float32(bm.sum())), (scale, bm.numel(), float(bm.sum()))
    return seeds


def _against_oracle(case, model, sd, batch_cpu, ld, seeds, grads=True, bound=2 * REL):
    leaf = O.leaf_state_dict(sd, requires_grad=grads)
    with torch.set_grad_enabled(grads):
        o = DB.gdrn_forward(leaf, batch_cpu, train=True, do_loss=True, seeds=seeds, update_stats=grads, **oracle_kwargs(case))
        if grads:
            sum(o["losses"].values()).backward()
    for k, v in ld.items():
        ref = float(o["losses"][k])
        print(f"[{case}] {k}: {v:.6f} vs oracle {ref:.6f} rel {abs(v - ref) / abs(ref):.2e}")
        assert abs(v - ref) <= bound * abs(ref), (k, v, ref)
    if grads:
        params = dict(model.named_parameters())
        for name in GRAD_KEYS:
            if params[name].grad is None:
                continue
            r = _rel(params[name].grad, leaf[name].grad)
            print(f"[{case}] grad {name}: rel-L2 vs oracle {r:.2e}")
            assert r < 0.06, (name, r)  # the bound of tests/test_mask_heads_gpu.py
    return o


@pytest.mark.parametrize("case", list(CASES))
def test_b4_matches_oracle_with_the_engine_seeds(case, golden_dir):
    g = golden(golden_dir, case)
    model, sd = _model(case)
    model.train()
    model.pnp_net.dropblock_step = int(g["step"])
    batch_cpu = _batch(case)
    ld = _train_step(model, _cuda(batch_cpu))
    assert model.pnp_net.dropblock_step == int(g["step"]) + 1
    seeds = _check_mask(model, case)
    assert 0 < int(seeds.sum()) < seeds.numel()
    _against_oracle(case, model, sd, batch_cpu, ld, seeds)
    assert list(ld) == [k[len("loss/"):] for k in g if k.startswith("loss/")]  # the reference's loss_dict order


@pytest.mark.parametrize("case", ["ship_b5", "r8_b3"])
def test_b64_mixed_matches_oracle(case):
    model, sd = _model(case)
    model.train()
    model.pnp_net.dropblock_step = 4999
    batch_cpu = _batch(case, B=64, seed=100)
    ld = _train_step(model, _cuda(batch_cpu))
    seeds = _check_mask(model, case)
    _against_oracle(case, model, sd, batch_cpu, ld, seeds, grads=False, bound=REL)
    assert all(torch.isfinite(p.grad).all() for p in model.parameters())


def _sampler(B, seed, p=0.25, k=5):
    from gdr_net_b200.capi import C

    step = torch.zeros(1, dtype=torch.int64, device="cuda")
    keep = torch.empty(B, 64, 64, dtype=torch.uint8, device="cuda")
    seeds = torch.empty_like(keep)
    counts = torch.empty(B, dtype=torch.int32, device="cuda")
    scale = torch.empty(1, device="cuda")

    def run(at=None):
        if at is not None:
            step.fill_(at)
        C.gdrn_dropblock_step(step.data_ptr(), seed, 0, p, k, 1, keep.data_ptr(), seeds.data_ptr(), counts.data_ptr(),
                              scale.data_ptr(), B, 64, 64, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        return seeds.clone(), keep.clone(), counts.clone(), scale.clone()

    return run, step


def test_seed_statistics_and_streams():
    B, n = 64, 64 * 4096
    run, step = _sampler(B, seed=7)
    draws = [run(4999 if i == 0 else None) for i in range(40)]
    assert int(step.item()) == 4999 + 40
    for s, kp, cnt, sc in draws:
        for p_, k_ in ((0.25, 5),):
            gamma = float(np.float32(p_ / k_**2))
            mean, sd = n * gamma, math.sqrt(n * gamma * (1 - gamma))
            assert abs(int(s.sum()) - mean) <= 5 * sd, (int(s.sum()), mean, sd)
        assert torch.equal(cnt.cpu(), kp.view(B, -1).sum(1, dtype=torch.int32).cpu())
        assert torch.equal(kp.float().cpu(), DB.block_mask(s.cpu(), 5))
    # masks differ between steps and between crops
    assert not torch.equal(draws[0][0], draws[1][0])
    assert all(not torch.equal(draws[0][0][0], draws[0][0][b]) for b in range(1, B))
    # the same seed repeats the sequence, another seed does not
    again, _ = _sampler(B, seed=7)
    assert torch.equal(again(4999)[0], draws[0][0]) and torch.equal(again()[0], draws[1][0])
    other, _ = _sampler(B, seed=8)
    assert not torch.equal(other(4999)[0], draws[0][0])
    # step 0 draws nothing (p = 0) and keeps everything with scale 1; mid-schedule gamma follows linspace
    s0, k0, _, sc0 = run(0)
    assert int(s0.sum()) == 0 and bool(k0.all()) and float(sc0) == 1.0
    mid = [run(2500 if i == 0 else None)[0] for i in range(10)]
    gamma = float(np.float32(DB.prob_at(0.25, 2500) / 25))
    tot = sum(int(s.sum()) for s in mid)
    assert abs(tot - 10 * n * gamma) <= 5 * math.sqrt(10 * n * gamma), (tot, 10 * n * gamma)


def test_schedule_first_step_eval_and_plateau():
    case = "ship_b5"
    batch = _cuda(_batch(case))
    m0, sd = _model(case, drop_prob=0.0)
    m1, _ = _model(case, sd=sd)
    for m in (m0, m1):
        m.train()
        m.engine.deterministic = True
    ld0, ld1 = _train_step(m0, batch), _train_step(m1, batch)
    assert ld0 == ld1  # forward 0 has probability 0: the Patch-PnP input is untouched
    assert m1.pnp_net.dropblock_step == 1 and int(m1.pnp_net.dropblock_seeds.sum()) == 0
    p0, p1 = dict(m0.named_parameters()), dict(m1.named_parameters())
    for name in GRAD_KEYS:
        assert _rel(p1[name].grad, p0[name].grad) < 1e-5, name
    # eval forwards (folded inference, and its captured graph) advance the counter as well
    m1.eval()
    with torch.no_grad():
        m1(batch["roi_img"], **synth.forward_kwargs(batch, train=False))
        m1.use_cuda_graphs = True
        for _ in range(3):
            m1(batch["roi_img"], **synth.forward_kwargs(batch, train=False))
    m1.use_cuda_graphs = False
    assert m1.pnp_net.dropblock_step == 5
    # past 5000 forwards p stays at drop_prob: the seed rate at step 20000 is that of p = 0.25
    m1.train()
    B = 64
    big = _cuda(synth.make_batch(B, seed=9))
    tot = 0
    for i in range(4):
        if i == 0:
            m1.pnp_net.dropblock_step = 20000
        with torch.no_grad():
            m1(big["roi_img"], **synth.forward_kwargs(big, train=False))
        tot += int(m1.pnp_net.dropblock_seeds.sum())
    gamma = float(np.float32(0.25 / 25))
    n = 4 * B * 4096
    assert abs(tot - n * gamma) <= 5 * math.sqrt(n * gamma), (tot, n * gamma)
    assert m1.pnp_net.dropblock_step == 20004


def test_graph_replay_equals_eager():
    case = "r8_b3"
    batch = _cuda(_batch(case))
    runs, sd = [], None
    for graphs in (False, True):
        model, sd = _model(case, sd=sd)
        model.train()
        model.engine.deterministic = True
        model.use_cuda_graphs = graphs
        model.pnp_net.dropblock_step = 4990
        seq = []
        for _ in range(3):
            ld = _train_step(model, batch)
            p = dict(model.named_parameters())
            seq.append((ld, model.pnp_net.dropblock_seeds.clone(), float(model.pnp_net.dropblock_scale),
                        {n: p[n].grad.clone() for n in ("rot_head_net.features.23.weight", "pnp_net.features.0.weight")}))
        assert model.pnp_net.dropblock_step == 4993
        runs.append(seq)
    for (ld_e, s_e, sc_e, g_e), (ld_g, s_g, sc_g, g_g) in zip(*runs):
        assert ld_e == ld_g and torch.equal(s_e, s_g) and sc_e == sc_g
        for n, v in g_e.items():
            assert torch.equal(g_g[n], v), n
    assert not torch.equal(runs[0][0][1], runs[0][1][1])


def test_frozen_pnp_still_drops():
    case = "ship_b5"
    model, sd = _model(case, freeze_pnp=True)
    model.train()
    model.pnp_net.dropblock_step = 4999
    batch_cpu = _batch(case)
    ld = _train_step(model, _cuda(batch_cpu))
    seeds = _check_mask(model, case)
    assert int(seeds.sum()) > 0
    _against_oracle(case, model, sd, batch_cpu, ld, seeds, grads=False)


@pytest.mark.parametrize("case", ["ship_b5", "r32_noatt_b4"])
def test_standalone_patch_pnp_train_mode(case):
    model, sd = _model(case)
    pn = model.pnp_net
    pn.train()
    pn.dropblock_step = 4999
    B = 8
    g = torch.Generator().manual_seed(3)
    n_reg = pn.nIn - 5
    coor = torch.rand(B, 5, 64, 64, generator=g)
    region = torch.softmax(torch.randn(B, n_reg, 64, 64, generator=g), 1) if n_reg else None
    ext = torch.rand(B, 3, generator=g) * 0.2 + 0.05
    rot, t = pn(coor.cuda(), None if region is None else region.cuda(), ext.cuda())
    torch.cuda.synchronize()
    seeds = pn.dropblock_seeds.cpu()
    assert pn.dropblock_step == 5000 and int(seeds.sum()) > 0
    leaf = O.leaf_state_dict(sd, requires_grad=False)
    reg = region if region is not None else torch.zeros(B, 0, 64, 64)
    r_o, t_o = DB.pnp_forward(coor.clone(), reg, ext, leaf, seeds=seeds, block_size=CASES[case][3])
    print(f"[{case}] stand-alone rot rel {_rel(rot, r_o):.2e} t rel {_rel(t, t_o):.2e}")
    assert _rel(rot, r_o) < REL and _rel(t, t_o) < REL
    # eval mode: no mask, the counter still advances
    pn.eval()
    rot_e, _ = pn(coor.cuda(), None if region is None else region.cuda(), ext.cuda())
    r_e, _ = DB.pnp_forward(coor.clone(), reg, ext, leaf)
    assert pn.dropblock_step == 5001 and _rel(rot_e, r_e) < REL


def test_no_new_launches_without_dropblock():
    from gdr_net_b200.capi import launch_count

    case = "ship_b5"
    batch = _cuda(_batch(case))
    counts = []
    for p in (0.0, 0.25):
        model, _ = _model(case, drop_prob=p)
        model.train()
        _train_step(model, batch)  # warm-up: workspaces, pack tables
        n0 = launch_count()
        _train_step(model, batch)
        counts.append(launch_count() - n0)
        if p == 0.0:
            assert model.pnp_net._db_step is None
    # DropBlock adds the sampler and its finish kernel; the glue and head backward replace their plain versions one for one
    assert counts[1] - counts[0] == 2, counts
