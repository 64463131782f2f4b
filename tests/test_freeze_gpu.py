"""GPU: frozen sub-networks (MODEL.CDPN.BACKBONE.FREEZE, ROT_HEAD.FREEZE, PNP_NET.FREEZE) through the whole model.

  * B = 4, "mixed": every case of tests/golden/train_freeze_<case>_b4.npz against the golden and the oracle (oracle/freeze_oracle.py)
    with the bounds of tests/test_mask_heads_gpu.py; frozen and unreachable parameters keep .grad None; with the head and the
    Patch-PnP frozen the losses do not require grad, so backward raises RuntimeError as the reference's does;
  * B = 64, "mixed": the frozen-backbone step against the oracle with the bounds of tests/test_parity_b64_gpu.py;
  * freezing removes work and changes none of the rest: in deterministic mode the live gradients are those of an unfrozen step;
  * the data-parallel hook sees exactly the live segments; a frozen backbone keeps no activations and needs less memory;
  * Ranger steps through TrainStep leave frozen parameters unchanged and still advance frozen BatchNorm statistics, and a
    graphed replay equals eager bit for bit."""
import os

import numpy as np
import pytest
import torch

from gdr_net_b200 import synth
from oracle import fixtures
from oracle import freeze_oracle as FO
from oracle import gdrn_oracle as O
from oracle.make_golden_freeze import BSEED, WSEED

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

REL = 1e-3
TRAINABLE = [c for c in sorted(FO.CASES) if c != "all"]
STAGES = ["pnp_net", "rot_head_net", "backbone.layer4", "backbone.layer3", "backbone.layer2", "backbone.stem"]


@pytest.fixture(scope="module", autouse=True)
def _gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _cfg(case):
    from gdr_net_b200.config import a6_config

    cfg = a6_config(device="cuda")
    cfg.MODEL.CDPN.BACKBONE.FREEZE, cfg.MODEL.CDPN.ROT_HEAD.FREEZE, cfg.MODEL.CDPN.PNP_NET.FREEZE = FO.CASES.get(case, (False,) * 3)
    return cfg


def _model(case, sd, precision="mixed"):
    from gdr_net_b200 import GDRN as G

    model, opt = G.build_model_optimizer(_cfg(case), precision=precision)
    model.load_state_dict(sd)
    model.train()
    return model, opt


def _cuda(batch):
    return {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in batch.items()}


def _forward(model, batch):
    for p in model.parameters():
        p.grad = None
    return model(batch["roi_img"], **synth.forward_kwargs(batch, train=True))[1]


def _step(model, batch):
    ld = _forward(model, batch)
    sum(ld.values()).backward()
    torch.cuda.synchronize()
    return {k: float(v.detach()) for k, v in ld.items()}


@pytest.mark.parametrize("case", TRAINABLE)
def test_b4_matches_golden_and_oracle(case, golden_dir):
    g = np.load(os.path.join(golden_dir, f"train_freeze_{case}_b4.npz"))
    freeze = FO.CASES[case]
    sd = fixtures.calibrated_state_dict(WSEED)
    model, _ = _model(case, sd)
    batch_cpu = synth.make_batch(4, seed=BSEED)
    batch = _cuda(batch_cpu)
    ld = _forward(model, batch)
    assert list(ld) == [k[len("loss/"):] for k in g.files if k.startswith("loss/")]
    leaf = O.leaf_state_dict(sd)
    o = FO.gdrn_forward(leaf, batch_cpu, train=True, do_loss=True, freeze=freeze, update_stats=True)
    for k, v in ld.items():
        v, ref = float(v.detach()), float(g["loss/" + k])
        print(f"[{case}] B=4 {k}: {v:.6f} vs golden {ref:.6f} rel {abs(v - ref) / abs(ref):.2e}")
        assert abs(v - ref) <= 2 * REL * abs(ref), (k, v, ref)
        assert abs(v - float(o["losses"][k])) <= 2 * REL * abs(ref), k
    # BatchNorm running statistics after the train-mode forward, frozen sub-networks included
    bufs = dict(model.named_buffers())
    for key in g.files:
        if key.startswith("bn/"):
            name = key[len("bn/"):]
            if name.endswith("num_batches_tracked"):
                assert int(bufs[name]) == int(g[key]), name
            else:
                assert _rel(bufs[name], g[key]) < REL, (name, _rel(bufs[name], g[key]))
    if case == "head_pnp":
        assert not any(v.requires_grad for v in ld.values())
        with pytest.raises(RuntimeError):
            sum(ld.values()).backward()
    else:
        sum(ld.values()).backward()
        sum(o["losses"].values()).backward()
    torch.cuda.synchronize()
    params = dict(model.named_parameters())
    assert [n for n, p in params.items() if p.grad is None] == list(g["none_grad"])
    for key in g.files:
        if key.startswith("grad/"):
            name = key[len("grad/"):]
            r_g, r_o = _rel(params[name].grad, g[key]), _rel(params[name].grad, leaf[name].grad)
            print(f"[{case}] grad {name}: rel-L2 vs golden {r_g:.2e}, vs oracle {r_o:.2e}")
            assert r_g < 0.06 and r_o < 0.06, (name, r_g, r_o)
    assert all(torch.isfinite(p.grad).all() for p in params.values() if p.grad is not None)


def test_b64_frozen_backbone_matches_oracle():
    """The benchmark's batch and weights (B = 64, seed 100) with a frozen backbone: every loss within 1e-3 of the oracle."""
    sd = synth.seeded_state_dict(fixtures.template_from_manifest(), 0)
    batch_cpu = synth.make_batch(64, seed=100)
    with torch.no_grad():
        o = FO.gdrn_forward(O.leaf_state_dict(sd, requires_grad=False), batch_cpu, train=True, do_loss=True, freeze=FO.CASES["bb"])
    model, _ = _model("bb", sd)
    ld = _step(model, _cuda(batch_cpu))
    assert list(ld) == list(o["losses"])
    for k, v in ld.items():
        ref = float(o["losses"][k])
        print(f"[bb] B=64 {k}: {v:.6f} vs {ref:.6f} rel {abs(v - ref) / abs(ref):.2e}")
        assert abs(v - ref) <= REL * abs(ref), (k, v, ref)
    for n, p in model.named_parameters():
        assert (p.grad is None) == n.startswith("backbone."), n
        assert p.grad is None or torch.isfinite(p.grad).all(), n


def _grads(model):
    return {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}


@pytest.mark.parametrize("case", ["bb", "head", "pnp"])
def test_live_gradients_equal_the_unfrozen_step(case):
    """Deterministic mode: the live gradients of a frozen step are those of an unfrozen step on the same weights and batch.
    Every gradient that two unfrozen runs reproduce bit for bit is reproduced bit for bit; the few that are summed with
    atomics (bias and GroupNorm entries) differ by no more than two unfrozen runs differ from each other."""
    sd = fixtures.calibrated_state_dict(WSEED)
    batch = _cuda(synth.make_batch(4, seed=BSEED))
    runs = []
    for c in (None, None, case):
        model, _ = _model(c, sd)
        model.engine.deterministic = True
        _step(model, batch)
        runs.append(_grads(model))
    full, full2, frozen = runs
    freeze = FO.CASES[case]
    assert sorted(frozen) == sorted(n for n in full if FO.live(n, freeze))
    n_exact = 0
    for n, g in frozen.items():
        if torch.equal(full[n], full2[n]):
            assert torch.equal(g, full[n]), n
            n_exact += 1
        else:
            assert (g - full[n]).abs().max() <= 4 * (full2[n] - full[n]).abs().max(), n
    assert n_exact >= len(frozen) // 2, (n_exact, len(frozen))


@pytest.mark.parametrize("case", ["none"] + TRAINABLE)
def test_grad_hook_sees_the_live_segments(case):
    sd = fixtures.calibrated_state_dict(WSEED)
    model, _ = _model(case, sd)
    seen = []
    eng = model.engine
    eng.grad_hook = lambda engine, stage: seen.append(stage)
    ld = _forward(model, _cuda(synth.make_batch(4, seed=BSEED)))
    if case != "head_pnp":
        sum(ld.values()).backward()
    torch.cuda.synchronize()
    freeze = FO.CASES.get(case, (False,) * 3)
    want = [s for s in STAGES if FO.live(s + ".", freeze)]
    assert seen == want, (seen, want)


def test_frozen_backbone_keeps_no_activations_and_needs_less_memory():
    B = 64
    sd = synth.seeded_state_dict(fixtures.template_from_manifest(), 0)
    batch = _cuda(synth.make_batch(B, seed=100))
    peaks = {}
    for case in ("none", "bb"):
        model, _ = _model(case, sd)
        _step(model, batch)  # warm: weight packs, split-K workspace
        eng = model.engine
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        ld = _forward(model, batch)
        S = eng.saved
        if case == "bb":
            assert not any(k in S for k in ("stem", "blocks")), sorted(S)
            assert "deconv" in S and "head" in S
        else:
            assert all(k in S for k in ("stem", "blocks", "deconv", "head"))
        sum(ld.values()).backward()
        torch.cuda.synchronize()
        peaks[case] = torch.cuda.max_memory_allocated()
        del model, eng, S, ld
        torch.cuda.empty_cache()
    a_col = B * 128 * 128 * 192 * 2 * 2  # the stem's im2col matrix: two 16-bit planes in "mixed"
    print(f"peak allocation: unfrozen {peaks['none'] / 2**30:.2f} GiB, frozen backbone {peaks['bb'] / 2**30:.2f} GiB")
    assert peaks["bb"] <= peaks["none"] - a_col, peaks


@pytest.mark.parametrize("case", ["bb", "head", "pnp", "bb_pnp"])
def test_ranger_steps_keep_frozen_parameters_and_advance_bn_statistics(case):
    from gdr_net_b200.train_harness import TrainStep

    sd = fixtures.calibrated_state_dict(WSEED)
    model, opt = _model(case, sd)
    freeze = FO.CASES[case]
    before = {n: p.detach().clone() for n, p in model.named_parameters()}
    bufs0 = {n: b.clone() for n, b in model.named_buffers()}
    step = TrainStep(model, opt, use_cuda_graphs=True)
    batch = _cuda(synth.make_batch(4, seed=BSEED))
    n_steps = 3
    for _ in range(n_steps):
        step(batch)
    torch.cuda.synchronize()
    for n, p in model.named_parameters():
        if FO.live(n, freeze):
            assert not torch.equal(p.detach(), before[n]) or n.endswith("bias"), n
        else:
            assert torch.equal(p.detach(), before[n]), n
            assert p.grad is None, n
    for n, b in model.named_buffers():  # every BatchNorm, frozen or not, normalises with batch statistics and updates
        if n.endswith("num_batches_tracked"):
            assert int(b) == int(bufs0[n]) + n_steps, n
        elif n.endswith("running_mean"):
            assert not torch.equal(b, bufs0[n]), n


@pytest.mark.parametrize("case", TRAINABLE)
def test_graph_replay_equals_eager(case):
    """Deterministic mode: losses and the gradients of parameters that are not atomically summed are bit-identical between
    eager steps and captured replays, as tests/test_mask_heads_gpu.py checks for the unfrozen step."""
    sd = fixtures.calibrated_state_dict(WSEED)
    batch = _cuda(synth.make_batch(4, seed=BSEED))
    keys = ("rot_head_net.features.23.weight", "rot_head_net.features.20.weight", "backbone.layer1.0.conv1.weight",
            "pnp_net.features.0.weight")
    runs = []
    for graphs in (False, True):
        model, _ = _model(case, sd)
        model.engine.deterministic = True
        model.use_cuda_graphs = graphs
        for _ in range(2):  # the second step replays when graphs are on
            ld = _forward(model, batch)
            if case != "head_pnp":
                sum(ld.values()).backward()
            torch.cuda.synchronize()
        p = dict(model.named_parameters())
        runs.append(({k: float(v.detach()) for k, v in ld.items()}, {n: p[n].grad for n in keys}))
    (l0, g0), (l1, g1) = runs
    assert l0 == l1
    for n in keys:
        assert (g0[n] is None) == (g1[n] is None) == (not FO.live(n, FO.CASES[case])), n
        if g0[n] is not None:
            assert torch.equal(g0[n], g1[n]), n


@pytest.mark.parametrize("case", TRAINABLE)
def test_eval_outputs_do_not_depend_on_freezing(case):
    sd = fixtures.calibrated_state_dict(WSEED)
    batch = _cuda(synth.make_batch(4, seed=BSEED))
    outs = []
    for c in (None, case):
        model, _ = _model(c, sd)
        model.eval()
        with torch.no_grad():
            outs.append(model(batch["roi_img"], **synth.forward_kwargs(batch, train=False)))
    for k in outs[0]:
        assert torch.equal(outs[0][k], outs[1][k]), k
