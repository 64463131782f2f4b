"""CPU: frozen sub-networks (MODEL.CDPN.BACKBONE.FREEZE, ROT_HEAD.FREEZE, PNP_NET.FREEZE; GDRN.py:550-700).

  * the freeze-aware oracle (oracle/freeze_oracle.py) against the unmodified reference built with those switches
    (tests/golden/train_freeze_<case>_b4.npz, oracle/make_golden_freeze.py): losses, which gradients are None, gradients and
    BatchNorm running statistics;
  * `build_model_optimizer` against the reference: requires_grad flags, param groups (count, order, learning rates), and the
    exception of the all-frozen case;
  * TRANS_HEAD.ENABLED and USE_MTL are still rejected, with their keys named."""
import os

import numpy as np
import pytest
import torch

from gdr_net_b200 import synth
from oracle import fixtures
from oracle import freeze_oracle as FO
from oracle import gdrn_oracle as O
from oracle.make_golden_freeze import BSEED, WSEED

SUBNET = {"backbone": "backbone.", "head": "rot_head_net.", "pnp": "pnp_net."}


def freeze_config(case, device="cpu"):
    from gdr_net_b200.config import a6_config

    cfg = a6_config(device=device)
    fb, fh, fp = FO.CASES[case]
    cfg.MODEL.CDPN.BACKBONE.FREEZE, cfg.MODEL.CDPN.ROT_HEAD.FREEZE, cfg.MODEL.CDPN.PNP_NET.FREEZE = fb, fh, fp
    return cfg


def _golden(golden_dir, case):
    return np.load(os.path.join(golden_dir, f"train_freeze_{case}_b4.npz"))


@pytest.mark.parametrize("case", [c for c in sorted(FO.CASES) if c != "all"])
def test_oracle_matches_reference_golden(golden_dir, case):
    g = _golden(golden_dir, case)
    freeze = FO.CASES[case]
    sd = fixtures.calibrated_state_dict(WSEED)
    batch = synth.make_batch(4, seed=BSEED)
    leaf = O.leaf_state_dict(sd)
    for k, v in leaf.items():  # requires_grad = False on the frozen sub-networks, as build_model_optimizer sets it
        if v.requires_grad and any(freeze[i] and k.startswith(p) for i, p in enumerate(SUBNET.values())):
            v.requires_grad_(False)
    o = FO.gdrn_forward(leaf, batch, train=True, do_loss=True, freeze=freeze, update_stats=True)
    # losses: the same CPU ops in the same order as the reference, bit for bit; a frozen head has no per-pixel losses
    assert list(o["losses"]) == [k[len("loss/"):] for k in g.files if k.startswith("loss/")]
    for k, v in o["losses"].items():
        assert float(v.detach()) == float(g["loss/" + k]), (k, float(v.detach()), float(g["loss/" + k]))
    # BatchNorm running statistics: a frozen backbone or head under no_grad still updates them
    for key in g.files:
        if key.startswith("bn/"):
            assert np.array_equal(leaf[key[len("bn/"):]].numpy(), g[key]), key
    if str(g["exc/backward"]):
        assert str(g["exc/backward"]) == "RuntimeError" and case == "head_pnp"
        assert not any(v.requires_grad for v in o["losses"].values())
        with pytest.raises(RuntimeError):
            sum(o["losses"].values()).backward()
    else:
        sum(o["losses"].values()).backward()
    params = [k for k, v in leaf.items() if v.dtype.is_floating_point and not k.endswith(("running_mean", "running_var"))]
    none = [k for k in params if leaf[k].grad is None]
    assert none == list(g["none_grad"])
    assert none == [k for k in params if not FO.live(k, freeze)]
    n_grads = 0
    for key in g.files:
        if key.startswith("grad/"):
            name = key[len("grad/"):]
            ref = g[key]
            err = np.abs(leaf[name].grad.numpy() - ref).max() / np.abs(ref).max()
            print(case, name, f"{err:.2e}")
            assert err <= 5e-6, (name, err)
            n_grads += 1
    live_nets = [p for p in SUBNET.values() if any(FO.live(k, freeze) for k in params if k.startswith(p))]
    assert n_grads > 0 or not live_nets
    for p in live_nets:  # every live sub-network has gradients in the golden
        assert any(k.startswith("grad/" + p) for k in g.files), p


@pytest.mark.parametrize("case", sorted(FO.CASES))
def test_build_model_optimizer_matches_reference(golden_dir, case):
    from gdr_net_b200 import GDRN as G

    g = _golden(golden_dir, case)
    cfg = freeze_config(case)
    if str(g["exc/build"]):
        # all three frozen: the optimizer gets an empty parameter list, and building it raises what the reference raises
        with pytest.raises(Exception) as ei:
            G.build_model_optimizer(cfg)
        assert type(ei.value).__name__ == str(g["exc/build"])
        return
    model, opt = G.build_model_optimizer(cfg)
    freeze = FO.CASES[case]
    for name, p in model.named_parameters():
        frozen = any(freeze[i] and name.startswith(pre) for i, pre in enumerate(SUBNET.values()))
        assert p.requires_grad == (not frozen), name
    assert [grp["lr"] for grp in opt.param_groups] == g["opt/lrs"].tolist()
    assert [len(grp["params"]) for grp in opt.param_groups] == g["opt/sizes"].tolist()
    # group order: backbone, head, Patch-PnP, each only if not frozen
    subnets = [pre for i, pre in enumerate(SUBNET.values()) if not freeze[i]]
    names = {id(p): n for n, p in model.named_parameters()}
    assert len(opt.param_groups) == len(subnets)
    for grp, pre in zip(opt.param_groups, subnets):
        assert all(names[id(p)].startswith(pre) for p in grp["params"]), pre
        assert len(grp["params"]) == sum(1 for n, _ in model.named_parameters() if n.startswith(pre))


def test_pnp_lr_mult_group_follows_pnp_freeze():
    """PNP_NET.LR_MULT scales the Patch-PnP group, which a frozen Patch-PnP does not have."""
    from gdr_net_b200 import GDRN as G

    for case, n in (("bb", 2), ("bb_pnp", 1)):
        cfg = freeze_config(case)
        cfg.MODEL.CDPN.PNP_NET.LR_MULT = 0.5
        _, opt = G.build_model_optimizer(cfg)
        lrs = [grp["lr"] for grp in opt.param_groups]
        assert len(lrs) == n
        assert lrs[-1] == (cfg.SOLVER.BASE_LR * 0.5 if case == "bb" else cfg.SOLVER.BASE_LR)


@pytest.mark.parametrize("key", ["TRANS_HEAD.ENABLED", "USE_MTL"])
def test_trans_head_and_mtl_still_rejected(key):
    from gdr_net_b200 import GDRN as G

    cfg = freeze_config("bb")
    if key == "USE_MTL":
        cfg.MODEL.CDPN.USE_MTL = True
    else:
        cfg.MODEL.CDPN.TRANS_HEAD.ENABLED = True
    with pytest.raises(NotImplementedError, match=key.replace(".", r"\.")):
        G.build_model_optimizer(cfg)


def test_freeze_message_no_longer_names_freeze():
    """Every non-empty freeze combination builds; none of the remaining rejections mentions FREEZE."""
    from gdr_net_b200 import GDRN as G

    for case in ("bb", "head", "pnp", "bb_pnp", "head_pnp"):
        G._check_supported(freeze_config(case))
    cfg = freeze_config("pnp")
    cfg.MODEL.CDPN.USE_MTL = True
    with pytest.raises(NotImplementedError) as ei:
        G.build_model_optimizer(cfg)
    assert "FREEZE" not in str(ei.value)


def test_oracle_without_switches_is_gdrn_oracle():
    """freeze = (False, False, False) is gdrn_oracle.gdrn_forward itself, bit for bit."""
    sd = fixtures.calibrated_state_dict(WSEED)
    batch = synth.make_batch(2, seed=BSEED)
    with torch.no_grad():
        a = O.gdrn_forward(O.leaf_state_dict(sd, requires_grad=False), batch, train=True, do_loss=True)
        b = FO.gdrn_forward(O.leaf_state_dict(sd, requires_grad=False), batch, train=True, do_loss=True)
    assert list(a["losses"]) == list(b["losses"])
    for k in a["losses"]:
        assert torch.equal(a["losses"][k], b["losses"][k]), k
    assert torch.equal(a["head"], b["head"])
