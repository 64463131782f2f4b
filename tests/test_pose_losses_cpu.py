"""CPU: the PNP_NET pose-loss switches (PM_*, ROT_*, CENTROID_/Z_LOSS_TYPE, TRANS_*, BIND_*; GDRN.py:402-514).

  * the oracle restatement (oracle/pose_loss_oracle.py) against the unmodified reference built with those switches
    (tests/golden/train_pose_losses_b4.npz, oracle/make_golden_pose_losses.py);
  * `build_model_optimizer` accepts every golden case, the engine's loss-name list is the reference's loss_dict keys in order,
    and the unsupported switches are rejected naming the key;
  * gdrn_pose_loss_ex / gdrn_loss_finalize_ex2 / gdrn_pose_loss_count are declared and exported."""
import ctypes
import os

import numpy as np
import pytest
import torch

from gdr_net_b200 import synth
from oracle import gdrn_oracle as O
from oracle import pose_loss_oracle as P

CASES = {  # as oracle/make_golden_pose_losses.py
    "rt_sl1": (dict(PM_R_ONLY=False, PM_LOSS_TYPE="Smooth_L1", PM_SMOOTH_L1_BETA=0.5, ROT_LW=1.0, ROT_LOSS_TYPE="angular",
                    TRANS_LW=1.0, TRANS_LOSS_TYPE="MSE", TRANS_LOSS_DISENTANGLE=True, BIND_LW=1.0, BIND_LOSS_TYPE="L1"), 7, 31, False),
    "disz_l2": (dict(PM_R_ONLY=False, PM_DISENTANGLE_Z=True, PM_T_USE_POINTS=True, PM_LOSS_TYPE="L2", ROT_LW=1.0,
                     ROT_LOSS_TYPE="L2", TRANS_LW=1.0, TRANS_LOSS_TYPE="L2", TRANS_LOSS_DISENTANGLE=False,
                     CENTROID_LOSS_TYPE="MSE", Z_LOSS_TYPE="L2"), 8, 37, False),
    "dist_nop_sym": (dict(PM_R_ONLY=False, PM_DISENTANGLE_T=True, PM_T_USE_POINTS=False, PM_LOSS_TYPE="MSE",
                          PM_NORM_BY_EXTENT=False, PM_LOSS_SYM=True, ROT_LW=1.0, ROT_LOSS_TYPE="angular", BIND_LW=1.0,
                          BIND_LOSS_TYPE="L1"), 9, 41, "ycbv"),
    "bind_mse": (dict(PM_R_ONLY=False, PM_DISENTANGLE_Z=True, PM_T_USE_POINTS=False, BIND_LW=1.0, BIND_LOSS_TYPE="MSE",
                      CENTROID_LOSS_TYPE="MSE"), 10, 43, False),
    "pm_off": (dict(PM_LW=0.0, ROT_LW=1.0, ROT_LOSS_TYPE="angular", TRANS_LW=1.0, TRANS_LOSS_TYPE="L1"), 11, 47, False),
}
PIXEL = ["loss_coor_x", "loss_coor_y", "loss_coor_z", "loss_mask", "loss_region"]


def pose_config(device="cpu", **switches):
    from gdr_net_b200.config import a6_config

    cfg = a6_config(device=device)
    for k, v in switches.items():
        setattr(cfg.MODEL.CDPN.PNP_NET, k, v)
    return cfg


def seeded_weights(cfg, seed):
    from gdr_net_b200 import GDRN as G

    model, _ = G.build_model_optimizer(cfg)
    return synth.seeded_state_dict(model.state_dict(), seed=seed)


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "train_pose_losses_b4.npz"))


# ------------------------------------------------------------------------------------------------ oracle vs reference goldens
@pytest.mark.parametrize("case", sorted(CASES))
def test_oracle_matches_reference_golden(golden, case):
    switches, wseed, bseed, with_sym = CASES[case]
    cfg = pose_config(**switches)
    sd = seeded_weights(pose_config(**switches), wseed)
    batch = synth.make_batch(4, seed=bseed, with_sym=with_sym)
    leaf = O.leaf_state_dict(sd)
    o = P.gdrn_forward(leaf, batch, cfg.MODEL.CDPN.PNP_NET, pm_sym=bool(switches.get("PM_LOSS_SYM")), update_stats=True)
    assert list(o["losses"]) == list(golden[f"{case}/names"])
    for k, v in o["losses"].items():
        ref = float(golden[f"{case}/loss/{k}"])
        err = abs(float(v.detach()) - ref) / abs(ref)
        print(case, k, f"{err:.2e}")
        assert err <= 1e-6, (k, float(v.detach()), ref)
    sum(o["losses"].values()).backward()
    prefix = f"{case}/grad/"
    for key in golden.files:
        if key.startswith(prefix):
            name = key[len(prefix):]
            ref = golden[key]
            err = np.abs(leaf[name].grad.numpy() - ref).max() / np.abs(ref).max()
            print(case, name, f"{err:.2e}")
            assert err <= 3e-6, (name, err)


def test_oracle_default_switches_are_gdrn_oracle():
    """With the shipped switches the restatement is gdrn_oracle.gdrn_losses' pose part, bit for bit."""
    batch = synth.make_batch(2, seed=3)
    g = torch.Generator().manual_seed(1)
    rot = O.quat2mat(torch.nn.functional.normalize(torch.randn(2, 4, generator=g), dim=1))
    t, pred_t = torch.randn(2, 3, generator=g), torch.randn(2, 3, generator=g)
    a = O.gdrn_losses(torch.randn(2, 69, 8, 8, generator=g), rot, pred_t, dict(batch, roi_xyz=torch.zeros(2, 3, 8, 8),
                      roi_mask_visib=torch.ones(2, 8, 8), roi_mask_trunc=torch.ones(2, 8, 8),
                      roi_region=torch.zeros(2, 8, 8, dtype=torch.long)))
    b = P.pose_losses(pose_config().MODEL.CDPN.PNP_NET, rot, t, pred_t, batch)
    assert list(b) == ["loss_PM_R", "loss_centroid", "loss_z"]
    for k in b:
        assert torch.equal(a[k], b[k]), k


def test_smooth_l1_is_fvcore():
    """fvcore's smooth_l1_loss: plain L1 below beta = 1e-5, torch's smooth L1 (continuous at |e| = beta) above."""
    a, b = torch.tensor([0.0, 0.3, -0.5, 2.0]), torch.zeros(4)
    assert torch.equal(P.smooth_l1(a, b, 1e-6), (a - b).abs().mean())
    v = P.smooth_l1(a, b, 0.5)
    assert torch.allclose(v, torch.tensor([0.0, 0.5 * 0.09 / 0.5, 0.25, 1.75]).mean())


# ------------------------------------------------------------------------------------------------ configuration surface
@pytest.mark.parametrize("case", sorted(CASES))
def test_build_accepts_case_and_names_match_golden(golden, case):
    from gdr_net_b200 import GDRN as G
    from gdr_net_b200.engine import pose_loss_switches

    switches = CASES[case][0]
    cfg = pose_config(**switches)
    G.build_model_optimizer(cfg)
    _, names = pose_loss_switches(cfg.MODEL.CDPN.PNP_NET)
    assert PIXEL + names == list(golden[f"{case}/names"])


def test_default_switches_keep_the_default_loss_list():
    from gdr_net_b200.engine import DEFAULT_POSE_SWITCHES, LOSS_NAMES, pose_loss_switches

    sw, names = pose_loss_switches(pose_config().MODEL.CDPN.PNP_NET)
    assert PIXEL + names == LOSS_NAMES
    assert all(sw[k] == v for k, v in DEFAULT_POSE_SWITCHES.items())


@pytest.mark.parametrize("key,value", [("PM_LOSS_TYPE", "Huber"), ("ROT_LOSS_TYPE", "geodesic"), ("CENTROID_LOSS_TYPE", "SmoothL1"),
                                       ("Z_LOSS_TYPE", "l1"), ("TRANS_LOSS_TYPE", "Huber"), ("BIND_LOSS_TYPE", "MSE"),
                                       ("ROT_TYPE", "allo_quat"), ("TRANS_TYPE", "trans"), ("Z_TYPE", "ABS"), ("R_ONLY", True)])
def test_build_rejects_unsupported_pose_switches(key, value):
    """Each raises NotImplementedError naming the key.  BIND_LOSS_TYPE = "MSE" with an L1 centroid loss is the reference's
    ValueError (GDRN.py:510 tests CENTROID_LOSS_TYPE); with CENTROID_LOSS_TYPE = "MSE" it is accepted (golden bind_mse)."""
    from gdr_net_b200 import GDRN as G

    extra = dict(ROT_LW=1.0, TRANS_LW=1.0, BIND_LW=1.0)
    with pytest.raises(NotImplementedError) as e:
        G.build_model_optimizer(pose_config(**dict(extra, **{key: value})))
    assert key in str(e.value), str(e.value)


def test_build_rejects_mtl():
    from gdr_net_b200 import GDRN as G

    cfg = pose_config()
    cfg.MODEL.CDPN.USE_MTL = True
    with pytest.raises(NotImplementedError) as e:
        G.build_model_optimizer(cfg)
    assert "USE_MTL" in str(e.value)


# ------------------------------------------------------------------------------------------------ C ABI
def test_pose_loss_ex_entry_points_declared_and_exported():
    from gdr_net_b200 import capi

    protos = capi.parse_header()
    want = {"gdrn_pose_loss_ex": 24, "gdrn_loss_finalize_ex2": 10, "gdrn_pose_loss_count": 1, "gdrn_pose_loss": 25}
    for name, nargs in want.items():
        assert name in protos and len(protos[name][1]) == nargs, (name, protos.get(name))
    assert protos["gdrn_pose_loss_ex"][1][22] is capi.PoseSwitches
    if not os.path.exists(capi.LIB_PATH):
        pytest.skip("library not built")
    dll = ctypes.CDLL(capi.LIB_PATH)
    for name in want:
        assert hasattr(dll, name), name


def test_pose_loss_count_matches_the_name_list():
    """The library's slot mask and the engine's name list agree for every golden case (by-value struct through ctypes)."""
    from gdr_net_b200 import capi
    from gdr_net_b200.engine import pose_loss_switches

    if not os.path.exists(capi.LIB_PATH):
        pytest.skip("library not built")
    dll = capi.C.load()
    for case in CASES:
        sw, names = pose_loss_switches(pose_config(**CASES[case][0]).MODEL.CDPN.PNP_NET)
        assert dll.gdrn_pose_loss_count(capi.PoseSwitches(**sw)) == len(names), case
    bad = dict(pose_loss_switches(pose_config().MODEL.CDPN.PNP_NET)[0], pm_type=7)
    rc = dll.gdrn_loss_finalize_ex2(None, None, None, None, None, 1, 4096, 1, capi.PoseSwitches(**bad), None)
    assert rc == -1 and b"pm_type" in dll.gdrn_last_error()
