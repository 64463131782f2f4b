"""CPU: any surface-region count (ROT_HEAD.NUM_REGIONS = 2..64) and Patch-PnP without region attention (PNP_NET.REGION_ATTENTION).

  * the oracle restatement (oracle/region_oracle.py) against the unmodified reference built with those switches
    (tests/golden/train_regions_b4.npz, oracle/make_golden_regions.py);
  * `build_model_optimizer` accepts every such configuration with the reference's parameter shapes and rejects R outside 2..64,
    naming the key; mask attention stays rejected;
  * the _ex2 entry points are declared and exported, report argument errors without a GPU, and their kernels keep everything
    in registers (no stack frame, no local memory)."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from gdr_net_b200 import synth
from oracle import gdrn_oracle as O
from oracle import region_oracle as RO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# as oracle/make_golden_regions.py: name -> (ROT_HEAD switches, PNP_NET switches, weight seed, batch seed, eval maps)
CASES = {
    "r8": (dict(NUM_REGIONS=8), dict(REGION_ATTENTION=True, WITH_2D_COORD=True), 31, 41, True),
    "r32_noatt": (dict(NUM_REGIONS=32), dict(REGION_ATTENTION=False, WITH_2D_COORD=True), 32, 42, True),
    "r64_noatt": (dict(NUM_REGIONS=64), dict(REGION_ATTENTION=False, WITH_2D_COORD=True), 33, 43, False),
    "r4_ce": (dict(NUM_REGIONS=4, MASK_LOSS_TYPE="CE", REGION_LOSS_MASK_GT="trunc"), dict(REGION_ATTENTION=True, WITH_2D_COORD=False),
              34, 44, False),
    "r60": (dict(NUM_REGIONS=60), dict(REGION_ATTENTION=True, WITH_2D_COORD=True), 35, 45, False),
}
N_IN = {"r8": 13, "r32_noatt": 5, "r64_noatt": 5, "r4_ce": 7, "r60": 65}


def region_config(case, device="cpu", **kw):
    from gdr_net_b200.config import a6_config

    rh, pn, *_ = CASES[case]
    cfg = a6_config(device=device, **kw)
    for k, v in rh.items():
        setattr(cfg.MODEL.CDPN.ROT_HEAD, k, v)
    for k, v in pn.items():
        setattr(cfg.MODEL.CDPN.PNP_NET, k, v)
    return cfg


def mask_gt(cfg):
    r = cfg.MODEL.CDPN.ROT_HEAD
    return (r.XYZ_LOSS_MASK_GT, r.MASK_LOSS_GT, r.REGION_LOSS_MASK_GT)


def oracle_kwargs(case):
    rh, pn, *_ = CASES[case]
    cfg = region_config(case)
    return dict(mask_loss_type=rh.get("MASK_LOSS_TYPE", "L1"), mask_gt=mask_gt(cfg), region_att=pn["REGION_ATTENTION"],
                with_2d=pn["WITH_2D_COORD"])


def seeded_weights(case):
    from gdr_net_b200 import GDRN as G

    model, _ = G.build_model_optimizer(region_config(case))
    return synth.seeded_state_dict(model.state_dict(), seed=CASES[case][2])


def _golden(golden_dir, case):
    g = np.load(os.path.join(golden_dir, "train_regions_b4.npz"))
    return {k[len(case) + 1:]: g[k] for k in g.files if k.startswith(case + "/")}


# ------------------------------------------------------------------------------------------------ oracle vs reference goldens
@pytest.mark.parametrize("case", list(CASES))
def test_oracle_matches_reference_golden(golden_dir, case):
    g = _golden(golden_dir, case)
    sd = seeded_weights(case)
    batch = synth.make_batch(4, seed=CASES[case][3], num_regions=CASES[case][0]["NUM_REGIONS"])
    kw = oracle_kwargs(case)
    if "eval/head" in g:
        # eval-mode head and pose: the same CPU ops in the same order as the reference, so bit-identical
        with torch.no_grad():
            o = RO.gdrn_forward(O.leaf_state_dict(sd, requires_grad=False), batch, train=False, do_loss=False, **kw)
        assert np.array_equal(o["head"][:, :, ::4, ::4].numpy(), g["eval/head"])
        assert np.array_equal(o["trans"].numpy(), g["eval/trans"])
        assert np.abs(o["rot"].numpy() - g["eval/rot"]).max() <= 1e-12
    leaf = O.leaf_state_dict(sd)
    o = RO.gdrn_forward(leaf, batch, train=True, do_loss=True, update_stats=True, **kw)
    assert o["layout"]["n_in"] == N_IN[case]
    assert list(o["losses"]) == [k[len("loss/"):] for k in g if k.startswith("loss/")]
    for k, v in o["losses"].items():
        assert float(v.detach()) == float(g["loss/" + k]), (k, float(v.detach()), float(g["loss/" + k]))
    sum(o["losses"].values()).backward()
    for key in g:
        if key.startswith("grad/"):
            name = key[len("grad/"):]
            ref = g[key]
            err = np.abs(leaf[name].grad.numpy() - ref).max() / np.abs(ref).max()
            print(case, name, f"{err:.2e}")
            # the accumulation order of autograd for a tensor used twice, as in tests/test_mask_heads_cpu.py
            assert err <= 5e-6, (name, err)


def test_layout_from_weight_shapes():
    for case in CASES:
        sd = seeded_weights(case)
        kw = oracle_kwargs(case)
        lay = RO.layout(sd, kw["mask_loss_type"])
        assert (lay["R"], lay["region_att"], lay["with_2d"], lay["n_in"]) == (
            CASES[case][0]["NUM_REGIONS"], kw["region_att"], kw["with_2d"], N_IN[case]), case


def test_make_batch_default_stream_and_labels():
    a, b = synth.make_batch(2, seed=7), synth.make_batch(2, seed=7, num_regions=64)
    for k, v in a.items():
        if isinstance(v, torch.Tensor):
            assert torch.equal(v, b[k]), k
    c = synth.make_batch(2, seed=7, num_regions=8)
    lab = c["roi_region"][c["roi_mask_obj"] > 0]
    assert int(lab.min()) == 1 and int(lab.max()) == 8
    assert int(c["roi_region"][c["roi_mask_obj"] == 0].abs().max()) == 0


# ------------------------------------------------------------------------------------------------ configuration surface
@pytest.mark.parametrize("case", list(CASES))
def test_build_model_accepts_region_configs(golden_dir, case):
    from gdr_net_b200 import GDRN as G

    model, _ = G.build_model_optimizer(region_config(case))
    R = CASES[case][0]["NUM_REGIONS"]
    mo = 2 if CASES[case][0].get("MASK_LOSS_TYPE") == "CE" else 1
    assert tuple(model.rot_head_net.features[23].weight.shape) == (mo + 4 + R, 256, 1, 1)
    assert model.pnp_net.features[0].in_channels == N_IN[case]
    # the parameter shapes of the reference's model (the golden gradients are its parameters' shapes)
    g = _golden(golden_dir, case)
    params = dict(model.named_parameters())
    for key in g:
        if key.startswith("grad/"):
            assert tuple(params[key[len("grad/"):]].shape) == g[key].shape, key
    missing, unexpected = model.load_state_dict(seeded_weights(case), strict=True)
    assert not missing and not unexpected


@pytest.mark.parametrize("R", [1, 65, 128])
def test_build_model_rejects_region_counts(R):
    from gdr_net_b200 import GDRN as G
    from gdr_net_b200.config import a6_config

    with pytest.raises(NotImplementedError) as e:
        G.build_model_optimizer(a6_config(device="cpu", num_regions=R))
    assert "ROT_HEAD.NUM_REGIONS" in str(e.value)


def test_mask_attention_still_rejected():
    from gdr_net_b200 import GDRN as G

    cfg = region_config("r32_noatt")
    cfg.MODEL.CDPN.PNP_NET.MASK_ATTENTION = "mul"
    with pytest.raises(NotImplementedError) as e:
        G.build_model_optimizer(cfg)
    assert "MASK_ATTENTION" in str(e.value)


# ------------------------------------------------------------------------------------------------ C ABI
NEW = {"gdrn_head_glue_fwd_ex2": 13, "gdrn_pixel_loss_fwd_ex2": 15, "gdrn_head_bwd_ex2": 22, "gdrn_pnp_pack_input_ex": 11}


def test_region_entry_points_declared_and_exported():
    from gdr_net_b200 import capi

    protos = capi.parse_header()
    for name, nargs in NEW.items():
        assert name in protos and len(protos[name][1]) == nargs, (name, protos.get(name))
    if not os.path.exists(capi.LIB_PATH):
        pytest.skip("library not built")
    dll = ctypes.CDLL(capi.LIB_PATH)
    for name in NEW:
        assert hasattr(dll, name), name


def test_region_argument_errors_without_a_gpu():
    from gdr_net_b200 import capi

    if not os.path.exists(capi.LIB_PATH):
        pytest.skip("library not built")
    dll = capi.C.load()
    for R, att, ld in ((1, 1, 64), (65, 1, 128), (0, 0, 64), (8, 2, 64), (8, 1, 96), (8, 1, 256)):
        rc = dll.gdrn_pixel_loss_fwd_ex2(None, None, None, None, None, None, None, 1, 4096, 0, 1, R, att, ld, None)
        assert rc == -1, (R, att, ld)
        err = dll.gdrn_last_error()
        assert any(w in err for w in (b"num_regions", b"region_att", b"pnp_ld")), err
    # the Patch-PnP input width must be round_up(nIn, 64): 8 regions + xyz + coord2d = 13 -> 64; 60 + 5 = 65 -> 128
    assert dll.gdrn_head_glue_fwd_ex2(None, None, None, None, None, 1, 4096, 1, 1, 8, 1, 128, None) == -1
    assert b"pnp_ld" in dll.gdrn_last_error()
    assert dll.gdrn_head_bwd_ex2(None, None, None, None, None, None, None, None, None, None, None, None, None, 1, 4096, 1, 0, 1,
                                 60, 1, 64, None) == -1
    assert b"pnp_ld" in dll.gdrn_last_error()
    assert dll.gdrn_pnp_pack_input_ex(None, 5, None, 8, None, None, None, 1, 4096, 128, None) == -1
    assert b"pnp_ld" in dll.gdrn_last_error()


def test_region_kernels_use_no_stack_or_local_memory():
    obj = os.path.join(ROOT, "gdr_net_b200", "_build", "losses.o")
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(obj) or not os.path.exists(tool):
        pytest.skip("needs the built objects and cuobjdump")
    out = subprocess.run([tool, "-res-usage", obj], capture_output=True, text=True, check=True).stdout
    found = 0
    name = None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        if name and re.search(r"(head_glue_fwd2|pixel_loss_fwd2|head_bwd2|pnp_pack_input2)_kernel", name):
            stack = int(re.search(r"STACK:(\d+)", line).group(1))
            local = int(re.search(r"LOCAL:(\d+)", line).group(1))
            assert stack == 0 and local == 0, (name, line)
            found += 1
        name = None
    # 8 glue (MO x W2D x ATT), 6 pixel loss (mask head x SEP), 24 backward (mask head x SEP x W2D x ATT), 1 pack
    assert found == 39, found
