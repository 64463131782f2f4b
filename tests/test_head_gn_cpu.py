"""CPU: the GroupNorm geometry head (ROT_HEAD.NORM = "GN", NUM_GN_GROUPS).

  * the oracle restatement (oracle/head_gn_oracle.py) against the unmodified reference built with a GN head
    (tests/golden/train_head_gn_b4.npz, oracle/make_golden_head_gn.py): eval maps and pose, losses and every parameter gradient;
  * `build_model_optimizer` gives the reference's state_dict keys and shapes (no head BatchNorm buffers), its parameter order and
    optimizer groups; other norms and group counts are refused naming the key;
  * the gdrn_head_gn_* entry points are declared and exported, report argument errors without a GPU, and their kernels keep
    everything in registers."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import gdrn_oracle as O
from oracle import head_gn_oracle as HG
from oracle.make_golden_head_gn import CASES, EVAL_STRIDE, grad_sample_index, make_batch, read_json


def case_config(case, device="cpu", **kw):
    from gdr_net_b200.config import a6_config

    rh, pn, *_ = CASES[case]
    cfg = a6_config(device=device, **kw)
    for k, v in rh.items():
        setattr(cfg.MODEL.CDPN.ROT_HEAD, k, v)
    for k, v in pn.items():
        setattr(cfg.MODEL.CDPN.PNP_NET, k, v)
    return cfg


def oracle_kwargs(case):
    rh, pn, *_ = CASES[case]
    return dict(G=rh["NUM_GN_GROUPS"], num_regions=rh["NUM_REGIONS"], mask_loss_type=rh.get("MASK_LOSS_TYPE", "L1"),
                region_att=pn["REGION_ATTENTION"], num_classes=rh.get("NUM_CLASSES", 1) if rh.get("ROT_CLASS_AWARE") else 1,
                rot_aware=rh.get("ROT_CLASS_AWARE", False))


def seeded_weights(case):
    from gdr_net_b200 import GDRN as G
    from gdr_net_b200 import synth

    model, _ = G.build_model_optimizer(case_config(case))
    return synth.seeded_state_dict(model.state_dict(), seed=CASES[case][3])


def golden(golden_dir, case):
    g = np.load(os.path.join(golden_dir, "train_head_gn_b4.npz"))
    return {k[len(case) + 1:]: g[k] for k in g.files if k.startswith(case + "/")}


# ------------------------------------------------------------------------------------------------ oracle vs reference goldens
@pytest.mark.parametrize("case", list(CASES))
def test_oracle_matches_reference_golden(golden_dir, case):
    g = golden(golden_dir, case)
    sd = seeded_weights(case)
    batch = make_batch(case)
    kw = oracle_kwargs(case)
    with torch.no_grad():
        o = HG.gdrn_forward(O.leaf_state_dict(sd, requires_grad=False), batch, train=False, do_loss=False, **kw)
    assert np.abs(o["head"][:, :, ::EVAL_STRIDE, ::EVAL_STRIDE].numpy() - g["eval/head"]).max() <= 1e-5
    assert np.abs(o["trans"].numpy() - g["eval/trans"]).max() <= 1e-5
    assert np.abs(o["rot"].numpy() - g["eval/rot"]).max() <= 1e-5
    leaf = O.leaf_state_dict(sd)
    o = HG.gdrn_forward(leaf, batch, train=True, do_loss=True, update_stats=True, **kw)
    assert list(o["losses"]) == [k[len("loss/"):] for k in g if k.startswith("loss/")]
    for k, v in o["losses"].items():
        ref = float(g["loss/" + k])
        assert abs(float(v.detach()) - ref) <= 5e-6 * abs(ref), (k, float(v.detach()), ref)
    sum(o["losses"].values()).backward()
    names = [k[len("grad/"):] for k in g if k.startswith("grad/")]
    assert names == [n for n in sd if not n.endswith(("running_mean", "running_var", "num_batches_tracked"))]
    for name in names:
        ref = g["grad/" + name]
        mine = leaf[name].grad.reshape(-1).numpy()[grad_sample_index(leaf[name].numel())]
        err = np.abs(mine - ref).max() / max(np.abs(ref).max(), 1e-30)
        assert err <= 5e-6, (name, err)


# ------------------------------------------------------------------------------------------------ configuration surface
@pytest.mark.parametrize("case", list(CASES))
def test_build_surface_matches_the_reference(golden_dir, case):
    from gdr_net_b200 import GDRN as G

    g = golden(golden_dir, case)
    model, optimizer = G.build_model_optimizer(case_config(case))
    sd = model.state_dict()
    assert list(sd) == read_json(g["sd_keys"])
    assert [list(v.shape) for v in sd.values()] == read_json(g["sd_shapes"])
    assert not [k for k in sd if k.startswith("rot_head_net.") and k.endswith(("running_mean", "running_var", "num_batches_tracked"))]
    gn = [i for i, m in enumerate(model.rot_head_net.features) if isinstance(m, torch.nn.GroupNorm)]
    assert gn == list(HG.NORM_AT)
    G_ = CASES[case][0]["NUM_GN_GROUPS"]
    for i in gn:
        m = model.rot_head_net.features[i]
        assert m.num_groups == G_ and m.num_channels == 256 and m.eps == 1e-5
        assert torch.equal(m.weight, torch.ones(256)) and torch.equal(m.bias, torch.zeros(256))
    names = {id(p): n for n, p in model.named_parameters()}
    groups = [dict(params=[names[id(p)] for p in grp["params"]], lr=grp["lr"]) for grp in optimizer.param_groups]
    assert groups == read_json(g["opt_groups"])
    assert model.load_state_dict(seeded_weights(case), strict=True) is not None


@pytest.mark.parametrize("key,value", [("NORM", "SyncBN"), ("NORM", "FrozenBN"), ("NORM", ""), ("NUM_GN_GROUPS", 3),
                                       ("NUM_GN_GROUPS", 128), ("NUM_GN_GROUPS", 256)])
def test_unsupported_head_norm_rejected(key, value):
    from gdr_net_b200 import GDRN as G
    from gdr_net_b200.config import a6_config

    cfg = a6_config(device="cpu")
    cfg.MODEL.CDPN.ROT_HEAD.NORM = "GN"
    setattr(cfg.MODEL.CDPN.ROT_HEAD, key, value)
    with pytest.raises(NotImplementedError) as e:
        G.build_model_optimizer(cfg)
    assert f"ROT_HEAD.{key}" in str(e.value)
    with pytest.raises(NotImplementedError) as e:
        G.RotWithRegionHead(norm=cfg.MODEL.CDPN.ROT_HEAD.NORM, num_gn_groups=cfg.MODEL.CDPN.ROT_HEAD.NUM_GN_GROUPS)
    assert f"ROT_HEAD.{key}" in str(e.value)


@pytest.mark.parametrize("groups", [1, 2, 4, 8, 16, 32, 64])
def test_every_supported_group_count_builds(groups):
    from gdr_net_b200 import GDRN as G

    head = G.RotWithRegionHead(norm="GN", num_gn_groups=groups)
    assert all(head.features[i].num_groups == groups for i in HG.NORM_AT)
    assert not any(isinstance(m, torch.nn.BatchNorm2d) for m in head.modules())


# ------------------------------------------------------------------------------------------------ C ABI
NEW = {"gdrn_head_gn_workspace": 2, "gdrn_head_gn_fwd": 15, "gdrn_head_gn_bwd": 17}


def test_head_gn_entry_points_declared_and_exported():
    from gdr_net_b200 import capi

    protos = capi.parse_header()
    for name, nargs in NEW.items():
        assert name in protos and len(protos[name][1]) == nargs, (name, protos.get(name))
    if not os.path.exists(capi.LIB_PATH):
        pytest.skip("library not built")
    dll = ctypes.CDLL(capi.LIB_PATH)
    for name in NEW:
        assert hasattr(dll, name), name


def test_head_gn_argument_errors_without_a_gpu():
    from gdr_net_b200 import capi

    if not os.path.exists(capi.LIB_PATH):
        pytest.skip("library not built")
    dll = capi.C.load()
    p = ctypes.c_void_p(16)  # never dereferenced: every call below fails its argument checks first
    assert dll.gdrn_head_gn_workspace(4, 4096) > 0 and dll.gdrn_head_gn_workspace(4, 2048) == -1
    assert dll.gdrn_head_gn_workspace(0, 256) == -1

    def fwd(B=4, HW=4096, C=256, G=32, ws=p):
        return dll.gdrn_head_gn_fwd(p, None, p, None, None, p, p, p, ws, B, HW, C, G, 1e-5, None)

    def bwd(B=4, HW=4096, C=256, G=32, mask=p):
        return dll.gdrn_head_gn_bwd(p, None, p, None, mask, p, p, p, None, p, p, p, B, HW, C, G, None)

    for call, kw, word in ((fwd, dict(C=128), b"C = 128"), (fwd, dict(G=3), b"G = 3"), (fwd, dict(G=128), b"G = 128"),
                           (fwd, dict(G=0), b"G = 0"), (fwd, dict(HW=2048), b"HW = 2048"), (fwd, dict(B=0), b"B = 0"),
                           (fwd, dict(ws=None), b"workspace"), (bwd, dict(G=256), b"G = 256"), (bwd, dict(HW=64), b"HW = 64"),
                           (bwd, dict(mask=None), b"mask")):
        assert call(**kw) == -1, kw
        assert word in dll.gdrn_last_error(), (kw, dll.gdrn_last_error())


def test_head_gn_kernels_use_no_stack_or_local_memory():
    from gdr_net_b200 import build, capi

    tool = shutil.which("cuobjdump") or os.path.join(os.path.dirname(build.NVCC), "cuobjdump")
    if not os.path.exists(capi.LIB_PATH) or not os.path.exists(tool):
        pytest.skip("needs the built library and cuobjdump")
    out = subprocess.run([tool, "-res-usage", capi.LIB_PATH], capture_output=True, text=True, check=True).stdout
    usage = dict(re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", out))
    mine = {n: r for n, r in usage.items() if "gn_head_" in n}
    assert len(mine) == 7, sorted(mine)
    for name, res in mine.items():
        assert "STACK:0 " in res and "LOCAL:0 " in res, (name, res)
