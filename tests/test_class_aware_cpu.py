"""CPU: class-aware geometry heads (ROT_HEAD.ROT_CLASS_AWARE / MASK_CLASS_AWARE / REGION_CLASS_AWARE).

  * the oracle restatement (oracle/class_aware_oracle.py) against the unmodified reference built with those switches
    (tests/golden/train_class_aware_b4.npz, oracle/make_golden_class_aware.py), including the exact-zero gradient rows of the
    classes no crop uses;
  * the engine's per-class row table (engine.class_rows) selects the same rows as the oracle;
  * `build_model_optimizer` accepts every flag combination with the reference's output-conv shape, a reference-shaped state dict
    loads strictly, roi_classes is required and range-checked, ROT_CONCAT stays rejected;
  * the grouped-GEMM and class-gradient entry points are declared and exported, report argument errors without a GPU, and their
    kernels keep everything in registers."""
import ctypes
import itertools
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from gdr_net_b200 import synth
from oracle import class_aware_oracle as CA
from oracle import gdrn_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# as oracle/make_golden_class_aware.py: name -> (ROT_HEAD switches, crop classes, weight seed, batch seed)
CASES = {
    "all13": (dict(NUM_CLASSES=13, ROT_CLASS_AWARE=True, MASK_CLASS_AWARE=True, REGION_CLASS_AWARE=True, NUM_REGIONS=64),
              [3, 0, 3, 12], 51, 61),
    "rot13": (dict(NUM_CLASSES=13, ROT_CLASS_AWARE=True, NUM_REGIONS=64), [3, 0, 3, 12], 52, 62),
    "mr_ce21": (dict(NUM_CLASSES=21, MASK_CLASS_AWARE=True, REGION_CLASS_AWARE=True, MASK_LOSS_TYPE="CE", NUM_REGIONS=8),
                [5, 0, 5, 20], 53, 63),
}
ROWS = {"all13": 897, "rot13": 105, "mr_ce21": 234}
FLAGS = ("ROT_CLASS_AWARE", "MASK_CLASS_AWARE", "REGION_CLASS_AWARE")


def case_config(case, device="cpu", **kw):
    from gdr_net_b200.config import a6_config

    cfg = a6_config(device=device, **kw)
    for k, v in CASES[case][0].items():
        setattr(cfg.MODEL.CDPN.ROT_HEAD, k, v)
    return cfg


def oracle_kwargs(case):
    rh = CASES[case][0]
    return dict(num_classes=rh["NUM_CLASSES"], rot_aware=rh.get("ROT_CLASS_AWARE", False), mask_aware=rh.get("MASK_CLASS_AWARE", False),
                region_aware=rh.get("REGION_CLASS_AWARE", False), num_regions=rh["NUM_REGIONS"],
                mask_loss_type=rh.get("MASK_LOSS_TYPE", "L1"))


def make_batch(case, B=4, seed=None):
    rh, classes, _w, bseed = CASES[case]
    batch = synth.make_batch(B, seed=bseed if seed is None else seed, num_regions=rh["NUM_REGIONS"])
    if B == len(classes):
        batch["roi_cls"] = torch.tensor(classes, dtype=torch.long)
    return batch


def seeded_weights(case):
    from gdr_net_b200 import GDRN as G

    model, _ = G.build_model_optimizer(case_config(case))
    return synth.seeded_state_dict(model.state_dict(), seed=CASES[case][2])


def golden(golden_dir, case):
    g = np.load(os.path.join(golden_dir, "train_class_aware_b4.npz"))
    return {k[len(case) + 1:]: g[k] for k in g.files if k.startswith(case + "/")}


def absent_rows(case):
    """Output-conv rows that no crop of the golden batch uses (their gradient is exactly 0)."""
    from gdr_net_b200.engine import class_rows

    kw = oracle_kwargs(case)
    mo = 2 if kw["mask_loss_type"] == "CE" else 1
    rows, n = class_rows(kw["num_classes"], mo, kw["num_regions"], kw["rot_aware"], kw["mask_aware"], kw["region_aware"])
    used = {r for c in CASES[case][1] for r in rows[c]}
    return sorted(set(range(n)) - used), n


# ------------------------------------------------------------------------------------------------ oracle vs reference goldens
@pytest.mark.parametrize("case", list(CASES))
def test_oracle_matches_reference_golden(golden_dir, case):
    g = golden(golden_dir, case)
    sd = seeded_weights(case)
    batch = make_batch(case)
    kw = oracle_kwargs(case)
    with torch.no_grad():
        o = CA.gdrn_forward(O.leaf_state_dict(sd, requires_grad=False), batch, train=False, do_loss=False, **kw)
    assert np.abs(o["head"][:, :, ::4, ::4].numpy() - g["eval/head"]).max() <= 1e-6
    assert np.abs(o["trans"].numpy() - g["eval/trans"]).max() <= 1e-6
    assert np.abs(o["rot"].numpy() - g["eval/rot"]).max() <= 1e-6
    leaf = O.leaf_state_dict(sd)
    o = CA.gdrn_forward(leaf, batch, train=True, do_loss=True, update_stats=True, **kw)
    assert list(o["losses"]) == [k[len("loss/"):] for k in g if k.startswith("loss/")]
    for k, v in o["losses"].items():
        ref = float(g["loss/" + k])
        assert abs(float(v.detach()) - ref) <= 1e-6 * abs(ref), (k, float(v.detach()), ref)
    sum(o["losses"].values()).backward()
    absent, n_rows = absent_rows(case)
    assert g["grad/rot_head_net.features.23.weight"].shape == (n_rows, 256, 1, 1) and n_rows == ROWS[case]
    for key in g:
        if key.startswith("grad/"):
            name = key[len("grad/"):]
            ref = g[key]
            err = np.abs(leaf[name].grad.numpy() - ref).max() / np.abs(ref).max()
            print(case, name, f"{err:.2e}")
            assert err <= 5e-6, (name, err)
            if name.startswith("rot_head_net.features.23."):
                # the rows of classes no crop uses: exactly zero in the reference and in the oracle
                assert absent and not ref[absent].any() and not leaf[name].grad.numpy()[absent].any(), name


@pytest.mark.parametrize("case", list(CASES))
def test_class_rows_select_what_the_oracle_selects(case):
    from gdr_net_b200.engine import class_rows

    kw = oracle_kwargs(case)
    mo = 2 if kw["mask_loss_type"] == "CE" else 1
    C_, R = kw["num_classes"], kw["num_regions"]
    rows, n = class_rows(C_, mo, R, kw["rot_aware"], kw["mask_aware"], kw["region_aware"])
    assert n == ROWS[case]
    full = torch.arange(n, dtype=torch.float64).view(1, n, 1, 1).expand(C_, n, 1, 1)
    sel = CA.select_class_maps(full, torch.arange(C_), C_, mo, R, kw["rot_aware"], kw["mask_aware"], kw["region_aware"])
    assert sel[:, :, 0, 0].long().tolist() == rows


# ------------------------------------------------------------------------------------------------ configuration surface
@pytest.mark.parametrize("flags", list(itertools.product((False, True), repeat=3)))
@pytest.mark.parametrize("num_classes", [1, 13])
def test_build_model_accepts_every_flag_combination(flags, num_classes):
    from gdr_net_b200 import GDRN as G
    from gdr_net_b200.config import a6_config

    cfg = a6_config(device="cpu")
    cfg.MODEL.CDPN.ROT_HEAD.NUM_CLASSES = num_classes
    for k, v in zip(FLAGS, flags):
        setattr(cfg.MODEL.CDPN.ROT_HEAD, k, v)
    model, _ = G.build_model_optimizer(cfg)
    rot, mask, region = ((num_classes if f else 1) for f in flags)
    rows = mask + 3 * rot + 65 * region
    assert tuple(model.rot_head_net.features[23].weight.shape) == (rows, 256, 1, 1)
    assert tuple(model.rot_head_net.features[23].bias.shape) == (rows,)


@pytest.mark.parametrize("case", list(CASES))
def test_reference_shaped_state_dict_loads_strictly(golden_dir, case):
    from gdr_net_b200 import GDRN as G

    model, _ = G.build_model_optimizer(case_config(case))
    g = golden(golden_dir, case)
    params = dict(model.named_parameters())
    for key in g:
        if key.startswith("grad/"):
            assert tuple(params[key[len("grad/"):]].shape) == g[key].shape, key
    missing, unexpected = model.load_state_dict(seeded_weights(case), strict=True)
    assert not missing and not unexpected


def test_roi_classes_are_required_and_range_checked():
    from gdr_net_b200 import GDRN as G

    model, _ = G.build_model_optimizer(case_config("all13"))
    batch = make_batch("all13")
    kw = synth.forward_kwargs(batch, train=False)
    for bad in (None, torch.tensor([0, 1, 2, 13]), torch.tensor([-1, 0, 0, 0]), torch.tensor([0.0, 1.0, 2.0, 3.0]),
                torch.tensor([0, 1, 2])):
        with pytest.raises(ValueError) as e:
            model(batch["roi_img"], **dict(kw, roi_classes=bad))
        assert "roi_classes" in str(e.value)
    # valid classes of any integer dtype pass the check (and then meet the CUDA-only engine)
    for ok in (torch.tensor([0, 12, 3, 3], dtype=torch.int32), torch.tensor([0, 12, 3, 3], dtype=torch.uint8), [0, 1, 2, 3]):
        with pytest.raises(RuntimeError) as e:
            model(batch["roi_img"], **dict(kw, roi_classes=ok))
        assert "CUDA" in str(e.value)


def test_rot_concat_still_rejected():
    from gdr_net_b200 import GDRN as G

    cfg = case_config("all13")
    cfg.MODEL.CDPN.ROT_HEAD.ROT_CONCAT = True
    with pytest.raises(NotImplementedError) as e:
        G.build_model_optimizer(cfg)
    assert "ROT_CONCAT" in str(e.value)


# ------------------------------------------------------------------------------------------------ C ABI
NEW = {"gdrn_conv_fwd_grouped": 26, "gdrn_gemm_fwd_grouped": 20, "gdrn_class_gather": 7, "gdrn_crop_colsum": 7,
       "gdrn_class_wgrad_reduce": 15}


def test_class_entry_points_declared_and_exported():
    from gdr_net_b200 import capi

    protos = capi.parse_header()
    for name, nargs in NEW.items():
        assert name in protos and len(protos[name][1]) == nargs, (name, protos.get(name))
    if not os.path.exists(capi.LIB_PATH):
        pytest.skip("library not built")
    dll = ctypes.CDLL(capi.LIB_PATH)
    for name in NEW:
        assert hasattr(dll, name), name


def test_class_argument_errors_without_a_gpu():
    from gdr_net_b200 import capi

    if not os.path.exists(capi.LIB_PATH):
        pytest.skip("library not built")
    dll = capi.C.load()
    grp = ctypes.c_void_p(16)  # never dereferenced: every call below fails its argument checks first

    def conv(group, rpg, G, N=2):
        return dll.gdrn_conv_fwd_grouped(None, None, None, None, None, None, None, None, N, 64, 64, 256, 69, 128, 1, 1, 1, 0, 72, 0,
                                         1, group, rpg, G, 128, None)

    for args, word in (((None, 4096, 13), b"group"), ((grp, 4000, 13), b"rows_per_group"), ((grp, 4096, 0), b"num_groups"),
                       ((grp, 3 * 4096, 13), b"groups of")):
        assert conv(*args) == -1, args
        assert word in dll.gdrn_last_error(), (args, dll.gdrn_last_error())
    assert dll.gdrn_gemm_fwd_grouped(None, None, None, None, None, None, None, None, 4096 * 2 + 128, 256, 256, 128, 256, 0, 1, grp,
                                     4096, 13, 0, None) == -1
    assert b"groups of" in dll.gdrn_last_error()
    assert dll.gdrn_gemm_fwd_grouped(None, None, None, None, None, None, None, None, 8192, 256, 256, 128, 256, 0, 1, grp, 64, 13, 0,
                                     None) == -1
    assert b"rows_per_group" in dll.gdrn_last_error()
    assert dll.gdrn_class_gather(None, None, None, 0, 256, 897, None) == -1
    assert dll.gdrn_crop_colsum(None, None, None, 4, 4096, 100, None) == -1 and b"ld" in dll.gdrn_last_error()
    assert dll.gdrn_crop_colsum(None, None, None, 0, 4096, 128, None) == -1
    # slots beyond the bias partial rows / a crop stride shorter than the slots
    assert dll.gdrn_class_wgrad_reduce(None, 128 * 256, 256, None, 128, None, 4, None, 13, 897, 129, 256, None, None, None) == -1
    assert dll.gdrn_class_wgrad_reduce(None, 64 * 256, 256, None, 128, None, 4, None, 13, 897, 69, 256, None, None, None) == -1
    assert b"partials" in dll.gdrn_last_error()
    assert dll.gdrn_class_wgrad_reduce(None, 128 * 256, 256, None, 128, None, 4, None, 0, 897, 69, 256, None, None, None) == -1


def test_class_kernels_use_no_stack_or_local_memory():
    from gdr_net_b200 import build, capi

    tool = shutil.which("cuobjdump") or os.path.join(os.path.dirname(build.NVCC), "cuobjdump")
    if not os.path.exists(capi.LIB_PATH) or not os.path.exists(tool):
        pytest.skip("needs the built library and cuobjdump")
    out = subprocess.run([tool, "-res-usage", capi.LIB_PATH], capture_output=True, text=True, check=True).stdout
    usage = dict(re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", out))
    mine = {n: r for n, r in usage.items() if re.search(r"gemm_fwd_grouped_kernel|class_gather|crop_colsum|class_wgrad_reduce", n)}
    assert sum("gemm_fwd_grouped_kernel" in n for n in mine) == 4, sorted(mine)  # BLOCK_N 64 / 128 x 1 / 3 passes
    assert len(mine) == 7, sorted(mine)
    for name, res in mine.items():
        assert "STACK:0 " in res and "LOCAL:0 " in res, (name, res)
