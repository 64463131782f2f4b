"""CPU: DropBlock on the Patch-PnP input (PNP_NET.PNP_HEAD_CFG.drop_prob / dropblock_size).

  * the oracle (oracle/dropblock_oracle.py), fed the seed masks the unmodified reference drew, reproduces its losses and
    gradients (tests/golden/train_dropblock_b4.npz, oracle/make_golden_dropblock.py), and its eval forward equals the model
    without DropBlock;
  * the device's schedule formula (csrc/dropblock.cu dropblock_prob) is np.linspace(0, p, 5000) bit for bit;
  * `build_model_optimizer` accepts drop_prob in [0, 1] and dropblock_size 1..15 with an unchanged state_dict and rejects
    other values, naming the key;
  * the DropBlock entry points are declared and exported, report argument errors without a GPU, and the new kernels keep
    everything in registers (no stack frame, no local memory)."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from gdr_net_b200 import synth
from oracle import dropblock_oracle as DB
from oracle import gdrn_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# as oracle/make_golden_dropblock.py: name -> (ROT_HEAD switches, PNP_NET switches, drop_prob, dropblock_size, step, weight seed,
# batch seed)
CASES = {
    "ship_b5": (dict(NUM_REGIONS=64), dict(REGION_ATTENTION=True, WITH_2D_COORD=True), 0.25, 5, 4999, 51, 61),
    "r8_b3": (dict(NUM_REGIONS=8), dict(REGION_ATTENTION=True, WITH_2D_COORD=True), 0.5, 3, 2500, 52, 62),
    "r32_noatt_b4": (dict(NUM_REGIONS=32), dict(REGION_ATTENTION=False, WITH_2D_COORD=True), 0.25, 4, 4200, 53, 63),
}
EVAL = ("ship_b5", 54, 64)


def db_config(case, device="cpu", drop_prob=None, block_size=None):
    from gdr_net_b200.config import a6_config

    rh, pn, p, k, *_ = CASES[case]
    k = k if block_size is None else block_size
    cfg = a6_config(device=device)
    for key, v in rh.items():
        setattr(cfg.MODEL.CDPN.ROT_HEAD, key, v)
    for key, v in pn.items():
        setattr(cfg.MODEL.CDPN.PNP_NET, key, v)
    cfg.MODEL.CDPN.PNP_NET.PNP_HEAD_CFG.update(drop_prob=p if drop_prob is None else drop_prob, dropblock_size=k)
    return cfg


def oracle_kwargs(case):
    return dict(region_att=CASES[case][1]["REGION_ATTENTION"], with_2d=CASES[case][1]["WITH_2D_COORD"], block_size=CASES[case][3])


def seeded_weights(case, wseed=None):
    from gdr_net_b200 import GDRN as G

    model, _ = G.build_model_optimizer(db_config(case))
    return synth.seeded_state_dict(model.state_dict(), seed=CASES[case][5] if wseed is None else wseed)


def golden(golden_dir, case):
    g = np.load(os.path.join(golden_dir, "train_dropblock_b4.npz"))
    return {k[len(case) + 1:]: g[k] for k in g.files if k.startswith(case + "/")}


def device_prob(p: float, k: int) -> float:
    """dropblock_prob of csrc/dropblock.cu, restated in float64."""
    if k >= 4999:
        return p
    step = np.float64(p) / np.float64(4999)
    return float((np.float64(k) / np.float64(4999)) * np.float64(p) if step == 0 else np.float64(k) * step)


# ------------------------------------------------------------------------------------------------ oracle vs reference goldens
@pytest.mark.parametrize("case", list(CASES))
def test_oracle_matches_reference_golden(golden_dir, case):
    g = golden(golden_dir, case)
    rh, _pn, p, k, step, _ws, bseed = CASES[case]
    assert int(g["step"]) == step
    seeds = torch.from_numpy(g["seeds"])
    assert 0 < int(seeds.sum()) < seeds.numel()
    leaf = O.leaf_state_dict(seeded_weights(case))
    batch = synth.make_batch(4, seed=bseed, num_regions=rh["NUM_REGIONS"])
    o = DB.gdrn_forward(leaf, batch, train=True, do_loss=True, seeds=seeds, update_stats=True, **oracle_kwargs(case))
    assert list(o["losses"]) == [key[len("loss/"):] for key in g if key.startswith("loss/")]
    for name, v in o["losses"].items():
        assert float(v.detach()) == float(g["loss/" + name]), (name, float(v.detach()), float(g["loss/" + name]))
    sum(o["losses"].values()).backward()
    for key in g:
        if key.startswith("grad/"):
            name = key[len("grad/"):]
            err = np.abs(leaf[name].grad.numpy() - g[key]).max() / np.abs(g[key]).max()
            print(case, name, f"{err:.2e}")
            assert err <= 5e-6, (name, err)
    # without the mask the losses move: the golden pins DropBlock, not a no-op
    with torch.no_grad():
        o0 = DB.gdrn_forward(O.leaf_state_dict(seeded_weights(case), requires_grad=False), batch, train=True, do_loss=True,
                             **oracle_kwargs(case))
    assert float(o0["losses"]["loss_PM_R"]) != float(g["loss/loss_PM_R"])


def test_oracle_eval_is_the_model_without_dropblock(golden_dir):
    g = np.load(os.path.join(golden_dir, "train_dropblock_b4.npz"))
    assert np.array_equal(g["eval/rot"], g["eval/rot_nodb"]) and np.array_equal(g["eval/trans"], g["eval/trans_nodb"])
    case, wseed, bseed = EVAL
    with torch.no_grad():
        o = DB.gdrn_forward(O.leaf_state_dict(seeded_weights(case, wseed), requires_grad=False), synth.make_batch(4, seed=bseed),
                            train=False, do_loss=False, seeds=torch.ones(4, 64, 64), **oracle_kwargs(case))
    assert np.array_equal(o["trans"].numpy(), g["eval/trans"])
    assert np.abs(o["rot"].numpy() - g["eval/rot"]).max() <= 1e-12


def test_block_mask_even_and_odd_sizes():
    seeds = torch.zeros(1, 64, 64)
    seeds[0, 10, 20] = 1
    seeds[0, 0, 63] = 1
    for k in (1, 2, 3, 4, 5, 15):
        bm = DB.block_mask(seeds, k)
        lo = k // 2
        want = torch.ones(1, 64, 64)
        for y, x in ((10, 20), (0, 63)):  # output (i, j) covers seeds (i - k // 2 .. i - k // 2 + k - 1)
            want[0, max(y - (k - 1 - lo), 0):y + lo + 1, max(x - (k - 1 - lo), 0):x + lo + 1] = 0
        assert torch.equal(bm, want), k


@pytest.mark.parametrize("p", [0.0, 0.25, 0.1, 0.3, 0.5, 1.0, 1e-300, 0.7777])
def test_device_schedule_is_numpy_linspace(p):
    ref = np.linspace(0, p, 5000)
    got = np.array([device_prob(p, k) for k in range(5000)])
    assert np.array_equal(got.view(np.uint64), ref.view(np.uint64)), p
    assert device_prob(p, 5000) == device_prob(p, 123456) == ref[-1]
    assert DB.prob_at(p, 0) == 0.0 and DB.prob_at(p, 10**6) == ref[-1]


# ------------------------------------------------------------------------------------------------ configuration surface
@pytest.mark.parametrize("p, k", [(0.25, 5), (1.0, 1), (0.5, 15), (0.1, 4)])
def test_build_accepts_dropblock_with_unchanged_state_dict(p, k):
    from gdr_net_b200 import GDRN as G

    model, _ = G.build_model_optimizer(db_config("ship_b5", drop_prob=p, block_size=k))
    ref, _ = G.build_model_optimizer(db_config("ship_b5", drop_prob=0.0))
    assert (model.pnp_net.drop_prob, model.pnp_net.dropblock_size, model.pnp_net.dropblock_step) == (p, k, 0)
    sd, sd0 = model.state_dict(), ref.state_dict()
    assert list(sd) == list(sd0) and all(sd[n].shape == sd0[n].shape for n in sd)
    assert [n for n, _ in model.named_buffers()] == [n for n, _ in ref.named_buffers()]
    assert isinstance(model.pnp_net.dropblock_seed, int)


@pytest.mark.parametrize("key, value", [("drop_prob", -0.1), ("drop_prob", 1.5), ("drop_prob", float("nan")),
                                        ("dropblock_size", 0), ("dropblock_size", 16), ("dropblock_size", 2.5)])
def test_out_of_range_dropblock_rejected(key, value):
    from gdr_net_b200 import GDRN as G

    cfg = db_config("ship_b5")
    cfg.MODEL.CDPN.PNP_NET.PNP_HEAD_CFG[key] = value
    with pytest.raises(NotImplementedError) as e:
        G.build_model_optimizer(cfg)
    assert f"PNP_HEAD_CFG.{key}" in str(e.value)


# ------------------------------------------------------------------------------------------------ C ABI
NEW = {"gdrn_dropblock_step": 14, "gdrn_head_glue_fwd_db": 15, "gdrn_head_bwd_db": 24, "gdrn_pnp_pack_input_db": 13}


def test_dropblock_entry_points_declared_and_exported():
    from gdr_net_b200 import capi

    protos = capi.parse_header()
    for name, nargs in NEW.items():
        assert name in protos and len(protos[name][1]) == nargs, (name, protos.get(name))
    if not os.path.exists(capi.LIB_PATH):
        pytest.skip("library not built")
    dll = ctypes.CDLL(capi.LIB_PATH)
    for name in NEW:
        assert hasattr(dll, name), name


def test_dropblock_argument_errors_without_a_gpu():
    from gdr_net_b200 import capi

    if not os.path.exists(capi.LIB_PATH):
        pytest.skip("library not built")
    dll = capi.C.load()
    fake = 16  # never dereferenced: the checks come first
    for p, k, H, W, what in ((-0.5, 5, 64, 64, b"drop_prob"), (1.01, 5, 64, 64, b"drop_prob"), (float("nan"), 5, 64, 64, b"drop_prob"),
                             (0.25, 0, 64, 64, b"block_size"), (0.25, 16, 64, 64, b"block_size"), (0.25, 5, 64, 65, b"width"),
                             (0.25, 5, 64, 0, b"width"), (0.25, 5, 0, 64, b"width")):
        assert dll.gdrn_dropblock_step(fake, 1, 0, p, k, 1, fake, fake, fake, fake, 4, H, W, None) == -1, (p, k, H, W)
        assert what in dll.gdrn_last_error(), dll.gdrn_last_error()
    assert dll.gdrn_dropblock_step(None, 1, 0, 0.25, 5, 0, None, None, None, None, 0, 64, 64, None) == -1
    assert dll.gdrn_dropblock_step(fake, 1, 0, 0.25, 5, 1, None, fake, fake, fake, 4, 64, 64, None) == -1
    assert b"keep" in dll.gdrn_last_error()
    # the _db kernels: region checks as the _ex2 ones, and keep / scale are required
    assert dll.gdrn_head_glue_fwd_db(None, None, None, None, None, 1, 4096, 1, 1, 8, 1, 128, fake, fake, None) == -1
    assert b"pnp_ld" in dll.gdrn_last_error()
    assert dll.gdrn_head_glue_fwd_db(None, fake, None, None, None, 1, 4096, 1, 1, 8, 1, 64, None, fake, None) == -1
    assert b"keep" in dll.gdrn_last_error()
    assert dll.gdrn_head_bwd_db(None, None, None, None, None, None, None, None, None, None, None, None, None, 1, 4096, 1, 0, 1,
                                64, 1, 128, fake, None, None) == -1
    assert b"scale" in dll.gdrn_last_error()
    assert dll.gdrn_pnp_pack_input_db(None, 5, None, 8, None, None, None, 1, 4096, 128, fake, fake, None) == -1
    assert b"pnp_ld" in dll.gdrn_last_error()


def test_dropblock_kernels_use_no_stack_or_local_memory():
    obj = os.path.join(ROOT, "gdr_net_b200", "_build", "dropblock.o")
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(obj) or not os.path.exists(tool):
        pytest.skip("needs the built objects and cuobjdump")
    out = subprocess.run([tool, "-res-usage", obj], capture_output=True, text=True, check=True).stdout
    found = {}
    name = None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        if name:
            kind = re.search(r"(head_glue_fwd2|head_bwd2|pnp_pack_input2|dropblock_sample|dropblock_finish)_kernel", name)
            assert kind, name
            stack = int(re.search(r"STACK:(\d+)", line).group(1))
            local = int(re.search(r"LOCAL:(\d+)", line).group(1))
            assert stack == 0 and local == 0, (name, line)
            found[kind.group(1)] = found.get(kind.group(1), 0) + 1
        name = None
    # 8 glue (MO x W2D x ATT), 24 backward (mask head x SEP x W2D x ATT), 1 pack, the sampler and its finish
    assert found == {"head_glue_fwd2": 8, "head_bwd2": 24, "pnp_pack_input2": 1, "dropblock_sample": 1, "dropblock_finish": 1}, found
