"""TEST INFRASTRUCTURE ONLY -- golden vectors for the GroupNorm geometry head (ROT_HEAD.NORM = "GN", NUM_GN_GROUPS), produced by
the UNMODIFIED reference model (GDRN.py, cdpn_rot_head_region.py, core/utils/layer_utils.get_norm) built from the a6 config with
only these switches changed (the GPU box has no reference install):

  ship_g32      the shipped head (64 regions, attention, 2-D coordinates), G = 32
  r8_noatt_g1   8 regions without region attention, G = 1 (one group of 256 channels)
  bce_rot_g64   BCE mask, class-aware xyz (13 classes), G = 64

Each case: a seeded batch of four crops, the eval-mode TEST.USE_PNP maps (every EVAL_STRIDE-th pixel of every EVAL_STRIDE-th
row) and pose, the train-mode losses and every parameter gradient after `sum(loss_dict.values()).backward()`, the state_dict
manifest and the optimizer groups.  A gradient of at most GRAD_WHOLE elements is stored whole, a larger one as the GRAD_SAMPLES
elements at grad_sample_index(numel) of its flattened view.
Output: tests/golden/train_head_gn_b4.npz, keys "<case>/loss/<name>", "<case>/grad/<param>", "<case>/eval/{head,rot,trans}",
"<case>/sd_keys", "<case>/sd_shapes", "<case>/opt_groups" (UTF-8 JSON bytes; the groups as parameter names and lr).
Usage: python -m oracle.make_golden_head_gn"""
import copy
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gdr_net_b200 import synth  # noqa: E402
from gdr_net_b200.config import Config, postprocess_like_main_gdrn  # noqa: E402
from oracle import ref_shim  # noqa: E402
from oracle.make_golden import REF_CFG  # noqa: E402

# name -> (ROT_HEAD switches, PNP_NET switches, crop classes, weight seed, batch seed)
CASES = {
    "ship_g32": (dict(NORM="GN", NUM_GN_GROUPS=32, NUM_REGIONS=64), dict(REGION_ATTENTION=True), [0, 0, 0, 0], 71, 81),
    "r8_noatt_g1": (dict(NORM="GN", NUM_GN_GROUPS=1, NUM_REGIONS=8), dict(REGION_ATTENTION=False), [0, 0, 0, 0], 72, 82),
    "bce_rot_g64": (dict(NORM="GN", NUM_GN_GROUPS=64, NUM_REGIONS=64, MASK_LOSS_TYPE="BCE", NUM_CLASSES=13, ROT_CLASS_AWARE=True),
                    dict(REGION_ATTENTION=True), [3, 0, 3, 12], 73, 83),
}
EVAL_STRIDE = 16
GRAD_SAMPLES = 96
GRAD_WHOLE = 256


def grad_sample_index(numel: int) -> np.ndarray:
    """Flat indices of the stored elements of a gradient with numel elements (all of them up to GRAD_WHOLE)."""
    if numel <= GRAD_WHOLE:
        return np.arange(numel)
    return np.linspace(0, numel - 1, GRAD_SAMPLES).round().astype(np.int64)


def json_bytes(obj) -> np.ndarray:
    return np.frombuffer(json.dumps(obj).encode(), dtype=np.uint8)


def read_json(arr: np.ndarray):
    return json.loads(arr.tobytes().decode())


def case_config(base, name):
    rh, pn, *_ = CASES[name]
    cfg = copy.deepcopy(base)
    cfg.MODEL.CDPN.ROT_HEAD.update(rh)
    cfg.MODEL.CDPN.PNP_NET.update(pn)
    return cfg


def make_batch(name, B=4):
    rh, _pn, classes, _w, bseed = CASES[name]
    batch = synth.make_batch(B, seed=bseed, num_regions=rh["NUM_REGIONS"])
    if B == len(classes):
        batch["roi_cls"] = torch.tensor(classes, dtype=torch.long)
    return batch


def run_case(ref_gdrn, base, name, save):
    wseed = CASES[name][3]
    torch.manual_seed(0)
    model, optimizer = ref_gdrn.build_model_optimizer(case_config(base, name))
    sd = synth.seeded_state_dict(model.state_dict(), seed=wseed)
    batch = make_batch(name)
    save[f"{name}/sd_keys"] = json_bytes(list(sd))
    save[f"{name}/sd_shapes"] = json_bytes([list(v.shape) for v in sd.values()])
    names = {id(p): n for n, p in model.named_parameters()}
    save[f"{name}/opt_groups"] = json_bytes([dict(params=[names[id(p)] for p in g["params"]], lr=g["lr"])
                                             for g in optimizer.param_groups])
    model.load_state_dict(sd)
    model.eval()
    model.cfg.TEST.USE_PNP = True
    with torch.no_grad():
        out = model(batch["roi_img"].clone(), **synth.forward_kwargs(batch, train=False))
    model.cfg.TEST.USE_PNP = False
    head = torch.cat([out["mask"], out["coor_x"], out["coor_y"], out["coor_z"], out["region"]], dim=1)
    save[f"{name}/eval/head"] = head[:, :, ::EVAL_STRIDE, ::EVAL_STRIDE].numpy()
    save[f"{name}/eval/rot"], save[f"{name}/eval/trans"] = np.asarray(out["rot"]), out["trans"].numpy()
    model.load_state_dict(sd)
    model.train()
    _, loss_dict = model(batch["roi_img"].clone(), **synth.forward_kwargs(batch, train=True))
    sum(loss_dict.values()).backward()
    for k, v in loss_dict.items():
        save[f"{name}/loss/{k}"] = np.array(float(v))
    for k, p in model.named_parameters():
        g = p.grad.detach().reshape(-1).numpy()
        save[f"{name}/grad/{k}"] = g[grad_sample_index(g.size)]
    print(name, {k: round(float(v), 6) for k, v in loss_dict.items()})


def main():
    torch.set_num_threads(os.cpu_count())
    ref_gdrn = ref_shim.import_reference_gdrn()
    base = Config.fromfile(os.path.join(ref_shim.REFERENCE_ROOT, REF_CFG))
    base = postprocess_like_main_gdrn(base, device="cpu")
    base.MODEL.CDPN.BACKBONE.PRETRAINED = ""
    save = {}
    for name in CASES:
        run_case(ref_gdrn, base, name, save)
    path = os.path.join(ROOT, "tests", "golden", "train_head_gn_b4.npz")
    np.savez_compressed(path, **save)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
