"""TEST INFRASTRUCTURE ONLY -- golden vectors for the geometry head's shape switches (ROT_HEAD.CONV_KERNEL_SIZE,
OUT_CONV_KERNEL_SIZE), produced by the UNMODIFIED reference model (GDRN.py, cdpn_rot_head_region.py) built from the a6 config with
only these switches changed (the GPU box has no reference install):

  k4_o1      4x4 deconv (pad 1), 1x1 output conv; otherwise the shipped head (64 regions, attention, 2-D coordinates)
  k2_o3_r8   2x2 deconv (pad 0), 3x3 output conv, 8 regions without region attention
  k3_o3_ca   the shipped deconv, 3x3 output conv, CE mask, class-aware xyz, mask and regions (13 classes)
  k4_o3_gn   4x4 deconv, 3x3 output conv, GroupNorm head with G = 32

Each case holds what oracle/make_golden_head_gn.py stores (same batch recipe, gradient sampling and map stride): the eval-mode
TEST.USE_PNP maps and pose, the train-mode losses, every parameter gradient, the state_dict manifest and the optimizer groups.
Output: tests/golden/train_head_shape_b4.npz, keys "<case>/loss/<name>", "<case>/grad/<param>", "<case>/eval/{head,rot,trans}",
"<case>/sd_keys", "<case>/sd_shapes", "<case>/opt_groups".
Usage: python -m oracle.make_golden_head_shape"""
import copy
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
from oracle.make_golden_head_gn import EVAL_STRIDE, grad_sample_index, json_bytes  # noqa: E402,F401

# name -> (ROT_HEAD switches, PNP_NET switches, crop classes, weight seed, batch seed)
CASES = {
    "k4_o1": (dict(CONV_KERNEL_SIZE=4, OUT_CONV_KERNEL_SIZE=1, NUM_REGIONS=64), dict(REGION_ATTENTION=True), [0, 0, 0, 0], 91, 101),
    "k2_o3_r8": (dict(CONV_KERNEL_SIZE=2, OUT_CONV_KERNEL_SIZE=3, NUM_REGIONS=8), dict(REGION_ATTENTION=False), [0, 0, 0, 0],
                 92, 102),
    "k3_o3_ca": (dict(CONV_KERNEL_SIZE=3, OUT_CONV_KERNEL_SIZE=3, NUM_REGIONS=64, MASK_LOSS_TYPE="CE", NUM_CLASSES=13,
                      ROT_CLASS_AWARE=True, MASK_CLASS_AWARE=True, REGION_CLASS_AWARE=True), dict(REGION_ATTENTION=True),
                 [3, 0, 3, 12], 93, 103),
    "k4_o3_gn": (dict(CONV_KERNEL_SIZE=4, OUT_CONV_KERNEL_SIZE=3, NORM="GN", NUM_GN_GROUPS=32, NUM_REGIONS=64),
                 dict(REGION_ATTENTION=True), [0, 0, 0, 0], 94, 104),
}


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
    path = os.path.join(ROOT, "tests", "golden", "train_head_shape_b4.npz")
    np.savez_compressed(path, **save)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
