"""TEST INFRASTRUCTURE ONLY -- golden vectors for other surface-region counts (ROT_HEAD.NUM_REGIONS) and Patch-PnP without region
attention (PNP_NET.REGION_ATTENTION), produced by the UNMODIFIED reference model (GDRN.py) built from the a6 config with only
these switches changed (the GPU box has no reference install):

  r8         8 regions, attention, 2-D coordinates           nIn 13, a 64-wide Patch-PnP input
  r32_noatt  32 regions, no attention, 2-D coordinates       nIn 5
  r64_noatt  the shipped head without attention              nIn 5
  r4_ce      4 regions, attention, no 2-D coordinates, CE mask head with REGION_LOSS_MASK_GT = trunc   nIn 7, MO 2
  r60        60 regions, attention, 2-D coordinates          nIn 65, a 128-wide input with a partly used last chunk

Each case: a seeded batch of four crops whose region labels run over 1..R (see oracle/make_golden_nin67.py for why four), the
train-mode losses and a few parameter gradients after `sum(loss_dict.values()).backward()`; for r8 and r32_noatt also the
eval-mode TEST.USE_PNP head maps (every 4th pixel of every 4th row) and pose.
Output: tests/golden/train_regions_b4.npz, keys "<case>/loss/<name>", "<case>/grad/<param>", "<case>/eval/{head,rot,trans}".
Usage: python -m oracle.make_golden_regions"""
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

# name -> (ROT_HEAD switches, PNP_NET switches, weight seed, batch seed, eval maps)
CASES = {
    "r8": (dict(NUM_REGIONS=8), dict(REGION_ATTENTION=True, WITH_2D_COORD=True), 31, 41, True),
    "r32_noatt": (dict(NUM_REGIONS=32), dict(REGION_ATTENTION=False, WITH_2D_COORD=True), 32, 42, True),
    "r64_noatt": (dict(NUM_REGIONS=64), dict(REGION_ATTENTION=False, WITH_2D_COORD=True), 33, 43, False),
    "r4_ce": (dict(NUM_REGIONS=4, MASK_LOSS_TYPE="CE", REGION_LOSS_MASK_GT="trunc"), dict(REGION_ATTENTION=True, WITH_2D_COORD=False),
              34, 44, False),
    "r60": (dict(NUM_REGIONS=60), dict(REGION_ATTENTION=True, WITH_2D_COORD=True), 35, 45, False),
}
GRAD_KEYS = ("rot_head_net.features.23.weight", "rot_head_net.features.23.bias", "rot_head_net.features.21.weight",
             "pnp_net.features.0.weight", "pnp_net.fc_r.weight", "backbone.bn1.weight")
EVAL_STRIDE = 4


def case_config(name, base):
    rh, pn, *_ = CASES[name]
    cfg = copy.deepcopy(base)
    cfg.MODEL.CDPN.ROT_HEAD.update(rh)
    cfg.MODEL.CDPN.PNP_NET.update(pn)
    return cfg


def run_case(ref_gdrn, base, name, save):
    rh, _pn, wseed, bseed, want_eval = CASES[name]
    cfg = case_config(name, base)
    torch.manual_seed(0)
    model, _ = ref_gdrn.build_model_optimizer(copy.deepcopy(cfg))
    sd = synth.seeded_state_dict(model.state_dict(), seed=wseed)
    batch = synth.make_batch(4, seed=bseed, num_regions=rh["NUM_REGIONS"])
    if want_eval:
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
    grads = dict(model.named_parameters())
    for k in GRAD_KEYS:
        save[f"{name}/grad/{k}"] = grads[k].grad.detach().numpy()
    print(name, "nIn", model.pnp_net.features[0].in_channels, {k: round(float(v), 6) for k, v in loss_dict.items()})


def main():
    torch.set_num_threads(os.cpu_count())
    ref_gdrn = ref_shim.import_reference_gdrn()
    base = Config.fromfile(os.path.join(ref_shim.REFERENCE_ROOT, REF_CFG))
    base = postprocess_like_main_gdrn(base, device="cpu")
    base.MODEL.CDPN.BACKBONE.PRETRAINED = ""
    save = {}
    for name in CASES:
        run_case(ref_gdrn, base, name, save)
    path = os.path.join(ROOT, "tests", "golden", "train_regions_b4.npz")
    np.savez_compressed(path, **save)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
