"""TEST INFRASTRUCTURE ONLY -- golden vectors for class-aware geometry heads (ROT_HEAD.ROT_CLASS_AWARE / MASK_CLASS_AWARE /
REGION_CLASS_AWARE), produced by the UNMODIFIED reference model (GDRN.py) built from the a6 config with only these switches changed
(the GPU box has no reference install):

  all13    all three switches, 13 classes, L1 mask, 64 regions        897 output-conv rows
  rot13    ROT_CLASS_AWARE only, 13 classes, 64 regions               105 rows
  mr_ce21  MASK_CLASS_AWARE with the CE mask + REGION_CLASS_AWARE, 8 regions, 21 classes   2 * 21 + 3 + 9 * 21 = 234 rows

Each case: a seeded batch of four crops whose classes repeat one class and leave most classes absent, the train-mode losses and
the gradients of the output conv (all rows: the rows of absent classes are exactly 0), features.21, fc_r and the stem BatchNorm
after `sum(loss_dict.values()).backward()`, and the eval-mode TEST.USE_PNP maps of each crop's class (every 4th pixel of every
4th row) and pose.
Output: tests/golden/train_class_aware_b4.npz, keys "<case>/loss/<name>", "<case>/grad/<param>", "<case>/eval/{head,rot,trans}".
Usage: python -m oracle.make_golden_class_aware"""
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

# name -> (ROT_HEAD switches, crop classes, weight seed, batch seed)
CASES = {
    "all13": (dict(NUM_CLASSES=13, ROT_CLASS_AWARE=True, MASK_CLASS_AWARE=True, REGION_CLASS_AWARE=True, NUM_REGIONS=64),
              [3, 0, 3, 12], 51, 61),
    "rot13": (dict(NUM_CLASSES=13, ROT_CLASS_AWARE=True, NUM_REGIONS=64), [3, 0, 3, 12], 52, 62),
    "mr_ce21": (dict(NUM_CLASSES=21, MASK_CLASS_AWARE=True, REGION_CLASS_AWARE=True, MASK_LOSS_TYPE="CE", NUM_REGIONS=8),
                [5, 0, 5, 20], 53, 63),
}
GRAD_KEYS = ("rot_head_net.features.23.weight", "rot_head_net.features.23.bias", "rot_head_net.features.21.weight",
             "pnp_net.fc_r.weight", "backbone.bn1.weight")
EVAL_STRIDE = 4


def run_case(ref_gdrn, base, name, save):
    rh, classes, wseed, bseed = CASES[name]
    cfg = copy.deepcopy(base)
    cfg.MODEL.CDPN.ROT_HEAD.update(rh)
    torch.manual_seed(0)
    model, _ = ref_gdrn.build_model_optimizer(copy.deepcopy(cfg))
    sd = synth.seeded_state_dict(model.state_dict(), seed=wseed)
    batch = synth.make_batch(4, seed=bseed, num_regions=rh["NUM_REGIONS"])
    batch["roi_cls"] = torch.tensor(classes, dtype=torch.long)
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
    print(name, "rows", model.rot_head_net.features[23].out_channels, {k: round(float(v), 6) for k, v in loss_dict.items()})


def main():
    torch.set_num_threads(os.cpu_count())
    ref_gdrn = ref_shim.import_reference_gdrn()
    base = Config.fromfile(os.path.join(ref_shim.REFERENCE_ROOT, REF_CFG))
    base = postprocess_like_main_gdrn(base, device="cpu")
    base.MODEL.CDPN.BACKBONE.PRETRAINED = ""
    save = {}
    for name in CASES:
        run_case(ref_gdrn, base, name, save)
    path = os.path.join(ROOT, "tests", "golden", "train_class_aware_b4.npz")
    np.savez_compressed(path, **save)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
