"""TEST INFRASTRUCTURE ONLY -- golden vectors for the mask-head switches of the geometric head, produced by the UNMODIFIED reference
(run in the build container; the GPU box has no /root/reference):

  * the reference model (GDRN.py) built from the a6 config with only ROT_HEAD switches changed, two cases:
      bce: MASK_LOSS_TYPE = BCE, MASK_LOSS_GT = visib, XYZ_LOSS_MASK_GT = obj     -> tests/golden/train_mask_bce_b4.npz
      ce:  MASK_LOSS_TYPE = CE,  MASK_LOSS_GT = obj,   REGION_LOSS_MASK_GT = trunc -> tests/golden/train_mask_ce_b4.npz
    each with the eval-mode head output (TEST.USE_PNP maps, cat(mask, coor_x, coor_y, coor_z, region), every 4th pixel of every 4th
    row) and pose, then the train-mode
    losses and a few parameter gradients after `sum(loss_dict.values()).backward()`, on a seeded batch of four crops (not three:
    see oracle/make_golden_nin67.py);
  * `engine_utils.get_out_mask` of a CE head (two channels, with exact z0 == z1 ties) followed by
    `GDRN_Evaluator.get_img_model_points_with_coords2d` (gdrn_evaluator.py:89-126)      -> tests/golden/pnp_ce_select_b3.npz

Usage: python -m oracle.make_golden_masks"""
import copy
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gdr_net_b200 import synth  # noqa: E402
from gdr_net_b200.config import Config, postprocess_like_main_gdrn  # noqa: E402
from oracle import ref_shim  # noqa: E402
from oracle.make_golden import REF_CFG  # noqa: E402

CASES = {  # name -> (ROT_HEAD switches, weight seed, batch seed)
    "bce": (dict(MASK_LOSS_TYPE="BCE", MASK_LOSS_GT="visib", XYZ_LOSS_MASK_GT="obj"), 5, 23),
    "ce": (dict(MASK_LOSS_TYPE="CE", MASK_LOSS_GT="obj", REGION_LOSS_MASK_GT="trunc"), 6, 29),
}
GRAD_KEYS = ("rot_head_net.features.23.weight", "rot_head_net.features.23.bias", "rot_head_net.features.21.weight",
             "pnp_net.features.1.weight", "pnp_net.fc_r.weight", "backbone.bn1.weight")
EVAL_STRIDE = 4  # the eval head is kept on every 4th row and column (all channels) to keep the file small


def train_case(ref_gdrn, name):
    switches, wseed, bseed = CASES[name]
    cfg = Config.fromfile(os.path.join(ref_shim.REFERENCE_ROOT, REF_CFG))
    cfg = postprocess_like_main_gdrn(cfg, device="cpu")
    cfg.MODEL.CDPN.BACKBONE.PRETRAINED = ""
    cfg.MODEL.CDPN.ROT_HEAD.update(switches)
    torch.manual_seed(0)
    model, _ = ref_gdrn.build_model_optimizer(copy.deepcopy(cfg))
    sd = synth.seeded_state_dict(model.state_dict(), seed=wseed)
    batch = synth.make_batch(4, seed=bseed)
    save = {}
    # eval-mode head output
    model.load_state_dict(sd)
    model.eval()
    model.cfg.TEST.USE_PNP = True
    with torch.no_grad():
        out = model(batch["roi_img"].clone(), **synth.forward_kwargs(batch, train=False))
    model.cfg.TEST.USE_PNP = False
    head = torch.cat([out["mask"], out["coor_x"], out["coor_y"], out["coor_z"], out["region"]], dim=1)
    save["eval/head"] = head[:, :, ::EVAL_STRIDE, ::EVAL_STRIDE].numpy()
    save["eval/rot"], save["eval/trans"] = np.asarray(out["rot"]), out["trans"].numpy()
    # train-mode forward + losses + backward
    model.load_state_dict(sd)
    model.train()
    _, loss_dict = model(batch["roi_img"].clone(), **synth.forward_kwargs(batch, train=True))
    sum(loss_dict.values()).backward()
    save.update({("loss/" + k): np.array(float(v)) for k, v in loss_dict.items()})
    grads = dict(model.named_parameters())
    for k in GRAD_KEYS:
        save["grad/" + k] = grads[k].grad.detach().numpy()
    path = os.path.join(ROOT, "tests", "golden", f"train_mask_{name}_b4.npz")
    np.savez_compressed(path, **save)
    print(name, {k: float(v) for k, v in loss_dict.items()}, "head", save["eval/head"].shape)
    print("wrote", path, os.path.getsize(path), "bytes")


def ce_selection_case():
    from oracle.make_golden_pnp import _stub_plotting

    _stub_plotting()
    import core.gdrn_modeling.engine_utils as engine_utils
    import core.gdrn_modeling.gdrn_evaluator as evaluator

    cfg = types.SimpleNamespace(MODEL=types.SimpleNamespace(CDPN=types.SimpleNamespace(ROT_HEAD=types.SimpleNamespace(MASK_LOSS_TYPE="CE"))))
    B = 3
    d = synth.make_pnp_maps(B, seed=13)
    g = torch.Generator().manual_seed(13)
    raw = d["mask"][:, 0]
    z0 = 0.475 + 0.02 * torch.randn(raw.shape, generator=g)  # class 1 (z1 > z0) on the object, where the raw map is 0.9
    z1 = raw.clone()
    tie = torch.zeros_like(raw, dtype=torch.bool)
    tie[:, 16:48:2, :] = True  # every other row through the object: z1 == z0 exactly, which get_out_mask resolves to class 0
    z1 = torch.where(tie, z0, z1)
    mask2 = torch.stack([z0, z1], dim=1).float().contiguous()  # [B, 2, 64, 64]
    out_mask = engine_utils.get_out_mask(cfg, mask2).numpy()
    save = dict(mask=mask2.numpy(), tie=tie.numpy(), xyz=d["xyz"].numpy(), coord_2d=d["coord_2d"].numpy(), extents=d["extents"].numpy(),
                im_wh=d["im_wh"].numpy(), cams=d["cams"].numpy(), R=d["R"].numpy(), t=d["t"].numpy(), out_mask=out_mask)
    for b in range(B):
        im_W, im_H = int(d["im_wh"][b, 0]), int(d["im_wh"][b, 1])
        xyz_i = d["xyz"][b].numpy().transpose(1, 2, 0).copy()
        coord_2d_i = d["coord_2d"][b].numpy().transpose(1, 2, 0).copy()
        img_points, model_points = evaluator.GDRN_Evaluator.get_img_model_points_with_coords2d(
            None, np.squeeze(out_mask[b]), xyz_i, coord_2d_i, im_H=im_H, im_W=im_W, extent=d["extents"][b].numpy(), mask_thr=0.5)
        save[f"img_points_{b}"] = img_points
        save[f"model_points_{b}"] = model_points
        print(b, "points", len(img_points), "tied pixels", int(tie[b].sum()))
    path = os.path.join(ROOT, "tests", "golden", "pnp_ce_select_b3.npz")
    np.savez_compressed(path, **save)
    print("wrote", path, os.path.getsize(path), "bytes")


def main():
    torch.set_num_threads(os.cpu_count())
    ref_gdrn = ref_shim.import_reference_gdrn()
    for name in CASES:
        train_case(ref_gdrn, name)
    ce_selection_case()


if __name__ == "__main__":
    main()
