"""TEST INFRASTRUCTURE ONLY -- golden vectors for the evaluator's network-initialised PnP modes (TEST.PNP_TYPE net_iter_pnp,
net_ransac_pnp, net_ransac_pnp_rot), produced by the UNMODIFIED reference method imported from /root/reference (run in the build
container; the GPU box has no /root/reference):

  * `GDRN_EvaluatorCustom.process_net_and_pnp` (gdrn_custom_evaluator.py:207-335) for pnp_type in {iter, ransac, ransac_rot},
    which calls get_out_coor / get_out_mask, get_img_model_points_with_coords2d, cv2.solvePnP / cv2.solvePnPRansac and te

on an evaluator instance created without __init__ (only the attributes the method reads are set) and the seeded synthetic head
outputs of `gdr_net_b200.synth.make_pnp_maps`.  The network pose is the true pose perturbed by a seeded rotation and translation;
ROI 2's translation is 2.5 m off: the `te > 1` rule fires there in the RANSAC mode, and in the
iterative mode the solution moves more than 1 m but is kept (the reference compares it with itself, see net_pnp_oracle).  Output: tests/golden/pnp_net_b4.npz
(inputs, network pose, the selected image / model points per ROI, the [3,4] pose per ROI and mode).
Usage: python -m oracle.make_golden_net_pnp"""
import logging
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gdr_net_b200 import synth  # noqa: E402
from oracle import ref_shim  # noqa: E402
from oracle.make_golden_pnp import _stub_plotting  # noqa: E402

B = 4


def net_pose(d, seed=1):
    """Seeded perturbation of the true pose: rotation by 0.05-0.3 rad about a random axis, translation by a few cm; ROI 2 is
    2.5 m too far.  float32, like the model's output."""
    import cv2

    rng = np.random.default_rng(seed)
    R = np.zeros((B, 3, 3), np.float32)
    t = np.zeros((B, 3), np.float32)
    for b in range(B):
        ax = rng.normal(size=3)
        ax *= rng.uniform(0.05, 0.3) / np.linalg.norm(ax)
        R[b] = (cv2.Rodrigues(ax)[0] @ d["R"][b].double().numpy()).astype(np.float32)
        t[b] = (d["t"][b].double().numpy() + rng.normal(scale=0.02, size=3)).astype(np.float32)
    t[2, 2] += 2.5
    return R, t


def main():
    import cv2

    ref_shim.install()
    _stub_plotting()
    import numpy.lib.npyio

    if not hasattr(numpy.lib.npyio, "save"):  # numpy 2 moved it; the module imports it unused
        numpy.lib.npyio.save = np.save
    import core.gdrn_modeling.gdrn_custom_evaluator as evaluator

    d = synth.make_pnp_maps(B, seed=9)
    R_net, t_net = net_pose(d)
    cfg = types.SimpleNamespace(MODEL=types.SimpleNamespace(CDPN=types.SimpleNamespace(ROT_HEAD=types.SimpleNamespace(
        MASK_LOSS_TYPE="L1", MASK_THR_TEST=0.5))))
    ev = evaluator.GDRN_EvaluatorCustom.__new__(evaluator.GDRN_EvaluatorCustom)
    ev.cfg = cfg
    ev._cpu_device = torch.device("cpu")
    ev._logger = logging.getLogger("make_golden_net_pnp")
    ev.train_objs = None
    ev.obj_names = ["obj"]
    save = {k: v.numpy() for k, v in d.items()}
    save["R_net"], save["t_net"] = R_net, t_net
    for pnp_type in ("iter", "ransac", "ransac_rot"):
        ev._predictions = {}
        inputs = [dict(
            roi_img=[None] * B, bbox_center=[(0.0, 0.0)] * B, scale=[1.0] * B, roi_coord_2d=d["coord_2d"].clone(),
            im_H=d["im_wh"][:, 1].long(), im_W=d["im_wh"][:, 0].long(), scene_im_id=[f"1/{b}" for b in range(B)], cam=d["cams"],
            roi_cls=[0] * B, score=[1.0] * B, file_name=[f"roi_{b}" for b in range(B)], roi_extent=d["extents"])]
        outputs = [dict(time=0.0)]
        # fresh copies per call: on CPU tensors `.cpu().numpy()` aliases, and the method scales coord_2d in place and cv2 writes
        # the iterative solution into the network translation
        out_dict = dict(mask=d["mask"].clone(), coor_x=d["xyz"][:, 0:1].clone(), coor_y=d["xyz"][:, 1:2].clone(),
                        coor_z=d["xyz"][:, 2:3].clone(), rot=torch.from_numpy(R_net.copy()), trans=torch.from_numpy(t_net.copy()))
        ev.process_net_and_pnp(inputs, outputs, out_dict, pnp_type=pnp_type)
        for b in range(B):
            res = ev._predictions["obj"][f"roi_{b}"]
            save[f"pose_{pnp_type}_{b}"] = np.concatenate([np.asarray(res["R"], np.float64),
                                                          np.asarray(res["t"], np.float64).reshape(3, 1)], axis=1)
            print(pnp_type, b, save[f"pose_{pnp_type}_{b}"][:, 3])
    # the point lists the method selected (same function, same inputs)
    from core.gdrn_modeling.engine_utils import get_out_coor, get_out_mask

    out_mask = get_out_mask(cfg, d["mask"]).numpy()
    out_xyz = get_out_coor(cfg, d["xyz"][:, 0:1], d["xyz"][:, 1:2], d["xyz"][:, 2:3]).numpy()
    for b in range(B):
        ip, mp = ev.get_img_model_points_with_coords2d(
            np.squeeze(out_mask[b]), out_xyz[b].transpose(1, 2, 0), d["coord_2d"][b].numpy().transpose(1, 2, 0).copy(),
            im_H=int(d["im_wh"][b, 1]), im_W=int(d["im_wh"][b, 0]), extent=d["extents"][b].numpy(), mask_thr=0.5)
        save[f"img_points_{b}"], save[f"model_points_{b}"] = ip, mp
    save["cv2_version"] = np.array(cv2.__version__)
    out = os.path.join(ROOT, "tests", "golden", "pnp_net_b4.npz")
    np.savez_compressed(out, **save)
    print("wrote", out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
