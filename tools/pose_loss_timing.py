"""Graphed B = 64 "mixed" train step with the shipped pose losses against a switch-heavy PNP_NET configuration (runs on the GPU).

The default configuration runs gdrn_pose_loss, the other gdrn_pose_loss_ex + gdrn_loss_finalize_ex2 (point matching on R and t
with Smooth-L1, angular rot, disentangled MSE translation and L1 bind losses).  Both steps are captured as one CUDA graph each
(engine.GraphedTrainStep) and timed in alternating windows, so that drift of the shared machine hits both alike; the output
is the per-window step times, their median and spread, and the GPU name and power limit they were measured on.

usage: python tools/pose_loss_timing.py [--windows 8] [--steps 25]"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from gdr_net_b200 import GDRN as G  # noqa: E402
from gdr_net_b200 import synth  # noqa: E402
from gdr_net_b200.config import a6_config  # noqa: E402
from gdr_net_b200.engine import GraphedTrainStep  # noqa: E402

SWITCH_HEAVY = dict(PM_R_ONLY=False, PM_LOSS_TYPE="Smooth_L1", PM_SMOOTH_L1_BETA=0.5, ROT_LW=1.0, ROT_LOSS_TYPE="angular",
                    TRANS_LW=1.0, TRANS_LOSS_TYPE="MSE", TRANS_LOSS_DISENTANGLE=True, BIND_LW=1.0, BIND_LOSS_TYPE="L1")
AUX = ["roi_coord_2d", "roi_cams", "roi_centers", "roi_whs", "roi_extents", "resize_ratios", "gt_xyz", "gt_mask_trunc",
       "gt_mask_visib", "gt_region", "gt_ego_rot", "gt_points", "gt_trans", "gt_trans_ratio"]


def graphed_step(switches, batch, B):
    cfg = a6_config(device="cuda")
    for k, v in switches.items():
        setattr(cfg.MODEL.CDPN.PNP_NET, k, v)
    model, _ = G.build_model_optimizer(cfg, precision="mixed")
    model.load_state_dict(synth.seeded_state_dict({k: v.cpu() for k, v in model.state_dict().items()}, seed=0))
    model.train()
    kw = synth.forward_kwargs(batch, train=True)
    aux = {k: (kw[k].float().contiguous() if kw[k].dtype != torch.long else kw[k]) for k in AUX}
    aux["sym_infos"] = None
    x = batch["roi_img"].float().contiguous()
    step = GraphedTrainStep(model.engine, x, aux, train_bn=True)
    return model, step


def window(step, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=8)
    ap.add_argument("--steps", type=int, default=25)
    ap.add_argument("--batch", type=int, default=64)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    batch = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in synth.make_batch(args.batch, seed=100).items()}
    steps = {}
    for name, sw in (("default", {}), ("switch_heavy", SWITCH_HEAVY)):
        model, step = graphed_step(sw, batch, args.batch)
        for _ in range(5):
            step()
        steps[name] = (model, step)
    torch.cuda.synchronize()
    times = {name: [] for name in steps}
    for w in range(args.windows):
        order = list(steps) if w % 2 == 0 else list(reversed(steps))
        for name in order:
            times[name].append(window(steps[name][1], args.steps))
    res = dict(gpu=gpu[0] if gpu else "unknown", batch=args.batch, precision="mixed", steps_per_window=args.steps,
               loss_names={n: steps[n][0].engine.loss_names for n in steps})
    for name, t in times.items():
        s = sorted(t)
        res[name] = dict(ms_per_step=[round(v, 4) for v in t], median=round(s[len(s) // 2], 4), min=round(s[0], 4), max=round(s[-1], 4))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
