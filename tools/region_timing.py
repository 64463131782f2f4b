"""Graphed B = 64 "mixed" train step for R = ROT_HEAD.NUM_REGIONS in {8, 32, 64} with PNP_NET.REGION_ATTENTION on and off (runs
on the GPU).

R = 64 with attention is the shipped head (the gdrn_*_ex loss kernels); every other configuration runs the gdrn_*_ex2 ones, a
Patch-PnP input of 64 channels (13 with R = 8, 5 without attention) or 128 (37 with R = 32, 69 with R = 64).  For each R the two
steps are captured as one CUDA graph each (engine.GraphedTrainStep) and timed in alternating windows, so that drift of the shared
machine hits both alike; the output is the per-window step times, their median and spread, and the GPU name and power limit
they were measured on.

usage: python tools/region_timing.py [--windows 8] [--steps 25]"""
import argparse
import gc
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

AUX = ["roi_coord_2d", "roi_cams", "roi_centers", "roi_whs", "roi_extents", "resize_ratios", "gt_xyz", "gt_mask_trunc",
       "gt_mask_visib", "gt_region", "gt_ego_rot", "gt_points", "gt_trans", "gt_trans_ratio"]


def graphed_step(R, att, batch):
    cfg = a6_config(device="cuda", num_regions=R)
    cfg.MODEL.CDPN.PNP_NET.REGION_ATTENTION = att
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
    res = dict(gpu=gpu[0] if gpu else "unknown", batch=args.batch, precision="mixed", steps_per_window=args.steps)
    for R in (8, 32, 64):
        batch = {k: (v.cuda() if isinstance(v, torch.Tensor) else v)
                 for k, v in synth.make_batch(args.batch, seed=100, num_regions=R).items()}
        steps = {}
        for att in (True, False):
            model, step = graphed_step(R, att, batch)
            for _ in range(5):
                step()
            steps[f"r{R}_{'att' if att else 'noatt'}"] = (model, step)
        torch.cuda.synchronize()
        times = {name: [] for name in steps}
        for w in range(args.windows):
            order = list(steps) if w % 2 == 0 else list(reversed(steps))
            for name in order:
                times[name].append(window(steps[name][1], args.steps))
        for name, t in times.items():
            s = sorted(t)
            res[name] = dict(pnp_in=steps[name][0].pnp_net.features[0].in_channels, ms_per_step=[round(v, 4) for v in t],
                             median=round(s[len(s) // 2], 4), min=round(s[0], 4), max=round(s[-1], 4))
        del steps, model, step
        gc.collect()
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
