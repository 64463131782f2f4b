"""Graphed B = 64 "mixed" train step of the class-agnostic a6 head against the class-aware head with all three switches
(ROT / MASK / REGION_CLASS_AWARE, 13 classes, L1 mask, 64 regions: 897 output-conv rows), the crops' classes spread over all 13
classes (runs on the GPU).

Both steps are captured as one CUDA graph each (engine.GraphedTrainStep) and timed in alternating windows, so that drift of the
shared machine hits both alike.  A separate eager class-aware step under torch.profiler gives the share of the step spent in the
class-aware launches (the grouped output conv and its dgrad, the gather, the per-crop bias sums and the gradient reduction; the
per-crop wgrad GEMM runs as gemm_wgrad_kernel and is not separated).  The output is one JSON line with the per-window step times,
their median and spread, the kernel shares, and the GPU name, power limit and SM clock they were measured on.

usage: python tools/class_aware_timing.py [--windows 8] [--steps 25]"""
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
CLASS_KERNELS = ("gemm_fwd_grouped_kernel", "class_gather", "crop_colsum", "class_wgrad_reduce")


def build(aware, batch):
    cfg = a6_config(device="cuda")
    if aware:
        rh = cfg.MODEL.CDPN.ROT_HEAD
        rh.NUM_CLASSES, rh.ROT_CLASS_AWARE, rh.MASK_CLASS_AWARE, rh.REGION_CLASS_AWARE = 13, True, True, True
    model, _ = G.build_model_optimizer(cfg, precision="mixed")
    model.load_state_dict(synth.seeded_state_dict({k: v.cpu() for k, v in model.state_dict().items()}, seed=0))
    model.train()
    kw = synth.forward_kwargs(batch, train=True)
    aux = {k: (kw[k].float().contiguous() if kw[k].dtype != torch.long else kw[k]) for k in AUX}
    aux["sym_infos"] = None
    if aware:
        aux["roi_classes"] = model.engine._classes(batch["roi_cls"], batch["roi_img"].shape[0])
    x = batch["roi_img"].float().contiguous()
    return model, GraphedTrainStep(model.engine, x, aux, train_bn=True)


def window(step, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def kernel_shares(model, batch):
    """Eager class-aware steps under torch.profiler: {kernel family: share of the summed kernel time}."""
    from torch.profiler import ProfilerActivity, profile

    def step():
        for p in model.parameters():
            p.grad = None
        _, ld = model(batch["roi_img"], **synth.forward_kwargs(batch, train=True))
        sum(ld.values()).backward()

    for _ in range(2):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            step()
        torch.cuda.synchronize()
    total, mine = 0.0, {k: 0.0 for k in CLASS_KERNELS}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
        if not t or e.key.startswith(("cudaLaunch", "cudaMemcpy", "Memcpy", "Memset", "cudaStream")):
            continue
        total += t
        for k in CLASS_KERNELS:
            if k in e.key:
                mine[k] += t
    return {k: round(v / total, 5) for k, v in mine.items()}, round(sum(mine.values()) / total, 5)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=8)
    ap.add_argument("--steps", type=int, default=25)
    ap.add_argument("--batch", type=int, default=64)
    args = ap.parse_args()
    q = "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm"
    smi = lambda: subprocess.run(["nvidia-smi", q, "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()  # noqa: E731
    res = dict(gpu_before=smi(), batch=args.batch, precision="mixed", steps_per_window=args.steps)
    batch = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in synth.make_batch(args.batch, seed=100).items()}
    batch["roi_cls"] = (torch.arange(args.batch, device="cuda") * 5) % 13  # every class, in mixed order
    steps = {}
    for name, aware in (("a6", False), ("class_aware_13", True)):
        model, step = build(aware, batch)
        for _ in range(5):
            step()
        steps[name] = (model, step)
    torch.cuda.synchronize()
    times = {name: [] for name in steps}
    for w in range(args.windows):
        order = list(steps) if w % 2 == 0 else list(reversed(steps))
        for name in order:
            times[name].append(window(steps[name][1], args.steps))
    res["gpu_after"] = smi()
    for name, t in times.items():
        s = sorted(t)
        res[name] = dict(rows=steps[name][0].rot_head_net.features[23].out_channels, ms_per_step=[round(v, 4) for v in t],
                         median=round(s[len(s) // 2], 4), min=round(s[0], 4), max=round(s[-1], 4))
    res["aware_over_agnostic_median"] = round(res["class_aware_13"]["median"] / res["a6"]["median"], 4)
    model = steps["class_aware_13"][0]
    del steps
    gc.collect()
    torch.cuda.empty_cache()
    res["class_kernel_share"], res["class_kernel_share_total"] = kernel_shares(model, batch)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
