"""B = 64 "mixed" train step with frozen sub-networks (BACKBONE / ROT_HEAD / PNP_NET .FREEZE) against the unfrozen step (runs on
the GPU).

Each combination runs one step through the module API (forward, sum of the loss dict, backward: the eager step a fine-tuning loop
takes) and one captured step (engine.GraphedTrainStep).  Eager and graphed steps are each timed with device events in windows
that alternate over the combinations, so that drift of the shared machine hits all of them alike.  Per combination the output
gives the per-window step times, their median and spread, and the step's peak allocation above what was allocated before it
(torch.cuda.max_memory_allocated).  With the head and the Patch-PnP frozen there is nothing to differentiate: that combination
is timed as the forward alone.  One JSON line, with the GPU name, power limit and SM clock before and after.

usage: python tools/freeze_timing.py [--windows 6] [--steps 20]"""
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
COMBOS = {"none": (False, False, False), "bb": (True, False, False), "head": (False, True, False), "pnp": (False, False, True),
          "bb_pnp": (True, False, True), "head_pnp": (False, True, True)}


def build(freeze, sd):
    cfg = a6_config(device="cuda")
    cfg.MODEL.CDPN.BACKBONE.FREEZE, cfg.MODEL.CDPN.ROT_HEAD.FREEZE, cfg.MODEL.CDPN.PNP_NET.FREEZE = freeze
    model, _ = G.build_model_optimizer(cfg, precision="mixed")
    model.load_state_dict(sd)
    model.train()
    return model


def eager_step(model, batch):
    kw = synth.forward_kwargs(batch, train=True)

    def step():
        for p in model.parameters():
            p.grad = None
        _, ld = model(batch["roi_img"], **kw)
        loss = sum(ld.values())
        if loss.requires_grad:
            loss.backward()

    return step


def graphed_step(model, batch):
    eng = model.engine
    if not eng.live_any:
        return None
    kw = synth.forward_kwargs(batch, train=True)
    aux = {k: (kw[k].float().contiguous() if kw[k].dtype != torch.long else kw[k]) for k in AUX}
    aux["sym_infos"] = None
    return GraphedTrainStep(eng, batch["roi_img"].float().contiguous(), aux, train_bn=True)


def window(step, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def peak_above_base(step):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    step()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def alternate(steps, windows, n):
    times = {name: [] for name in steps}
    for w in range(windows):
        order = list(steps) if w % 2 == 0 else list(reversed(steps))
        for name in order:
            times[name].append(window(steps[name], n))
    out = {}
    for name, t in times.items():
        s = sorted(t)
        out[name] = dict(ms_per_step=[round(v, 4) for v in t], median=round(s[len(s) // 2], 4), min=round(s[0], 4), max=round(s[-1], 4))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=6)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--batch", type=int, default=64)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/freeze_timing.py measures on the GPU; no CUDA device found")
    q = "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm"
    smi = lambda: subprocess.run(["nvidia-smi", q, "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()  # noqa: E731
    res = dict(gpu_before=smi(), batch=args.batch, precision="mixed", steps_per_window=args.steps)
    batch = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in synth.make_batch(args.batch, seed=100).items()}
    sd = synth.seeded_state_dict(_template(), seed=0)  # the seeded weights bench.py uses
    models = {name: build(freeze, sd) for name, freeze in COMBOS.items()}
    # eager: the module API step
    eager = {name: eager_step(m, batch) for name, m in models.items()}
    for step in eager.values():
        for _ in range(3):
            step()
    res["peak_alloc_mib_eager"] = {name: round(peak_above_base(step) / 2**20, 1) for name, step in eager.items()}
    res["eager"] = alternate(eager, args.windows, args.steps)
    gc.collect()
    torch.cuda.empty_cache()
    # graphed: one CUDA graph per step; each frozen combination alternates with the unfrozen graph, one pair at a time (every
    # graph keeps a memory pool of a whole step)
    g_none = graphed_step(models["none"], batch)
    res["graphed"], res["graphed_over_unfrozen"] = {}, {}
    for name, m in models.items():
        g = None if name == "none" else graphed_step(m, batch)
        if g is None:
            continue
        for _ in range(3):
            g()
            g_none()
        t = alternate({"none": g_none, name: g}, args.windows, args.steps)
        res["graphed"][name] = dict(t[name], unfrozen_median=t["none"]["median"])
        res["graphed_over_unfrozen"][name] = round(t[name]["median"] / t["none"]["median"], 4)
        del g, t
        gc.collect()
        torch.cuda.empty_cache()
    res["gpu_after"] = smi()
    base = res["eager"]["none"]["median"]
    res["eager_over_unfrozen"] = {k: round(v["median"] / base, 4) for k, v in res["eager"].items()}
    print(json.dumps(res))


def _template():
    m, _ = G.build_model_optimizer(a6_config(device="cpu"), precision="mixed")
    return m.state_dict()


if __name__ == "__main__":
    main()
