"""B = 64 "mixed" train step with DropBlock on the Patch-PnP input (PNP_HEAD_CFG.drop_prob = 0.25, dropblock_size 5) against
the same step without it (drop_prob = 0) (runs on the GPU).

Both models run the captured train step (engine.GraphedTrainStep) and the eager step of the module API (forward, sum of the loss
dict, backward).  The DropBlock model's counter is set past the end of the schedule, so every step samples a mask at p = 0.25.
The two are timed with device events in windows that alternate between them, so that drift of the shared machine hits both
alike.  One JSON line: per-window step times, median and spread, the overhead of DropBlock, and the GPU name, power limit and SM
clock before and after.

usage: python tools/dropblock_timing.py [--windows 8] [--steps 20]"""
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
from tools.freeze_timing import AUX, alternate, eager_step  # noqa: E402
from gdr_net_b200.engine import GraphedTrainStep  # noqa: E402


def build(drop_prob, sd):
    cfg = a6_config(device="cuda")
    cfg.MODEL.CDPN.PNP_NET.PNP_HEAD_CFG.update(drop_prob=drop_prob, dropblock_size=5)
    model, _ = G.build_model_optimizer(cfg, precision="mixed")
    model.load_state_dict(sd)
    model.train()
    if drop_prob > 0:
        model.pnp_net.dropblock_step = 5000
    return model


def graphed_step(model, batch):
    kw = synth.forward_kwargs(batch, train=True)
    aux = {k: (kw[k].float().contiguous() if kw[k].dtype != torch.long else kw[k]) for k in AUX}
    aux["sym_infos"] = None
    return GraphedTrainStep(model.engine, batch["roi_img"].float().contiguous(), aux, train_bn=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=8)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--batch", type=int, default=64)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/dropblock_timing.py measures on the GPU; no CUDA device found")
    q = "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm"
    smi = lambda: subprocess.run(["nvidia-smi", q, "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()  # noqa: E731
    res = dict(gpu_before=smi(), batch=args.batch, precision="mixed", steps_per_window=args.steps)
    batch = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in synth.make_batch(args.batch, seed=100).items()}
    m, _ = G.build_model_optimizer(a6_config(device="cpu"), precision="mixed")
    sd = synth.seeded_state_dict(m.state_dict(), seed=0)  # the seeded weights bench.py uses
    models = {"p0": build(0.0, sd), "p0.25": build(0.25, sd)}
    graphed = {name: graphed_step(m, batch) for name, m in models.items()}
    for _ in range(3):
        for g in graphed.values():
            g()
    res["graphed"] = alternate(graphed, args.windows, args.steps)
    eager = {name: eager_step(m, batch) for name, m in models.items()}
    for _ in range(3):
        for s in eager.values():
            s()
    res["eager"] = alternate(eager, args.windows, args.steps)
    for mode in ("graphed", "eager"):
        t = res[mode]
        res[f"{mode}_overhead_ms"] = round(t["p0.25"]["median"] - t["p0"]["median"], 4)
        res[f"{mode}_ratio"] = round(t["p0.25"]["median"] / t["p0"]["median"], 4)
    res["dropblock_step_after"] = models["p0.25"].pnp_net.dropblock_step
    res["gpu_after"] = smi()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
