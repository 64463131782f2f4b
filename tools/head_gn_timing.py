"""B = 64 "mixed" model with a GroupNorm geometry head (ROT_HEAD.NORM = "GN", NUM_GN_GROUPS = 32) against the same weights with
the BatchNorm head (runs on the GPU).

Three measurements, each alternating the two models window by window (device events), so that drift of the shared machine hits
both alike: the captured train step (engine.GraphedTrainStep), the eager step of the module API (forward, sum of the loss dict,
backward) and folded inference (eval mode, the cached inference graph), reported in crops/s.  One JSON line with per-window
times, medians and ratios, and the GPU name, power limit and SM clock before and after.

usage: python tools/head_gn_timing.py [--windows 8] [--steps 20]"""
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
from tools.dropblock_timing import graphed_step  # noqa: E402
from tools.freeze_timing import alternate, eager_step  # noqa: E402


def build(norm, sd):
    cfg = a6_config(device="cuda")
    cfg.MODEL.CDPN.ROT_HEAD.NORM = norm
    cfg.MODEL.CDPN.ROT_HEAD.NUM_GN_GROUPS = 32
    model, _ = G.build_model_optimizer(cfg, precision="mixed")
    own = model.state_dict()
    model.load_state_dict({k: v for k, v in sd.items() if k in own}, strict=True)
    model.train()
    return model


def infer_step(model, batch):
    kw = synth.forward_kwargs(batch, train=False)

    def step():
        with torch.no_grad():
            model(batch["roi_img"], **kw)

    return step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=8)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--batch", type=int, default=64)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/head_gn_timing.py measures on the GPU; no CUDA device found")
    q = "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm"
    smi = lambda: subprocess.run(["nvidia-smi", q, "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()  # noqa: E731
    res = dict(gpu_before=smi(), batch=args.batch, precision="mixed", groups=32, steps_per_window=args.steps)
    batch = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in synth.make_batch(args.batch, seed=100).items()}
    m, _ = G.build_model_optimizer(a6_config(device="cpu"), precision="mixed")
    sd = synth.seeded_state_dict(m.state_dict(), seed=0)  # the seeded weights bench.py uses
    models = {"BN": build("BN", sd), "GN": build("GN", sd)}
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
    for m in models.values():
        m.eval()
        m.use_cuda_graphs = True
    infer = {name: infer_step(m, batch) for name, m in models.items()}
    for _ in range(3):
        for s in infer.values():
            s()
    res["inference"] = alternate(infer, args.windows, args.steps)
    for mode in ("graphed", "eager", "inference"):
        t = res[mode]
        res[f"{mode}_ratio_gn_over_bn"] = round(t["GN"]["median"] / t["BN"]["median"], 4)
    res["inference_crops_per_s"] = {n: round(args.batch / (t["median"] * 1e-3), 1) for n, t in res["inference"].items()}
    res["gpu_after"] = smi()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
