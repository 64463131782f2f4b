"""B = 64 "mixed" model with the geometry head's shape switches (ROT_HEAD.CONV_KERNEL_SIZE, OUT_CONV_KERNEL_SIZE) against the shipped
head (k3 deconv, 1x1 output conv), all with the same seeded weights wherever the shapes agree (runs on the GPU).

Heads: "k3_o1" (shipped), "k4_o1", "k3_o3", "k4_o3".  Three measurements, each alternating the models window by window (device
events), so that drift of the shared machine hits all alike: the captured train step (engine.GraphedTrainStep), the eager step of
the module API (forward, sum of the loss dict, backward) and folded inference (eval mode, the cached inference graph), reported in
crops/s.  One JSON line with per-window times, medians, ratios to the shipped head, and the GPU name, power limit and SM clock
before and after.

usage: python tools/head_shape_timing.py [--windows 8] [--steps 20]"""
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
from tools.head_gn_timing import infer_step  # noqa: E402

HEADS = {"k3_o1": (3, 1), "k4_o1": (4, 1), "k3_o3": (3, 3), "k4_o3": (4, 3)}


def build(k, k_out, seed):
    cfg = a6_config(device="cuda")
    cfg.MODEL.CDPN.ROT_HEAD.CONV_KERNEL_SIZE = k
    cfg.MODEL.CDPN.ROT_HEAD.OUT_CONV_KERNEL_SIZE = k_out
    model, _ = G.build_model_optimizer(cfg, precision="mixed")
    # the seeded weights bench.py uses (seed 0) for every tensor whose shape does not depend on the head shape
    model.load_state_dict(synth.seeded_state_dict({n: v.cpu() for n, v in model.state_dict().items()}, seed=seed), strict=True)
    model.train()
    return model


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=8)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--batch", type=int, default=64)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/head_shape_timing.py measures on the GPU; no CUDA device found")
    q = "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm"
    smi = lambda: subprocess.run(["nvidia-smi", q, "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()  # noqa: E731
    res = dict(gpu_before=smi(), batch=args.batch, precision="mixed", steps_per_window=args.steps)
    batch = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in synth.make_batch(args.batch, seed=100).items()}
    models = {name: build(k, k_out, 0) for name, (k, k_out) in HEADS.items()}
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
        res[f"{mode}_ratio_to_k3_o1"] = {n: round(t[n]["median"] / t["k3_o1"]["median"], 4) for n in HEADS if n != "k3_o1"}
    res["inference_crops_per_s"] = {n: round(args.batch / (t["median"] * 1e-3), 1) for n, t in res["inference"].items()}
    res["gpu_after"] = smi()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
