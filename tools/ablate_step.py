"""In-situ cost of each non-GEMM kernel family inside the graphed train step (runs on the GPU box).

ncu's per-launch durations are cold-cache and serialised; producer/consumer pairs that live in the 50 MB L2 (split-K
workspace -> unpack, conv output -> BN) look 2-5x more expensive there than they are inside the step.  Here each family's
C entry point is replaced by a no-op, the whole step is re-captured as a CUDA graph and re-timed: baseline - ablated = the
family's real share.  (The ablated step computes garbage; only its duration is used.)

usage: python tools/ablate_step.py [B] [precision]"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from gdr_net_b200 import GDRN as G
from gdr_net_b200 import synth
from gdr_net_b200.capi import C
from gdr_net_b200.config import a6_config
from gdr_net_b200.engine import GraphedTrainStep

FAMILIES = {
    "unpack_wgrad": ["gdrn_unpack_wgrad"],
    "pack_weights": ["gdrn_pack_weight_batched"],
    "bn_fwd": ["gdrn_bn_fwd"],
    "bn_bwd": ["gdrn_bn_bwd"],
    "stem_im2col": ["gdrn_stem_im2col"],
    "maxpool": ["gdrn_maxpool_fwd", "gdrn_maxpool_bwd"],
    "upsample": ["gdrn_upsample2x_fwd", "gdrn_upsample2x_bwd"],
    "zero_insert": ["gdrn_zero_insert"],
    "groupnorm": ["gdrn_gn_relu_fwd", "gdrn_gn_relu_bwd"],
}


def main():
    B = int(sys.argv[1]) if len(sys.argv) > 1 else 64
    precision = sys.argv[2] if len(sys.argv) > 2 else "half"
    cfg = a6_config(device="cuda")
    model, _ = G.build_model_optimizer(cfg, precision=precision)
    model.train()
    eng = model.engine
    batch = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in synth.make_batch(B, seed=100).items()}
    kw = synth.forward_kwargs(batch, train=True)
    names = ["roi_coord_2d", "roi_cams", "roi_centers", "roi_whs", "roi_extents", "resize_ratios", "gt_xyz", "gt_mask_trunc",
             "gt_mask_visib", "gt_region", "gt_ego_rot", "gt_points", "gt_trans", "gt_trans_ratio"]
    aux = {k: kw[k] for k in names}
    aux["sym_infos"] = None
    aux = {k: (v.float().contiguous() if isinstance(v, torch.Tensor) and v.dtype != torch.long else v) for k, v in aux.items()}
    x = batch["roi_img"].float().contiguous()

    def timed(steps=20):
        g = GraphedTrainStep(eng, x, aux, train_bn=True, warmup=1)
        for _ in range(3):
            g()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(steps):
            g()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps

    eng.forward(x, aux, train_bn=True, do_loss=True)  # sizes workspaces / job tables with the real kernels
    eng.backward(torch.ones(8, device="cuda"))
    torch.cuda.synchronize()
    base = timed()
    print(f"baseline                {base:8.3f} ms/step  (B={B}, {precision})")
    if len(sys.argv) > 3 and sys.argv[3] == "base":
        print(f"baseline again          {timed():8.3f} ms/step")
        return
    for fam, entries in FAMILIES.items():
        missing = [e for e in entries if not hasattr(C.load(), e)]
        if missing:
            print(f"{fam:22s}  skipped (no entry {missing})")
            continue
        saved = {}
        for e in entries:
            getattr(C, e)  # materialise the checked wrapper
            saved[e] = C.__dict__.get(e)
            setattr(C, e, lambda *a, **k: 0)
        try:
            t = timed()
        finally:
            for e, fn in saved.items():
                if fn is None:
                    delattr(C, e)
                else:
                    setattr(C, e, fn)
        print(f"{fam:22s}  {t:8.3f} ms/step   in-situ cost {base - t:7.3f} ms  ({(base - t) / base * 100:5.1f} %)")
    print(f"baseline again          {timed():8.3f} ms/step")


if __name__ == "__main__":
    main()
