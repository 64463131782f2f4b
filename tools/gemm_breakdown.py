"""Per-launch timing of every wgmma GEMM/conv launch in one B=64 train step (CUDA events), with algorithmic TFLOP/s."""
import os, sys, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench
from gdr_net_b200 import ops, synth

def main():
    precision = sys.argv[1] if len(sys.argv) > 1 else "half"
    model, _ = bench.build(precision)
    eng = model.engine
    dev = torch.device("cuda")
    batch = bench.device_batch(synth.make_batch(64, seed=100), dev)
    x = batch["roi_img"].float().contiguous()
    aux = {k: (v.float().contiguous() if isinstance(v, torch.Tensor) and v.dtype != torch.long else v) for k, v in bench.aux_from_batch(batch).items()}
    gl = torch.ones(8, device=dev)
    recs = []
    orig = {n: getattr(ops, n) for n in ("conv_fwd", "gemm_fwd", "conv_wgrad", "gemm_wgrad")}
    def wrap(name, fn, desc):
        def w(*a, **k):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); r = fn(*a, **k); e1.record()
            recs.append((name, desc(*a, **k), e0, e1)); return r
        return w
    def d_conv(x_, wp, Cout, KH, KW, stride, pad, **k):
        N, H, W, Cin = x_.shape
        return (f"{H}x{W} {Cin}->{Cout} k{KH} s{stride}" + (" zi" if k.get("algo_scale", 1) != 1 else ""), 2.0 * N * (H // stride) * (W // stride) * Cout * Cin * KH * KW * k.get("algo_scale", 1.0))
    def d_gemm(a, wp, N, **k):
        return (f"gemm M{a.shape[0]} N{N} K{a.shape[1]}", 2.0 * a.shape[0] * N * a.shape[1])
    def d_cw(dy, x_, ws, Cout, KH, KW, stride, pad, ksplit=0):
        N, H, W, Cin = x_.shape
        return (f"{H}x{W} {Cin}->{Cout} k{KH} s{stride}", 2.0 * N * (H // stride) * (W // stride) * Cout * Cin * KH * KW)
    def d_gw(dy, x_, ws, ksplit=0):
        return (f"gemm P{dy.shape[0]} M{dy.shape[1]} N{x_.shape[1]}", 2.0 * dy.shape[0] * dy.shape[1] * x_.shape[1])
    ops.conv_fwd = wrap("conv_fwd", orig["conv_fwd"], d_conv); ops.gemm_fwd = wrap("gemm_fwd", orig["gemm_fwd"], d_gemm)
    ops.conv_wgrad = wrap("conv_wgrad", orig["conv_wgrad"], d_cw); ops.gemm_wgrad = wrap("gemm_wgrad", orig["gemm_wgrad"], d_gw)
    for it in range(3):
        recs.clear()
        eng.forward(x, aux, train_bn=True, do_loss=True); eng.backward(gl)
    torch.cuda.synchronize()
    agg = {}
    for name, (desc, fl), a, b in recs:
        key = (name, desc)
        d = agg.setdefault(key, [0, 0.0, 0.0]); d[0] += 1; d[1] += a.elapsed_time(b); d[2] += fl
    tot = sum(v[1] for v in agg.values())
    print(f"{'op':11s} {'shape':34s} {'n':>3s} {'ms':>8s} {'TF/s':>8s} {'share':>6s}")
    for (name, desc), v in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print(f"{name:11s} {desc:34s} {v[0]:3d} {v[1]:8.3f} {v[2]/v[1]/1e9:8.1f} {v[1]/tot:6.3f}")
    print("total ms", round(tot, 3), "TF/s", round(sum(v[2] for v in agg.values()) / tot / 1e9, 1))

if __name__ == "__main__":
    main()
