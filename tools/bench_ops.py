"""Micro-benchmark of the wgmma conv kernels on the GDR-Net layer shapes (B=64), CUDA-event timed."""
import json
import sys
import os

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from gdr_net_b200 import ops

SHAPES = [  # name, N, H, W, Cin, Cout, k, stride, pad
    ("layer1 3x3 64->64 @64", 64, 64, 64, 64, 64, 3, 1, 1),
    ("layer2 3x3 128->128 @32", 64, 32, 32, 128, 128, 3, 1, 1),
    ("layer3 3x3 256->256 @16", 64, 16, 16, 256, 256, 3, 1, 1),
    ("layer4 3x3 512->512 @8", 64, 8, 8, 512, 512, 3, 1, 1),
    ("head 3x3 256->256 @32", 64, 32, 32, 256, 256, 3, 1, 1),
    ("head 3x3 256->256 @64", 64, 64, 64, 256, 256, 3, 1, 1),
    ("layer2.0 3x3 s2 64->128", 64, 64, 64, 64, 128, 3, 2, 1),
    ("head 1x1 256->69 @64", 64, 64, 64, 256, 69, 1, 1, 0),
]


def timeit(fn, iters=10, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def main():
    planes_list = [1, 2] if "--x3" in sys.argv else [1]
    rows = []
    for planes in planes_list:
        for name, N, H, W, Cin, Cout, k, stride, pad in SHAPES:
            x = ops.PT((N, H, W, Cin), planes)
            x.buf.normal_()
            w = torch.randn(Cout, Cin, k, k, device="cuda") * 0.05
            wp = ops.pack_conv_fwd(w, planes)
            Ho, Wo = H // stride, W // stride
            ldc = (Cout + 63) // 64 * 64
            out = ops.PT((N, Ho, Wo, ldc), planes)
            stats = torch.zeros(2, Cout, device="cuda")
            flops = 2.0 * N * Ho * Wo * Cout * Cin * k * k
            t = timeit(lambda: ops.conv_fwd(x, wp, Cout, k, k, stride, pad, out=out, stats=stats))
            row = dict(op="fwd", planes=planes, shape=name, ms=round(t, 4), tflops=round(flops / t / 1e9, 1))
            rows.append(row)
            print(row, flush=True)
            dy = ops.PT((N, Ho, Wo, ldc), planes)
            dy.buf.normal_()
            ws = ops.Workspace()
            t = timeit(lambda: ops.conv_wgrad(dy, x, ws, Cout, k, k, stride, pad))
            row = dict(op="wgrad", planes=planes, shape=name, ms=round(t, 4), tflops=round(flops / t / 1e9, 1))
            rows.append(row)
            print(row, flush=True)
    os.makedirs("gpurun_out", exist_ok=True)
    json.dump(rows, open("gpurun_out/bench_ops.json", "w"), indent=1)


if __name__ == "__main__":
    main()
