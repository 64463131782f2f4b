"""Experiment: fp32 accumulation behaviour of the GEMM kernels' tensor-core MMAs (bias / growth with K) vs fp64 truth."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from gdr_net_b200 import ops
torch.backends.cuda.matmul.allow_tf32 = False
for dist in ("uniform01", "normal"):
    for K in (64, 256, 1024, 4096, 16384, 65536):
        M, N = 256, 128
        g = torch.Generator(device="cuda").manual_seed(K)
        if dist == "uniform01":
            a = torch.rand(M, K, device="cuda", generator=g); w = torch.rand(N, K, device="cuda", generator=g)
        else:
            a = torch.randn(M, K, device="cuda", generator=g); w = torch.randn(N, K, device="cuda", generator=g)
        for planes in (1, 2):
            ae = a.bfloat16().float() if planes == 1 else a
            we = w.bfloat16().float() if planes == 1 else w
            ref = ae.double() @ we.double().t()
            out = torch.zeros(M, N, device="cuda")
            ops.gemm_fwd(ops.PT.from_float(a, planes), ops.pack_linear(w, planes), N, out_f32=out, want_planes=False)
            t32 = ae @ we.t()
            scale = ref.abs().mean()
            e = (out.double() - ref)
            et = (t32.double() - ref)
            print(f"{dist:9s} K={K:6d} planes={planes}  ours: rms {float(e.pow(2).mean().sqrt()/scale):.2e} bias {float(e.mean()/scale):+.2e}"
                  f"   torch-fp32: rms {float(et.pow(2).mean().sqrt()/scale):.2e} bias {float(et.mean()/scale):+.2e}")
