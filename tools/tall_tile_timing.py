"""128-row against 256-row forward GEMM tiles on the single-pass dgrad shapes of the B = 64 step (CUDA events).

Loads two builds of libgdrn_b200.so side by side: BASE, whose launches all run on 128-row tiles, and NEW (default: the library
of this tree), which picks 256-row tiles for these shapes (pick_block_m, gemm_fwd.cu).  Each shape is launched from both
libraries on the same operands, alternating windows of --iters launches (A, B, A, B, ...), and the outputs are compared bit for
bit.  Prints the card's name, power limit and SM clock, then per shape the tile height each library used, the median window
time per launch and the executed TFLOP/s.

usage: python tools/tall_tile_timing.py BASE_LIB [--new NEW_LIB] [--windows 5] [--iters 50]"""
import argparse
import ctypes
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VP, I = ctypes.c_void_p, ctypes.c_int

# (name, kind, shape): conv (N, H, W, Cin, Cout, k) with pad k // 2, or gemm (M, N, K)
SHAPES = [
    ("head 64^2 dgrad 3x3 256->256", "conv", (64, 64, 64, 256, 256, 3)),
    ("head 32^2 dgrad 3x3 256->256", "conv", (64, 32, 32, 256, 256, 3)),
    ("head 16^2 / layer3 dgrad 3x3 256->256", "conv", (64, 16, 16, 256, 256, 3)),
    ("layer2 dgrad 3x3 128->128", "conv", (64, 32, 32, 128, 128, 3)),
    ("head output-conv dgrad gemm", "gemm", (262144, 256, 128)),
]


def smi(query):
    r = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unavailable"


def load(path):
    dll = ctypes.CDLL(os.path.abspath(path), mode=ctypes.RTLD_LOCAL)
    dll.gdrn_conv_fwd.argtypes = [VP] * 11 + [I] * 13 + [VP]
    dll.gdrn_gemm_fwd.argtypes = [VP] * 9 + [I] * 7 + [VP]
    dll.gdrn_last_error.restype = ctypes.c_char_p
    return dll


def block_m(dll):
    return dll.gdrn_last_gemm_block_m() if hasattr(dll, "gdrn_last_gemm_block_m") else 128


def operands(kind, shape, dtype, gen):
    if kind == "conv":
        n, h, w, cin, cout, k = shape
        a = torch.randn((n, h, w, cin), device="cuda", generator=gen).to(dtype)
        wt = (torch.randn((cout, k * k * cin), device="cuda", generator=gen) / (k * k * cin) ** 0.5).to(dtype)
        rows, cols, depth = n * h * w, cout, k * k * cin
    else:
        rows, cols, depth = shape
        a = torch.randn((rows, depth), device="cuda", generator=gen).to(dtype)
        wt = (torch.randn((cols, depth), device="cuda", generator=gen) / depth ** 0.5).to(dtype)
    bias = torch.randn(cols, device="cuda", generator=gen)
    return a, wt, bias, rows, cols, depth


def launcher(dll, kind, shape, a, wt, bias, out):
    stream = VP(torch.cuda.current_stream().cuda_stream)
    if kind == "conv":
        n, h, w, cin, cout, k = shape
        args = (a.data_ptr(), None, wt.data_ptr(), None, out.data_ptr(), None, None, bias.data_ptr(), None, None, None,
                n, h, w, cin, cout, cout, k, k, 1, k // 2, cout, 1, 1, stream)
        fn = dll.gdrn_conv_fwd
    else:
        m, ncol, kdim = shape
        args = (a.data_ptr(), None, wt.data_ptr(), None, out.data_ptr(), None, None, bias.data_ptr(), None, m, ncol, ncol, kdim,
                ncol, 1, 1, stream)
        fn = dll.gdrn_gemm_fwd

    def run():
        if fn(*args) != 0:
            raise RuntimeError(dll.gdrn_last_error().decode())

    return run


def time_window(run, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        run()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("base")
    ap.add_argument("--new", default=os.path.join(ROOT, "gdr_net_b200", "lib", "libgdrn_b200.so"))
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("tall_tile_timing needs a GPU")
    torch.cuda.init()
    libs = {"A": load(args.base), "B": load(args.new)}
    dtype = torch.float16 if libs["B"].gdrn_storage_format() else torch.bfloat16
    print(f"gpu: {smi('name')}, power limit {smi('power.limit')}, max SM clock {smi('clocks.max.sm')}", flush=True)
    print(f"A = {args.base}\nB = {args.new}")
    gen = torch.Generator(device="cuda").manual_seed(0)
    ok = True
    for name, kind, shape in SHAPES:
        a, wt, bias, rows, cols, depth = operands(kind, shape, dtype, gen)
        flop = 2.0 * rows * cols * depth
        outs, runs, bm = {}, {}, {}
        for tag, dll in libs.items():
            outs[tag] = torch.empty((rows, cols), dtype=dtype, device="cuda")
            runs[tag] = launcher(dll, kind, shape, a, wt, bias, outs[tag])
            runs[tag]()  # warm-up: module load, tensor-map encode
            bm[tag] = block_m(dll)
            time_window(runs[tag], max(1, args.iters // 5))
        same = torch.equal(outs["A"].view(torch.int16), outs["B"].view(torch.int16))
        ok &= same
        ms = {"A": [], "B": []}
        for _ in range(args.windows):
            for tag in ("A", "B"):
                ms[tag].append(time_window(runs[tag], args.iters))
        med = {t: statistics.median(v) for t, v in ms.items()}
        print(f"{name:40s} M {rows:7d} N {cols:4d} K {depth:5d} | A {bm['A']}-row {med['A'] * 1e3:8.1f} us "
              f"{flop / med['A'] / 1e9:6.1f} TF/s | B {bm['B']}-row {med['B'] * 1e3:8.1f} us {flop / med['B'] / 1e9:6.1f} TF/s | "
              f"B/A {med['B'] / med['A']:.3f} | B faster in every window: {max(ms['B']) < min(ms['A'])} | bit-identical: {same}",
              flush=True)
        del a, wt, bias, outs
    print(f"SM clock now {smi('clocks.sm')}")
    if not ok:
        sys.exit("outputs differ")


if __name__ == "__main__":
    main()
