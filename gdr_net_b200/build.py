"""In-tree build of libgdrn_b200.so (hand-written sm_90a CUDA behind a C ABI).

    python -m gdr_net_b200.build            # incremental
    python -m gdr_net_b200.build --force

nvcc cross-compiles for sm_90a (H100) without a GPU.  Objects go to gdr_net_b200/_build/, the shared
library to gdr_net_b200/lib/ (both git-ignored build products).
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
BUILD = os.path.join(HERE, "_build")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libgdrn_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC",
    "-diag-suppress", "550",
    # 16-bit storage format of the activation / weight planes: 1 = fp16 (11-bit mantissa, TF32-equivalent; default),
    # 0 = bf16.  See csrc/ptx.cuh.
    "-DGDRN_STORE_F16=" + os.environ.get("GDRN_STORE_F16", "1"),
]


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest(paths):
    h = hashlib.sha256()
    for p in paths:
        with open(p, "rb") as f:
            h.update(f.read())
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(BUILD, exist_ok=True)
    os.makedirs(LIBDIR, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith((".h", ".cuh"))]
    jobs = []
    objs = []
    for src in _sources():
        sp = os.path.join(CSRC, src)
        obj = os.path.join(BUILD, src[:-3] + ".o")
        stamp = obj + ".sha"
        dig = _digest([sp] + headers)
        objs.append(obj)
        if not force and os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == dig:
            continue
        jobs.append((sp, obj, stamp, dig))

    def compile_one(job):
        sp, obj, stamp, dig = job
        cmd = [NVCC] + FLAGS + ["-I", CSRC, "-c", sp, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {sp}:\n{r.stdout}\n{r.stderr}")
        if verbose and (r.stdout or r.stderr):
            print(r.stdout, r.stderr)
        with open(stamp, "w") as f:
            f.write(dig)

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            list(ex.map(compile_one, jobs))
    if jobs or force or not os.path.exists(LIB):
        # link to a temporary name and rename atomically: a concurrent reader (a gpurun snapshot, another process importing
        # the package) must never see a half-written library
        tmp = LIB + f".tmp{os.getpid()}"
        cmd = [NVCC, "-shared", "-o", tmp] + objs + ["-cudart", "shared", "-Xlinker", "-rpath,/usr/local/cuda/lib64"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
        os.replace(tmp, LIB)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
