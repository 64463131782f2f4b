"""A/B of two builds of libgdrn_b200.so on the flagship step: alternates `bench.py --quick` runs with GDRN_LIB_PATH pointing at
library A and at library B (A, B, A, B, ...), so slow drifts of clock, temperature and neighbouring load fall on both alike.
Prints every window as it finishes, then the medians and ranges of each library and the card's name, power limit and SM clock.

usage: python tools/ab_libs.py LIB_A LIB_B [--windows 6] [--steps 30] [--warmup 5] [--json OUT]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def smi(query):
    r = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unavailable"


def window(lib, steps, warmup):
    env = dict(os.environ, GDRN_LIB_PATH=os.path.abspath(lib))
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--quick", "--steps", str(steps), "--warmup", str(warmup)]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, cwd=ROOT)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    if r.returncode != 0 or not lines:
        raise RuntimeError(f"bench.py failed with {lib} (exit {r.returncode}):\n{r.stdout[-2000:]}\n{r.stderr[-4000:]}")
    out = json.loads(lines[-1])
    return out["ms_per_step"], out["value"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("lib_a")
    ap.add_argument("lib_b")
    ap.add_argument("--windows", type=int, default=6, help="windows per library")
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--json", default=None, help="also write the windows and medians to this file")
    args = ap.parse_args()
    for lib in (args.lib_a, args.lib_b):
        if not os.path.exists(lib):
            sys.exit(f"no such library: {lib}")
    gpu = {"name": smi("name"), "power_limit": smi("power.limit"), "sm_clock_max": smi("clocks.max.sm")}
    print(f"gpu: {gpu['name']}, power limit {gpu['power_limit']}, max SM clock {gpu['sm_clock_max']}", flush=True)
    names = {"A": args.lib_a, "B": args.lib_b}
    ms = {"A": [], "B": []}
    for w in range(args.windows):
        for tag in ("A", "B"):
            t, crops = window(names[tag], args.steps, args.warmup)
            ms[tag].append(t)
            print(f"window {w} {tag} {os.path.basename(names[tag])}: {t:.3f} ms/step  {crops:.1f} crops/s  "
                  f"(SM clock now {smi('clocks.sm')})", flush=True)
    res = {"gpu": gpu, "steps": args.steps, "libs": names, "ms_per_step": ms, "sm_clock_end": smi("clocks.sm")}
    for tag in ("A", "B"):
        v = ms[tag]
        res[f"median_{tag}"] = statistics.median(v)
        print(f"{tag} {os.path.basename(names[tag])}: median {statistics.median(v):.3f} ms/step, range {min(v):.3f}-{max(v):.3f}")
    gain = (res["median_A"] - res["median_B"]) / res["median_A"]
    res["b_faster_in_every_window"] = max(ms["B"]) < min(ms["A"])
    print(f"B vs A: {100 * gain:+.2f} % of A's median step time faster; every B window faster than every A window: "
          f"{res['b_faster_in_every_window']}")
    print(f"SM clock at the end: {res['sm_clock_end']}")
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
