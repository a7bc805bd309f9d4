"""Times the essential-graph optimisation (pkg.EssentialGraphOptimizer, csrc/essential.cu) on seeded loop-closing maps
of 250, 1,000 and 4,096 keyframes: device time (CUDA events over the solver's stream segments), host wall time of the
whole call, and the reference's own Optimizer::OptimizeEssentialGraph on one CPU thread (oracle/_ref/
libref_essential.so, where it was built) at the sizes where its dense stand-in storage fits.  Prints the card's name and
power limit from the same run.  Usage: python tools/essential_time.py [--ref-max 1000] [--repeats 3]"""
import argparse
import ctypes
import importlib
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import eg_binding as eb  # noqa: E402
from synth_essential import synth_essential  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="250,1000,4096")
    ap.add_argument("--ref-max", type=int, default=1000)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    pkg = importlib.import_module("self_commit_orb-slam2_b200")
    if pkg.device_count() < 1:
        raise SystemExit("no CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    print("card:", q)
    opt = pkg.EssentialGraphOptimizer()
    ref = ctypes.CDLL(eb.REF_LIB) if os.path.exists(eb.REF_LIB) else None
    print("| keyframes | edges | LM trials | device ms | host wall ms | reference ms (1 CPU thread) |")
    print("|---|---|---|---|---|---|")
    for n in [int(x) for x in a.sizes.split(",")]:
        m = synth_essential(n_kf=n, n_mp=25 * n, seed=n, mono=True, closures=3)
        d, _, _ = eb.flatten(m)
        opt.OptimizeEssentialGraph(d)  # warm-up: module load, tile storage
        dev, wall = [], []
        for _ in range(a.repeats):
            t = time.perf_counter()
            out = opt.OptimizeEssentialGraph(d)
            wall.append((time.perf_counter() - t) * 1e3)
            dev.append(opt.last_ms()[0])
        rms = "not measured"
        if ref is not None and n <= a.ref_max:
            t = time.perf_counter()
            eb.call_map(ref.ref_essential_graph, m)
            rms = "%.0f" % ((time.perf_counter() - t) * 1e3)
        print("| %d | %d | %d | %.1f | %.1f | %s |" % (n, len(d["edges"]), out["n_trials"], min(dev), min(wall), rms))


if __name__ == "__main__":
    main()
