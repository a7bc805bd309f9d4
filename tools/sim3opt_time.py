"""Times OptimizeSim3: the device (b2s_sim3opt_last_ms: upload, one launch, download) for batches of 1, 64 and 1,024
problems of 50, 200 and 800 candidate matches, and the reference's own function on one CPU thread
(oracle/_ref/libref_sim3opt.so, when it was built) at the same sizes, each with its spread over repeats.  Prints the
card's name and power limit.  Usage: python tools/sim3opt_time.py [--repeats R]"""
import argparse
import ctypes
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import sim3_binding as sb  # noqa: E402
from synth_sim3 import flatten, synth_sim3  # noqa: E402


def spread(xs):
    xs = np.asarray(xs)
    return "median %.3f [min %.3f, max %.3f]" % (np.median(xs), xs.min(), xs.max())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=7)
    args = ap.parse_args()
    import importlib
    pkg = importlib.import_module("self_commit_orb-slam2_b200")
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                         capture_output=True, text=True).stdout.strip())
    sizes = (50, 200, 800)
    opt = pkg.Sim3Optimizer(max_matches=1024, max_batch=1024)
    for n in sizes:
        pool = [flatten(synth_sim3(n=n, seed=1000 + i, mono=bool(i % 2), outliers=0.2))[0] for i in range(64)]
        for batch in (1, 64, 1024):
            ds = [pool[i % len(pool)] for i in range(batch)]
            opt.OptimizeSim3Batch(ds)  # warm-up
            ms, trials = [], 0
            for _ in range(args.repeats):
                opt.OptimizeSim3Batch(ds)
                t, trials = opt.last_ms()
                ms.append(t)
            print("device  matches %4d  batch %4d  ms/call %s  us/problem %.1f  LM trials/problem %.1f" %
                  (n, batch, spread(ms), 1e3 * np.median(ms) / batch, trials / batch))
    if not os.path.exists(sb.REF_LIB):
        print("reference: not measured (oracle/_ref/libref_sim3opt.so not built)")
        return
    ref = ctypes.CDLL(sb.REF_LIB).ref_optimize_sim3
    for n in sizes:
        scenes = [synth_sim3(n=n, seed=1000 + i, mono=bool(i % 2), outliers=0.2) for i in range(16)]
        sb.call_graph(ref, scenes[0])
        per = []
        for _ in range(args.repeats):
            t0 = time.perf_counter()
            for sc in scenes:
                sb.call_graph(ref, sc)
            per.append((time.perf_counter() - t0) * 1e3 / len(scenes))
        print("reference (one CPU thread, object graph included)  matches %4d  ms/problem %s" % (n, spread(per)))


if __name__ == "__main__":
    main()
