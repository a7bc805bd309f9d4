"""Times the global bundle adjustment (Optimizer::GlobalBundleAdjustemnt as LoopClosing runs it: 10 iterations, no robust
kernel, nLoopKF > 0) on the device against the reference's own src/Optimizer.cc + g2o on one CPU thread
(oracle/_ref/libref_gba.so, built by build() where the reference's sources are present), on closed-loop stereo maps
(tests/synth_gba.py synth_global_ba) of about 100, 300 and 1,000 keyframes and the largest supported size (2,048 keyframes).

Per map size it prints one JSON line: the device time of the call (CUDA events around its stream segments, the host's LM
decisions between trials excluded), the host wall time of the whole call (upload, structure, LM loop, write-back), the LM
trials, and the reference's wall time where it runs (sizes up to --ref-max keyframes), as medians over --reps calls,
with the card's name and power limit.

    python tools/gba_time.py [--sizes 100,300,1000,2048] [--reps 3] [--ref-max 100] [--out DIR/gba_time.jsonl]"""
import argparse
import ctypes
import importlib
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402

import gba_binding as gb  # noqa: E402
from synth_gba import synth_global_ba  # noqa: E402


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        name, power = [s.strip() for s in out.splitlines()[0].split(",")]
        return name, power
    except Exception as e:  # the numbers are still device events; say where they came from
        return "unknown (%s)" % e, "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="100,300,1000,2048")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ref-max", type=int, default=100)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    pkg = importlib.import_module("self_commit_orb-slam2_b200")
    ref = ctypes.CDLL(gb.REF_LIB) if os.path.exists(gb.REF_LIB) else None
    name, power = card()
    opt = pkg.GlobalOptimizer(max_kf=2048, max_mp=262144, max_edges=1 << 21)
    lines = []
    for n in [int(s) for s in a.sizes.split(",")]:
        m = synth_global_ba(n_kf=n, n_mp=min(100 * n, 200000), obs_range=(2, 10), seed=n, pert_deg=0.1, pert_t=0.02)
        d, _, _ = gb.flatten(m)
        opt.BundleAdjustment(d, iterations=10, robust=False)  # warm-up: grows the reduced-system storage
        dev, wall, trials = [], [], []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            opt.BundleAdjustment(d, iterations=10, robust=False)
            wall.append((time.perf_counter() - t0) * 1e3)
            ms, tr = opt.last_ms()
            dev.append(ms)
            trials.append(tr)
        row = dict(n_kf=n, n_mp=len(d["points"]), n_edges=len(d["edges"]), lm_trials=int(np.median(trials)),
                   device_ms=float(np.median(dev)), device_ms_min=float(np.min(dev)), device_ms_max=float(np.max(dev)),
                   host_wall_ms=float(np.median(wall)), reps=a.reps, card=name, power_limit=power)
        if ref is not None and n <= a.ref_max:
            rw = []
            for _ in range(max(1, min(a.reps, 2))):
                t0 = time.perf_counter()
                gb.call_map(ref.ref_global_ba, m, 10, False, n - 1)
                rw.append((time.perf_counter() - t0) * 1e3)
            row["reference_ms_1thread"] = float(np.median(rw))
        print(json.dumps(row), flush=True)
        lines.append(row)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
