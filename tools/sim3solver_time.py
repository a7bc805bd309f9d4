"""Device time of the Sim3 RANSAC (b2s_sim3solver_iterate) per call, against the reference's own Sim3Solver on the CPU
(oracle/_ref/libref_sim3solver.so: src/Sim3Solver.cc compiled in place against the cv2-pinned stand-in, one thread).

For batch 1 / 16 / 256 solvers of 50 / 200 / 800 correspondences (30 % true matches, so few calls return early), it
times iterate(5) (LoopClosing::ComputeSim3's call) and find() (300 iterations).  Device time is the CUDA-event time of
the call (upload, three launches, download), median of the repetitions; the CPU column is one reference solver's call.
Prints one JSON line per configuration.

    python tools/sim3solver_time.py [--reps 20]
"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import sim3solver_binding as sb  # noqa: E402
from synth_sim3solver import problem, scene  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    pkg = importlib.import_module("self_commit_orb-slam2_b200")
    if pkg.device_count() < 1:
        raise SystemExit("no CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    handle = pkg.Sim3SolverBatch(max_matches=1024, max_sets=300, max_batch=256)
    for n in (50, 200, 800):
        scenes = [scene(n=n, inliers=0.3, seed=100 + i, skips=0.0) for i in range(16)]
        probs = [problem(sc, 20) for sc in scenes]
        for mode in ("iterate5", "find"):
            ref_ms = []
            if os.path.exists(sb.REF_LIB):
                for sc in scenes[:4]:
                    for rep in range(3):
                        r = sb.RefSolver(sb.REF_LIB, sc)
                        r.set_ransac_parameters(0.99, 20, 300)
                        r.srand(rep)
                        t0 = time.perf_counter()
                        r.iterate(5 if mode == "iterate5" else None)
                        ref_ms.append((time.perf_counter() - t0) * 1e3)
                        r.close()
            for batch in (1, 16, 256):
                rng = np.random.default_rng(batch)
                solvers, sets = [], []
                for i in range(batch):
                    pr = probs[i % len(probs)]
                    sv = handle.solver(pr["X1c"], pr["X2c"], pr["sigma2_1"], pr["sigma2_2"], pr["K1"], pr["K2"],
                                       fix_scale=False)
                    sv.set_ransac_parameters(0.99, 20, 300)
                    nN = len(pr["X1c"])
                    solvers.append(sv)
                    sets.append(np.array([rng.choice(nN, 3, replace=False) for _ in range(300)], np.int32))
                nit = 5 if mode == "iterate5" else 300
                ms = []
                for rep in range(args.reps + 2):
                    for sv in solvers:
                        sv.iterations, sv.best_inliers = 0, 0
                    pkg.Sim3Solver.iterate_batch(solvers, [nit] * batch, sets, handle=handle)
                    if rep >= 2:
                        ms.append(handle.last_ms())
                row = dict(n=n, mode=mode, batch=batch, device_ms=float(np.median(ms)),
                           device_us_per_solver=float(np.median(ms)) * 1e3 / batch,
                           ref_cpu_ms_per_solver=float(np.median(ref_ms)) if ref_ms else None, gpu=gpu)
                print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
