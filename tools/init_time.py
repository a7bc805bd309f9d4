"""Times the monocular initialiser (b2s_initialize): batch 1 and batch 64, 200 iterations, about 150, 600 and 1,500
matches among 2,000 keypoints per frame, planar and general scenes; and, on the CPUs of the same machine, the
reference's own Initialize (oracle/_ref/libref_init.so: src/Initializer.cc compiled in place, H and F on its two
std::threads, its own draws) and the CPU restatement (oracle/liborb_init.so, one thread) on the same problems.  Prints the card and its
power limit with the numbers, and one JSON line per configuration.

    python tools/init_time.py [--reps 20]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import init_binding as ib  # noqa: E402
from synth_init import synth_init  # noqa: E402


def problem(n, seed, kind):
    # 2,000 keypoints per frame: n matched, the rest unmatched
    return synth_init(n=n, seed=seed, kind=kind, outliers=0.2, extra=(2000 - n) / n, iterations=200)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    import importlib
    pkg = importlib.import_module("self_commit_orb-slam2_b200")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print("device:", q)
    ini = pkg.MonoInitializer(max_keys=2048, max_iterations=200, max_batch=64)
    for kind in ("planar", "general"):
        for n in (150, 600, 1500):
            ds = [problem(n, 1000 + s, kind) for s in range(64)]
            for batch in (1, 64):
                work = ds[:batch]
                for _ in range(3):
                    ini.InitializeBatch(work)
                ms = []
                for _ in range(args.reps):
                    ini.InitializeBatch(work)
                    ms.append(ini.last_ms())
                t0 = time.perf_counter()
                for d in work[:8]:
                    ib.oracle(d)
                cpu_ms = (time.perf_counter() - t0) / min(batch, 8) * 1e3
                ref_ms = None
                if os.path.exists(ib.REF_LIB):
                    t0 = time.perf_counter()
                    for d in work[:8]:
                        ib.call_initialize(ib.REF_LIB, "ref_initialize", d)
                    ref_ms = (time.perf_counter() - t0) / min(batch, 8) * 1e3
                rec = dict(kind=kind, matches=n, keypoints=2000, iterations=200, batch=batch,
                           device_ms_median=float(np.median(ms)), device_ms_per_problem=float(np.median(ms)) / batch,
                           reference_ms_per_problem=ref_ms, cpu_oracle_ms_per_problem=cpu_ms, device=q)
                print(json.dumps(rec), flush=True)
    ini.close()


if __name__ == "__main__":
    main()
