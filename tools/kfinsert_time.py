"""Times the keyframe insertion (b2s_process_new_keyframe) and the standalone UpdateNormalAndDepth on the GPU: device
time (CUDA events on the matcher's stream, upload to download), the host wall time of the call, and, where
oracle/_ref is built, the reference's own ProcessNewKeyFrame + MapPointCulling on one CPU thread (the association and
culling alone, timed inside the glue).  Prints one JSON line per case.

  python tools/kfinsert_time.py [--reps 20]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import numpy as np  # noqa: E402

import kfinsert_binding as kb  # noqa: E402

pkg = kb.pkg


def stats(xs):
    xs = np.sort(np.asarray(xs))
    return {"median": float(np.median(xs)), "p10": float(xs[int(0.1 * (len(xs) - 1))]),
            "p90": float(xs[int(0.9 * (len(xs) - 1))])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    if pkg.device_count() < 1:
        sys.exit("kfinsert_time: no CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    m = pkg.ORBmatcher(max_features=64)
    ref = kb.Reference() if os.path.exists(kb.REF_LIB) else None
    for slots in (500, 2000):
        for batch in (1, 32):
            ds = [kb.scene(1000 + i, n_kf=40, n_slots=slots, mono=False, n_recent=slots // 2) for i in range(batch)]
            for _ in range(3):
                m.ProcessNewKeyFrame(ds)
            dev, wall = [], []
            for _ in range(a.reps):
                t0 = time.perf_counter()
                m.ProcessNewKeyFrame(ds)
                wall.append((time.perf_counter() - t0) * 1e3)
                dev.append(m.last_ms())
            row = {"case": "ProcessNewKeyFrame+MapPointCulling", "slots": slots, "batch": batch,
                   "device_ms": stats(dev), "host_wall_ms": stats(wall), "gpu": gpu}
            if ref is not None:
                row["reference_cpu_ms_per_keyframe"] = stats([ref(ds[0])["wall_ns"] * 1e-6 for _ in range(5)])
            print(json.dumps(row), flush=True)
    for n_mp in (10000, 100000):
        d = kb.normal_depth_scene(7, n_mp=n_mp, n_kf=300)
        for _ in range(3):
            m.UpdateNormalAndDepth(d)
        dev, wall = [], []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            m.UpdateNormalAndDepth(d)
            wall.append((time.perf_counter() - t0) * 1e3)
            dev.append(m.last_ms())
        print(json.dumps({"case": "UpdateNormalAndDepth", "points": n_mp, "device_ms": stats(dev),
                          "host_wall_ms": stats(wall), "gpu": gpu}), flush=True)


if __name__ == "__main__":
    main()
