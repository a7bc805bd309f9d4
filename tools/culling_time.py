"""Times b2s_keyframe_culling (pkg.KeyFrameCulling) against the reference's own LocalMapping::KeyFrameCulling
(oracle/_ref/libref_localmapping.so, with its real SetBadFlag) on one CPU thread of the same machine.

Local lists of about 30, 100 and 300 keyframes with about 2,000 slots each, stereo and monocular, on paths where each
point is seen by a run of 2-12 keyframes.  Batches of 1 (one LocalMapping iteration) and 32 (32 copies of the same
problem: independent local maps of the same size).  Reported: device time (CUDA events: upload, kernels, download) and
host wall time of the library call (validation, packing, device work, unpacking), medians of 20 after warm-up; the
reference's time is the median wall time of its KeyFrameCulling alone (times 32 for a batch of 32), without building the
object graph.  The device result is checked against the reference's and the restatement's before timing.

  python tools/culling_time.py [--out FILE]"""
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
import culling_binding as cb  # noqa: E402


def gpu_info():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    pkg = cb.pkg
    h = pkg.KeyFrameCulling(max_kf=512, max_mp=1 << 18, max_obs=1 << 21, max_local=320, max_slots=1 << 20,
                            max_batch=32)
    ref, orc = cb.Reference(), cb.Oracle()
    rows = []
    for size in (30, 100, 300):
        for mono in (False, True):
            w = cb.trajectory(seed=size + mono, n_kf=size + 1, pts_per_kf=300, stereo=not mono)
            rng = np.random.default_rng(size)
            cur = size
            local = cb.local_list(w, rng, cur, size=size)
            d = w.problem(local, monocular=mono)
            slots = int(d["slot_off"][-1]) / size
            want = ref(w, d, cur)
            got = h(d)
            cb.same(want, got, counts=False)
            cb.same(orc(d), got)
            ref_ns = [ref(w, d, cur)["wall_ns"] for _ in range(max(3, args.reps // 4))]
            for B in (1, 32):
                ds = [d] * B
                for _ in range(3):
                    h(ds)
                dev, wall = [], []
                for _ in range(args.reps):
                    t0 = time.perf_counter()
                    h(ds)
                    wall.append((time.perf_counter() - t0) * 1e3)
                    dev.append(h.last_ms())
                row = {"local": size, "mode": "monocular" if mono else "stereo", "batch": B,
                       "slots_per_kf": round(slots), "culled": int(got["n_culled"]),
                       "device_ms": round(float(np.median(dev)), 4), "host_wall_ms": round(float(np.median(wall)), 4),
                       "reference_ms": round(float(np.median(ref_ns)) * 1e-6 * B, 4)}
                rows.append(row)
                print(json.dumps(row), flush=True)
    res = {"gpu": gpu_info(), "rows": rows}
    print(json.dumps({"gpu": res["gpu"]}))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
