"""Times b2s_undistort_keypoints_device and b2s_stereo_from_depth_device on the GPU (CUDA events around `reps` launches on
one stream, 2,000 records per image, batch 1 and 32) and, on the same run, the host path a caller has without them:
cv2.undistortPoints on the same keypoints plus the ComputeStereoFromRGBD gather (numpy) on one CPU thread.  Prints one
JSON line per batch with the card's name and power limit.

  python tools/undistort_time.py [--reps 200]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import importlib  # noqa: E402

import numpy as np  # noqa: E402

import undistort_binding as ub  # noqa: E402

pkg = importlib.import_module("self_commit_orb-slam2_b200")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    a = ap.parse_args()
    if pkg.device_count() < 1:
        sys.exit("undistort_time: no CUDA device")
    import cv2
    import torch
    cv2.setNumThreads(1)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    w, h, cap = 640, 480, 2000
    K4, dist = ub.calib("tum1")
    ex = pkg.ORBextractor(1000, 1.2, 8, 20, 7, max_width=w, max_height=h)
    s = torch.cuda.Stream()
    for B in (1, 32):
        rng = np.random.default_rng(B)
        rec = np.zeros((B, cap), ub.kp_dtype)
        rec["x"], rec["y"] = rng.uniform(0, w - 1, (B, cap)), rng.uniform(0, h - 1, (B, cap))
        depth_h = np.stack([ub.depth_image(w, h, seed=b) for b in range(B)])
        kps = torch.from_numpy(rec.view(np.uint8).reshape(B, cap, 28)).cuda()
        counts = torch.full((B,), cap, dtype=torch.int32, device="cuda")
        depth = torch.from_numpy(depth_h).cuda()
        un = torch.empty_like(kps)
        ur = torch.empty((B, cap), device="cuda")
        dd = torch.empty((B, cap), device="cuda")
        torch.cuda.synchronize()
        ms = {}
        for name, call in (("undistort", lambda: ex.undistort_keypoints_device(kps, counts, B, cap, K4, dist, un,
                                                                                 stream=s.cuda_stream)),
                           ("depth", lambda: ex.stereo_from_depth_device(kps, un, counts, B, cap, depth, 40.0, ur, dd,
                                                                         stream=s.cuda_stream))):
            for _ in range(10):
                call()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(s)
            for _ in range(a.reps):
                call()
            e1.record(s)
            e1.synchronize()
            ms[name] = e0.elapsed_time(e1) / a.reps
        # the host path on one thread: cv2.undistortPoints + the depth gather, per image as Frame does it
        K33 = ub.K33(K4)
        host = []
        for _ in range(5):
            t0 = time.perf_counter()
            for b in range(B):
                xy = np.stack([rec["x"][b], rec["y"][b]], 1).reshape(-1, 1, 2)
                u = cv2.undistortPoints(xy, K33, dist, P=K33).reshape(-1, 2)
                d = depth_h[b][rec["y"][b].astype(np.int64), rec["x"][b].astype(np.int64)]
                ok = d > 0
                np.where(ok, u[:, 0] - np.float32(40.0) / np.where(ok, d, 1), -1)
            host.append((time.perf_counter() - t0) * 1e3)
        print(json.dumps({"gpu": gpu, "batch": B, "records_per_image": cap, "undistort_device_ms": round(ms["undistort"], 5),
                          "depth_device_ms": round(ms["depth"], 5), "host_cv2_plus_depth_ms": round(float(np.median(host)), 3),
                          "reps": a.reps}))


if __name__ == "__main__":
    main()
