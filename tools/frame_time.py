"""Per-frame wall time of the drop-in Frame constructors (host/adapters/Frame_b200.cc over libb200slam.so) and of the
reference's own Frame (src/Frame.cc with its CPU ORBextractor) on this host's CPU, on the same inputs:

  kitti_stereo  1241 x 376 stereo pair, KITTI calibration, 2000 features
  tum_rgbd      640 x 480 grey image + float depth, TUM1 calibration (five coefficients), 1000 features
  tum_mono      640 x 480 grey image, TUM1 calibration, 1000 features

Each drop-in frame ends in its synchronous downloads (keypoints, descriptors, mvuRight / mvDepth), so the wall time of
one constructor call is what Tracking waits for.  Both sides run through oracle/ref_frame_seq_glue.cpp
(oracle/_ref/libadapter_frame.so and libref_frame_seq.so, built by oracle/frame.mk); the reference allocates from the
system allocator, as it does in a real build, and extracts left and right on its own two threads.  Median of `reps`
calls after `warmup`.  Also printed: the card's name and power limit, read in the same run, and the pyramid bytes a
drop-in stereo frame no longer downloads (both images' mvImagePyramid at 1241 x 376, 8 levels of 1.2).

  python tools/frame_time.py [--reps 50] [--warmup 5] [--ref-reps 10]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402

import frame_binding as fb  # noqa: E402
import undistort_binding as ub  # noqa: E402
from synth import synth_image, synth_stereo  # noqa: E402


def _median_ms(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(t))


def pyramid_bytes(w, h, nlevels=8, scale=1.2):
    """bytes of one image's mvImagePyramid: level l is lrintf(w * inv_l) x lrintf(h * inv_l), inv_l = 1 / scale^l in
    float (src/ORBextractor.cc:500-554, 1078-1084)"""
    s = np.float32(1.0)
    total = 0
    for _ in range(nlevels):
        inv = np.float32(1.0) / s
        total += int(np.rint(np.float32(w) * inv)) * int(np.rint(np.float32(h) * inv))
        s = np.float32(np.float64(s) * scale)
    return total


def cases(L):
    """(name, call) for one library; every call builds one frame"""
    L.reset()
    K4s, dists, bf, th, nf = fb.STEREO["kitti"]
    imL, imR = synth_stereo(1241, 376, 3)
    exl, exr = L.extractor(nf), L.extractor(nf)
    K4, dist = fb.MONO["tum1"]
    img = synth_image(640, 480, 31)
    depth = ub.depth_image(640, 480, seed=9, special=False)
    ex_d, ex_m = L.extractor(1000), L.extractor(1000)
    return [("kitti_stereo", lambda: L.stereo(exl, exr, imL, imR, K4s, dists, bf, th)),
            ("tum_rgbd", lambda: L.mono_rgbd(ex_d, img, K4, dist, 40.0, 40.0, depth=depth)),
            ("tum_mono", lambda: L.mono_rgbd(ex_m, img, K4, dist, 40.0, 40.0))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--ref-reps", type=int, default=10)
    a = ap.parse_args()
    for p in (fb.ADAPTER_LIB, fb.REF_LIB):
        if not os.path.exists(p):
            sys.exit("frame_time: %s is missing (make -C oracle -f frame.mk frame-ref REF=<reference tree>)" % p)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    drop_in = fb.FrameLib(fb.ADAPTER_LIB, monotonic=0)
    ref = fb.FrameLib(fb.REF_LIB, monotonic=0)
    ref_ms = {name: _median_ms(call, a.ref_reps, 1) for name, call in cases(ref)}
    ref.reset()
    for name, call in cases(drop_in):
        ms = _median_ms(call, a.reps, a.warmup)
        print(json.dumps(dict(case=name, gpu=gpu, drop_in_ms=round(ms, 3), reference_cpu_ms=round(ref_ms[name], 3),
                              reps=a.reps, ref_reps=a.ref_reps, host_cpus=os.cpu_count())))
    drop_in.reset()
    print(json.dumps(dict(case="kitti_stereo_pyramid_not_downloaded", bytes_per_frame=2 * pyramid_bytes(1241, 376))))


if __name__ == "__main__":
    main()
