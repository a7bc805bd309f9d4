"""Times the frame ingest on the GPU and the host OpenCV path it replaces, and the stereo stream with and without it.

Kernel cases (CUDA events around `reps` C calls on one stream after a warm-up, batch 1 and 32; each call's arguments are
converted once, so the loop measures the device, not the Python wrapper):
  euroc_rect   752 x 480 grey stereo pair, each camera rectified (b2s_prepare_images_device twice, left and right maps)
  tum_rgbd     640 x 480 colour (3 channels) to grey, plus b2s_stereo_from_depth_u16_device on 2,000 keypoints of a
               16-bit depth image
  kitti_colour 1241 x 376 colour stereo pair to grey (one call over both images)
Achieved bandwidth counts the compulsory bytes: per output pixel C source bytes and 1 output byte, plus the two float
maps (8 bytes per output pixel) once per call when rectifying, since a batch shares them; the u16 depth gather's 2 bytes
per keypoint and the records it reads are counted too.  It is set against the H100 SXM's data-sheet 3.35 TB/s.
Beside each case: cv2 on this host's CPU (cv2.remap + cv2.cvtColor per image, and the u16 -> f32 scaling in numpy),
with cv2's default thread count.

Stream: StereoStream(F, 1241, 376, stereo=True) fed from resident grey frames, against the same stream fed resident
colour frames and rectifying both cameras (source_channels=3, rectify=near-identity maps), alternated `rounds` times in
one run; frames/s = F * steps / wall time of the steps ending in a synchronise.

Prints one JSON line per case with the card's name and power limit read in the same run.

  python tools/ingest_time.py [--reps 200] [--frames 32] [--steps 20] [--rounds 3]"""
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

import ingest_binding as ib  # noqa: E402
import undistort_binding as ub  # noqa: E402
from synth import synth_stereo  # noqa: E402

pkg = importlib.import_module("self_commit_orb-slam2_b200")
HBM = 3.35e12  # B/s, H100 SXM data sheet


def _time(call, s, reps, torch):
    for _ in range(10):
        call()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(s)
    for _ in range(reps):
        call()
    e1.record(s)
    e1.synchronize()
    return e0.elapsed_time(e1) / reps


def _prep_call(ex, src, out, rgb, maps, st):
    """b2s_prepare_images_device with its arguments converted once: the timed loop is one ctypes call per launch, so the
    events time the kernels, not the Python wrapper's checks."""
    import ctypes
    vp = ctypes.c_void_p
    B, H, W = src.shape[:3]
    C = 1 if src.dim() == 3 else src.shape[3]
    h, w = out.shape[1:]
    mx, my = maps if maps is not None else (None, None)
    args = (ex._h, vp(src.data_ptr()), src.stride(1), src.stride(0), B, W, H, C, int(rgb),
            vp(mx.data_ptr()) if mx is not None else None, vp(my.data_ptr()) if my is not None else None,
            mx.stride(0) * 4 if mx is not None else 0, w, h, vp(out.data_ptr()), out.stride(1), out.stride(0), vp(st))
    fn = pkg.lib().b2s_prepare_images_device
    torch_sync()  # the uploads ran on torch's stream
    ex.prepare_images_device(src, out, rgb=rgb, maps=maps, stream=st)  # the checked path once
    return lambda: fn(*args)


def torch_sync():
    import torch
    torch.cuda.synchronize()


def _host(fn, n=5):
    t = []
    for _ in range(n):
        t0 = time.perf_counter()
        fn()
        t.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(t))


def kernels(a, gpu, torch, cv2):
    s = torch.cuda.Stream()
    st = s.cuda_stream
    ex = pkg.ORBextractor(1000, 1.2, 8, 20, 7, max_width=1241, max_height=480)
    for B in (1, 32):
        # EuRoC: grey pair, both cameras rectified
        w, h = 752, 480
        maps = ib.rectify_maps("barrel_752x480")
        raw = np.stack([synth_stereo(w, h, b)[k] for k in range(2) for b in range(B)])  # left images, then right
        d_raw = torch.from_numpy(raw).cuda()
        d_out = torch.empty((2 * B, h, w), dtype=torch.uint8, device="cuda")
        dm = [tuple(torch.from_numpy(m).cuda() for m in side) for side in maps]

        calls = [_prep_call(ex, d_raw[k * B:(k + 1) * B], d_out[k * B:(k + 1) * B], True, dm[k], st) for k in range(2)]

        def euroc():
            calls[0]()
            calls[1]()

        ms = _time(euroc, s, a.reps, torch)
        nbytes = 2 * (B * w * h * (1 + 1) + w * h * 8)
        host = _host(lambda: [cv2.remap(raw[i], *maps[i // B], cv2.INTER_LINEAR) for i in range(2 * B)])
        yield dict(case="euroc_rect", batch=B, device_ms=ms, bytes=nbytes, host_ms=host)

        # TUM RGB-D: colour to grey + u16 depth at the keypoints
        w, h, cap = 640, 480, 2000
        col = np.stack([ib.colour_frame(w, h, b) for b in range(B)])
        depth16 = np.stack([np.rint(ub.depth_image(w, h, seed=b, special=False) * 5000).astype(np.uint16)
                            for b in range(B)])
        d_col = torch.from_numpy(col).cuda()
        d_grey = torch.empty((B, h, w), dtype=torch.uint8, device="cuda")
        d_dep = torch.from_numpy(depth16.view(np.int16)).cuda()
        rng = np.random.default_rng(B)
        rec = np.zeros((B, cap), ub.kp_dtype)
        rec["x"], rec["y"] = rng.uniform(0, w - 1, (B, cap)), rng.uniform(0, h - 1, (B, cap))
        kps = torch.from_numpy(rec.view(np.uint8).reshape(B, cap, 28)).cuda()
        counts = torch.full((B,), cap, dtype=torch.int32, device="cuda")
        ur = torch.empty((B, cap), device="cuda")
        dd = torch.empty((B, cap), device="cuda")

        prep = _prep_call(ex, d_col, d_grey, True, None, st)
        import ctypes
        vp = ctypes.c_void_p
        dargs = (ex._h, vp(kps.data_ptr()), vp(kps.data_ptr()), vp(counts.data_ptr()), B, cap, vp(d_dep.data_ptr()), w * 2,
                 w, h, 5000.0, 40.0, vp(ur.data_ptr()), vp(dd.data_ptr()), vp(st))
        dfn = pkg.lib().b2s_stereo_from_depth_u16_device
        torch_sync()
        ex.stereo_from_depth_u16_device(kps, kps, counts, B, cap, d_dep, 5000.0, 40.0, ur, dd, stream=st)

        def tum():
            prep()
            dfn(*dargs)

        ms = _time(tum, s, a.reps, torch)
        nbytes = B * w * h * (3 + 1) + B * cap * (2 * 28 + 2 + 8)
        f = ib.depth_multiplier(5000.0)
        host = _host(lambda: [(cv2.cvtColor(col[b], cv2.COLOR_RGB2GRAY), depth16[b].astype(np.float32) * f)
                              for b in range(B)])
        yield dict(case="tum_rgbd", batch=B, device_ms=ms, bytes=nbytes, host_ms=host)

        # KITTI colour: both images of each pair, no rectification
        w, h = 1241, 376
        col = np.stack([ib.colour_frame(w, h, b) for b in range(2 * B)])
        d_col = torch.from_numpy(col).cuda()
        d_grey = torch.empty((2 * B, h, w), dtype=torch.uint8, device="cuda")
        ms = _time(_prep_call(ex, d_col, d_grey, False, None, st), s, a.reps, torch)
        nbytes = 2 * B * w * h * (3 + 1)
        host = _host(lambda: [cv2.cvtColor(col[i], cv2.COLOR_BGR2GRAY) for i in range(2 * B)])
        yield dict(case="kitti_colour", batch=B, device_ms=ms, bytes=nbytes, host_ms=host)


def stream(a, torch):
    stream_mod = importlib.import_module("self_commit_orb-slam2_b200.stream")
    F, w, h, D = a.frames, 1241, 376, 2 * a.frames
    pairs = [synth_stereo(w, h, 300 + i) for i in range(D)]
    grey = np.stack([np.stack([p[k] for p in pairs]) for k in range(2)])
    colour = np.stack([np.repeat(grey[k][..., None], 3, -1) for k in range(2)])
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    ident = (xx + np.float32(0.25), yy)  # a quarter-pixel shift: every pixel interpolated
    plain = stream_mod.StereoStream(F, w, h, 2000, stereo=True)
    ingest = stream_mod.StereoStream(F, w, h, 2000, stereo=True, source_channels=3, rgb=True,
                                     rectify=(ident[0], ident[1], ident[0], ident[1]))
    d_grey, d_col = torch.from_numpy(grey).cuda(), torch.from_numpy(colour).cuda()
    fps = {"plain": [], "ingest": []}
    for r in range(a.rounds + 1):
        for name, ss, d_all in (("plain", plain, d_grey), ("ingest", ingest, d_col)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i in range(a.steps):
                ss.load_window(d_all, (i * F) % D)
                ss.step_device()
            torch.cuda.synchronize()
            if r:  # round 0 warms both up
                fps[name].append(F * a.steps / (time.perf_counter() - t0))
    return {k: [round(v, 1) for v in vs] for k, vs in fps.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--frames", type=int, default=32)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if pkg.device_count() < 1:
        sys.exit("ingest_time: no CUDA device")
    import cv2
    import torch
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    for r in kernels(a, gpu, torch, cv2):
        r.update(gpu=gpu, reps=a.reps, cv2_threads=cv2.getNumThreads(), device_ms=round(r["device_ms"], 5),
                 host_ms=round(r["host_ms"], 3), achieved_GBps=round(r["bytes"] / (r["device_ms"] * 1e-3) / 1e9, 1),
                 of_hbm=round(r["bytes"] / (r["device_ms"] * 1e-3) / HBM, 3))
        print(json.dumps(r), flush=True)
    fps = stream(a, torch)
    print(json.dumps({"case": "stream_fps", "gpu": gpu, "frames_per_step": a.frames, "steps": a.steps, "width": 1241,
                      "height": 376, "plain_fps": fps["plain"], "ingest_fps": fps["ingest"]}), flush=True)


if __name__ == "__main__":
    main()
