"""Batched stereo-stream mode: frames sharded over GPUs, one process per GPU (SURVEY.md §8e).

Per step a rank owns F stereo frames (2F images).  Device-resident path:
  1. b2s_extract_batch_device  : 2F images -> fixed-size feature records written straight into the buffer that is the
                                 NCCL all-gather input (no staging copy)
  2. all_gather (world > 1)    : left-image records of every rank over NVLink/NVSwitch (torch.distributed, NCCL)
  3. b2s_search_by_bow_device  : temporal match left(t-1) -> left(t) for the rank's F frames, all features in one
                                 vocabulary node (2000x2000 brute force); the frame before the shard's first one comes
                                 from the previous rank's gathered records
  3b. b2s_track_queries_device + b2s_search_by_projection_last_device (project=True): the motion-model matcher of
                                 Tracking::TrackWithMotionModel, SearchByProjection(CurrentFrame, LastFrame), for the same
                                 F pairs: the last frame's stereo points are moved by the relative pose and searched in
                                 the current frame's grid windows
  4. b2s_local_ba_batch        : one LocalBA window per `ba_every` frames (replicas; its own stream, overlaps 1-3)
torch is plumbing only: device memory, streams, torch.distributed.
"""
import ctypes
import threading

import numpy as np
import torch

from . import (ORBextractor, ORBmatcher, Optimizer, _check, _vp, ba_edge_dtype, keypoint_dtype, lib, proj_query_dtype)
from . import sharding

KP_BYTES = keypoint_dtype.itemsize  # 28


class StereoStream:
    def __init__(self, frames_per_step, width, height, nfeatures=2000, scale=1.2, nlevels=8, ini_th=20, min_th=7,
                 ba_problem=None, ba_every=5, device=0, rank=0, world=1, nnratio=0.7, ba_depth=1,
                 exchange="boundary", ba_problems=None, pose_problems=None, stereo=False, bf=386.1448, project=False,
                 intrinsics=(718.856, 718.856, 607.1928, 185.2157), motion=None, ba_sms=64, source_channels=1, rgb=True,
                 rectify=None, source_size=None):
        """ba_problems: list of LocalBA windows (a step solves ceil(F / ba_every) of them, taken round-robin);
        pose_problems: list of per-frame PoseOptimization problems (F per step, round-robin); stereo: run
        Frame::ComputeStereoMatches for the F pairs of every step on the resident pyramids; project (needs stereo): also
        run SearchByProjection(CurrentFrame, LastFrame) for every frame against its predecessor, the predecessor's stereo
        points moved by `motion` (Tcl, 3 x 4; default: 0.8 m forward with a small yaw, the KITTI-like case that takes the
        reference's forward branch, src/ORBmatcher.cc:1595-1598).  ba_sms: SMs one LocalBA batch may occupy (0 = all): the LM
        kernel shares the GPU with extraction and matching, and about half of the SMs gives the best stream throughput
        (DESIGN.md §6).
        Frame ingest (all off by default): source_channels (1, 3, 4) and rgb (mbRGB) say what a raw frame holds; rectify =
        (left mapx, left mapy, right mapx, right mapy), float32 [height, width] each, the stereo examples'
        initUndistortRectifyMap maps; source_size = the raw (width, height), default (width, height).  When colour or
        rectification is asked for, upload / load_window take raw frames and every step first runs
        b2s_prepare_images_device (left maps, then right maps) into the grey input of the extractor."""
        self.F, self.w, self.h = frames_per_step, width, height
        self.rank, self.world = rank, world
        self.dev = torch.device("cuda", device)
        # a real (non-default) stream: the C ABI treats stream == NULL as "the handle's own stream"
        self.stream = torch.cuda.Stream(self.dev)
        self.ex = ORBextractor(nfeatures, scale, nlevels, ini_th, min_th, max_width=max(width, 64),
                               max_height=max(height, 64), max_batch=2 * self.F, device=device)
        self.cap = self.ex.cap
        self.matcher = ORBmatcher(nnratio, True, max_features=self.cap, max_batch=self.F, device=device)
        self.windows = list(ba_problems) if ba_problems else ([ba_problem] if ba_problem is not None else [])
        self.ba_problem = self.windows[0] if self.windows else None
        self.ba_every = ba_every
        self.n_ba = (self.F + ba_every - 1) // ba_every if self.windows else 0
        self.pose_problems = list(pose_problems) if pose_problems else []
        self.stereo, self.bf = bool(stereo), float(bf)
        self.opt = None
        self.opts = []
        self._prep = {}
        if self.n_ba or self.pose_problems:
            # ba_depth solver handles: with depth 2 the host preparation / upload / write-back of one LocalBA batch
            # overlaps the LM kernel of the previous one (pipelined mode only)
            mk = max([16] + [w["n_kf"] for w in self.windows])
            mm = max([16] + [len(w["points"]) for w in self.windows])
            me = max([64] + [len(w["edges"]) for w in self.windows])
            # PoseOptimization has its own handle (own stream, own worker thread): the Tracking-side solver does not queue
            # behind the LocalMapping-side one.  (Created first: see the shared-memory attribute note in b2s_ba_create.)
            self.pose_opt = Optimizer(max_kf=4, max_mp=16, max_edges=64, max_batch=max(1, self.F), device=device) \
                if self.pose_problems else None
            for _ in range(max(1, int(ba_depth))):
                self.opts.append(Optimizer(max_kf=mk, max_mp=mm, max_edges=me, max_batch=max(1, self.n_ba), device=device))
                self.opts[-1].set_sm_budget(ba_sms)
            self.opt = self.opts[0]
        F, cap = self.F, self.cap
        S = 1 + 2 * F  # slot 0: the frame before this shard; 1..F left images; F+1..2F right images
        z = dict(device=self.dev)
        self.kps = torch.zeros((S, cap, KP_BYTES), dtype=torch.uint8, **z)
        self.desc = torch.zeros((S, cap, 32), dtype=torch.uint8, **z)
        self.counts = torch.zeros(S, dtype=torch.int32, **z)
        self.node = torch.zeros((1 + F, cap), dtype=torch.int32, **z)   # every feature in vocabulary node 0
        self.valid = torch.ones((1 + F, cap), dtype=torch.uint8, **z)
        self.ang = torch.zeros((1 + F, cap), dtype=torch.float32, **z)
        self.match = torch.full((F, cap), -1, dtype=torch.int32, **z)
        self.nmatch = torch.zeros(F, dtype=torch.int32, **z)
        # exchange: "boundary" all-gathers only each rank's LAST left-image record (the only frame another rank's temporal
        # matcher reads: 123 KB per rank); "all" gathers every left-image record of the step (SURVEY §8e: any rank can then
        # match any frame pair; 20 MB per rank and step)
        self.exchange = exchange
        self.G = F if exchange == "all" else 1
        if world > 1:
            self.g_kps = torch.zeros((world, self.G, cap, KP_BYTES), dtype=torch.uint8, **z)
            self.g_desc = torch.zeros((world, self.G, cap, 32), dtype=torch.uint8, **z)
            self.g_counts = torch.zeros((world, self.G), dtype=torch.int32, **z)
        self.d_imgs = torch.zeros((2 * F, height, width), dtype=torch.uint8, **z)
        self.src_c, self.rgb = int(source_channels), bool(rgb)
        self.sw, self.sh = (width, height) if source_size is None else (int(source_size[0]), int(source_size[1]))
        if self.src_c not in (1, 3, 4):
            raise ValueError("source_channels must be 1, 3 or 4")
        if rectify is None and (self.sw, self.sh) != (width, height):
            raise ValueError("source_size differs from the output size: only rectification changes the size")
        self.ingest = self.src_c != 1 or rectify is not None
        self.maps = None
        if self.ingest:  # raw frames: [2F, sh, sw] or [2F, sh, sw, C]
            self.d_src = torch.zeros((2 * F, self.sh, self.sw) + ((self.src_c,) if self.src_c > 1 else ()),
                                     dtype=torch.uint8, **z)
            if rectify is not None:
                if len(rectify) != 4:
                    raise ValueError("rectify: (left mapx, left mapy, right mapx, right mapy)")
                ms = [torch.as_tensor(m, dtype=torch.float32).to(self.dev).contiguous() for m in rectify]
                for m in ms:
                    if tuple(m.shape) != (height, width):
                        raise ValueError("rectify: every map must be [height, width]")
                self.maps = ((ms[0], ms[1]), (ms[2], ms[3]))
        if self.stereo:  # mvuRight / mvDepth per left feature, matches per pair
            self.ur = torch.zeros((F, cap), dtype=torch.float32, **z)
            self.dp_all = torch.zeros((1 + F, cap), dtype=torch.float32, **z)  # slot 0: depth of the shard's predecessor
            self.dp = self.dp_all[1:]
            self.nstereo = torch.zeros(F, dtype=torch.int32, **z)
        self.project = bool(project) and self.stereo
        if self.project:
            self.fx, self.fy, self.cx, self.cy = [float(v) for v in intrinsics]
            if motion is None:
                a = 0.01  # rad of yaw per frame
                motion = np.array([[np.cos(a), 0, np.sin(a), 0.02], [0, 1, 0, 0.0], [-np.sin(a), 0, np.cos(a), -0.8]])
            self.motion = np.ascontiguousarray(motion, np.float32).reshape(3, 4)
            self.proj_mode = self.projection_mode(self.motion, self.bf / self.fx)
            self.proj_th = 7.0  # stereo / RGB-D window of Tracking::TrackWithMotionModel (src/Tracking.cc:892-897)
            self.geom = dict(mnMinX=0.0, mnMinY=0.0, mnMaxX=float(width), mnMaxY=float(height), bf=self.bf,
                             scale_factors=np.asarray(self.ex.GetScaleFactors(), np.float32))
            self.Tcl = torch.from_numpy(np.tile(self.motion.reshape(1, 12), (F, 1))).to(self.dev)
            self.q = torch.zeros((F, cap, proj_query_dtype.itemsize), dtype=torch.uint8, **z)
            self.nq = torch.zeros(F, dtype=torch.int32, **z)
            self.pmatch = torch.full((F, cap), -1, dtype=torch.int32, **z)
            self.npmatch = torch.zeros(F, dtype=torch.int32, **z)
            if world > 1:
                self.g_dp = torch.zeros((world, self.G, cap), dtype=torch.float32, **z)
        self._step_no = 0
        self._pool = None
        self._ba_future = None
        self._ba_futures = []  # (pipelined) in-flight LocalBA batches, oldest first; at most len(self.opts)
        self._ba_next = 0
        self._last_lock = threading.Lock()
        self.last_solved = {}  # "ba" / "pose" -> (step, LocalBA outputs / PoseOptimization batch) of the latest step solved

    @staticmethod
    def projection_mode(Tcl, mb):
        """0 / 1 (forward) / 2 (backward) as src/ORBmatcher.cc:1589-1598 decides it for a stereo frame: tlc = position of
        the current camera centre in the last camera's frame."""
        R, t = np.asarray(Tcl, np.float64)[:, :3], np.asarray(Tcl, np.float64)[:, 3]
        tlc_z = float((-R.T @ t)[2])
        return 1 if tlc_z > mb else (2 if -tlc_z > mb else 0)

    @staticmethod
    def track_queries_host(kps, desc, depth, n, Tcl, fx, fy, cx, cy, has_obs=1):
        """numpy restatement of b2s_track_queries_device (same single-precision operation order), for host-buffer callers
        and tests: kps [B, cap] keypoint_dtype, desc [B, cap, 32], depth [B, cap], n [B], Tcl [B, 3, 4]."""
        f = np.float32
        B, cap = depth.shape
        q = np.zeros((B, cap), proj_query_dtype)
        T = np.asarray(Tcl, f).reshape(B, 12)
        z = depth.astype(f)
        live = (np.arange(cap)[None, :] < np.asarray(n)[:, None])
        ok = live & (z > 0)
        invfx, invfy = f(1.0) / f(fx), f(1.0) / f(fy)
        with np.errstate(all="ignore"):
            x = (kps["x"] - f(cx)) * z * invfx
            y = (kps["y"] - f(cy)) * z * invfy
            c = lambda k: T[:, k:k + 1]
            xc = ((c(0) * x + c(1) * y) + c(2) * z) + c(3)
            yc = ((c(4) * x + c(5) * y) + c(6) * z) + c(7)
            zc = ((c(8) * x + c(9) * y) + c(10) * z) + c(11)
            invz = f(1.0) / zc
            ok2 = ok & ~(invz < 0)
            u = (f(fx) * xc) * invz + f(cx)
            v = (f(fy) * yc) * invz + f(cy)
        q["u"] = np.where(ok2, u, f(0))
        q["v"] = np.where(ok2, v, f(0))
        q["invz"] = np.where(ok2, invz, f(-1))
        q["angle"] = kps["angle"]
        q["octave"] = kps["octave"]
        q["has_obs"] = has_obs
        q["desc"] = desc
        q[~live] = np.zeros((), proj_query_dtype)
        return q

    # ------------------------------------------------------------------ device-resident step
    def upload(self, imgs_host):
        """imgs_host: uint8 [2F, h, w] (L_0..L_F-1, R_0..R_F-1), ideally pinned."""
        with torch.cuda.stream(self.stream):
            (self.d_src if self.ingest else self.d_imgs).copy_(imgs_host, non_blocking=True)

    def load_window(self, d_all, start):
        """d_all: device uint8 [2, D, h, w] (left / right images of D resident frames).  Copies frames start .. start+F-1
        (modulo D) into the step's input batch on the stream (device-to-device, part of the timed step)."""
        D, F = d_all.shape[1], self.F
        dst = self.d_src if self.ingest else self.d_imgs  # raw frames [2, D, sh, sw(, C)] when ingesting
        with torch.cuda.stream(self.stream):
            done = 0
            while done < F:
                a = (start + done) % D
                n = min(F - done, D - a)
                dst[done:done + n].copy_(d_all[0, a:a + n], non_blocking=True)
                dst[F + done:F + done + n].copy_(d_all[1, a:a + n], non_blocking=True)
                done += n

    def step_device(self, run_ba=True, pipelined=False):
        """Enqueue extraction (+ all-gather) + matching on the stream, then LocalBA of this step's windows.

        pipelined=True runs the LocalBA batch on a worker thread (the C call releases the GIL and uses the solver's own
        CUDA streams), so the caller can already enqueue the next step while it runs; at most one batch is in flight
        (finish() joins the last one).  This also keeps ranks from waiting on each other's host-blocking LocalBA inside
        the all-gather."""
        with torch.cuda.stream(self.stream):
            self._enqueue_extract_match()
        ba_out = None
        if run_ba and (self.n_ba or self.pose_problems):  # own stream inside the solver; overlaps the work enqueued above
            if pipelined:
                ba_out = self._submit_ba()
            else:
                self._solve_pose(self._step_no)
                ba_out = self._solve(self.opt, self._step_no)
        self._step_no += 1
        return ba_out

    def _step_windows(self, step):
        if not self.n_ba:
            return []
        n = len(self.windows)
        return [self.windows[(step * self.n_ba + i) % n] for i in range(self.n_ba)]

    def _step_poses(self, step):
        if not self.pose_problems:
            return []
        n = len(self.pose_problems)
        return [self.pose_problems[(step * self.F + i) % n] for i in range(self.F)]

    def _solve(self, opt, step):
        """PoseOptimization of the step's F frames, then LocalBA of its windows, on solver handle `opt`.  The ctypes problem
        arrays of a (handle, window set) are built once and reused (the per-step Python cost is one C call each)."""
        out = None
        wins = self._step_windows(step)
        if wins:
            key = ("ba", id(opt), (step * self.n_ba) % len(self.windows) if len(self.windows) > self.n_ba else 0)
            if key not in self._prep:
                self._prep[key] = opt.prepare_ba_batch(wins)
            out = opt.run_prepared_ba(self._prep[key])
            self._record("ba", step, out)
        return out

    def _record(self, kind, step, out):
        with self._last_lock:
            if step >= self.last_solved.get(kind, (-1, None))[0]:
                self.last_solved[kind] = (step, out)

    def _solve_pose(self, step):
        poses = self._step_poses(step)
        if not poses:
            return None
        key = ("pose", (step * self.F) % len(self.pose_problems) if len(self.pose_problems) > self.F else 0)
        if key not in self._prep:
            self._prep[key] = self.pose_opt.prepare_pose_batch(poses)
        out = self.pose_opt.run_prepared_pose(self._prep[key])
        self._record("pose", step, self._prep[key])
        return out

    def _submit_ba(self):
        """Queue this step's LocalBA batch on the next solver handle; returns the result of the batch that used that
        handle before (or None)."""
        if self._pool is None:
            from concurrent.futures import ThreadPoolExecutor
            self._pool = ThreadPoolExecutor(max_workers=len(self.opts) + 1)
            self._pose_future = None
        out = None
        if len(self._ba_futures) >= len(self.opts):
            out = self._ba_futures.pop(0).result()
        opt = self.opts[self._ba_next % len(self.opts)]
        self._ba_next += 1
        self._ba_futures.append(self._pool.submit(self._solve, opt, self._step_no))
        if self.pose_problems:  # one PoseOptimization batch in flight, on its own handle / thread
            if self._pose_future is not None:
                self._pose_future.result()
            self._pose_future = self._pool.submit(self._solve_pose, self._step_no)
        return out

    def finish(self):
        """Join the LocalBA batches still in flight (pipelined mode); returns the last result or None."""
        out = None
        while self._ba_futures:
            out = self._ba_futures.pop(0).result()
        if getattr(self, "_pose_future", None) is not None:
            self._pose_future.result()
            self._pose_future = None
        return out

    def _enqueue_extract_match(self):
        F, cap = self.F, self.cap
        st = self.stream.cuda_stream
        if self.ingest:  # Tracking::GrabImageStereo's grey conversion, after the examples' rectification of each camera
            if self.maps is None:
                self.ex.prepare_images_device(self.d_src, self.d_imgs, rgb=self.rgb, stream=st)
            else:
                for side in range(2):
                    self.ex.prepare_images_device(self.d_src[side * F:(side + 1) * F], self.d_imgs[side * F:(side + 1) * F],
                                                  rgb=self.rgb, maps=self.maps[side], stream=st)
        self.ex.extract_batch_device(self.d_imgs.data_ptr(), self.w * self.h, 2 * F, self.w, self.h, self.w,
                                     self.kps[1:].data_ptr(), self.desc[1:].data_ptr(), self.counts[1:].data_ptr(), cap,
                                     stream=st)
        if self.stereo:  # Frame::ComputeStereoMatches, left image i <-> right image F + i, on the resident pyramids
            self.ex.stereo_match_device(0, F, F, self.kps[1:].data_ptr(), self.desc[1:].data_ptr(),
                                        self.counts[1:].data_ptr(), cap, self.bf, 0.0, self.ur.data_ptr(), self.dp.data_ptr(),
                                        self.nstereo.data_ptr(), stream=st)
        if self.world > 1:
            lo = 1 + F - self.G  # first gathered slot: all F left images, or just the last one
            sharding.gather_records(self.kps[lo:1 + F], self.desc[lo:1 + F], self.counts[lo:1 + F], self.g_kps, self.g_desc,
                                    self.g_counts)
            sharding.take_predecessor(self.g_kps, self.g_desc, self.g_counts, self.rank, self.world, self.kps[0],
                                      self.desc[0], self.counts[0:1])
            if self.project:  # the predecessor's stereo depths travel with its record
                sharding.gather_array(self.dp_all[lo:1 + F], self.g_dp)
                self.dp_all[0].copy_(self.g_dp[sharding.predecessor_source(self.rank, self.world), self.G - 1])
        else:  # ring inside the shard
            self.kps[0].copy_(self.kps[F])
            self.desc[0].copy_(self.desc[F])
            self.counts[0:1].copy_(self.counts[F:F + 1])
            if self.project:
                self.dp_all[0].copy_(self.dp_all[F])
        # angles of the left images (kpUn.angle), gathered out of the 28-byte records
        self.ang.copy_(self.kps[:1 + F].view(torch.float32)[:, :, 3])
        L = lib()
        _check(L.b2s_search_by_bow_device(self.matcher._h, F, _vp(self.desc.data_ptr()), _vp(self.node.data_ptr()),
                                          _vp(self.valid.data_ptr()), _vp(self.ang.data_ptr()),
                                          _vp(self.counts.data_ptr()), cap, _vp(self.desc[1:].data_ptr()),
                                          _vp(self.node[1:].data_ptr()), None, _vp(self.ang[1:].data_ptr()),
                                          _vp(self.counts[1:].data_ptr()), cap, 50, float(self.matcher.mfNNratio), 0, 1,
                                          _vp(self.match.data_ptr()), _vp(self.nmatch.data_ptr()), _vp(st)))
        if self.project:  # pair f: last = left image f-1 (slot f), current = left image f (slot f+1)
            m = self.matcher
            m.track_queries_device(F, self.kps.data_ptr(), self.desc.data_ptr(), self.dp_all.data_ptr(), self.counts.data_ptr(),
                                   cap, self.Tcl.data_ptr(), self.fx, self.fy, self.cx, self.cy, 1, self.q.data_ptr(),
                                   self.nq.data_ptr(), stream=st)
            m.search_by_projection_last_device(F, self.q.data_ptr(), self.nq.data_ptr(), cap, self.kps[1:].data_ptr(),
                                               self.ur.data_ptr(), self.desc[1:].data_ptr(), self.counts[1:].data_ptr(), cap,
                                               self.geom, self.proj_th, self.proj_mode, self.pmatch.data_ptr(),
                                               self.npmatch.data_ptr(), stream=st)

    # ------------------------------------------------------------------ end-to-end step through the host-buffer C ABI
    def step_host(self, imgs_host_np, run_ba=True, pipelined=False, img_ptrs=None):
        """imgs_host_np: numpy uint8 [2F, h, w] (or img_ptrs: 2F host addresses of dense h x w images, left images first).
        Returns (counts, nmatches, ba_out); everything ends up in host memory."""
        if self.ingest:
            raise ValueError("step_host takes grey images: a stream with source_channels or rectify ingests on the device")
        F, cap = self.F, self.cap
        if getattr(self, "_h_kps", None) is None:  # pinned result buffers, allocated once
            # slot 0 = the frame before the shard's first one (ring), slots 1..2F = this step's images: both sides of the
            # temporal matcher are then contiguous views, exactly like the device-resident layout
            self._h_kps_t = torch.zeros((1 + 2 * F, cap, KP_BYTES), dtype=torch.uint8).pin_memory()
            self._h_desc_t = torch.zeros((1 + 2 * F, cap, 32), dtype=torch.uint8).pin_memory()
            self._h_kps = self._h_kps_t.numpy().view(keypoint_dtype).reshape(1 + 2 * F, cap)
            self._h_desc = self._h_desc_t.numpy()
            self._h_n = np.zeros(1 + 2 * F, np.int32)
            self._h_ang = torch.zeros((1 + F, cap), dtype=torch.float32).pin_memory().numpy()
            self._h_node = torch.zeros((1 + F, cap), dtype=torch.int32).pin_memory().numpy()
            self._h_valid = torch.ones((1 + F, cap), dtype=torch.uint8).pin_memory().numpy()
            self._h_match = torch.zeros((F, cap), dtype=torch.int32).pin_memory().numpy()
            self._h_nm = np.zeros(F, np.int32)
            self._h_ptrs = (_vp * (2 * F))()
        all_kps, all_desc, all_n = self._h_kps, self._h_desc, self._h_n
        res_kps, res_desc, n = all_kps[1:], all_desc[1:], all_n[1:]
        if img_ptrs is not None:
            for i in range(2 * F):
                self._h_ptrs[i] = img_ptrs[i]
        else:
            base, stride0 = imgs_host_np.ctypes.data, imgs_host_np.strides[0]
            for i in range(2 * F):
                self._h_ptrs[i] = base + i * stride0
        L = lib()
        _check(L.b2s_extract_batch(self.ex._h, ctypes.cast(self._h_ptrs, _vp), 2 * F, self.w, self.h, self.w,
                                   res_kps.ctypes.data_as(_vp), res_desc.ctypes.data_as(_vp), cap,
                                   n.ctypes.data_as(_vp)))
        # ring: pair f = (left f-1, left f); slot 0 <- the last left image
        all_kps[0] = all_kps[F]
        all_desc[0] = all_desc[F]
        all_n[0] = all_n[F]
        np.copyto(self._h_ang, all_kps["angle"][:1 + F])
        ang, node, valid, match, nm = self._h_ang, self._h_node, self._h_valid, self._h_match, self._h_nm
        p = lambda a: a.ctypes.data_as(_vp)
        _check(L.b2s_search_by_bow_batch(self.matcher._h, F, p(all_desc), p(node), p(valid), p(ang), p(all_n), cap,
                                         p(all_desc[1:]), p(node[1:]), None, p(ang[1:]), p(all_n[1:]), cap, 50,
                                         float(self.matcher.mfNNratio), 0, 1, p(match), p(nm)))
        if self.stereo:  # mvuRight / mvDepth of the F left images, host arrays (the pyramids are still on the device)
            if getattr(self, "_h_ur", None) is None:
                self._h_ur = torch.zeros((F, cap), dtype=torch.float32).pin_memory().numpy()
                self._h_dp_all = torch.zeros((1 + F, cap), dtype=torch.float32).pin_memory().numpy()
                self._h_dp = self._h_dp_all[1:]
                self._h_ns = np.zeros(F, np.int32)
                self._h_pm = torch.zeros((F, cap), dtype=torch.int32).pin_memory().numpy()
                self._h_npm = np.zeros(F, np.int32)
                self._h_Tcl = np.tile(self.motion.reshape(1, 12), (F, 1)) if self.project else None
            L.b2s_stereo_match.argtypes = [_vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float, _vp,
                                           _vp, ctypes.c_int, _vp]
            _check(L.b2s_stereo_match(self.ex._h, 0, F, F, ctypes.c_float(self.bf), ctypes.c_float(0.0), p(self._h_ur),
                                      p(self._h_dp), cap, p(self._h_ns)))
            if self.project:  # SearchByProjection(CurrentFrame, LastFrame): frame f against f-1 (slot 0 = ring predecessor)
                self._h_dp_all[0] = self._h_dp_all[F]
                self.matcher.SearchByProjectionSequence(all_kps[:1 + F], all_desc[:1 + F], self._h_dp_all, self._h_ur,
                                                        all_n[:1 + F], self._h_Tcl, self.fx, self.fy, self.cx, self.cy,
                                                        self.geom, self.proj_th, self.proj_mode,
                                                        out=(self._h_npm, self._h_pm))
        ba_out = None
        if run_ba and (self.n_ba or self.pose_problems):
            if pipelined:  # results of an earlier step's windows are returned; finish() joins the rest
                ba_out = self._submit_ba()
            else:
                self._solve_pose(self._step_no)
                ba_out = self._solve(self.opt, self._step_no)
        self._step_no += 1
        return n, nm, ba_out, (res_kps, res_desc, match)

    def launch_count(self):
        c = self.ex.launch_count() + self.matcher.launch_count()
        for o in self.opts:
            c += o.launch_count()
        if getattr(self, "pose_opt", None) is not None:
            c += self.pose_opt.launch_count()
        return c

    def h2d_bytes_per_step(self):
        b = 2 * self.F * self.sw * self.sh * self.src_c
        b += self.F * self.cap * (32 + 4 + 4 + 1) * 2  # descriptors, nodes, angles, valid for both sides of the matcher
        if self.project:  # records + depths of F + 1 frames, mvuRight of F, relative poses
            b += (self.F + 1) * self.cap * (KP_BYTES + 32 + 4) + self.F * self.cap * 4 + self.F * 48
        for pr in self._step_windows(0):
            b += pr["n_kf"] * 64 + len(pr["points"]) * 12 + len(pr["edges"]) * ba_edge_dtype.itemsize
        for pp in self._step_poses(0):
            b += 64 + len(pp["has_mp"]) * (1 + 12 + 4 * 4)
        return int(b)

    def d2h_bytes_per_step(self):
        b = 2 * self.F * self.cap * (KP_BYTES + 32) + 2 * self.F * 4
        b += self.F * self.cap * 4 + self.F * 4
        if self.stereo:
            b += self.F * self.cap * 8 + self.F * 4
        if self.project:
            b += self.F * self.cap * 4 + self.F * 4
        for pr in self._step_windows(0):
            b += pr["n_local"] * 64 + len(pr["points"]) * 12 + len(pr["edges"])
        for pp in self._step_poses(0):
            b += 64 + len(pp["has_mp"])
        return int(b)
