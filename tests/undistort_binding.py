"""Shared pieces of the undistortion / RGB-D depth tests: the calibrations, a numpy restatement of cv::undistortPoints
(OpenCV 4) and of Frame::ComputeStereoFromRGBD, the oracle's orc_undistort_points, and the reference's own monocular and
RGB-D Frame constructors (oracle/_ref/libref_frame_undistort.so, oracle/undistort.mk)."""
import ctypes
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_LIB = os.path.join(ROOT, "oracle", "liborb_undistort.so")
GRID_ORACLE_LIB = os.path.join(ROOT, "oracle", "liborb_oracle.so")
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libref_frame_undistort.so")
vp, c_f, c_i = ctypes.c_void_p, ctypes.c_float, ctypes.c_int

# Examples/{Monocular,RGB-D}/TUM{1,2,3}.yaml and Examples/Monocular/EuRoC.yaml: (fx, fy, cx, cy), (k1, k2, p1, p2[, k3])
CALIB = {
    "tum1": ((517.306408, 516.469215, 318.643040, 255.313989), (0.262383, -0.953104, -0.005358, 0.002628, 1.163314)),
    "tum1_4": ((517.306408, 516.469215, 318.643040, 255.313989), (0.262383, -0.953104, -0.005358, 0.002628)),
    "tum2": ((520.908620, 521.007327, 325.141442, 249.701764), (0.231222, -0.784899, -0.003257, -0.000105, 0.917205)),
    "tum2_4": ((520.908620, 521.007327, 325.141442, 249.701764), (0.231222, -0.784899, -0.003257, -0.000105)),
    "tum3": ((535.4, 539.2, 320.1, 247.6), (0.0, 0.0, 0.0, 0.0)),
    "euroc": ((458.654, 457.296, 367.215, 248.375), (-0.28340811, 0.07395907, 0.00019359, 1.76187114e-05)),
    "euroc_5": ((458.654, 457.296, 367.215, 248.375), (-0.28340811, 0.07395907, 0.00019359, 1.76187114e-05, 0.0)),
    # not undistorted by Frame::UndistortKeyPoints (only k1 is tested), still undistorted by cv::undistortPoints
    "k1zero_p1": ((517.306408, 516.469215, 318.643040, 255.313989), (0.0, 0.0, 0.004, -0.002, 0.0)),
    # strong pincushion: the corners move inwards more than the edges, so undistorted keypoints fall outside the bounds
    "pincushion": ((300.0, 300.0, 320.0, 240.0), (0.6, 0.0, 0.0, 0.0)),
    # strong barrel: some iterations reach icdist < 0 (OpenCV 4's early exit)
    "barrel": ((300.0, 300.0, 320.0, 240.0), (-1.5, 0.2, 0.001, -0.002, -2.0)),
}


def calib(name):
    K, d = CALIB[name]
    return np.float32(K), np.float32(d)


def K33(K4):
    return np.float32([[K4[0], 0, K4[2]], [0, K4[1], K4[3]], [0, 0, 1]])


def np_undistort(xy, K4, dist, count_early=False):
    """cvUndistortPointsInternal (P = K, R = I, 5 iterations) restated over numpy doubles; with count_early also the
    number of points that took the icdist < 0 exit."""
    xy = np.asarray(xy, np.float32).reshape(-1, 2)
    k = np.zeros(14)
    k[:len(dist)] = np.asarray(dist, np.float32).astype(np.float64)
    fx, fy, cx, cy = [np.float64(np.float32(v)) for v in K4]
    ifx, ify = 1. / fx, 1. / fy
    u, v = xy[:, 0].astype(np.float64), xy[:, 1].astype(np.float64)
    x, y = (u - cx) * ifx, (v - cy) * ify
    x0, y0 = x.copy(), y.copy()
    live = np.ones(len(u), bool)
    for _ in range(5):
        r2 = x * x + y * y
        icdist = (1 + ((k[7] * r2 + k[6]) * r2 + k[5]) * r2) / (1 + ((k[4] * r2 + k[1]) * r2 + k[0]) * r2)
        stop = live & (icdist < 0)
        x[stop], y[stop] = x0[stop], y0[stop]
        live &= ~stop
        dX = 2 * k[2] * x * y + k[3] * (r2 + 2 * x * x) + k[8] * r2 + k[9] * r2 * r2
        dY = k[2] * (r2 + 2 * y * y) + 2 * k[3] * x * y + k[10] * r2 + k[11] * r2 * r2
        x = np.where(live, (x0 - dX) * icdist, x)
        y = np.where(live, (y0 - dY) * icdist, y)
    out = np.stack([(fx * x + 0 * y + cx).astype(np.float32), (0 * x + fy * y + cy).astype(np.float32)], 1)
    return (out, int((~live).sum())) if count_early else out


def np_stereo_from_depth(kps, kps_un, depth, bf):
    """Frame::ComputeStereoFromRGBD (src/Frame.cc:1423-1461): (mvuRight, mvDepth)."""
    u = kps["x"].astype(np.int64)  # float -> int truncation, as imDepth.at<float>(v, u)
    v = kps["y"].astype(np.int64)
    d = depth[v, u].astype(np.float32)
    ok = d > 0
    ur = np.full(len(kps), -1, np.float32)
    dd = np.full(len(kps), -1, np.float32)
    dd[ok] = d[ok]
    with np.errstate(divide="ignore", invalid="ignore"):
        ur[ok] = kps_un["x"][ok].astype(np.float32) - np.float32(bf) / d[ok]
    return ur, dd


def bounds_from_corners(c):
    """Frame::ComputeImageBounds from the undistorted corners (0,0), (cols,0), (0,rows), (cols,rows)."""
    return np.float32([min(c[0, 0], c[2, 0]), max(c[1, 0], c[3, 0]), min(c[0, 1], c[1, 1]), max(c[2, 1], c[3, 1])])


def image_bounds(w, h, K4, dist, undistort):
    if dist[0] == 0:
        return np.float32([0, w, 0, h])
    return bounds_from_corners(undistort(np.float32([[0, 0], [w, 0], [0, h], [w, h]]), K4, dist))


class Oracle:
    def __init__(self):
        L = self.L = ctypes.CDLL(ORACLE_LIB)
        L.orc_undistort_points.argtypes = [vp, c_i, vp, vp, c_i, vp]
        L.orc_undistort_points.restype = None

    def undistort(self, xy, K4, dist):
        xy = np.ascontiguousarray(np.asarray(xy, np.float32).reshape(-1, 2))
        K4, dist = np.ascontiguousarray(K4, np.float32), np.ascontiguousarray(dist, np.float32)
        out = np.empty_like(xy)
        self.L.orc_undistort_points(xy.ctypes.data, len(xy), K4.ctypes.data, dist.ctypes.data, len(dist), out.ctypes.data)
        return out


kp_dtype = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"), ("octave", "<i4"),
                     ("class_id", "<i4")])


def _kps(a):
    k = np.zeros(len(a), kp_dtype)
    for i, f in enumerate(("x", "y", "size", "angle", "response")):
        k[f] = a[:, i]
    k["octave"] = a[:, 5].astype(np.int32)
    k["class_id"] = a[:, 6].astype(np.int32)
    return k


class RefMonoFrame:
    """The reference's monocular (depth None) or RGB-D Frame, built by its own constructor (src/Frame.cc:238-458) with
    ORBextractor(nf, 1.2, 8, 20, 7).  The construction runs on the glue's bump allocator, so the reference's extraction
    breaks DistributeOctTree's ties the way the oracle and the device do and mvKeys equals their keypoints."""

    def __init__(self, img, K4, dist, depth=None, nf=1000, bf=40.0):
        R = self.R = ctypes.CDLL(REF_LIB)
        R.ref_frame_mono_rgbd.argtypes = [vp, vp, c_i, c_i, c_i, c_f, c_i, c_i, c_i, vp, vp, c_i, c_f, c_f]
        R.ref_frame_get_un.argtypes = [vp] * 5
        R.ref_frame_get_un.restype = None
        R.ref_frame_features_in_area.argtypes = [c_f, c_f, c_f, c_i, c_i, vp, c_i]
        img = np.ascontiguousarray(img, np.uint8)
        h, w = img.shape
        K4, dist = np.ascontiguousarray(K4, np.float32), np.ascontiguousarray(dist, np.float32)
        dep = None if depth is None else np.ascontiguousarray(depth, np.float32)
        R.ref_frame_set_monotonic_allocator(1)
        self.N = R.ref_frame_mono_rgbd(img.ctypes.data, None if dep is None else dep.ctypes.data, w, h, nf, 1.2, 8, 20, 7,
                                       K4.ctypes.data, dist.ctypes.data, len(dist), bf, 40.0)
        R.ref_frame_set_monotonic_allocator(0)
        k, ku = np.zeros((self.N, 7), np.float32), np.zeros((self.N, 7), np.float32)
        self.uright, self.depth = np.zeros(self.N, np.float32), np.zeros(self.N, np.float32)
        self.bounds = np.zeros(4, np.float32)  # mnMinX, mnMaxX, mnMinY, mnMaxY
        R.ref_frame_get_un(k.ctypes.data, ku.ctypes.data, self.uright.ctypes.data, self.depth.ctypes.data,
                           self.bounds.ctypes.data)
        self.kps, self.kps_un = _kps(k), _kps(ku)

    def features_in_area(self, x, y, r, min_level=-1, max_level=-1):
        out = np.zeros(max(self.N, 1), np.int32)
        n = self.R.ref_frame_features_in_area(x, y, r, min_level, max_level, out.ctypes.data, len(out))
        assert n >= 0
        return out[:n].copy()


def depth_image(w, h, seed, special=True):
    """A float depth image in metres (0.3 .. 8 m) with, when `special`, blocks of 0, negative, NaN and +inf values."""
    rng = np.random.default_rng(seed)
    d = rng.uniform(0.3, 8.0, (h, w)).astype(np.float32)
    if special:
        for val in (0.0, -1.5, np.nan, np.inf, -0.0):
            m = rng.random((h, w)) < 0.04
            d[m] = val
    return d
