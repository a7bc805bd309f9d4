"""The Frame checkers of oracle/frame.mk behind one Python class: the reference's own Frame constructors
(oracle/_ref/libref_frame_seq.so) and the drop-in host/adapters/Frame_b200.cc (oracle/_ref/libadapter_frame.so), both
driven by oracle/ref_frame_seq_glue.cpp, and the calibrations of the reference's example settings."""
import ctypes
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libref_frame_seq.so")
ADAPTER_LIB = os.path.join(ROOT, "oracle", "_ref", "libadapter_frame.so")
vp, c_f, c_i = ctypes.c_void_p, ctypes.c_float, ctypes.c_int
GRID_COLS, GRID_ROWS = 64, 48

# (fx, fy, cx, cy), (k1, k2, p1, p2[, k3]), bf, ThDepth, nFeatures of Examples/{Stereo,RGB-D,Monocular}/*.yaml
STEREO = {
    "kitti": ((718.856, 718.856, 607.1928, 185.2157), (0.0, 0.0, 0.0, 0.0), 386.1448, 35.0, 2000),
    "euroc": ((435.2046959714599, 435.2046959714599, 367.4517211914062, 252.2008514404297), (0.0, 0.0, 0.0, 0.0),
              47.90639384423901, 35.0, 1200),
    # the EuRoC left camera before rectification (Examples/Monocular/EuRoC.yaml): k1 != 0, so mvKeysUn differs from the
    # mvKeys the stereo search reads
    "euroc_raw": ((458.654, 457.296, 367.215, 248.375), (-0.28340811, 0.07395907, 0.00019359, 1.76187114e-05), 47.90639384423901,
                  35.0, 1200),
}
TUM1 = (517.306408, 516.469215, 318.643040, 255.313989)
MONO = {
    "tum1": (TUM1, (0.262383, -0.953104, -0.005358, 0.002628, 1.163314)),
    "tum1_4": (TUM1, (0.262383, -0.953104, -0.005358, 0.002628)),  # k3 == 0: Tracking builds 4 coefficients
    "k1zero": (TUM1, (0.0, 0.0, 0.004, -0.002)),  # not undistorted: only k1 is tested
}

KP_FIELDS = ("x", "y", "size", "angle", "response", "octave", "class_id")


class FrameLib:
    """One of the two libraries.  Every frame and extractor lives in the library until reset()."""

    def __init__(self, path, monotonic):
        L = self.L = ctypes.CDLL(path)
        self.monotonic = monotonic
        L.rfs_reset.argtypes = [c_i]
        L.rfs_reset.restype = None
        L.rfs_extractor.argtypes = [c_i, c_f, c_i, c_i, c_i]
        L.rfs_stereo.argtypes = [c_i, c_i, vp, c_i, c_i, c_i, vp, c_i, c_i, c_i, vp, vp, c_i, c_f, c_f]
        L.rfs_mono_rgbd.argtypes = [c_i, vp, c_i, c_i, vp, vp, vp, c_i, c_f, c_f]
        L.rfs_copy.argtypes = [c_i]
        L.rfs_info.argtypes = [c_i, vp, vp]
        L.rfs_info.restype = None
        L.rfs_get.argtypes = [c_i] + [vp] * 8
        L.rfs_get.restype = None
        L.rfs_statics.argtypes = [vp, vp]
        L.rfs_statics.restype = None
        L.rfs_grid.argtypes = [c_i, vp, vp, c_i]
        L.rfs_features_in_area.argtypes = [c_i, c_f, c_f, c_f, c_i, c_i, vp, c_i]
        L.rfs_is_in_frustum.argtypes = [c_i, vp, vp, vp, vp, vp, c_i, c_f, vp, vp, vp]
        L.rfs_is_in_frustum.restype = None
        L.rfs_unproject_stereo.argtypes = [c_i, c_i, vp]
        L.rfs_pyramid_level.argtypes = [c_i, c_i, vp, vp]
        self._keep = []

    def reset(self):
        self._keep = []
        self.L.rfs_reset(self.monotonic)

    def extractor(self, nf, scale=1.2, nlevels=8, ini=20, mn=7):
        return self.L.rfs_extractor(nf, scale, nlevels, ini, mn)

    @staticmethod
    def _img(a):
        assert a.dtype == np.uint8 and a.strides[1] == 1
        return a

    def stereo(self, exL, exR, imL, imR, K4, dist, bf, th):
        imL, imR = self._img(imL), self._img(imR)
        K4, dist = np.ascontiguousarray(K4, np.float32), np.ascontiguousarray(dist, np.float32)
        return self.L.rfs_stereo(exL, exR, imL.ctypes.data, imL.shape[1], imL.shape[0], imL.strides[0], imR.ctypes.data,
                                 imR.shape[1], imR.shape[0], imR.strides[0], K4.ctypes.data, dist.ctypes.data, len(dist), bf, th)

    def mono_rgbd(self, ex, img, K4, dist, bf, th, depth=None):
        img = np.ascontiguousarray(img, np.uint8)
        K4, dist = np.ascontiguousarray(K4, np.float32), np.ascontiguousarray(dist, np.float32)
        d = None if depth is None else np.ascontiguousarray(depth, np.float32)
        h, w = img.shape
        return self.L.rfs_mono_rgbd(ex, img.ctypes.data, w, h, None if d is None else d.ctypes.data, K4.ctypes.data,
                                    dist.ctypes.data, len(dist), bf, th)

    def copy(self, f):
        return self.L.rfs_copy(f)

    def frame(self, f):
        """Every per-frame member the glue exposes, as numpy arrays."""
        counts = np.zeros(13, np.int64)
        sc = np.zeros(5, np.float32)
        self.L.rfs_info(f, counts.ctypes.data, sc.ctypes.data)
        N, nk, nku, nkr, nur, nd, nmp, mnId, nde, nder, L, nset, nout = [int(v) for v in counts]
        kps, kun, kr = np.zeros((nk, 7), np.float32), np.zeros((nku, 7), np.float32), np.zeros((nkr, 7), np.float32)
        desc, descr = np.zeros((nde, 32), np.uint8), np.zeros((nder, 32), np.uint8)
        ur, dp = np.zeros(nur, np.float32), np.zeros(nd, np.float32)
        tables = np.zeros((4, L), np.float32)
        self.L.rfs_get(f, kps.ctypes.data, kun.ctypes.data, kr.ctypes.data, desc.ctypes.data, descr.ctypes.data,
                       ur.ctypes.data, dp.ctypes.data, tables.ctypes.data)
        return dict(N=N, sizes=counts[1:7].copy(), mnId=mnId, mvbOutlier=nout, set_entries=nset, mnScaleLevels=L,
                    mvKeys=kps, mvKeysUn=kun, mvKeysRight=kr, mDescriptors=desc, mDescriptorsRight=descr, mvuRight=ur,
                    mvDepth=dp, mbf=sc[0:1], mb=sc[1:2], mThDepth=sc[2:3], mfScaleFactor=sc[3:4], mfLogScaleFactor=sc[4:5],
                    tables=tables)

    def statics(self):
        """(fx fy cx cy invfx invfy mnMinX mnMaxX mnMinY mnMaxY mfGridElementWidthInv mfGridElementHeightInv,
        nNextId, mbInitialComputations)"""
        v = np.zeros(12, np.float32)
        i = np.zeros(2, np.int64)
        self.L.rfs_statics(v.ctypes.data, i.ctypes.data)
        return v, int(i[0]), int(i[1])

    def grid(self, f):
        counts = np.zeros(GRID_COLS * GRID_ROWS, np.int32)
        idx = np.zeros(16384, np.int32)
        n = self.L.rfs_grid(f, counts.ctypes.data, idx.ctypes.data, len(idx))
        assert n >= 0
        return counts, idx[:n].copy()

    def features_in_area(self, f, x, y, r, lo=-1, hi=-1):
        out = np.zeros(16384, np.int32)
        n = self.L.rfs_features_in_area(f, x, y, r, lo, hi, out.ctypes.data, len(out))
        assert n >= 0
        return out[:n].copy()

    def is_in_frustum(self, f, T, pos, nrm, mind, maxd, cos_limit):
        n = len(pos)
        T, pos, nrm = [np.ascontiguousarray(a, np.float32) for a in (T, pos, nrm)]
        mind, maxd = np.ascontiguousarray(mind, np.float32), np.ascontiguousarray(maxd, np.float32)
        out, level, inv = np.zeros((n, 4), np.float32), np.zeros(n, np.int32), np.zeros(n, np.uint8)
        self.L.rfs_is_in_frustum(f, T.ctypes.data, pos.ctypes.data, nrm.ctypes.data, mind.ctypes.data, maxd.ctypes.data, n,
                                 cos_limit, out.ctypes.data, level.ctypes.data, inv.ctypes.data)
        return out, level, inv

    def unproject(self, f, i):
        xyz = np.zeros(3, np.float32)
        ok = self.L.rfs_unproject_stereo(f, i, xyz.ctypes.data)
        return xyz if ok else None

    def pyramid(self, ex):
        """[(w, h)] of the extractor's mvImagePyramid levels ((0, 0) = never written)"""
        w, h = ctypes.c_int(0), ctypes.c_int(0)
        n = self.L.rfs_pyramid_level(ex, 0, ctypes.byref(w), ctypes.byref(h))
        out = []
        for l in range(n):
            self.L.rfs_pyramid_level(ex, l, ctypes.byref(w), ctypes.byref(h))
            out.append((w.value, h.value))
        return out


def bits(a):
    a = np.ascontiguousarray(a, np.float32)
    return a.view(np.uint32)


def assert_same_frame(a, b, right=False):
    """Frame members of the two libraries, floats compared as bits."""
    assert a["N"] == b["N"]
    assert np.array_equal(a["sizes"], b["sizes"]), (a["sizes"], b["sizes"])
    assert a["mnId"] == b["mnId"] and a["mvbOutlier"] == b["mvbOutlier"] and a["set_entries"] == b["set_entries"] == 0
    for k in ("mvKeys", "mvKeysUn", "mvKeysRight"):
        assert a[k].shape == b[k].shape, k
        for i, f in enumerate(KP_FIELDS):
            assert np.array_equal(bits(a[k][:, i]), bits(b[k][:, i])), (k, f)
    for k in ("mDescriptors", "mDescriptorsRight", ):
        assert np.array_equal(a[k], b[k]), k
    for k in ("mvuRight", "mvDepth", "mbf", "mb", "mThDepth", "mfScaleFactor", "mfLogScaleFactor", "tables"):
        assert np.array_equal(bits(a[k]), bits(b[k])), k
    assert a["mnScaleLevels"] == b["mnScaleLevels"]
