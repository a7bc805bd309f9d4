"""self_commit_orb-slam2_b200 — H100-native hot path of ORB-SLAM2 (extract -> match -> LocalBA).

This package is a thin ctypes binding over ``libb200slam.so`` (hand-written sm_90a CUDA behind the C ABI of
``include/b200slam.h``).  The Python classes mirror the reference's operator interface
(``ORBextractor.__call__`` = ``ORBextractor::operator()``, ``ORBmatcher.SearchByBoW`` ...), so the tests read like
calls into the reference.  There is no CPU fallback: if the CUDA library is missing or no GPU is present the calls
raise ``B200SlamError``.

The directory name contains a dash, so import it with
``importlib.import_module("self_commit_orb-slam2_b200")`` (or ``from b200slam_loader import pkg`` in tests).
"""
import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200slam.so")

OK, ERR_NO_DEVICE, ERR_BAD_ARG, ERR_CUDA, ERR_CAPACITY, ERR_ABORTED = range(6)

keypoint_dtype = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"),
                           ("octave", "<i4"), ("class_id", "<i4")])
win_query_dtype = np.dtype([("u", "<f4"), ("v", "<f4"), ("ur", "<f4"), ("radius", "<f4"), ("min_level", "<i4"),
                            ("max_level", "<i4"), ("valid", "u1"), ("pad", "u1", 3), ("desc", "u1", 32)])
map_query_dtype = np.dtype([("u", "<f4"), ("v", "<f4"), ("ur", "<f4"), ("view_cos", "<f4"), ("level", "<i4"),
                            ("in_view", "u1"), ("has_obs", "u1"), ("pad", "u1", 2), ("desc", "u1", 32)])
proj_query_dtype = np.dtype([("u", "<f4"), ("v", "<f4"), ("invz", "<f4"), ("angle", "<f4"), ("octave", "<i4"),
                             ("has_obs", "<i4"), ("desc", "u1", 32)])
ba_edge_dtype = np.dtype([("kf", "<i4"), ("mp", "<i4"), ("obs", "<f4", 3), ("inv_sigma2", "<f4")])

TH_HIGH, TH_LOW, HISTO_LENGTH = 100, 50, 30  # src/ORBmatcher.cc:49-51


class B200SlamError(RuntimeError):
    def __init__(self, code, text):
        super().__init__("libb200slam error %d: %s" % (code, text))
        self.code = code


_vp = ctypes.c_void_p
_lib = None


class _FrameGeom(ctypes.Structure):
    _fields_ = [("mnMinX", ctypes.c_float), ("mnMinY", ctypes.c_float), ("mnMaxX", ctypes.c_float),
                ("mnMaxY", ctypes.c_float), ("bf", ctypes.c_float), ("scale_factors", _vp), ("nlevels", ctypes.c_int)]


class _KfFeatures(ctypes.Structure):
    _fields_ = [("desc", ctypes.c_void_p), ("node", ctypes.c_void_p), ("has_mp", ctypes.c_void_p),
                ("stereo", ctypes.c_void_p), ("x", ctypes.c_void_p), ("y", ctypes.c_void_p), ("octave", ctypes.c_void_p),
                ("angle", ctypes.c_void_p), ("n", ctypes.c_int32)]


class _BaProblem(ctypes.Structure):
    _fields_ = [("n_kf", ctypes.c_int), ("n_local", ctypes.c_int), ("Tcw", _vp), ("fixed", _vp), ("n_mp", ctypes.c_int),
                ("points", _vp), ("n_edges", ctypes.c_int), ("edges", _vp), ("fx", ctypes.c_float),
                ("fy", ctypes.c_float), ("cx", ctypes.c_float), ("cy", ctypes.c_float), ("bf", ctypes.c_float),
                ("its1", ctypes.c_int), ("its2", ctypes.c_int)]


class _BaResult(ctypes.Structure):
    _fields_ = [("Tcw_out", _vp), ("points_out", _vp), ("edge_outlier", _vp), ("trace", _vp),
                ("chi2_final", ctypes.c_double), ("n_trials", ctypes.c_int)]


class _PoseProblem(ctypes.Structure):
    _fields_ = [("Tcw", _vp), ("n", ctypes.c_int32), ("has_mp", _vp), ("Xw", _vp), ("kpx", _vp), ("kpy", _vp),
                ("uright", _vp), ("inv_sigma2", _vp), ("fx", ctypes.c_float), ("fy", ctypes.c_float),
                ("cx", ctypes.c_float), ("cy", ctypes.c_float), ("bf", ctypes.c_float)]


class _PoseResult(ctypes.Structure):
    _fields_ = [("Tcw_out", _vp), ("outlier", _vp), ("trace", _vp), ("n_inliers", ctypes.c_int32),
                ("n_trials", ctypes.c_int32)]


class _GbaProblem(ctypes.Structure):
    _fields_ = [("n_kf", ctypes.c_int), ("Tcw", _vp), ("fixed", _vp), ("n_mp", ctypes.c_int), ("points", _vp),
                ("n_edges", ctypes.c_int), ("edges", _vp), ("fx", ctypes.c_float), ("fy", ctypes.c_float),
                ("cx", ctypes.c_float), ("cy", ctypes.c_float), ("bf", ctypes.c_float), ("iterations", ctypes.c_int),
                ("robust", ctypes.c_int)]


class _EgProblem(ctypes.Structure):
    _fields_ = [("n_kf", ctypes.c_int), ("Siw", _vp), ("fixed_kf", ctypes.c_int), ("fix_scale", ctypes.c_int),
                ("n_edges", ctypes.c_int), ("edges", _vp), ("n_mp", ctypes.c_int), ("points", _vp), ("ref_kf", _vp)]


class _EgResult(ctypes.Structure):
    _fields_ = [("Tcw_out", _vp), ("points_out", _vp), ("trace", _vp), ("chi2_initial", ctypes.c_double),
                ("chi2_final", ctypes.c_double), ("n_trials", ctypes.c_int)]


# b2s_sim3_edge: EdgeSim3 between keyframes i (vertex 0) and j (vertex 1), measurement S_ji as qx qy qz qw tx ty tz s
sim3_edge_dtype = np.dtype([("i", np.int32), ("j", np.int32), ("meas", np.float64, 8)])


class _Sim3(ctypes.Structure):
    _fields_ = [("v", ctypes.c_double * 8)]  # b2s_sim3: qx qy qz qw tx ty tz s


class _Sim3Problem(ctypes.Structure):
    _fields_ = [("n", ctypes.c_int32), ("X1c", _vp), ("X2c", _vp), ("obs1", _vp), ("obs2", _vp), ("inv_sigma2_1", _vp),
                ("inv_sigma2_2", _vp)] + [(k, ctypes.c_float) for k in ("fx1", "fy1", "cx1", "cy1", "fx2", "fy2", "cx2",
                                                                         "cy2")] + [
        ("S12", _Sim3), ("th2", ctypes.c_float), ("fix_scale", ctypes.c_int32)]


class _Sim3Result(ctypes.Structure):
    _fields_ = [("S12_out", _Sim3), ("keep", _vp), ("trace", _vp), ("n_inliers", ctypes.c_int32),
                ("n_trials", ctypes.c_int32)]


class _InitProblem(ctypes.Structure):  # b2s_init_problem
    _fields_ = [("n1", ctypes.c_int32), ("n2", ctypes.c_int32), ("kp1", _vp), ("kp2", _vp), ("matches12", _vp),
                ("K", ctypes.c_float * 9), ("sigma", ctypes.c_float), ("iterations", ctypes.c_int32), ("sets", _vp)]


class _InitResult(ctypes.Structure):  # b2s_init_result
    _fields_ = [("ret", ctypes.c_int32), ("model", ctypes.c_int32), ("rt_state", ctypes.c_int32),
                ("R21", ctypes.c_float * 9), ("t21", ctypes.c_float * 3), ("p3d", _vp), ("triangulated", _vp),
                ("inliers_h", _vp), ("inliers_f", _vp), ("n_matches", ctypes.c_int32), ("best_h_iter", ctypes.c_int32),
                ("best_f_iter", ctypes.c_int32), ("SH", ctypes.c_float), ("SF", ctypes.c_float),
                ("RH", ctypes.c_float), ("H21", ctypes.c_float * 9), ("F21", ctypes.c_float * 9),
                ("n_hyp", ctypes.c_int32), ("n_good", ctypes.c_int32 * 8), ("parallax", ctypes.c_float * 8)]


class _Sim3SolverProblem(ctypes.Structure):  # b2s_sim3solver_problem
    _fields_ = [("n", ctypes.c_int32), ("X1c", _vp), ("X2c", _vp), ("sigma2_1", _vp), ("sigma2_2", _vp),
                ("K1", ctypes.c_float * 4), ("K2", ctypes.c_float * 4), ("fix_scale", ctypes.c_int32),
                ("min_inliers", ctypes.c_int32), ("max_its", ctypes.c_int32), ("iterations_done", ctypes.c_int32),
                ("best_inliers", ctypes.c_int32), ("k", ctypes.c_int32), ("sets", _vp)]


class _Sim3SolverResult(ctypes.Structure):  # b2s_sim3solver_result
    _fields_ = [("returned", ctypes.c_int32), ("T12", ctypes.c_float * 16), ("best_changed", ctypes.c_int32),
                ("R", ctypes.c_float * 9), ("t", ctypes.c_float * 3), ("s", ctypes.c_float), ("inliers", _vp),
                ("n_inliers", ctypes.c_int32), ("no_more", ctypes.c_int32), ("iterations_used", ctypes.c_int32),
                ("iterations_done", ctypes.c_int32), ("best_inliers", ctypes.c_int32)]


class _PnPsolverProblem(ctypes.Structure):  # b2s_pnpsolver_problem
    _fields_ = [("n", ctypes.c_int32), ("P3Dw", _vp), ("P2D", _vp), ("sigma2", _vp), ("fu", ctypes.c_float),
                ("fv", ctypes.c_float), ("uc", ctypes.c_float), ("vc", ctypes.c_float), ("th2", ctypes.c_float),
                ("min_inliers", ctypes.c_int32), ("max_its", ctypes.c_int32), ("min_set", ctypes.c_int32),
                ("iterations_done", ctypes.c_int32), ("best_inliers", ctypes.c_int32), ("best_Tcw", _vp),
                ("best_mask", _vp), ("k", ctypes.c_int32), ("sets", _vp)]


class _PnPsolverResult(ctypes.Structure):  # b2s_pnpsolver_result
    _fields_ = [("returned", ctypes.c_int32), ("Tcw", ctypes.c_float * 16), ("inliers", _vp),
                ("n_inliers", ctypes.c_int32), ("no_more", ctypes.c_int32), ("iterations_used", ctypes.c_int32),
                ("iterations_done", ctypes.c_int32), ("best_inliers", ctypes.c_int32), ("best_changed", ctypes.c_int32),
                ("best_Tcw", ctypes.c_float * 16), ("best_mask", _vp)]


class _GbaResult(ctypes.Structure):
    _fields_ = [("Tcw_out", _vp), ("points_out", _vp), ("point_included", _vp), ("trace", _vp),
                ("chi2_final", ctypes.c_double), ("n_trials", ctypes.c_int)]


def lib():
    """Loads libb200slam.so (built in-tree by build.py). Fails loudly if it is missing."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise B200SlamError(-1, "%s not found: run `python -c 'import __graft_entry__ as g; g.build()'` "
                                    "(there is no CPU fallback)" % LIB_PATH)
        L = ctypes.CDLL(LIB_PATH)
        L.b2s_last_error.restype = ctypes.c_char_p
        L.b2s_extractor_launch_count.restype = ctypes.c_longlong
        L.b2s_extractor_launch_count.argtypes = [_vp]
        L.b2s_extractor_create.argtypes = [ctypes.c_int, ctypes.c_float, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                           ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, _vp]
        L.b2s_extractor_destroy.argtypes = [_vp]
        L.b2s_extractor_destroy.restype = None
        L.b2s_extractor_tables.argtypes = [_vp] * 6
        L.b2s_extractor_max_keypoints.argtypes = [_vp]
        L.b2s_extract.argtypes = [_vp, _vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, _vp, _vp, ctypes.c_int, _vp, _vp]
        L.b2s_extract_batch.argtypes = [_vp, _vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, _vp, _vp,
                                        ctypes.c_int, _vp]
        L.b2s_extract_batch_device.argtypes = [_vp, _vp, ctypes.c_size_t, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                               ctypes.c_int, _vp, _vp, _vp, ctypes.c_int, _vp]
        L.b2s_extractor_check.argtypes = [_vp]
        L.b2s_extractor_set_timing.argtypes = [_vp, ctypes.c_int]
        L.b2s_extractor_get_timing.argtypes = [_vp, _vp, _vp]
        L.b2s_extractor_debug_level.argtypes = [_vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, _vp, _vp, _vp]
        L.b2s_extractor_debug_candidates.argtypes = [_vp, ctypes.c_int, ctypes.c_int, _vp, _vp, ctypes.c_int, _vp]
        if hasattr(L, "b2s_matcher_create"):
            L.b2s_matcher_create.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, _vp]
            L.b2s_matcher_destroy.argtypes = [_vp]
            L.b2s_matcher_destroy.restype = None
            L.b2s_matcher_launch_count.restype = ctypes.c_longlong
            L.b2s_matcher_launch_count.argtypes = [_vp]
            L.b2s_descriptor_distance.argtypes = [_vp, _vp, _vp, ctypes.c_int, _vp]
            L.b2s_search_by_bow.argtypes = [_vp, _vp, _vp, _vp, _vp, ctypes.c_int, _vp, _vp, _vp, _vp, ctypes.c_int,
                                            ctypes.c_int, ctypes.c_float, ctypes.c_int, ctypes.c_int, _vp, _vp]
            L.b2s_search_by_bow_batch.argtypes = [_vp, ctypes.c_int, _vp, _vp, _vp, _vp, _vp, ctypes.c_int, _vp, _vp, _vp,
                                                  _vp, _vp, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_int,
                                                  ctypes.c_int, _vp, _vp]
            L.b2s_search_by_bow_device.argtypes = [_vp, ctypes.c_int, _vp, _vp, _vp, _vp, _vp, ctypes.c_int, _vp, _vp,
                                                   _vp, _vp, _vp, ctypes.c_int, ctypes.c_int, ctypes.c_float,
                                                   ctypes.c_int, ctypes.c_int, _vp, _vp, _vp]
            L.b2s_search_by_projection_last.argtypes = [_vp, _vp, ctypes.c_int, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                                        ctypes.c_int, _vp, ctypes.c_float, ctypes.c_int, ctypes.c_int,
                                                        ctypes.c_int, _vp, _vp]
            L.b2s_search_by_projection_last_device.argtypes = [_vp, ctypes.c_int, _vp, _vp, ctypes.c_int, _vp, _vp, _vp, _vp,
                                                               ctypes.c_int, _vp, ctypes.c_float, ctypes.c_int,
                                                               ctypes.c_int, ctypes.c_int, _vp, _vp, _vp]
            L.b2s_search_by_projection_last_batch.argtypes = [_vp, ctypes.c_int, _vp, _vp, ctypes.c_int, _vp, _vp, _vp, _vp,
                                                              ctypes.c_int, _vp, ctypes.c_float, ctypes.c_int,
                                                              ctypes.c_int, ctypes.c_int, _vp, _vp]
            L.b2s_search_by_projection_sequence.argtypes = [_vp, ctypes.c_int, _vp, _vp, _vp, _vp, _vp, ctypes.c_int, _vp,
                                                            ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_float,
                                                            ctypes.c_int, _vp, ctypes.c_float, ctypes.c_int, ctypes.c_int,
                                                            ctypes.c_int, _vp, _vp]
            L.b2s_track_queries_device.argtypes = [_vp, ctypes.c_int, _vp, _vp, _vp, _vp, ctypes.c_int, _vp, ctypes.c_float,
                                                   ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_int, _vp, _vp,
                                                   _vp]
            L.b2s_search_by_projection_map.argtypes = [_vp, _vp, ctypes.c_int, _vp, _vp, _vp, _vp, _vp, _vp, ctypes.c_int,
                                                       _vp, ctypes.c_float, ctypes.c_int, ctypes.c_float, _vp, _vp]
        if hasattr(L, "b2s_ba_create"):
            L.b2s_ba_create.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, _vp]
            L.b2s_ba_destroy.argtypes = [_vp]
            L.b2s_ba_destroy.restype = None
            L.b2s_ba_launch_count.restype = ctypes.c_longlong
            L.b2s_ba_launch_count.argtypes = [_vp]
            L.b2s_ba_last_kernel_ms.restype = ctypes.c_float
            L.b2s_ba_last_kernel_ms.argtypes = [_vp, _vp]
            L.b2s_local_ba.argtypes = [_vp, _vp, _vp, _vp]
            L.b2s_ba_set_sm_budget.argtypes = [_vp, ctypes.c_int]
            L.b2s_local_ba_batch.argtypes = [_vp, ctypes.c_int, _vp, _vp]
            L.b2s_pose_optimization_batch.argtypes = [_vp, ctypes.c_int, _vp, _vp]
        if hasattr(L, "b2s_gba_create"):
            L.b2s_gba_create.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, _vp]
            L.b2s_gba_destroy.argtypes = [_vp]
            L.b2s_gba_destroy.restype = None
            L.b2s_global_ba.argtypes = [_vp, _vp, _vp, _vp]
            L.b2s_gba_last_ms.restype = ctypes.c_float
            L.b2s_gba_last_ms.argtypes = [_vp, _vp]
        if hasattr(L, "b2s_eg_create"):
            L.b2s_eg_create.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, _vp]
            L.b2s_eg_destroy.argtypes = [_vp]
            L.b2s_eg_destroy.restype = None
            L.b2s_optimize_essential_graph.argtypes = [_vp, _vp, _vp]
            L.b2s_eg_last_ms.restype = ctypes.c_float
            L.b2s_eg_last_ms.argtypes = [_vp, _vp]
        if hasattr(L, "b2s_sim3opt_create"):
            L.b2s_sim3opt_create.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, _vp]
            L.b2s_sim3opt_destroy.argtypes = [_vp]
            L.b2s_sim3opt_destroy.restype = None
            L.b2s_optimize_sim3.argtypes = [_vp, ctypes.c_int, _vp, _vp]
            L.b2s_sim3opt_last_ms.restype = ctypes.c_float
            L.b2s_sim3opt_last_ms.argtypes = [_vp, _vp]
        if hasattr(L, "b2s_init_create"):
            L.b2s_init_create.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, _vp]
            L.b2s_init_destroy.argtypes = [_vp]
            L.b2s_init_destroy.restype = None
            L.b2s_initialize.argtypes = [_vp, ctypes.c_int, _vp, _vp]
            L.b2s_init_last_ms.restype = ctypes.c_float
            L.b2s_init_last_ms.argtypes = [_vp]
        if hasattr(L, "b2s_sim3solver_create"):
            L.b2s_sim3solver_create.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, _vp]
            L.b2s_sim3solver_destroy.argtypes = [_vp]
            L.b2s_sim3solver_destroy.restype = None
            L.b2s_sim3solver_iterate.argtypes = [_vp, ctypes.c_int, _vp, _vp]
            L.b2s_sim3solver_last_ms.restype = ctypes.c_float
            L.b2s_sim3solver_last_ms.argtypes = [_vp]
        if hasattr(L, "b2s_pnpsolver_create"):
            L.b2s_pnpsolver_create.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, _vp]
            L.b2s_pnpsolver_destroy.argtypes = [_vp]
            L.b2s_pnpsolver_destroy.restype = None
            L.b2s_pnpsolver_iterate.argtypes = [_vp, ctypes.c_int, _vp, _vp]
            L.b2s_pnpsolver_last_ms.restype = ctypes.c_float
            L.b2s_pnpsolver_last_ms.argtypes = [_vp]
        _lib = L
    return _lib


def _check(rc):
    if rc != OK:
        raise B200SlamError(rc, lib().b2s_last_error().decode("utf-8", "replace"))


def _p(a):
    return None if a is None else a.ctypes.data_as(_vp)


def device_count():
    return lib().b2s_device_count()


class ORBextractor:
    """Mirror of ORB_SLAM2::ORBextractor (include/ORBextractor.h:92-161)."""

    def __init__(self, nfeatures, scaleFactor, nlevels, iniThFAST, minThFAST, max_width=1280, max_height=1024,
                 max_batch=1, device=0):
        self._h = _vp()
        self.nfeatures, self.nlevels = nfeatures, nlevels
        self.max_batch = max_batch
        _check(lib().b2s_extractor_create(nfeatures, scaleFactor, nlevels, iniThFAST, minThFAST, max_width, max_height,
                                          max_batch, device, ctypes.byref(self._h)))
        self.cap = lib().b2s_extractor_max_keypoints(self._h)
        s = [np.zeros(nlevels, np.float32) for _ in range(4)]
        nf = np.zeros(nlevels, np.int32)
        _check(lib().b2s_extractor_tables(self._h, _p(s[0]), _p(s[1]), _p(s[2]), _p(s[3]), _p(nf)))
        self.mvScaleFactor, self.mvInvScaleFactor, self.mvLevelSigma2, self.mvInvLevelSigma2 = s
        self.mnFeaturesPerLevel = nf
        self.mvImagePyramid = []

    def close(self):
        if self._h:
            lib().b2s_extractor_destroy(self._h)
            self._h = _vp()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # getters of include/ORBextractor.h:118-161
    def GetLevels(self):
        return self.nlevels

    def GetScaleFactors(self):
        return self.mvScaleFactor

    def GetInverseScaleFactors(self):
        return self.mvInvScaleFactor

    def GetScaleSigmaSquares(self):
        return self.mvLevelSigma2

    def GetInverseScaleSigmaSquares(self):
        return self.mvInvLevelSigma2

    def __call__(self, image, mask=None, want_pyramid=False):
        """operator()(image, mask, keypoints, descriptors): returns (keypoints[N], descriptors[N,32])."""
        if image is None or image.size == 0:
            return np.zeros(0, keypoint_dtype), np.zeros((0, 32), np.uint8)
        assert image.dtype == np.uint8 and image.ndim == 2  # assert(image.type() == CV_8UC1)
        h, w = image.shape
        kps = np.zeros(self.cap, keypoint_dtype)
        desc = np.zeros((self.cap, 32), np.uint8)
        n = ctypes.c_int(0)
        pyr_ptrs = None
        if want_pyramid:
            dims = self.level_dims(w, h)
            self.mvImagePyramid = [np.zeros((lh, lw), np.uint8) for (lw, lh) in dims]
            arr = (_vp * self.nlevels)(*[p.ctypes.data for p in self.mvImagePyramid])
            pyr_ptrs = ctypes.cast(arr, _vp)
        _check(lib().b2s_extract(self._h, image.ctypes.data_as(_vp), w, h, image.strides[0], _p(kps), _p(desc), self.cap,
                                 ctypes.byref(n), pyr_ptrs))
        return kps[:n.value].copy(), desc[:n.value].copy()

    def level_dims(self, w, h):
        return [(int(np.rint(np.float32(w) * s)), int(np.rint(np.float32(h) * s))) for s in self.mvInvScaleFactor]

    def extract_batch(self, images):
        B = len(images)
        h, w = images[0].shape
        kps = np.zeros((B, self.cap), keypoint_dtype)
        desc = np.zeros((B, self.cap, 32), np.uint8)
        n = np.zeros(B, np.int32)
        imgs = [np.ascontiguousarray(im) for im in images]
        ptrs = (_vp * B)(*[im.ctypes.data for im in imgs])
        _check(lib().b2s_extract_batch(self._h, ctypes.cast(ptrs, _vp), B, w, h, w, _p(kps), _p(desc), self.cap, _p(n)))
        return [(kps[b, :n[b]].copy(), desc[b, :n[b]].copy()) for b in range(B)]

    def extract_batch_device(self, d_imgs_ptr, img_pitch_bytes, batch, w, h, stride, d_kps_ptr, d_desc_ptr, d_counts_ptr,
                             cap, stream=None):
        _check(lib().b2s_extract_batch_device(self._h, _vp(d_imgs_ptr), img_pitch_bytes, batch, w, h, stride,
                                              _vp(d_kps_ptr), _vp(d_desc_ptr), _vp(d_counts_ptr), cap,
                                              _vp(stream) if stream else None))

    def stereo_match(self, first_left, first_right, n_pairs, bf, mb=0.0):
        """Frame::ComputeStereoMatches (src/Frame.cc:1026-1421) on the pairs of the batch extracted last with
        extract_batch(); returns (uright [n_pairs, cap], depth [n_pairs, cap], n_matched [n_pairs])."""
        ur = np.full((n_pairs, self.cap), -1, np.float32)
        dp = np.full((n_pairs, self.cap), -1, np.float32)
        nm = np.zeros(n_pairs, np.int32)
        L = lib()
        L.b2s_stereo_match.argtypes = [_vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float, _vp,
                                       _vp, ctypes.c_int, _vp]
        _check(L.b2s_stereo_match(self._h, first_left, first_right, n_pairs, float(bf), float(mb), _p(ur), _p(dp),
                                  self.cap, _p(nm)))
        return ur, dp, nm

    def stereo_match_device(self, first_left, first_right, n_pairs, d_kps_ptr, d_desc_ptr, d_counts_ptr, cap, bf, mb,
                            d_uright_ptr, d_depth_ptr, d_nmatched_ptr, stream=0):
        L = lib()
        L.b2s_stereo_match_device.argtypes = [_vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, _vp, _vp, _vp, ctypes.c_int,
                                              ctypes.c_float, ctypes.c_float, _vp, _vp, _vp, _vp]
        _check(L.b2s_stereo_match_device(self._h, first_left, first_right, n_pairs, _vp(d_kps_ptr), _vp(d_desc_ptr),
                                         _vp(d_counts_ptr), cap, float(bf), float(mb), _vp(d_uright_ptr),
                                         _vp(d_depth_ptr), _vp(d_nmatched_ptr), _vp(stream)))

    def check(self):
        _check(lib().b2s_extractor_check(self._h))

    def launch_count(self):
        return lib().b2s_extractor_launch_count(self._h)

    # test hooks
    def debug_level(self, b, level, blurred=False):
        w, h = ctypes.c_int(0), ctypes.c_int(0)
        _check(lib().b2s_extractor_debug_level(self._h, b, level, int(blurred), None, ctypes.byref(w), ctypes.byref(h)))
        out = np.zeros((h.value, w.value), np.uint8)
        _check(lib().b2s_extractor_debug_level(self._h, b, level, int(blurred), _p(out), None, None))
        return out

    def debug_candidates(self, b, level):
        n = ctypes.c_int(0)
        _check(lib().b2s_extractor_debug_candidates(self._h, b, level, None, None, 0, ctypes.byref(n)))
        cap = max(n.value, 1)
        xy = np.zeros((cap, 2), np.int32)
        resp = np.zeros(cap, np.int32)
        _check(lib().b2s_extractor_debug_candidates(self._h, b, level, _p(xy), _p(resp), cap, ctypes.byref(n)))
        return xy[:n.value].copy(), resp[:n.value].copy()


class ORBmatcher:
    """Mirror of ORB_SLAM2::ORBmatcher (include/ORBmatcher.h:57-215) on flattened arrays."""
    TH_HIGH, TH_LOW, HISTO_LENGTH = TH_HIGH, TH_LOW, HISTO_LENGTH

    def __init__(self, nnratio=0.6, checkOri=True, max_features=4096, max_batch=1, device=0):
        self.mfNNratio = np.float32(nnratio)
        self.mbCheckOrientation = bool(checkOri)
        self._h = _vp()
        _check(lib().b2s_matcher_create(max_features, max_batch, device, ctypes.byref(self._h)))

    def close(self):
        if self._h:
            lib().b2s_matcher_destroy(self._h)
            self._h = _vp()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def launch_count(self):
        return lib().b2s_matcher_launch_count(self._h)

    def DescriptorDistance(self, a, b):
        a = np.ascontiguousarray(a, np.uint8).reshape(-1, 32)
        b = np.ascontiguousarray(b, np.uint8).reshape(-1, 32)
        out = np.zeros(len(a), np.int32)
        _check(lib().b2s_descriptor_distance(self._h, _p(a), _p(b), len(a), _p(out)))
        return out

    def SearchByBoW(self, descA, nodeA, validA, angA, descB, nodeB, angB, validB=None, strict_lt=False, th_low=TH_LOW):
        nA, nB = len(descA), len(descB)
        match = np.full(nB, -1, np.int32)
        nm = ctypes.c_int(0)
        _check(lib().b2s_search_by_bow(self._h, _p(descA), _p(nodeA), _p(validA), _p(angA), nA, _p(descB), _p(nodeB),
                                       _p(validB), _p(angB), nB, th_low, float(self.mfNNratio), int(strict_lt),
                                       int(self.mbCheckOrientation), _p(match), ctypes.byref(nm)))
        return nm.value, match

    def SearchByProjection(self, queries, kpx, kpy, octave, angle, uright, occupied, desc, geom, th, mode=0,
                           th_high=TH_HIGH):
        nf = len(kpx)
        g, sf = self.frame_geom(geom)
        match = np.full(nf, -1, np.int32)
        nm = ctypes.c_int(0)
        _check(lib().b2s_search_by_projection_last(self._h, _p(queries), len(queries), _p(kpx), _p(kpy), _p(octave),
                                                   _p(angle), _p(uright), _p(occupied), _p(desc), nf, ctypes.byref(g),
                                                   float(th), mode, th_high, int(self.mbCheckOrientation), _p(match),
                                                   ctypes.byref(nm)))
        return nm.value, match


    @staticmethod
    def frame_geom(geom):
        """ctypes b2s_frame_geom (+ the array it points to, which the caller keeps alive) from a dict."""
        sf = np.ascontiguousarray(geom["scale_factors"], np.float32)
        return _FrameGeom(geom["mnMinX"], geom["mnMinY"], geom["mnMaxX"], geom["mnMaxY"], geom["bf"], sf.ctypes.data,
                          len(sf)), sf

    def track_queries_device(self, batch, d_kps_last, d_desc_last, d_depth_last, d_n_last, cap, d_Tcl, fx, fy, cx, cy, has_obs,
                             d_q, d_nq, stream=None):
        """Projection half of SearchByProjection(CurrentFrame, LastFrame) (src/ORBmatcher.cc:1600-1626) for `batch` stereo
        frame pairs on the device (b2s_track_queries_device); all d_* are device addresses."""
        _check(lib().b2s_track_queries_device(self._h, batch, _vp(d_kps_last), _vp(d_desc_last), _vp(d_depth_last),
                                              _vp(d_n_last), cap, _vp(d_Tcl), float(fx), float(fy), float(cx), float(cy),
                                              int(has_obs), _vp(d_q), _vp(d_nq), _vp(stream) if stream else None))

    def search_by_projection_last_device(self, batch, d_q, d_nq, cap_q, d_kps, d_uright, d_desc, d_nf, cap_f, geom, th, mode,
                                         d_match, d_nmatches, th_high=TH_HIGH, stream=None):
        """Batched device-resident SearchByProjection(CurrentFrame, LastFrame) (b2s_search_by_projection_last_device)."""
        g, keep = self.frame_geom(geom)
        _check(lib().b2s_search_by_projection_last_device(self._h, batch, _vp(d_q), _vp(d_nq), cap_q, _vp(d_kps), _vp(d_uright),
                                                          _vp(d_desc), _vp(d_nf), cap_f, ctypes.byref(g), float(th), int(mode),
                                                          th_high, int(self.mbCheckOrientation), _vp(d_match),
                                                          _vp(d_nmatches), _vp(stream) if stream else None))

    def SearchByProjectionBatch(self, queries, nq, kps, uright, desc, nf, geom, th, mode=0, th_high=TH_HIGH):
        """Host-buffer batch (b2s_search_by_projection_last_batch): queries [B, capQ] proj_query_dtype, kps [B, capF]
        keypoint_dtype, uright [B, capF] f32, desc [B, capF, 32] u8.  Returns (nmatches [B], match_cur [B, capF])."""
        queries, kps = np.ascontiguousarray(queries), np.ascontiguousarray(kps)
        uright, desc = np.ascontiguousarray(uright, np.float32), np.ascontiguousarray(desc, np.uint8)
        B, capQ = queries.shape
        capF = kps.shape[1]
        g, keep = self.frame_geom(geom)
        match = np.full((B, capF), -1, np.int32)
        nm = np.zeros(B, np.int32)
        nq = np.ascontiguousarray(nq, np.int32)
        nf = np.ascontiguousarray(nf, np.int32)
        _check(lib().b2s_search_by_projection_last_batch(self._h, B, _p(queries), _p(nq), capQ, _p(kps), _p(uright), _p(desc),
                                                         _p(nf), capF, ctypes.byref(g), float(th), int(mode), th_high,
                                                         int(self.mbCheckOrientation), _p(match), _p(nm)))
        return nm, match

    def SearchByProjectionSequence(self, kps, desc, depth, uright, n, Tcl, fx, fy, cx, cy, geom, th, mode=0, has_obs=1,
                                   th_high=TH_HIGH, out=None):
        """b2s_search_by_projection_sequence: kps / desc / depth of B + 1 consecutive frames ([B + 1, cap, ...], C-contiguous
        host arrays), uright [B, cap] of frames 1..B, Tcl [B, 12]; frame b + 1 is matched against frame b.  Returns
        (nmatches [B], match_cur [B, cap]) (written into `out` = (nm, match) when given)."""
        B, cap = uright.shape
        g, keep = self.frame_geom(geom)
        nm, match = out if out is not None else (np.zeros(B, np.int32), np.full((B, cap), -1, np.int32))
        _check(lib().b2s_search_by_projection_sequence(self._h, B, _p(kps), _p(desc), _p(depth), _p(uright), _p(n), cap, _p(Tcl),
                                                       float(fx), float(fy), float(cx), float(cy), int(has_obs),
                                                       ctypes.byref(g), float(th), int(mode), th_high,
                                                       int(self.mbCheckOrientation), _p(match), _p(nm)))
        return nm, match

    def SearchForInitialization(self, prev, octave1, angle1, desc1, kpx2, kpy2, octave2, angle2, desc2, geom, window=10,
                                th_low=TH_LOW):
        """ORBmatcher::SearchForInitialization (src/ORBmatcher.cc:515-643).  prev: [n1, 2] vbPrevMatched (updated in place
        like the reference does, :636-638).  Returns (nmatches, vnMatches12)."""
        n1, n2 = len(octave1), len(kpx2)
        prev_in = np.ascontiguousarray(prev, np.float32)
        px, py = np.ascontiguousarray(prev_in[:, 0]), np.ascontiguousarray(prev_in[:, 1])
        g, sf = self.frame_geom(geom)
        keep = [np.ascontiguousarray(octave1, np.int32), np.ascontiguousarray(angle1, np.float32),
                np.ascontiguousarray(desc1, np.uint8), np.ascontiguousarray(kpx2, np.float32),
                np.ascontiguousarray(kpy2, np.float32), np.ascontiguousarray(octave2, np.int32),
                np.ascontiguousarray(angle2, np.float32), np.ascontiguousarray(desc2, np.uint8)]
        m12 = np.full(n1, -1, np.int32)
        nm = ctypes.c_int(0)
        L = lib()
        L.b2s_search_for_initialization.argtypes = [_vp, _vp, _vp, _vp, _vp, _vp, ctypes.c_int, _vp, _vp, _vp, _vp, _vp,
                                                    ctypes.c_int, _vp, ctypes.c_int, ctypes.c_int, ctypes.c_float,
                                                    ctypes.c_int, _vp, _vp]
        _check(L.b2s_search_for_initialization(self._h, _p(px), _p(py), _p(keep[0]), _p(keep[1]), _p(keep[2]), n1, _p(keep[3]),
                                               _p(keep[4]), _p(keep[5]), _p(keep[6]), _p(keep[7]), n2, ctypes.byref(g),
                                               int(window), int(th_low), float(self.mfNNratio),
                                               int(self.mbCheckOrientation), _p(m12), ctypes.byref(nm)))
        hit = m12 >= 0
        prev[hit, 0] = keep[3][m12[hit]]
        prev[hit, 1] = keep[4][m12[hit]]
        return nm.value, m12

    def SearchByProjectionReloc(self, queries, kpx, kpy, octave, angle, occupied, desc, geom, th, orb_dist):
        """SearchByProjection(Frame& Cur, KeyFrame*, sAlreadyFound, th, ORBdist) (src/ORBmatcher.cc:1731-1862, relocalisation):
        queries = the keyframe's projected map points with octave = predicted level; occupied[j] = the frame feature holds
        any map point.  Same kernel as the last-frame search: levels [l-1, l+1], no stereo gate, th_high = ORBdist."""
        q = np.ascontiguousarray(queries).copy()
        q["invz"] = 1.0
        q["has_obs"] = 1
        return self.SearchByProjection(q, kpx, kpy, octave, angle, np.full(len(kpx), -1, np.float32), occupied, desc, geom, th,
                                       mode=0, th_high=orb_dist)

    def SearchByProjectionMap(self, queries, kpx, kpy, octave, uright, occupied, desc, geom, th=1.0, th_high=TH_HIGH):
        """SearchByProjection(Frame&, const vector<MapPoint*>&, th) (src/ORBmatcher.cc:70-175); queries: map_query_dtype."""
        nf = len(kpx)
        g, sf = self.frame_geom(geom)
        match = np.full(nf, -1, np.int32)
        nm = ctypes.c_int(0)
        _check(lib().b2s_search_by_projection_map(self._h, _p(queries), len(queries), _p(kpx), _p(kpy), _p(octave),
                                                  _p(uright), _p(occupied), _p(desc), nf, ctypes.byref(g), float(th),
                                                  th_high, float(self.mfNNratio), _p(match), ctypes.byref(nm)))
        return nm.value, match


    def SearchWindows(self, queries, kpx, kpy, octave, uright, inv_level_sigma2, occupied, desc, geom, chi2=False,
                      greedy=False, th_dist=TH_LOW):
        """Search core of Fuse (src/ORBmatcher.cc:1020-1174, :1179-1310) and SearchByProjection(KeyFrame*, Scw, ...)
        (:388-512); queries: win_query_dtype.  Returns (n_accepted, best_idx, best_dist)."""
        nq, nf = len(queries), len(kpx)
        g, sf = self.frame_geom(geom)
        best = np.full(nq, -1, np.int32)
        bdist = np.full(nq, 256, np.int32)
        nacc = ctypes.c_int(0)
        L = lib()
        L.b2s_search_windows.argtypes = [_vp, _vp, ctypes.c_int, _vp, _vp, _vp, _vp, _vp, _vp, _vp, ctypes.c_int, _vp,
                                         ctypes.c_int, ctypes.c_int, _vp, _vp, _vp]
        is2 = None if inv_level_sigma2 is None else np.ascontiguousarray(inv_level_sigma2, np.float32)
        _check(L.b2s_search_windows(self._h, _p(queries), nq, _p(kpx), _p(kpy), _p(octave), _p(uright), _p(is2),
                                    _p(occupied), _p(desc), nf, ctypes.byref(g), (1 if chi2 else 0) | (2 if greedy else 0),
                                    th_dist, _p(best), _p(bdist), ctypes.byref(nacc)))
        return nacc.value, best, bdist


    def DistinctiveDescriptors(self, desc, offsets):
        """MapPoint::ComputeDistinctiveDescriptors (src/MapPoint.cc:359-440) for a batch of map points."""
        desc = np.ascontiguousarray(desc, np.uint8)
        offsets = np.ascontiguousarray(offsets, np.int32)
        best = np.full(len(offsets) - 1, -1, np.int32)
        L = lib()
        L.b2s_distinctive_descriptors.argtypes = [_vp, _vp, _vp, ctypes.c_int, _vp]
        _check(L.b2s_distinctive_descriptors(self._h, _p(desc), _p(offsets), len(offsets) - 1, _p(best)))
        return best

    def SearchForTriangulation(self, kf1, kf2, F12, ex, ey, scale_factors, level_sigma2, only_stereo=False):
        """ORBmatcher::SearchForTriangulation (src/ORBmatcher.cc:810-1009). kf1/kf2: dicts with desc, node, has_mp, stereo,
        x, y, octave, angle.  Returns (nmatches, match12)."""
        keep = []

        def side(k):
            arrs = [np.ascontiguousarray(k["desc"], np.uint8), np.ascontiguousarray(k["node"], np.int32),
                    np.ascontiguousarray(k["has_mp"], np.uint8), np.ascontiguousarray(k["stereo"], np.uint8),
                    np.ascontiguousarray(k["x"], np.float32), np.ascontiguousarray(k["y"], np.float32),
                    np.ascontiguousarray(k["octave"], np.int32), np.ascontiguousarray(k["angle"], np.float32)]
            keep.append(arrs)
            return _KfFeatures(*[a.ctypes.data for a in arrs], len(arrs[0]))

        a, b = side(kf1), side(kf2)
        F = np.ascontiguousarray(F12, np.float32).reshape(9)
        sf = np.ascontiguousarray(scale_factors, np.float32)
        s2 = np.ascontiguousarray(level_sigma2, np.float32)
        match12 = np.full(a.n, -1, np.int32)
        nm = ctypes.c_int(0)
        L = lib()
        L.b2s_search_for_triangulation.argtypes = [_vp, _vp, _vp, _vp, ctypes.c_float, ctypes.c_float, _vp, _vp,
                                                   ctypes.c_int, ctypes.c_int, ctypes.c_int, _vp, _vp]
        _check(L.b2s_search_for_triangulation(self._h, ctypes.byref(a), ctypes.byref(b), _p(F), float(ex), float(ey), _p(sf),
                                              _p(s2), len(sf), int(only_stereo), int(self.mbCheckOrientation),
                                              _p(match12), ctypes.byref(nm)))
        return nm.value, match12


class _VocDesc(ctypes.Structure):
    _fields_ = [("k", ctypes.c_int32), ("L", ctypes.c_int32), ("n_nodes", ctypes.c_int32), ("parent", ctypes.c_void_p),
                ("leaf_flag", ctypes.c_void_p), ("desc", ctypes.c_void_p), ("weight", ctypes.c_void_p)]


class FrameGrid:
    """Frame::AssignFeaturesToGrid / GetFeaturesInArea (src/Frame.cc:461-491, 741-852) kept on the device: build once per
    frame, then run several projection matchers that upload only their queries (SURVEY §8f rank 4)."""

    def __init__(self, matcher, kpx=None, kpy=None, octave=None, angle=None, uright=None, desc=None, geom=None,
                 inv_level_sigma2=None, d_kps_ptr=None, d_desc_ptr=None, d_uright_ptr=None, nf=None, stream=0):
        self.matcher = matcher
        self._h = _vp()
        L = lib()
        L.b2s_frame_grid_create.argtypes = [_vp, _vp, _vp, _vp, _vp, _vp, _vp, ctypes.c_int, _vp, _vp, _vp]
        L.b2s_frame_grid_create_device.argtypes = [_vp, _vp, _vp, ctypes.c_int, _vp, _vp, _vp, _vp, _vp]
        L.b2s_frame_grid_destroy.argtypes = [_vp]
        L.b2s_frame_grid_destroy.restype = None
        L.b2s_frame_grid_size.argtypes = [_vp]
        L.b2s_frame_grid_features_in_area.argtypes = [_vp, ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_int,
                                                      ctypes.c_int, _vp, ctypes.c_int, _vp]
        L.b2s_search_by_projection_last_grid.argtypes = [_vp, _vp, _vp, ctypes.c_int, _vp, ctypes.c_float, ctypes.c_int,
                                                         ctypes.c_int, ctypes.c_int, _vp, _vp]
        L.b2s_search_by_projection_map_grid.argtypes = [_vp, _vp, _vp, ctypes.c_int, _vp, ctypes.c_float, ctypes.c_int,
                                                        ctypes.c_float, _vp, _vp]
        L.b2s_search_windows_grid.argtypes = [_vp, _vp, _vp, ctypes.c_int, _vp, ctypes.c_int, ctypes.c_int, _vp, _vp, _vp]
        g, sf = ORBmatcher.frame_geom(geom)
        is2 = None if inv_level_sigma2 is None else np.ascontiguousarray(inv_level_sigma2, np.float32)
        if d_kps_ptr is not None:
            _check(L.b2s_frame_grid_create_device(matcher._h, _vp(d_kps_ptr), _vp(d_desc_ptr), int(nf),
                                                  _vp(d_uright_ptr) if d_uright_ptr else None, ctypes.byref(g), _p(is2),
                                                  _vp(stream), ctypes.byref(self._h)))
        else:
            a = [np.ascontiguousarray(kpx, np.float32), np.ascontiguousarray(kpy, np.float32),
                 np.ascontiguousarray(octave, np.int32), np.ascontiguousarray(angle, np.float32),
                 np.ascontiguousarray(uright, np.float32), np.ascontiguousarray(desc, np.uint8)]
            _check(L.b2s_frame_grid_create(matcher._h, _p(a[0]), _p(a[1]), _p(a[2]), _p(a[3]), _p(a[4]), _p(a[5]), len(a[0]),
                                           ctypes.byref(g), _p(is2), ctypes.byref(self._h)))
        self.n = lib().b2s_frame_grid_size(self._h)

    def close(self):
        if self._h:
            lib().b2s_frame_grid_destroy(self._h)
            self._h = _vp()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def GetFeaturesInArea(self, x, y, r, minLevel=-1, maxLevel=-1):
        out = np.zeros(max(self.n, 1), np.int32)
        n = ctypes.c_int(0)
        _check(lib().b2s_frame_grid_features_in_area(self._h, float(x), float(y), float(r), int(minLevel), int(maxLevel),
                                                     _p(out), len(out), ctypes.byref(n)))
        return out[:n.value].copy()

    def SearchByProjection(self, queries, occupied, th, mode=0, th_high=TH_HIGH):
        m = np.full(self.n, -1, np.int32)
        nm = ctypes.c_int(0)
        q = np.ascontiguousarray(queries)
        occ = None if occupied is None else np.ascontiguousarray(occupied, np.uint8)
        _check(lib().b2s_search_by_projection_last_grid(self.matcher._h, self._h, _p(q), len(q), _p(occ), float(th), int(mode),
                                                        int(th_high), int(self.matcher.mbCheckOrientation), _p(m),
                                                        ctypes.byref(nm)))
        return nm.value, m

    def SearchByProjectionMap(self, queries, occupied, th=1.0, th_high=TH_HIGH):
        m = np.full(self.n, -1, np.int32)
        nm = ctypes.c_int(0)
        q = np.ascontiguousarray(queries)
        occ = None if occupied is None else np.ascontiguousarray(occupied, np.uint8)
        _check(lib().b2s_search_by_projection_map_grid(self.matcher._h, self._h, _p(q), len(q), _p(occ), float(th), int(th_high),
                                                       float(self.matcher.mfNNratio), _p(m), ctypes.byref(nm)))
        return nm.value, m

    def SearchWindows(self, queries, occupied, chi2=False, greedy=False, th_dist=TH_LOW):
        q = np.ascontiguousarray(queries)
        best = np.full(len(q), -1, np.int32)
        bd = np.full(len(q), 256, np.int32)
        na = ctypes.c_int(0)
        occ = None if occupied is None else np.ascontiguousarray(occupied, np.uint8)
        _check(lib().b2s_search_windows_grid(self.matcher._h, self._h, _p(q), len(q), _p(occ), (1 if chi2 else 0) | (2 if greedy else 0),
                                             int(th_dist), _p(best), _p(bd), ctypes.byref(na)))
        return na.value, best, bd


class ORBVocabulary:
    """Mirror of ORBVocabulary::transform (DBoW2 TemplatedVocabulary.h:1127-1256) on a flattened vocabulary."""

    def __init__(self, k, L, parent, leaf_flag, desc, weight, device=0):
        self._h = _vp()
        self._keep = [np.ascontiguousarray(parent, np.int32), np.ascontiguousarray(leaf_flag, np.uint8),
                      np.ascontiguousarray(desc, np.uint8), np.ascontiguousarray(weight, np.float64)]
        d = _VocDesc(k, L, len(self._keep[0]), *[a.ctypes.data for a in self._keep])
        L_ = lib()
        L_.b2s_vocabulary_create.argtypes = [_vp, ctypes.c_int, _vp]
        L_.b2s_vocabulary_destroy.argtypes = [_vp]
        L_.b2s_vocabulary_destroy.restype = None
        L_.b2s_bow_transform.argtypes = [_vp, _vp, ctypes.c_int, ctypes.c_int, _vp, _vp, _vp]
        L_.b2s_bow_transform_device.argtypes = [_vp, _vp, ctypes.c_int, ctypes.c_int, _vp, _vp, _vp, _vp]
        _check(L_.b2s_vocabulary_create(ctypes.byref(d), device, ctypes.byref(self._h)))

    def close(self):
        if self._h:
            lib().b2s_vocabulary_destroy(self._h)
            self._h = _vp()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def transform_features(self, features, levelsup=4):
        """Per feature (word_id, weight, node_id)."""
        features = np.ascontiguousarray(features, np.uint8)
        n = len(features)
        word = np.zeros(n, np.int32)
        w = np.zeros(n, np.float64)
        node = np.zeros(n, np.int32)
        _check(lib().b2s_bow_transform(self._h, _p(features), n, levelsup, _p(word), _p(w), _p(node)))
        return word, w, node

    def transform(self, features, levelsup=4):
        """transform(features, BowVector&, FeatureVector&, levelsup) (:1127-1187) for TF_IDF / L1: returns
        (bow: dict word -> value, feat: dict node -> [feature indices])."""
        word, w, node = self.transform_features(features, levelsup)
        bow, feat = {}, {}
        for i in range(len(word)):
            if w[i] > 0:  # not stopped
                bow[int(word[i])] = bow.get(int(word[i]), 0.0) + float(w[i])  # BowVector::addWeight, feature order
                feat.setdefault(int(node[i]), []).append(i)                   # FeatureVector::addFeature
        norm = 0.0
        for k in sorted(bow):  # BowVector::normalize(L1) iterates the std::map in key order
            norm += abs(bow[k])
        if norm > 0.0:
            for k in bow:
                bow[k] /= norm
        return bow, feat


class _KfdbState(ctypes.Structure):
    _fields_ = [("loop_query", ctypes.c_uint64), ("loop_words", ctypes.c_int32), ("loop_score", ctypes.c_float),
                ("reloc_query", ctypes.c_uint64), ("reloc_words", ctypes.c_int32), ("reloc_score", ctypes.c_float)]


class _KfdbCovis(ctypes.Structure):
    _fields_ = [("ids", _vp), ("n", _vp), ("n_rows", ctypes.c_int32)]


class KeyFrameDatabase:
    """Mirror of ORB_SLAM2::KeyFrameDatabase (include/KeyFrameDatabase.h) on the device (b2s_kfdb_*).

    A BowVector is (words, values): ascending uint32 word ids and their float64 values.  `covis` is the
    GetBestCovisibilityKeyFrames(10) table at query time, (ids [n_rows, 10] uint64, n [n_rows] int32) indexed by keyframe
    id, or None.  The Detect* methods return the candidate keyframe ids in the reference's order."""

    def __init__(self, n_words, device=0):
        self._h = _vp()
        L = lib()
        L.b2s_kfdb_create.argtypes = [ctypes.c_int, ctypes.c_int, _vp]
        L.b2s_kfdb_destroy.argtypes = [_vp]
        L.b2s_kfdb_destroy.restype = None
        L.b2s_kfdb_add.argtypes = [_vp, ctypes.c_uint64, _vp, _vp, ctypes.c_int]
        L.b2s_kfdb_erase.argtypes = [_vp, ctypes.c_uint64]
        L.b2s_kfdb_clear.argtypes = [_vp]
        L.b2s_kfdb_size.argtypes = [_vp, _vp]
        L.b2s_kfdb_detect_loop_candidates.argtypes = [_vp, ctypes.c_uint64, _vp, _vp, ctypes.c_int, _vp, ctypes.c_int,
                                                      ctypes.c_float, _vp, _vp, ctypes.c_int, _vp]
        L.b2s_kfdb_detect_relocalization_candidates.argtypes = [_vp, ctypes.c_uint64, _vp, _vp, ctypes.c_int, _vp, _vp,
                                                                ctypes.c_int, _vp]
        L.b2s_kfdb_keyframe_state.argtypes = [_vp, ctypes.c_uint64, _vp]
        L.b2s_kfdb_last_query_ms.argtypes = [_vp]
        L.b2s_kfdb_last_query_ms.restype = ctypes.c_float
        _check(L.b2s_kfdb_create(int(n_words), device, ctypes.byref(self._h)))

    def close(self):
        if self._h:
            lib().b2s_kfdb_destroy(self._h)
            self._h = _vp()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @staticmethod
    def _bow(words, values):
        return np.ascontiguousarray(words, np.uint32), np.ascontiguousarray(values, np.float64)

    def add(self, kf_id, words, values):
        w, v = self._bow(words, values)
        _check(lib().b2s_kfdb_add(self._h, int(kf_id), _p(w), _p(v), len(w)))

    def erase(self, kf_id):
        _check(lib().b2s_kfdb_erase(self._h, int(kf_id)))

    def clear(self):
        _check(lib().b2s_kfdb_clear(self._h))

    def size(self):
        n = ctypes.c_int(0)
        _check(lib().b2s_kfdb_size(self._h, ctypes.byref(n)))
        return n.value

    @staticmethod
    def _covis(covis):
        if covis is None:
            return _KfdbCovis(None, None, 0), None
        ids = np.ascontiguousarray(covis[0], np.uint64).reshape(-1, 10)
        n = np.ascontiguousarray(covis[1], np.int32)
        assert len(n) == len(ids)
        return _KfdbCovis(ids.ctypes.data, n.ctypes.data, len(n)), (ids, n)

    def _detect(self, fn, *args, covis):
        c, keep = self._covis(covis)
        cap = self.size() + 1
        out = np.zeros(cap, np.uint64)
        n = ctypes.c_int(0)
        _check(fn(self._h, *args, ctypes.byref(c), _p(out), cap, ctypes.byref(n)))
        return out[:n.value].tolist()

    def DetectLoopCandidates(self, kf_id, words, values, connected, min_score, covis=None):
        w, v = self._bow(words, values)
        conn = np.ascontiguousarray(list(connected), np.uint64)
        return self._detect(lib().b2s_kfdb_detect_loop_candidates, int(kf_id), _p(w), _p(v), len(w), _p(conn), len(conn),
                            float(min_score), covis=covis)

    def DetectRelocalizationCandidates(self, frame_id, words, values, covis=None):
        w, v = self._bow(words, values)
        return self._detect(lib().b2s_kfdb_detect_relocalization_candidates, int(frame_id), _p(w), _p(v), len(w),
                            covis=covis)

    def keyframe_state(self, kf_id):
        """(mnLoopQuery, mnLoopWords, mLoopScore, mnRelocQuery, mnRelocWords, mRelocScore) of keyframe kf_id."""
        s = _KfdbState()
        _check(lib().b2s_kfdb_keyframe_state(self._h, int(kf_id), ctypes.byref(s)))
        return (s.loop_query, s.loop_words, s.loop_score, s.reloc_query, s.reloc_words, s.reloc_score)

    def last_query_ms(self):
        """Device time of the last query's kernels (CUDA events on the database's stream)."""
        return float(lib().b2s_kfdb_last_query_ms(self._h))


class Optimizer:
    """Mirror of ORB_SLAM2::Optimizer::LocalBundleAdjustment (include/Optimizer.h:112) on a flattened window."""

    def __init__(self, max_kf=64, max_mp=8192, max_edges=65536, max_batch=1, device=0):
        self._h = _vp()
        _check(lib().b2s_ba_create(max_kf, max_mp, max_edges, max_batch, device, ctypes.byref(self._h)))

    def close(self):
        if self._h:
            lib().b2s_ba_destroy(self._h)
            self._h = _vp()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def launch_count(self):
        return lib().b2s_ba_launch_count(self._h)

    def set_sm_budget(self, sms):
        """SMs one batched LocalBA call may occupy (b2s_ba_set_sm_budget); 0 = all."""
        _check(lib().b2s_ba_set_sm_budget(self._h, int(sms)))

    def last_kernel_ms(self):
        """(ms, trials): duration of the persistent LM kernel of the last LocalBundleAdjustment(Batch) call, measured with
        CUDA events on the solver's stream, and the LM trials it ran over all windows."""
        n = ctypes.c_longlong(0)
        ms = lib().b2s_ba_last_kernel_ms(self._h, ctypes.byref(n))
        return float(ms), int(n.value)

    @staticmethod
    def _problem(d, its1=5, its2=10):
        keep = dict(Tcw=np.ascontiguousarray(d["Tcw"], np.float32), fixed=np.ascontiguousarray(d["fixed"], np.uint8),
                    points=np.ascontiguousarray(d["points"], np.float32), edges=np.ascontiguousarray(d["edges"]))
        assert keep["edges"].dtype == ba_edge_dtype
        p = _BaProblem(d["n_kf"], d["n_local"], keep["Tcw"].ctypes.data, keep["fixed"].ctypes.data, len(keep["points"]),
                       keep["points"].ctypes.data, len(keep["edges"]), keep["edges"].ctypes.data, d["fx"], d["fy"],
                       d["cx"], d["cy"], d["bf"], its1, its2)
        return p, keep

    @staticmethod
    def _result(d):
        out = dict(Tcw=np.zeros((d["n_local"], 16), np.float32), points=np.zeros((len(d["points"]), 3), np.float32),
                   outlier=np.zeros(len(d["edges"]), np.uint8), trace=np.full(256, -1, np.int32))
        r = _BaResult(out["Tcw"].ctypes.data, out["points"].ctypes.data, out["outlier"].ctypes.data,
                      out["trace"].ctypes.data, 0.0, 0)
        return r, out

    def LocalBundleAdjustment(self, d, stop=None, its1=5, its2=10):
        p, keep = self._problem(d, its1, its2)
        r, out = self._result(d)
        rc = lib().b2s_local_ba(self._h, ctypes.byref(p), _p(stop), ctypes.byref(r))
        if rc == ERR_ABORTED:
            return None
        _check(rc)
        out["chi2"] = r.chi2_final
        out["n_trials"] = r.n_trials
        return out

    def PoseOptimizationBatch(self, ds):
        """Optimizer::PoseOptimization (src/Optimizer.cc:363-605) for a batch of independent frames; ds: dicts with Tcw,
        has_mp, Xw, kpx, kpy, uright, inv_sigma2, fx, fy, cx, cy, bf.  Returns a list of result dicts."""
        B = len(ds)
        probs, ress, keep, outs = (_PoseProblem * B)(), (_PoseResult * B)(), [], []
        for i, d in enumerate(ds):
            a = dict(Tcw=np.ascontiguousarray(d["Tcw"], np.float32).reshape(16),
                     has_mp=np.ascontiguousarray(d["has_mp"], np.uint8), Xw=np.ascontiguousarray(d["Xw"], np.float32),
                     kpx=np.ascontiguousarray(d["kpx"], np.float32), kpy=np.ascontiguousarray(d["kpy"], np.float32),
                     uright=np.ascontiguousarray(d["uright"], np.float32),
                     inv_sigma2=np.ascontiguousarray(d["inv_sigma2"], np.float32))
            n = len(a["has_mp"])
            o = dict(Tcw=np.zeros(16, np.float32), outlier=np.zeros(max(n, 1), np.uint8), trace=np.full(256, -1, np.int32))
            keep.append((a, o))
            probs[i] = _PoseProblem(a["Tcw"].ctypes.data, n, a["has_mp"].ctypes.data, a["Xw"].ctypes.data,
                                    a["kpx"].ctypes.data, a["kpy"].ctypes.data, a["uright"].ctypes.data,
                                    a["inv_sigma2"].ctypes.data, float(d["fx"]), float(d["fy"]), float(d["cx"]),
                                    float(d["cy"]), float(d["bf"]))
            ress[i] = _PoseResult(o["Tcw"].ctypes.data, o["outlier"].ctypes.data, o["trace"].ctypes.data, 0, 0)
            outs.append((o, n))
        _check(lib().b2s_pose_optimization_batch(self._h, B, ctypes.cast(probs, _vp), ctypes.cast(ress, _vp)))
        return [dict(n_inliers=ress[i].n_inliers, n_trials=ress[i].n_trials, Tcw=o["Tcw"], outlier=o["outlier"][:n],
                     trace=o["trace"]) for i, (o, n) in enumerate(outs)]

    def PoseOptimization(self, d):
        return self.PoseOptimizationBatch([d])[0]

    # ---- prepared batches: the ctypes problem / result arrays are built once, a step is then one C call (stream.py)
    def prepare_pose_batch(self, ds):
        B = len(ds)
        probs, ress, keep = (_PoseProblem * B)(), (_PoseResult * B)(), []
        for i, d in enumerate(ds):
            a = [np.ascontiguousarray(d["Tcw"], np.float32).reshape(16), np.ascontiguousarray(d["has_mp"], np.uint8),
                 np.ascontiguousarray(d["Xw"], np.float32), np.ascontiguousarray(d["kpx"], np.float32),
                 np.ascontiguousarray(d["kpy"], np.float32), np.ascontiguousarray(d["uright"], np.float32),
                 np.ascontiguousarray(d["inv_sigma2"], np.float32)]
            n = len(a[1])
            o = [np.zeros(16, np.float32), np.zeros(max(n, 1), np.uint8)]
            keep.append((a, o))
            probs[i] = _PoseProblem(a[0].ctypes.data, n, a[1].ctypes.data, a[2].ctypes.data, a[3].ctypes.data,
                                    a[4].ctypes.data, a[5].ctypes.data, a[6].ctypes.data, float(d["fx"]), float(d["fy"]),
                                    float(d["cx"]), float(d["cy"]), float(d["bf"]))
            ress[i] = _PoseResult(o[0].ctypes.data, o[1].ctypes.data, None, 0, 0)
        return dict(B=B, probs=probs, ress=ress, keep=keep)

    def run_prepared_pose(self, prep):
        _check(lib().b2s_pose_optimization_batch(self._h, prep["B"], ctypes.cast(prep["probs"], _vp),
                                                 ctypes.cast(prep["ress"], _vp)))
        return prep["ress"]

    def prepare_ba_batch(self, ds, its1=5, its2=10):
        B = len(ds)
        probs, ress, keeps, outs = (_BaProblem * B)(), (_BaResult * B)(), [], []
        for i, d in enumerate(ds):
            p, keep = self._problem(d, its1, its2)
            r, out = self._result(d)
            probs[i], ress[i] = p, r
            keeps.append(keep)
            outs.append(out)
        return dict(B=B, probs=probs, ress=ress, keeps=keeps, outs=outs)

    def run_prepared_ba(self, prep):
        _check(lib().b2s_local_ba_batch(self._h, prep["B"], ctypes.cast(prep["probs"], _vp), ctypes.cast(prep["ress"], _vp)))
        for i in range(prep["B"]):
            prep["outs"][i]["chi2"] = prep["ress"][i].chi2_final
            prep["outs"][i]["n_trials"] = prep["ress"][i].n_trials
        return prep["outs"]

    def LocalBundleAdjustmentBatch(self, ds, its1=5, its2=10):
        return self.run_prepared_ba(self.prepare_ba_batch(ds, its1, its2))


class GlobalOptimizer:
    """Mirror of ORB_SLAM2::Optimizer::BundleAdjustment (include/Optimizer.h, src/Optimizer.cc:86-341), the body of
    GlobalBundleAdjustemnt, on a flattened map (b2s_global_ba).  The handle's capacities bound the problem sizes; the
    reduced-system storage grows with the maps it is given."""

    def __init__(self, max_kf=2048, max_mp=262144, max_edges=1 << 21, device=0):
        self._h = _vp()
        _check(lib().b2s_gba_create(max_kf, max_mp, max_edges, device, ctypes.byref(self._h)))

    def close(self):
        if self._h:
            lib().b2s_gba_destroy(self._h)
            self._h = _vp()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def last_ms(self):
        """(ms, trials): device time of the last call (its stream segments between the host's LM decisions, CUDA
        events) and the LM trials it ran."""
        n = ctypes.c_longlong(0)
        ms = lib().b2s_gba_last_ms(self._h, ctypes.byref(n))
        return float(ms), int(n.value)

    def BundleAdjustment(self, d, iterations=10, robust=True, stop=None):
        """d: Tcw (n_kf x 16, the non-bad keyframes by ascending mnId), fixed (n_kf), points (n_mp x 3, the non-bad map
        points by ascending mnId), edges (ba_edge_dtype, grouped by point, one per (keyframe, point)), fx, fy, cx, cy, bf.
        Returns Tcw (every keyframe), points (rows of excluded points keep their input), point_included, trace, n_trials,
        chi2 (robustified chi2 of the returned estimate)."""
        keep = dict(Tcw=np.ascontiguousarray(d["Tcw"], np.float32).reshape(-1, 16),
                    fixed=np.ascontiguousarray(d["fixed"], np.uint8),
                    points=np.ascontiguousarray(d["points"], np.float32).reshape(-1, 3),
                    edges=np.ascontiguousarray(d["edges"]))
        assert keep["edges"].dtype == ba_edge_dtype
        nkf, nmp = len(keep["Tcw"]), len(keep["points"])
        p = _GbaProblem(nkf, keep["Tcw"].ctypes.data, keep["fixed"].ctypes.data, nmp, keep["points"].ctypes.data,
                        len(keep["edges"]), keep["edges"].ctypes.data, float(d["fx"]), float(d["fy"]), float(d["cx"]),
                        float(d["cy"]), float(d["bf"]), int(iterations), int(bool(robust)))
        out = dict(Tcw=np.zeros((nkf, 16), np.float32), points=keep["points"].copy(),
                   point_included=np.zeros(nmp, np.uint8), trace=np.full(256, -1, np.int32))
        r = _GbaResult(out["Tcw"].ctypes.data, out["points"].ctypes.data, out["point_included"].ctypes.data,
                       out["trace"].ctypes.data, 0.0, 0)
        _check(lib().b2s_global_ba(self._h, ctypes.byref(p), _p(stop), ctypes.byref(r)))
        out["chi2"] = r.chi2_final
        out["n_trials"] = r.n_trials
        return out


class EssentialGraphOptimizer:
    """Mirror of ORB_SLAM2::Optimizer::OptimizeEssentialGraph (src/Optimizer.cc:1017-1339) on a flattened pose graph
    (b2s_optimize_essential_graph).  The handle's capacities bound the problem sizes; the factorisation's tile storage
    grows with the graphs it is given."""

    def __init__(self, max_kf=4096, max_edges=1 << 17, max_mp=1 << 22, device=0):
        self._h = _vp()
        _check(lib().b2s_eg_create(max_kf, max_edges, max_mp, device, ctypes.byref(self._h)))

    def close(self):
        if self._h:
            lib().b2s_eg_destroy(self._h)
            self._h = _vp()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def last_ms(self):
        """(ms, trials): device time of the last call (CUDA events) and the LM trials it ran."""
        n = ctypes.c_longlong(0)
        ms = lib().b2s_eg_last_ms(self._h, ctypes.byref(n))
        return float(ms), int(n.value)

    def OptimizeEssentialGraph(self, d):
        """d: Siw (n_kf x 8: qx qy qz qw tx ty tz s, the keyframes by ascending mnId), fixed_kf, fix_scale, edges
        (sim3_edge_dtype, in the reference's insertion order), points (n_mp x 3), ref_kf (n_mp, -1: unchanged).
        Returns Tcw (every keyframe), points, trace, n_trials, chi2_initial, chi2_final."""
        keep = dict(Siw=np.ascontiguousarray(d["Siw"], np.float64).reshape(-1, 8),
                    edges=np.ascontiguousarray(d["edges"]),
                    points=np.ascontiguousarray(d["points"], np.float32).reshape(-1, 3),
                    ref_kf=np.ascontiguousarray(d["ref_kf"], np.int32))
        assert keep["edges"].dtype == sim3_edge_dtype
        nkf, nmp = len(keep["Siw"]), len(keep["points"])
        p = _EgProblem(nkf, keep["Siw"].ctypes.data, int(d["fixed_kf"]), int(bool(d["fix_scale"])), len(keep["edges"]),
                       keep["edges"].ctypes.data, nmp, keep["points"].ctypes.data, keep["ref_kf"].ctypes.data)
        out = dict(Tcw=np.zeros((nkf, 16), np.float32), points=np.zeros((nmp, 3), np.float32),
                   trace=np.full(256, -1, np.int32))
        r = _EgResult(out["Tcw"].ctypes.data, out["points"].ctypes.data, out["trace"].ctypes.data, 0.0, 0.0, 0)
        _check(lib().b2s_optimize_essential_graph(self._h, ctypes.byref(p), ctypes.byref(r)))
        out["chi2_initial"] = r.chi2_initial
        out["chi2"] = r.chi2_final
        out["n_trials"] = r.n_trials
        return out


class Sim3Optimizer:
    """Mirror of ORB_SLAM2::Optimizer::OptimizeSim3 (src/Optimizer.cc:1364-1590) on flattened correspondences
    (b2s_optimize_sim3).  A batch of independent problems runs in one launch."""

    def __init__(self, max_matches=4096, max_batch=64, device=0):
        self._h = _vp()
        _check(lib().b2s_sim3opt_create(max_matches, max_batch, device, ctypes.byref(self._h)))

    def close(self):
        if self._h:
            lib().b2s_sim3opt_destroy(self._h)
            self._h = _vp()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def last_ms(self):
        """(ms, trials): device time of the last call (CUDA events) and the LM trials of all its problems."""
        n = ctypes.c_longlong(0)
        ms = lib().b2s_sim3opt_last_ms(self._h, ctypes.byref(n))
        return float(ms), int(n.value)

    def OptimizeSim3(self, d):
        """d: X1c, X2c (n x 3 float32), obs1, obs2 (n x 2), inv_sigma2_1, inv_sigma2_2 (n), K1, K2 (fx fy cx cy), S12
        (qx qy qz qw tx ty tz s), th2, fix_scale.  Returns S12, keep (n, uint8), trace, n_inliers, n_trials."""
        return self.OptimizeSim3Batch([d])[0]

    def OptimizeSim3Batch(self, ds):
        keep, probs, outs = [], (_Sim3Problem * len(ds))(), []
        res = (_Sim3Result * len(ds))()
        for i, d in enumerate(ds):
            a = dict(X1c=np.ascontiguousarray(d["X1c"], np.float32).reshape(-1, 3),
                     X2c=np.ascontiguousarray(d["X2c"], np.float32).reshape(-1, 3),
                     obs1=np.ascontiguousarray(d["obs1"], np.float32).reshape(-1, 2),
                     obs2=np.ascontiguousarray(d["obs2"], np.float32).reshape(-1, 2),
                     inv_sigma2_1=np.ascontiguousarray(d["inv_sigma2_1"], np.float32).reshape(-1),
                     inv_sigma2_2=np.ascontiguousarray(d["inv_sigma2_2"], np.float32).reshape(-1))
            keep.append(a)
            n = len(a["X1c"])
            P = probs[i]
            P.n = n
            for k in a:
                setattr(P, k, a[k].ctypes.data)
            for k, v in zip(("fx1", "fy1", "cx1", "cy1"), d["K1"]):
                setattr(P, k, float(v))
            for k, v in zip(("fx2", "fy2", "cx2", "cy2"), d["K2"]):
                setattr(P, k, float(v))
            P.S12.v[:] = [float(v) for v in np.asarray(d["S12"], np.float64).reshape(8)]
            P.th2 = float(d["th2"])
            P.fix_scale = int(bool(d["fix_scale"]))
            out = dict(keep=np.zeros(n, np.uint8), trace=np.full(256, -1, np.int32))
            outs.append(out)
            res[i].keep = out["keep"].ctypes.data
            res[i].trace = out["trace"].ctypes.data
        _check(lib().b2s_optimize_sim3(self._h, len(ds), probs, res))
        for i, out in enumerate(outs):
            out["S12"] = np.array(res[i].S12_out.v[:], np.float64)
            out["n_inliers"] = res[i].n_inliers
            out["n_trials"] = res[i].n_trials
        return outs


class MonoInitializer:
    """Mirror of ORB_SLAM2::Initializer::Initialize (src/Initializer.cc:68-231) with the minimal sets given
    (b2s_initialize): H and F RANSAC over the sets, the model choice and the two-view reconstruction.  A batch of
    independent problems runs in one call."""

    def __init__(self, max_keys=4096, max_iterations=300, max_batch=64, device=0):
        self._h = _vp()
        _check(lib().b2s_init_create(max_keys, max_iterations, max_batch, device, ctypes.byref(self._h)))

    def close(self):
        if self._h:
            lib().b2s_init_destroy(self._h)
            self._h = _vp()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def last_ms(self):
        """Device time of the last call (CUDA events: upload, kernels, download)."""
        return float(lib().b2s_init_last_ms(self._h))

    def Initialize(self, d):
        """d: kp1 (n1 x 2, mvKeysUn of the reference frame), kp2 (n2 x 2), matches12 (n1, -1: unmatched), K (3 x 3),
        sigma, sets (iterations x 8, indices into the matches compacted in frame-1 order).  Returns ret, model (1: H,
        2: F), rt_state (1 written, -1 emptied, 0 untouched), R21 (3 x 3), t21 (3), p3d (n1 x 3) and triangulated (n1)
        (None unless ret), n_matches, SH, SF, RH, best_h_iter, best_f_iter, H21, F21 (3 x 3), inliers_h, inliers_f
        (n_matches, bool), n_good and parallax (per motion hypothesis checked)."""
        return self.InitializeBatch([d])[0]

    def InitializeBatch(self, ds):
        keep, probs, outs = [], (_InitProblem * len(ds))(), []
        res = (_InitResult * len(ds))()
        for i, d in enumerate(ds):
            a = dict(kp1=np.ascontiguousarray(d["kp1"], np.float32).reshape(-1, 2),
                     kp2=np.ascontiguousarray(d["kp2"], np.float32).reshape(-1, 2),
                     matches12=np.ascontiguousarray(d["matches12"], np.int32).reshape(-1),
                     sets=np.ascontiguousarray(d["sets"], np.int32).reshape(-1, 8))
            keep.append(a)
            P = probs[i]
            P.n1, P.n2, P.iterations = len(a["kp1"]), len(a["kp2"]), len(a["sets"])
            for k in a:
                setattr(P, k, a[k].ctypes.data)
            P.K[:] = [float(v) for v in np.asarray(d["K"], np.float32).reshape(9)]
            P.sigma = float(d["sigma"])
            nm = int((a["matches12"] >= 0).sum())
            out = dict(p3d=np.zeros((P.n1, 3), np.float32), triangulated=np.zeros(P.n1, np.uint8),
                       inliers_h=np.zeros(max(nm, 1), np.uint8), inliers_f=np.zeros(max(nm, 1), np.uint8))
            outs.append(out)
            for k in out:
                setattr(res[i], k, out[k].ctypes.data)
        _check(lib().b2s_initialize(self._h, len(ds), probs, res))
        for r, out in zip(res, outs):
            n = r.n_matches
            out.update(ret=r.ret, model=r.model, rt_state=r.rt_state, n_matches=n, SH=np.float32(r.SH),
                       SF=np.float32(r.SF), RH=np.float32(r.RH), best_h_iter=r.best_h_iter, best_f_iter=r.best_f_iter,
                       R21=np.array(r.R21[:], np.float32).reshape(3, 3), t21=np.array(r.t21[:], np.float32),
                       H21=np.array(r.H21[:], np.float32).reshape(3, 3), F21=np.array(r.F21[:], np.float32).reshape(3, 3),
                       n_good=np.array(r.n_good[:r.n_hyp], np.int32), parallax=np.array(r.parallax[:r.n_hyp], np.float32))
            out["inliers_h"] = out["inliers_h"][:n].astype(bool)
            out["inliers_f"] = out["inliers_f"][:n].astype(bool)
            out["triangulated"] = out["triangulated"].astype(bool)
            if not r.ret:
                out["p3d"] = out["triangulated"] = None
        return outs


def _c_log(x):
    """C's log, with its IEEE special cases."""
    import math
    return math.log(x) if 0 < x < math.inf else (-math.inf if x == 0 else (x if x > 0 else math.nan))


def _x86_int(x):
    """A float or double converted to int as x86 converts it (truncation; NaN and out-of-range values become
    INT_MIN)."""
    import math
    return int(x) if math.isfinite(x) and -2 ** 31 <= math.trunc(x) < 2 ** 31 else -2 ** 31


def _ransac_iterations(probability, epsilon, power):
    """ceil(log(1-p) / log(1-pow(epsilon, power))) in double, converted to int as x86 converts it."""
    import math
    with np.errstate(all="ignore"):
        c = float(np.float64(_c_log(1 - probability)) / np.float64(_c_log(1 - math.pow(epsilon, power))))
    return _x86_int(math.ceil(c) if math.isfinite(c) else c)


def sim3_ransac_max_its(n, probability=0.99, min_inliers=6, max_iterations=300):
    """Sim3Solver::SetRansacParameters (src/Sim3Solver.cc:143-196) on the host: the mRansacMaxIts it leaves for n
    correspondences.  epsilon = min_inliers / n is a float; the iteration count ceil(log(1-p) / log(1-epsilon^3)) is
    double, converted to int as x86 converts (NaN and out-of-range values become INT_MIN); min_inliers == n gives 1; the
    result is max(1, min(count, max_iterations))."""
    with np.errstate(all="ignore"):
        if min_inliers == n:
            it = 1
        else:
            it = _ransac_iterations(probability, float(np.float32(min_inliers) / np.float32(n)), 3)
    return max(1, min(it, max_iterations))


def pnp_ransac_parameters(n, probability=0.99, min_inliers=8, max_iterations=300, min_set=4, epsilon=0.4):
    """PnPsolver::SetRansacParameters (src/PnPsolver.cc:181-230) on the host: (mRansacMinInliers, mRansacMaxIts) for n
    correspondences.  min_inliers is raised to (int)(n*epsilon) (a float product, converted as x86 converts) and to
    min_set; epsilon is raised to the float min_inliers / n; the iteration count is ceil(log(1-p) / log(1-epsilon^3)) in
    double (3, although the minimal set is 4), 1 when min_inliers == n; the result is max(1, min(count,
    max_iterations)).  The reference's defaults."""
    with np.errstate(all="ignore"):
        eps = np.float32(epsilon)
        m = _x86_int(float(np.float32(n) * eps))
        m = max(m, int(min_inliers), int(min_set))
        q = np.float32(m) / np.float32(n) if n else np.float32(np.inf)
        if eps < q:
            eps = q
        it = 1 if m == n else _ransac_iterations(probability, float(eps), 3)
    return m, max(1, min(it, int(max_iterations)))


class Sim3Solver:
    """Mirror of ORB_SLAM2::Sim3Solver (src/Sim3Solver.cc) for one loop candidate, with the minimal sets drawn by the
    caller (b2s_sim3solver_iterate).  The constructor takes what the reference's constructor keeps: X1c / X2c (n x 3,
    mvX3Dc1 / mvX3Dc2), sigma2_1 / sigma2_2 (n, mvLevelSigma2 of each keypoint's octave), K1 / K2 (fx, fy, cx, cy) and
    fix_scale; the object keeps mnIterations, mnBestInliers and the best model across calls as the reference does.
    `iterate` and `find` run on the device; `iterate_batch` runs the calls of many solvers in one launch sequence."""

    def __init__(self, X1c, X2c, sigma2_1, sigma2_2, K1, K2, fix_scale=True, max_matches=None, max_sets=300,
                 device=0, _handle=None):
        self.X1c = np.ascontiguousarray(X1c, np.float32).reshape(-1, 3)
        self.X2c = np.ascontiguousarray(X2c, np.float32).reshape(-1, 3)
        self.sigma2_1 = np.ascontiguousarray(sigma2_1, np.float32).reshape(-1)
        self.sigma2_2 = np.ascontiguousarray(sigma2_2, np.float32).reshape(-1)
        self.K1 = [float(v) for v in np.asarray(K1, np.float32).reshape(4)]
        self.K2 = [float(v) for v in np.asarray(K2, np.float32).reshape(4)]
        self.fix_scale = bool(fix_scale)
        self.N = len(self.X1c)
        self.iterations = 0
        self.best_inliers = 0
        self.R = self.t = self.s = None
        self.set_ransac_parameters()
        self._own = _handle is None
        self._h = _handle._h if _handle is not None else _vp()
        if self._own:
            _check(lib().b2s_sim3solver_create(max(3, max_matches or self.N), max_sets, 1, device,
                                               ctypes.byref(self._h)))

    def close(self):
        if self._own and self._h:
            lib().b2s_sim3solver_destroy(self._h)
        self._h = _vp()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def last_ms(self):
        """Device time of the last call (CUDA events: upload, kernels, download)."""
        return float(lib().b2s_sim3solver_last_ms(self._h))

    def set_ransac_parameters(self, probability=0.99, min_inliers=6, max_iterations=300):
        """SetRansacParameters: resets the iteration count, keeps the best inlier count."""
        self.min_inliers = int(min_inliers)
        self.max_its = sim3_ransac_max_its(self.N, probability, min_inliers, max_iterations)
        self.iterations = 0

    def sets_needed(self, n_iterations):
        """How many minimal sets iterate(n_iterations) may consume: 0 when N < min_inliers (the reference draws
        nothing), else min(n_iterations, max_its - iterations)."""
        if self.N < self.min_inliers:
            return 0
        return max(0, min(int(n_iterations), self.max_its - self.iterations))

    def iterate(self, n_iterations, sets):
        """iterate(n_iterations) with its minimal sets (at least sets_needed(n_iterations) rows of 3 indices into
        [0, N), in draw order; the extra rows are ignored).  Returns a dict: T12 (4 x 4, or None for the empty matrix),
        no_more, inliers (N, compacted order), n_inliers, iterations_used."""
        return Sim3Solver.iterate_batch([self], [n_iterations], [sets])[0]

    def find(self, sets):
        """find(): iterate(mRansacMaxIts)."""
        return self.iterate(self.max_its, sets)

    @staticmethod
    def iterate_batch(solvers, n_iterations, sets, handle=None):
        """One iterate call per solver, all in one device call (on `handle`, a Sim3SolverBatch, or the first solver's
        handle)."""
        h = handle._h if handle is not None else solvers[0]._h
        probs = (_Sim3SolverProblem * len(solvers))()
        res = (_Sim3SolverResult * len(solvers))()
        keep, outs = [], []
        for i, (sv, nit, st) in enumerate(zip(solvers, n_iterations, sets)):
            k = sv.sets_needed(nit)
            st = np.ascontiguousarray(np.asarray(st, np.int32).reshape(-1, 3)[:k])
            if len(st) < k:
                raise ValueError("iterate: %d sets given, %d needed" % (len(st), k))
            keep.append(st)
            P = probs[i]
            P.n, P.X1c, P.X2c = sv.N, sv.X1c.ctypes.data, sv.X2c.ctypes.data
            P.sigma2_1, P.sigma2_2 = sv.sigma2_1.ctypes.data, sv.sigma2_2.ctypes.data
            P.K1[:], P.K2[:] = sv.K1, sv.K2
            P.fix_scale, P.min_inliers, P.max_its = int(sv.fix_scale), sv.min_inliers, sv.max_its
            P.iterations_done, P.best_inliers, P.k, P.sets = sv.iterations, sv.best_inliers, k, st.ctypes.data
            out = np.zeros(max(sv.N, 1), np.uint8)
            outs.append(out)
            res[i].inliers = out.ctypes.data
        _check(lib().b2s_sim3solver_iterate(h, len(solvers), probs, res))
        ret = []
        for sv, r, out in zip(solvers, res, outs):
            sv.iterations, sv.best_inliers = r.iterations_done, r.best_inliers
            if r.best_changed:
                sv.R = np.array(r.R[:], np.float32).reshape(3, 3)
                sv.t = np.array(r.t[:], np.float32).reshape(3, 1)
                sv.s = np.float32(r.s)
            ret.append(dict(T12=np.array(r.T12[:], np.float32).reshape(4, 4) if r.returned else None,
                            no_more=bool(r.no_more), inliers=out[:sv.N].astype(bool), n_inliers=r.n_inliers,
                            iterations_used=r.iterations_used))
        return ret

    def GetEstimatedRotation(self):
        return None if self.R is None else self.R.copy()

    def GetEstimatedTranslation(self):
        return None if self.t is None else self.t.copy()

    def GetEstimatedScale(self):
        return self.s


class Sim3SolverBatch:
    """A device handle sized for batched Sim3Solver.iterate_batch calls (max_matches per solver, max_sets per call,
    max_batch solvers)."""

    def __init__(self, max_matches=4096, max_sets=300, max_batch=64, device=0):
        self._h = _vp()
        _check(lib().b2s_sim3solver_create(max_matches, max_sets, max_batch, device, ctypes.byref(self._h)))

    def close(self):
        if self._h:
            lib().b2s_sim3solver_destroy(self._h)
            self._h = _vp()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def last_ms(self):
        return float(lib().b2s_sim3solver_last_ms(self._h))

    def solver(self, *args, **kw):
        """A Sim3Solver on this handle (Sim3Solver's constructor arguments)."""
        return Sim3Solver(*args, _handle=self, **kw)


class PnPsolver:
    """Mirror of ORB_SLAM2::PnPsolver (src/PnPsolver.cc) for one relocalisation candidate, with the minimal sets drawn by
    the caller (b2s_pnpsolver_iterate).  The constructor takes what the reference's constructor keeps: P3Dw (n x 3,
    mvP3Dw), P2D (n x 2, mvP2D), sigma2 (n, mvLevelSigma2 of each keypoint's octave) and K (fx, fy, cx, cy); the object
    keeps mnIterations, mnBestInliers, mBestTcw and mvbBestInliers across calls as the reference does.  `iterate` and
    `find` run on the device; `iterate_batch` runs the calls of many solvers in one launch sequence."""

    def __init__(self, P3Dw, P2D, sigma2, K, max_matches=None, max_sets=300, device=0, _handle=None):
        self.P3Dw = np.ascontiguousarray(P3Dw, np.float32).reshape(-1, 3)
        self.P2D = np.ascontiguousarray(P2D, np.float32).reshape(-1, 2)
        self.sigma2 = np.ascontiguousarray(sigma2, np.float32).reshape(-1)
        self.K = [float(v) for v in np.asarray(K, np.float32).reshape(4)]
        self.N = len(self.P3Dw)
        self.iterations = 0
        self.best_inliers = 0
        self.best_Tcw = np.eye(4, dtype=np.float32)
        self.best_mask = np.zeros(max(self.N, 1), np.uint8)
        self.set_ransac_parameters()
        self._own = _handle is None
        self._h = _handle._h if _handle is not None else _vp()
        if self._own:
            _check(lib().b2s_pnpsolver_create(max(4, max_matches or self.N), max_sets, 1, device, ctypes.byref(self._h)))

    def close(self):
        if self._own and self._h:
            lib().b2s_pnpsolver_destroy(self._h)
        self._h = _vp()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def last_ms(self):
        """Device time of the last call (CUDA events: upload, kernels, download)."""
        return float(lib().b2s_pnpsolver_last_ms(self._h))

    def set_ransac_parameters(self, probability=0.99, min_inliers=8, max_iterations=300, min_set=4, epsilon=0.4,
                              th2=5.991):
        """SetRansacParameters with the reference's defaults.  Like the reference it resets neither the iteration
        count nor the best model.  Only min_set = 4 is supported (the device rejects any other)."""
        self.min_inliers, self.max_its = pnp_ransac_parameters(self.N, probability, min_inliers, max_iterations,
                                                               min_set, epsilon)
        self.min_set = int(min_set)
        self.th2 = float(np.float32(th2))

    def sets_needed(self, n_iterations):
        """How many minimal sets iterate(n_iterations) may consume: 0 when N < min_inliers (the reference draws
        nothing), else max(n_iterations, max_its - iterations): the loop runs while either bound is not reached."""
        if self.N < self.min_inliers:
            return 0
        return max(0, int(n_iterations), self.max_its - self.iterations)

    def iterate(self, n_iterations, sets):
        """iterate(n_iterations) with its minimal sets (at least sets_needed(n_iterations) rows of 4 indices into
        [0, N), in draw order; the extra rows are ignored).  Returns a dict: Tcw (4 x 4, or None for the empty matrix),
        no_more, inliers (N, compacted order), n_inliers, iterations_used."""
        return PnPsolver.iterate_batch([self], [n_iterations], [sets])[0]

    def find(self, sets):
        """find(): iterate(mRansacMaxIts)."""
        return self.iterate(self.max_its, sets)

    @staticmethod
    def iterate_batch(solvers, n_iterations, sets, handle=None):
        """One iterate call per solver, all in one device call (on `handle`, a PnPsolverBatch, or the first solver's
        handle)."""
        h = handle._h if handle is not None else solvers[0]._h
        probs = (_PnPsolverProblem * len(solvers))()
        res = (_PnPsolverResult * len(solvers))()
        keep, outs = [], []
        for i, (sv, nit, st) in enumerate(zip(solvers, n_iterations, sets)):
            k = sv.sets_needed(nit)
            st = np.ascontiguousarray(np.asarray(st, np.int32).reshape(-1, 4)[:k])
            if len(st) < k:
                raise ValueError("iterate: %d sets given, %d needed" % (len(st), k))
            tcw = np.ascontiguousarray(sv.best_Tcw, np.float32)
            keep += [st, tcw]
            P = probs[i]
            P.n, P.P3Dw, P.P2D, P.sigma2 = sv.N, sv.P3Dw.ctypes.data, sv.P2D.ctypes.data, sv.sigma2.ctypes.data
            P.fu, P.fv, P.uc, P.vc, P.th2 = sv.K + [sv.th2]
            P.min_inliers, P.max_its, P.min_set = sv.min_inliers, sv.max_its, sv.min_set
            P.iterations_done, P.best_inliers = sv.iterations, sv.best_inliers
            P.best_Tcw, P.best_mask, P.k, P.sets = tcw.ctypes.data, sv.best_mask.ctypes.data, k, st.ctypes.data
            out, bm = np.zeros(max(sv.N, 1), np.uint8), np.zeros(max(sv.N, 1), np.uint8)
            outs.append((out, bm))
            res[i].inliers, res[i].best_mask = out.ctypes.data, bm.ctypes.data
        _check(lib().b2s_pnpsolver_iterate(h, len(solvers), probs, res))
        ret = []
        for sv, r, (out, bm) in zip(solvers, res, outs):
            sv.iterations, sv.best_inliers = r.iterations_done, r.best_inliers
            sv.best_Tcw = np.array(r.best_Tcw[:], np.float32).reshape(4, 4)
            sv.best_mask = bm
            ret.append(dict(Tcw=np.array(r.Tcw[:], np.float32).reshape(4, 4) if r.returned else None,
                            no_more=bool(r.no_more), inliers=out[:sv.N].astype(bool), n_inliers=r.n_inliers,
                            iterations_used=r.iterations_used))
        return ret


class PnPsolverBatch:
    """A device handle sized for batched PnPsolver.iterate_batch calls (max_matches per solver, max_sets per call,
    max_batch solvers)."""

    def __init__(self, max_matches=4096, max_sets=300, max_batch=64, device=0):
        self._h = _vp()
        _check(lib().b2s_pnpsolver_create(max_matches, max_sets, max_batch, device, ctypes.byref(self._h)))

    def close(self):
        if self._h:
            lib().b2s_pnpsolver_destroy(self._h)
            self._h = _vp()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def last_ms(self):
        return float(lib().b2s_pnpsolver_last_ms(self._h))

    def solver(self, *args, **kw):
        """A PnPsolver on this handle (PnPsolver's constructor arguments)."""
        return PnPsolver(*args, _handle=self, **kw)
