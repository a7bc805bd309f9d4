"""ctypes binding of oracle/liborb_oracle.so — the CPU checker (test infrastructure only)."""
import ctypes
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
ORACLE_LIB = os.path.join(ORACLE_DIR, "liborb_oracle.so")
vp = ctypes.c_void_p

kp_dtype = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"),
                     ("octave", "<i4"), ("class_id", "<i4")])
proj_query_dtype = np.dtype([("u", "<f4"), ("v", "<f4"), ("invz", "<f4"), ("angle", "<f4"), ("octave", "<i4"),
                             ("has_obs", "<i4"), ("desc", "u1", 32)])
ba_edge_dtype = np.dtype([("kf", "<i4"), ("mp", "<i4"), ("obs", "<f4", 3), ("inv_sigma2", "<f4")])


class FrameGeom(ctypes.Structure):
    _fields_ = [("mnMinX", ctypes.c_float), ("mnMinY", ctypes.c_float), ("mnMaxX", ctypes.c_float),
                ("mnMaxY", ctypes.c_float), ("bf", ctypes.c_float), ("scale_factors", vp), ("nlevels", ctypes.c_int)]


class BaProblem(ctypes.Structure):
    _fields_ = [("n_kf", ctypes.c_int), ("n_local", ctypes.c_int), ("Tcw", vp), ("fixed", vp), ("n_mp", ctypes.c_int),
                ("points", vp), ("n_edges", ctypes.c_int), ("edges", vp), ("fx", ctypes.c_float), ("fy", ctypes.c_float),
                ("cx", ctypes.c_float), ("cy", ctypes.c_float), ("bf", ctypes.c_float), ("its1", ctypes.c_int),
                ("its2", ctypes.c_int)]


class BaResult(ctypes.Structure):
    _fields_ = [("Tcw_out", vp), ("points_out", vp), ("edge_outlier", vp), ("trace", vp), ("chi2_final", ctypes.c_double),
                ("n_trials", ctypes.c_int)]


class PoseProblem(ctypes.Structure):
    _fields_ = [("Tcw", vp), ("n", ctypes.c_int32), ("has_mp", vp), ("Xw", vp), ("kpx", vp), ("kpy", vp),
                ("uright", vp), ("inv_sigma2", vp), ("fx", ctypes.c_float), ("fy", ctypes.c_float),
                ("cx", ctypes.c_float), ("cy", ctypes.c_float), ("bf", ctypes.c_float)]


class PoseResult(ctypes.Structure):
    _fields_ = [("Tcw_out", vp), ("outlier", vp), ("trace", vp), ("n_trials", ctypes.c_int32)]


def P(a):
    return None if a is None else a.ctypes.data_as(vp)


def call_pose_optimization(fn, d):
    """fn(const orc_pose_problem*, orc_pose_result*) -> inliers: the oracle's orc_pose_optimization or the reference's own
    Optimizer::PoseOptimization behind oracle/ref_optimizer_glue.cpp (same flattened problem)."""
    arrs = pose_problem_arrays(d)
    n = len(arrs["has_mp"])
    p = PoseProblem(arrs["Tcw"].ctypes.data, n, arrs["has_mp"].ctypes.data, arrs["Xw"].ctypes.data, arrs["kpx"].ctypes.data,
                    arrs["kpy"].ctypes.data, arrs["uright"].ctypes.data, arrs["inv_sigma2"].ctypes.data, d["fx"], d["fy"],
                    d["cx"], d["cy"], d["bf"])
    Tout = np.zeros(16, np.float32)
    outl = np.zeros(n, np.uint8)
    trace = np.full(256, -1, np.int32)
    r = PoseResult(Tout.ctypes.data, outl.ctypes.data, trace.ctypes.data, 0)
    fn.argtypes = [vp, vp]
    ninl = fn(ctypes.byref(p), ctypes.byref(r))
    return dict(n_inliers=ninl, Tcw=Tout, outlier=outl, trace=trace, n_trials=r.n_trials)


def call_local_ba(fn, d, stop=None, its1=5, its2=10):
    """fn(const orc_ba_problem*, const uint8_t* stop, orc_ba_result*): orc_local_ba or ref_local_ba."""
    Tcw = np.ascontiguousarray(d["Tcw"], np.float32)
    fixed = np.ascontiguousarray(d["fixed"], np.uint8)
    pts = np.ascontiguousarray(d["points"], np.float32)
    edges = np.ascontiguousarray(d["edges"])
    p = BaProblem(d["n_kf"], d["n_local"], Tcw.ctypes.data, fixed.ctypes.data, len(pts), pts.ctypes.data, len(edges),
                  edges.ctypes.data, d["fx"], d["fy"], d["cx"], d["cy"], d["bf"], its1, its2)
    out = dict(Tcw=np.zeros((d["n_local"], 16), np.float32), points=np.zeros((len(pts), 3), np.float32),
               outlier=np.zeros(len(edges), np.uint8), trace=np.full(256, -1, np.int32))
    r = BaResult(out["Tcw"].ctypes.data, out["points"].ctypes.data, out["outlier"].ctypes.data,
                 out["trace"].ctypes.data, 0.0, 0)
    fn.argtypes = [vp, vp, vp]
    rc = fn(ctypes.byref(p), P(stop), ctypes.byref(r))
    if rc == 1:
        return None
    assert rc == 0, "local_ba: window not expressible (rc=%d)" % rc
    out["chi2"] = r.chi2_final
    out["n_trials"] = r.n_trials
    return out


def call_ref_local_ba(fn, d, stop=None):
    """ref_local_ba / adp_local_ba (oracle/ref_optimizer_glue.cpp) for any window.  The glue's keyframe 0 is the triggering
    keyframe with mnId 0, which the reference keeps fixed (src/Optimizer.cc:722), so the glue takes only windows whose
    keyframe 0 is fixed.  A window whose current keyframe is free (every LocalBA after the map's first keyframe) goes in
    behind one extra keyframe: a fixed pKF with mnId 0 and no observation.  Its vertex has no edge, so g2o leaves it out of
    the optimisation (initializeOptimization activates only vertices with an edge at the level), and keyframe k of the
    window becomes the free local keyframe with mnId k + 1.  Returns the result of the window as given."""
    if d["fixed"][0]:
        return call_local_ba(fn, d, stop)
    e = dict(d)
    e["n_kf"], e["n_local"] = d["n_kf"] + 1, d["n_local"] + 1
    e["Tcw"] = np.concatenate([np.eye(4, dtype=np.float32).reshape(1, 16), np.asarray(d["Tcw"], np.float32).reshape(-1, 16)])
    e["fixed"] = np.concatenate([[1], d["fixed"]]).astype(np.uint8)
    e["edges"] = np.array(d["edges"], copy=True)
    e["edges"]["kf"] += 1
    out = call_local_ba(fn, e, stop)
    if out is not None:
        out["Tcw"] = np.ascontiguousarray(out["Tcw"][1:])
    return out


class Oracle:
    def __init__(self, L):
        self.L = L
        L.orc_extractor_create.restype = vp
        L.orc_extractor_create.argtypes = [ctypes.c_int, ctypes.c_float, ctypes.c_int, ctypes.c_int, ctypes.c_int]
        L.orc_extractor_destroy.argtypes = [vp]
        L.orc_extract.argtypes = [vp, vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, vp, vp, ctypes.c_int]
        L.orc_extractor_tables.argtypes = [vp] * 7
        L.orc_level_dims.argtypes = [vp, ctypes.c_int, vp, vp]
        L.orc_level_image.restype = ctypes.POINTER(ctypes.c_uint8)
        L.orc_level_image.argtypes = [vp, ctypes.c_int]
        L.orc_level_blurred.restype = ctypes.POINTER(ctypes.c_uint8)
        L.orc_level_blurred.argtypes = [vp, ctypes.c_int]
        L.orc_level_candidates.argtypes = [vp, ctypes.c_int, vp, ctypes.c_int]
        L.orc_level_keypoints.argtypes = [vp, ctypes.c_int, vp, ctypes.c_int]
        L.orc_resize_linear_u8.argtypes = [vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, vp, ctypes.c_int, ctypes.c_int,
                                           ctypes.c_int]
        L.orc_gaussian_blur7_s2_u8.argtypes = [vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, vp, ctypes.c_int]
        L.orc_fast9_16_nms.argtypes = [vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, vp, vp, ctypes.c_int]
        L.orc_fast_atan2.restype = ctypes.c_float
        L.orc_fast_atan2.argtypes = [ctypes.c_float, ctypes.c_float]
        L.orc_distribute_octtree.argtypes = [vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                             ctypes.c_int, vp, ctypes.c_int]
        L.orc_descriptor_distance.argtypes = [vp, vp]
        L.orc_search_by_bow.argtypes = [vp, vp, vp, vp, ctypes.c_int, vp, vp, vp, vp, ctypes.c_int, ctypes.c_int,
                                        ctypes.c_float, ctypes.c_int, ctypes.c_int, vp]
        L.orc_search_by_projection_last.argtypes = [vp, ctypes.c_int, vp, vp, vp, vp, vp, vp, vp, ctypes.c_int, vp,
                                                    ctypes.c_float, ctypes.c_int, ctypes.c_int, ctypes.c_int, vp]
        L.orc_search_by_projection_map.argtypes = [vp, ctypes.c_int, vp, vp, vp, vp, vp, vp, ctypes.c_int, vp,
                                                   ctypes.c_float, ctypes.c_int, ctypes.c_float, vp]
        L.orc_local_ba.argtypes = [vp, vp, vp]
        L.orc_sincosf_batch.argtypes = [vp, ctypes.c_long, vp, vp, ctypes.c_int]
        L.orc_extract_many.argtypes = [ctypes.c_int, ctypes.c_float, ctypes.c_int, ctypes.c_int, ctypes.c_int, vp,
                                       ctypes.c_int, ctypes.c_int, ctypes.c_int, vp, vp, ctypes.c_int, vp, ctypes.c_int]

    # ---- extractor ----
    def extractor(self, nfeatures, scaleFactor, nlevels, iniTh, minTh):
        return OracleExtractor(self, nfeatures, scaleFactor, nlevels, iniTh, minTh)

    def extract_many(self, params, imgs, threads):
        nf, sf, nl, ini, mn = params
        count, h, w = imgs.shape
        cap = nf + 4 * nl + 16
        kps = np.zeros((count, cap), kp_dtype)
        desc = np.zeros((count, cap, 32), np.uint8)
        n = np.zeros(count, np.int32)
        rc = self.L.orc_extract_many(nf, sf, nl, ini, mn, P(imgs), count, w, h, P(kps), P(desc), cap, P(n), threads)
        assert rc == 0
        return kps, desc, n

    def resize(self, src, dw, dh):
        src = np.ascontiguousarray(src)
        dst = np.zeros((dh, dw), np.uint8)
        self.L.orc_resize_linear_u8(P(src), src.shape[1], src.shape[0], src.shape[1], P(dst), dw, dh, dw)
        return dst

    def blur(self, src):
        src = np.ascontiguousarray(src)
        dst = np.zeros_like(src)
        self.L.orc_gaussian_blur7_s2_u8(P(src), src.shape[1], src.shape[0], src.shape[1], P(dst), src.shape[1])
        return dst

    def fast(self, img, th):
        img = np.ascontiguousarray(img)
        h, w = img.shape
        cap = w * h
        xy = np.zeros((cap, 2), np.int32)
        rs = np.zeros(cap, np.int32)
        n = self.L.orc_fast9_16_nms(P(img), w, h, w, th, P(xy), P(rs), cap)
        return xy[:n].copy(), rs[:n].copy()

    def fast_atan2(self, y, x):
        return self.L.orc_fast_atan2(float(y), float(x))

    def distribute_octtree(self, kps, minX, maxX, minY, maxY, N):
        out = np.zeros(N + 16 + 64, kp_dtype)
        n = self.L.orc_distribute_octtree(P(kps), len(kps), minX, maxX, minY, maxY, N, P(out), len(out))
        assert n >= 0
        return out[:n].copy()

    # ---- matcher ----
    def descriptor_distance(self, a, b):
        return self.L.orc_descriptor_distance(P(np.ascontiguousarray(a)), P(np.ascontiguousarray(b)))

    def search_by_bow(self, descA, nodeA, validA, angA, descB, nodeB, angB, validB=None, th_low=50, nnratio=0.7,
                      strict_lt=False, check_ori=True):
        m = np.full(len(descB), -1, np.int32)
        n = self.L.orc_search_by_bow(P(descA), P(nodeA), P(validA), P(angA), len(descA), P(descB), P(nodeB), P(validB),
                                     P(angB), len(descB), th_low, nnratio, int(strict_lt), int(check_ori), P(m))
        return n, m

    def search_by_projection_last(self, queries, kpx, kpy, octave, angle, uright, occupied, desc, geom, th, mode=0,
                                  th_high=100, check_ori=True):
        sf = np.ascontiguousarray(geom["scale_factors"], np.float32)
        g = FrameGeom(geom["mnMinX"], geom["mnMinY"], geom["mnMaxX"], geom["mnMaxY"], geom["bf"], sf.ctypes.data, len(sf))
        m = np.full(len(kpx), -1, np.int32)
        n = self.L.orc_search_by_projection_last(P(queries), len(queries), P(kpx), P(kpy), P(octave), P(angle), P(uright),
                                                 P(occupied), P(desc), len(kpx), ctypes.byref(g), th, mode, th_high,
                                                 int(check_ori), P(m))
        return n, m

    def search_by_projection_map(self, queries, kpx, kpy, octave, uright, occupied, desc, geom, th=1.0, th_high=100,
                                 nnratio=0.8):
        sf = np.ascontiguousarray(geom["scale_factors"], np.float32)
        g = FrameGeom(geom["mnMinX"], geom["mnMinY"], geom["mnMaxX"], geom["mnMaxY"], geom["bf"], sf.ctypes.data, len(sf))
        m = np.full(len(kpx), -1, np.int32)
        n = self.L.orc_search_by_projection_map(P(queries), len(queries), P(kpx), P(kpy), P(octave), P(uright),
                                                P(occupied), P(desc), len(kpx), ctypes.byref(g), th, th_high, nnratio, P(m))
        return n, m

    def search_for_initialization(self, prev, octave1, angle1, desc1, kpx2, kpy2, octave2, angle2, desc2, geom, window=10,
                                  th_low=50, nnratio=0.9, check_ori=True):
        prev_in = np.ascontiguousarray(prev, np.float32)
        px, py = np.ascontiguousarray(prev_in[:, 0]), np.ascontiguousarray(prev_in[:, 1])
        sf = np.ascontiguousarray(geom["scale_factors"], np.float32)
        g = FrameGeom(geom["mnMinX"], geom["mnMinY"], geom["mnMaxX"], geom["mnMaxY"], geom["bf"], sf.ctypes.data, len(sf))
        a = [np.ascontiguousarray(octave1, np.int32), np.ascontiguousarray(angle1, np.float32),
             np.ascontiguousarray(desc1, np.uint8), np.ascontiguousarray(kpx2, np.float32), np.ascontiguousarray(kpy2, np.float32),
             np.ascontiguousarray(octave2, np.int32), np.ascontiguousarray(angle2, np.float32), np.ascontiguousarray(desc2, np.uint8)]
        m12 = np.full(len(a[0]), -1, np.int32)
        self.L.orc_search_for_initialization.argtypes = [vp, vp, vp, vp, vp, ctypes.c_int, vp, vp, vp, vp, vp, ctypes.c_int, vp,
                                                         ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_int, vp]
        n = self.L.orc_search_for_initialization(P(px), P(py), P(a[0]), P(a[1]), P(a[2]), len(a[0]), P(a[3]), P(a[4]), P(a[5]),
                                                 P(a[6]), P(a[7]), len(a[3]), ctypes.byref(g), int(window), int(th_low),
                                                 float(nnratio), int(check_ori), P(m12))
        hit = m12 >= 0
        prev[hit, 0] = a[3][m12[hit]]
        prev[hit, 1] = a[4][m12[hit]]
        return n, m12

    def search_for_triangulation(self, kf1, kf2, F12, ex, ey, scale_factors, level_sigma2, only_stereo=False,
                                 check_ori=True):
        class KF(ctypes.Structure):
            _fields_ = [("desc", vp), ("node", vp), ("has_mp", vp), ("stereo", vp), ("x", vp), ("y", vp), ("octave", vp),
                        ("angle", vp), ("n", ctypes.c_int32)]
        keep = []

        def side(k):
            arrs = [np.ascontiguousarray(k["desc"], np.uint8), np.ascontiguousarray(k["node"], np.int32),
                    np.ascontiguousarray(k["has_mp"], np.uint8), np.ascontiguousarray(k["stereo"], np.uint8),
                    np.ascontiguousarray(k["x"], np.float32), np.ascontiguousarray(k["y"], np.float32),
                    np.ascontiguousarray(k["octave"], np.int32), np.ascontiguousarray(k["angle"], np.float32)]
            keep.append(arrs)
            return KF(*[a.ctypes.data for a in arrs], len(arrs[0]))

        a, b = side(kf1), side(kf2)
        F = np.ascontiguousarray(F12, np.float32).reshape(9)
        sf = np.ascontiguousarray(scale_factors, np.float32)
        s2 = np.ascontiguousarray(level_sigma2, np.float32)
        m = np.full(a.n, -1, np.int32)
        self.L.orc_search_for_triangulation.argtypes = [vp, vp, vp, ctypes.c_float, ctypes.c_float, vp, vp, ctypes.c_int,
                                                        ctypes.c_int, vp]
        n = self.L.orc_search_for_triangulation(ctypes.byref(a), ctypes.byref(b), P(F), ex, ey, P(sf), P(s2),
                                                int(only_stereo), int(check_ori), P(m))
        return n, m

    def search_windows(self, queries, kpx, kpy, octave, uright, inv_level_sigma2, occupied, desc, geom, chi2=False,
                       greedy=False, th_dist=50):
        sf = np.ascontiguousarray(geom["scale_factors"], np.float32)
        g = FrameGeom(geom["mnMinX"], geom["mnMinY"], geom["mnMaxX"], geom["mnMaxY"], geom["bf"], sf.ctypes.data, len(sf))
        best = np.full(len(queries), -1, np.int32)
        bdist = np.full(len(queries), 256, np.int32)
        self.L.orc_search_windows.argtypes = [vp, ctypes.c_int, vp, vp, vp, vp, vp, vp, vp, ctypes.c_int, vp, ctypes.c_int,
                                              ctypes.c_int, vp, vp]
        is2 = None if inv_level_sigma2 is None else np.ascontiguousarray(inv_level_sigma2, np.float32)
        n = self.L.orc_search_windows(P(queries), len(queries), P(kpx), P(kpy), P(octave), P(uright), P(is2), P(occupied),
                                      P(desc), len(kpx), ctypes.byref(g), (1 if chi2 else 0) | (2 if greedy else 0), th_dist,
                                      P(best), P(bdist))
        return n, best, bdist

    def compute_stereo_matches(self, exL, exR, kpsL, descL, kpsR, descR, bf, mb=0.0, reason=None):
        """exL / exR: OracleExtractor objects that just extracted the left / right image (their pyramids are used).
        reason: None, or an int32 array of len(kpsL) that receives each left keypoint's ORC_ST_* decision."""
        nl = exL.nlevels
        lv_l = [exL.level(l) for l in range(nl)]
        lv_r = [exR.level(l) for l in range(nl)]
        W = np.array([a.shape[1] for a in lv_l], np.int32)
        H = np.array([a.shape[0] for a in lv_l], np.int32)
        pl = (vp * nl)(*[a.ctypes.data for a in lv_l])
        pr = (vp * nl)(*[a.ctypes.data for a in lv_r])
        (sc, isc, _, _), _, _ = exL.tables()
        kpsL, descL = np.ascontiguousarray(kpsL), np.ascontiguousarray(descL)
        kpsR, descR = np.ascontiguousarray(kpsR), np.ascontiguousarray(descR)
        ur = np.zeros(len(kpsL), np.float32)
        dp = np.zeros(len(kpsL), np.float32)
        fn = self.L.orc_compute_stereo_matches_reason
        fn.argtypes = [vp, vp, ctypes.c_int, vp, vp, ctypes.c_int, vp, vp, vp, vp, vp, vp, ctypes.c_int, ctypes.c_float,
                       ctypes.c_float, vp, vp, vp]
        n = fn(P(kpsL), P(descL), len(kpsL), P(kpsR), P(descR), len(kpsR), pl, pr, P(W), P(H),
                 P(sc), P(isc), nl, bf, mb, P(ur), P(dp), P(reason))
        return n, ur, dp

    def distinctive_descriptors(self, desc, offsets):
        desc = np.ascontiguousarray(desc, np.uint8)
        offsets = np.ascontiguousarray(offsets, np.int32)
        best = np.full(len(offsets) - 1, -1, np.int32)
        self.L.orc_distinctive_descriptors.argtypes = [vp, vp, ctypes.c_int, vp]
        self.L.orc_distinctive_descriptors.restype = None
        self.L.orc_distinctive_descriptors(P(desc), P(offsets), len(offsets) - 1, P(best))
        return best

    # ---- DBoW2 transform ----
    def bow_transform(self, voc, features, levelsup=4):
        class V(ctypes.Structure):
            _fields_ = [("k", ctypes.c_int32), ("L", ctypes.c_int32), ("n_nodes", ctypes.c_int32), ("parent", vp),
                        ("leaf_flag", vp), ("desc", vp), ("weight", vp)]
        arrs = [np.ascontiguousarray(voc["parent"], np.int32), np.ascontiguousarray(voc["leaf_flag"], np.uint8),
                np.ascontiguousarray(voc["desc"], np.uint8), np.ascontiguousarray(voc["weight"], np.float64)]
        v = V(voc["k"], voc["L"], len(arrs[0]), *[a.ctypes.data for a in arrs])
        features = np.ascontiguousarray(features, np.uint8)
        n = len(features)
        word, w, node = np.zeros(n, np.int32), np.zeros(n, np.float64), np.zeros(n, np.int32)
        self.L.orc_bow_transform.argtypes = [vp, vp, ctypes.c_int, ctypes.c_int, vp, vp, vp]
        nw = self.L.orc_bow_transform(ctypes.byref(v), P(features), n, levelsup, P(word), P(w), P(node))
        return nw, word, w, node

    # ---- PoseOptimization ----
    def pose_optimization(self, d):
        return call_pose_optimization(self.L.orc_pose_optimization, d)

    # ---- LocalBA ----
    def local_ba(self, d, stop=None, its1=5, its2=10):
        return call_local_ba(self.L.orc_local_ba, d, stop, its1, its2)

    def sincosf(self, x, threads=8):
        x = np.ascontiguousarray(x, np.float32)
        s = np.zeros_like(x)
        c = np.zeros_like(x)
        self.L.orc_sincosf_batch(P(x), len(x), P(s), P(c), threads)
        return s, c


def pose_problem_arrays(d):
    return dict(Tcw=np.ascontiguousarray(d["Tcw"], np.float32).reshape(16),
                has_mp=np.ascontiguousarray(d["has_mp"], np.uint8), Xw=np.ascontiguousarray(d["Xw"], np.float32),
                kpx=np.ascontiguousarray(d["kpx"], np.float32), kpy=np.ascontiguousarray(d["kpy"], np.float32),
                uright=np.ascontiguousarray(d["uright"], np.float32),
                inv_sigma2=np.ascontiguousarray(d["inv_sigma2"], np.float32))


class OracleExtractor:
    def __init__(self, o, nfeatures, scaleFactor, nlevels, iniTh, minTh):
        self.o = o
        self.L = o.L
        self.nlevels = nlevels
        self.cap = nfeatures + 4 * nlevels + 16
        self.h = vp(self.L.orc_extractor_create(nfeatures, scaleFactor, nlevels, iniTh, minTh))

    def __del__(self):
        try:
            self.L.orc_extractor_destroy(self.h)
        except Exception:
            pass

    def tables(self):
        t = [np.zeros(self.nlevels, np.float32) for _ in range(4)]
        nf = np.zeros(self.nlevels, np.int32)
        um = np.zeros(16, np.int32)
        self.L.orc_extractor_tables(self.h, P(t[0]), P(t[1]), P(t[2]), P(t[3]), P(nf), P(um))
        return t, nf, um

    def __call__(self, img):
        img = np.ascontiguousarray(img)
        h, w = img.shape
        kps = np.zeros(self.cap, kp_dtype)
        desc = np.zeros((self.cap, 32), np.uint8)
        n = self.L.orc_extract(self.h, P(img), w, h, w, P(kps), P(desc), self.cap)
        assert n >= 0
        return kps[:n].copy(), desc[:n].copy()

    def level(self, l, blurred=False):
        w, h = ctypes.c_int(0), ctypes.c_int(0)
        self.L.orc_level_dims(self.h, l, ctypes.byref(w), ctypes.byref(h))
        ptr = self.L.orc_level_blurred(self.h, l) if blurred else self.L.orc_level_image(self.h, l)
        if not ptr:
            return None
        return np.ctypeslib.as_array(ptr, shape=(h.value, w.value)).copy()

    def candidates(self, l):
        n = self.L.orc_level_candidates(self.h, l, None, 0)
        out = np.zeros(max(n, 1), kp_dtype)
        self.L.orc_level_candidates(self.h, l, P(out), n)
        return out[:n]

    def keypoints(self, l):
        n = self.L.orc_level_keypoints(self.h, l, None, 0)
        out = np.zeros(max(n, 1), kp_dtype)
        self.L.orc_level_keypoints(self.h, l, P(out), n)
        return out[:n]


def load():
    if not os.path.exists(ORACLE_LIB):
        subprocess.check_call(["make", "-s", "-C", ORACLE_DIR, "liborb_oracle.so"])
    return Oracle(ctypes.CDLL(ORACLE_LIB))
