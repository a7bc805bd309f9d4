"""Monocular initialiser checkers (test infrastructure): ctypes bindings of the CPU restatement oracle/liborb_init.so
(orc_initialize and the OpenCV linear algebra it restates: orc_svd, orc_inv3, orc_det3, orc_gemm).  The problem and
result structures are the C ABI's (b2s_init_problem / b2s_init_result in include/b200slam.h); pkg.MonoInitializer
uses the same ones."""
import ctypes
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
ORACLE_LIB = os.path.join(ORACLE_DIR, "liborb_init.so")
vp = ctypes.c_void_p
f32p = ctypes.POINTER(ctypes.c_float)


class Problem(ctypes.Structure):
    _fields_ = [("n1", ctypes.c_int32), ("n2", ctypes.c_int32), ("kp1", vp), ("kp2", vp), ("matches12", vp),
                ("K", ctypes.c_float * 9), ("sigma", ctypes.c_float), ("iterations", ctypes.c_int32), ("sets", vp)]


class Result(ctypes.Structure):
    _fields_ = [("ret", ctypes.c_int32), ("model", ctypes.c_int32), ("rt_state", ctypes.c_int32),
                ("R21", ctypes.c_float * 9), ("t21", ctypes.c_float * 3), ("p3d", vp), ("triangulated", vp),
                ("inliers_h", vp), ("inliers_f", vp), ("n_matches", ctypes.c_int32), ("best_h_iter", ctypes.c_int32),
                ("best_f_iter", ctypes.c_int32), ("SH", ctypes.c_float), ("SF", ctypes.c_float),
                ("RH", ctypes.c_float), ("H21", ctypes.c_float * 9), ("F21", ctypes.c_float * 9),
                ("n_hyp", ctypes.c_int32), ("n_good", ctypes.c_int32 * 8), ("parallax", ctypes.c_float * 8)]


# Untouched outputs keep this marker, so a test sees what a call wrote (as the reference leaves its arguments alone)
UNTOUCHED = np.float32(-12345.0)


def pack(d):
    """(Problem, arrays kept alive) from a dict with kp1 (n1 x 2), kp2, matches12 (n1), K (3 x 3), sigma, sets."""
    a = dict(kp1=np.ascontiguousarray(d["kp1"], np.float32), kp2=np.ascontiguousarray(d["kp2"], np.float32),
             m=np.ascontiguousarray(d["matches12"], np.int32), sets=np.ascontiguousarray(d["sets"], np.int32))
    p = Problem()
    p.n1, p.n2 = len(a["kp1"]), len(a["kp2"])
    p.kp1, p.kp2, p.matches12, p.sets = (a[k].ctypes.data for k in ("kp1", "kp2", "m", "sets"))
    p.K[:] = [float(x) for x in np.asarray(d["K"], np.float32).ravel()]
    p.sigma = float(d["sigma"])
    p.iterations = len(a["sets"])
    return p, a


def new_result(n1, n_matches):
    """(Result, output arrays) with p3d / triangulated / R21 / t21 pre-filled with UNTOUCHED (triangulated with 7)."""
    out = dict(p3d=np.full((n1, 3), UNTOUCHED, np.float32), triangulated=np.full(n1, 7, np.uint8),
               inliers_h=np.zeros(max(n_matches, 1), np.uint8), inliers_f=np.zeros(max(n_matches, 1), np.uint8))
    r = Result()
    r.R21[:] = [float(UNTOUCHED)] * 9
    r.t21[:] = [float(UNTOUCHED)] * 3
    for k, v in out.items():
        setattr(r, k, v.ctypes.data)
    return r, out


def unpack(r, out):
    n = r.n_matches
    res = dict(ret=r.ret, model=r.model, rt_state=r.rt_state, R21=np.array(r.R21[:], np.float32),
               t21=np.array(r.t21[:], np.float32), p3d=out["p3d"], triangulated=out["triangulated"],
               inliers_h=out["inliers_h"][:n].astype(bool), inliers_f=out["inliers_f"][:n].astype(bool),
               n_matches=n, best_h_iter=r.best_h_iter, best_f_iter=r.best_f_iter, SH=np.float32(r.SH),
               SF=np.float32(r.SF), RH=np.float32(r.RH), H21=np.array(r.H21[:], np.float32),
               F21=np.array(r.F21[:], np.float32), n_hyp=r.n_hyp, n_good=np.array(r.n_good[:r.n_hyp], np.int32),
               parallax=np.array(r.parallax[:r.n_hyp], np.float32))
    return res


def _lib():
    if not os.path.exists(ORACLE_LIB):
        subprocess.check_call(["make", "-s", "-C", ORACLE_DIR, "-f", "init.mk", "liborb_init.so"])
    L = ctypes.CDLL(ORACLE_LIB)
    L.orc_initialize.argtypes = [vp, vp]
    L.orc_svd.argtypes = [vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, vp, vp, vp]
    L.orc_inv3.argtypes = [vp, vp]
    L.orc_det3.argtypes = [vp]
    L.orc_det3.restype = ctypes.c_double
    L.orc_gemm.argtypes = [vp, vp, vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_double, ctypes.c_int, vp]
    return L


def oracle(d):
    """orc_initialize on one problem (a dict as pack() takes it)."""
    p, keep = pack(d)
    n = int((keep["m"] >= 0).sum())
    r, out = new_result(p.n1, n)
    assert _lib().orc_initialize(ctypes.byref(p), ctypes.byref(r)) == 0
    return unpack(r, out)


def svd(A, full_uv):
    """orc_svd: (w, u, vt) with OpenCV's shapes."""
    A = np.ascontiguousarray(A, np.float32)
    rows, cols = A.shape
    m, n = max(rows, cols), min(rows, cols)
    urows = m if full_uv else n
    w = np.zeros(n, np.float32)
    if rows >= cols:
        u, vt = np.zeros((rows, urows), np.float32), np.zeros((n, n), np.float32)
    else:
        u, vt = np.zeros((n, n), np.float32), np.zeros((urows, cols), np.float32)
    _lib().orc_svd(A.ctypes.data, rows, cols, int(full_uv), w.ctypes.data, u.ctypes.data, vt.ctypes.data)
    return w, u, vt


def inv3(A):
    A = np.ascontiguousarray(A, np.float32)
    o = np.zeros((3, 3), np.float32)
    ok = _lib().orc_inv3(A.ctypes.data, o.ctypes.data)
    return bool(ok), o


def det3(A):
    A = np.ascontiguousarray(A, np.float32)
    return _lib().orc_det3(A.ctypes.data)


def gemm(A, B, alpha=1.0, C=None, tA=False):
    A, B = np.ascontiguousarray(A, np.float32), np.ascontiguousarray(B, np.float32)
    m, k = (A.shape[1], A.shape[0]) if tA else A.shape
    n = B.shape[1]
    D = np.zeros((m, n), np.float32)
    Cc = None if C is None else np.ascontiguousarray(C, np.float32)
    _lib().orc_gemm(A.ctypes.data, B.ctypes.data, None if Cc is None else Cc.ctypes.data, m, k, n, float(alpha),
                    int(tA), D.ctypes.data)
    return D


REF_LIB = os.path.join(ORACLE_DIR, "_ref", "libref_init.so")
ADP_LIB = os.path.join(ORACLE_DIR, "_ref", "libadapter_init.so")


def find(d, homography):
    """orc_find: (best iteration, score, X (9), inlier flags)."""
    p, keep = pack(d)
    n = int((keep["m"] >= 0).sum())
    score, X, inl = ctypes.c_float(0), np.zeros(9, np.float32), np.zeros(max(n, 1), np.uint8)
    L = _lib()
    L.orc_find.argtypes = [vp, ctypes.c_int, vp, vp, vp]
    best = L.orc_find(ctypes.byref(p), int(homography), ctypes.byref(score), X.ctypes.data, inl.ctypes.data)
    return best, np.float32(score.value), X, inl[:n].astype(bool)


def reconstruct(d, homography, inliers, X):
    """orc_reconstruct: the result fields ReconstructH / ReconstructF set (p3d / triangulated only when ret)."""
    p, keep = pack(d)
    n = int((keep["m"] >= 0).sum())
    r, out = new_result(p.n1, n)
    inl = np.ascontiguousarray(inliers, np.uint8)
    X = np.ascontiguousarray(X, np.float32)
    L = _lib()
    L.orc_reconstruct.argtypes = [vp, ctypes.c_int, vp, vp, vp]
    L.orc_reconstruct(ctypes.byref(p), int(homography), inl.ctypes.data, X.ctypes.data, ctypes.byref(r))
    r.n_matches = n
    return unpack(r, out)


def _graph_out(n1):
    return dict(R21=np.full(9, UNTOUCHED, np.float32), t21=np.full(3, UNTOUCHED, np.float32),
                rt_state=ctypes.c_int32(0), p3d=np.zeros((n1, 3), np.float32), triangulated=np.zeros(n1, np.uint8))


def _graph_result(ret, o):
    return dict(ret=ret, R21=o["R21"], t21=o["t21"], rt_state=o["rt_state"].value, p3d=o["p3d"],
                triangulated=o["triangulated"])


def call_initialize(lib_path, fn, d):
    """ref_initialize / adp_initialize: Initializer(F1, sigma, iterations).Initialize(F2, vMatches12, ...) after srand(0)
    on two stand-in Frames.  Returns ret, R21, t21, rt_state, p3d / triangulated (vP3D / vbTriangulated as left: n1
    points of UNTOUCHED and n1 x true when the call did not write them) and sets (the object's mvSets)."""
    p, keep = pack(d)
    o = _graph_out(p.n1)
    sets = np.zeros((p.iterations, 8), np.int32)
    f = getattr(ctypes.CDLL(lib_path), fn)
    f.argtypes = [vp] * 7
    ret = f(ctypes.byref(p), o["R21"].ctypes.data, o["t21"].ctypes.data, ctypes.byref(o["rt_state"]),
            o["p3d"].ctypes.data, o["triangulated"].ctypes.data, sets.ctypes.data)
    out = _graph_result(ret, o)
    out["sets"] = sets
    return out


def ref_find(d, homography):
    p, keep = pack(d)
    n = int((keep["m"] >= 0).sum())
    score, X, inl = ctypes.c_float(0), np.zeros(9, np.float32), np.zeros(max(n, 1), np.uint8)
    f = ctypes.CDLL(REF_LIB).ref_find
    f.argtypes = [vp, ctypes.c_int, vp, vp, vp]
    f(ctypes.byref(p), int(homography), ctypes.byref(score), X.ctypes.data, inl.ctypes.data)
    return np.float32(score.value), X, inl[:n].astype(bool)


def ref_reconstruct(d, homography, inliers, X):
    p, keep = pack(d)
    o = _graph_out(p.n1)
    inl = np.ascontiguousarray(inliers, np.uint8)
    X = np.ascontiguousarray(X, np.float32)
    f = ctypes.CDLL(REF_LIB).ref_reconstruct
    f.argtypes = [vp, ctypes.c_int, vp, vp, vp, vp, vp, vp, vp]
    ret = f(ctypes.byref(p), int(homography), inl.ctypes.data, X.ctypes.data, o["R21"].ctypes.data,
            o["t21"].ctypes.data, ctypes.byref(o["rt_state"]), o["p3d"].ctypes.data, o["triangulated"].ctypes.data)
    return _graph_result(ret, o)
