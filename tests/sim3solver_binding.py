"""Sim3 RANSAC checkers (test infrastructure): ctypes bindings of the CPU restatement oracle/liborb_sim3solver.so
(orc_s3s_iterate and the OpenCV operations it restates) and of the reference's own Sim3Solver compiled in place
(oracle/_ref/libref_sim3solver.so) and the drop-in (oracle/_ref/libadapter_sim3solver.so).  The problem and result
structures are the C ABI's (b2s_sim3solver_problem / b2s_sim3solver_result in include/b200slam.h); pkg.Sim3Solver uses
the same ones."""
import ctypes
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
ORACLE_LIB = os.path.join(ORACLE_DIR, "liborb_sim3solver.so")
REF_LIB = os.path.join(ORACLE_DIR, "_ref", "libref_sim3solver.so")
ADP_LIB = os.path.join(ORACLE_DIR, "_ref", "libadapter_sim3solver.so")
vp = ctypes.c_void_p
i32 = ctypes.c_int32


class Problem(ctypes.Structure):
    _fields_ = [("n", i32), ("X1c", vp), ("X2c", vp), ("sigma2_1", vp), ("sigma2_2", vp),
                ("K1", ctypes.c_float * 4), ("K2", ctypes.c_float * 4), ("fix_scale", i32), ("min_inliers", i32),
                ("max_its", i32), ("iterations_done", i32), ("best_inliers", i32), ("k", i32), ("sets", vp)]


class Result(ctypes.Structure):
    _fields_ = [("returned", i32), ("T12", ctypes.c_float * 16), ("best_changed", i32), ("R", ctypes.c_float * 9),
                ("t", ctypes.c_float * 3), ("s", ctypes.c_float), ("inliers", vp), ("n_inliers", i32),
                ("no_more", i32), ("iterations_used", i32), ("iterations_done", i32), ("best_inliers", i32)]


def pack(d, state, sets):
    """(Problem, arrays kept alive).  d: X1c, X2c (n x 3), sigma2_1, sigma2_2 (n), K1, K2 (fx, fy, cx, cy), fix_scale,
    min_inliers, max_its; state: (iterations_done, best_inliers); sets: k x 3."""
    a = dict(X1c=np.ascontiguousarray(d["X1c"], np.float32).reshape(-1, 3),
             X2c=np.ascontiguousarray(d["X2c"], np.float32).reshape(-1, 3),
             sigma2_1=np.ascontiguousarray(d["sigma2_1"], np.float32).reshape(-1),
             sigma2_2=np.ascontiguousarray(d["sigma2_2"], np.float32).reshape(-1),
             sets=np.ascontiguousarray(sets, np.int32).reshape(-1, 3))
    p = Problem()
    p.n = len(a["X1c"])
    for k in ("X1c", "X2c", "sigma2_1", "sigma2_2", "sets"):
        setattr(p, k, a[k].ctypes.data)
    p.K1[:] = [float(v) for v in np.asarray(d["K1"], np.float32)]
    p.K2[:] = [float(v) for v in np.asarray(d["K2"], np.float32)]
    p.fix_scale, p.min_inliers, p.max_its = int(d["fix_scale"]), int(d["min_inliers"]), int(d["max_its"])
    p.iterations_done, p.best_inliers = int(state[0]), int(state[1])
    p.k = len(a["sets"])
    return p, a


def new_result(n):
    out = np.full(max(n, 1), 7, np.uint8)
    r = Result()
    r.inliers = out.ctypes.data
    return r, out


def unpack(r, out, n):
    return dict(returned=r.returned, T12=np.array(r.T12[:], np.float32).reshape(4, 4), best_changed=r.best_changed,
                R=np.array(r.R[:], np.float32).reshape(3, 3), t=np.array(r.t[:], np.float32), s=np.float32(r.s),
                inliers=out[:n].astype(bool), n_inliers=r.n_inliers, no_more=r.no_more,
                iterations_used=r.iterations_used, iterations_done=r.iterations_done, best_inliers=r.best_inliers)


_L = None


def _lib():
    global _L
    if _L is None:
        if not os.path.exists(ORACLE_LIB):
            subprocess.check_call(["make", "-s", "-C", ORACLE_DIR, "-f", "sim3solver.mk", "liborb_sim3solver.so"])
        L = ctypes.CDLL(ORACLE_LIB)
        L.orc_s3s_reduce_sum_cols.argtypes = [vp, ctypes.c_int, ctypes.c_int, vp]
        L.orc_s3s_eigen.argtypes = [vp, ctypes.c_int, vp, vp]
        L.orc_s3s_rodrigues.argtypes = [vp, vp]
        L.orc_s3s_norm.argtypes = [vp, ctypes.c_int]
        L.orc_s3s_norm.restype = ctypes.c_double
        L.orc_s3s_dot.argtypes = [vp, vp, ctypes.c_int]
        L.orc_s3s_dot.restype = ctypes.c_double
        L.orc_s3s_pow2.argtypes = [vp, ctypes.c_int, vp]
        L.orc_s3s_gemm_bt.argtypes = [vp, vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, vp]
        L.orc_s3s_ransac_max_its.argtypes = [ctypes.c_int, ctypes.c_double, ctypes.c_int, ctypes.c_int]
        L.orc_s3s_compute_sim3.argtypes = [vp, vp, ctypes.c_int, vp]
        L.orc_s3s_iterate.argtypes = [vp, vp, vp]
        L.orc_gemm.argtypes = [vp, vp, vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_double, ctypes.c_int, vp]
        _L = L
    return _L


def _f32(a):
    return np.ascontiguousarray(a, np.float32)


def reduce_sum_cols(P):
    P = _f32(P)
    C = np.zeros(P.shape[0], np.float32)
    _lib().orc_s3s_reduce_sum_cols(P.ctypes.data, P.shape[0], P.shape[1], C.ctypes.data)
    return C


def eigen(A):
    A = _f32(A)
    n = A.shape[0]
    w, v = np.zeros(n, np.float32), np.zeros((n, n), np.float32)
    _lib().orc_s3s_eigen(A.ctypes.data, n, w.ctypes.data, v.ctypes.data)
    return w, v


def rodrigues(v):
    v = _f32(v).reshape(3)
    R = np.zeros((3, 3), np.float32)
    _lib().orc_s3s_rodrigues(v.ctypes.data, R.ctypes.data)
    return R


def norm(a):
    a = _f32(a).ravel()
    return _lib().orc_s3s_norm(a.ctypes.data, a.size)


def dot(a, b):
    a, b = _f32(a).ravel(), _f32(b).ravel()
    return _lib().orc_s3s_dot(a.ctypes.data, b.ctypes.data, a.size)


def pow2(a):
    a = _f32(a)
    o = np.zeros_like(a)
    _lib().orc_s3s_pow2(a.ctypes.data, a.size, o.ctypes.data)
    return o


def gemm_bt(A, B):
    A, B = _f32(A), _f32(B)
    D = np.zeros((A.shape[0], B.shape[0]), np.float32)
    _lib().orc_s3s_gemm_bt(A.ctypes.data, B.ctypes.data, A.shape[0], A.shape[1], B.shape[0], D.ctypes.data)
    return D


def gemm(A, B, alpha=1.0, C=None):
    A, B = _f32(A), _f32(B)
    D = np.zeros((A.shape[0], B.shape[1]), np.float32)
    Cc = None if C is None else _f32(C)
    _lib().orc_gemm(A.ctypes.data, B.ctypes.data, None if Cc is None else Cc.ctypes.data, A.shape[0], A.shape[1],
                    B.shape[1], float(alpha), 0, D.ctypes.data)
    return D


def ransac_max_its(N, probability, min_inliers, max_iterations):
    return _lib().orc_s3s_ransac_max_its(int(N), float(probability), int(min_inliers), int(max_iterations))


def compute_sim3(P1, P2, fix_scale):
    """orc_s3s_compute_sim3: dict R, t, s, T12, T21."""
    P1, P2 = _f32(P1), _f32(P2)
    h = np.zeros(45, np.float32)
    _lib().orc_s3s_compute_sim3(P1.ctypes.data, P2.ctypes.data, int(fix_scale), h.ctypes.data)
    return dict(R=h[:9].reshape(3, 3), t=h[9:12], s=h[12], T12=h[13:29].reshape(4, 4), T21=h[29:45].reshape(4, 4))


def oracle(d, state, sets):
    """orc_s3s_iterate on one solver state: (result dict, margin)."""
    p, keep = pack(d, state, sets)
    r, out = new_result(p.n)
    m = ctypes.c_double(0)
    _lib().orc_s3s_iterate(ctypes.byref(p), ctypes.byref(r), ctypes.byref(m))
    return unpack(r, out, p.n), m.value


def camera_points(Tcw, Xw):
    """Rcw*Xw + tcw as the cv::Mat expression evaluates it (gemm's float path for an inner size of 3, then the float
    addition of C): the constructor's mvX3Dc."""
    Tcw = _f32(Tcw)
    R, t = Tcw[:3, :3], Tcw[:3, 3]
    Xw = _f32(Xw).reshape(-1, 3)
    f = (R[None, :, 0] * Xw[:, 0:1] + R[None, :, 1] * Xw[:, 1:2]) + R[None, :, 2] * Xw[:, 2:3]
    return (f + t[None, :]).astype(np.float32)


class Scene(ctypes.Structure):  # s3s_scene (oracle/ref_sim3solver_glue.cpp)
    _fields_ = [("m", i32), ("nk2", i32), ("fix_scale", i32), ("Tcw1", vp), ("Tcw2", vp), ("K1", vp), ("K2", vp),
                ("n_levels", i32), ("level_sigma2_1", vp), ("level_sigma2_2", vp), ("octave1", vp), ("octave2", vp),
                ("matched", vp), ("has_mp1", vp), ("bad1", vp), ("bad2", vp), ("idx1", vp), ("idx2", vp),
                ("Xw1", vp), ("Xw2", vp)]


class RefSolver:
    """The reference's own Sim3Solver (REF_LIB) or the drop-in (ADP_LIB) on a flattened scene (synth_sim3solver)."""

    def __init__(self, lib_path, sc):
        L = ctypes.CDLL(lib_path)
        L.s3s_create.restype = vp
        L.s3s_create.argtypes = [vp]
        L.s3s_destroy.argtypes = [vp]
        L.s3s_set_ransac_parameters.argtypes = [vp, ctypes.c_double, ctypes.c_int, ctypes.c_int]
        L.s3s_iterate.argtypes = [vp, ctypes.c_int, vp, vp, vp, vp]
        L.s3s_state.argtypes = [vp] * 6
        L.s3s_members.argtypes = [vp] * 6
        L.s3s_srand.argtypes = [ctypes.c_uint]
        L.s3s_random_int.argtypes = [ctypes.c_int, ctypes.c_int]
        self.L = L
        keep = {}
        s = Scene()
        for k, t in (("Tcw1", np.float32), ("Tcw2", np.float32), ("K1", np.float32), ("K2", np.float32),
                     ("level_sigma2_1", np.float32), ("level_sigma2_2", np.float32), ("octave1", np.int32),
                     ("octave2", np.int32), ("matched", np.int32), ("has_mp1", np.int32), ("bad1", np.int32),
                     ("bad2", np.int32), ("idx1", np.int32), ("idx2", np.int32), ("Xw1", np.float32),
                     ("Xw2", np.float32)):
            keep[k] = np.ascontiguousarray(sc[k], t)
            setattr(s, k, keep[k].ctypes.data)
        s.m, s.nk2, s.fix_scale, s.n_levels = sc["m"], sc["nk2"], sc["fix_scale"], len(sc["level_sigma2_1"])
        self.m = sc["m"]
        self.h = L.s3s_create(ctypes.byref(s))

    def close(self):
        if self.h:
            self.L.s3s_destroy(self.h)
            self.h = None

    def set_ransac_parameters(self, probability=0.99, min_inliers=6, max_iterations=300):
        self.L.s3s_set_ransac_parameters(self.h, probability, min_inliers, max_iterations)

    def iterate(self, n_iterations):
        """iterate(n) (find() when n is None): T12 (None: empty), no_more (None for find), inliers (mN1), n_inliers."""
        nm, ni = ctypes.c_int32(0), ctypes.c_int32(0)
        inl = np.zeros(max(self.m, 1), np.uint8)
        T = np.zeros(16, np.float32)
        ret = self.L.s3s_iterate(self.h, -1 if n_iterations is None else int(n_iterations), ctypes.byref(nm),
                                 inl.ctypes.data, ctypes.byref(ni), T.ctypes.data)
        return dict(T12=T.reshape(4, 4) if ret else None, no_more=None if n_iterations is None else bool(nm.value),
                    inliers=inl[:self.m].astype(bool), n_inliers=ni.value)

    def state(self):
        c = np.zeros(6, np.int32)
        R, t, s, hb = np.zeros(9, np.float32), np.zeros(3, np.float32), ctypes.c_float(0), ctypes.c_int32(0)
        self.L.s3s_state(self.h, c.ctypes.data, R.ctypes.data, t.ctypes.data, ctypes.byref(s), ctypes.byref(hb))
        return dict(N=int(c[0]), mN1=int(c[1]), iterations=int(c[2]), best_inliers=int(c[3]), max_its=int(c[4]),
                    min_inliers=int(c[5]), has_best=bool(hb.value), R=R.reshape(3, 3), t=t, s=np.float32(s.value))

    def members(self):
        N = self.state()["N"]
        idx, X1, X2 = np.zeros(N, np.int32), np.zeros((N, 3), np.float32), np.zeros((N, 3), np.float32)
        e1, e2 = np.zeros(N, np.uint64), np.zeros(N, np.uint64)
        self.L.s3s_members(self.h, idx.ctypes.data, X1.ctypes.data, X2.ctypes.data, e1.ctypes.data, e2.ctypes.data)
        return dict(indices1=idx, X1c=X1, X2c=X2, max_err1=e1, max_err2=e2)

    def srand(self, seed):
        self.L.s3s_srand(seed)

    def rand_draws(self, n, count):
        """The sets `count` iterations over n correspondences draw next from rand() (DUtils::Random::RandomInt)."""
        out = np.zeros((count, 3), np.int32)
        for it in range(count):
            avail = list(range(n))
            for j in range(3):
                ri = self.L.s3s_random_int(0, len(avail) - 1)
                out[it, j] = avail[ri]
                avail[ri] = avail[-1]
                avail.pop()
        return out


def expand(inl, indices1, m):
    """vbInliers (mN1) from the compacted flags."""
    v = np.zeros(m, bool)
    v[np.asarray(indices1)[np.asarray(inl, bool)]] = True
    return v
