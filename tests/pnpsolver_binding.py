"""EPnP RANSAC checkers (test infrastructure): ctypes bindings of the CPU restatement oracle/liborb_pnpsolver.so
(orc_pnp_iterate and the OpenCV C API operations it restates) and of the reference's own PnPsolver compiled in place
(oracle/_ref/libref_pnpsolver.so).  The problem and result structures are the C ABI's (b2s_pnpsolver_problem /
b2s_pnpsolver_result in include/b200slam.h), shared with pkg.PnPsolver."""
import ctypes
import importlib
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
ORACLE_LIB = os.path.join(ORACLE_DIR, "liborb_pnpsolver.so")
REF_LIB = os.path.join(ORACLE_DIR, "_ref", "libref_pnpsolver.so")
ADP_LIB = os.path.join(ORACLE_DIR, "_ref", "libadapter_pnpsolver.so")
vp = ctypes.c_void_p
pkg = importlib.import_module("self_commit_orb-slam2_b200")
Problem, Result = pkg._PnPsolverProblem, pkg._PnPsolverResult


def pack(d, state, sets):
    """(Problem, arrays kept alive).  d: a scene of synth_pnp (P3Dw, P2D, sigma2, K, th2, min_inliers, max_its);
    state: (iterations_done, best_inliers, best_Tcw, best_mask); sets: k x 4."""
    n = len(d["P3Dw"])
    a = dict(P3Dw=np.ascontiguousarray(d["P3Dw"], np.float32), P2D=np.ascontiguousarray(d["P2D"], np.float32),
             sigma2=np.ascontiguousarray(d["sigma2"], np.float32),
             best_Tcw=np.ascontiguousarray(state[2], np.float32).reshape(16),
             best_mask=np.ascontiguousarray(np.resize(np.asarray(state[3], np.uint8), max(n, 1))),
             sets=np.ascontiguousarray(sets, np.int32).reshape(-1, 4))
    p = Problem()
    p.n = n
    for k in ("P3Dw", "P2D", "sigma2", "best_Tcw", "best_mask", "sets"):
        setattr(p, k, a[k].ctypes.data)
    p.fu, p.fv, p.uc, p.vc = [float(v) for v in np.asarray(d["K"], np.float32)]
    p.th2 = float(np.float32(d["th2"]))
    p.min_inliers, p.max_its, p.min_set = int(d["min_inliers"]), int(d["max_its"]), 4
    p.iterations_done, p.best_inliers = int(state[0]), int(state[1])
    p.k = len(a["sets"])
    return p, a


def new_result(n):
    out, bm = np.full(max(n, 1), 7, np.uint8), np.full(max(n, 1), 7, np.uint8)
    r = Result()
    r.inliers, r.best_mask = out.ctypes.data, bm.ctypes.data
    return r, (out, bm)


def unpack(r, arrs, n):
    out, bm = arrs
    return dict(returned=r.returned, Tcw=np.array(r.Tcw[:], np.float32).reshape(4, 4) if r.returned else None,
                inliers=out[:n].astype(bool), n_inliers=r.n_inliers, no_more=r.no_more,
                iterations_used=r.iterations_used, iterations_done=r.iterations_done, best_inliers=r.best_inliers,
                best_changed=r.best_changed, best_Tcw=np.array(r.best_Tcw[:], np.float32).reshape(4, 4),
                best_mask=bm[:n].copy())


def next_state(res):
    """The solver state a result leaves, for the next call's pack."""
    return (res["iterations_done"], res["best_inliers"], res["best_Tcw"], res["best_mask"])


INITIAL = (0, 0, np.eye(4, dtype=np.float32), np.zeros(1, np.uint8))

_L = None


def lib():
    global _L
    if _L is None:
        if not os.path.exists(ORACLE_LIB):
            subprocess.check_call(["make", "-s", "-C", ORACLE_DIR, "-f", "pnpsolver.mk", "liborb_pnpsolver.so"])
        L = ctypes.CDLL(ORACLE_LIB)
        L.orc_pnp_mul_transposed.argtypes = [vp, ctypes.c_int, ctypes.c_int, vp]
        L.orc_pnp_svd.argtypes = [vp, ctypes.c_int, vp, vp, vp]
        L.orc_pnp_invert_svd.argtypes = [vp, ctypes.c_int, vp]
        L.orc_pnp_solve_svd.argtypes = [vp, ctypes.c_int, ctypes.c_int, vp, vp]
        L.orc_pnp_ransac_parameters.argtypes = [ctypes.c_int, ctypes.c_double, ctypes.c_int, ctypes.c_int,
                                                ctypes.c_int, ctypes.c_float, vp, vp]
        L.orc_pnp_compute_pose.argtypes = [vp, vp, vp, ctypes.c_int, vp, vp, vp]
        L.orc_pnp_compute_pose.restype = ctypes.c_double
        L.orc_pnp_iterate.argtypes = [vp, vp, vp, vp]
        _L = L
    return _L


def _d(a):
    return np.ascontiguousarray(a, np.float64)


def mul_transposed(A):
    A = _d(A)
    D = np.zeros((A.shape[1], A.shape[1]))
    lib().orc_pnp_mul_transposed(A.ctypes.data, A.shape[0], A.shape[1], D.ctypes.data)
    return D


def svd(A):
    A = _d(A)
    n = A.shape[0]
    w, u, vt = np.zeros(n), np.zeros((n, n)), np.zeros((n, n))
    lib().orc_pnp_svd(A.ctypes.data, n, w.ctypes.data, u.ctypes.data, vt.ctypes.data)
    return w, u, vt


def invert_svd(A):
    A = _d(A)
    D = np.zeros_like(A)
    lib().orc_pnp_invert_svd(A.ctypes.data, A.shape[0], D.ctypes.data)
    return D


def solve_svd(A, b):
    A, b = _d(A), _d(b).reshape(-1)
    x = np.zeros(A.shape[1])
    lib().orc_pnp_solve_svd(A.ctypes.data, A.shape[0], A.shape[1], b.ctypes.data, x.ctypes.data)
    return x


def ransac_parameters(n, probability=0.99, min_inliers=8, max_iterations=300, min_set=4, epsilon=0.4):
    m, it = ctypes.c_int(), ctypes.c_int()
    lib().orc_pnp_ransac_parameters(n, probability, min_inliers, max_iterations, min_set, epsilon, ctypes.byref(m),
                                    ctypes.byref(it))
    return m.value, it.value


def compute_pose(d, idx):
    idx = np.ascontiguousarray(idx, np.int32)
    R, t = np.zeros(9), np.zeros(3)
    K = np.ascontiguousarray(d["K"], np.float32)
    e = lib().orc_pnp_compute_pose(np.ascontiguousarray(d["P3Dw"], np.float32).ctypes.data,
                                   np.ascontiguousarray(d["P2D"], np.float32).ctypes.data, idx.ctypes.data, len(idx),
                                   K.ctypes.data, R.ctypes.data, t.ctypes.data)
    return R.reshape(3, 3), t, e


def iterate(d, state, sets):
    """orc_pnp_iterate: the result dict, plus margin and trace (k x 15: R, t, error, inliers, refined inliers)."""
    p, keep = pack(d, state, sets)
    r, arrs = new_result(p.n)
    margin = ctypes.c_double()
    hyp = np.zeros((max(p.k, 1), 15))
    lib().orc_pnp_iterate(ctypes.byref(p), ctypes.byref(r), ctypes.byref(margin), hyp.ctypes.data)
    out = unpack(r, arrs, p.n)
    out["margin"], out["trace"] = margin.value, hyp[:p.k]
    return out


def draw_sets(n, k, random_int):
    """k minimal sets as PnPsolver::iterate draws them: 4 RandomInt calls per set over the available indices, each
    pick swap-removed."""
    sets = np.zeros((k, 4), np.int32)
    for j in range(k):
        avail = list(range(n))
        for i in range(4):
            r = random_int(0, len(avail) - 1)
            sets[j, i] = avail[r]
            avail[r] = avail[-1]
            avail.pop()
    return sets


class Ref:
    """The reference's own PnPsolver (REF_LIB, oracle/_ref/libref_pnpsolver.so) or the drop-in (ADP_LIB,
    oracle/_ref/libadapter_pnpsolver.so) on one scene."""
    _L = {}

    @classmethod
    def lib(cls, path=REF_LIB):
        if path not in cls._L:
            L = ctypes.CDLL(path)
            L.pnp_create.restype = vp
            L.pnp_create.argtypes = [ctypes.c_int, vp, vp, vp, vp]
            L.pnp_destroy.argtypes = [vp]
            L.pnp_set_ransac_parameters.argtypes = [vp, ctypes.c_double, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                                    ctypes.c_float, ctypes.c_float]
            L.pnp_iterate.argtypes = [vp, ctypes.c_int, vp, vp, vp, vp]
            L.pnp_state.argtypes = [vp, vp, vp, vp]
            if hasattr(L, "pnp_compute_pose"):  # the reference's own EPnP (the drop-in runs it on the device)
                L.pnp_compute_pose.argtypes = [vp, vp, ctypes.c_int, vp, vp]
                L.pnp_compute_pose.restype = ctypes.c_double
            L.pnp_srand.argtypes = [ctypes.c_uint]
            L.pnp_random_int.argtypes = [ctypes.c_int, ctypes.c_int]
            cls._L[path] = L
        return cls._L[path]

    def __init__(self, d, path=REF_LIB):
        self.n = len(d["P3Dw"])
        self.L = self.lib(path)
        self.keep = [np.ascontiguousarray(d[k], np.float32) for k in ("P3Dw", "P2D", "sigma2", "K")]
        self.h = self.L.pnp_create(self.n, *[a.ctypes.data for a in self.keep])
        self.L.pnp_set_ransac_parameters(self.h, *d["params"])

    def __del__(self):
        if getattr(self, "h", None):
            self.L.pnp_destroy(self.h)

    def iterate(self, n_iterations):
        """iterate(n_iterations), or find() for None."""
        nm, ni = ctypes.c_int32(), ctypes.c_int32()
        inl, T = np.zeros(max(self.n, 1), np.uint8), np.zeros(16, np.float32)
        ret = self.L.pnp_iterate(self.h, -1 if n_iterations is None else n_iterations, ctypes.byref(nm),
                                     inl.ctypes.data, ctypes.byref(ni), T.ctypes.data)
        return dict(Tcw=T.reshape(4, 4) if ret else None, no_more=None if n_iterations is None else bool(nm.value),
                    n_inliers=ni.value,
                    inliers=inl[:self.n].astype(bool))

    def state(self):
        c, T, m = np.zeros(4, np.int32), np.zeros(16, np.float32), np.zeros(max(self.n, 1), np.uint8)
        has = self.L.pnp_state(self.h, c.ctypes.data, T.ctypes.data, m.ctypes.data)
        return dict(iterations=int(c[0]), best_inliers=int(c[1]), min_inliers=int(c[2]), max_its=int(c[3]),
                    best_Tcw=T.reshape(4, 4) if has else None, best_mask=m[:self.n].copy())

    def compute_pose(self, idx):
        idx = np.ascontiguousarray(idx, np.int32)
        R, t = np.zeros(9), np.zeros(3)
        e = self.L.pnp_compute_pose(self.h, idx.ctypes.data, len(idx), R.ctypes.data, t.ctypes.data)
        return R.reshape(3, 3), t, e

    @classmethod
    def srand(cls, seed):
        cls.lib().pnp_srand(seed)

    @classmethod
    def random_int(cls, lo, hi):
        return cls.lib().pnp_random_int(lo, hi)


def probe_count(d, s):
    """CheckInliers' count for the hypothesis of set s, from a one-iteration call on a solver whose best mask holds every
    correspondence (so the iteration never replaces it) and that has run max_its iterations (so k = 1 is valid)."""
    n = len(d["P3Dw"])
    st = (d["max_its"], n, np.eye(4, dtype=np.float32), np.ones(n, np.uint8))
    return int(iterate(d, st, np.asarray(s, np.int32).reshape(1, 4))["trace"][0, 13])


def refine_paths(n, seed):
    """(scene, state, sets) of one call that reaches every branch of the scan's Refine handling: the state carries a
    best mask of wrong matches only, with best_inliers = c1, the smallest qualifying count among probed sets of true
    matches; the sets are [S1, S1, S2] with S1 of count c1 and S2 of a larger count.  Iteration 1 qualifies without
    beating the best, so Refine fits the carried mask and fails; iteration 2 repeats it with the mask unchanged (the
    device skips that Refine, the reference runs it again and fails again); iteration 3 replaces the mask and its Refine
    succeeds.  Returns None when the scene does not allow it (the caller tries another seed)."""
    import synth_pnp as sp
    d = sp.scene(n, 0.5, seed, params=(0.99, 20, 300, 4, 0.1, 5.991))
    rng = np.random.default_rng(seed)
    good, wrong = np.where(d["truth"])[0], np.where(~d["truth"])[0]
    sets = [rng.choice(good, 4, replace=False) for _ in range(40)]
    counts = [probe_count(d, s) for s in sets]
    q = [i for i, c in enumerate(counts) if c >= d["min_inliers"]]
    if len(q) < 2:
        return None
    i1 = min(q, key=lambda i: counts[i])
    i2 = max(q, key=lambda i: counts[i])
    c1 = counts[i1]
    if counts[i2] <= c1 or c1 > len(wrong):
        return None
    mask = np.zeros(n, np.uint8)
    mask[rng.choice(wrong, c1, replace=False)] = 1
    state = (d["max_its"] - 3, c1, np.eye(4, dtype=np.float32), mask)
    S = np.array([sets[i1], sets[i1], sets[i2]], np.int32)
    tr = iterate(d, state, S)["trace"]
    m = d["min_inliers"]
    if not (0 <= tr[0, 14] <= m and 0 <= tr[1, 14] <= m and tr[2, 14] > m):
        return None
    return d, state, S


def refine_path_cases(n, count=2):
    """The first `count` seeds for which refine_paths(n, seed) exists."""
    out, seed = [], 0
    while len(out) < count and seed < 200:
        c = refine_paths(n, seed)
        if c is not None:
            out.append(c)
        seed += 1
    return out
