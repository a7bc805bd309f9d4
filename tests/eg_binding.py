"""Essential-graph checkers (test infrastructure): the CPU restatement oracle/liborb_essential.so
(orc_optimize_essential_graph) and the reference's own Optimizer::OptimizeEssentialGraph behind
oracle/ref_essential_glue.cpp (oracle/_ref/libref_essential.so, ref_essential_graph), and the product's drop-in body
behind the same glue (oracle/_ref/libadapter_essential.so, adp_essential_graph).

A map (tests/synth_essential.py) is what the object graph holds.  flatten() is the gather of the reference's steps 2-4
(src/Optimizer.cc:1059-1262): the non-bad keyframes by ascending id, their initial Sim3s, and the edges in the
reference's insertion order with its own measurement expressions, computed with the oracle's g2o::Sim3 operations.
expand() is the scatter (:1274-1338)."""
import ctypes
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
ORACLE_LIB = os.path.join(ORACLE_DIR, "liborb_essential.so")
REF_LIB = os.path.join(ORACLE_DIR, "_ref", "libref_essential.so")
ADP_LIB = os.path.join(ORACLE_DIR, "_ref", "libadapter_essential.so")
vp = ctypes.c_void_p
# Bar against the reference.  The reference is this sensitive on its own: on the 12 maps of
# test_essential_graph_random_sweep, moving one keyframe's tx by one float32 ulp moves the reference's output poses by up
# to 1.1e-3 of its largest pose delta (sweep map 3; 1.9e-4 on map 7, 2e-5 on map 9, below 1e-5 elsewhere) and changes
# the accept / reject tail of map 8.  Lambda 1e-16 with numeric Jacobians (delta = 1e-9) amplifies rounding that much,
# so a restatement with another summation order or libm cannot be held closer than that; deltas are held to 5e-3.
RTOL = 5e-3
# Bar between the device and the CPU restatement: the same arithmetic except the Cholesky's summation order and the
# device libm, on a map whose run is one accepted step (the first iteration's linearisation and solve) and then rejections.
RTOL_DEVICE = 1e-6
MIN_FEAT = 100
edge_dtype = np.dtype([("i", np.int32), ("j", np.int32), ("meas", np.float64, 8)])


class EgProblem(ctypes.Structure):
    _fields_ = [("n_kf", ctypes.c_int), ("Siw", vp), ("fixed_kf", ctypes.c_int), ("fix_scale", ctypes.c_int),
                ("n_edges", ctypes.c_int), ("edges", vp), ("n_mp", ctypes.c_int), ("points", vp), ("ref_kf", vp)]


class EgResult(ctypes.Structure):
    _fields_ = [("Tcw_out", vp), ("points_out", vp), ("trace", vp), ("chi2_initial", ctypes.c_double),
                ("chi2_final", ctypes.c_double), ("n_trials", ctypes.c_int)]


class EgMap(ctypes.Structure):
    _fields_ = [("n_kf", ctypes.c_int), ("Tcw", vp), ("kf_bad", vp), ("parent", vp), ("n_loop", ctypes.c_int),
                ("loop_edges", vp), ("n_cov", ctypes.c_int), ("cov", vp), ("loop_kf", ctypes.c_int),
                ("cur_kf", ctypes.c_int), ("n_corr", ctypes.c_int), ("corr_kf", vp), ("corr_S", vp), ("noncorr_S", vp),
                ("n_conn", ctypes.c_int), ("conn", vp), ("n_mp", ctypes.c_int), ("points", vp), ("mp_bad", vp),
                ("mp_ref", vp), ("mp_corrected_by", vp), ("mp_corrected_ref", vp), ("fix_scale", ctypes.c_int)]


class EgMapResult(ctypes.Structure):
    _fields_ = [("Tcw_out", vp), ("points_out", vp), ("mp_updates", vp), ("trace", vp), ("n_trials", ctypes.c_int)]


def _lib():
    if not os.path.exists(ORACLE_LIB):
        subprocess.check_call(["make", "-s", "-C", ORACLE_DIR, "-f", "essential.mk", "liborb_essential.so"])
    return ctypes.CDLL(ORACLE_LIB)


class Sim3Ops:
    """g2o::Sim3 operations of a library (prefix orc_ or ref_) on 8-vectors qx qy qz qw tx ty tz s."""

    def __init__(self, L, prefix):
        self.f = {k: getattr(L, prefix + k) for k in ("exp", "log", "mul", "inverse", "map")}
        self.from_Rt = getattr(L, prefix + "from_Rt", None)

    def _out(self, n):
        return np.zeros(n, np.float64)

    def exp(self, u):
        o = self._out(8)
        self.f["exp"](np.ascontiguousarray(u, np.float64).ctypes.data_as(vp), o.ctypes.data_as(vp))
        return o

    def log(self, a):
        o = self._out(7)
        self.f["log"](np.ascontiguousarray(a, np.float64).ctypes.data_as(vp), o.ctypes.data_as(vp))
        return o

    def mul(self, a, b):
        o = self._out(8)
        self.f["mul"](np.ascontiguousarray(a, np.float64).ctypes.data_as(vp),
                      np.ascontiguousarray(b, np.float64).ctypes.data_as(vp), o.ctypes.data_as(vp))
        return o

    def inverse(self, a):
        o = self._out(8)
        self.f["inverse"](np.ascontiguousarray(a, np.float64).ctypes.data_as(vp), o.ctypes.data_as(vp))
        return o

    def map(self, a, x):
        o = self._out(3)
        self.f["map"](np.ascontiguousarray(a, np.float64).ctypes.data_as(vp),
                      np.ascontiguousarray(x, np.float64).ctypes.data_as(vp), o.ctypes.data_as(vp))
        return o

    def Rt(self, R, t, s):
        o = self._out(8)
        self.from_Rt(np.ascontiguousarray(R, np.float64).ctypes.data_as(vp),
                     np.ascontiguousarray(t, np.float64).ctypes.data_as(vp), ctypes.c_double(s), o.ctypes.data_as(vp))
        return o


def flatten(m, ops=None):
    """The drop-in body's gather: returns (problem dict, keyframe ids, point ids)."""
    ops = ops or Sim3Ops(_lib(), "orc_sim3_")
    n = len(m["kf_bad"])
    kf_ids = np.where(m["kf_bad"] == 0)[0]
    idx = np.full(n, -1, np.int64)
    idx[kf_ids] = np.arange(len(kf_ids))
    corr = {int(k): m["corr_S"][a] for a, k in enumerate(m["corr_kf"])}
    noncorr = {int(k): m["noncorr_S"][a] for a, k in enumerate(m["corr_kf"])}
    vScw = {}
    for k in kf_ids:
        k = int(k)
        if k in corr:
            vScw[k] = corr[k]
        else:
            T = m["Tcw"][k].reshape(4, 4).astype(np.float64)
            vScw[k] = ops.Rt(T[:3, :3], T[:3, 3], 1.0)
    W = {}
    covis = {k: [] for k in range(n)}
    for k, j, w in m["cov"]:
        W[(int(k), int(j))] = int(w)
        covis[int(k)].append(int(j))
    children = {k: set() for k in range(n)}
    for k in kf_ids:
        if m["parent"][k] >= 0:
            children[int(m["parent"][k])].add(int(k))
    loops = {k: set() for k in range(n)}
    for a, b in m["loop_edges"]:
        loops[int(a)].add(int(b))
    conns = {}
    for a, b in m["conn"]:
        conns.setdefault(int(a), set()).add(int(b))
    cur, loop = int(m["cur_kf"]), int(m["loop_kf"])
    edges, inserted = [], set()

    def add(i, j, S):
        edges.append((idx[i], idx[j], S))

    for k in sorted(conns):  # LoopConnections (:1108-1143)
        Swi = ops.inverse(vScw[k])
        for j in sorted(conns[k]):
            if (k != cur or j != loop) and W.get((k, j), 0) < MIN_FEAT:
                continue
            add(k, j, ops.mul(vScw[j], Swi))
            inserted.add((min(k, j), max(k, j)))
    for k in kf_ids:  # normal edges (:1147-1262)
        k = int(k)
        Swi = ops.inverse(noncorr[k]) if k in noncorr else ops.inverse(vScw[k])
        par = int(m["parent"][k])
        if par >= 0:
            add(k, par, ops.mul(noncorr[par] if par in noncorr else vScw[par], Swi))
        for l in sorted(loops[k]):
            if l < k:
                add(k, l, ops.mul(noncorr[l] if l in noncorr else vScw[l], Swi))
        for nb in covis[k]:
            if W[(k, nb)] < MIN_FEAT:
                continue
            if nb != par and nb not in children[k] and nb not in loops[k]:
                if not m["kf_bad"][nb] and nb < k:
                    if (min(k, nb), max(k, nb)) in inserted:
                        continue
                    add(k, nb, ops.mul(noncorr[nb] if nb in noncorr else vScw[nb], Swi))
    e = np.zeros(len(edges), edge_dtype)
    for a, (i, j, S) in enumerate(edges):
        e[a] = (i, j, S)
    mp_ids = np.where(m["mp_bad"] == 0)[0]
    nid = np.where(m["mp_corrected_by"][mp_ids] == cur, m["mp_corrected_ref"][mp_ids], m["mp_ref"][mp_ids])
    ref_kf = idx[nid].astype(np.int32)
    d = dict(Siw=np.array([vScw[int(k)] for k in kf_ids], np.float64).reshape(-1, 8), fixed_kf=int(idx[loop]),
             fix_scale=bool(m["fix_scale"]), edges=e, points=np.ascontiguousarray(m["points"][mp_ids]), ref_kf=ref_kf)
    return d, kf_ids, mp_ids


def expand(m, flat, kf_ids, mp_ids):
    """The scatter (:1274-1338): SetPose of every map keyframe, SetWorldPos + UpdateNormalAndDepth of every good point."""
    out = dict(Tcw=np.array(m["Tcw"], np.float32, copy=True), points=np.array(m["points"], np.float32, copy=True),
               mp_updates=np.zeros(len(m["mp_bad"]), np.int32))
    out["Tcw"][kf_ids] = flat["Tcw"]
    out["points"][mp_ids] = flat["points"]
    out["mp_updates"][mp_ids] = 1
    out["trace"], out["n_trials"] = flat["trace"], flat["n_trials"]
    return out


def call_flat(fn, d):
    Siw = np.ascontiguousarray(d["Siw"], np.float64).reshape(-1, 8)
    edges = np.ascontiguousarray(d["edges"])
    pts = np.ascontiguousarray(d["points"], np.float32).reshape(-1, 3)
    ref = np.ascontiguousarray(d["ref_kf"], np.int32)
    p = EgProblem(len(Siw), Siw.ctypes.data, int(d["fixed_kf"]), int(bool(d["fix_scale"])), len(edges), edges.ctypes.data,
                  len(pts), pts.ctypes.data, ref.ctypes.data)
    out = dict(Tcw=np.zeros((len(Siw), 16), np.float32), points=np.zeros((len(pts), 3), np.float32),
               trace=np.full(256, -1, np.int32))
    r = EgResult(out["Tcw"].ctypes.data, out["points"].ctypes.data, out["trace"].ctypes.data, 0.0, 0.0, 0)
    fn.argtypes = [vp, vp]
    assert fn(ctypes.byref(p), ctypes.byref(r)) == 0
    out["chi2_initial"], out["chi2"], out["n_trials"] = r.chi2_initial, r.chi2_final, r.n_trials
    return out


def call_map(fn, m):
    """fn = ref_essential_graph on the object graph of map m.  Returns the map-wide outputs."""
    arrs = {k: np.ascontiguousarray(m[k]) for k in ("Tcw", "kf_bad", "parent", "loop_edges", "cov", "corr_kf", "corr_S",
                                                    "noncorr_S", "conn", "points", "mp_bad", "mp_ref", "mp_corrected_by",
                                                    "mp_corrected_ref")}
    a = {k: v.ctypes.data for k, v in arrs.items()}
    nk, nm = len(arrs["kf_bad"]), len(arrs["mp_bad"])
    p = EgMap(nk, a["Tcw"], a["kf_bad"], a["parent"], len(arrs["loop_edges"]), a["loop_edges"], len(arrs["cov"]), a["cov"],
              int(m["loop_kf"]), int(m["cur_kf"]), len(arrs["corr_kf"]), a["corr_kf"], a["corr_S"], a["noncorr_S"],
              len(arrs["conn"]), a["conn"], nm, a["points"], a["mp_bad"], a["mp_ref"], a["mp_corrected_by"],
              a["mp_corrected_ref"], int(bool(m["fix_scale"])))
    out = dict(Tcw=np.zeros((nk, 16), np.float32), points=np.zeros((nm, 3), np.float32), mp_updates=np.zeros(nm, np.int32),
               trace=np.full(256, -1, np.int32))
    r = EgMapResult(out["Tcw"].ctypes.data, out["points"].ctypes.data, out["mp_updates"].ctypes.data,
                    out["trace"].ctypes.data, 0)
    fn.argtypes = [vp, vp]
    rc = fn(ctypes.byref(p), ctypes.byref(r))
    assert rc == 0, rc
    out["n_trials"] = r.n_trials
    return out


def traces_agree(tg, tw):
    """Accept / reject sequences of two runs agree up to the converged tail: identical up to their first difference,
    after which each run accepts at most one more (noise-level) step."""
    tg, tw = list(tg), list(tw)
    i = 0
    while i < min(len(tg), len(tw)) and tg[i] == tw[i]:
        i += 1
    return sum(tg[i:]) <= 1 and sum(tw[i:]) <= 1 and (i > 0 or not tw)


def close(got, want, init, rtol=RTOL):
    """Deltas within RTOL of the largest reference delta, plus one float32 ulp of the written value (of 1 for values
    below 1: rotation entries near zero)."""
    got, want, init = (np.asarray(x, np.float64) for x in (got, want, init))
    scale = max(np.abs(want - init).max(), 1e-12) if want.size else 1e-12
    ulp = np.spacing(np.maximum(np.abs(want), 1.0).astype(np.float32)).astype(np.float64)
    err = np.abs(got - want)
    return bool((err <= rtol * scale + ulp).all()), float((err / scale).max()) if err.size else 0.0


class Oracle:
    def __init__(self):
        self.L = _lib()

    def essential_graph(self, d):
        return call_flat(self.L.orc_optimize_essential_graph, d)


class Cuda:
    def __init__(self, pkg, **caps):
        self.opt = pkg.EssentialGraphOptimizer(**caps) if caps else pkg.EssentialGraphOptimizer(
            max_kf=1024, max_edges=1 << 14, max_mp=1 << 16)

    def essential_graph(self, d):
        return self.opt.OptimizeEssentialGraph(d)
