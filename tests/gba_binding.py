"""Global bundle adjustment checkers (test infrastructure): the CPU restatement oracle/liborb_gba.so (orc_global_ba), the
reference's own Optimizer::GlobalBundleAdjustemnt behind oracle/ref_gba_glue.cpp (oracle/_ref/libref_gba.so,
ref_global_ba) and the product's drop-in body behind the same glue (oracle/_ref/libadapter_gba.so, adp_global_ba).

A map (tests/synth_gba.py synth_global_ba) is what the object graph holds: every keyframe and point, bad ones included, and
every observation.  flatten() is the gather the drop-in body performs (src/Optimizer.cc:86-275): the non-bad keyframes
and points by ascending id, the observations of non-bad keyframes, mnId == 0 fixed."""
import ctypes
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
ORACLE_LIB = os.path.join(ORACLE_DIR, "liborb_gba.so")
REF_LIB = os.path.join(ORACLE_DIR, "_ref", "libref_gba.so")
ADP_LIB = os.path.join(ORACLE_DIR, "_ref", "libadapter_gba.so")
vp = ctypes.c_void_p
RTOL = 1e-5


class GbaProblem(ctypes.Structure):
    _fields_ = [("n_kf", ctypes.c_int), ("Tcw", vp), ("fixed", vp), ("n_mp", ctypes.c_int), ("points", vp),
                ("n_edges", ctypes.c_int), ("edges", vp), ("fx", ctypes.c_float), ("fy", ctypes.c_float),
                ("cx", ctypes.c_float), ("cy", ctypes.c_float), ("bf", ctypes.c_float), ("iterations", ctypes.c_int),
                ("robust", ctypes.c_int)]


class GbaResult(ctypes.Structure):
    _fields_ = [("Tcw_out", vp), ("points_out", vp), ("point_included", vp), ("trace", vp),
                ("chi2_final", ctypes.c_double), ("n_trials", ctypes.c_int)]


class GbaMap(ctypes.Structure):
    _fields_ = [("n_kf", ctypes.c_int), ("Tcw", vp), ("kf_bad", vp), ("n_mp", ctypes.c_int), ("points", vp),
                ("mp_bad", vp), ("n_obs", ctypes.c_int), ("obs", vp), ("fx", ctypes.c_float), ("fy", ctypes.c_float),
                ("cx", ctypes.c_float), ("cy", ctypes.c_float), ("bf", ctypes.c_float), ("iterations", ctypes.c_int),
                ("robust", ctypes.c_int), ("loop_kf", ctypes.c_uint64)]


class GbaMapResult(ctypes.Structure):
    _fields_ = [("Tcw_out", vp), ("points_out", vp), ("kf_gba", vp), ("mp_gba", vp), ("kf_ba_global", vp),
                ("mp_ba_global", vp), ("mp_updates", vp), ("trace", vp), ("n_trials", ctypes.c_int)]


def flatten(m):
    """The drop-in body's gather: returns (problem dict, keyframe ids, point ids)."""
    kf_ids = np.where(m["kf_bad"] == 0)[0]
    mp_ids = np.where(m["mp_bad"] == 0)[0]
    max_kf = int(kf_ids.max()) if len(kf_ids) else 0
    kf_new = np.full(len(m["kf_bad"]), -1, np.int64)
    kf_new[kf_ids] = np.arange(len(kf_ids))
    mp_new = np.full(len(m["mp_bad"]), -1, np.int64)
    mp_new[mp_ids] = np.arange(len(mp_ids))
    o = m["obs"]
    keep = (m["mp_bad"][o["mp"]] == 0) & (m["kf_bad"][o["kf"]] == 0) & (o["kf"] <= max_kf)
    e = o[keep].copy()
    e["kf"] = kf_new[e["kf"]]
    e["mp"] = mp_new[e["mp"]]
    d = dict(Tcw=np.ascontiguousarray(m["Tcw"][kf_ids]), fixed=(kf_ids == 0).astype(np.uint8),
             points=np.ascontiguousarray(m["points"][mp_ids]), edges=np.ascontiguousarray(e),
             fx=m["fx"], fy=m["fy"], cx=m["cx"], cy=m["cy"], bf=m["bf"])
    return d, kf_ids, mp_ids


def call_flat(fn, d, iterations, robust, stop=None):
    """fn(const orc_gba_problem*, const uint8_t* stop, orc_gba_result*): orc_global_ba."""
    Tcw = np.ascontiguousarray(d["Tcw"], np.float32).reshape(-1, 16)
    fixed = np.ascontiguousarray(d["fixed"], np.uint8)
    pts = np.ascontiguousarray(d["points"], np.float32).reshape(-1, 3)
    edges = np.ascontiguousarray(d["edges"])
    p = GbaProblem(len(Tcw), Tcw.ctypes.data, fixed.ctypes.data, len(pts), pts.ctypes.data, len(edges), edges.ctypes.data,
                   d["fx"], d["fy"], d["cx"], d["cy"], d["bf"], int(iterations), int(bool(robust)))
    out = dict(Tcw=np.zeros((len(Tcw), 16), np.float32), points=pts.copy(), point_included=np.zeros(len(pts), np.uint8),
               trace=np.full(256, -1, np.int32))
    r = GbaResult(out["Tcw"].ctypes.data, out["points"].ctypes.data, out["point_included"].ctypes.data,
                  out["trace"].ctypes.data, 0.0, 0)
    fn.argtypes = [vp, vp, vp]
    rc = fn(ctypes.byref(p), None if stop is None else stop.ctypes.data_as(vp), ctypes.byref(r))
    assert rc == 0
    out["chi2"] = r.chi2_final
    out["n_trials"] = r.n_trials
    return out


def call_map(fn, m, iterations, robust, loop_kf, stop=None):
    """fn = ref_global_ba / adp_global_ba on the object graph of map m.  Returns the map-wide outputs."""
    Tcw = np.ascontiguousarray(m["Tcw"], np.float32)
    pts = np.ascontiguousarray(m["points"], np.float32)
    kb = np.ascontiguousarray(m["kf_bad"], np.uint8)
    mb = np.ascontiguousarray(m["mp_bad"], np.uint8)
    obs = np.ascontiguousarray(m["obs"])
    nk, nm = len(Tcw), len(pts)
    p = GbaMap(nk, Tcw.ctypes.data, kb.ctypes.data, nm, pts.ctypes.data, mb.ctypes.data, len(obs), obs.ctypes.data,
               m["fx"], m["fy"], m["cx"], m["cy"], m["bf"], int(iterations), int(bool(robust)), int(loop_kf))
    out = dict(Tcw=np.zeros((nk, 16), np.float32), points=np.zeros((nm, 3), np.float32), kf_gba=np.zeros(nk, np.uint8),
               mp_gba=np.zeros(nm, np.uint8), kf_ba_global=np.zeros(nk, np.uint64), mp_ba_global=np.zeros(nm, np.uint64),
               mp_updates=np.zeros(nm, np.int32), trace=np.full(256, -1, np.int32))
    r = GbaMapResult(*[out[k].ctypes.data for k in ("Tcw", "points", "kf_gba", "mp_gba", "kf_ba_global", "mp_ba_global",
                                                    "mp_updates", "trace")], 0)
    fn.argtypes = [vp, vp, vp]
    rc = fn(ctypes.byref(p), None if stop is None else stop.ctypes.data_as(vp), ctypes.byref(r))
    assert rc == 0, rc
    out["n_trials"] = r.n_trials
    return out


def expand(m, flat, kf_ids, mp_ids, loop_kf):
    """The map-wide outputs the drop-in body's scatter produces from a flattened result (src/Optimizer.cc:287-340)."""
    nk, nm = len(m["kf_bad"]), len(m["mp_bad"])
    none = np.uint64(0xFFFFFFFFFFFFFFFF)
    out = dict(Tcw=np.array(m["Tcw"], np.float32, copy=True), points=np.array(m["points"], np.float32, copy=True),
               kf_gba=np.zeros(nk, np.uint8), mp_gba=np.zeros(nm, np.uint8), kf_ba_global=np.full(nk, none, np.uint64),
               mp_ba_global=np.full(nm, none, np.uint64), mp_updates=np.zeros(nm, np.int32))
    out["Tcw"][kf_ids] = flat["Tcw"]
    inc = mp_ids[flat["point_included"] != 0]
    out["points"][inc] = flat["points"][flat["point_included"] != 0]
    if loop_kf:
        out["kf_gba"][kf_ids] = 1
        out["kf_ba_global"][kf_ids] = loop_kf
        out["mp_gba"][inc] = 1
        out["mp_ba_global"][inc] = loop_kf
    else:
        out["mp_updates"][inc] = 1
    out["trace"], out["n_trials"] = flat["trace"], flat["n_trials"]
    return out


def close(got, want, init):
    """Deltas within RTOL of the largest reference delta, plus one float32 ulp of the written value."""
    got, want, init = (np.asarray(a, np.float64) for a in (got, want, init))
    scale = max(np.abs(want - init).max(), 1e-12) if want.size else 1e-12
    ulp = np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
    err = np.abs(got - want)
    return bool((err <= RTOL * scale + ulp).all()), float((err / scale).max()) if err.size else 0.0


class Oracle:
    def __init__(self):
        if not os.path.exists(ORACLE_LIB):
            subprocess.check_call(["make", "-s", "-C", ORACLE_DIR, "-f", "gba.mk", "liborb_gba.so"])
        self.L = ctypes.CDLL(ORACLE_LIB)

    def global_ba(self, d, iterations=10, robust=True, stop=None):
        return call_flat(self.L.orc_global_ba, d, iterations, robust, stop)


class Cuda:
    def __init__(self, pkg, **caps):
        self.opt = pkg.GlobalOptimizer(**caps) if caps else pkg.GlobalOptimizer(max_kf=512, max_mp=65536, max_edges=1 << 19)

    def global_ba(self, d, iterations=10, robust=True, stop=None):
        return self.opt.BundleAdjustment(d, iterations=iterations, robust=robust, stop=stop)
