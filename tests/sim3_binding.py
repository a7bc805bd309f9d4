"""OptimizeSim3 checkers (test infrastructure): the CPU restatement orc_optimize_sim3 (oracle/liborb_sim3opt.so), the
reference's own Optimizer::OptimizeSim3 behind oracle/ref_sim3opt_glue.cpp (oracle/_ref/libref_sim3opt.so,
ref_optimize_sim3) and the product's drop-in body behind the same glue (oracle/_ref/libadapter_sim3opt.so,
adp_optimize_sim3)."""
import ctypes
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
ORACLE_LIB = os.path.join(ORACLE_DIR, "liborb_sim3opt.so")
REF_LIB = os.path.join(ORACLE_DIR, "_ref", "libref_sim3opt.so")
ADP_LIB = os.path.join(ORACLE_DIR, "_ref", "libadapter_sim3opt.so")
vp = ctypes.c_void_p
# Bar against the reference (its own g2o with FMA contraction, LDLT and glibc): S12 deltas within 1e-5 of the largest
# component of the reference's delta, as LocalBA's bar is.
RTOL = 1e-5
# Bar between the device and the CPU restatement: the same arithmetic in the same order except the device libm.
RTOL_DEVICE = 1e-6


class Sim3(ctypes.Structure):
    _fields_ = [("v", ctypes.c_double * 8)]


class Problem(ctypes.Structure):
    _fields_ = [("n", ctypes.c_int32)] + [(k, vp) for k in ("X1c", "X2c", "obs1", "obs2", "inv_sigma2_1",
                                                             "inv_sigma2_2")] + [
        (k, ctypes.c_float) for k in ("fx1", "fy1", "cx1", "cy1", "fx2", "fy2", "cx2", "cy2")] + [
        ("S12", Sim3), ("th2", ctypes.c_float), ("fix_scale", ctypes.c_int32)]


class Result(ctypes.Structure):
    _fields_ = [("S12_out", Sim3), ("keep", vp), ("trace", vp), ("n_inliers", ctypes.c_int32),
                ("n_trials", ctypes.c_int32)]


class Graph(ctypes.Structure):
    _fields_ = [("Tcw1", vp), ("Tcw2", vp), ("K1", vp), ("K2", vp), ("n1", ctypes.c_int), ("kp1", vp), ("oct1", vp),
                ("n2", ctypes.c_int), ("kp2", vp), ("oct2", vp), ("n_levels", ctypes.c_int), ("inv_sigma2_1", vp),
                ("inv_sigma2_2", vp), ("n_mp", ctypes.c_int), ("points", vp), ("mp_bad", vp), ("mp_idx2", vp),
                ("mp1", vp), ("matches1", vp), ("S12", Sim3), ("th2", ctypes.c_float), ("fix_scale", ctypes.c_int)]


class GraphResult(ctypes.Structure):
    _fields_ = [("match_kept", vp), ("S12_out", Sim3), ("trace", vp), ("n_trials", ctypes.c_int),
                ("ret", ctypes.c_int)]


def _lib():
    if not os.path.exists(ORACLE_LIB):
        subprocess.check_call(["make", "-s", "-C", ORACLE_DIR, "-f", "sim3opt.mk", "liborb_sim3opt.so"])
    return ctypes.CDLL(ORACLE_LIB)


def oracle(d):
    """orc_optimize_sim3 on a flattened problem; also returns the final classification's chi2 (2n)."""
    L = _lib()
    a = {k: np.ascontiguousarray(d[k], np.float32) for k in ("X1c", "X2c", "obs1", "obs2", "inv_sigma2_1",
                                                            "inv_sigma2_2")}
    n = len(a["X1c"])
    p = Problem()
    p.n = n
    for k, v in a.items():
        setattr(p, k, v.ctypes.data)
    for k, v in zip(("fx1", "fy1", "cx1", "cy1"), d["K1"]):
        setattr(p, k, float(v))
    for k, v in zip(("fx2", "fy2", "cx2", "cy2"), d["K2"]):
        setattr(p, k, float(v))
    p.S12.v[:] = [float(x) for x in d["S12"]]
    p.th2, p.fix_scale = float(d["th2"]), int(bool(d["fix_scale"]))
    out = dict(keep=np.zeros(max(n, 1), np.uint8), trace=np.full(256, -1, np.int32), chi2=np.zeros(max(2 * n, 1)))
    r = Result()
    r.keep, r.trace = out["keep"].ctypes.data, out["trace"].ctypes.data
    L.orc_optimize_sim3.argtypes = [vp, vp, vp]
    assert L.orc_optimize_sim3(ctypes.byref(p), ctypes.byref(r), out["chi2"].ctypes.data) == 0
    out["keep"], out["chi2"] = out["keep"][:n], out["chi2"][:2 * n]
    out["S12"] = np.array(r.S12_out.v[:])
    out["n_inliers"], out["n_trials"] = r.n_inliers, r.n_trials
    return out


def call_graph(fn, sc):
    """fn = ref_optimize_sim3 / adp_optimize_sim3 on the object graph of scene sc."""
    a = dict(Tcw1=np.ascontiguousarray(sc["Tcw1"], np.float32), Tcw2=np.ascontiguousarray(sc["Tcw2"], np.float32),
             K1=np.ascontiguousarray(sc["K1"], np.float32), K2=np.ascontiguousarray(sc["K2"], np.float32),
             kp1=np.ascontiguousarray(sc["kp1"], np.float32), oct1=np.ascontiguousarray(sc["oct1"], np.int32),
             kp2=np.ascontiguousarray(sc["kp2"], np.float32), oct2=np.ascontiguousarray(sc["oct2"], np.int32),
             isg=np.ascontiguousarray(sc["inv_sigma2"], np.float32), points=np.ascontiguousarray(sc["points"], np.float32),
             mp_bad=np.ascontiguousarray(sc["mp_bad"], np.uint8), mp_idx2=np.ascontiguousarray(sc["mp_idx2"], np.int32),
             mp1=np.ascontiguousarray(sc["mp1"], np.int32), matches1=np.ascontiguousarray(sc["matches1"], np.int32))
    n1, n2 = len(a["kp1"]), len(a["kp2"])
    g = Graph(a["Tcw1"].ctypes.data, a["Tcw2"].ctypes.data, a["K1"].ctypes.data, a["K2"].ctypes.data, n1,
              a["kp1"].ctypes.data, a["oct1"].ctypes.data, n2, a["kp2"].ctypes.data, a["oct2"].ctypes.data,
              len(a["isg"]), a["isg"].ctypes.data, a["isg"].ctypes.data, len(a["points"]), a["points"].ctypes.data,
              a["mp_bad"].ctypes.data, a["mp_idx2"].ctypes.data, a["mp1"].ctypes.data, a["matches1"].ctypes.data)
    g.S12.v[:] = [float(x) for x in sc["S12"]]
    g.th2, g.fix_scale = float(sc["th2"]), int(bool(sc["fix_scale"]))
    out = dict(kept=np.zeros(n1, np.uint8), trace=np.full(256, -1, np.int32))
    r = GraphResult()
    r.match_kept, r.trace = out["kept"].ctypes.data, out["trace"].ctypes.data
    fn.argtypes = [vp, vp]
    rc = fn(ctypes.byref(g), ctypes.byref(r))
    assert rc == 0, rc
    out["kept"] = out["kept"].astype(bool)
    out["S12"] = np.array(r.S12_out.v[:])
    out["ret"], out["n_trials"] = r.ret, r.n_trials
    return out


def s12_close(got, want, init, rtol):
    """S12 deltas within rtol of the largest component of the wanted delta (exact when the wanted S12 is the input)."""
    got, want, init = (np.asarray(x, np.float64) for x in (got, want, init))
    scale = np.abs(want - init).max()
    if scale == 0:
        return bool(np.array_equal(got, want)), 0.0
    err = np.abs(got - want).max() / scale
    return bool(err <= rtol), float(err)
