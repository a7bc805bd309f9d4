"""ctypes bindings of the covisibility-update checkers, behind the call of pkg.Covisibility.UpdateConnections:

  Oracle()                  oracle/liborb_covis.so, the CPU restatement (oracle/covis.cpp)
  Reference()               oracle/_ref/libref_keyframe.so, the reference's own src/KeyFrame.cc on a fresh object graph
  Reference(adapter=True)   oracle/_ref/libadapter_covis.so, the product's host/adapters/Covisibility_b200.cc on the same
                            glue (one device call per batch)

and World, a keyframe graph whose state is carried from call to call, with the seeded maps the tests and
tools/covis_time.py replay."""
import ctypes
import importlib
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_LIB = os.path.join(ROOT, "oracle", "liborb_covis.so")
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libref_keyframe.so")
ADP_LIB = os.path.join(ROOT, "oracle", "_ref", "libadapter_covis.so")
pkg = importlib.import_module("self_commit_orb-slam2_b200")
vp = ctypes.c_void_p
CAP = 1 << 22


class Oracle:
    def __init__(self):
        self.L = ctypes.CDLL(ORACLE_LIB)
        self.L.orc_update_connections.argtypes = [vp, vp]

    def UpdateConnections(self, d):
        rc, o = pkg.covis_call(self.L.orc_update_connections, d, CAP)
        assert rc == 0
        return pkg.covis_state(d, o)


class Reference:
    """The reference's KeyFrame::UpdateConnections on the members one after another.  UpdateConnections(d) also takes
    d["kf_bad"] (KeyFrame::mbBad, which the call never reads) and d["children"] (mspChildrens on entry, a list of
    sets); the result has "children" after the batch and "wall_ns", the time of the calls alone."""

    def __init__(self, adapter=False):
        self.L = ctypes.CDLL(ADP_LIB if adapter else REF_LIB)
        self.f = getattr(self.L, ("adp_" if adapter else "ref_") + "update_connections")
        self.f.argtypes = [vp, vp, vp, vp, vp, vp, vp, ctypes.c_int, vp]

    def UpdateConnections(self, d):
        n = len(d["kf_id"])
        bad = np.ascontiguousarray(d.get("kf_bad", np.zeros(n, np.uint8)), np.uint8)
        ch = d.get("children") or [set() for _ in range(n)]
        c_off = np.concatenate([[0], np.cumsum([len(c) for c in ch])]).astype(np.int32)
        c_kf = np.array([k for c in ch for k in sorted(c)] or [0], np.int32)
        oc_off = np.zeros(n + 1, np.int32)
        oc_kf = np.zeros(c_off[-1] + len(d["member"]) + 1, np.int32)
        ns = ctypes.c_double(0)
        rc, o = pkg.covis_call(lambda p, r: self.f(p, bad.ctypes.data, c_off.ctypes.data, c_kf.ctypes.data, r,
                                                   oc_off.ctypes.data, oc_kf.ctypes.data, len(oc_kf),
                                                   ctypes.byref(ns)), d, CAP)
        assert rc == 0, rc
        s = pkg.covis_state(d, o)
        s["children"] = [set(oc_kf[oc_off[i]:oc_off[i + 1]].tolist()) for i in range(n)]
        s["wall_ns"] = ns.value
        return s


def counters(d):
    """The counter KFcounter of each call, {partner: weight} (only to check which cases a test reaches)."""
    out = []
    for b, m in enumerate(d["member"]):
        c = {}
        for s in d["slot_mp"][d["slot_off"][b]:d["slot_off"][b + 1]]:
            if s < 0 or d["mp_bad"][s]:
                continue
            for o in d["obs_kf"][d["obs_off"][s]:d["obs_off"][s + 1]]:
                if o != m:
                    c[int(o)] = c.get(int(o), 0) + 1
        out.append(c)
    return out


class World:
    """n keyframes (ids ascending) with connection state, slots and map points; problem() flattens it for a batch and
    apply() takes a call's state back.  Observers of a point are kept ascending."""

    def __init__(self, ids):
        self.ids = np.asarray(ids, np.uint64)
        n = len(ids)
        self.conn = [dict() for _ in range(n)]
        self.ordKf = [[] for _ in range(n)]
        self.ordW = [[] for _ in range(n)]
        self.first = np.ones(n, np.uint8)
        self.parent = np.full(n, -1, np.int32)
        self.children = [set() for _ in range(n)]
        self.kf_bad = np.zeros(n, np.uint8)
        self.slots = [[] for _ in range(n)]
        self.obs = []
        self.mp_bad = []

    def add_point(self, observers=()):
        self.obs.append(sorted(set(observers)))
        self.mp_bad.append(0)
        return len(self.obs) - 1

    def problem(self, members):
        n = len(self.ids)
        d = {"kf_id": self.ids, "first_connection": self.first.copy(), "parent": self.parent.copy(),
             "mp_bad": np.array(self.mp_bad, np.uint8), "member": np.array(members, np.int32),
             "kf_bad": self.kf_bad.copy(), "children": [set(c) for c in self.children]}
        mk = [sorted(c) for c in self.conn]
        d["map_off"] = np.concatenate([[0], np.cumsum([len(x) for x in mk])]).astype(np.int32)
        d["map_kf"] = np.array([k for x in mk for k in x], np.int32)
        d["map_w"] = np.array([self.conn[i][k] for i, x in enumerate(mk) for k in x], np.int32)
        d["list_off"] = np.concatenate([[0], np.cumsum([len(x) for x in self.ordKf])]).astype(np.int32)
        d["list_kf"] = np.array([k for x in self.ordKf for k in x], np.int32)
        d["list_w"] = np.array([w for x in self.ordW for w in x], np.int32)
        d["obs_off"] = np.concatenate([[0], np.cumsum([len(x) for x in self.obs])]).astype(np.int32)
        d["obs_kf"] = np.array([k for x in self.obs for k in x], np.int32)
        sl = [self.slots[m] for m in members]
        d["slot_off"] = np.concatenate([[0], np.cumsum([len(x) for x in sl])]).astype(np.int32)
        d["slot_mp"] = np.array([s for x in sl for s in x], np.int32)
        return d

    def apply(self, s):
        for i in range(len(self.ids)):
            a, b = s["map_off"][i], s["map_off"][i + 1]
            self.conn[i] = dict(zip(s["map_kf"][a:b].tolist(), s["map_w"][a:b].tolist()))
            a, b = s["list_off"][i], s["list_off"][i + 1]
            self.ordKf[i] = s["list_kf"][a:b].tolist()
            self.ordW[i] = s["list_w"][a:b].tolist()
        self.first = s["first_connection"].copy()
        self.parent = s["parent"].copy()
        if "children" in s:  # the reference reports mspChildrens itself
            self.children = [set(c) for c in s["children"]]
        for p, c in s["pairs"]:
            self.children[p].add(int(c))


def same(want, got, n_kf):
    """Asserts two states are equal: every keyframe's map, list, parent, first flag, and the per-call reads."""
    for k in ("parent", "first_connection", "map_off", "map_kf", "map_w", "list_off", "list_kf", "list_w", "start_off",
              "start_kf", "after_off", "after_kf", "after_w"):
        assert np.array_equal(np.asarray(want[k]), np.asarray(got[k])), k


# ------------------------------------------------------------------------------------------------ seeded maps
def trajectory(seed, n_kf, pts_per_kf=120, null_frac=0.05, bad_frac=0.03, revisit=None, ids=None):
    """A camera path: keyframe i creates pts_per_kf points, each observed by a run of 2-10 consecutive keyframes from i
    (and, with revisit = P, also by keyframes around i + P: the path comes back).  Returns the World, with the points'
    full observer lists in w.runs and no observation yet (add them with observe(i))."""
    rng = np.random.default_rng(seed)
    w = World(np.arange(n_kf) * 2 + 1 if ids is None else ids)
    runs = []
    for i in range(n_kf):
        for _ in range(pts_per_kf):
            L = int(rng.integers(2, 11))
            run = list(range(i, min(n_kf, i + L)))
            if revisit and i + revisit < n_kf and rng.random() < 0.3:
                run += list(range(i + revisit, min(n_kf, i + revisit + int(rng.integers(1, 4)))))
            p = w.add_point()
            runs.append(sorted(set(run)))
            if rng.random() < bad_frac:
                w.mp_bad[p] = 1
    slots = [[] for _ in range(n_kf)]
    for p, run in enumerate(runs):
        for k in run:
            slots[k].append(p)
    for k in range(n_kf):
        rng.shuffle(slots[k])
        sl = slots[k]
        for _ in range(int(null_frac * len(sl))):
            sl.insert(int(rng.integers(0, len(sl) + 1)), -1)
        w.slots[k] = sl
    w.runs = runs
    return w


def observe(w, i):
    """Keyframe i's observations join its points' observer lists (KeyFrame insertion)."""
    for p in w.slots[i]:
        if p >= 0 and i in w.runs[p] and i not in w.obs[p]:
            w.obs[p] = sorted(w.obs[p] + [i])


def random_map(seed, n_kf, slots_per_kf=200, zipf=1.6):
    """n_kf keyframes, points with Zipf-distributed observation counts (2..12) over clustered keyframes, NULL slots and
    bad points; every keyframe's observations are in place."""
    rng = np.random.default_rng(seed)
    ids = np.sort(rng.choice(10 * n_kf, n_kf, replace=False)).astype(np.uint64)
    if rng.random() < 0.5:
        ids[0] = 0
    w = World(ids)
    n_pts = n_kf * slots_per_kf // 4
    slots = [[] for _ in range(n_kf)]
    for _ in range(n_pts):
        k = int(min(12, max(2, rng.zipf(zipf) + 1)))
        c = int(rng.integers(0, n_kf))
        obs = set()
        while len(obs) < min(k, n_kf):
            obs.add(int(np.clip(c + rng.integers(-8, 9), 0, n_kf - 1)) if rng.random() < 0.85 else int(rng.integers(0, n_kf)))
        p = w.add_point(obs)
        if rng.random() < 0.03:
            w.mp_bad[p] = 1
        for o in obs:
            slots[o].append(p)
    for k in range(n_kf):
        rng.shuffle(slots[k])
        w.slots[k] = slots[k] + [-1] * int(rng.integers(0, 5))
    w.kf_bad[rng.random(n_kf) < 0.05] = 1
    return w
