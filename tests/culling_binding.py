"""ctypes bindings of the keyframe-culling checkers, beside pkg.KeyFrameCulling:

  Oracle()                  oracle/liborb_culling.so, the CPU restatement (oracle/culling.cpp), one problem per call
  Reference()               oracle/_ref/libref_localmapping.so, the reference's own LocalMapping::KeyFrameCulling (with
                            its real KeyFrame::SetBadFlag and MapPoint code) on a fresh object graph
  Reference(adapter=True)   oracle/_ref/libadapter_culling.so, the product's host/adapters/LocalMapping_b200.cc on the
                            same glue

and World, a keyframe / map-point graph with each keyframe's per-index octaves, right coordinates and depths, with the
seeded maps the tests and tools/culling_time.py use."""
import ctypes
import importlib
import os

import numpy as np
import scipy.sparse as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_LIB = os.path.join(ROOT, "oracle", "liborb_culling.so")
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libref_localmapping.so")
ADP_LIB = os.path.join(ROOT, "oracle", "_ref", "libadapter_culling.so")
pkg = importlib.import_module("self_commit_orb-slam2_b200")
vp = ctypes.c_void_p
OUT_KEYS = ("verdict", "n_mps", "n_redundant", "mp_bad", "mp_nobs", "obs_alive", "slot_mp")


class Oracle:
    def __init__(self):
        self.L = ctypes.CDLL(ORACLE_LIB)
        self.L.orc_keyframe_culling.argtypes = [vp, vp]

    def __call__(self, ds):
        one = isinstance(ds, dict)
        outs = []
        for d in ([ds] if one else ds):
            p, keep = pkg.culling_problem(d)
            r, o = pkg.culling_outputs(d)
            assert self.L.orc_keyframe_culling(ctypes.byref(p), ctypes.byref(r)) == 0
            o["n_culled"] = r.n_culled
            outs.append(o)
        return outs[0] if one else outs


class Reference:
    """The reference's KeyFrameCulling on a World's object graph: __call__(w, d, cur) with d = w.problem(...) and cur
    the current keyframe.  The result has the fields of b2s_culling_result (n_mps and n_redundant -1) and the keyframe
    state after the call: kf_bad, to_be_erased, parent, conn (a dict per keyframe), children (a set per keyframe),
    erased (the culls in SetBadFlag order) and wall_ns (the time of the culling alone)."""

    def __init__(self, adapter=False):
        self.L = ctypes.CDLL(ADP_LIB if adapter else REF_LIB)
        self.f = getattr(self.L, ("adp_" if adapter else "ref_") + "keyframe_culling")
        self.f.argtypes = [vp, ctypes.c_int] + [vp] * 13 + [ctypes.c_int, vp, vp, ctypes.c_int, vp]

    def __call__(self, w, d, cur):
        n = len(w.ids)
        parent = np.ascontiguousarray(w.parent, np.int32)
        c_off, c_kf, c_w = w.connections()
        p, keep = pkg.culling_problem(d)
        r, o = pkg.culling_outputs(d)
        cap = len(c_kf) + 1
        kb, tb = np.zeros(n, np.uint8), np.zeros(n, np.uint8)
        po, er, ne = np.zeros(n, np.int32), np.zeros(n, np.int32), ctypes.c_int32(0)
        co_off, co_kf, co_w = np.zeros(n + 1, np.int32), np.zeros(cap, np.int32), np.zeros(cap, np.int32)
        ch_off, ch_kf = np.zeros(n + 1, np.int32), np.zeros(n + 1, np.int32)
        ns = ctypes.c_double(0)
        a = lambda x: x.ctypes.data  # noqa: E731
        rc = self.f(ctypes.byref(p), cur, a(parent), a(c_off), a(c_kf), a(c_w), ctypes.byref(r), a(kb), a(tb), a(po),
                    a(er), ctypes.byref(ne), a(co_off), a(co_kf), a(co_w), cap, a(ch_off), a(ch_kf), n + 1,
                    ctypes.byref(ns))
        assert rc == 0, rc
        o["n_culled"] = r.n_culled
        o.update(kf_bad=kb, to_be_erased=tb, parent=po, erased=er[:ne.value].tolist(), wall_ns=ns.value,
                 conn=[dict(zip(co_kf[co_off[i]:co_off[i + 1]].tolist(), co_w[co_off[i]:co_off[i + 1]].tolist()))
                       for i in range(n)],
                 children=[set(ch_kf[ch_off[i]:ch_off[i + 1]].tolist()) for i in range(n)])
        return o


def same(want, got, counts=True):
    """Asserts two results are equal: verdicts, every point's bad flag, nObs and observers, the local slots and the
    culled count; with counts, also nMPs and nRedundant (the reference does not report them)."""
    for k in OUT_KEYS if counts else ("verdict", "mp_bad", "mp_nobs", "obs_alive", "slot_mp"):
        assert np.array_equal(np.asarray(want[k]), np.asarray(got[k])), k
    assert want["n_culled"] == got["n_culled"]


class World:
    """n keyframes (table indices, ids ascending) with per-index slots, octaves, right coordinates (stereo flags) and
    depths; map points with bad flags, nObs and observations {keyframe: idx}; a spanning tree (parent) over the table,
    rooted at index 0 (mnId 0).  problem() flattens it for one local list."""

    def __init__(self, ids):
        self.ids = np.asarray(ids, np.uint64)
        n = len(ids)
        self.not_erase = np.zeros(n, np.uint8)
        self.th_depth = np.full(n, 5.0, np.float32)
        self.slots = [[] for _ in range(n)]
        self.octave = [[] for _ in range(n)]
        self.stereo = [[] for _ in range(n)]
        self.depth = [[] for _ in range(n)]
        self.parent = np.array([-1] + list(range(n - 1)), np.int32)
        self.bad, self.nobs, self.obs = [], [], []

    def add_point(self, bad=0):
        self.bad.append(bad)
        self.nobs.append(0)
        self.obs.append({})
        return len(self.obs) - 1

    def add_slot(self, k, mp, octave=0, stereo=False, depth=1.0, observe=True):
        """Appends a slot holding mp (-1: NULL) to keyframe k; with observe, mp's observation of k points at it."""
        self.slots[k].append(mp)
        self.octave[k].append(int(octave))
        self.stereo[k].append(bool(stereo))
        self.depth[k].append(float(depth))
        i = len(self.slots[k]) - 1
        if observe and mp >= 0:
            self.obs[mp][k] = i
        return i

    def count_nobs(self):
        """nObs as AddObservation leaves it: 2 per stereo observation, 1 per other."""
        self.nobs = [sum(2 if self.stereo[k][i] else 1 for k, i in o.items()) for o in self.obs]

    def problem(self, local, monocular=False):
        d = {"kf_id": self.ids, "not_erase": self.not_erase.copy(), "th_depth": self.th_depth.copy(),
             "mp_bad": np.array(self.bad, np.uint8), "mp_nobs": np.array(self.nobs, np.int32),
             "local_kf": np.array(local, np.int32), "monocular": monocular}
        rows = [sorted(o.items()) for o in self.obs]
        d["obs_off"] = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int32)
        d["obs_kf"] = np.array([k for r in rows for k, _ in r], np.int32)
        d["obs_idx"] = np.array([i for r in rows for _, i in r], np.int32)
        d["obs_octave"] = np.array([self.octave[k][i] for r in rows for k, i in r], np.int32)
        d["obs_stereo"] = np.array([self.stereo[k][i] for r in rows for k, i in r], np.uint8)
        d["slot_off"] = np.concatenate([[0], np.cumsum([len(self.slots[k]) for k in local])]).astype(np.int32)
        d["slot_mp"] = np.array([s for k in local for s in self.slots[k]], np.int32)
        d["slot_octave"] = np.array([s for k in local for s in self.octave[k]], np.int32)
        d["slot_depth"] = np.array([s for k in local for s in self.depth[k]], np.float32)
        return d

    def connections(self):
        """mConnectedKeyFrameWeights as UpdateConnections would build them: shared non-bad points per pair, as a CSR."""
        n = len(self.ids)
        r = [m for m, o in enumerate(self.obs) for _ in o if not self.bad[m]]
        c = [k for m, o in enumerate(self.obs) for k in o if not self.bad[m]]
        A = sp.csr_matrix((np.ones(len(r), np.int32), (r, c)), shape=(len(self.obs), n))
        W = (A.T @ A).tolil()
        W.setdiag(0)
        W = W.tocsr()
        W.eliminate_zeros()
        W.sort_indices()
        return W.indptr.astype(np.int32), W.indices.astype(np.int32), W.data.astype(np.int32)

    def covisible(self, k):
        """GetVectorCovisibleKeyFrames() of keyframe k: its connections by weight descending (index descending)."""
        off, kf, wt = self.connections()
        row = sorted(zip(wt[off[k]:off[k + 1]].tolist(), kf[off[k]:off[k + 1]].tolist()), reverse=True)
        return [j for _, j in row]


def _octave(rng, n):
    return rng.choice(8, n, p=[0.45, 0.25, 0.12, 0.07, 0.05, 0.03, 0.02, 0.01])


def trajectory(seed, n_kf, pts_per_kf=60, stereo=True, revisit=None):
    """A camera path over n_kf keyframes (index 0 is mnId 0): keyframe i creates pts_per_kf points, each seen by a run
    of 2-12 keyframes from i (with revisit = P, some also by keyframes around i + P).  Stereo slots have a right
    coordinate with probability 0.7 and depths around mThDepth; monocular ones have neither."""
    rng = np.random.default_rng(seed)
    w = World(np.arange(n_kf) * 3)
    w.th_depth[:] = rng.uniform(3, 8, n_kf)
    for i in range(n_kf):
        for _ in range(pts_per_kf):
            run = list(range(i, min(n_kf, i + int(rng.integers(2, 13)))))
            if revisit and i + revisit < n_kf and rng.random() < 0.3:
                run += list(range(i + revisit, min(n_kf, i + revisit + int(rng.integers(1, 4)))))
            m = w.add_point()
            for k in sorted(set(run)):
                st = stereo and rng.random() < 0.7
                z = float(rng.uniform(0.2, 1.3) * w.th_depth[k]) if stereo else -1.0
                w.add_slot(k, m, _octave(rng, 1)[0], st, z)
    for k in range(n_kf):  # NULL slots
        for _ in range(int(0.03 * len(w.slots[k]))):
            w.add_slot(k, -1, 0, False, -1.0)
    w.count_nobs()
    for m in np.nonzero(rng.random(len(w.obs)) < 0.02)[0]:
        w.bad[m] = 1
    return w


def random_world(seed, n_kf, slots_per_kf=80, stereo=True, odd=0.05):
    """Clustered points with 1-12 observers (mostly 4 or more) over n_kf keyframes (index 0 is mnId 0), with the inconsistencies Replace
    and Fuse leave at rate `odd`: duplicate slots, slots whose point does not list the keyframe, observations whose slot
    holds another point, bad points that keep their observers, and nObs off by one; plus depths exactly mThDepth,
    negative and NaN, and keyframes with mbNotErase."""
    rng = np.random.default_rng(seed)
    ids = np.concatenate([[0], np.sort(rng.choice(np.arange(1, 10 * n_kf), n_kf - 1, replace=False))])
    w = World(ids)
    w.th_depth[:] = rng.uniform(3, 8, n_kf)
    w.not_erase[rng.random(n_kf) < 0.15] = 1
    w.parent = np.array([-1] + [int(rng.integers(0, i)) for i in range(1, n_kf)], np.int32)
    for _ in range(n_kf * slots_per_kf // 5):
        c = int(rng.integers(0, n_kf))
        obs = set()
        for _ in range(int(rng.integers(4, 13)) if rng.random() < 0.85 else int(rng.integers(1, 4))):
            obs.add(int(np.clip(c + rng.integers(-6, 7), 0, n_kf - 1)) if rng.random() < 0.9 else int(rng.integers(0, n_kf)))
        m = w.add_point()
        for k in sorted(obs):
            z = float(rng.choice([w.th_depth[k], -0.5, np.nan, rng.uniform(0, 1.4) * w.th_depth[k]],
                                 p=[odd, odd, odd, 1 - 3 * odd])) if stereo else -1.0
            w.add_slot(k, m, _octave(rng, 1)[0], stereo and rng.random() < 0.7, z)
    w.count_nobs()
    n_mp = len(w.obs)
    for k in range(n_kf):
        for _ in range(int(odd * len(w.slots[k])) + int(rng.integers(0, 3))):
            kind = int(rng.integers(0, 4))
            if kind == 0:                                  # NULL slot
                w.add_slot(k, -1, 0, False, 1.0)
            elif kind == 1 and w.slots[k]:                 # the same point twice
                m = w.slots[k][int(rng.integers(0, len(w.slots[k])))]
                w.add_slot(k, m, _octave(rng, 1)[0], False, 1.0, observe=False)
            elif kind == 2:                                # a point that does not list k
                w.add_slot(k, int(rng.integers(0, n_mp)), _octave(rng, 1)[0], False, 1.0, observe=False)
            elif len(w.slots[k]) >= 2:                     # two slots swap points; the observations stay
                i, j = rng.choice(len(w.slots[k]), 2, replace=False)
                w.slots[k][i], w.slots[k][j] = w.slots[k][j], w.slots[k][i]
    for m in range(n_mp):
        u = rng.random()
        if u < 0.03:
            w.bad[m] = 1                                   # bad, observers kept
        elif u < 0.03 + odd:
            w.nobs[m] += int(rng.choice([-1, 1]))
    return w


def local_list(w, rng, cur, size=None):
    """A local list for current keyframe cur: its covisible keyframes in order, topped up with random others (mnId 0
    among them sometimes)."""
    n = len(w.ids)
    lst = w.covisible(cur)
    rest = [k for k in rng.permutation(n).tolist() if k != cur and k not in lst]
    size = min(n - 1, size if size is not None else len(lst) + int(rng.integers(0, 4)))
    lst = (lst + rest)[:size]
    return lst


def entry_verdicts(orc, d):
    """Each local keyframe's verdict from the entry state (as if it were the only one in the list)."""
    out = []
    for l, k in enumerate(d["local_kf"]):
        e = dict(d)
        e["local_kf"] = np.array([k], np.int32)
        a, b = d["slot_off"][l], d["slot_off"][l + 1]
        e["slot_off"] = np.array([0, b - a], np.int32)
        for f in ("slot_mp", "slot_octave", "slot_depth"):
            e[f] = np.asarray(d[f])[a:b]
        out.append(int(orc(e)["verdict"][0]))
    return out
