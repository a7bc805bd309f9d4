"""ctypes bindings of the keyframe-insertion checkers, beside pkg.ORBmatcher.ProcessNewKeyFrame / UpdateNormalAndDepth:

  Oracle()                  oracle/liborb_kfinsert.so, the CPU restatement (oracle/kfinsert.cpp)
  Reference()               oracle/_ref/libref_kfinsert.so, the reference's own ProcessNewKeyFrame + MapPointCulling and
                            UpdateNormalAndDepth on a fresh object graph
  Reference(adapter=True)   oracle/_ref/libadapter_kfinsert.so, the product's host/adapters/LocalMapping_b200.cc on the
                            same glue

and the seeded scenes the tests and tools/kfinsert_time.py use: scene() for one keyframe insertion, normal_depth_scene()
for a map of points."""
import ctypes
import importlib
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_LIB = os.path.join(ROOT, "oracle", "liborb_kfinsert.so")
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libref_kfinsert.so")
ADP_LIB = os.path.join(ROOT, "oracle", "_ref", "libadapter_kfinsert.so")
pkg = importlib.import_module("self_commit_orb-slam2_b200")
vp = ctypes.c_void_p
OUT_KEYS = ("mp_nobs", "mp_bad", "mp_added", "obs_alive", "mp_updated", "mp_normal", "mp_min_dist", "mp_max_dist",
            "mp_desc", "slot_mp", "list_mp", "list_verdict", "n_list", "n_culled")
CULLS = (pkg.KFI_CULLED_RATIO, pkg.KFI_CULLED_OBS)


class Oracle:
    def __init__(self):
        self.L = ctypes.CDLL(ORACLE_LIB)
        self.L.orc_process_new_keyframe.argtypes = [vp, vp]
        self.L.orc_update_normal_and_depth.argtypes = [vp, vp]

    def __call__(self, ds):
        one = isinstance(ds, dict)
        outs = []
        for d in ([ds] if one else ds):
            p, keep = pkg.kfinsert_problem(d)
            r, o = pkg.kfinsert_outputs(d)
            assert self.L.orc_process_new_keyframe(ctypes.byref(p), ctypes.byref(r)) == 0
            o["n_list"], o["n_culled"] = r.n_list, r.n_culled
            o["list_mp"], o["list_verdict"] = o["list_mp"][:r.n_list], o["list_verdict"][:r.n_list]
            outs.append(o)
        return outs[0] if one else outs

    def normal_and_depth(self, d):
        p, keep = pkg.normal_depth_problem(d)
        return _nd_call(self.L.orc_update_normal_and_depth, p)


def _nd_call(f, p):
    M = p.n_mp
    o = {"normal": np.zeros((M, 3), np.float32), "min_dist": np.zeros(M, np.float32),
         "max_dist": np.zeros(M, np.float32), "updated": np.zeros(M, np.uint8)}
    r = pkg._NormalDepthResult(*[o[k].ctypes.data_as(vp) for k in ("normal", "min_dist", "max_dist", "updated")])
    assert f(ctypes.byref(p), ctypes.byref(r)) == 0
    return o


class Reference:
    """The reference's ProcessNewKeyFrame (BoW and the map insertion stubbed) + MapPointCulling on the object graph of
    a scene: __call__(d) returns the state after the call (see ref_kfinsert_glue.cpp): mp_nobs, mp_bad, obs_alive,
    cur_idx, normal, min_dist, max_dist, desc (n_mp, 32), slot_mp, recent, erased, conn (one dict per keyframe) and
    wall_ns."""

    def __init__(self, adapter=False):
        self.L = ctypes.CDLL(ADP_LIB if adapter else REF_LIB)
        self.f = getattr(self.L, ("adp_" if adapter else "ref_") + "process_new_keyframe")
        self.f.argtypes = [vp] * 18 + [ctypes.c_int, vp]
        if not adapter:
            self.L.ref_update_normal_and_depth.argtypes = [vp, vp]

    def __call__(self, d):
        p, keep = pkg.kfinsert_problem(d)
        M, S, R, n = p.n_mp, p.n_slots, p.n_recent, p.n_kf
        cap = 4 * n * n + 16
        o = {"mp_nobs": np.zeros(M, np.int32), "mp_bad": np.zeros(M, np.uint8),
             "obs_alive": np.zeros(int(np.asarray(d["obs_off"])[-1]), np.uint8), "cur_idx": np.zeros(M, np.int32),
             "normal": np.zeros((M, 3), np.float32), "min_dist": np.zeros(M, np.float32),
             "max_dist": np.zeros(M, np.float32), "desc": np.zeros((M, 32), np.uint8), "slot_mp": np.zeros(S, np.int32),
             "recent": np.zeros(R + S, np.int32), "erased": np.zeros(M, np.int32)}
        desc_in = np.ascontiguousarray(d["mp_desc_in"], np.uint8)
        nr, ne = ctypes.c_int32(0), ctypes.c_int32(0)
        c_off, c_kf, c_w = np.zeros(n + 1, np.int32), np.zeros(cap, np.int32), np.zeros(cap, np.int32)
        wall = ctypes.c_double(0)
        P = lambda a: a.ctypes.data_as(vp)
        rc = self.f(ctypes.byref(p), P(desc_in), P(o["mp_nobs"]), P(o["mp_bad"]), P(o["obs_alive"]), P(o["cur_idx"]),
                    P(o["normal"]), P(o["min_dist"]), P(o["max_dist"]), P(o["desc"]), P(o["slot_mp"]), P(o["recent"]),
                    ctypes.byref(nr), P(o["erased"]), ctypes.byref(ne), P(c_off), P(c_kf), P(c_w), cap,
                    ctypes.byref(wall))
        assert rc == 0, rc
        o["recent"], o["erased"] = o["recent"][:nr.value].tolist(), o["erased"][:ne.value].tolist()
        o["conn"] = [dict(zip(c_kf[c_off[i]:c_off[i + 1]].tolist(), c_w[c_off[i]:c_off[i + 1]].tolist()))
                     for i in range(n)]
        o["wall_ns"] = wall.value
        return o

    def normal_and_depth(self, d):
        p, keep = pkg.normal_depth_problem(d)
        return _nd_call(self.L.ref_update_normal_and_depth, p)


def view(d, o):
    """A b2s_kfinsert_result dict (device or restatement) in the terms the reference glue reports."""
    off = np.asarray(d["obs_off"])
    obs_kf, obs_idx = np.asarray(d["obs_kf"]), np.asarray(d["obs_idx"])
    M = len(d["mp_bad"])
    cur_idx = np.full(M, -1, np.int32)
    desc = np.array(d["mp_desc_in"], np.uint8).copy()
    set_bad = (o["mp_bad"] != 0) & (np.asarray(d["mp_bad"]) == 0)
    for m in range(M):
        row = list(zip(obs_kf[off[m]:off[m + 1]].tolist(), range(off[m], off[m + 1])))
        hit = [o_ for k, o_ in row if k == d["cur"]]
        if hit:
            cur_idx[m] = obs_idx[hit[0]]
        elif o["mp_added"][m] >= 0:
            cur_idx[m] = o["mp_added"][m]
        if set_bad[m]:
            cur_idx[m] = -1
        j = o["mp_desc"][m]
        if j >= 0:  # position j of the row with the new observation at the current keyframe's table position
            merged = sorted(row + [(d["cur"], -1 - int(o["mp_added"][m]))])
            src = merged[j][1]
            desc[m] = d["obs_desc"][src] if src >= 0 else d["slot_desc"][-1 - src]
    lm, lv = np.asarray(o["list_mp"]), np.asarray(o["list_verdict"])
    return {"mp_nobs": o["mp_nobs"], "mp_bad": o["mp_bad"], "obs_alive": o["obs_alive"], "cur_idx": cur_idx,
            "normal": o["mp_normal"], "min_dist": o["mp_min_dist"], "max_dist": o["mp_max_dist"], "desc": desc,
            "slot_mp": o["slot_mp"], "recent": lm[lv == pkg.KFI_KEPT].tolist(),
            "erased": lm[np.isin(lv, CULLS)].tolist(), "updated": o["mp_updated"]}


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def same_as_reference(d, want, o):
    """The device's or the restatement's result o equals the reference glue's state want: integers, lists and
    descriptors identical, every float of a refreshed point bit-identical (others keep the reference's initial 0)."""
    v = view(d, o)
    for k in ("mp_nobs", "mp_bad", "obs_alive", "cur_idx", "desc", "slot_mp"):
        assert np.array_equal(np.asarray(v[k]), np.asarray(want[k])), k
    assert v["recent"] == want["recent"] and v["erased"] == want["erased"]
    u = v["updated"] != 0
    for k in ("normal", "min_dist", "max_dist"):
        assert np.array_equal(bits(v[k])[u], bits(want[k])[u]), k
        assert not np.asarray(want[k])[~u].any(), k


def same(a, b):
    """Two b2s_kfinsert_result dicts are identical (floats bit for bit)."""
    for k in OUT_KEYS:
        x, y = np.asarray(a[k]), np.asarray(b[k])
        if x.dtype == np.float32:
            x, y = bits(x), bits(y)
        assert np.array_equal(x, y), k


SF = (1.2 ** np.arange(8)).astype(np.float32)


def scene(seed, n_kf=40, n_slots=500, mono=False, max_obs=12, big_obs=0, p_listed=0.1, p_dup=0.03, p_bad=0.03,
          p_kf_bad=0.05, n_recent=None, cur_id=None):
    """One keyframe insertion.  Keyframes in table (= address) order with camera centres in a 10 m box; the current
    keyframe at a random position; points 20-40 m out, each seen by 1..max_obs other keyframes (big_obs of them by up
    to every keyframe), with descriptors scattered around a per-point base so that medians differ.  Slots: about 70 %
    hold a point; p_listed of those points already list the current keyframe (stereo points Tracking made); p_dup of
    the slots repeat an earlier point, p_bad hold bad points.  The recent list draws points with repeats.  mnFound /
    mnVisible include 0 visible and a ratio of exactly 1/4; mnFirstKFid spans cur_id - {0..4}, and cur_id may cross
    2^32 so that the (int) casts wrap."""
    rng = np.random.default_rng(seed)
    cur = int(rng.integers(n_kf))
    if cur_id is None:
        cur_id = int(rng.choice([n_kf + 7, 1 << 20, (1 << 32) + 1]))
    centers = rng.uniform(-5, 5, (n_kf, 3)).astype(np.float32)
    kf_bad = (rng.random(n_kf) < p_kf_bad).astype(np.uint8)
    n_mp = max(1, int(n_slots * 0.7))
    pos = np.empty((n_mp, 3), np.float32)
    dirs = rng.standard_normal((n_mp, 3))
    pos[:] = dirs / np.linalg.norm(dirs, axis=1, keepdims=True) * rng.uniform(20, 40, (n_mp, 1))
    slot_mp = np.full(n_slots, -1, np.int32)
    filled = rng.permutation(n_slots)[:n_mp]
    slot_mp[filled] = np.arange(n_mp)
    for s in np.where((slot_mp < 0) & (rng.random(n_slots) < p_dup / 0.3))[0]:
        slot_mp[s] = rng.integers(n_mp)  # a repeated point
    first_slot = {}
    for s, m in enumerate(slot_mp.tolist()):
        if m >= 0:
            first_slot.setdefault(m, s)
    slot_stereo = (np.zeros(n_slots) if mono else rng.random(n_slots) < 0.6).astype(np.uint8)
    slot_desc = rng.integers(0, 256, (n_slots, 32), dtype=np.uint8)
    base = rng.integers(0, 256, (n_mp, 32), dtype=np.uint8)
    others = np.array([k for k in range(n_kf) if k != cur])
    next_idx = np.zeros(n_kf, np.int64)
    next_idx[cur] = n_slots
    obs_off, obs_kf, obs_idx, obs_oct, obs_desc, ref = [0], [], [], [], [], []
    big = set(rng.choice(n_mp, min(big_obs, n_mp), replace=False).tolist())
    for m in range(n_mp):
        k_n = len(others) if m in big else int(rng.integers(1, max_obs + 1))
        row = sorted(rng.choice(others, min(k_n, len(others)), replace=False).tolist())
        if m in first_slot and rng.random() < p_listed:
            row = sorted(row + [cur])
        ref.append(int(rng.choice([k for k in row if k != cur])))
        for k in row:
            obs_kf.append(k)
            if k == cur:
                obs_idx.append(first_slot[m])
                obs_desc.append(slot_desc[first_slot[m]])
            else:
                obs_idx.append(int(next_idx[k]))
                next_idx[k] += 1
                d = base[m].copy()
                flip = rng.integers(0, 256, 32, dtype=np.uint8) & rng.integers(0, 256, 32, dtype=np.uint8) & \
                    rng.integers(0, 256, 32, dtype=np.uint8)
                obs_desc.append(d ^ flip)
            obs_oct.append(int(rng.integers(8)))
        obs_off.append(len(obs_kf))
    for s, m in enumerate(slot_mp.tolist()):  # the current keyframe's descriptors near the points' too
        if m >= 0 and rng.random() < 0.8:
            slot_desc[s] = base[m] ^ (rng.integers(0, 256, 32, dtype=np.uint8) & rng.integers(0, 256, 32, dtype=np.uint8)
                                      & rng.integers(0, 256, 32, dtype=np.uint8))
    for o, k in enumerate(obs_kf):  # an observation of cur carries the slot's descriptor
        if k == cur:
            obs_desc[o] = slot_desc[obs_idx[o]]
    visible = rng.integers(0, 9, n_mp).astype(np.int32)
    found = (rng.random(n_mp) * (visible + 1)).astype(np.int32)
    q = rng.random(n_mp)
    visible[q < 0.05], found[q < 0.05] = 0, rng.integers(0, 3, int((q < 0.05).sum()))
    visible[(q >= 0.05) & (q < 0.1)], found[(q >= 0.05) & (q < 0.1)] = 4, 1  # exactly 1/4
    first = (cur_id - rng.integers(0, 5, n_mp)).astype(np.int64)
    n_recent = n_mp // 3 if n_recent is None else n_recent
    recent = rng.integers(0, n_mp, n_recent).astype(np.int32)
    return {"kf_center": centers, "kf_bad": kf_bad, "cur": cur, "cur_id": cur_id, "slot_mp": slot_mp,
            "slot_stereo": slot_stereo, "slot_desc": slot_desc, "mp_pos": pos,
            "mp_bad": (rng.random(n_mp) < p_bad).astype(np.uint8), "mp_ref": np.array(ref, np.int32),
            "mp_nobs": rng.integers(1, 7, n_mp).astype(np.int32), "mp_found": found, "mp_visible": visible,
            "mp_first_kf": first, "obs_off": np.array(obs_off, np.int32), "obs_kf": np.array(obs_kf, np.int32),
            "obs_idx": np.array(obs_idx, np.int32), "obs_octave": np.array(obs_oct, np.int32),
            "obs_desc": np.array(obs_desc, np.uint8).reshape(-1, 32), "recent": recent, "scale_factors": SF,
            "monocular": mono, "mp_desc_in": rng.integers(0, 256, (n_mp, 32), dtype=np.uint8)}


def normal_depth_scene(seed, n_mp=10000, n_kf=200, max_obs=8, p_bad=0.02):
    """A map for the standalone UpdateNormalAndDepth: n_kf camera centres, n_mp points with 0..max_obs observers (an
    empty row and bad points are left unchanged), the reference keyframe one of the observers."""
    rng = np.random.default_rng(seed)
    counts = rng.integers(1, max_obs + 1, n_mp)
    counts[rng.random(n_mp) < 0.02] = 0
    obs_off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    obs_kf = np.concatenate([np.sort(rng.choice(n_kf, c, replace=False)) for c in counts] + [np.zeros(0)]).astype(
        np.int32)
    ref = np.array([obs_kf[obs_off[m] + rng.integers(counts[m])] if counts[m] else -1 for m in range(n_mp)], np.int32)
    dirs = rng.standard_normal((n_mp, 3))
    pos = (dirs / np.linalg.norm(dirs, axis=1, keepdims=True) * rng.uniform(15, 60, (n_mp, 1))).astype(np.float32)
    return {"kf_center": rng.uniform(-10, 10, (n_kf, 3)).astype(np.float32), "mp_pos": pos,
            "mp_bad": (rng.random(n_mp) < p_bad).astype(np.uint8), "mp_ref": ref, "obs_off": obs_off,
            "obs_kf": obs_kf, "obs_octave": rng.integers(0, 8, int(obs_off[-1])).astype(np.int32),
            "scale_factors": SF}
