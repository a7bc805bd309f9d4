"""Times b2s_update_connections (pkg.Covisibility) against the reference's own KeyFrame::UpdateConnections
(oracle/_ref/libref_keyframe.so) called one keyframe at a time on one CPU thread of the same machine.

Maps of 500, 2,000 and 8,000 keyframes, about 2,000 slots per keyframe, 2-10 observers per point (consecutive keyframes
around a centre), entry connection maps of the 40 nearest keyframes.  Batches of 1 (LocalMapping::ProcessNewKeyFrame)
and 64 (a loop correction).  Each problem holds what the adapter gathers: the members, the observers of their points and
the keyframes their maps name.  Reported: device time (CUDA events: upload, kernels, download) and host wall time of the
library call (validation, packing, device work, unpacking), medians of 20 after warm-up; the reference's time is the median wall time of its calls alone.  The device result
is checked against the reference's before timing.

  python tools/covis_time.py [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import covis_binding as cb  # noqa: E402


def make_map(rng, n_kf, slots=2000):
    n_pts = n_kf * slots // 6
    k = rng.integers(2, 11, n_pts)
    c = (rng.random(n_pts) * (n_kf - k + 1)).astype(np.int64)
    obs_off = np.concatenate([[0], np.cumsum(k)])
    obs = np.repeat(c, k) + (np.arange(obs_off[-1]) - np.repeat(obs_off[:-1], k))
    pt = np.repeat(np.arange(n_pts), k)
    order = np.argsort(obs, kind="stable")
    kf_slot_off = np.concatenate([[0], np.cumsum(np.bincount(obs, minlength=n_kf))])
    return {"n_kf": n_kf, "obs_off": obs_off, "obs": obs, "slot_pt": pt[order], "slot_off": kf_slot_off,
            "bad": rng.random(n_pts) < 0.03}


def problem(m, members, rng):
    """The table the adapter would gather for `members` (renumbered, ascending id)."""
    n = m["n_kf"]
    pts = np.unique(np.concatenate([m["slot_pt"][m["slot_off"][k]:m["slot_off"][k + 1]] for k in members]))
    obs_kf = np.concatenate([m["obs"][m["obs_off"][p]:m["obs_off"][p + 1]] for p in pts])
    core = np.unique(np.concatenate([obs_kf, members]))
    ring = np.unique(np.clip(core[:, None] + np.arange(-20, 21)[None, :], 0, n - 1))
    table = np.unique(np.concatenate([core, ring]))
    idx = -np.ones(n, np.int64)
    idx[table] = np.arange(len(table))
    incore = np.zeros(n, bool)
    incore[core] = True
    map_kf, map_w, list_kf, list_w, map_off, list_off = [], [], [], [], [0], [0]
    for t in table:
        if incore[t]:
            nb = np.array([j for j in range(max(0, t - 20), min(n, t + 21)) if j != t])
            w = rng.integers(1, 60, len(nb))
            map_kf += idx[nb].tolist()
            map_w += w.tolist()
            o = sorted(zip(w.tolist(), idx[nb].tolist()), reverse=True)
            list_kf += [b for a, b in o if a >= 15]
            list_w += [a for a, b in o if a >= 15]
        map_off.append(len(map_kf))
        list_off.append(len(list_kf))
    pidx = {int(p): i for i, p in enumerate(pts)}
    obs_off = np.concatenate([[0], np.cumsum([m["obs_off"][p + 1] - m["obs_off"][p] for p in pts])])
    slot_mp, slot_off = [], [0]
    for k in members:
        s = m["slot_pt"][m["slot_off"][k]:m["slot_off"][k + 1]]
        slot_mp += [pidx[int(p)] for p in s]
        slot_off.append(len(slot_mp))
    return {"kf_id": table.astype(np.uint64) + 1, "map_off": map_off, "map_kf": map_kf, "map_w": map_w,
            "list_off": list_off, "list_kf": list_kf, "list_w": list_w,
            "first_connection": np.zeros(len(table), np.uint8), "parent": np.full(len(table), -1, np.int32),
            "mp_bad": m["bad"][pts].astype(np.uint8), "obs_off": obs_off, "obs_kf": idx[obs_kf],
            "member": idx[np.asarray(members)], "slot_off": slot_off, "slot_mp": slot_mp}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    import importlib
    pkg = importlib.import_module("self_commit_orb-slam2_b200")
    if pkg.device_count() < 1:
        raise SystemExit("covis_time: no CUDA device")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    ref = cb.Reference()
    dev = pkg.Covisibility(max_kf=8192, max_mp=1 << 19, max_obs=1 << 22, max_slots=1 << 18, max_conn=1 << 22,
                           max_batch=64)
    rng = np.random.default_rng(0)
    rows = []
    for n_kf in (500, 2000, 8000):
        m = make_map(rng, n_kf)
        for B in (1, 64):
            members = [int(x) for x in rng.choice(np.arange(20, n_kf - 20), B, replace=False)]
            d = problem(m, members, rng)
            want = ref.UpdateConnections(d)
            cb.same(want, dev.UpdateConnections(d), len(d["kf_id"]))
            need = max(dev.raw(d)[1]["need"])
            dev_ms, wall_ms, ref_ms = [], [], []
            for rep in range(a.reps + 3):
                wall = []

                def call(p, r):  # the host wall time of the library call alone
                    t0 = time.perf_counter()
                    rc = pkg.lib().b2s_update_connections(dev._h, p, r)
                    wall.append(time.perf_counter() - t0)
                    return rc
                rc, _ = pkg.covis_call(call, d, need)
                assert rc == 0
                r = ref.UpdateConnections(d)["wall_ns"] * 1e-6
                if rep >= 3:
                    dev_ms.append(dev.last_ms())
                    wall_ms.append(wall[0] * 1e3)
                    ref_ms.append(r)
            row = {"n_kf": n_kf, "batch": B, "table_kf": len(d["kf_id"]), "points": len(d["mp_bad"]),
                   "slots": len(d["slot_mp"]), "device_ms": float(np.median(dev_ms)),
                   "host_wall_ms": float(np.median(wall_ms)), "reference_cpu_ms": float(np.median(ref_ms))}
            rows.append(row)
            print(json.dumps(row), flush=True)
    res = {"gpu": smi, "rows": rows}
    print("card, power limit:", smi)
    print("| keyframes | batch | table kfs | slots | device ms | host wall ms | reference 1 thread ms |")
    for r in rows:
        print("| %d | %d | %d | %d | %.3f | %.3f | %.3f |" % (r["n_kf"], r["batch"], r["table_kf"], r["slots"],
                                                          r["device_ms"], r["host_wall_ms"], r["reference_cpu_ms"]))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
