"""Seeded maps that look like what LoopClosing::CorrectLoop hands to Optimizer::OptimizeEssentialGraph (test data).

A drifting trajectory (with scale drift when monocular) around a loop, a spanning tree whose parent is usually k-1 and
sometimes k-2, covisibility weights on both sides of minFeat = 100, loop edges of earlier closures, the current keyframe's
connected set with CorrectedSim3 / NonCorrectedSim3 (their keyframes already moved to the corrected pose), LoopConnections
that include the current / loop pair below minFeat and one that duplicates a spanning-tree edge, bad keyframes only as
covisible neighbours, bad points, and points with mnCorrectedByKF == the current keyframe."""
import numpy as np


def _rot(axis, ang):
    a = np.asarray(axis, np.float64)
    a = a / np.linalg.norm(a)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * K @ K


def _quat(R):
    """Unit quaternion (x, y, z, w) of a rotation matrix (a test value; the products below are what matters)."""
    w = np.sqrt(max(0.0, 1 + R[0, 0] + R[1, 1] + R[2, 2])) / 2
    x = np.copysign(np.sqrt(max(0.0, 1 + R[0, 0] - R[1, 1] - R[2, 2])) / 2, R[2, 1] - R[1, 2])
    y = np.copysign(np.sqrt(max(0.0, 1 - R[0, 0] + R[1, 1] - R[2, 2])) / 2, R[0, 2] - R[2, 0])
    z = np.copysign(np.sqrt(max(0.0, 1 - R[0, 0] - R[1, 1] + R[2, 2])) / 2, R[1, 0] - R[0, 1])
    q = np.array([x, y, z, w])
    return q / np.linalg.norm(q)


def synth_essential(n_kf=60, n_mp=500, seed=0, mono=False, closures=1, n_bad_kf=2, n_bad_mp=5, drift=0.01,
                    scale_drift=0.004, n_connected=6):
    rng = np.random.RandomState(seed)
    n = n_kf
    # ground truth on a circle, the estimate drifts (rotation, translation, and scale when monocular)
    Rw, tw = [], []
    for k in range(n):
        ang = 2 * np.pi * k / max(n, 2) * 0.95
        Rw.append(_rot([0, 1, 0], ang))
        tw.append(np.array([5 * np.sin(ang), 0.1 * np.sin(3 * ang), 5 * np.cos(ang)]))
    Rd, td, sd = [Rw[0]], [tw[0]], [1.0]
    for k in range(1, n):
        dR = Rw[k - 1].T @ Rw[k]
        dt = Rw[k - 1].T @ (tw[k] - tw[k - 1])
        dR = dR @ _rot(rng.randn(3), drift * rng.uniform(0.2, 1.0))
        dt = dt + drift * rng.randn(3)
        s = sd[-1] * (1 + (scale_drift * rng.uniform(0.5, 1.5) if mono else 0.0))
        Rd.append(Rd[-1] @ dR)
        td.append(td[-1] + Rd[-2] @ dt * (s / sd[-1]) if mono else td[-1] + Rd[-2] @ dt)
        sd.append(s)
    Tcw = np.zeros((n, 16), np.float32)
    for k in range(n):
        T = np.eye(4)
        T[:3, :3] = Rd[k].T
        T[:3, 3] = -Rd[k].T @ td[k]
        Tcw[k] = T.reshape(-1).astype(np.float32)
    kf_bad = np.zeros(n, np.uint8)
    cur, loop = n - 1, min(int(rng.randint(0, 3)), n - 1)
    cands = np.arange(4, n - n_connected - 2)
    bad = rng.choice(cands, size=min(n_bad_kf, len(cands)), replace=False) if len(cands) and n_bad_kf else []
    kf_bad[np.asarray(bad, np.int64)] = 1
    good = [k for k in range(n) if not kf_bad[k]]
    parent = np.full(n, -1, np.int32)
    prev = [k for k in good]
    for a, k in enumerate(prev[1:], 1):
        parent[k] = prev[a - 2] if a >= 2 and rng.uniform() < 0.2 else prev[a - 1]
    # covisibility: neighbours up to 4 keyframes apart, weights on both sides of 100
    W = {}
    for k in range(n):
        for d in range(1, 5):
            j = k + d
            if j < n:
                W[(k, j)] = W[(j, k)] = int(rng.randint(30, 260) if d > 1 else rng.randint(90, 300))
    loops = []
    for c in range(closures - 1):  # earlier closures: loop edges both ways
        a, b = int(rng.randint(n // 3, n // 2)), int(rng.randint(0, n // 6))
        if kf_bad[a] or kf_bad[b] or a == b:
            continue
        loops += [(a, b), (b, a)]
        W[(a, b)] = W[(b, a)] = int(rng.randint(100, 200))
    # the current keyframe's connected set, corrected by the loop's Sim3
    connected = [k for k in range(n - n_connected, n) if not kf_bad[k]]
    corr_kf, corr_S, noncorr_S = [], [], []
    s_corr = 1.0 / sd[cur] if mono else 1.0
    for k in connected:
        Rcw_d, tcw_d = Tcw[k].reshape(4, 4)[:3, :3].astype(np.float64), Tcw[k].reshape(4, 4)[:3, 3].astype(np.float64)
        Rcw_t = Rw[k].T
        tcw_t = -Rw[k].T @ tw[k] + 0.002 * rng.randn(3)
        corr_kf.append(k)
        corr_S.append(np.concatenate([_quat(Rcw_t), s_corr * tcw_t, [s_corr]]))
        noncorr_S.append(np.concatenate([_quat(Rcw_d), tcw_d, [1.0]]))
        T = np.eye(4)
        T[:3, :3] = Rcw_t
        T[:3, 3] = tcw_t
        Tcw[k] = T.reshape(-1).astype(np.float32)
    # LoopConnections: around the loop keyframe; the current / loop pair below minFeat; one duplicating a tree edge
    conn = []
    near_loop = [j for j in range(0, min(n, loop + 5)) if not kf_bad[j] and j not in connected]
    for k in connected:
        for j in near_loop:
            if rng.uniform() < 0.5 or (k == cur and j == loop):
                conn.append((k, j))
                if (k, j) not in W:
                    W[(k, j)] = W[(j, k)] = int(40 if (k == cur and j == loop) else rng.randint(60, 200))
    k0 = connected[len(connected) // 2]
    if parent[k0] >= 0 and parent[k0] not in near_loop:
        conn.append((k0, int(parent[k0])))
        W[(k0, int(parent[k0]))] = W[(int(parent[k0]), k0)] = 150
    if cur != loop:
        if (cur, loop) not in conn:
            conn.append((cur, loop))
        W[(cur, loop)] = W[(loop, cur)] = 40
    adj = {}
    for (a, j), w in W.items():
        adj.setdefault(a, []).append((w, j))
    cov = []
    for k in range(n):
        cov += [(k, j, w) for w, j in sorted(adj.get(k, []), key=lambda x: (-x[0], x[1]))]
    # points
    P = np.zeros((n_mp, 3), np.float32)
    ref = np.zeros(n_mp, np.int32)
    for m in range(n_mp):
        k = int(rng.randint(0, n))
        ref[m] = k
        P[m] = (td[k] + Rd[k] @ np.array([rng.uniform(-2, 2), rng.uniform(-1, 1), rng.uniform(2, 8)])).astype(np.float32)
    mp_bad = np.zeros(n_mp, np.uint8)
    if n_bad_mp and n_mp:
        mp_bad[rng.choice(n_mp, size=min(n_bad_mp, n_mp), replace=False)] = 1
    corrected_by = np.zeros(n_mp, np.int32)
    corrected_ref = np.zeros(n_mp, np.int32)
    for m in range(n_mp):
        if rng.uniform() < 0.1:
            corrected_by[m] = cur
            corrected_ref[m] = connected[int(rng.randint(0, len(connected)))]
    return dict(Tcw=Tcw, kf_bad=kf_bad, parent=parent, loop_edges=np.array(loops, np.int32).reshape(-1, 2),
                cov=np.array(cov, np.int32).reshape(-1, 3), loop_kf=loop, cur_kf=cur,
                corr_kf=np.array(corr_kf, np.int32), corr_S=np.array(corr_S, np.float64).reshape(-1, 8),
                noncorr_S=np.array(noncorr_S, np.float64).reshape(-1, 8), conn=np.array(conn, np.int32).reshape(-1, 2),
                points=P, mp_bad=mp_bad, mp_ref=ref, mp_corrected_by=corrected_by, mp_corrected_ref=corrected_ref,
                fix_scale=not mono)
