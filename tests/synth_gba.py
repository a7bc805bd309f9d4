"""Synthetic whole maps for the global bundle adjustment (Optimizer::GlobalBundleAdjustemnt) tests, in the style of
tests/synth.py: float32 values as Converter hands them over."""
import numpy as np


def synth_global_ba(n_kf=60, n_mp=3000, obs_range=(2, 10), seed=11, mono_frac=0.0, outlier_frac=0.0, loop=True,
                    n_bad_kf=0, n_bad_mp=0, n_excluded_mp=0, edgeless_kf=False, pert_deg=0.2, pert_t=0.02, pert_p=0.05):
    """A whole map for Optimizer::GlobalBundleAdjustemnt (src/Optimizer.cc:55-341), as the object graph holds it.

    loop=True: keyframes on a closed circle (radius 20 m) looking outwards, so the last keyframes re-observe the first
    keyframes' points and the reduced camera system is not a band; loop=False: a straight forward path (1 m spacing,
    monocular initialisation).  Each point is seen by randint(obs_range) keyframes nearest (along the trajectory) to an
    anchor keyframe in whose frustum it was placed; keyframe k has mnId k, point m has mnId m.  Optional: gross outliers
    (+30 px), n_bad_kf bad keyframes (their observations stay in the map), n_bad_mp bad points, n_excluded_mp points
    whose only observers are bad keyframes, and one keyframe whose observations are all removed (edgeless_kf).
    float32 values as Converter hands them over.  obs: ba_edge-style records grouped by point (ascending), keyframes
    ascending inside a point."""
    rng = np.random.RandomState(seed)
    fx = fy = 718.856
    cx, cy, bf = 607.1928, 185.2157, 386.1448
    W, H = 1241, 376
    R = np.zeros((n_kf, 3, 3))
    center = np.zeros((n_kf, 3))
    for k in range(n_kf):
        if loop:
            th = 2 * np.pi * k / n_kf
            zc = np.array([np.sin(th), 0.0, np.cos(th)])        # optical axis: outwards
            xc = np.array([np.cos(th), 0.0, -np.sin(th)])
            center[k] = 20.0 * zc + rng.normal(0, 0.05, 3)
        else:
            yaw = np.deg2rad(rng.uniform(-2, 2))
            zc = np.array([np.sin(yaw), 0.0, np.cos(yaw)])
            xc = np.array([np.cos(yaw), 0.0, -np.sin(yaw)])
            center[k] = np.array([rng.uniform(-0.1, 0.1), rng.uniform(-0.05, 0.05), 1.0 * k])
        R[k] = np.stack([xc, np.array([0.0, 1.0, 0.0]), zc])   # rows: camera axes in world coordinates (R_cw)
    t = -np.einsum("kij,kj->ki", R, center)
    lo, hi = obs_range
    want = rng.randint(lo, hi + 1, n_mp)
    pts = np.zeros((n_mp, 3))
    chosen = [None] * n_mp
    todo = np.arange(n_mp)
    kidx = np.arange(n_kf)
    for _ in range(60):
        if len(todo) == 0:
            break
        for c0 in range(0, len(todo), 2000):
            part = todo[c0:c0 + 2000]
            m = len(part)
            ka = rng.randint(0, n_kf, m)
            z = rng.uniform(5, 40, m)
            u = rng.uniform(50, W - 50, m)
            v = rng.uniform(30, H - 30, m)
            Xc = np.stack([(u - cx) * z / fx, (v - cy) * z / fy, z], 1)
            Xw = np.einsum("mji,mj->mi", R[ka], Xc - t[ka])
            Xk = np.einsum("kij,mj->mki", R, Xw) + t[None]
            zz = Xk[..., 2]
            uu = fx * Xk[..., 0] / np.where(zz > 0, zz, 1) + cx
            vv = fy * Xk[..., 1] / np.where(zz > 0, zz, 1) + cy
            vis = (zz >= 2.0) & (uu > 0) & (uu < W) & (vv > 0) & (vv < H)
            dk = np.abs(kidx[None] - ka[:, None])
            if loop:
                dk = np.minimum(dk, n_kf - dk)
            dist = np.where(vis, dk, 10 ** 6)
            order = np.argsort(dist, 1, kind="stable")
            for i in range(m):
                n_want = min(want[part[i]], n_kf)
                if vis[i].sum() >= n_want:
                    pts[part[i]] = Xw[i]
                    chosen[part[i]] = np.sort(order[i, :n_want])
        todo = np.array([i for i in todo if chosen[i] is None], np.int64)
    keep = np.array([c is not None for c in chosen])
    pts = pts[keep]
    chosen = [c for c in chosen if c is not None]
    n_mp = len(pts)
    kf = np.concatenate(chosen).astype(np.int64)
    mp = np.repeat(np.arange(n_mp), [len(c) for c in chosen])
    Xk = np.einsum("eij,ej->ei", R[kf], pts[mp]) + t[kf]
    uu = fx * Xk[:, 0] / Xk[:, 2] + cx
    vv = fy * Xk[:, 1] / Xk[:, 2] + cy
    ur = uu - bf / Xk[:, 2]
    ne = len(kf)
    octv = rng.randint(0, 8, ne)
    sig = 1.2 ** octv
    noise = rng.normal(0, 1, (ne, 3)) * sig[:, None]
    noise[:, 0] += np.where(rng.uniform(size=ne) < outlier_frac, 30.0, 0.0)
    mono = rng.uniform(size=ne) < mono_frac
    edge_dt = np.dtype([("kf", "i4"), ("mp", "i4"), ("obs", "f4", 3), ("inv_sigma2", "f4")])
    E = np.zeros(ne, edge_dt)
    E["kf"] = kf
    E["mp"] = mp
    E["obs"][:, 0] = (uu + noise[:, 0]).astype(np.float32)
    E["obs"][:, 1] = (vv + noise[:, 1]).astype(np.float32)
    E["obs"][:, 2] = np.where(mono, -1.0, ur + noise[:, 2]).astype(np.float32)
    E["inv_sigma2"] = (1.0 / (1.2 ** (2 * octv))).astype(np.float32)
    kf_bad = np.zeros(n_kf, np.uint8)
    if n_bad_kf:
        kf_bad[1 + rng.choice(n_kf - 1, n_bad_kf, replace=False)] = 1
    bad_ids = np.where(kf_bad)[0]
    if n_excluded_mp and len(bad_ids):
        # points whose only observers are bad keyframes: every observation is moved to bad keyframes
        for m in rng.choice(n_mp, n_excluded_mp, replace=False):
            sel = np.where(E["mp"] == m)[0]
            ks = np.sort(rng.choice(bad_ids, min(len(sel), len(bad_ids)), replace=False))
            E["kf"][sel[:len(ks)]] = ks
            E["mp"][sel[len(ks):]] = -1
        E = E[E["mp"] >= 0]
    if edgeless_kf:
        cand = [k for k in range(1, n_kf) if not kf_bad[k]]
        k0 = cand[len(cand) // 2]
        drop = E["kf"] == k0
        # a point must keep one observation
        cnt = np.bincount(E["mp"][~drop], minlength=n_mp)
        lonely = np.where(drop & (cnt[E["mp"]] == 0))[0]
        if len(lonely):
            alt = (k0 + 1) % n_kf
            E["kf"][lonely] = alt
            drop[lonely] = False
            E = E[~drop]
            # (k0 + 1 may already observe such a point: keep the first of each (keyframe, point) pair)
            _, first = np.unique(E["mp"].astype(np.int64) * n_kf + E["kf"], return_index=True)
            E = E[np.sort(first)]
        else:
            E = E[~drop]
    E = E[np.lexsort((E["kf"], E["mp"]))]
    mp_bad = np.zeros(n_mp, np.uint8)
    if n_bad_mp:
        mp_bad[rng.choice(n_mp, n_bad_mp, replace=False)] = 1
    Tcw0 = np.zeros((n_kf, 4, 4))
    Tcw0[:, :3, :3] = R
    Tcw0[:, :3, 3] = t
    Tcw0[:, 3, 3] = 1
    for k in range(1, n_kf):
        a = np.deg2rad(rng.normal(0, pert_deg, 3))
        Rx = np.array([[1, 0, 0], [0, np.cos(a[0]), -np.sin(a[0])], [0, np.sin(a[0]), np.cos(a[0])]])
        Ry = np.array([[np.cos(a[1]), 0, np.sin(a[1])], [0, 1, 0], [-np.sin(a[1]), 0, np.cos(a[1])]])
        dR = Rx @ Ry
        Tcw0[k, :3, :3] = dR @ R[k]
        Tcw0[k, :3, 3] = dR @ t[k] + rng.normal(0, pert_t, 3)
    pts0 = pts + rng.normal(0, pert_p, pts.shape)
    return dict(Tcw=Tcw0.astype(np.float32).reshape(n_kf, 16), kf_bad=kf_bad, points=pts0.astype(np.float32),
                mp_bad=mp_bad, obs=E, fx=np.float32(fx), fy=np.float32(fy), cx=np.float32(cx), cy=np.float32(cy),
                bf=np.float32(bf))
