"""Two-view scenes for the monocular initialiser: a 640 x 480 pinhole K, keypoints with sub-pixel noise, unmatched
keypoints in both frames, a share of wrong matches, and the minimal sets drawn as Initializer::Initialize draws them
(without replacement within a set; the C rand() stream itself is the caller's business)."""
import numpy as np

K = np.array([[520.0, 0, 320.0], [0, 520.0, 240.0], [0, 0, 1]], np.float32)


def _rot(axis, ang):
    axis = np.asarray(axis, np.float64)
    axis = axis / np.linalg.norm(axis)
    x, y, z = axis
    S = np.array([[0, -z, y], [z, 0, -x], [-y, x, 0]])
    return np.eye(3) + np.sin(ang) * S + (1 - np.cos(ang)) * S @ S


def _project(X):
    x = (K.astype(np.float64) @ X.T).T
    return x[:, :2] / x[:, 2:3]


def synth_init(n, seed, kind="general", outliers=0.2, extra=0.3, iterations=200, noise=0.5, sigma=1.0):
    """kind: 'planar' (a plane, H should win), 'general' (3-D points, F should win), 'rotation' (a pure rotation: fails on
    parallax), 'ambiguous' (a short baseline along the optical axis over a shallow scene)."""
    rng = np.random.default_rng(seed)
    R = _rot(rng.normal(size=3), np.deg2rad(rng.uniform(2, 6)))
    t = np.array([rng.uniform(-1, 1), rng.uniform(-0.2, 0.2), rng.uniform(-0.1, 0.1)])
    t = t / np.linalg.norm(t) * rng.uniform(0.4, 0.8)
    if kind == "rotation":
        t = np.zeros(3)
    if kind == "ambiguous":
        t = np.array([0.0, 0.0, 0.05])
    pts, m = [], 0
    while m < n:
        u = rng.uniform(20, 620, 4 * n)
        v = rng.uniform(20, 460, 4 * n)
        if kind == "planar":
            d = 5.0 + 0.3 * (u - 320) / 320
        elif kind == "ambiguous":
            d = rng.uniform(20, 21, 4 * n)
        else:
            d = rng.uniform(3, 9, 4 * n)
        X = np.stack([(u - 320) / 520 * d, (v - 240) / 520 * d, d], 1)
        X2 = X @ R.T + t
        ok = X2[:, 2] > 0.5
        p2 = _project(X2[ok])
        ok2 = (p2[:, 0] > 0) & (p2[:, 0] < 640) & (p2[:, 1] > 0) & (p2[:, 1] < 480)
        pts.append(np.concatenate([np.stack([u[ok][ok2], v[ok][ok2]], 1), p2[ok2]], 1))
        m += int(ok2.sum())
    P = np.concatenate(pts)[:n]
    P[:, :2] += rng.normal(scale=noise, size=(n, 2))
    P[:, 2:] += rng.normal(scale=noise, size=(n, 2))
    n_out = int(round(outliers * n))
    bad = rng.choice(n, n_out, replace=False) if n_out else np.zeros(0, int)
    P[bad, 2] = rng.uniform(0, 640, n_out)
    P[bad, 3] = rng.uniform(0, 480, n_out)
    # unmatched keypoints in both frames, all shuffled
    e1, e2 = int(extra * n) + 1, int(extra * n) + 2
    kp1 = np.concatenate([P[:, :2], np.stack([rng.uniform(0, 640, e1), rng.uniform(0, 480, e1)], 1)])
    kp2 = np.concatenate([P[:, 2:], np.stack([rng.uniform(0, 640, e2), rng.uniform(0, 480, e2)], 1)])
    o1, o2 = rng.permutation(len(kp1)), rng.permutation(len(kp2))
    inv2 = np.argsort(o2)
    kp1, kp2 = kp1[o1], kp2[o2]
    matches12 = np.full(len(kp1), -1, np.int32)
    for new1, old1 in enumerate(o1):
        if old1 < n:
            matches12[new1] = inv2[old1]
    sets = np.stack([rng.choice(n, 8, replace=False) for _ in range(iterations)]).astype(np.int32)
    return dict(kp1=kp1.astype(np.float32), kp2=kp2.astype(np.float32), matches12=matches12, K=K, sigma=sigma,
                sets=sets, R=R, t=t)


# (n, seed, kind, outliers, iterations): the seeds kept are those whose decisions are clear of every threshold
CASES = {
    "planar_150": dict(n=150, seed=1, kind="planar", outliers=0.1),
    "planar_500": dict(n=500, seed=28, kind="planar", outliers=0.1, noise=0.3),
    "planar_500_b": dict(n=500, seed=35, kind="planar", outliers=0.1, noise=0.3),
    "planar_600": dict(n=600, seed=2, kind="planar", outliers=0.3),
    "planar_1500": dict(n=1500, seed=3, kind="planar", outliers=0.45),
    "general_150": dict(n=150, seed=4, kind="general", outliers=0.1),
    "general_600": dict(n=600, seed=5, kind="general", outliers=0.2),
    "general_1500": dict(n=1500, seed=6, kind="general", outliers=0.3),
    "general_3000": dict(n=3000, seed=7, kind="general", outliers=0.0, iterations=300),
    "rotation_400": dict(n=400, seed=8, kind="rotation", outliers=0.1),
    "ambiguous_400": dict(n=400, seed=9, kind="ambiguous", outliers=0.05, iterations=50),
    "general_8": dict(n=8, seed=10, kind="general", outliers=0.0, iterations=1),
    "planar_100_it1": dict(n=100, seed=11, kind="planar", outliers=0.0, iterations=1),
}
