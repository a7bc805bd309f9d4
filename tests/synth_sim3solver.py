"""Loop-closure candidates for Sim3Solver, built from first principles: two keyframes whose map points are related by
a similarity S12 = (s, R, t) (X1c = s*R*X2c + t in camera coordinates), with pixel noise, wrong matches, mixed pyramid
levels and the constructor's skip cases (no match, no map point in KF1, bad points, points not observed).

scene(...) returns the flattened keyframes the reference's constructor reads (see oracle/ref_sim3solver_glue.cpp's
s3s_scene) and problem(sc) the b2s_sim3solver_problem fields that constructor produces (X1c, X2c, sigma2 per kept
correspondence, K, fix_scale) with mvnIndices1."""
import numpy as np

from sim3solver_binding import camera_points

SCALE_FACTOR = np.float32(1.2)
N_LEVELS = 8


def level_sigma2():
    """ORBextractor's mvLevelSigma2: float products of the scale factor, squared in float."""
    f = [np.float32(1.0)]
    for _ in range(1, N_LEVELS):
        f.append(np.float32(f[-1] * SCALE_FACTOR))
    return np.array([np.float32(v * v) for v in f], np.float32)


def _rot(rng, deg):
    axis = rng.standard_normal(3)
    axis /= np.linalg.norm(axis)
    a = np.deg2rad(deg)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + np.sin(a) * K + (1 - np.cos(a)) * K @ K


def _pose(rng):
    T = np.eye(4)
    T[:3, :3] = _rot(rng, rng.uniform(0, 40))
    T[:3, 3] = rng.uniform(-2, 2, 3)
    return T.astype(np.float32)


def scene(n=200, inliers=0.7, seed=0, fix_scale=False, rot_deg=20.0, scale=1.3, noise_px=0.6, levels=N_LEVELS,
          skips=0.1, kind="loop"):
    """n keypoint slots in KF1.  kind: 'loop' (a true Sim3 between the two maps), 'identity' (S12 = I: the same camera
    points in both keyframes) or 'degenerate' (every kept correspondence repeats one of three points, or lies on a
    line, so every minimal set is singular)."""
    rng = np.random.default_rng(seed)
    K1 = np.array([[520.0, 0, 320.0], [0, 521.0, 240.0], [0, 0, 1]], np.float32)
    K2 = np.array([[518.0, 0, 318.0], [0, 517.0, 242.0], [0, 0, 1]], np.float32)
    s = 1.0 if fix_scale or kind == "identity" else scale
    R = np.eye(3) if kind == "identity" else _rot(rng, rot_deg)
    t = np.zeros(3) if kind == "identity" else rng.uniform(-0.5, 0.5, 3)
    # camera-1 points in front of both cameras
    X1 = np.stack([rng.uniform(-3, 3, n), rng.uniform(-2, 2, n), rng.uniform(4, 12, n)], 1)
    if kind == "degenerate":
        base = X1[:3].copy()
        line = base[0] + np.outer(rng.uniform(0, 1, n), base[1] - base[0])
        X1 = np.where((np.arange(n) % 2 == 0)[:, None], base[np.arange(n) % 3], line)
    X2 = ((X1 - t) @ R) / s  # R^T (X1 - t) / s
    octave1 = rng.integers(0, levels, n).astype(np.int32)
    octave2 = rng.integers(0, levels, n).astype(np.int32)
    sig2 = level_sigma2()
    # pixel noise in each image, scaled with the level as the detector's would be
    def perturb(X, K, oct_):
        z = X[:, 2:3]
        px = rng.standard_normal((len(X), 2)) * noise_px * np.sqrt(sig2[oct_])[:, None]
        return X + np.concatenate([px / np.array([K[0, 0], K[1, 1]]) * z, np.zeros_like(z)], 1)
    if kind == "loop":
        X1 = perturb(X1, K1, octave1)
        X2 = perturb(X2, K2, octave2)
    wrong = rng.uniform(0, 1, n) >= inliers
    X2[wrong] = np.stack([rng.uniform(-3, 3, wrong.sum()), rng.uniform(-2, 2, wrong.sum()),
                          rng.uniform(4, 12, wrong.sum())], 1) / s
    Tcw1, Tcw2 = _pose(rng), _pose(rng)

    def world(T, Xc):
        Rm, tv = T[:3, :3].astype(np.float64), T[:3, 3].astype(np.float64)
        return ((Xc - tv) @ Rm).astype(np.float32)

    u = rng.uniform(0, 1, (5, n))
    matched = (u[0] >= skips / 2).astype(np.int32)
    has_mp1 = (u[1] >= skips / 4).astype(np.int32)
    bad1 = (u[2] < skips / 4).astype(np.int32)
    bad2 = (u[3] < skips / 4).astype(np.int32)
    idx1 = np.arange(n, dtype=np.int32)
    idx2 = rng.permutation(n).astype(np.int32)
    unobs = u[4] < skips / 4
    idx1[unobs & (np.arange(n) % 2 == 0)] = -1
    idx2[unobs & (np.arange(n) % 2 == 1)] = -1
    oct2_by_idx = np.zeros(n, np.int32)
    oct2_by_idx[idx2[idx2 >= 0]] = octave2[idx2 >= 0]
    return dict(m=n, nk2=n, fix_scale=int(fix_scale), Tcw1=Tcw1, Tcw2=Tcw2, K1=K1, K2=K2, level_sigma2_1=sig2,
                level_sigma2_2=sig2, octave1=octave1, octave2=oct2_by_idx, matched=matched, has_mp1=has_mp1,
                bad1=bad1, bad2=bad2, idx1=idx1, idx2=idx2, Xw1=world(Tcw1, X1), Xw2=world(Tcw2, X2),
                true_wrong=wrong, S=(s, R, t))


def problem(sc, min_inliers=20, max_its=300):
    """The constructor's correspondences (:78-127) as b2s_sim3solver_problem fields, and mvnIndices1."""
    keep = [i for i in range(sc["m"]) if sc["matched"][i] and sc["has_mp1"][i] and not sc["bad1"][i]
            and not sc["bad2"][i] and sc["idx1"][i] >= 0 and sc["idx2"][i] >= 0]
    keep = np.array(keep, np.int64)
    sig = sc["level_sigma2_1"]
    K1, K2 = sc["K1"], sc["K2"]
    return dict(X1c=camera_points(sc["Tcw1"], sc["Xw1"][keep]), X2c=camera_points(sc["Tcw2"], sc["Xw2"][keep]),
                sigma2_1=sig[sc["octave1"][sc["idx1"][keep]]], sigma2_2=sig[sc["octave2"][sc["idx2"][keep]]],
                K1=np.array([K1[0, 0], K1[1, 1], K1[0, 2], K1[1, 2]], np.float32),
                K2=np.array([K2[0, 0], K2[1, 1], K2[0, 2], K2[1, 2]], np.float32), fix_scale=sc["fix_scale"],
                min_inliers=min_inliers, max_its=max_its, indices1=keep.astype(np.int32))


# name -> (scene kwargs, (probability, minInliers, maxIterations))
CASES = {
    "loop_90_free": (dict(n=200, inliers=0.9, seed=1), (0.99, 20, 300)),
    "loop_60_free": (dict(n=300, inliers=0.6, seed=2), (0.99, 20, 300)),
    "loop_30_free": (dict(n=400, inliers=0.3, seed=3), (0.99, 20, 300)),
    "loop_70_fixed": (dict(n=250, inliers=0.7, seed=4, fix_scale=True), (0.99, 20, 300)),
    "loop_40_fixed_levels": (dict(n=500, inliers=0.4, seed=5, fix_scale=True, noise_px=1.2), (0.99, 20, 300)),
    "loop_50_free_800": (dict(n=800, inliers=0.5, seed=6, noise_px=1.0), (0.99, 20, 300)),
    "loop_demanding": (dict(n=300, inliers=0.35, seed=7), (0.99, 60, 300)),
    "outliers_only": (dict(n=150, inliers=0.0, seed=8), (0.99, 20, 300)),
    "outliers_only_fixed": (dict(n=120, inliers=0.0, seed=9, fix_scale=True), (0.99, 20, 40)),
    "too_few": (dict(n=24, inliers=0.9, seed=10), (0.99, 20, 300)),
    "min_equals_n": (dict(n=30, inliers=0.9, seed=11, skips=0.0), (0.99, 30, 300)),
    "identity": (dict(n=120, inliers=0.8, seed=12, kind="identity", skips=0.0), (0.99, 20, 300)),
    "degenerate": (dict(n=60, inliers=1.0, seed=13, kind="degenerate", skips=0.0), (0.99, 6, 300)),
}
