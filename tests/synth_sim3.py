"""Synthetic loop-closure candidates for Optimizer::OptimizeSim3 (src/Optimizer.cc:1364-1590).

A scene is the object graph the reference's function reads: two keyframes with different intrinsics and poses, a pool
of map points (those of pKF1's map, then those of pKF2's map), pKF1's map-point matches, pKF2's observations and the
candidate matches vpMatches1.  The true S12 maps pKF2's camera frame into pKF1's (scale 1 for stereo, 0.7-1.4 for
monocular); each map carries its own point noise, observations carry pixel noise 1.2^octave, a share of the matches are
gross mismatches, and the initial S12 is perturbed by about 1 degree, a few % of the translation and (monocular) 3 % of
the scale, the accuracy Sim3Solver hands over.  Null matches, null and bad points and points pKF2 does not observe
exercise every skip rule.  Everything the reference holds in float is float32.

flatten() is the drop-in body's gather: the skip rules in the reference's order and the camera-frame points by the
cv::Mat expression R*P + t (a gemm with double accumulation, rounded to float, then a float addition)."""
import numpy as np

N_LEVELS = 8
INV_SIGMA2 = (1.0 / 1.2 ** (2 * np.arange(N_LEVELS))).astype(np.float32)


def _rot(rng, deg):
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    a = np.deg2rad(deg)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + np.sin(a) * K + (1 - np.cos(a)) * K @ K


def _quat(R):
    """Eigen::Quaterniond(Matrix3d) as qx qy qz qw."""
    t = np.trace(R)
    q = np.zeros(4)
    if t > 0:
        s = np.sqrt(t + 1.0)
        q[3] = 0.5 * s
        s = 0.5 / s
        q[0], q[1], q[2] = (R[2, 1] - R[1, 2]) * s, (R[0, 2] - R[2, 0]) * s, (R[1, 0] - R[0, 1]) * s
    else:
        i = 0
        if R[1, 1] > R[0, 0]:
            i = 1
        if R[2, 2] > R[i, i]:
            i = 2
        j, k = (i + 1) % 3, (i + 2) % 3
        s = np.sqrt(R[i, i] - R[j, j] - R[k, k] + 1.0)
        q[i] = 0.5 * s
        s = 0.5 / s
        q[3] = (R[k, j] - R[j, k]) * s
        q[j] = (R[j, i] + R[i, j]) * s
        q[k] = (R[k, i] + R[i, k]) * s
    return q


def synth_sim3(n=200, seed=0, mono=False, outliers=0.1, point_noise=0.01, px=1.0, n_null=None, n_skip=None):
    """n candidate matches (keypoints of pKF1); a share `outliers` of them are gross mismatches."""
    rng = np.random.default_rng(seed)
    K1 = np.array([520.0, 518.0, 320.0, 240.0], np.float32)
    K2 = np.array([458.5, 457.2, 367.2, 248.4], np.float32)
    s_true = float(rng.uniform(0.7, 1.4)) if mono else 1.0
    R12, t12 = _rot(rng, rng.uniform(5, 20)), rng.normal(size=3) * 0.5
    T1 = np.eye(4)
    T1[:3, :3], T1[:3, 3] = _rot(rng, 30), rng.normal(size=3) * 2
    T2 = np.eye(4)
    T2[:3, :3], T2[:3, 3] = _rot(rng, 30), rng.normal(size=3) * 2
    T1, T2 = T1.astype(np.float32), T2.astype(np.float32)
    # true points in pKF1's camera frame, seen by both cameras
    X1 = np.stack([rng.uniform(-4, 4, n), rng.uniform(-3, 3, n), rng.uniform(5, 15, n)], 1)
    X2 = ((X1 - t12) @ R12) / s_true  # S12^-1 X1 = R12^T (X1 - t12) / s
    bad_z = X2[:, 2] < 1.0
    X2[bad_z, 2] += 6.0  # keep every point in front of pKF2 (the correspondence is then slightly off: an outlier)
    R1, t1 = T1[:3, :3].astype(np.float64), T1[:3, 3].astype(np.float64)
    R2, t2 = T2[:3, :3].astype(np.float64), T2[:3, 3].astype(np.float64)
    P1 = (X1 - t1) @ R1 + rng.normal(size=(n, 3)) * point_noise
    P2 = (X2 - t2) @ R2 + rng.normal(size=(n, 3)) * point_noise / s_true
    oct1, oct2 = rng.integers(0, N_LEVELS, n), rng.integers(0, N_LEVELS, n)

    def proj(K, X):
        return np.stack([X[:, 0] / X[:, 2] * K[0] + K[2], X[:, 1] / X[:, 2] * K[1] + K[3]], 1)

    kp1 = proj(K1, X1) + rng.normal(size=(n, 2)) * px * 1.2 ** oct1[:, None]
    kp2 = proj(K2, X2) + rng.normal(size=(n, 2)) * px * 1.2 ** oct2[:, None]
    n_out = int(round(outliers * n))
    out_idx = rng.choice(n, n_out, replace=False)
    kp2[out_idx] = np.stack([rng.uniform(0, 640, n_out), rng.uniform(0, 480, n_out)], 1)
    # object graph: point m < n is pKF1's map point of keypoint m, point n + m the pKF2 point it is matched with, observed
    # as pKF2's keypoint m
    mp1 = np.arange(n, dtype=np.int32)
    matches1 = (n + np.arange(n)).astype(np.int32)
    mp_bad = np.zeros(2 * n, np.uint8)
    mp_idx2 = np.full(2 * n, -1, np.int32)
    mp_idx2[n:] = np.arange(n)
    n_null = max(1, n // 20) if n_null is None else n_null
    n_skip = max(1, n // 40) if n_skip is None else n_skip
    perm = rng.permutation(n)
    c = 0
    matches1[perm[c:c + n_null]] = -1; c += n_null          # vpMatches1[i] null
    mp1[perm[c:c + n_skip]] = -1; c += n_skip              # pKF1 has no map point there
    mp_bad[perm[c:c + n_skip]] = 1; c += n_skip            # pMP1 bad
    mp_bad[n + perm[c:c + n_skip]] = 1; c += n_skip        # pMP2 bad
    mp_idx2[n + perm[c:c + n_skip]] = -1; c += n_skip      # pMP2 not observed in pKF2
    # initial estimate: the truth perturbed as Sim3Solver leaves it
    R0 = _rot(rng, 1.0) @ R12
    t0 = t12 + rng.normal(size=3) * 0.03 * max(np.linalg.norm(t12), 0.1)
    s0 = s_true * (1 + 0.03 * rng.choice([-1, 1])) if mono else 1.0
    S12 = np.concatenate([_quat(R0), t0, [s0]])
    return dict(Tcw1=T1.reshape(16), Tcw2=T2.reshape(16), K1=K1, K2=K2, kp1=kp1.astype(np.float32),
                oct1=oct1.astype(np.int32), kp2=kp2.astype(np.float32), oct2=oct2.astype(np.int32),
                inv_sigma2=INV_SIGMA2, points=np.concatenate([P1, P2]).astype(np.float32), mp_bad=mp_bad,
                mp_idx2=mp_idx2, mp1=mp1, matches1=matches1, S12=S12, th2=np.float32(10.0), fix_scale=not mono,
                s_true=s_true)


def _cam(T, P):
    """R*P + t as the reference's cv::Mat expression evaluates it."""
    R = T.reshape(4, 4)[:3, :3].astype(np.float64)
    t = T.reshape(4, 4)[:3, 3]
    acc = np.zeros((len(P), 3))
    for k in range(3):
        acc = acc + R[None, :, k] * P[:, k:k + 1].astype(np.float64)
    return acc.astype(np.float32) + t[None, :]


def flatten(sc):
    """The drop-in body's gather: returns (problem dict for b2s_optimize_sim3 / orc_optimize_sim3, vnIndexEdge)."""
    idx = []
    for i in range(len(sc["matches1"])):
        j2, j1 = int(sc["matches1"][i]), int(sc["mp1"][i])
        if j2 < 0 or j1 < 0:
            continue
        if sc["mp_bad"][j1] or sc["mp_bad"][j2] or sc["mp_idx2"][j2] < 0:
            continue
        idx.append(i)
    idx = np.array(idx, np.int64)
    j1 = sc["mp1"][idx]
    j2 = sc["matches1"][idx]
    i2 = sc["mp_idx2"][j2]
    d = dict(X1c=_cam(sc["Tcw1"], sc["points"][j1]), X2c=_cam(sc["Tcw2"], sc["points"][j2]),
             obs1=sc["kp1"][idx], obs2=sc["kp2"][i2], inv_sigma2_1=sc["inv_sigma2"][sc["oct1"][idx]],
             inv_sigma2_2=sc["inv_sigma2"][sc["oct2"][i2]], K1=sc["K1"], K2=sc["K2"], S12=sc["S12"], th2=sc["th2"],
             fix_scale=sc["fix_scale"])
    return d, idx


def expand(sc, keep, idx):
    """The scatter: vpMatches1[i] is non-null afterwards."""
    kept = sc["matches1"] >= 0
    kept[idx[np.asarray(keep) == 0]] = False
    return kept


# seeds of the oracle-vs-reference and device-vs-oracle tests: every branch of the function
CASES = {
    "stereo_200_outliers": dict(n=200, seed=1, mono=False, outliers=0.15),           # nMore = 10
    "mono_400_outliers": dict(n=400, seed=2, mono=True, outliers=0.3),               # nMore = 10
    "stereo_1500": dict(n=1500, seed=3, mono=False, outliers=0.05),                  # nMore = 10
    "mono_800_clean": dict(n=800, seed=4, mono=True, outliers=0.2, px=0.5),          # nMore = 10
    "stereo_60_clean": dict(n=60, seed=5, mono=False, outliers=0.0, point_noise=0.001, px=0.3),  # nMore = 5
    "mono_40_clean": dict(n=40, seed=6, mono=True, outliers=0.0, point_noise=0.001, px=0.3),     # nMore = 5
    "mono_12_early": dict(n=12, seed=7, mono=True, outliers=0.5, n_null=0, n_skip=0),           # early return
    "empty": dict(n=10, seed=8, mono=False, outliers=0.0, n_null=10, n_skip=0),                 # no correspondence
}
