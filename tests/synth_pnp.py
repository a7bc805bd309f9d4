"""Synthetic relocalisation scenes for PnPsolver: map points seen by a 640 x 480 camera, true matches with pixel noise
and wrong matches, octave-dependent sigma2 at scale factor 1.2 (mvLevelSigma2[octave] = 1.2^(2 octave)), and the
geometries that stress EPnP: a plane, a nearly collinear set, a repeated world point, outliers behind the camera."""
import numpy as np

K = np.array([520.0, 518.0, 320.5, 240.25], np.float32)
RELOC = (0.99, 10, 300, 4, 0.5, 5.991)    # Tracking::Relocalization's SetRansacParameters
DEFAULT = (0.99, 8, 300, 4, 0.4, 5.991)   # the header's defaults


def _rot(rng, scale):
    w = rng.normal(size=3) * scale
    th = np.linalg.norm(w)
    k = w / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx


def scene(n, inlier_frac=0.7, seed=0, kind="general", noise=0.7, params=RELOC):
    """A scene dict: P3Dw (n x 3), P2D (n x 2), sigma2 (n), K, th2, params (SetRansacParameters' arguments),
    min_inliers and max_its (what SetRansacParameters leaves), truth (n bools) and the true Tcw."""
    import importlib
    pkg = importlib.import_module("self_commit_orb-slam2_b200")
    rng = np.random.default_rng(seed)
    R = _rot(rng, 0.3)
    t = rng.normal(size=3) * 0.5
    # camera-frame points, then to the world frame
    z = rng.uniform(2.0, 8.0, n)
    u = rng.uniform(20, 620, n)
    v = rng.uniform(20, 460, n)
    Xc = np.stack([(u - K[2]) / K[0] * z, (v - K[3]) / K[1] * z, z], 1)
    Xw = (Xc - t) @ R  # R^T (Xc - t)
    if kind == "planar":  # every point on the world plane through the first one, normal (0.2, 0.1, 1)
        nrm = np.array([0.2, 0.1, 1.0])
        Xw = Xw - np.outer((Xw - Xw[0]) @ nrm / (nrm @ nrm), nrm)
    elif kind == "collinear":  # a line with a millimetre of spread
        d = rng.normal(size=3)
        Xw = Xw[0] + np.outer(rng.uniform(-3, 3, n), d / np.linalg.norm(d)) + rng.normal(size=(n, 3)) * 1e-3
    elif kind == "repeated":
        Xw[1] = Xw[0]
        Xw[3] = Xw[2]
    Xw = Xw.astype(np.float32)
    Xc = Xw.astype(np.float64) @ R.T + t
    P2D = np.stack([K[0] * Xc[:, 0] / Xc[:, 2] + K[2], K[1] * Xc[:, 1] / Xc[:, 2] + K[3]], 1)
    octave = rng.integers(0, 8, n)
    sigma2 = (1.2 ** (2 * octave)).astype(np.float32)
    truth = rng.random(n) < inlier_frac
    P2D = P2D + rng.normal(size=(n, 2)) * noise * np.sqrt(sigma2)[:, None]
    out = ~truth
    P2D[out] = np.stack([rng.uniform(0, 640, out.sum()), rng.uniform(0, 480, out.sum())], 1)
    if kind == "behind":  # a quarter of the wrong matches are map points behind the camera
        b = np.where(out)[0][::4]
        Xb = Xc[b] * np.array([1, 1, -1.0])
        Xw[b] = ((Xb - t) @ R).astype(np.float32)
    m, its = pkg.pnp_ransac_parameters(n, *params[:5])
    Tcw = np.eye(4)
    Tcw[:3, :3], Tcw[:3, 3] = R, t
    return dict(P3Dw=Xw, P2D=P2D.astype(np.float32), sigma2=sigma2, K=K, th2=np.float32(params[5]), params=params,
                min_inliers=m, max_its=its, truth=truth, Tcw=Tcw)


# (name, n, inlier fraction, kind, SetRansacParameters)
CASES = [
    ("below_min", 12, 0.9, "general", (0.99, 20, 300, 4, 0.5, 5.991)),
    ("n15", 15, 0.9, "general", RELOC),
    ("n50", 50, 0.6, "general", RELOC),
    ("n200", 200, 0.3, "general", RELOC),
    ("n200_default", 200, 0.5, "general", DEFAULT),
    ("n1000", 1000, 0.5, "general", RELOC),
    ("n1000_dense", 1000, 0.9, "general", RELOC),  # qualifies: Refine over ~900 correspondences
    ("planar", 120, 0.7, "planar", RELOC),
    ("collinear", 60, 0.8, "collinear", RELOC),
    ("repeated", 40, 0.8, "repeated", RELOC),
    ("behind", 150, 0.5, "behind", RELOC),
    ("no_inliers", 80, 0.0, "general", RELOC),
]


def case(name, seed=0):
    for c in CASES:
        if c[0] == name:
            return scene(c[1], c[2], seed, c[3], params=c[4])
    raise KeyError(name)
