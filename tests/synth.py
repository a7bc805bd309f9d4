"""Deterministic synthetic inputs (integer-only numpy so they reproduce bit-for-bit on any box).

SURVEY.md §8(d): textured images that fill the per-level quotas; stereo pairs with band disparity;
descriptor sets with known correspondences; a KITTI-shaped LocalBA window.
"""
import numpy as np


def _blur5(a):
    """separable [1,4,6,4,1]/16 integer blur with edge replication"""
    a = a.astype(np.int32)
    k = (1, 4, 6, 4, 1)
    p = np.pad(a, ((0, 0), (2, 2)), mode="edge")
    h = sum(k[i] * p[:, i:i + a.shape[1]] for i in range(5))
    p = np.pad(h, ((2, 2), (0, 0)), mode="edge")
    v = sum(k[i] * p[i:i + a.shape[0], :] for i in range(5))
    return (v + 128) >> 8


def synth_image(w, h, seed, blocks=True):
    rng = np.random.RandomState(seed)
    noise = rng.randint(0, 256, size=(h, w)).astype(np.int32)
    base = _blur5(noise) // 2 + 40
    if blocks:
        bs = 12
        gh, gw = (h + bs - 1) // bs, (w + bs - 1) // bs
        on = rng.randint(0, 100, size=(gh, gw)) < 22
        amp = rng.randint(60, 121, size=(gh, gw)) * on
        amp = np.kron(amp, np.ones((bs, bs), dtype=np.int32))[:h, :w]
        base = base + amp
    # a few smooth gradients so low-texture cells exist (exercise the minThFAST fallback)
    yy, xx = np.mgrid[0:h, 0:w]
    flat = ((xx // 97 + yy // 61) % 5 == 0)
    base = np.where(flat, 90 + ((xx + yy) >> 5), base)
    return np.clip(base, 0, 255).astype(np.uint8)


TEXTURES = ("noise", "saltpepper", "dark", "bright", "checker2", "checker3", "checker4", "checker5", "checker6", "corner",
            "fallback", "dense")


def level_sizes(W, H, scale_factor, nlevels):
    """(w, h) of every pyramid level as the extractor rounds them: cvRound(W * mvInvScaleFactor[l]) in float32, with
    mvScaleFactor[l] = (float)(mvScaleFactor[l-1] * (double)scaleFactor) (src/ORBextractor.cc:500-520, :1680-1682)."""
    sf = np.float64(np.float32(scale_factor))
    s, out = np.float32(1.0), []
    for l in range(nlevels):
        if l:
            s = np.float32(np.float64(s) * sf)
        inv = np.float32(1.0) / s
        out.append((int(np.rint(np.float32(W) * inv)), int(np.rint(np.float32(H) * inv))))
    return out


def grid_ok(w, h):
    """The 30-px cell grid of a level exists (nCols, nRows >= 1) and its width is >= height / 2 (quadtree roots)."""
    width, height = np.float32(w - 32), np.float32(h - 32)
    return int(width / np.float32(30)) >= 1 and int(height / np.float32(30)) >= 1 and round(float(width / height)) >= 1


def residue_shapes(scale_factor=1.2, nlevels=8):
    """A small set of image sizes such that, over all of them, some level's width is 0, 1 and 127 mod 128 (the tile
    width) and some level's height is 0, 1 and 31 mod 32 (the tile height).  Returns [(W, H)] and the residues covered."""
    shapes, xs, ys = [], set(), set()
    want_x, want_y = {0, 1, 127}, {0, 1, 31}
    W, H = 640, 480
    for Wc in range(640, 1100):
        lv = level_sizes(Wc, H, scale_factor, nlevels)
        got = {w % 128 for w, _ in lv} & (want_x - xs)
        if got:
            shapes.append((Wc, H))
            xs |= {w % 128 for w, _ in lv} & want_x
        if xs == want_x:
            break
    for Hc in range(400, 700):
        lv = level_sizes(W, Hc, scale_factor, nlevels)
        got = {h % 32 for _, h in lv} & (want_y - ys)
        if got:
            shapes.append((W, Hc))
            ys |= {h % 32 for _, h in lv} & want_y
        if ys == want_y:
            break
    return shapes, xs, ys


def synth_texture(kind, w, h, seed):
    """Extractor stress textures: uniform noise 0..255 (dense candidates), salt-and-pepper 0/255, dark 0..30 and bright
    225..255 noise (FAST's p - t < 0 and p + t > 255 lanes), checkerboards of period 2..6, one isolated corner on a
    constant image, and weak noise with strong noise only in the first 30 columns after the border (every other level-0
    cell has no maximum above iniThFAST and goes through the minThFAST pass)."""
    rng = np.random.RandomState(seed)
    if kind == "noise":
        return rng.randint(0, 256, size=(h, w)).astype(np.uint8)
    if kind == "saltpepper":
        return (rng.randint(0, 2, size=(h, w)) * 255).astype(np.uint8)
    if kind == "dark":
        return rng.randint(0, 31, size=(h, w)).astype(np.uint8)
    if kind == "bright":
        return (225 + rng.randint(0, 31, size=(h, w))).astype(np.uint8)
    if kind.startswith("checker"):
        p = int(kind[7:])
        yy, xx = np.mgrid[0:h, 0:w]
        return np.where((xx // p + yy // p) % 2 == 0, 40, 210).astype(np.uint8)
    if kind == "corner":
        img = np.full((h, w), 90, np.uint8)
        img[h // 2:, w // 2:] = 180
        return img
    if kind == "dense":  # a 2 x 7 tile on which 56 % of all pixels are FAST corners at threshold 20
        tile = np.array([[8, 214], [84, 9], [201, 3], [103, 31], [90, 160], [135, 41], [132, 109]], np.uint8)
        return np.tile(tile, (h // 7 + 1, w // 2 + 1))[:h, :w].copy()
    if kind == "fallback":
        img = (100 + rng.randint(0, 18, size=(h, w))).astype(np.uint8)
        img[:, 19:49] = rng.randint(0, 256, size=(h, 30))
        return img
    raise ValueError(kind)


_CIRCLE = ((0, 3), (1, 3), (2, 2), (3, 1), (3, 0), (3, -1), (2, -2), (1, -3), (0, -3), (-1, -3), (-2, -2), (-3, -1), (-3, 0),
           (-3, 1), (-2, 2), (-1, 3))


def fast_strength(img):
    """FAST-9/16 arc strength of every pixel (0 on the 3-pixel rim): M = max over the 16 arcs of 9 circle pixels of
    min |I_k - p| with one sign; a pixel is a corner at threshold t iff M > t."""
    a = img.astype(np.int32)
    h, w = a.shape
    c = a[3:h - 3, 3:w - 3]
    ring = np.stack([a[3 + dy:h - 3 + dy, 3 + dx:w - 3 + dx] for dx, dy in _CIRCLE])
    ring = np.concatenate([ring, ring[:8]])
    bright = np.max([ring[s:s + 9].min(axis=0) for s in range(16)], axis=0) - c
    dark = c - np.min([ring[s:s + 9].max(axis=0) for s in range(16)], axis=0)
    M = np.zeros((h, w), np.int32)
    M[3:h - 3, 3:w - 3] = np.maximum(np.maximum(bright, dark), 0)
    return M


def synth_stereo(w, h, seed):
    left = synth_image(w, h, seed)
    rng = np.random.RandomState(seed + 100003)
    right = np.empty_like(left)
    band = 47
    for y0 in range(0, h, band):
        d = int(rng.randint(5, 61))
        rows = left[y0:y0 + band]
        shifted = np.empty_like(rows)
        shifted[:, :w - d] = rows[:, d:]
        shifted[:, w - d:] = rows[:, w - d - 1:w - d]  # replicate
        right[y0:y0 + band] = shifted
    jitter = rng.randint(-2, 3, size=(h, w))
    right = np.clip(right.astype(np.int32) + jitter, 0, 255).astype(np.uint8)
    return left, right


def synth_descriptors(n, seed=1234, match_frac=0.7, max_flips=40, n_nodes=100):
    """A (keyframe side) and B (frame side) descriptor sets, node ids, angles (SURVEY §8d Matching)."""
    rng = np.random.RandomState(seed)
    A = rng.randint(0, 256, size=(n, 32)).astype(np.uint8)
    perm = rng.permutation(n)
    B = rng.randint(0, 256, size=(n, 32)).astype(np.uint8)
    angA = (rng.randint(0, 360000, size=n) / 1000.0).astype(np.float32)
    angB = (rng.randint(0, 360000, size=n) / 1000.0).astype(np.float32)
    nodeA = rng.randint(0, n_nodes, size=n).astype(np.int32)
    nodeB = rng.randint(0, n_nodes, size=n).astype(np.int32)
    for i in range(n):
        if rng.randint(0, 1000) < match_frac * 1000:
            j = perm[i]
            d = A[j].copy()
            k = int(rng.randint(0, max_flips + 1))
            bits = rng.choice(256, size=k, replace=False)
            for b in bits:
                d[b >> 3] ^= np.uint8(1 << (b & 7))
            B[i] = d
            nodeB[i] = nodeA[j]
            a = float(angA[j]) + float(rng.randint(-15000, 15001)) / 3000.0
            angB[i] = np.float32(a % 360.0)
    validA = (rng.randint(0, 100, size=n) < 95).astype(np.uint8)
    return A, nodeA, validA, angA, B, nodeB, angB


def _path_position(n_kf, revisit):
    """Position of every keyframe along the path (metres): a straight forward path, or with `revisit` one that runs
    twice over the same ground, so that keyframes k and k + ceil(n_kf / 2) see the same points."""
    k = np.arange(n_kf)
    return k % -(-n_kf // 2) if revisit else k


def synth_local_ba(n_kf=50, n_fixed=10, n_mp=5000, obs_per_mp=6, seed=42, mono_frac=0.0, outlier_frac=0.03,
                   fix_first=True, revisit=False):
    """KITTI-shaped LocalBA window (SURVEY §8d): forward path, stereo edges, 3 % gross outliers.

    Returns dict with float32 arrays exactly as Converter would hand them over.
    Keyframes [0, n_kf-n_fixed) are local: free, except keyframe 0 when fix_first (it plays the map's first keyframe,
    mnId == 0); the last n_fixed are fixed cameras.  A point is observed by the obs_per_mp keyframes that see it and lie
    nearest its anchor keyframe along the path; with `revisit` the path passes twice over the same ground, so the
    covisibility graph is not banded (see _path_position).  The defaults reproduce the windows of earlier versions bit for
    bit.
    """
    rng = np.random.RandomState(seed)
    fx = fy = 718.856
    cx, cy, bf = 607.1928, 185.2157, 386.1448
    W, H = 1241, 376
    n_local = n_kf - n_fixed
    pos = _path_position(n_kf, revisit)
    # true poses: camera moves along +z, 1 m spacing, small yaw jitter. Tcw = [R | -R*c]
    Tcw_true = np.zeros((n_kf, 4, 4))
    for k in range(n_kf):
        yaw = np.deg2rad(rng.uniform(-2, 2))
        c, s = np.cos(yaw), np.sin(yaw)
        R = np.array([[c, 0, -s], [0, 1, 0], [s, 0, c]])
        center = np.array([rng.uniform(-0.1, 0.1), rng.uniform(-0.05, 0.05), 1.0 * pos[k]])
        Tcw_true[k, :3, :3] = R
        Tcw_true[k, :3, 3] = -R @ center
        Tcw_true[k, 3, 3] = 1
    pts_true = np.zeros((n_mp, 3))
    edges = []
    order = rng.permutation(n_kf)
    for m in range(n_mp):
        # pick an anchor KF, place the point in its frustum 5-60 m ahead
        for _ in range(100):
            ka = int(rng.randint(0, n_kf))
            z = rng.uniform(5, 60)
            u = rng.uniform(50, W - 50)
            v = rng.uniform(30, H - 30)
            Xc = np.array([(u - cx) * z / fx, (v - cy) * z / fy, z])
            Ra, ta = Tcw_true[ka, :3, :3], Tcw_true[ka, :3, 3]
            Xw = Ra.T @ (Xc - ta)
            # which KFs see it
            vis = []
            for k in range(n_kf):
                Xk = Tcw_true[k, :3, :3] @ Xw + Tcw_true[k, :3, 3]
                if Xk[2] < 2.0:
                    continue
                uu = fx * Xk[0] / Xk[2] + cx
                vv = fy * Xk[1] / Xk[2] + cy
                if 0 < uu < W and 0 < vv < H:
                    vis.append((abs(int(pos[k]) - int(pos[ka])), k, uu, vv, Xk[2]))
            if len(vis) >= obs_per_mp:
                break
        vis.sort()
        pts_true[m] = Xw
        for (_, k, uu, vv, zz) in sorted(vis[:obs_per_mp], key=lambda t: t[1]):
            octv = int(rng.randint(0, 8))
            sig = 1.2 ** octv
            nu, nv, nr = rng.normal(0, sig, 3)
            ur = uu - bf / zz
            if rng.uniform() < outlier_frac:
                nu += 30.0
            mono = rng.uniform() < mono_frac
            edges.append((k, m, uu + nu, vv + nv, -1.0 if mono else ur + nr, 1.0 / (1.2 ** (2 * octv))))
    # perturbed initial state
    Tcw0 = Tcw_true.copy()
    for k in range(n_local):
        dyaw = np.deg2rad(rng.normal(0, 0.2))
        c, s = np.cos(dyaw), np.sin(dyaw)
        dR = np.array([[c, 0, -s], [0, 1, 0], [s, 0, c]])
        Tcw0[k, :3, :3] = dR @ Tcw_true[k, :3, :3]
        Tcw0[k, :3, 3] = dR @ Tcw_true[k, :3, 3] + rng.normal(0, 0.02, 3)
    pts0 = pts_true + rng.normal(0, 0.05, pts_true.shape)
    fixed = np.zeros(n_kf, np.uint8)
    fixed[n_local:] = 1
    if fix_first:
        fixed[0] = 1  # plays the role of mnId==0
    edge_dt = np.dtype([("kf", "i4"), ("mp", "i4"), ("obs", "f4", 3), ("inv_sigma2", "f4")])
    E = np.zeros(len(edges), edge_dt)
    for i, (k, m, a, b_, c_, w) in enumerate(edges):
        E[i] = (k, m, (np.float32(a), np.float32(b_), np.float32(c_)), np.float32(w))
    return dict(n_kf=n_kf, n_local=n_local, Tcw=Tcw0.astype(np.float32).reshape(n_kf, 16), fixed=fixed,
                points=pts0.astype(np.float32), edges=E, fx=np.float32(fx), fy=np.float32(fy), cx=np.float32(cx),
                cy=np.float32(cy), bf=np.float32(bf), Tcw_true=Tcw_true, pts_true=pts_true)


CROWD_F, CROWD_Q = np.arange(100, 112), np.arange(5, 21)


def synth_projection(nf=2000, nq=1800, seed=7, w=1241, h=376, cluster=False, th=7.0, crowd=False):
    """Current-frame features + projected last-frame map points (SURVEY A5 / src/ORBmatcher.cc:1569).
    crowd: the 12 features CROWD_F share one descriptor inside one window and the 16 queries CROWD_Q (the first valid
    ones) carry it too, so from the ninth of them on the K-list (8 entries) holds only taken features while the window
    has more than 8 candidates."""
    rng = np.random.RandomState(seed)
    scale = np.array([np.float32(1.2) ** i for i in range(8)], np.float32)
    if cluster:
        kpx = (300 + rng.randint(0, 1200, size=nf) / 10.0).astype(np.float32)
        kpy = (150 + rng.randint(0, 600, size=nf) / 10.0).astype(np.float32)
    else:
        kpx = (rng.randint(0, w * 10, size=nf) / 10.0).astype(np.float32)
        kpy = (rng.randint(0, h * 10, size=nf) / 10.0).astype(np.float32)
    octave = rng.randint(0, 8, size=nf).astype(np.int32)
    angle = (rng.randint(0, 360000, size=nf) / 1000.0).astype(np.float32)
    desc = rng.randint(0, 256, size=(nf, 32)).astype(np.uint8)
    if cluster:  # near-duplicate descriptors so that K-lists run dry
        base = rng.randint(0, 256, size=(4, 32)).astype(np.uint8)
        desc = base[rng.randint(0, 4, size=nf)].copy()
        for i in range(nf):
            for b in rng.choice(256, size=int(rng.randint(0, 12)), replace=False):
                desc[i, b >> 3] ^= np.uint8(1 << (b & 7))
    bf = np.float32(386.1448)
    depth = rng.uniform(4, 60, size=nf).astype(np.float32)
    uright = (kpx - bf / depth).astype(np.float32)
    uright[rng.randint(0, 100, size=nf) < 20] = -1.0
    occupied = (rng.randint(0, 100, size=nf) < 5).astype(np.uint8)
    qdt = np.dtype([("u", "<f4"), ("v", "<f4"), ("invz", "<f4"), ("angle", "<f4"), ("octave", "<i4"),
                    ("has_obs", "<i4"), ("desc", "u1", 32)])
    q = np.zeros(nq, qdt)
    src = rng.randint(0, nf, size=nq)
    for i in range(nq):
        j = src[i]
        q["u"][i] = kpx[j] + np.float32(rng.randint(-40, 41) / 10.0)
        q["v"][i] = kpy[j] + np.float32(rng.randint(-40, 41) / 10.0)
        q["invz"][i] = np.float32(1.0) / depth[j] if rng.randint(0, 100) > 2 else np.float32(-0.1)
        q["angle"][i] = np.float32((float(angle[j]) + rng.randint(-12000, 12001) / 1000.0) % 360.0)
        q["octave"][i] = min(7, max(0, int(octave[j]) + int(rng.randint(-1, 2))))
        q["has_obs"][i] = 1 if rng.randint(0, 100) < 85 else 0
        d = desc[j].copy()
        for b in rng.choice(256, size=int(rng.randint(0, 30)), replace=False):
            d[b >> 3] ^= np.uint8(1 << (b & 7))
        q["desc"][i] = d
    # a few queries out of bounds
    q["u"][:5] = -3.0
    if crowd:
        x0, y0 = np.float32(w / 2), np.float32(h / 2)
        k = np.arange(len(CROWD_F))
        kpx[CROWD_F] = x0 + ((k % 4) - np.float32(1.5)) / np.float32(4)
        kpy[CROWD_F] = y0 + ((k // 4) - np.float32(1)) / np.float32(4)
        octave[CROWD_F], uright[CROWD_F], occupied[CROWD_F] = 0, -1.0, 0
        desc[CROWD_F], angle[CROWD_F] = desc[CROWD_F[0]], angle[CROWD_F[0]]
        q["u"][CROWD_Q], q["v"][CROWD_Q], q["invz"][CROWD_Q] = x0, y0, np.float32(0.1)
        q["angle"][CROWD_Q], q["octave"][CROWD_Q], q["has_obs"][CROWD_Q] = angle[CROWD_F[0]], 0, 1
        q["desc"][CROWD_Q] = desc[CROWD_F[0]]
    geom = dict(mnMinX=np.float32(0), mnMinY=np.float32(0), mnMaxX=np.float32(w), mnMaxY=np.float32(h), bf=bf,
                scale_factors=scale)
    return dict(q=q, kpx=kpx, kpy=kpy, octave=octave, angle=angle, uright=uright, occupied=occupied, desc=desc,
                geom=geom, th=np.float32(th))


def synth_projection_map(nf=2000, nq=2500, seed=9, w=1241, h=376, cluster=False, crowd=False):
    """Current-frame features + local map points after isInFrustum (SURVEY M4 / src/ORBmatcher.cc:70-175)."""
    d = synth_projection(nf=nf, nq=nq, seed=seed, w=w, h=h, cluster=cluster, crowd=crowd)
    rng = np.random.RandomState(seed + 77)
    q0 = d["q"]
    qdt = np.dtype([("u", "<f4"), ("v", "<f4"), ("ur", "<f4"), ("view_cos", "<f4"), ("level", "<i4"), ("in_view", "u1"),
                    ("has_obs", "u1"), ("pad", "u1", 2), ("desc", "u1", 32)])
    q = np.zeros(nq, qdt)
    q["u"], q["v"], q["desc"] = q0["u"], q0["v"], q0["desc"]
    q["u"][:5] = np.float32(-30.0)  # far outside: GetFeaturesInArea returns nothing
    invz = np.where(q0["invz"] > 0, q0["invz"], np.float32(0.05)).astype(np.float32)
    q["ur"] = (q0["u"] - d["geom"]["bf"] * invz + rng.randint(-30, 31, size=nq).astype(np.float32) / np.float32(10.0)).astype(np.float32)
    q["view_cos"] = np.where(rng.randint(0, 100, size=nq) < 50, np.float32(0.9995), np.float32(0.99)).astype(np.float32)
    q["view_cos"][::17] = np.float32(0.998)  # exactly at the (double) threshold of RadiusByViewingCos
    q["level"] = q0["octave"]
    q["in_view"] = (rng.randint(0, 100, size=nq) < 90).astype(np.uint8)
    q["has_obs"] = (rng.randint(0, 100, size=nq) < 85).astype(np.uint8)
    if crowd:
        q["in_view"][CROWD_Q], q["has_obs"][CROWD_Q] = 1, 1
    d = dict(d)
    d["q"] = q
    return d


def synth_windows(nf=2000, nq=2500, seed=13, th=3.0, cluster=False, crowd=False):
    """Keyframe features + projected map points for the Fuse / SearchByProjection(KeyFrame*, Scw, ...) search core."""
    d = synth_projection(nf=nf, nq=nq, seed=seed, cluster=cluster, crowd=crowd)
    rng = np.random.RandomState(seed + 5)
    q0 = d["q"]
    qdt = np.dtype([("u", "<f4"), ("v", "<f4"), ("ur", "<f4"), ("radius", "<f4"), ("min_level", "<i4"), ("max_level", "<i4"),
                    ("valid", "u1"), ("pad", "u1", 3), ("desc", "u1", 32)])
    q = np.zeros(nq, qdt)
    # small reprojection offsets so that the chi-square gate passes for some candidates and fails for others
    q["u"] = (q0["u"] + rng.randint(-15, 16, size=nq).astype(np.float32) / np.float32(10.0)).astype(np.float32)
    q["v"] = q0["v"]
    q["desc"] = q0["desc"]
    invz = np.where(q0["invz"] > 0, q0["invz"], np.float32(0.05)).astype(np.float32)
    q["ur"] = (q["u"] - d["geom"]["bf"] * invz).astype(np.float32)
    lvl = q0["octave"].astype(np.int32)
    q["radius"] = (np.float32(th) * d["geom"]["scale_factors"][lvl]).astype(np.float32)
    q["min_level"], q["max_level"] = lvl - 1, lvl
    q["valid"] = (rng.randint(0, 100, size=nq) < 92).astype(np.uint8)
    if crowd:
        q["valid"][CROWD_Q] = 1
    d = dict(d)
    d["q"] = q
    d["inv_sigma2"] = (np.float32(1.0) / (d["geom"]["scale_factors"] * d["geom"]["scale_factors"])).astype(np.float32)
    return d


def synth_triangulation(n=2000, seed=17, n_nodes=100, w=1241, h=376):
    """Two keyframes observing the same 3-D points (SearchForTriangulation, src/ORBmatcher.cc:810): keypoints scattered
    around the true projections, F12 / epipole computed like LocalMapping::ComputeF12 (src/LocalMapping.cc:1009-1035)."""
    rng = np.random.RandomState(seed)
    fx = fy = 718.856
    cx, cy = 607.1928, 185.2157
    K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1.0]])
    scale = np.array([np.float32(1.2) ** i for i in range(8)], np.float32)
    sigma2 = (scale * scale).astype(np.float32)
    yaw = np.deg2rad(3.0)
    R2 = np.array([[np.cos(yaw), 0, -np.sin(yaw)], [0, 1, 0], [np.sin(yaw), 0, np.cos(yaw)]])
    c2 = np.array([0.6, 0.02, 1.1])  # camera-2 centre in the frame of camera 1 (= world)
    t2 = -R2 @ c2
    R1, t1 = np.eye(3), np.zeros(3)
    R12 = R1 @ R2.T
    t12 = -R1 @ R2.T @ t2 + t1
    tx = np.array([[0, -t12[2], t12[1]], [t12[2], 0, -t12[0]], [-t12[1], t12[0], 0]])
    F12 = (np.linalg.inv(K).T @ tx @ R12 @ np.linalg.inv(K)).astype(np.float32)
    C2 = R2 @ np.zeros(3) + t2  # camera-1 centre in camera-2 coordinates
    ex = np.float32(fx * C2[0] / C2[2] + cx)
    ey = np.float32(fy * C2[1] / C2[2] + cy)
    z = rng.uniform(4, 60, size=n)
    u = rng.uniform(20, w - 20, size=n)
    v = rng.uniform(20, h - 20, size=n)
    X = np.stack([(u - cx) * z / fx, (v - cy) * z / fy, z], 1)
    X2 = (R2 @ X.T).T + t2
    u2 = fx * X2[:, 0] / X2[:, 2] + cx
    v2 = fy * X2[:, 1] / X2[:, 2] + cy
    octv = rng.randint(0, 8, size=n).astype(np.int32)
    noise = scale[octv].astype(np.float64)

    def kf(uu, vv, perm, flip_max):
        d = dict()
        d["x"] = (uu + rng.normal(0, 0.7, n) * noise).astype(np.float32)[perm]
        d["y"] = (vv + rng.normal(0, 0.7, n) * noise).astype(np.float32)[perm]
        # a fraction of gross outliers off the epipolar line
        bad = rng.randint(0, 100, size=n) < 15
        d["y"] = np.where(bad, d["y"] + np.float32(25.0), d["y"]).astype(np.float32)
        d["octave"] = np.clip(octv + rng.randint(-1, 2, size=n), 0, 7).astype(np.int32)[perm]
        d["angle"] = ((base_angle + rng.normal(0, 4, n)) % 360.0).astype(np.float32)[perm]
        dd = base_desc.copy()
        for i in range(n):
            for b in rng.choice(256, size=int(rng.randint(0, flip_max)), replace=False):
                dd[i, b >> 3] ^= np.uint8(1 << (b & 7))
        d["desc"] = dd[perm]
        d["node"] = base_node[perm].astype(np.int32)
        d["has_mp"] = (rng.randint(0, 100, size=n) < 35).astype(np.uint8)
        d["stereo"] = (rng.randint(0, 100, size=n) < 70).astype(np.uint8)
        return d

    base_angle = rng.uniform(0, 360, n)
    base_desc = rng.randint(0, 256, size=(n, 32)).astype(np.uint8)
    base_node = rng.randint(0, n_nodes, size=n)
    # near-duplicate descriptors inside a node so that ties and contention for the same feature occur
    dup = rng.randint(0, 100, size=n) < 20
    for i in np.nonzero(dup)[0]:
        same = np.nonzero(base_node == base_node[i])[0]
        base_desc[i] = base_desc[same[0]]
    kf1 = kf(u, v, np.arange(n), 20)
    kf2 = kf(u2, v2, rng.permutation(n), 25)
    return dict(kf1=kf1, kf2=kf2, F12=F12, ex=ex, ey=ey, scale=scale, sigma2=sigma2)


def synth_pose_problem(n=2000, seed=23, mp_frac=0.6, mono_frac=0.2, outlier_frac=0.1, pert_t=0.05, pert_deg=0.5):
    """One tracked frame for Optimizer::PoseOptimization (src/Optimizer.cc:363): map points seen from a true pose,
    noisy observations (sigma = 1 px * 1.2^octave), gross outliers, initial pose = motion-model prediction."""
    rng = np.random.RandomState(seed)
    fx = fy = np.float32(718.856)
    cx, cy, bf = np.float32(607.1928), np.float32(185.2157), np.float32(386.1448)
    W, H = 1241, 376
    yaw = np.deg2rad(rng.uniform(-3, 3))
    R = np.array([[np.cos(yaw), 0, -np.sin(yaw)], [0, 1, 0], [np.sin(yaw), 0, np.cos(yaw)]])
    c = np.array([rng.uniform(-0.3, 0.3), rng.uniform(-0.05, 0.05), rng.uniform(0, 2.0)])
    T = np.eye(4)
    T[:3, :3] = R
    T[:3, 3] = -R @ c
    z = rng.uniform(4, 60, size=n)
    u = rng.uniform(5, W - 5, size=n)
    v = rng.uniform(5, H - 5, size=n)
    Xc = np.stack([(u - cx) * z / fx, (v - cy) * z / fy, z], 1)
    Xw = (R.T @ (Xc - T[:3, 3]).T).T
    octv = rng.randint(0, 8, size=n)
    sig = 1.2 ** octv
    kpx = u + rng.normal(0, 1, n) * sig
    kpy = v + rng.normal(0, 1, n) * sig
    ur = u - bf / z + rng.normal(0, 1, n) * sig
    bad = rng.uniform(size=n) < outlier_frac
    kpx = np.where(bad, kpx + rng.choice([-1, 1], n) * rng.uniform(15, 60, n), kpx)
    mono = rng.uniform(size=n) < mono_frac
    ur = np.where(mono, -1.0, ur)
    has_mp = (rng.uniform(size=n) < mp_frac).astype(np.uint8)
    dyaw = np.deg2rad(rng.normal(0, pert_deg))
    dR = np.array([[np.cos(dyaw), 0, -np.sin(dyaw)], [0, 1, 0], [np.sin(dyaw), 0, np.cos(dyaw)]])
    T0 = np.eye(4)
    T0[:3, :3] = dR @ R
    T0[:3, 3] = dR @ T[:3, 3] + rng.normal(0, pert_t, 3)
    return dict(Tcw=T0.astype(np.float32).reshape(16), Tcw_true=T, has_mp=has_mp, Xw=Xw.astype(np.float32),
                kpx=kpx.astype(np.float32), kpy=kpy.astype(np.float32), uright=ur.astype(np.float32),
                inv_sigma2=(1.0 / (1.2 ** (2 * octv))).astype(np.float32), fx=fx, fy=fy, cx=cx, cy=cy, bf=bf)


def synth_vocabulary(k=10, L=4, seed=3, stop_frac=0.05, ragged=True):
    """A DBoW2-shaped vocabulary tree (k children per node, L levels) in text-file order (breadth-first like the k-means
    training writes it): children descriptors are noisy copies of their parent so the descent is meaningful; a few
    branches stop early (leaves above level L) when `ragged`."""
    rng = np.random.RandomState(seed)
    parent, leaf, desc, weight, level = [-1], [0], [np.zeros(32, np.uint8)], [0.0], [0]
    frontier = [0]
    for lv in range(1, L + 1):
        nxt = []
        for p in frontier:
            nchild = k if not ragged else int(rng.choice([k, k, k, k - 3]))
            for c in range(nchild):
                d = desc[p].copy() if lv > 1 else rng.randint(0, 256, 32).astype(np.uint8)
                flips = rng.choice(256, size=int(256 // (2 ** lv)), replace=False)
                for b in flips:
                    d[b >> 3] ^= np.uint8(1 << (b & 7))
                nid = len(parent)
                parent.append(p)
                is_leaf = lv == L or (ragged and lv >= 2 and rng.uniform() < 0.03)
                leaf.append(1 if is_leaf else 0)
                desc.append(d)
                weight.append(0.0 if (is_leaf and rng.uniform() < stop_frac) else float(rng.uniform(0.5, 9.0)))
                level.append(lv)
                if not is_leaf:
                    nxt.append(nid)
        frontier = nxt
    return dict(k=k, L=L, parent=np.array(parent, np.int32), leaf_flag=np.array(leaf, np.uint8),
                desc=np.stack(desc).astype(np.uint8), weight=np.array(weight, np.float64))


def synth_voc_features(voc, n=2000, seed=5):
    """Features near random leaves of the vocabulary (plus pure-noise features)."""
    rng = np.random.RandomState(seed)
    leaves = np.nonzero(voc["leaf_flag"])[0]
    f = voc["desc"][rng.choice(leaves, size=n)].copy()
    for i in range(n):
        for b in rng.choice(256, size=int(rng.randint(0, 40)), replace=False):
            f[i, b >> 3] ^= np.uint8(1 << (b & 7))
    noise = rng.uniform(size=n) < 0.1
    f[noise] = rng.randint(0, 256, size=(int(noise.sum()), 32)).astype(np.uint8)
    return f


def synth_local_ba_fast(n_kf=50, n_fixed=10, n_mp=5000, obs_per_mp=6, seed=42, mono_frac=0.0, outlier_frac=0.03,
                        fix_first=True, revisit=False):
    """Vectorised variant of synth_local_ba (same construction: KITTI-shaped forward path, points in the frustum of an
    anchor keyframe, the obs_per_mp observing keyframes nearest to it, noise ~ 1.2^octave, gross outliers, perturbed
    initial state, the same fix_first and revisit options) for callers that need many different windows quickly
    (bench.py).  Not stream-compatible with synth_local_ba: the parity tests keep that one."""
    rng = np.random.RandomState(seed)
    fx = fy = 718.856
    cx, cy, bf = 607.1928, 185.2157, 386.1448
    W, H = 1241, 376
    n_local = n_kf - n_fixed
    pos = _path_position(n_kf, revisit)
    yaw = np.deg2rad(rng.uniform(-2, 2, n_kf))
    c, s = np.cos(yaw), np.sin(yaw)
    R = np.zeros((n_kf, 3, 3))
    R[:, 0, 0] = c; R[:, 0, 2] = -s; R[:, 1, 1] = 1; R[:, 2, 0] = s; R[:, 2, 2] = c
    center = np.stack([rng.uniform(-0.1, 0.1, n_kf), rng.uniform(-0.05, 0.05, n_kf), 1.0 * pos], 1)
    t = -np.einsum("kij,kj->ki", R, center)
    pts = np.zeros((n_mp, 3))
    chosen = np.full((n_mp, obs_per_mp), -1, np.int64)
    todo = np.arange(n_mp)
    for _ in range(50):
        if len(todo) == 0:
            break
        m = len(todo)
        ka = rng.randint(0, n_kf, m)
        z = rng.uniform(5, 60, m)
        u = rng.uniform(50, W - 50, m)
        v = rng.uniform(30, H - 30, m)
        Xc = np.stack([(u - cx) * z / fx, (v - cy) * z / fy, z], 1)
        Xw = np.einsum("mji,mj->mi", R[ka], Xc - t[ka])
        Xk = np.einsum("kij,mj->mki", R, Xw) + t[None]          # m x n_kf x 3
        zz = Xk[..., 2]
        uu = fx * Xk[..., 0] / np.where(zz > 0, zz, 1) + cx
        vv = fy * Xk[..., 1] / np.where(zz > 0, zz, 1) + cy
        vis = (zz >= 2.0) & (uu > 0) & (uu < W) & (vv > 0) & (vv < H)
        ok = vis.sum(1) >= obs_per_mp
        dist = np.where(vis, np.abs(pos[None] - pos[ka][:, None]), 10 ** 6)
        near = np.sort(np.argsort(dist, 1, kind="stable")[:, :obs_per_mp], 1)
        pts[todo[ok]] = Xw[ok]
        chosen[todo[ok]] = near[ok]
        todo = todo[~ok]
    good = chosen[:, 0] >= 0
    pts, chosen = pts[good], chosen[good]
    n_mp = len(pts)
    kf = chosen.reshape(-1)
    mp = np.repeat(np.arange(n_mp), obs_per_mp)
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
    Tcw0 = np.zeros((n_kf, 4, 4))
    Tcw0[:, :3, :3] = R
    Tcw0[:, :3, 3] = t
    Tcw0[:, 3, 3] = 1
    dyaw = np.deg2rad(rng.normal(0, 0.2, n_local))
    dc, ds = np.cos(dyaw), np.sin(dyaw)
    dR = np.zeros((n_local, 3, 3))
    dR[:, 0, 0] = dc; dR[:, 0, 2] = -ds; dR[:, 1, 1] = 1; dR[:, 2, 0] = ds; dR[:, 2, 2] = dc
    Tcw0[:n_local, :3, :3] = np.einsum("kij,kjl->kil", dR, R[:n_local])
    Tcw0[:n_local, :3, 3] = np.einsum("kij,kj->ki", dR, t[:n_local]) + rng.normal(0, 0.02, (n_local, 3))
    pts0 = pts + rng.normal(0, 0.05, pts.shape)
    fixed = np.zeros(n_kf, np.uint8)
    fixed[n_local:] = 1
    if fix_first:
        fixed[0] = 1
    edge_dt = np.dtype([("kf", "i4"), ("mp", "i4"), ("obs", "f4", 3), ("inv_sigma2", "f4")])
    E = np.zeros(ne, edge_dt)
    E["kf"] = kf
    E["mp"] = mp
    E["obs"][:, 0] = (uu + noise[:, 0]).astype(np.float32)
    E["obs"][:, 1] = (vv + noise[:, 1]).astype(np.float32)
    E["obs"][:, 2] = np.where(mono, -1.0, ur + noise[:, 2]).astype(np.float32)
    E["inv_sigma2"] = (1.0 / (1.2 ** (2 * octv))).astype(np.float32)
    return dict(n_kf=n_kf, n_local=n_local, Tcw=Tcw0.astype(np.float32).reshape(n_kf, 16), fixed=fixed,
                points=pts0.astype(np.float32), edges=E, fx=np.float32(fx), fy=np.float32(fy), cx=np.float32(cx),
                cy=np.float32(cy), bf=np.float32(bf))


def synth_stereo_kitti(seed):
    """1241 x 376 stereo pair number `seed` (module-level so that process pools can pickle it)."""
    return synth_stereo(1241, 376, seed)
