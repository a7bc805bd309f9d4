"""The drop-in Frame (self_commit_orb-slam2_b200/host/adapters/Frame_b200.cc over the drop-in ORBextractor and
libb200slam.so) against the reference's own src/Frame.cc, on the same inputs and through the same glue
(oracle/ref_frame_seq_glue.cpp, oracle/frame.mk).  Every member the later stages read must be identical, floats compared
as bits: N, mvKeys / mvKeysUn / mvKeysRight, both descriptor matrices, mvuRight, mvDepth, mb, mbf, mThDepth, the scale
tables, the static calibration, bounds and grid constants, and every cell of mGrid.

  * stereo pairs of tests/synth.py at 1241 x 376 (KITTI), 752 x 480 and 640 x 480 (EuRoC), one calibration with k1 != 0,
    and a right image with its own row stride;
  * RGB-D at 640 x 480 with the TUM1 calibration and depth images holding 0, negatives, NaN and inf;
  * monocular TUM1 with five and four coefficients and with k1 == 0, and the initialisation extractor (2 x nFeatures);
  * sequences: mnId, the first-frame-only computations, the copy constructor;
  * GetFeaturesInArea, isInFrustum and UnprojectStereo;
  * the refused stereo pairs (one stderr line, N = 0) and the pyramid that is never downloaded.

The reference runs on the glue's bump allocator, so its extraction breaks DistributeOctTree's ties the way the device
does (tests/test_oracle_reference_extractor.py)."""
import os

import numpy as np
import pytest

import frame_binding as fb
from synth import synth_image, synth_stereo

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not (os.path.exists(fb.REF_LIB) and os.path.exists(fb.ADAPTER_LIB)),
                                 reason="oracle/_ref not built (needs the reference's sources: make -f oracle/frame.mk)")]


@pytest.fixture(scope="module")
def libs(pkg):
    if pkg.device_count() < 1:
        pytest.skip("no CUDA device")
    return fb.FrameLib(fb.REF_LIB, monotonic=1), fb.FrameLib(fb.ADAPTER_LIB, monotonic=0)


def _both(libs, build):
    """build(lib) on both libraries after a reset; returns the two results"""
    out = []
    for L in libs:
        L.reset()
        out.append(build(L))
    return out


def _same_statics(libs):
    (sa, na, ia), (sb, nb, ib) = libs[0].statics(), libs[1].statics()
    assert np.array_equal(fb.bits(sa), fb.bits(sb)), (sa, sb)
    assert (na, ia) == (nb, ib)
    return sa


def _same_grid(libs, fa, fb_):
    ca, ia = libs[0].grid(fa)
    cb, ib = libs[1].grid(fb_)
    assert np.array_equal(ca, cb) and np.array_equal(ia, ib)
    return ca


def _stereo(L, name, imL, imR):
    K4, dist, bf, th, nf = fb.STEREO[name]
    ex_l, ex_r = L.extractor(nf), L.extractor(nf)
    return L.stereo(ex_l, ex_r, imL, imR, K4, dist, bf, th)


@pytest.mark.parametrize("name,w,h,seed", [("kitti", 1241, 376, 3), ("kitti", 1241, 376, 11), ("euroc", 752, 480, 21),
                                           ("euroc", 752, 480, 5), ("euroc", 640, 480, 9), ("euroc_raw", 752, 480, 7)])
def test_stereo_frame_equals_reference(libs, name, w, h, seed):
    imL, imR = synth_stereo(w, h, seed)
    fa, fb_ = _both(libs, lambda L: _stereo(L, name, imL, imR))
    A, B = libs[0].frame(fa), libs[1].frame(fb_)
    fb.assert_same_frame(A, B)
    nf = fb.STEREO[name][4]
    assert A["N"] > 0.8 * nf and len(A["mvKeysRight"]) > 0.8 * nf
    assert (A["mvuRight"] >= 0).sum() > 100  # the stereo search found matches
    assert A["mb"][0] == np.float32(np.float32(fb.STEREO[name][2]) / np.float32(fb.STEREO[name][0][0]))
    s = _same_statics(libs)
    if fb.STEREO[name][1][0] != 0:  # undistorted keypoints and bounds
        assert not np.array_equal(A["mvKeysUn"][:, :2], A["mvKeys"][:, :2]) and s[6] != 0
    assert _same_grid(libs, fa, fb_).sum() > 0


def test_stereo_right_image_with_its_own_stride(libs):
    """The right image is a view into a wider buffer: the drop-in packs it to the left image's stride."""
    imL, imR = synth_stereo(1241, 376, 4)
    wide = np.zeros((376, 1300), np.uint8)
    wide[:, :1241] = imR
    fa, fb_ = _both(libs, lambda L: _stereo(L, "kitti", imL, wide[:, :1241]))
    A, B = libs[0].frame(fa), libs[1].frame(fb_)
    fb.assert_same_frame(A, B)
    assert A["N"] > 1000
    _same_grid(libs, fa, fb_)


@pytest.mark.parametrize("name", ["tum1", "tum1_4"])
@pytest.mark.parametrize("seed", [31, 8])
def test_rgbd_frame_equals_reference(libs, name, seed):
    import undistort_binding as ub
    K4, dist = fb.MONO[name]
    img = synth_image(640, 480, seed)
    depth = ub.depth_image(640, 480, seed=seed + 1)  # blocks of 0, -1.5, NaN, inf and -0
    fa, fb_ = _both(libs, lambda L: L.mono_rgbd(L.extractor(1000), img, K4, dist, 40.0, 40.0, depth=depth))
    A, B = libs[0].frame(fa), libs[1].frame(fb_)
    fb.assert_same_frame(A, B)
    assert A["N"] > 800 and (A["mvDepth"] == -1).sum() > 10 and (A["mvDepth"] > 0).sum() > 500
    _same_statics(libs)
    _same_grid(libs, fa, fb_)


@pytest.mark.parametrize("name,nf", [("tum1", 1000), ("tum1_4", 1000), ("k1zero", 1000), ("tum1", 2000)])
def test_monocular_frame_equals_reference(libs, name, nf):
    """nf = 2000: Tracking's initialisation extractor (2 x nFeatures, src/Tracking.cc:191-192)"""
    K4, dist = fb.MONO[name]
    img = synth_image(640, 480, 17)
    fa, fb_ = _both(libs, lambda L: L.mono_rgbd(L.extractor(nf), img, K4, dist, 40.0, 40.0))
    A, B = libs[0].frame(fa), libs[1].frame(fb_)
    fb.assert_same_frame(A, B)
    assert A["N"] > 0.8 * nf and np.all(A["mvuRight"] == -1) and np.all(A["mvDepth"] == -1)
    if name == "k1zero":
        assert np.array_equal(A["mvKeysUn"], A["mvKeys"])
    _same_statics(libs)
    _same_grid(libs, fa, fb_)


def test_sequence_ids_first_frame_computations_and_copies(libs):
    """Stereo frames in a row, then one with another calibration: mnId counts up, the calibration and bounds stay the
    first frame's; copies (one made after SetPose) equal their originals in both libraries."""
    pairs = [synth_stereo(752, 480, s) for s in (40, 41, 42)]
    K4r, distr, bf, th, nf = fb.STEREO["euroc_raw"]
    K4, dist = fb.STEREO["euroc"][0], fb.STEREO["euroc"][1]

    def run(L):
        exl, exr = L.extractor(nf), L.extractor(nf)
        ids = [L.stereo(exl, exr, a, b, K4r, distr, bf, th) for a, b in pairs[:2]]
        s_first = L.statics()
        ids.append(L.stereo(exl, exr, pairs[2][0], pairs[2][1], K4, dist, bf, th))  # another calibration
        ids.append(L.copy(ids[1]))
        T = np.eye(4, dtype=np.float32)
        T[:3, 3] = (0.1, -0.2, 0.3)
        L.is_in_frustum(ids[0], T, np.zeros((1, 3)), np.float32([[0, 0, 1]]), [0.1], [10.0], 0.5)  # SetPose
        ids.append(L.copy(ids[0]))
        return ids, s_first

    (ia, sa), (ib, sb) = _both(libs, run)
    assert np.array_equal(fb.bits(sa[0]), fb.bits(sb[0])) and sa[1:] == sb[1:] == (2, 0)
    assert sa[0][6] != 0  # the distorted first calibration moved the bounds
    s = _same_statics(libs)
    assert np.array_equal(fb.bits(s), fb.bits(sa[0]))  # the third frame changed none of them
    assert libs[0].statics()[1] == 3
    frames = [(libs[0].frame(a), libs[1].frame(b)) for a, b in zip(ia, ib)]
    for (A, B), want_id in zip(frames, [0, 1, 2, 1, 0]):
        fb.assert_same_frame(A, B)
        assert A["mnId"] == want_id
    fb.assert_same_frame(frames[3][1], frames[1][1])  # a copy equals its original
    for f in range(len(ia)):
        _same_grid(libs, ia[f], ib[f])
    # the copy made after SetPose carries the pose: UnprojectStereo on it
    n_ok = 0
    for i in range(0, frames[4][0]["N"], 7):
        ra, rb = libs[0].unproject(ia[4], i), libs[1].unproject(ib[4], i)
        assert (ra is None) == (rb is None)
        if ra is not None:
            assert np.array_equal(fb.bits(ra), fb.bits(rb))
            n_ok += 1
    assert n_ok > 20


def test_monocular_sequence_keeps_the_first_bounds(libs):
    img0, img1 = synth_image(640, 480, 50), synth_image(640, 480, 51)

    def run(L):
        ex = L.extractor(1000)
        a = L.mono_rgbd(ex, img0, *fb.MONO["tum1"], 40.0, 40.0)
        b = L.mono_rgbd(ex, img1, *fb.MONO["k1zero"], 40.0, 40.0)
        return a, b

    (a0, a1), (b0, b1) = _both(libs, run)
    for a, b in ((a0, b0), (a1, b1)):
        fb.assert_same_frame(libs[0].frame(a), libs[1].frame(b))
        _same_grid(libs, a, b)
    s = _same_statics(libs)
    assert s[6] != 0.0 and libs[1].statics()[1:] == (2, 0)


def test_queries_equal_reference(libs):
    """GetFeaturesInArea (600 queries), isInFrustum and UnprojectStereo on a KITTI stereo frame."""
    imL, imR = synth_stereo(1241, 376, 5)
    fa, fb_ = _both(libs, lambda L: _stereo(L, "kitti", imL, imR))
    A = libs[0].frame(fa)
    rng = np.random.RandomState(3)
    W, H = 1241, 376
    total = 0
    for t in range(600):
        if t % 3 == 0:
            j = rng.randint(0, A["N"])
            x, y = float(A["mvKeys"][j, 0]) + rng.uniform(-3, 3), float(A["mvKeys"][j, 1]) + rng.uniform(-3, 3)
        else:
            x, y = rng.uniform(-60, W + 60), rng.uniform(-60, H + 60)
        r = float(rng.choice([2.5, 7.0, 15.0, 40.0, 120.0]))
        lo, hi = [(-1, -1), (0, 3), (2, -1), (3, 4), (0, 0), (1, 7)][rng.randint(0, 6)]
        ra, rb = libs[0].features_in_area(fa, x, y, r, lo, hi), libs[1].features_in_area(fb_, x, y, r, lo, hi)
        assert np.array_equal(ra, rb)
        total += len(ra)
    assert total > 5000
    # map points near the features, some behind the camera, some out of range, some seen from behind
    K4, _, bf, _, _ = fb.STEREO["kitti"]
    fx, fy, cx, cy = K4
    n = 2000
    ang = 0.02
    Rm = np.array([[np.cos(ang), 0, np.sin(ang)], [0, 1, 0], [-np.sin(ang), 0, np.cos(ang)]])
    t = np.array([0.2, -0.1, 0.4])
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = Rm, t
    src = rng.randint(0, A["N"], size=n)
    z = rng.uniform(3, 50, n)
    u = A["mvKeys"][src, 0] + rng.normal(0, 1.5, n)
    v = A["mvKeys"][src, 1] + rng.normal(0, 1.0, n)
    Xc = np.stack([(u - cx) * z / fx, (v - cy) * z / fy, z], 1)
    Xw = (Rm.T @ (Xc - t).T).T
    Ow = -Rm.T @ t
    dist = np.linalg.norm(Xw - Ow, axis=1)
    nrm = (Xw - Ow) / dist[:, None] + rng.normal(0, 0.35, (n, 3))
    nrm /= np.linalg.norm(nrm, axis=1)[:, None]
    nrm[rng.randint(0, 100, size=n) < 5] *= -1
    maxd = (dist * 1.2 ** rng.randint(0, 8, n) * rng.uniform(0.8, 1.0, n)).astype(np.float32)
    mind = (maxd / 1.2 ** 7).astype(np.float32)
    behind = rng.randint(0, 100, size=n) < 3
    Xw[behind] = Ow + (Ow - Xw[behind])
    oa = libs[0].is_in_frustum(fa, T, Xw, nrm, mind, maxd, 0.5)
    ob = libs[1].is_in_frustum(fb_, T, Xw, nrm, mind, maxd, 0.5)
    assert np.array_equal(oa[2], ob[2]) and 0.3 * n < oa[2].sum() < n
    assert np.array_equal(fb.bits(oa[0]), fb.bits(ob[0])) and np.array_equal(oa[1], ob[1])
    n_ok = 0
    for i in range(A["N"]):
        ra, rb = libs[0].unproject(fa, i), libs[1].unproject(fb_, i)
        assert (ra is None) == (rb is None)
        if ra is not None:
            assert np.array_equal(fb.bits(ra), fb.bits(rb))
            n_ok += 1
    assert n_ok > 100


def test_refused_stereo_pairs_give_an_empty_frame(libs, capfd):
    """A right extractor with other parameters, or images of different sizes: one stderr line and N = 0; the next
    frame is built normally."""
    L = libs[1]
    L.reset()
    K4, dist, bf, th, nf = fb.STEREO["kitti"]
    imL, imR = synth_stereo(1241, 376, 3)
    exl, exr_other = L.extractor(nf), L.extractor(nf + 100)
    capfd.readouterr()
    f0 = L.stereo(exl, exr_other, imL, imR, K4, dist, bf, th)
    err = capfd.readouterr().err
    assert len(err.strip().splitlines()) == 1 and "Frame" in err, err
    f1 = L.stereo(exl, L.extractor(nf), imL, np.ascontiguousarray(imR[:300]), K4, dist, bf, th)
    err = capfd.readouterr().err
    assert len(err.strip().splitlines()) == 1 and "Frame" in err, err
    for f, want_id in ((f0, 0), (f1, 1)):
        F = L.frame(f)
        assert F["N"] == 0 and F["mnId"] == want_id and np.all(F["sizes"] == 0)
        assert len(F["mDescriptors"]) == 0 and len(F["mDescriptorsRight"]) == 0
    assert L.statics()[2] == 1  # no first-frame computations yet
    f2 = L.stereo(exl, L.extractor(nf), imL, imR, K4, dist, bf, th)
    F = L.frame(f2)
    assert F["N"] > 1000 and F["mnId"] == 2 and L.statics()[2] == 0
    assert capfd.readouterr().err == ""


def test_drop_in_frames_never_download_the_pyramid(libs):
    """After stereo, RGB-D and monocular drop-in frames, no level of any extractor's mvImagePyramid was written (the
    reference's extractors fill theirs)."""
    imL, imR = synth_stereo(1241, 376, 3)
    img = synth_image(640, 480, 31)

    def run(L):
        K4, dist, bf, th, nf = fb.STEREO["kitti"]
        exs = [L.extractor(nf), L.extractor(nf), L.extractor(1000), L.extractor(1000)]
        L.stereo(exs[0], exs[1], imL, imR, K4, dist, bf, th)
        L.mono_rgbd(exs[2], img, *fb.MONO["tum1"], 40.0, 40.0, depth=np.ones((480, 640), np.float32))
        L.mono_rgbd(exs[3], img, *fb.MONO["tum1"], 40.0, 40.0)
        return [L.pyramid(e) for e in exs]

    ref, drop_in = _both(libs, run)
    assert all(len(p) == 8 for p in ref + drop_in)
    assert ref[0][0] == (1241, 376) and all(w > 0 for p in ref for w, _ in p)
    assert all(wh == (0, 0) for p in drop_in for wh in p)
