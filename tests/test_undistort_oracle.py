"""Pins the undistortion and RGB-D depth recipes on the CPU.

  * orc_undistort_points (oracle/orb_undistort.cpp) and the numpy restatement equal cv2.undistortPoints(pts, K, D, P=K)
    bit for bit: the TUM fr1 / fr2 / fr3 and EuRoC calibrations with 4 and 5 coefficients, points over the whole image,
    the corners, points outside the image, a strong barrel model that takes OpenCV 4's icdist < 0 exit, and +-0.
  * The reference's own monocular and RGB-D Frame constructors (src/Frame.cc:238-458, compiled in place with
    refshim/refshim_cv_undistort.h, whose undistortPoints is the restatement) equal the restatement plus a numpy ComputeStereoFromRGBD: every mvKeysUn bit,
    mvuRight / mvDepth and the four image bounds; GetFeaturesInArea equals the oracle's grid over those bounds."""
import ctypes
import os

import numpy as np
import pytest

import undistort_binding as ub
from synth import synth_image

cv2 = pytest.importorskip("cv2")
NAMES = ["tum1", "tum1_4", "tum2", "tum2_4", "tum3", "euroc", "euroc_5", "k1zero_p1", "pincushion", "barrel"]


@pytest.fixture(scope="module")
def orc():
    return ub.Oracle()


def _points(w=640, h=480, seed=0):
    rng = np.random.default_rng(seed)
    gx, gy = np.meshgrid(np.arange(0, w + 1, 8, dtype=np.float32), np.arange(0, h + 1, 8, dtype=np.float32))
    grid = np.stack([gx.ravel(), gy.ravel()], 1)
    inside = rng.uniform([0, 0], [w, h], (20000, 2)).astype(np.float32)
    outside = rng.uniform([-0.5 * w, -0.5 * h], [1.5 * w, 1.5 * h], (5000, 2)).astype(np.float32)
    corners = np.float32([[0, 0], [w, 0], [0, h], [w, h]])
    zeros = np.float32([[0.0, 0.0], [-0.0, 0.0], [0.0, -0.0], [-0.0, -0.0], [-0.0, 240.0], [320.0, -0.0]])
    return np.concatenate([grid, inside, outside, corners, zeros])


def _cv2(xy, K4, dist):
    return cv2.undistortPoints(xy.reshape(-1, 1, 2), ub.K33(K4), dist, P=ub.K33(K4)).reshape(-1, 2)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("name", NAMES)
def test_restatement_equals_cv2(orc, name):
    K4, dist = ub.calib(name)
    xy = _points(seed=NAMES.index(name))
    ref = _cv2(xy, K4, dist)
    assert np.array_equal(_bits(orc.undistort(xy, K4, dist)), _bits(ref))
    assert np.array_equal(_bits(ub.np_undistort(xy, K4, dist)), _bits(ref))


def test_barrel_model_takes_the_icdist_exit(orc):
    """The synthetic barrel model reaches OpenCV 4's `icdist < 0` branch (absent from OpenCV 3.2) for part of the points
    and the restatement follows it there."""
    K4, dist = ub.calib("barrel")
    xy = _points(seed=3)
    out, early = ub.np_undistort(xy, K4, dist, count_early=True)
    assert 100 < early < len(xy) - 100
    assert np.array_equal(_bits(orc.undistort(xy, K4, dist)), _bits(_cv2(xy, K4, dist)))


def test_in_place_and_1241x376(orc):
    K4, dist = ub.calib("euroc")
    xy = _points(1241, 376, seed=5)
    ref = _cv2(xy, K4, dist)
    buf = np.ascontiguousarray(xy.copy())
    orc.L.orc_undistort_points(buf.ctypes.data, len(buf), K4.ctypes.data, dist.ctypes.data, len(dist), buf.ctypes.data)
    assert np.array_equal(_bits(buf), _bits(ref))


# ---------------------------------------------------------------- the reference's own monocular / RGB-D Frame
needs_ref = pytest.mark.skipif(not os.path.exists(ub.REF_LIB), reason="oracle/_ref not built (make -C oracle ref)")


def _check_frame(orc, F, K4, dist, w, h, depth=None, bf=40.0):
    assert F.N > 200
    # UndistortKeyPoints: only x, y change; k1 == 0 copies the keypoints
    for f in ("size", "angle", "response", "octave", "class_id"):
        assert np.array_equal(F.kps_un[f], F.kps[f]), f
    xy = np.stack([F.kps["x"], F.kps["y"]], 1)
    un = orc.undistort(xy, K4, dist) if dist[0] != 0 else xy
    assert np.array_equal(_bits(np.stack([F.kps_un["x"], F.kps_un["y"]], 1)), _bits(un))
    # ComputeImageBounds
    assert np.array_equal(_bits(F.bounds), _bits(ub.image_bounds(w, h, K4, dist, orc.undistort)))
    if depth is None:
        assert (F.uright == -1).all() and (F.depth == -1).all()
    else:
        ur, dd = ub.np_stereo_from_depth(F.kps, F.kps_un, depth, bf)
        assert np.array_equal(_bits(F.uright), _bits(ur)) and np.array_equal(_bits(F.depth), _bits(dd))


@needs_ref
@pytest.mark.parametrize("name", ["tum1", "tum2_4", "tum3", "euroc", "k1zero_p1", "barrel"])
def test_reference_monocular_frame(orc, name):
    K4, dist = ub.calib(name)
    img = synth_image(640, 480, 11)
    F = ub.RefMonoFrame(img, K4, dist, nf=1500)
    _check_frame(orc, F, K4, dist, 640, 480)
    if name == "k1zero_p1":  # p1, p2 != 0 but k1 == 0: not undistorted by the frame, undistorted by cv::undistortPoints
        xy = np.stack([F.kps["x"], F.kps["y"]], 1)
        assert not np.array_equal(orc.undistort(xy, K4, dist), xy)


@needs_ref
@pytest.mark.parametrize("name", ["tum1", "tum2", "tum3", "euroc_5", "k1zero_p1", "pincushion"])
def test_reference_rgbd_frame(orc, name):
    """Depth 0, -1.5, -0, NaN and +inf at keypoints."""
    K4, dist = ub.calib(name)
    w, h = 640, 480
    img = synth_image(w, h, 12)
    depth = ub.depth_image(w, h, seed=7)
    F = ub.RefMonoFrame(img, K4, dist, depth=depth, nf=2000)
    _check_frame(orc, F, K4, dist, w, h, depth=depth)
    d = depth[F.kps["y"].astype(int), F.kps["x"].astype(int)]
    for special in (lambda a: a == 0, lambda a: a < 0, np.isnan, np.isposinf):
        assert special(d).any()
    assert (F.depth == -1).any() and np.isposinf(F.depth).any()


@needs_ref
def test_reference_frame_keypoints_equal_the_oracle_extractor():
    """On the bump allocator the reference frame's mvKeys are the oracle extractor's keypoints (what the device extractor
    reproduces), whatever the calibration: the device chain can be compared with the reference's RGB-D Frame."""
    import oracle_binding
    img = synth_image(640, 480, 31)
    k, _ = oracle_binding.load().extractor(2000, 1.2, 8, 20, 7)(img)
    for name in ("tum1", "pincushion"):
        K4, dist = ub.calib(name)
        F = ub.RefMonoFrame(img, K4, dist, depth=ub.depth_image(640, 480, seed=9), nf=2000)
        assert F.N == len(k)
        for f in ("x", "y", "size", "angle", "response", "octave"):
            assert np.array_equal(F.kps[f], k[f]), f


def _oracle_grid_query(L, kps_un, bounds, x, y, r, lo, hi):
    import oracle_binding  # the oracle's Frame grid (orc_features_in_area)
    L.orc_features_in_area.argtypes = [ctypes.c_void_p] * 5 + [ctypes.c_float] * 3 + [ctypes.c_int] * 2 + [ctypes.c_void_p,
                                                                                                           ctypes.c_int]
    kx, ky = np.ascontiguousarray(kps_un["x"]), np.ascontiguousarray(kps_un["y"])
    oc = np.ascontiguousarray(kps_un["octave"])
    sf = np.float32(1.2) ** np.arange(8, dtype=np.float32)
    g = oracle_binding.FrameGeom(bounds[0], bounds[2], bounds[1], bounds[3], 40.0, sf.ctypes.data, 8)
    out = np.zeros(len(kx) + 1, np.int32)
    n = L.orc_features_in_area(kx.ctypes.data, ky.ctypes.data, oc.ctypes.data, len(kx), ctypes.byref(g), x, y, r, lo, hi,
                               out.ctypes.data, len(out))
    return out[:n].copy()


@needs_ref
@pytest.mark.parametrize("name", ["tum1", "euroc", "pincushion"])
def test_reference_grid_over_undistorted_bounds(name):
    """The reference's grid (AssignFeaturesToGrid over the undistorted bounds, GetFeaturesInArea) equals the oracle's
    grid on the same mvKeysUn and bounds, including the keypoints PosInGrid drops."""
    K4, dist = ub.calib(name)
    w, h = 640, 480
    grid_oracle = ctypes.CDLL(ub.GRID_ORACLE_LIB)
    F = ub.RefMonoFrame(synth_image(w, h, 13), K4, dist, depth=ub.depth_image(w, h, seed=8), nf=2000)
    x, y = F.kps_un["x"], F.kps_un["y"]
    mnMinX, mnMaxX, mnMinY, mnMaxY = F.bounds
    outside = (x < mnMinX) | (x >= mnMaxX) | (y < mnMinY) | (y >= mnMaxY)
    if name == "pincushion":
        assert outside.any()
    rng = np.random.default_rng(2)
    for _ in range(300):
        qx, qy = float(rng.uniform(mnMinX - 40, mnMaxX + 40)), float(rng.uniform(mnMinY - 40, mnMaxY + 40))
        r = float(rng.choice([3.0, 15.0, 60.0, 200.0]))
        lo, hi = [(-1, -1), (0, 2), (1, -1)][rng.integers(3)]
        a = F.features_in_area(qx, qy, r, lo, hi)
        b = _oracle_grid_query(grid_oracle, F.kps_un, F.bounds, qx, qy, r, lo, hi)
        assert np.array_equal(a, b)


def test_entry_points_without_a_device(pkg):
    """No handle can exist without a device; each entry point then fails with B2S_ERR_NO_DEVICE, never on the CPU."""
    if pkg.device_count() > 0:
        pytest.skip("a CUDA device is present")
    L = pkg.lib()
    K4, dist = ub.calib("tum1")
    xy = np.float32([[1, 2]])
    out = np.zeros_like(xy)
    assert L.b2s_undistort_points(None, xy.ctypes.data, 1, K4.ctypes.data, dist.ctypes.data, 5,
                                  out.ctypes.data) == pkg.ERR_NO_DEVICE
    assert L.b2s_undistort_keypoints_device(None, None, None, 1, 1, K4.ctypes.data, dist.ctypes.data, 5, None,
                                            None) == pkg.ERR_NO_DEVICE
    assert L.b2s_stereo_from_depth_device(None, None, None, None, 1, 1, None, 2560, 640, 480, 40.0, None, None,
                                          None) == pkg.ERR_NO_DEVICE
    assert (out == 0).all()
