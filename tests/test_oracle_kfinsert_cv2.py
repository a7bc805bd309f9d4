"""Pins the OpenCV primitives MapPoint::UpdateNormalAndDepth is restated with (oracle/kfinsert.cpp, csrc/mappoint.cu,
refshim_cv_kfinsert.h) against cv2, bit for bit.  `normal + normali/norm(normali)` is a
MatOp_AddEx with alpha = 1/norm and beta = 1, which OpenCV evaluates with cv::scaleAdd (read from its source; cv2 binds no
MatExpr); `normal/n` is convertTo with the scale rounded to float, the arithmetic of scaleAdd with a zero addend."""
import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")


def vectors(seed, n):
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal((n, 3)) * rng.choice([1e-3, 1, 10, 1e3], (n, 1))).astype(np.float32)
    y = (rng.standard_normal((n, 3)) * rng.choice([1e-3, 1, 10], (n, 1))).astype(np.float32)
    return x, y, rng.uniform(1e-2, 1e4, n)


def test_scale_add_is_fused_with_alpha_rounded_to_float():
    x, y, s = vectors(1, 5000)
    fused = two_roundings = 0
    for i in range(len(x)):
        a = np.float32(1.0 / s[i])
        got = cv2.scaleAdd(x[i].reshape(3, 1), 1.0 / s[i], y[i].reshape(3, 1)).ravel()
        want = (x[i].astype(np.float64) * np.float64(a) + y[i]).astype(np.float32)  # exact product, one rounding
        fused += np.array_equal(got.view(np.uint32), want.view(np.uint32))
        two_roundings += np.array_equal(got.view(np.uint32), (x[i] * a + y[i]).view(np.uint32))
    assert fused == len(x)
    assert two_roundings < len(x)  # the inputs tell the forms apart


def test_add_weighted_is_another_form():
    """addWeighted computes in double and rounds once: it is not the form `normal + normali/s` takes."""
    x, y, s = vectors(2, 2000)
    differ = 0
    for i in range(len(x)):
        got = cv2.addWeighted(x[i].reshape(3, 1), 1.0 / s[i], y[i].reshape(3, 1), 1, 0).ravel()
        want = (x[i].astype(np.float64) * (1.0 / s[i]) + y[i]).astype(np.float32)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
        a = np.float32(1.0 / s[i])
        differ += not np.array_equal(got.view(np.uint32),
                                     (x[i].astype(np.float64) * np.float64(a) + y[i]).astype(np.float32).view(np.uint32))
    assert differ > 0


def test_scale_by_float_scalar():
    x, _, _ = vectors(3, 3000)
    for i, n in enumerate(np.resize(np.arange(1, 300), len(x))):
        a = np.float32(1.0 / n)
        got = cv2.scaleAdd(x[i].reshape(3, 1), 1.0 / n, np.zeros((3, 1), np.float32)).ravel()
        assert np.array_equal(got.view(np.uint32), (x[i] * a + np.float32(0)).view(np.uint32))


def test_norm_of_a_column_sums_in_order():
    """mWorldPos - Owi is a 3 x 1 column: cv::norm sums its squares in double in order (a 1 x 3 row, as in Sim3Solver,
    takes two lanes, (x0^2 + x2^2) + x1^2)."""
    x, _, _ = vectors(4, 5000)
    for v in x:
        d = v.astype(np.float64)
        assert cv2.norm(v.reshape(3, 1)) == np.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2])
