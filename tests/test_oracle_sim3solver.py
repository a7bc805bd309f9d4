"""The Sim3 RANSAC's CPU restatement (oracle/sim3solver.cpp): its OpenCV operations pinned bit for bit against cv2 at
the shapes Sim3Solver.cc uses, SetRansacParameters' arithmetic at its edges, and its decisions on the loop candidates of
tests/synth_sim3solver.py."""
import numpy as np
import pytest

import sim3solver_binding as sb
from synth_sim3solver import CASES, problem, scene

cv2 = pytest.importorskip("cv2")


def test_reduce_norm_pow_gemm_match_cv2():
    rng = np.random.default_rng(0)
    for _ in range(2000):
        P = (rng.standard_normal((3, 3)) * rng.choice([1e-3, 1, 10, 1e3])).astype(np.float32)
        assert np.array_equal(sb.reduce_sum_cols(P), cv2.reduce(P, 1, cv2.REDUCE_SUM).ravel())
        B = rng.standard_normal((3, 3)).astype(np.float32)
        assert np.array_equal(sb.gemm_bt(P, B), cv2.gemm(P, B, 1, None, 0, flags=cv2.GEMM_2_T))  # Pr2*Pr1.t()
        x = (rng.standard_normal(3) * rng.choice([1e-6, 1, 100])).astype(np.float32)
        assert sb.norm(x) == cv2.norm(x.reshape(1, 3))
        assert np.array_equal(sb.pow2(P), cv2.pow(P, 2))
        c = rng.standard_normal((3, 1)).astype(np.float32)
        s = float(np.float32(rng.uniform(0.5, 2)))
        assert np.array_equal(sb.gemm(B, c, -s, c), cv2.gemm(B, c, -s, c, 1))  # O1 - s*R*O2


def _sym(rng, n=4):
    A = rng.standard_normal((n, n)).astype(np.float32)
    return (A + A.T).astype(np.float32)


def test_eigen_matches_cv2():
    """cv::eigen of a symmetric float 4 x 4: lapack.cpp's Jacobi (this cv2 has no Eigen backend), with its own float
    hypot, including repeated eigenvalues, already-diagonal input and the N matrices ComputeSim3 builds."""
    rng = np.random.default_rng(1)
    mats = [_sym(rng) * np.float32(rng.choice([1e-4, 1, 1e4])) for _ in range(2000)]
    mats += [np.diag(rng.standard_normal(4)).astype(np.float32) for _ in range(20)]
    mats += [np.eye(4, dtype=np.float32) * 3, np.zeros((4, 4), np.float32), np.diag([2, 2, -1, -1]).astype(np.float32)]
    for _ in range(50):  # repeated eigenvalues in a rotated basis
        Q = np.linalg.qr(rng.standard_normal((4, 4)))[0]
        mats.append((Q @ np.diag([5.0, 5.0, 1.0, 1.0]) @ Q.T).astype(np.float32))
    for _ in range(300):  # Horn's N from three random point pairs
        P1, P2 = rng.standard_normal((3, 3)).astype(np.float32), rng.standard_normal((3, 3)).astype(np.float32)
        M = sb.gemm_bt(P2 - P2.mean(1, keepdims=True), P1 - P1.mean(1, keepdims=True))
        N = np.array([[M[0, 0] + M[1, 1] + M[2, 2], M[1, 2] - M[2, 1], M[2, 0] - M[0, 2], M[0, 1] - M[1, 0]],
                      [0, M[0, 0] - M[1, 1] - M[2, 2], M[0, 1] + M[1, 0], M[2, 0] + M[0, 2]],
                      [0, 0, -M[0, 0] + M[1, 1] - M[2, 2], M[1, 2] + M[2, 1]],
                      [0, 0, 0, -M[0, 0] - M[1, 1] + M[2, 2]]], np.float32)
        mats.append(np.triu(N) + np.triu(N, 1).T)
    for A in mats:
        A = np.ascontiguousarray(A, np.float32)
        ok, w, v = cv2.eigen(A)
        ow, ov = sb.eigen(A)
        assert np.array_equal(ow, w.ravel()) and np.array_equal(ov, v)


def test_rodrigues_matches_cv2():
    """cv::Rodrigues: double arithmetic rounded once, near 0 (the theta < DBL_EPSILON identity branch) and near pi."""
    rng = np.random.default_rng(2)
    vs = []
    for scale in (1e-20, 1e-17, 1e-16, 1e-12, 1e-7, 1e-3, 0.5, 1, 2, 3):
        vs += list(rng.standard_normal((100, 3)) * scale)
    for _ in range(200):
        a = rng.standard_normal(3)
        vs.append(a / np.linalg.norm(a) * (np.pi - rng.uniform(0, 1e-3)))
        vs.append(a / np.linalg.norm(a) * np.pi)
    vs += [np.zeros(3), np.array([np.pi, 0, 0]), np.array([0, 0, -np.pi])]
    for v in vs:
        v = np.asarray(v, np.float32)
        assert np.array_equal(sb.rodrigues(v), cv2.Rodrigues(v.reshape(1, 3))[0]), v
    assert np.array_equal(sb.rodrigues(np.array([1e-17, 0, 0], np.float32)), np.eye(3, dtype=np.float32))


def test_dot_is_dot_prod():
    """Mat::dot (cv2 binds none): dotProd_'s double products, unrolled by 4, which dotProd_32f runs below one
    AVX-512 vector (16 floats)."""
    rng = np.random.default_rng(3)
    for n in (2, 9):
        for _ in range(200):
            a, b = rng.standard_normal(n).astype(np.float32), rng.standard_normal(n).astype(np.float32)
            p = a.astype(np.float64) * b.astype(np.float64)
            want = 0.0
            i = 0
            while i + 4 <= n:
                want += p[i] + p[i + 1] + p[i + 2] + p[i + 3]
                i += 4
            for j in range(i, n):
                want += p[j]
            assert sb.dot(a, b) == want


@pytest.mark.parametrize("n,p,mi,mx", [
    (100, 0.99, 20, 300), (20, 0.99, 20, 300), (21, 0.99, 20, 300), (19, 0.99, 20, 300), (0, 0.99, 20, 300),
    (0, 0.99, 0, 300), (50, 0.99, 0, 300), (1000, 0.99, 20, 300), (1000, 0.99, 6, 300), (30, 1.0, 20, 300),
    (30, 0.0, 20, 300), (30, 0.5, 29, 300), (300, 0.99, 299, 5), (40, 0.99, 20, 1), (40, 0.99, 20, 0),
    (40, 0.99, 20, -3), (7, 0.99, 6, 300), (10 ** 6, 0.99, 3, 10 ** 9), (3, 0.99, 2, 300)])
def test_ransac_parameters_at_the_edges(pkg, n, p, mi, mx):
    """SetRansacParameters: epsilon a float, the count in double, NaN / infinite counts through x86's int conversion,
    minInliers == N giving 1, max(1, min(count, maxIterations))."""
    want = sb.ransac_max_its(n, p, mi, mx)
    assert pkg.sim3_ransac_max_its(n, p, mi, mx) == want
    assert want >= 1


def test_ransac_parameters_sweep(pkg):
    for n in range(0, 400, 7):
        for mi in (0, 3, 6, 20, 50, n):
            for p in (0.5, 0.9, 0.99, 0.999):
                assert pkg.sim3_ransac_max_its(n, p, mi, 300) == sb.ransac_max_its(n, p, mi, 300), (n, mi, p)


def test_degenerate_sets():
    """Repeated points, collinear points and an exact identity go through Horn's closed form unguarded; the exact
    identity gives a NaN model, as the reference does."""
    rng = np.random.default_rng(4)
    X = rng.uniform(1, 5, (3, 3)).astype(np.float32)
    dup = X.copy()
    dup[:, 2] = dup[:, 0]
    h = sb.compute_sim3(dup, dup, False)  # two equal points: still Horn's closed form, no guard
    assert h["T12"][3].tolist() == [0, 0, 0, 1]
    same = sb.compute_sim3(X, X, False)  # q = (1, 0, 0, 0): norm(vec) = 0, so vec = 0 * inf
    assert np.isnan(same["R"]).all() and np.isnan(same["T12"][:3]).all()
    line = np.stack([X[:, 0], X[:, 0] * 2, X[:, 0] * 3], 1).astype(np.float32)
    h = sb.compute_sim3(line, line, True)
    assert h["s"] == 1.0


def check_case(name):
    kw, (p, mi, mx) = CASES[name]
    sc = scene(**kw)
    pr = problem(sc, mi)
    pr["max_its"] = sb.ransac_max_its(len(pr["X1c"]), p, mi, mx)
    return sc, pr


@pytest.mark.parametrize("case", sorted(CASES))
def test_oracle_cases(case):
    sc, pr = check_case(case)
    rng = np.random.default_rng(7)
    n = len(pr["X1c"])
    k = pr["max_its"] if n >= pr["min_inliers"] else 0
    sets = np.array([rng.choice(n, 3, replace=False) for _ in range(k)], np.int32).reshape(-1, 3)
    r, margin = sb.oracle(pr, (0, 0), sets)
    assert margin > 1e-6  # no error within rounding of its threshold
    if n < pr["min_inliers"]:
        assert r["no_more"] and not r["returned"] and r["iterations_used"] == 0
    elif case.startswith("loop"):
        assert r["returned"] and r["n_inliers"] > pr["min_inliers"]
        s, R, t = sc["S"]
        # a model from three noisy points, close to the scene's
        assert np.abs(r["R"] - R).max() < 0.06
        assert abs(float(r["s"]) - s) < 0.08
        # the inliers are (nearly all) true matches
        assert (r["inliers"] & sc["true_wrong"][pr["indices1"]]).sum() <= 0.02 * r["n_inliers"]
    elif case.startswith("outliers"):
        assert not r["returned"] and r["no_more"] and r["iterations_done"] == pr["max_its"]
    if case == "min_equals_n":
        assert pr["max_its"] == 1
