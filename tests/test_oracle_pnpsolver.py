"""The OpenCV C API operations EPnP calls, as the restatement (oracle/pnpsolver.cpp) computes them, pinned bit for bit
against cv2 on CV_64F data: cvMulTransposed (MulTransposedR's serial sums), cvSVD (JacobiSVDImpl_<double> with
lapack.cpp's hypot template, including the basis completion of rank-deficient input), cvInvert and cvSolve with CV_SVD;
then SetRansacParameters (pkg.pnp_ransac_parameters against the restatement) and the scene decisions."""
import importlib

import numpy as np
import pytest

import pnpsolver_binding as pb
import synth_pnp as sp

cv2 = pytest.importorskip("cv2")
pkg = importlib.import_module("self_commit_orb-slam2_b200")


def fill_M(rng, n):
    """A 2n x 12 matrix with fill_M's zero pattern."""
    M = np.zeros((2 * n, 12))
    a = rng.normal(size=(n, 4))
    u, v = rng.uniform(0, 640, n), rng.uniform(0, 480, n)
    for j in range(4):
        M[0::2, 3 * j] = a[:, j] * 520.0
        M[0::2, 3 * j + 2] = a[:, j] * (320.5 - u)
        M[1::2, 3 * j + 1] = a[:, j] * 518.0
        M[1::2, 3 * j + 2] = a[:, j] * (240.25 - v)
    return M


@pytest.mark.parametrize("n", [4, 5, 17, 100, 1000, 4000])
def test_mul_transposed(n):
    rng = np.random.default_rng(n)
    for A in (rng.normal(size=(n, 3)) * 3.0, fill_M(rng, n)):
        assert np.array_equal(pb.mul_transposed(A), cv2.mulTransposed(A, True))


def svd_inputs():
    rng = np.random.default_rng(7)
    out = [rng.normal(size=(12, 12)) for _ in range(4)]
    for n in (4, 5, 9, 39):  # M^T M of n points: rank <= 8 at n = 4
        out.append(cv2.mulTransposed(fill_M(rng, n), True))
    P = rng.normal(size=(6, 3))
    out.append(cv2.mulTransposed(P - P.mean(0), True))
    P[:, 2] = 0.0  # planar: an exact zero singular value
    out.append(cv2.mulTransposed(P - P.mean(0), True))
    out.append(np.diag([3.0, 2.0, 0.0]))
    out.append(np.zeros((3, 3)))
    out.append(rng.normal(size=(3, 3)))
    return out


@pytest.mark.parametrize("i", range(len(svd_inputs())))
def test_svd(i):
    A = svd_inputs()[i]
    w, u, vt = cv2.SVDecomp(A)
    ow, ou, ovt = pb.svd(A)
    assert np.array_equal(ow, w.reshape(-1)) and np.array_equal(ou, u) and np.array_equal(ovt, vt)


def invert_inputs():
    rng = np.random.default_rng(11)
    out = [rng.normal(size=(3, 3)) for _ in range(3)]
    S = rng.normal(size=(3, 3))
    S[:, 2] = 0  # the planar case: cws[3] == cws[0]
    out.append(S)
    out.append(np.outer(rng.normal(size=3), rng.normal(size=3)))
    out.append(np.zeros((3, 3)))
    return out


@pytest.mark.parametrize("i", range(len(invert_inputs())))
def test_invert_svd(i):
    A = invert_inputs()[i]
    _, D = cv2.invert(A, flags=cv2.DECOMP_SVD)
    assert np.array_equal(pb.invert_svd(A), D)


@pytest.mark.parametrize("cols", [4, 3, 5])
def test_solve_svd(cols):
    rng = np.random.default_rng(cols)
    cases = [rng.normal(size=(6, cols)) for _ in range(4)]
    Z = rng.normal(size=(6, cols))
    Z[:, 1] = 0  # a zero column: a zero singular value, the basis completed
    cases.append(Z)
    for A in cases:
        b = rng.normal(size=(6, 1))
        _, x = cv2.solve(A, b, flags=cv2.DECOMP_SVD)
        assert np.array_equal(pb.solve_svd(A, b), x.reshape(-1))


@pytest.mark.parametrize("n", [0, 1, 4, 8, 9, 10, 12, 15, 19, 20, 21, 25, 50, 200, 1000, 65536])
@pytest.mark.parametrize("params", [sp.RELOC, sp.DEFAULT, (0.99, 4, 300, 4, 0.5, 5.991), (0.5, 8, 50, 4, 0.3, 5.991),
                                    (0.99, 8, 300, 4, 1.0, 5.991), (0.99, 8, 300, 4, 0.35, 5.991)])
def test_ransac_parameters(n, params):
    assert pkg.pnp_ransac_parameters(n, *params[:5]) == pb.ransac_parameters(n, *params[:5])


def test_ransac_parameters_edges():
    assert pkg.pnp_ransac_parameters(10, *sp.RELOC[:5]) == (10, 1)  # min == N: one iteration
    assert pkg.pnp_ransac_parameters(0, *sp.RELOC[:5]) == (10, 1)
    assert pkg.pnp_ransac_parameters(100, *sp.RELOC[:5]) == (50, 35)  # (int)(N*epsilon)
    for n in range(1, 300):  # N*epsilon in float, truncated
        for eps in (0.1, 0.3, 0.35, 0.7):
            assert pkg.pnp_ransac_parameters(n, 0.99, 4, 300, 4, eps) == pb.ransac_parameters(n, 0.99, 4, 300, 4, eps)


def test_scene_decisions():
    """What each synthetic scene exercises, on the restatement with random sets."""
    seen = set()
    for name, *_ in sp.CASES:
        for seed in range(3):
            d = sp.case(name, seed)
            n = len(d["P3Dw"])
            rng = np.random.default_rng(seed + 100)
            k = d["max_its"] if n >= d["min_inliers"] else 0
            sets = np.array([rng.choice(n, 4, replace=False) for _ in range(k)], np.int32).reshape(-1, 4)
            r = pb.iterate(d, pb.INITIAL, sets)
            tr = r["trace"][:r["iterations_used"]]
            refines = tr[tr[:, 14] >= 0]
            if name == "below_min":
                assert r["no_more"] and not r["returned"] and r["iterations_used"] == 0
            if name == "no_inliers":
                assert not r["returned"] and r["best_inliers"] == 0
            if r["returned"] and not r["no_more"]:
                seen.add("early")
                if len(refines) == 1 and r["iterations_used"] == int(np.argmax(tr[:, 13] >= d["min_inliers"])) + 1:
                    seen.add("first_refine_succeeds")
                if (refines[:-1, 14] <= d["min_inliers"]).any():
                    seen.add("refine_failed_then_succeeded")
            if len(refines) and not r["returned"]:
                seen.add("refine_failed")
            if len(refines) and n >= 1000:
                seen.add("refine_at_1000")
            assert r["margin"] > 1e-6
    assert {"early", "first_refine_succeeds", "refine_at_1000"} <= seen  # failed Refines: test_refine_paths


@pytest.mark.parametrize("n", [100, 1200])
def test_refine_paths(n):
    """The scan's Refine branches, reached on purpose (pnpsolver_binding.refine_paths): a Refine of the carried-in best
    mask fails; a second qualifying iteration repeats it with the mask unchanged and fails again; a third replaces the
    mask and its Refine succeeds, here over hundreds of correspondences at n = 1200."""
    cases = pb.refine_path_cases(n)
    assert len(cases) == 2
    for d, state, sets in cases:
        r = pb.iterate(d, state, sets)
        tr, m = r["trace"], d["min_inliers"]
        assert m <= tr[0, 13] <= state[1] and 0 <= tr[0, 14] <= m  # qualifies, keeps the carried mask, fails
        assert tr[1, 13] == tr[0, 13] and tr[1, 14] == tr[0, 14]   # the same mask again: the same failure
        assert tr[2, 13] > state[1] and tr[2, 14] > m              # a new mask, and its Refine succeeds
        assert r["returned"] and not r["no_more"] and r["iterations_used"] == 3 and r["n_inliers"] == tr[2, 14]
        assert r["best_changed"] and r["best_inliers"] == tr[2, 13]
        if n >= 1000:
            assert tr[2, 13] > 32 * 8  # the compacted mask spans many words
        assert r["margin"] > 1e-6
