"""The monocular initialiser's CPU restatement (oracle/init.cpp): its OpenCV linear algebra pinned bit for bit against
cv2 at the shapes Initializer.cc uses, and its decisions on the two-view scenes of tests/synth_init.py."""
import numpy as np
import pytest

import init_binding as ib
from synth_init import CASES, synth_init

cv2 = pytest.importorskip("cv2")

# (rows, cols, FULL_UV): ComputeH21 (:509), ComputeF21 (:584, :606), ReconstructH (:1174), Triangulate (:1492),
# DecomposeE (:1810)
SVD_SHAPES = [(16, 9, True), (8, 9, True), (3, 3, True), (4, 4, True), (3, 3, False)]


@pytest.mark.parametrize("rows,cols,full", SVD_SHAPES)
def test_svd_matches_cv2(rows, cols, full):
    rng = np.random.default_rng(rows * 100 + cols)
    for trial in range(200):
        A = rng.standard_normal((rows, cols)).astype(np.float32)
        if rows == cols == 3 and trial % 2:
            A[2] = A[0] * np.float32(0.5) + A[1] * np.float32(0.25)  # rank 2, as Fpre after w[2] = 0
        w, u, vt = ib.svd(A, full)
        cw, cu, cvt = cv2.SVDecomp(A.copy(), flags=cv2.SVD_FULL_UV if full else 0)
        assert np.array_equal(w, cw.ravel())
        assert np.array_equal(u, cu)
        assert np.array_equal(vt, cvt)  # for 8 x 9 this includes the 9th row, completed beyond the rank


def test_inv_det_gemm_match_cv2():
    rng = np.random.default_rng(3)
    for _ in range(300):
        M = rng.standard_normal((3, 3)).astype(np.float32)
        B = rng.standard_normal((3, 4)).astype(np.float32)
        c = rng.standard_normal((3, 1)).astype(np.float32)
        s = float(np.float32(rng.uniform(0.99, 1.01)))
        ok, inv = ib.inv3(M)
        assert ok and np.array_equal(inv, cv2.invert(M)[1])
        assert ib.det3(M) == cv2.determinant(M)
        assert np.array_equal(ib.gemm(M, B), cv2.gemm(M, B, 1, None, 0))  # K*[R|t]
        assert np.array_equal(ib.gemm(M, M, s), cv2.gemm(M, M, s, None, 0))  # s*U*Rp
        assert np.array_equal(ib.gemm(M, c, 1.0, c), cv2.gemm(M, c, 1, c, 1))  # R*x3D + t
        assert np.array_equal(ib.gemm(M, c, -1.0, None, True), cv2.gemm(M, c, -1, None, 0, flags=cv2.GEMM_1_T))
        assert np.array_equal(ib.gemm(M, M, 1.0, None, True), cv2.gemm(M, M, 1, None, 0, flags=cv2.GEMM_1_T))
    singular = np.array([[1, 2, 3], [2, 4, 6], [0, 1, 0]], np.float32)
    ok, inv = ib.inv3(singular)
    assert not ok and not inv.any() and not cv2.invert(singular)[1].any()


def test_triangulate_rows_are_add_weighted():
    """A.row(0) = x*P.row(2) - P.row(0) (:1484-1487) evaluates as addWeighted(P.row(2), x, P.row(0), -1, 0): one
    rounding of the double expression, which init.cpp writes out."""
    rng = np.random.default_rng(4)
    for _ in range(500):
        r2 = rng.standard_normal((1, 4)).astype(np.float32) * 400
        r0 = rng.standard_normal((1, 4)).astype(np.float32) * 400
        x = np.float32(rng.uniform(0, 640))
        want = cv2.addWeighted(r2, float(x), r0, -1, 0)
        assert np.array_equal((np.float64(x) * r2.astype(np.float64) - r0.astype(np.float64)).astype(np.float32), want)


def decisions_clear(r):
    """No decision of the case sits within rounding of its threshold."""
    assert abs(float(r["RH"]) - 0.40) > 1e-6
    assert not (np.abs(r["parallax"].astype(np.float64) - 1.0) <= 1e-4).any()


@pytest.mark.parametrize("case", sorted(CASES))
def test_oracle_cases(case):
    d = synth_init(**CASES[case])
    r = ib.oracle(d)
    decisions_clear(r)
    assert r["n_matches"] == int((d["matches12"] >= 0).sum())
    if r["ret"]:
        # the recovered motion is the scene's (t up to scale)
        R = r["R21"].reshape(3, 3)
        assert np.abs(R - d["R"]).max() < 0.02
        assert r["t21"] @ (d["t"] / np.linalg.norm(d["t"])) > 0.99
        assert r["rt_state"] == 1 and r["triangulated"].sum() > 50
        assert (r["p3d"][d["matches12"] < 0] == 0).all()
    else:
        assert (r["p3d"] == ib.UNTOUCHED).all() and (r["triangulated"] == 7).all()
        assert r["rt_state"] == (-1 if r["n_hyp"] == 4 else 0)
        if r["rt_state"] == 0:
            assert (r["R21"] == ib.UNTOUCHED).all()


def test_cases_cover_the_branches():
    seen = set()
    for case, kw in CASES.items():
        r = ib.oracle(synth_init(**kw))
        seen.add(("H" if r["model"] == 1 else "F") + ("ok" if r["ret"] else "fail"))
        if kw["kind"] == "rotation":
            assert not r["ret"] and r["n_hyp"] and max(r["parallax"]) < 1.0
        if kw["kind"] == "ambiguous":
            # rejected by the ambiguity tests, not by parallax or point count: ReconstructH's second-best rule
            # (secondBestGood >= 0.75*bestGood) or ReconstructF's nsimilar > 1
            g = r["n_good"].astype(np.int64)
            assert not r["ret"] and len(g)
            if r["model"] == 1:
                assert np.sort(g)[-2] >= 0.75 * g.max()
            else:
                assert (g > 0.7 * g.max()).sum() > 1
            seen.add("ambiguous")
    assert seen >= {"Hok", "Fok", "Hfail", "Ffail", "ambiguous"}, seen
