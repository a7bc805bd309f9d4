"""The CPU restatement of Sim3Solver (oracle/sim3solver.cpp) against the reference's own src/Sim3Solver.cc, compiled in
place (oracle/_ref/libref_sim3solver.so), bit for bit: after srand(seed) the reference draws its sets; the restatement,
fed the same sets, gives the same returned T12, vbInliers, nInliers, bNoMore, getters and counters on every call."""
import os

import numpy as np
import pytest

import sim3solver_binding as sb
from synth_sim3solver import CASES, problem, scene

pytestmark = pytest.mark.skipif(not os.path.exists(sb.REF_LIB),
                                reason="oracle/_ref not built (make -C oracle -f sim3solver.mk sim3solver-ref)")


def ref_call(ref, n_iterations):
    """One iterate (find() when None) on the reference: its outputs and the state before and after."""
    before = ref.state()
    out = ref.iterate(n_iterations)
    out["before"], out["after"] = before, ref.state()
    return out


def assert_same(got, want, pr, m):
    """The restatement's result (got) against one reference call (want)."""
    after = want["after"]
    assert (want["T12"] is not None) == bool(got["returned"])
    if want["T12"] is not None:
        assert np.array_equal(got["T12"], want["T12"])
    assert got["n_inliers"] == want["n_inliers"]
    assert np.array_equal(sb.expand(got["inliers"], pr["indices1"], m), want["inliers"])
    if want["no_more"] is not None:
        assert bool(got["no_more"]) == want["no_more"]
    assert got["iterations_done"] == after["iterations"] and got["best_inliers"] == after["best_inliers"]
    if got["best_changed"]:
        assert np.array_equal(got["R"], after["R"]) and np.array_equal(got["t"], after["t"]) and got["s"] == after["s"]
    else:
        before = want["before"]
        assert after["has_best"] == before["has_best"]
        assert np.array_equal(after["R"], before["R"]) and after["s"] == before["s"]


def solver(name, lib=sb.REF_LIB):
    kw, (p, mi, mx) = CASES[name]
    sc = scene(**kw)
    ref = sb.RefSolver(lib, sc)
    ref.set_ransac_parameters(p, mi, mx)
    pr = problem(sc, mi)
    st = ref.state()
    pr["max_its"] = st["max_its"]
    return sc, pr, ref


@pytest.mark.parametrize("case", sorted(CASES))
def test_constructor_and_parameters(case):
    sc, pr, ref = solver(case)
    st, mem = ref.state(), ref.members()
    kw, (p, mi, mx) = CASES[case]
    assert st["N"] == len(pr["X1c"]) and st["mN1"] == sc["m"] and st["iterations"] == 0 and st["best_inliers"] == 0
    assert np.array_equal(mem["indices1"], pr["indices1"])
    assert np.array_equal(mem["X1c"], pr["X1c"]) and np.array_equal(mem["X2c"], pr["X2c"])
    # (size_t)(9.210 * sigma2): 9 at level 0, 13 at level 1
    assert np.array_equal(mem["max_err1"], (9.210 * pr["sigma2_1"].astype(np.float64)).astype(np.uint64))
    assert np.array_equal(mem["max_err2"], (9.210 * pr["sigma2_2"].astype(np.float64)).astype(np.uint64))
    assert st["max_its"] == sb.ransac_max_its(st["N"], p, mi, mx) and st["min_inliers"] == mi
    ref.close()


@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("case", sorted(CASES))
def test_find_matches_reference(case, seed):
    sc, pr, ref = solver(case)
    ref.srand(seed)
    want = ref_call(ref, None)
    used = want["after"]["iterations"]
    ref.srand(seed)
    sets = ref.rand_draws(len(pr["X1c"]), used) if len(pr["X1c"]) >= pr["min_inliers"] else np.zeros((0, 3))
    got, margin = sb.oracle(pr, (0, 0), sets)
    assert margin > 1e-6
    assert_same(got, want, pr, sc["m"])
    ref.close()


ROUND_ROBIN = [["loop_30_free", "outliers_only", "loop_demanding", "too_few"],
               ["loop_40_fixed_levels", "outliers_only_fixed", "loop_60_free"],
               ["degenerate", "identity", "min_equals_n", "loop_50_free_800"]]


def round_robin(names, seed, lib=sb.REF_LIB, rounds=8):
    """LoopClosing::ComputeSim3's pattern: iterate(5) on every candidate in turn from one srand(seed); a candidate
    stays after bNoMore is false, including after a returned model (OptimizeSim3 may reject it).  Returns the solvers
    and the calls in order as (candidate, outputs)."""
    solvers = [solver(n, lib) for n in names]
    solvers[0][2].srand(seed)
    calls, dead = [], set()
    for _ in range(rounds):
        for c, (sc, pr, ref) in enumerate(solvers):
            if c in dead:
                continue
            out = ref_call(ref, 5)
            calls.append((c, out))
            if out["no_more"]:
                dead.add(c)
    return solvers, calls


@pytest.mark.parametrize("seed", [0, 3])
@pytest.mark.parametrize("group", range(len(ROUND_ROBIN)))
def test_round_robin_matches_reference(group, seed):
    solvers, calls = round_robin(ROUND_ROBIN[group], seed)
    ref0 = solvers[0][2]
    ref0.srand(seed)
    returned_then_continued = False
    last_returned = set()
    for c, want in calls:
        sc, pr, ref = solvers[c]
        n = len(pr["X1c"])
        k = want["after"]["iterations"] - want["before"]["iterations"]
        sets = ref0.rand_draws(n, k) if n >= pr["min_inliers"] else np.zeros((0, 3), np.int32)
        pr = dict(pr)
        got, margin = sb.oracle(pr, (want["before"]["iterations"], want["before"]["best_inliers"]), sets)
        assert margin > 1e-6
        assert got["iterations_used"] == k
        assert_same(got, want, pr, sc["m"])
        returned_then_continued |= c in last_returned
        if want["T12"] is not None:
            last_returned.add(c)
    assert calls
    if (group, seed) == (0, 0):  # this sequence continues a solver after its early return
        assert returned_then_continued
    for _, _, ref in solvers:
        ref.close()
