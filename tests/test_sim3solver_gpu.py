"""GPU tests of the Sim3 RANSAC (csrc/sim3solver.cu, pkg.Sim3Solver): parity with the CPU restatement on every loop
candidate of tests/synth_sim3solver.py, a mixed batch against single calls, bit-identical repeats, the error codes, and
the drop-in host/adapters/Sim3Solver_b200.cc against the reference's own Sim3Solver after srand(seed)."""
import os

import numpy as np
import pytest

import sim3solver_binding as sb
from synth_sim3solver import CASES, problem, scene

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def batch(pkg):
    b = pkg.Sim3SolverBatch(max_matches=1024, max_sets=300, max_batch=64)
    yield b
    b.close()


def ulps(a, b):
    a, b = np.asarray(a, np.float32).view(np.int32).astype(np.int64), np.asarray(b, np.float32).view(np.int32)
    return np.abs(a - b.astype(np.int64))


def close_floats(got, want):
    """Bit-identical, or within 1 ulp: the device's double atan2 / sin / cos (CUDA's) may differ from glibc's in the
    last bit and move a float rounding of the rotation (DESIGN §7).  NaN equals NaN."""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    return bool(((ulps(got, want) <= 1) | (np.isnan(got) & np.isnan(want))).all())


def same(got, want, n):
    """A device result (pkg dict plus the solver's state) against the restatement's."""
    assert (got["T12"] is not None) == bool(want["returned"])
    if want["returned"]:
        assert close_floats(got["T12"], want["T12"])
    assert got["n_inliers"] == want["n_inliers"] and got["no_more"] == bool(want["no_more"])
    assert np.array_equal(got["inliers"], want["inliers"][:n])
    assert got["iterations_used"] == want["iterations_used"]


def make(pkg, handle, pr):
    sv = handle.solver(pr["X1c"], pr["X2c"], pr["sigma2_1"], pr["sigma2_2"], pr["K1"], pr["K2"], pr["fix_scale"])
    sv.min_inliers, sv.max_its = pr["min_inliers"], pr["max_its"]
    return sv


def case_problem(name):
    kw, (p, mi, mx) = CASES[name]
    sc = scene(**kw)
    pr = problem(sc, mi)
    pr["max_its"] = sb.ransac_max_its(len(pr["X1c"]), p, mi, mx)
    return sc, pr


def random_sets(rng, n, k):
    return np.array([rng.choice(n, 3, replace=False) for _ in range(k)], np.int32).reshape(-1, 3)


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("case", sorted(CASES))
def test_device_matches_oracle(pkg, batch, case, seed):
    """find() and then iterate(5) calls until bNoMore, each against the restatement from the same state."""
    sc, pr = case_problem(case)
    n = len(pr["X1c"])
    sv = make(pkg, batch, pr)
    rng = np.random.default_rng(seed)
    for call in range(4):
        nit = sv.max_its if call == 0 else 5
        k = sv.sets_needed(nit)
        sets = random_sets(rng, n, k) if n >= 3 else np.zeros((0, 3), np.int32)
        state = (sv.iterations, sv.best_inliers)
        want, margin = sb.oracle(pr, state, sets)
        assert margin > 1e-6
        R0 = sv.R
        got = sv.iterate(nit, sets)
        same(got, want, n)
        assert (sv.iterations, sv.best_inliers) == (want["iterations_done"], want["best_inliers"])
        if want["best_changed"]:
            assert close_floats(sv.R, want["R"]) and close_floats(sv.t.ravel(), want["t"])
            assert close_floats(sv.s, want["s"])
        else:
            assert sv.R is R0
        if got["no_more"]:
            break


def test_degenerate_sets_match_oracle(pkg, batch):
    """Sets with repeated points and collinear points, and the identity scene: NaN models or 0 inliers are still
    accepted by the 0 >= 0 rule, on the device as in the restatement."""
    sc, pr = case_problem("degenerate")
    n = len(pr["X1c"])
    sets = np.array([[0, 3, 6], [1, 4, 7], [2, 5, 8], [0, 2, 4], [1, 3, 5]] * 4, np.int32)  # repeated / on the line
    for fix in (0, 1):
        d = dict(pr, fix_scale=fix, min_inliers=n)
        sv = make(pkg, batch, d)
        want, _ = sb.oracle(d, (0, 0), sets)
        got = sv.iterate(len(sets), sets)
        same(got, want, n)
        assert sv.best_inliers == want["best_inliers"]
        if want["best_changed"]:
            assert close_floats(sv.R, want["R"]) and close_floats(sv.s, want["s"])
    sc, pr = case_problem("identity")
    X = pr["X1c"]
    d = dict(pr, X2c=X)  # exactly the same points: q = (1, 0, 0, 0), vec = 0 * inf
    sv = make(pkg, batch, d)
    sets = random_sets(np.random.default_rng(3), len(X), 10)
    want, _ = sb.oracle(d, (0, 0), sets)
    same(sv.iterate(10, sets), want, len(X))
    assert np.isnan(sv.R).all() and want["best_inliers"] == 0


def test_batch_equals_single_calls(pkg, batch):
    rng = np.random.default_rng(11)
    names = sorted(CASES)
    probs, solvers, sets, nits = [], [], [], []
    for i in range(64):
        sc, pr = case_problem(names[i % len(names)])
        n = len(pr["X1c"])
        sv = make(pkg, batch, pr)
        sv.iterations = int(rng.integers(0, 3)) if n >= pr["min_inliers"] else 0
        nit = int(rng.choice([1, 5, 300]))
        k = sv.sets_needed(nit)
        probs.append(pr)
        solvers.append(sv)
        sets.append(random_sets(rng, n, k) if n >= 3 else np.zeros((0, 3), np.int32))
        nits.append(nit)
    start = [(s.iterations, s.best_inliers) for s in solvers]
    outs = pkg.Sim3Solver.iterate_batch(solvers, nits, sets, handle=batch)
    assert batch.last_ms() > 0
    for pr, sv, st, nit, s0, b in zip(probs, solvers, sets, nits, start, outs):
        one = make(pkg, batch, pr)
        one.iterations, one.best_inliers = s0
        a = one.iterate(nit, st)
        assert (a["T12"] is None) == (b["T12"] is None)
        if a["T12"] is not None:
            assert a["T12"].tobytes() == b["T12"].tobytes()
        for k in ("no_more", "n_inliers", "iterations_used"):
            assert a[k] == b[k], k
        assert np.array_equal(a["inliers"], b["inliers"])
        assert (one.iterations, one.best_inliers) == (sv.iterations, sv.best_inliers)
        if one.R is not None:
            assert one.R.tobytes() == sv.R.tobytes() and one.s == sv.s
        want, margin = sb.oracle(pr, s0, st)
        assert margin > 1e-6
        same(b, want, len(pr["X1c"]))


def test_repeats_are_bit_identical(pkg, batch):
    sc, pr = case_problem("loop_30_free")
    sets = random_sets(np.random.default_rng(5), len(pr["X1c"]), pr["max_its"])
    outs = []
    for _ in range(3):
        sv = make(pkg, batch, pr)
        r = sv.find(sets)
        outs.append((r["T12"].tobytes(), r["inliers"].tobytes(), sv.R.tobytes(), sv.t.tobytes(), sv.iterations))
    assert outs[0] == outs[1] == outs[2]


def test_capacity_and_bad_arguments(pkg):
    small = pkg.Sim3SolverBatch(max_matches=100, max_sets=10, max_batch=2)
    sc, pr = case_problem("loop_90_free")
    pr = dict(pr, X1c=pr["X1c"][:80], X2c=pr["X2c"][:80], sigma2_1=pr["sigma2_1"][:80], sigma2_2=pr["sigma2_2"][:80],
              max_its=10)
    sets = random_sets(np.random.default_rng(0), 80, 10)

    def code(prs, sts, nits=None, tweak=None):
        svs = [make(pkg, small, p) for p in prs]
        if tweak:
            tweak(svs)
        with pytest.raises(pkg.B200SlamError) as e:
            pkg.Sim3Solver.iterate_batch(svs, nits or [10] * len(svs), sts, handle=small)
        return e.value.code

    big = dict(pr, X1c=np.tile(pr["X1c"], (2, 1)), X2c=np.tile(pr["X2c"], (2, 1)),
               sigma2_1=np.tile(pr["sigma2_1"], 2), sigma2_2=np.tile(pr["sigma2_2"], 2))
    assert code([big], [sets]) == pkg.ERR_CAPACITY  # correspondences
    assert code([dict(pr, max_its=20)], [np.tile(sets, (2, 1))], [20]) == pkg.ERR_CAPACITY  # sets
    assert code([pr, pr, pr], [sets] * 3) == pkg.ERR_CAPACITY  # batch
    for bad in (-1, 80):
        s = sets.copy()
        s[4, 1] = bad
        assert code([pr], [s]) == pkg.ERR_BAD_ARG
    s = sets.copy()
    s[2, 2] = s[2, 0]
    assert code([pr], [s]) == pkg.ERR_BAD_ARG  # repeated within a set
    sig = pr["sigma2_1"].copy()
    sig[3] = -1
    assert code([dict(pr, sigma2_1=sig)], [sets]) == pkg.ERR_BAD_ARG
    sig[3] = np.inf
    assert code([dict(pr, sigma2_1=sig)], [sets]) == pkg.ERR_BAD_ARG
    two = dict(pr, X1c=pr["X1c"][:2], X2c=pr["X2c"][:2], sigma2_1=pr["sigma2_1"][:2], sigma2_2=pr["sigma2_2"][:2],
               min_inliers=1)
    assert code([two], [np.zeros((10, 3), np.int32)]) == pkg.ERR_BAD_ARG  # n < 3 where an iteration runs

    def more_sets(svs):  # more sets than max_its - iterations_done
        svs[0].iterations = 5
        svs[0].sets_needed = lambda nit: 10
    assert code([pr], [sets], tweak=more_sets) == pkg.ERR_BAD_ARG
    # a bad problem anywhere in the batch: nothing is written
    good = make(pkg, small, pr)
    s = sets.copy()
    s[0, 0] = -5
    bad = make(pkg, small, pr)
    with pytest.raises(pkg.B200SlamError):
        pkg.Sim3Solver.iterate_batch([good, bad], [10, 10], [sets, s], handle=small)
    assert good.iterations == 0 and good.R is None
    r = small.solver(pr["X1c"], pr["X2c"], pr["sigma2_1"], pr["sigma2_2"], pr["K1"], pr["K2"])
    r.min_inliers, r.max_its = pr["min_inliers"], 10
    assert r.iterate(10, sets)["iterations_used"] >= 1
    # too few correspondences for min_inliers: no_more, no set read, no error
    few = make(pkg, small, dict(pr, min_inliers=81))
    out = few.iterate(10, np.zeros((0, 3), np.int32))
    assert out["no_more"] and out["iterations_used"] == 0 and out["T12"] is None
    with pytest.raises(pkg.B200SlamError) as e:
        pkg.Sim3SolverBatch(max_matches=2, max_sets=1, max_batch=1)
    assert e.value.code == pkg.ERR_BAD_ARG
    small.close()


@pytest.mark.skipif(not (os.path.exists(sb.REF_LIB) and os.path.exists(sb.ADP_LIB)),
                    reason="oracle/_ref not built (make -C oracle -f sim3solver.mk sim3solver-ref)")
@pytest.mark.parametrize("seed", [0, 3])
@pytest.mark.parametrize("group", [0, 1, 2])
def test_drop_in_matches_reference(group, seed):
    """host/adapters/Sim3Solver_b200.cc against the reference's own Sim3Solver, both in LoopClosing's round-robin of
    iterate(5) after srand(seed): every call is identical up to and including the first early return (after it, the
    drop-in's rand() stream is ahead by the draws the reference did not make); with no early return, the whole
    sequences are identical."""
    from test_oracle_reference_sim3solver import ROUND_ROBIN, round_robin
    _, want = round_robin(ROUND_ROBIN[group], seed, sb.REF_LIB)
    _, got = round_robin(ROUND_ROBIN[group], seed, sb.ADP_LIB)
    first_return = next((i for i, (_, w) in enumerate(want) if w["T12"] is not None), None)
    upto = len(want) if first_return is None else first_return + 1
    if first_return is None:
        assert len(got) == len(want)
    for (cg, g), (cw, w) in zip(got[:upto], want[:upto]):
        assert cg == cw
        assert (g["T12"] is None) == (w["T12"] is None)
        if w["T12"] is not None:
            assert close_floats(g["T12"], w["T12"])
        assert g["no_more"] == w["no_more"] and g["n_inliers"] == w["n_inliers"]
        assert np.array_equal(g["inliers"], w["inliers"])
        ga, wa = g["after"], w["after"]
        for k in ("N", "mN1", "iterations", "best_inliers", "max_its", "min_inliers", "has_best"):
            assert ga[k] == wa[k], k
        assert close_floats(ga["R"], wa["R"]) and close_floats(ga["t"], wa["t"]) and close_floats(ga["s"], wa["s"])
