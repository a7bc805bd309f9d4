"""The CPU restatement of PnPsolver (oracle/pnpsolver.cpp) against the reference's own src/PnPsolver.cc, compiled in
place (oracle/_ref/libref_pnpsolver.so), bit for bit: per-hypothesis compute_pose, Refine's compute_pose, find(), and
Tracking::Relocalization's round-robin of iterate(5) over several candidates.  After srand(seed) the reference draws its
sets; the restatement is fed the same sets (replayed from the same rand() stream) and the state the previous call left."""
import os

import numpy as np
import pytest

import pnpsolver_binding as pb
import synth_pnp as sp

pytestmark = pytest.mark.skipif(not os.path.exists(pb.REF_LIB),
                                reason="oracle/_ref not built (make -C oracle -f pnpsolver.mk pnpsolver-ref)")

NAMES = [c[0] for c in sp.CASES]


@pytest.mark.parametrize("name", NAMES)
def test_compute_pose(name):
    d = sp.case(name, 1)
    n = len(d["P3Dw"])
    if n < 4:
        return
    ref = pb.Ref(d)
    rng = np.random.default_rng(5)
    for idx in [rng.choice(n, 4, replace=False) for _ in range(20)] + [np.arange(n), np.where(d["truth"])[0]]:
        if len(idx) < 4:
            continue
        R, t, e = ref.compute_pose(idx)
        oR, ot, oe = pb.compute_pose(d, idx)
        assert np.array_equal(R, oR) and np.array_equal(t, ot), name
        assert e == oe or (np.isnan(e) and np.isnan(oe))


def run_calls(scenes, calls, seed):
    """calls: a list of (solver index, n_iterations or None for find()).  Runs the reference after srand(seed), then
    replays its draws into the restatement call by call; asserts every output and the state after each call."""
    refs = [pb.Ref(d) for d in scenes]
    pb.Ref.srand(seed)
    want = []
    for s, nit in calls:
        out = refs[s].iterate(nit)
        out["after"] = refs[s].state()
        want.append(out)
    pb.Ref.srand(seed)
    states = [pb.INITIAL] * len(scenes)
    for (s, nit), w in zip(calls, want):
        d = scenes[s]
        n = len(d["P3Dw"])
        it = states[s][0]
        nit = d["max_its"] if nit is None else nit
        k = 0 if n < d["min_inliers"] else max(nit, d["max_its"] - it)
        used = w["after"]["iterations"] - it if n >= d["min_inliers"] else 0
        sets = pb.draw_sets(n, used, pb.Ref.random_int)
        full = np.zeros((k, 4), np.int32)
        full[:used] = sets
        full[used:] = np.arange(4)  # never reached: the reference returned before
        got = pb.iterate(d, states[s], full)
        assert (w["Tcw"] is not None) == bool(got["returned"])
        if w["Tcw"] is not None:
            assert np.array_equal(got["Tcw"], w["Tcw"])
            assert np.array_equal(got["inliers"], w["inliers"]) and got["n_inliers"] == w["n_inliers"]
        if w["no_more"] is not None:  # find() keeps bNoMore to itself
            assert bool(got["no_more"]) == w["no_more"]
        assert got["iterations_used"] == used
        a = w["after"]
        assert got["iterations_done"] == a["iterations"] and got["best_inliers"] == a["best_inliers"]
        if a["best_Tcw"] is not None:
            assert np.array_equal(got["best_Tcw"], a["best_Tcw"])
            assert np.array_equal(got["best_mask"].astype(bool), a["best_mask"].astype(bool))
        states[s] = pb.next_state(got)


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("seed", [0, 1])
def test_find(name, seed):
    run_calls([sp.case(name, seed)], [(0, None)], seed)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_relocalization_round_robin(seed):
    """Relocalization: iterate(5) on each candidate in turn until one returns or all are exhausted, then further calls
    on the solvers that remain (a solver that continues after an early return carries its best mask)."""
    names = ["n15", "n50", "planar", "repeated", "behind", "no_inliers"]
    scenes = [sp.case(nm, seed + 10) for nm in names]
    calls = [(s, 5) for _ in range(9) for s in range(len(scenes))]
    run_calls(scenes, calls, seed)
