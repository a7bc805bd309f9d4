"""The device PnPsolver (b2s_pnpsolver_iterate) against the CPU restatement (oracle/pnpsolver.cpp, itself bit-identical
to the reference's own PnPsolver): every output bit-identical on every scene and several seeds, including calls that
continue from a carried-in best mask; a mixed batch of 64 against single calls; bit-identical repeats; every error
code.  Threshold margins are asserted on every compared scene so that bit-identity is not luck at a threshold."""
import ctypes
import importlib
import os

import numpy as np
import pytest

import pnpsolver_binding as pb
import synth_pnp as sp

pkg = importlib.import_module("self_commit_orb-slam2_b200")
pytestmark = pytest.mark.gpu

NAMES = [c[0] for c in sp.CASES]


def device(h, probs):
    """One b2s_pnpsolver_iterate over packed problems: (rc, results)."""
    res = (pkg._PnPsolverResult * len(probs))()
    arrs = []
    for i, (p, _) in enumerate(probs):
        r, a = pb.new_result(p.n)
        res[i] = r
        arrs.append(a)
    P = (pkg._PnPsolverProblem * len(probs))(*[p for p, _ in probs])
    rc = pkg.lib().b2s_pnpsolver_iterate(h, len(probs), P, res)
    return rc, [pb.unpack(res[i], arrs[i], probs[i][0].n) for i in range(len(probs))]


def same(a, b):
    for k in ("returned", "n_inliers", "no_more", "iterations_used", "iterations_done", "best_inliers",
              "best_changed"):
        assert a[k] == b[k], k
    assert (a["Tcw"] is None) == (b["Tcw"] is None)
    if a["Tcw"] is not None:
        assert a["Tcw"].tobytes() == b["Tcw"].tobytes()
    assert np.array_equal(a["inliers"], b["inliers"])
    assert a["best_Tcw"].tobytes() == b["best_Tcw"].tobytes()
    assert np.array_equal(a["best_mask"], b["best_mask"])


@pytest.fixture(scope="module")
def handle():
    h = ctypes.c_void_p()
    assert pkg.lib().b2s_pnpsolver_create(4096, 400, 64, 0, ctypes.byref(h)) == 0
    yield h
    pkg.lib().b2s_pnpsolver_destroy(h)


def sets_for(d, rng, iterations_done, n_iterations):
    """Random minimal sets for one iterate(n_iterations) call on a solver that has run iterations_done iterations."""
    n = len(d["P3Dw"])
    k = 0 if n < d["min_inliers"] else max(n_iterations, d["max_its"] - iterations_done)
    return np.array([rng.choice(n, 4, replace=False) for _ in range(k)], np.int32).reshape(-1, 4)


def first_sets(d, seed):
    return sets_for(d, np.random.default_rng(seed), 0, 5)


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_device_vs_restatement(handle, name, seed):
    d = sp.case(name, seed)
    state = pb.INITIAL
    rng = np.random.default_rng(seed)
    for c in range(4):  # the first call a find() when seed is odd, then iterate(5)
        sets = sets_for(d, rng, state[0], d["max_its"] if (c == 0 and seed % 2) else 5)
        want = pb.iterate(d, state, sets)
        assert want["margin"] > 1e-6, "a compared error2 lies within 1e-6 of its threshold"
        rc, (got,) = device(handle, [pb.pack(d, state, sets)])
        assert rc == 0, pkg.lib().b2s_last_error()
        same(got, want)
        state = pb.next_state(want)


@pytest.mark.parametrize("n", [100, 1200])
def test_refine_paths(handle, n):
    """A failed Refine of the carried-in mask, its skipped repeat with the mask unchanged, then a new mask whose Refine
    succeeds (pnpsolver_binding.refine_paths; at n = 1200 the Refine runs over hundreds of correspondences)."""
    cases = pb.refine_path_cases(n)
    assert len(cases) == 2
    for d, state, sets in cases:
        want = pb.iterate(d, state, sets)
        rc, (got,) = device(handle, [pb.pack(d, state, sets)])
        assert rc == 0, pkg.lib().b2s_last_error()
        assert want["returned"] and not want["no_more"] and want["iterations_used"] == 3
        same(got, want)


def test_compute_pose_bits(handle):
    """A call whose first qualifying hypothesis returns: the refined Tcw carries the double R, t rounded once, so the
    device's pose equals the restatement's to the bit on a scene that returns."""
    d = sp.case("n50", 0)
    sets = first_sets(d, 0)
    want = pb.iterate(d, pb.INITIAL, sets)
    rc, (got,) = device(handle, [pb.pack(d, pb.INITIAL, sets)])
    assert rc == 0 and want["returned"]
    same(got, want)


def test_batch_of_64_equals_singles(handle):
    probs, wants = [], []
    for i in range(64):
        name = NAMES[i % len(NAMES)]
        d = sp.case(name, 100 + i)
        sets = first_sets(d, i)
        probs.append(pb.pack(d, pb.INITIAL, sets))
        wants.append(pb.iterate(d, pb.INITIAL, sets))
    rc, got = device(handle, probs)
    assert rc == 0
    for g, w in zip(got, wants):
        same(g, w)
    for i in range(0, 64, 9):
        rc, (one,) = device(handle, [probs[i]])
        assert rc == 0
        same(one, got[i])


def test_repeats_bit_identical(handle):
    d = sp.case("n200_default", 3)
    sets = first_sets(d, 3)
    p = pb.pack(d, pb.INITIAL, sets)
    first = device(handle, [p])[1][0]
    for _ in range(3):
        same(device(handle, [p])[1][0], first)


def test_package_api(handle):
    d = sp.case("planar", 4)
    sv = pkg.PnPsolver(d["P3Dw"], d["P2D"], d["sigma2"], d["K"])
    sv.set_ransac_parameters(*d["params"])
    state = pb.INITIAL
    rng = np.random.default_rng(4)
    for c in range(4):
        sets = sets_for(d, rng, state[0], 5)
        want = pb.iterate(d, state, sets)
        got = sv.iterate(5, sets)
        assert (got["Tcw"] is None) == (want["Tcw"] is None)
        if want["Tcw"] is not None:
            assert got["Tcw"].tobytes() == want["Tcw"].tobytes()
        assert got["n_inliers"] == want["n_inliers"] and got["no_more"] == bool(want["no_more"])
        assert sv.iterations == want["iterations_done"] and sv.best_inliers == want["best_inliers"]
        state = pb.next_state(want)
    b = pkg.PnPsolverBatch(max_matches=1024, max_sets=400, max_batch=4)
    svs = [b.solver(sp.case(nm, 5)["P3Dw"], sp.case(nm, 5)["P2D"], sp.case(nm, 5)["sigma2"], sp.K)
           for nm in ("n15", "n50", "repeated")]
    for sv in svs:
        sv.set_ransac_parameters(*sp.RELOC)
    outs = pkg.PnPsolver.iterate_batch(svs, [5] * 3, [first_sets(sp.case(nm, 5), 5) for nm in
                                                      ("n15", "n50", "repeated")], handle=b)
    assert len(outs) == 3 and b.last_ms() > 0


def test_error_codes(handle):
    L = pkg.lib()
    d = sp.case("n50", 0)
    good = pb.pack(d, pb.INITIAL, first_sets(d, 0))
    assert device(handle, [good])[0] == 0
    BAD, CAP = pkg.ERR_BAD_ARG, pkg.ERR_CAPACITY
    h = ctypes.c_void_p()
    assert L.b2s_pnpsolver_create(3, 10, 1, 0, ctypes.byref(h)) == BAD
    assert L.b2s_pnpsolver_create(65537, 10, 1, 0, ctypes.byref(h)) == BAD
    assert L.b2s_pnpsolver_create(64, 10, 65536, 0, ctypes.byref(h)) == BAD  # the batch is a grid's y extent

    def rc_with(**kw):
        p, keep = pb.pack(d, pb.INITIAL, first_sets(d, 0))
        for k, v in kw.items():
            if k == "sets_value":
                keep["sets"][0, 1] = v
            elif k == "sigma":
                keep["sigma2"][3] = v
            else:
                setattr(p, k, v)
        return device(handle, [(p, keep)])[0]

    assert rc_with(min_set=3) == BAD and rc_with(min_set=5) == BAD
    assert rc_with(k=3) == BAD                      # below max_its - iterations_done
    assert rc_with(sets_value=-1) == BAD and rc_with(sets_value=50) == BAD
    assert rc_with(sets_value=int(good[1]["sets"][0, 0])) == BAD  # repeated within its set
    assert rc_with(sigma=-1.0) == BAD and rc_with(sigma=float("nan")) == BAD and rc_with(sigma=float("inf")) == BAD
    assert rc_with(P3Dw=None) == BAD and rc_with(sets=None) == BAD and rc_with(best_Tcw=None) == BAD
    assert rc_with(iterations_done=-1) == BAD and rc_with(best_inliers=-1) == BAD and rc_with(max_its=0) == BAD
    assert rc_with(best_inliers=3) == BAD            # the mask does not hold 3 entries
    assert rc_with(n=5000) == CAP and rc_with(k=401) == CAP
    res = (pkg._PnPsolverResult * 65)()
    P = (pkg._PnPsolverProblem * 65)(*([good[0]] * 65))
    assert L.b2s_pnpsolver_iterate(handle, 65, P, res) == CAP
    assert L.b2s_pnpsolver_iterate(handle, 0, P, res) == BAD
    # nothing is written unless every problem is valid
    r, arrs = pb.new_result(good[0].n)
    bad, keep = pb.pack(d, pb.INITIAL, first_sets(d, 0))
    bad.min_set = 3
    res2 = (pkg._PnPsolverResult * 2)(r, r)
    res2[0].iterations_done = -7
    P2 = (pkg._PnPsolverProblem * 2)(good[0], bad)
    assert L.b2s_pnpsolver_iterate(handle, 2, P2, res2) == BAD and res2[0].iterations_done == -7
    assert np.all(arrs[0] == 7)


needs_drop_in = pytest.mark.skipif(not (os.path.exists(pb.REF_LIB) and os.path.exists(pb.ADP_LIB)),
                                   reason="oracle/_ref not built (make -C oracle -f pnpsolver.mk pnpsolver-ref)")
ROUND = ["n15", "n50", "planar", "repeated", "behind", "no_inliers", "n1000_dense"]


def drop_in_round_robin(path, scenes, seed, rounds):
    """Relocalization's round-robin of iterate(5) after srand(seed) on the library at path: per call, the outputs and
    the state after; stops after the first call that returns a pose (when rand() streams part)."""
    sv = [pb.Ref(d, path) for d in scenes]
    pb.Ref.srand(seed)
    out = []
    for _ in range(rounds):
        for s, r in enumerate(sv):
            o = r.iterate(5)
            o["solver"], o["after"] = s, r.state()
            out.append(o)
            if o["Tcw"] is not None and not o["no_more"]:
                return out
    return out


@needs_drop_in
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_drop_in_matches_reference(seed):
    """host/adapters/PnPsolver_b200.cc against the reference's own PnPsolver in Relocalization's round-robin of
    iterate(5): every call, up to and including the first early return, gives the same Tcw, vbInliers, nInliers,
    bNoMore and the same mnIterations, mnBestInliers, mBestTcw and mvbBestInliers."""
    scenes = [sp.case(nm, seed + 20) for nm in ROUND]
    want = drop_in_round_robin(pb.REF_LIB, scenes, seed, 8)
    got = drop_in_round_robin(pb.ADP_LIB, scenes, seed, 8)
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert (g["Tcw"] is None) == (w["Tcw"] is None)
        if w["Tcw"] is not None:
            assert g["Tcw"].tobytes() == w["Tcw"].tobytes()
        assert np.array_equal(g["inliers"], w["inliers"]) and g["n_inliers"] == w["n_inliers"]
        assert g["no_more"] == w["no_more"]
        a, b = g["after"], w["after"]
        for k in ("iterations", "best_inliers", "min_inliers", "max_its"):
            assert a[k] == b[k], k
        assert (a["best_Tcw"] is None) == (b["best_Tcw"] is None)
        if b["best_Tcw"] is not None:
            assert a["best_Tcw"].tobytes() == b["best_Tcw"].tobytes()
        assert np.array_equal(a["best_mask"], b["best_mask"])


@needs_drop_in
@pytest.mark.parametrize("name", ["no_inliers", "n1000", "behind"])
def test_drop_in_whole_sequence(name):
    """Where no call returns early the draws stay in step: a whole sequence of calls, past bNoMore, is identical."""
    d = sp.case(name, 7)
    res = []
    for path in (pb.REF_LIB, pb.ADP_LIB):
        r = pb.Ref(d, path)
        pb.Ref.srand(7)
        res.append([(r.iterate(n), r.state()) for n in (5, 5, 5, None, 5, 40)])
    for (g, ga), (w, wa) in zip(res[1], res[0]):
        assert (g["Tcw"] is None) == (w["Tcw"] is None)
        if w["Tcw"] is not None:
            assert g["Tcw"].tobytes() == w["Tcw"].tobytes()
        assert np.array_equal(g["inliers"], w["inliers"]) and g["no_more"] == w["no_more"]
        assert ga["iterations"] == wa["iterations"] and ga["best_inliers"] == wa["best_inliers"]
        assert np.array_equal(ga["best_mask"], wa["best_mask"])


@needs_drop_in
def test_drop_in_rand_lead():
    """The documented difference: after an early return at iteration j of the k a call may run, the drop-in has drawn
    4*(k-j) more values from rand() than the reference."""
    d = sp.case("n15", 1)
    r = pb.Ref(d, pb.REF_LIB)
    pb.Ref.srand(3)
    o = r.iterate(5)
    j = r.state()["iterations"]
    assert o["Tcw"] is not None and not o["no_more"]
    k = max(5, d["max_its"])
    after_ref = [pb.Ref.random_int(0, 1 << 30) for _ in range(4 * (k - j) + 1)]
    a = pb.Ref(d, pb.ADP_LIB)
    pb.Ref.srand(3)
    oa = a.iterate(5)
    assert oa["Tcw"].tobytes() == o["Tcw"].tobytes()
    assert pb.Ref.random_int(0, 1 << 30) == after_ref[4 * (k - j)]
    assert k > j  # the case the lead is about
