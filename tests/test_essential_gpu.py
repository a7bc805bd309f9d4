"""GPU tests of the essential-graph optimisation (csrc/essential.cu, pkg.EssentialGraphOptimizer): parity with the CPU
restatement on a map of 1,000 keyframes with three closures, bit-identical repeats on 4,096 keyframes, the error codes,
and the drop-in body (host/adapters/Optimizer_b200.cc) against the reference on one object graph."""
import ctypes
import os

import numpy as np
import pytest

import eg_binding as eb
from synth_essential import synth_essential

pytestmark = pytest.mark.gpu


def test_device_matches_oracle_1000_keyframes(pkg):
    """1,000 monocular keyframes, three closures: the run is one accepted step and then rejections, so the outputs are
    the first iteration's linearisation, solve and update; they are held to the oracle at 1e-6."""
    m = synth_essential(n_kf=1000, n_mp=20000, seed=7, mono=True, closures=3, n_bad_kf=5, n_bad_mp=30)
    d, _, _ = eb.flatten(m)
    want = eb.Oracle().essential_graph(d)
    got = eb.Cuda(pkg, max_kf=1024, max_edges=1 << 14, max_mp=1 << 15).essential_graph(d)
    ta, tb = got["trace"][:got["n_trials"]].tolist(), want["trace"][:want["n_trials"]].tolist()
    assert ta == tb and tb[0] == 1 and sum(tb) == 1, (ta, tb)
    assert abs(got["chi2_initial"] - want["chi2_initial"]) <= 1e-9 * want["chi2_initial"]
    assert abs(got["chi2"] - want["chi2"]) <= eb.RTOL_DEVICE * want["chi2"], (got["chi2"], want["chi2"])
    assert got["chi2"] < 0.5 * got["chi2_initial"]
    ok, worst = eb.close(got["Tcw"], want["Tcw"], m["Tcw"][np.where(m["kf_bad"] == 0)[0]], eb.RTOL_DEVICE)
    assert ok, worst
    ok, worst = eb.close(got["points"], want["points"], d["points"], eb.RTOL_DEVICE)
    assert ok, worst


def test_4096_keyframes_bit_identical_repeats(pkg):
    m = synth_essential(n_kf=4096, n_mp=100000, seed=8, mono=False, closures=3)
    d, _, _ = eb.flatten(m)
    opt = pkg.EssentialGraphOptimizer()
    a = opt.OptimizeEssentialGraph(d)
    b = opt.OptimizeEssentialGraph(d)
    assert a["n_trials"] >= 1
    for k in ("Tcw", "points", "trace"):
        assert np.array_equal(a[k], b[k]), k
    assert a["chi2"] == b["chi2"] and a["chi2"] <= a["chi2_initial"]


def test_capacity_and_bad_arguments(pkg):
    m = synth_essential(n_kf=20, n_mp=100, seed=9)
    d, _, _ = eb.flatten(m)
    small = pkg.EssentialGraphOptimizer(max_kf=8, max_edges=1024, max_mp=1024)
    with pytest.raises(pkg.B200SlamError) as e:
        small.OptimizeEssentialGraph(d)
    assert e.value.code == pkg.ERR_CAPACITY
    opt = pkg.EssentialGraphOptimizer(max_kf=32, max_edges=1024, max_mp=1024)
    n = len(d["Siw"])
    for how in ("i_range", "j_range", "self", "fixed", "ref"):
        bad = dict(d)
        e2 = d["edges"].copy()
        if how == "i_range":
            e2["i"][0] = n
        elif how == "j_range":
            e2["j"][1] = -1
        elif how == "self":
            e2["j"][2] = e2["i"][2]
        elif how == "fixed":
            bad["fixed_kf"] = n
        else:
            r = d["ref_kf"].copy()
            r[0] = n
            bad["ref_kf"] = r
        bad["edges"] = e2
        with pytest.raises(pkg.B200SlamError) as e:
            opt.OptimizeEssentialGraph(bad)
        assert e.value.code == pkg.ERR_BAD_ARG, how
    with pytest.raises(pkg.B200SlamError) as e:
        pkg.EssentialGraphOptimizer(max_kf=0, max_edges=1, max_mp=1)
    assert e.value.code == pkg.ERR_BAD_ARG


@pytest.mark.skipif(not (os.path.exists(eb.REF_LIB) and os.path.exists(eb.ADP_LIB)),
                    reason="oracle/_ref not built (make -C oracle -f essential.mk essential-ref)")
@pytest.mark.parametrize("kw", [dict(n_kf=60, n_mp=600, seed=1, mono=False),
                                dict(n_kf=120, n_mp=800, seed=3, mono=True, closures=2),
                                dict(n_kf=1, n_mp=40, seed=5, n_bad_kf=0, n_connected=1)])
def test_optimize_essential_graph_signature(kw):
    """Optimizer::OptimizeEssentialGraph(Map*, KeyFrame*, KeyFrame*, const KeyFrameAndPose&, const KeyFrameAndPose&,
    const map<KeyFrame*, set<KeyFrame*>>&, const bool&): the drop-in body (gather -> b2s_optimize_essential_graph ->
    scatter) against the reference's own function on one object graph."""
    ref, adp = ctypes.CDLL(eb.REF_LIB), ctypes.CDLL(eb.ADP_LIB)
    m = synth_essential(**kw)
    want = eb.call_map(ref.ref_essential_graph, m)
    got = eb.call_map(adp.adp_essential_graph, m)
    assert np.array_equal(got["mp_updates"], want["mp_updates"])
    ok, worst = eb.close(got["Tcw"], want["Tcw"], m["Tcw"])
    assert ok, worst
    ok, worst = eb.close(got["points"], want["points"], m["points"])
    assert ok, worst
    # the drop-in body's gather is the Python one: the same problem gives the same outputs as the flattened call
    d, kf_ids, mp_ids = eb.flatten(m)
    flat = eb.expand(m, eb.Oracle().essential_graph(d), kf_ids, mp_ids)
    assert eb.close(got["Tcw"], flat["Tcw"], m["Tcw"])[0]
