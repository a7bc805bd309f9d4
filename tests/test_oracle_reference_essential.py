"""Pins the essential-graph optimisation against the REFERENCE'S OWN Optimizer::OptimizeEssentialGraph
(src/Optimizer.cc:1017-1339 with the vendored g2o and src/Converter.cc, compiled in place -> oracle/_ref/
libref_essential.so, driven on an object graph by oracle/ref_essential_glue.cpp).

Every case runs twice: the CPU restatement (oracle/essential.cpp) and, marked gpu, the CUDA path (csrc/essential.cu
behind pkg.EssentialGraphOptimizer), each on the flattened problem of eg_binding.flatten, scattered back by
eg_binding.expand.  Bar: the same accept / reject sequence of the LM trials up to the converged tail, pose / point
deltas within eg_binding.RTOL of the largest reference delta plus one float32 ulp, and the same
UpdateNormalAndDepth counts."""
import ctypes
import os

import numpy as np
import pytest

import eg_binding as eb
from synth_essential import synth_essential

pytestmark = pytest.mark.skipif(not os.path.exists(eb.REF_LIB),
                                reason="oracle/_ref not built (needs the reference's sources: make -C oracle -f "
                                       "essential.mk essential-ref)")


@pytest.fixture(scope="module")
def ref():
    return ctypes.CDLL(eb.REF_LIB)


@pytest.fixture(params=["oracle", pytest.param("cuda", marks=pytest.mark.gpu)])
def checker(request):
    if request.param == "oracle":
        return eb.Oracle()
    return eb.Cuda(request.getfixturevalue("pkg"))


def run_both(checker, ref, m):
    want = eb.call_map(ref.ref_essential_graph, m)
    d, kf_ids, mp_ids = eb.flatten(m)
    got = eb.expand(m, checker.essential_graph(d), kf_ids, mp_ids)
    return got, want, d


def check(got, want, m):
    """With lambda 1e-16 and numeric Jacobians, a converged graph accepts or rejects its last trials on rounding noise,
    so the traces are compared up to the converged tail (eg_binding.traces_agree)."""
    assert np.array_equal(got["mp_updates"], want["mp_updates"])
    tg, tw = got["trace"][:got["n_trials"]].tolist(), want["trace"][:want["n_trials"]].tolist()
    assert eb.traces_agree(tg, tw), (tg, tw)
    ok, worst = eb.close(got["Tcw"], want["Tcw"], m["Tcw"])
    assert ok, "pose deltas differ from the reference: %g" % worst
    ok, worst = eb.close(got["points"], want["points"], m["points"])
    assert ok, "point deltas differ from the reference: %g" % worst
    return tg, tw


CASES = {
    "stereo_60": lambda: synth_essential(n_kf=60, n_mp=600, seed=1, mono=False),
    "mono_80": lambda: synth_essential(n_kf=80, n_mp=600, seed=2, mono=True),
    "two_closures_mono_120": lambda: synth_essential(n_kf=120, n_mp=800, seed=3, mono=True, closures=2),
    "two_closures_stereo_120": lambda: synth_essential(n_kf=120, n_mp=800, seed=4, mono=False, closures=3),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_essential_graph_matches_reference_source(checker, ref, case):
    m = CASES[case]()
    got, want, d = run_both(checker, ref, m)
    assert want["n_trials"] >= 1
    check(got, want, m)
    assert (m["mp_corrected_by"] == m["cur_kf"]).any() and m["mp_bad"].any()


def test_essential_graph_empty_edge_set(checker, ref):
    """A map of one keyframe: no edge, no iteration; the keyframe and the points are still written back."""
    m = synth_essential(n_kf=1, n_mp=40, seed=5, n_bad_kf=0, n_connected=1)
    m["conn"] = m["conn"][:0]
    got, want, d = run_both(checker, ref, m)
    assert len(d["edges"]) == 0 and want["n_trials"] == 0 and got["n_trials"] == 0
    check(got, want, m)


def test_essential_graph_edgeless_keyframes(checker, ref):
    """Only the loop connections, no tree or covisibility edge: keyframes without an edge keep their Sim3 (inactive
    vertices) and are written back through [R t/s; 0 1]."""
    m = synth_essential(n_kf=30, n_mp=200, seed=6, mono=True)
    m["parent"][:] = -1
    m["cov"] = m["cov"][np.isin(m["cov"][:, 0], m["conn"][:, 0]) & np.isin(m["cov"][:, 1], m["conn"][:, 1])]
    m["loop_edges"] = m["loop_edges"][:0]
    got, want, d = run_both(checker, ref, m)
    assert len(d["edges"]) >= 1
    check(got, want, m)


def test_essential_graph_random_sweep(checker, ref):
    """12 seeded maps up to 300 keyframes, monocular and stereo, one to three closures."""
    for sd in range(12):
        rng = np.random.RandomState(900 + sd)
        m = synth_essential(n_kf=int(rng.randint(12, 301)), n_mp=int(rng.randint(50, 1500)), seed=100 + sd,
                            mono=bool(sd % 2), closures=int(rng.randint(1, 4)), n_bad_kf=int(rng.randint(0, 4)),
                            n_bad_mp=int(rng.randint(0, 6)), drift=float(rng.uniform(0.002, 0.03)),
                            n_connected=int(rng.randint(2, 9)))
        got, want, _ = run_both(checker, ref, m)
        check(got, want, m)


# exp branches: (sigma small, theta small), (sigma small, theta large), (sigma large, theta small), both large
UPDATES = [[1e-7, -2e-7, 3e-7, 0.1, -0.2, 0.3, 1e-7], [0.3, -0.2, 0.5, 0.1, -0.2, 0.3, 2e-6],
           [2e-7, 1e-7, -1e-7, 0.4, 0.1, -0.3, 0.2], [0.4, 0.7, -0.2, -0.5, 0.2, 0.9, -0.3], [0, 0, 0, 0, 0, 0, 0],
           [1.2, -0.9, 2.0, 3.0, -1.0, 0.5, 0.8]]


def _rel(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return float(np.abs(a - b).max() / max(1.0, np.abs(b).max()))


def test_oracle_sim3_matches_reference_header(ref):
    """The oracle's Sim3 exp / log / product / inverse / map agree with g2o::Sim3 of the reference's header to 1e-12
    relative across all exp and log branches."""
    o, g = eb.Sim3Ops(eb._lib(), "orc_sim3_"), eb.Sim3Ops(ref, "ref_sim3_")
    X = np.array([0.3, -1.2, 4.5])
    for u in UPDATES:
        a, b = o.exp(u), g.exp(u)
        assert _rel(a, b) < 1e-12, u
        for v in UPDATES:
            c = o.exp(v)
            assert _rel(o.mul(a, c), g.mul(a, c)) < 1e-12
        assert _rel(o.inverse(a), g.inverse(a)) < 1e-12
        assert _rel(o.map(a, X), g.map(a, X)) < 1e-12
        assert _rel(o.log(a), g.log(a)) < 1e-12, u
        assert _rel(o.log(a), u if np.linalg.norm(u[:3]) < 3 else o.log(a)) < 1e-6
