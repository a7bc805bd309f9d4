"""Pins the global bundle adjustment against the REFERENCE'S OWN Optimizer::GlobalBundleAdjustemnt / BundleAdjustment
(src/Optimizer.cc:55-341 with the vendored g2o and src/Converter.cc, compiled in place -> oracle/_ref/libref_gba.so,
driven on an object graph by oracle/ref_gba_glue.cpp).

Every case runs twice: the CPU restatement (oracle/gba.cpp) and, marked gpu, the CUDA path (csrc/gba.cu behind
pkg.GlobalOptimizer), each on the flattened problem the drop-in body gathers (gba_binding.flatten), its result scattered
back the way the drop-in body does it (gba_binding.expand).  Bar, as for LocalBA: the same accept / reject sequence of the
LM trials (on the sweep: up to the converged tail), pose / point deltas within 1e-5 relative plus one float32 ulp, the same
excluded points and the same choice between SetPose / SetWorldPos (nLoopKF == 0) and mTcwGBA / mPosGBA with
mnBAGlobalForKF = nLoopKF."""
import ctypes
import os

import numpy as np
import pytest

import gba_binding as gb
from synth_gba import synth_global_ba

pytestmark = pytest.mark.skipif(not os.path.exists(gb.REF_LIB),
                                reason="oracle/_ref not built (needs the reference's sources: make -C oracle -f gba.mk gba-ref)")


@pytest.fixture(scope="module")
def ref():
    return ctypes.CDLL(gb.REF_LIB)


@pytest.fixture(params=["oracle", pytest.param("cuda", marks=pytest.mark.gpu)])
def checker(request):
    if request.param == "oracle":
        return gb.Oracle()
    return gb.Cuda(request.getfixturevalue("pkg"))


def run_both(checker, ref, m, iterations, robust, loop_kf, stop=None):
    want = gb.call_map(ref.ref_global_ba, m, iterations, robust, loop_kf, stop)
    d, kf_ids, mp_ids = gb.flatten(m)
    got = gb.expand(m, checker.global_ba(d, iterations, robust, stop), kf_ids, mp_ids, loop_kf)
    return got, want


def check(got, want, m, exact_trace=True):
    for k in ("kf_gba", "mp_gba", "kf_ba_global", "mp_ba_global", "mp_updates"):
        assert np.array_equal(got[k], want[k]), k
    tg, tw = got["trace"][:got["n_trials"]].tolist(), want["trace"][:want["n_trials"]].tolist()
    if exact_trace:
        assert tg == tw, (tg, tw)
    ok, worst = gb.close(got["Tcw"], want["Tcw"], m["Tcw"])
    assert ok, "pose deltas differ from the reference: %g" % worst
    ok, worst = gb.close(got["points"], want["points"], m["points"])
    assert ok, "point deltas differ from the reference: %g" % worst
    return tg, tw


CASES = {
    # Tracking::CreateInitialMapMonocular (src/Tracking.cc:1081): two keyframes, monocular, 20 iterations, Huber on
    "monocular_init": (lambda: synth_global_ba(n_kf=2, n_mp=300, obs_range=(2, 2), seed=4, mono_frac=1.0, loop=False,
                                               pert_deg=0.3, pert_t=0.03), 20, True, 0),
    # LoopClosing::RunGlobalBundleAdjustment (src/LoopClosing.cc:880-895): stereo, 10 iterations, no robust kernel
    "stereo_loop_60": (lambda: synth_global_ba(n_kf=60, n_mp=3000, seed=6), 10, False, 59),
    "mixed_robust_40": (lambda: synth_global_ba(n_kf=40, n_mp=2500, seed=8, mono_frac=0.5, outlier_frac=0.05), 10, True, 39),
    "bad_objects": (lambda: synth_global_ba(n_kf=30, n_mp=1500, seed=10, mono_frac=0.3, n_bad_kf=3, n_bad_mp=25,
                                            n_excluded_mp=6, edgeless_kf=True), 10, True, 0),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_global_ba_matches_reference_source(checker, ref, case):
    make, its, robust, loop_kf = CASES[case]
    m = make()
    got, want = run_both(checker, ref, m, its, robust, loop_kf)
    assert want["n_trials"] >= 2
    check(got, want, m)
    if case == "bad_objects":
        d, _, _ = gb.flatten(m)
        counts = np.bincount(d["edges"]["kf"], minlength=len(d["Tcw"]))
        assert (counts == 0).any()  # an edgeless keyframe (inactive vertex) is written back unchanged up to rounding
        assert (want["mp_updates"] == 0).sum() > m["mp_bad"].sum()  # points whose observers are all bad are excluded


def test_global_ba_stop_flag_before_call(checker, ref):
    """pbStopFlag already set: no iteration runs, the write-back still happens (every keyframe through Converter)."""
    m = synth_global_ba(n_kf=20, n_mp=800, seed=12)
    stop = np.ones(1, np.uint8)
    got, want = run_both(checker, ref, m, 10, True, 19, stop)
    assert want["n_trials"] == 0 and got["n_trials"] == 0
    check(got, want, m)
    assert want["kf_gba"].all()


def test_global_ba_empty_map(checker, ref):
    """No edge at all: g2o optimises nothing; the keyframes are still written back."""
    m = synth_global_ba(n_kf=5, n_mp=50, seed=13, loop=False)
    m["obs"] = m["obs"][:0]
    got, want = run_both(checker, ref, m, 10, True, 0)
    assert want["n_trials"] == 0 and got["n_trials"] == 0
    check(got, want, m)
    assert not want["mp_updates"].any()


def test_global_ba_random_sweep(checker, ref):
    """16 small random maps (open and closed trajectories, mono / stereo mixes, robust or not, outliers, bad objects,
    strongly perturbed starts): outputs within the bar; the trace identical up to the converged tail."""
    exact = 0
    for sd in range(16):
        rng = np.random.RandomState(500 + sd)
        nkf = int(rng.randint(3, 25))
        m = synth_global_ba(n_kf=nkf, n_mp=int(rng.randint(60, 600)), obs_range=(2, int(rng.randint(2, 11))), seed=sd,
                            mono_frac=float(rng.choice([0, 0.3, 1.0])), outlier_frac=float(rng.choice([0, 0.05])),
                            loop=bool(rng.uniform() < 0.5) and nkf >= 12, n_bad_kf=int(rng.randint(0, 2)) if nkf > 3 else 0,
                            n_bad_mp=int(rng.randint(0, 5)), pert_deg=float(rng.uniform(0.05, 1.0)),
                            pert_t=float(rng.uniform(0.01, 0.3)), pert_p=float(rng.uniform(0.01, 0.5)))
        its, robust, loop_kf = int(rng.choice([5, 10, 20])), bool(rng.uniform() < 0.5), int(rng.choice([0, nkf - 1]))
        got, want = run_both(checker, ref, m, its, robust, loop_kf)
        tg, tw = check(got, want, m, exact_trace=False)
        k = max(min(len(tg), len(tw)) - 8, min(len(tg), len(tw), 5))
        assert tg[:k] == tw[:k], (sd, tg, tw)
        exact += tg == tw
    assert exact >= 12
