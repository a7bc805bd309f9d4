"""LocalBundleAdjustment against the reference's own source across what the C ABI accepts and a running system sends it:
windows up to the 128-keyframe capacity of b2s_ba_create (127 free poses, a 762-row reduced camera system, 24 Cholesky
block columns), a free current keyframe (every LocalBA after the map's first keyframe), non-banded covisibility
(shuffled keyframe ids, a path that comes back over the same ground), the first LocalBA calls of a map (1 and 2 free
poses) and points with a single observation (the close points a stereo keyframe creates).

Every case runs twice (conftest.py `checker`): oracle vs reference source on the CPU, and, marked gpu, the CUDA kernels
vs the reference source directly.  The bar is that of test_oracle_reference_optimizer.py: identical LM accept / reject
sequence, identical outlier sets, pose / landmark deltas within 1e-5 relative (+ 1 float32 ulp).

A window with a free keyframe 0 reaches the reference behind a fixed, unobserved first keyframe
(oracle_binding.call_ref_local_ba); the oracle and the CUDA path get the window as it is."""
import ctypes
import os

import numpy as np
import pytest

from oracle_binding import call_ref_local_ba
from synth import synth_local_ba, synth_local_ba_fast
from test_oracle_reference_optimizer import _check_ba, _result_equal_ba

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "oracle", "_ref", "libref_optimizer.so")
pytestmark = pytest.mark.skipif(not os.path.exists(LIB), reason="oracle/_ref not built (needs /root/reference: make -C oracle ref)")


@pytest.fixture(scope="module")
def ref():
    return ctypes.CDLL(LIB)


def _shuffled(d, seed):
    """Local keyframe ids permuted (keyframe 0 stays in place when it is the fixed first keyframe): the covisibility
    pattern of the reduced system is scattered instead of banded."""
    rng = np.random.RandomState(seed)
    nl = d["n_local"]
    first = 1 if d["fixed"][0] else 0
    perm = np.arange(d["n_kf"])
    perm[first:nl] = first + rng.permutation(nl - first)  # new index -> old index
    inv = np.argsort(perm)
    d["Tcw"] = np.ascontiguousarray(d["Tcw"][perm])
    d["fixed"] = np.ascontiguousarray(d["fixed"][perm])
    d["edges"]["kf"] = inv[d["edges"]["kf"]].astype(np.int32)
    return d


def _single_observations(d, every, mono_every=0):
    """Every `every`-th point keeps only its first observation; of those, every `mono_every`-th observation is made
    monocular (its 3x3 Hessian block then has rank 2, and only the Levenberg damping keeps it invertible)."""
    E = d["edges"]
    first = np.r_[True, E["mp"][1:] != E["mp"][:-1]]
    single = E["mp"] % every == 0
    E = E[~single | first].copy()
    if mono_every:
        m = (E["mp"] % (every * mono_every) == 0)
        E["obs"][m, 2] = np.float32(-1.0)
    d["edges"] = E
    return d


def _perturbed(d, seed, ps, ts):
    """Strong perturbation of the points and of the free poses' translations (rejected LM trials, early terminations)."""
    rng = np.random.RandomState(seed)
    d["points"] = (d["points"] + rng.normal(0, ps, d["points"].shape)).astype(np.float32)
    T = d["Tcw"].reshape(-1, 4, 4).copy()
    free = np.nonzero(d["fixed"][:d["n_local"]] == 0)[0]
    T[free, :3, 3] += rng.normal(0, ts, (len(free), 3)).astype(np.float32)
    d["Tcw"] = T.reshape(-1, 16)
    return d


CASES = {
    # beyond 64 keyframes (the adapter's default handle) up to the 128-keyframe capacity
    "kf65": lambda: synth_local_ba_fast(n_kf=65, n_fixed=8, n_mp=2000, obs_per_mp=4, seed=65),
    "kf96_free_current": lambda: synth_local_ba_fast(n_kf=96, n_fixed=10, n_mp=3000, obs_per_mp=5, seed=96, fix_first=False),
    # 127 free poses: 762 rows, 24 block columns of 32
    "kf128_nfree127_first_fixed": lambda: synth_local_ba_fast(n_kf=128, n_fixed=0, n_mp=2500, obs_per_mp=4, seed=128),
    "kf128_nfree127_current_free": lambda: synth_local_ba_fast(n_kf=128, n_fixed=1, n_mp=2500, obs_per_mp=4, seed=127,
                                                               fix_first=False),
    "kf128_all_mono": lambda: synth_local_ba_fast(n_kf=128, n_fixed=8, n_mp=2500, obs_per_mp=5, seed=131, mono_frac=1.0,
                                                  fix_first=False),
    "kf128_shuffled": lambda: _shuffled(synth_local_ba_fast(n_kf=128, n_fixed=6, n_mp=2500, obs_per_mp=5, seed=133,
                                                            fix_first=False), 3),
    "kf128_shuffled_first_fixed": lambda: _shuffled(synth_local_ba_fast(n_kf=128, n_fixed=4, n_mp=2500, obs_per_mp=4,
                                                                        seed=134), 4),
    "kf128_revisit": lambda: synth_local_ba_fast(n_kf=128, n_fixed=6, n_mp=2500, obs_per_mp=6, seed=129, revisit=True,
                                                 fix_first=False),
    # a free current keyframe at the other sizes
    "small_current_free": lambda: synth_local_ba(n_kf=8, n_fixed=2, n_mp=200, obs_per_mp=4, seed=5, fix_first=False),
    "kitti_50_5000_current_free": lambda: synth_local_ba(n_kf=50, n_fixed=10, n_mp=5000, obs_per_mp=6, seed=42,
                                                         fix_first=False),
    "revisit_40_current_free": lambda: synth_local_ba(n_kf=40, n_fixed=6, n_mp=1500, obs_per_mp=6, seed=40, revisit=True,
                                                      fix_first=False),
    # the first LocalBA calls of a map: one and two free poses
    "nfree1_first_fixed": lambda: synth_local_ba(n_kf=2, n_fixed=0, n_mp=150, obs_per_mp=2, seed=61),
    "nfree1_current_free": lambda: synth_local_ba(n_kf=2, n_fixed=1, n_mp=150, obs_per_mp=2, seed=62, fix_first=False),
    "nfree2_first_fixed": lambda: synth_local_ba(n_kf=3, n_fixed=0, n_mp=200, obs_per_mp=3, seed=63, mono_frac=0.3),
    "nfree2_current_free": lambda: synth_local_ba(n_kf=3, n_fixed=1, n_mp=200, obs_per_mp=2, seed=64, fix_first=False),
    # single-observation points: stereo ones mixed with normal points, and a few monocular ones
    "single_obs_stereo": lambda: _single_observations(synth_local_ba(n_kf=12, n_fixed=3, n_mp=600, obs_per_mp=4, seed=71,
                                                                     fix_first=False), 3),
    "single_obs_mono": lambda: _single_observations(synth_local_ba(n_kf=12, n_fixed=3, n_mp=600, obs_per_mp=4, seed=72),
                                                    3, mono_every=40),
    "kf128_single_obs": lambda: _single_observations(synth_local_ba_fast(n_kf=128, n_fixed=4, n_mp=2500, obs_per_mp=5,
                                                                         seed=135, fix_first=False), 4, mono_every=50),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_local_ba_capacity_matches_reference_source(checker, ref, case):
    d = CASES[case]()
    nfree = int((d["fixed"] == 0).sum())
    if case.startswith("kf128_nfree127"):
        assert nfree == 127
    if case.startswith("nfree"):
        assert nfree == int(case[5])
    if case.startswith("single_obs") or case == "kf128_single_obs":
        deg = np.bincount(d["edges"]["mp"])
        assert (deg == 1).sum() >= 100 and (deg > 1).sum() >= 100
        if "mono" in case or case == "kf128_single_obs":
            single = np.nonzero(deg == 1)[0]
            mono = d["edges"]["obs"][np.isin(d["edges"]["mp"], single), 2] < 0
            assert 3 <= mono.sum() <= 20
    want = call_ref_local_ba(ref.ref_local_ba, d)
    assert want["n_trials"] >= 2
    _check_ba(checker.local_ba(d), want, d)


def test_local_ba_capacity_random_sweep(checker, ref):
    """12 random windows of 20-128 keyframes, current keyframe fixed or free, 1-8 observations per point, mono / stereo
    mixes, half of them strongly perturbed.  Poses, landmarks and outlier sets must equal the reference's; the accept /
    reject sequence must agree on the common prefix minus the converged tail (the rule of the reference sweep in
    test_oracle_reference_optimizer.py)."""
    exact = 0
    for sd in range(12):
        rng = np.random.RandomState(3000 + sd)
        nkf = int(rng.randint(20, 129))
        fix_first = bool(rng.randint(0, 2))
        d = synth_local_ba_fast(n_kf=nkf, n_fixed=int(rng.randint(0 if fix_first else 1, max(2, nkf // 4))),
                                n_mp=int(rng.randint(200, 2500)), obs_per_mp=1 + sd % 8, seed=4000 + sd,
                                mono_frac=float(rng.choice([0, 0.3, 1.0])), outlier_frac=float(rng.choice([0, 0.05, 0.2])),
                                fix_first=fix_first)
        if rng.uniform() < 0.5:
            _perturbed(d, 5000 + sd, rng.uniform(0.5, 5), rng.uniform(0.1, 2))
        want = call_ref_local_ba(ref.ref_local_ba, d)
        out = checker.local_ba(d)
        assert _result_equal_ba(out, want, d), "window %d differs from the reference" % sd
        to, tw = out["trace"][:out["n_trials"]].tolist(), want["trace"][:want["n_trials"]].tolist()
        k = max(min(len(to), len(tw)) - 8, min(len(to), len(tw), 5))
        assert to[:k] == tw[:k], (sd, to, tw)
        exact += to == tw
    assert exact >= 9
