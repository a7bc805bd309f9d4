"""GPU LocalBundleAdjustment at the 128-keyframe capacity in every launch shape, against the CPU oracle (the reference's
own source cannot express batches, SM budgets, iteration counts other than 5 / 10, or several handles): a 762-row window
(127 free poses, current keyframe free) solved by 1-16 CTAs next to small windows, in a batch larger than the SM count,
with other its1 / its2, twice on one handle, alternately with a 16-keyframe handle, and after rejected calls.  The bar
is that of test_localba_gpu.py."""
import numpy as np
import pytest

from synth import synth_local_ba, synth_local_ba_fast
from test_localba_gpu import _check, _num_sms

pytestmark = pytest.mark.gpu


def _big(seed=127):
    """128 keyframes, 127 of them free (keyframe 0 is the free current keyframe, one fixed camera), 10 k stereo edges."""
    d = synth_local_ba_fast(n_kf=128, n_fixed=1, n_mp=2500, obs_per_mp=4, seed=seed, fix_first=False)
    assert (d["fixed"] == 0).sum() == 127
    return d


def _small(n, seed0):
    """n small windows of 5-14 keyframes, alternately with a fixed and a free current keyframe."""
    return [synth_local_ba(n_kf=5 + i % 10, n_fixed=1 + i % 3, n_mp=60 + 20 * (i % 7), obs_per_mp=4, seed=seed0 + i,
                           fix_first=i % 2 == 0) for i in range(n)]


def _hard(seed):
    """Strongly perturbed window with a free current keyframe: rejected trials and early terminations."""
    rng = np.random.RandomState(seed)
    d = synth_local_ba(n_kf=20, n_fixed=4, n_mp=600, obs_per_mp=5, seed=seed, outlier_frac=0.1, fix_first=False)
    d["points"] = (d["points"] + rng.normal(0, 12.0, d["points"].shape)).astype(np.float32)
    T = d["Tcw"].reshape(-1, 4, 4).copy()
    T[:d["n_local"], :3, 3] += rng.normal(0, 3.0, (d["n_local"], 3)).astype(np.float32)
    d["Tcw"] = T.reshape(-1, 16)
    return d


def _handle(pkg, ds, max_kf=128):
    return pkg.Optimizer(max_kf=max_kf, max_mp=max(len(d["points"]) for d in ds),
                         max_edges=max(len(d["edges"]) for d in ds), max_batch=len(ds))


@pytest.mark.parametrize("budget", [0, 2, 5])
def test_big_window_in_batch_sm_budget(pkg, oracle, budget):
    """The 128-keyframe window next to three small ones: budget 2 leaves it one CTA, 5 two, 0 (all SMs) sixteen."""
    ds = _small(3, 300)
    ds.insert(1, _big())
    opt = _handle(pkg, ds)
    opt.set_sm_budget(budget)
    for d, out in zip(ds, opt.LocalBundleAdjustmentBatch(ds)):
        _check(out, oracle.local_ba(d), d)


def test_big_window_in_batch_larger_than_sms(pkg, oracle):
    """SM count + 4 windows, one CTA each, the 128-keyframe window among them, in two cooperative launches."""
    ds = _small(_num_sms() + 3, 400)
    ds.insert(2, _big())
    opt = _handle(pkg, ds)
    before = opt.launch_count()
    outs = opt.LocalBundleAdjustmentBatch(ds)
    assert opt.launch_count() - before == 5 + -(-len(ds) // _num_sms())
    for d, out in zip(ds, outs):
        _check(out, oracle.local_ba(d), d)


# The 128-keyframe window does not run (10, 20): after 20 and more accepted steps its final chi2 is conditioned at the
# level of the 1e-7 bar itself (moving one input coordinate by one float32 ulp changes the oracle's own value by up to
# 1.1e-7 relative), so that comparison would measure rounding, not the kernel.
@pytest.mark.parametrize("window,its", [("hard", (1, 0)), ("hard", (5, 0)), ("hard", (2, 3)), ("hard", (10, 20)),
                                        ("big", (1, 0)), ("big", (5, 0)), ("big", (2, 3))])
def test_iteration_counts(pkg, oracle, window, its):
    """its1 / its2 other than 5 / 10; its2 = 0 skips round 2, whose active set (the inliers, no robust kernel) still
    defines the final chi2."""
    d = _hard(52) if window == "hard" else _big()
    ref = oracle.local_ba(d, its1=its[0], its2=its[1])
    if window == "hard" and its == (10, 20):
        assert ref["n_trials"] > 15  # more iterations than the 5 + 10 schedule allows
        assert "01" in "".join(map(str, ref["trace"][:ref["n_trials"]].tolist()))  # rejected, then accepted
    out = _handle(pkg, [d]).LocalBundleAdjustment(d, its1=its[0], its2=its[1])
    _check(out, ref, d)


def test_repeat_is_bit_identical(pkg):
    """The same batch twice on one handle: every output bit-identical (fixed-order reductions, no float atomics)."""
    ds = _small(3, 500)
    ds.insert(0, _big())
    opt = _handle(pkg, ds)
    opt.set_sm_budget(7)
    a = opt.LocalBundleAdjustmentBatch(ds)
    a = [{k: np.copy(v) for k, v in o.items()} for o in a]
    b = opt.LocalBundleAdjustmentBatch(ds)
    for oa, ob in zip(a, b):
        assert oa["n_trials"] == ob["n_trials"] and oa["chi2"] == ob["chi2"]
        for k in ("Tcw", "points", "outlier", "trace"):
            assert np.array_equal(oa[k], ob[k]), k


def test_handles_of_different_capacity_alternate(pkg, oracle):
    """A 128-keyframe handle, then a 16-keyframe handle created after it (which lowers the kernel's shared-memory limit),
    used alternately: both keep matching the oracle."""
    big = [_big(127), _big(129)]
    small = _small(2, 600)
    h128 = _handle(pkg, big)
    h16 = _handle(pkg, small, max_kf=16)
    for i in range(2):
        _check(h128.LocalBundleAdjustment(big[i]), oracle.local_ba(big[i]), big[i])
        _check(h16.LocalBundleAdjustment(small[i]), oracle.local_ba(small[i]), small[i])


def test_capacity_errors_leave_handle_usable(pkg, oracle):
    """Windows beyond a handle's capacities and a handle beyond 128 keyframes are rejected with an error; the handle
    keeps working afterwards."""
    ok = synth_local_ba(n_kf=16, n_fixed=3, n_mp=300, obs_per_mp=4, seed=81, fix_first=False)
    opt = pkg.Optimizer(max_kf=16, max_mp=300, max_edges=len(ok["edges"]), max_batch=1)
    bad = {"n_kf": synth_local_ba(n_kf=17, n_fixed=3, n_mp=200, obs_per_mp=4, seed=82),
           "n_mp": synth_local_ba(n_kf=10, n_fixed=3, n_mp=301, obs_per_mp=2, seed=83),
           "n_edges": synth_local_ba(n_kf=16, n_fixed=3, n_mp=300, obs_per_mp=5, seed=84)}
    assert len(bad["n_edges"]["edges"]) > len(ok["edges"])
    for d in bad.values():
        with pytest.raises(pkg.B200SlamError):
            opt.LocalBundleAdjustment(d)
        _check(opt.LocalBundleAdjustment(ok), oracle.local_ba(ok), ok)
    with pytest.raises(pkg.B200SlamError):
        opt.LocalBundleAdjustmentBatch([ok, ok])  # more windows than max_batch
    with pytest.raises(pkg.B200SlamError):
        pkg.Optimizer(max_kf=129, max_mp=300, max_edges=2048)
    _check(opt.LocalBundleAdjustment(ok), oracle.local_ba(ok), ok)
