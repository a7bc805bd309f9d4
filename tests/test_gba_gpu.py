"""GPU tests of the global bundle adjustment (csrc/gba.cu, pkg.GlobalOptimizer): parity with the CPU restatement on a
map of hundreds of keyframes, bit-identical repeats on a map of 1,500 keyframes, monotone chi2, the error codes, and the
drop-in body (host/adapters/Optimizer_b200.cc) against the reference on one object graph."""
import ctypes
import os

import numpy as np
import pytest

import gba_binding as gb
from synth_gba import synth_global_ba

pytestmark = pytest.mark.gpu


def _prefix_equal(a, b):
    ta, tb = a["trace"][:a["n_trials"]].tolist(), b["trace"][:b["n_trials"]].tolist()
    k = max(min(len(ta), len(tb)) - 8, min(len(ta), len(tb), 5))
    return ta[:k] == tb[:k], ta, tb


def test_device_matches_oracle_large_map(pkg):
    """300 keyframes on a closed loop, ~30k points, ~200k edges, mono / stereo mix, outliers, robust."""
    m = synth_global_ba(n_kf=300, n_mp=30000, obs_range=(4, 10), seed=5, mono_frac=0.3, outlier_frac=0.02)
    d, _, _ = gb.flatten(m)
    assert len(d["edges"]) > 150000
    want = gb.Oracle().global_ba(d, iterations=10, robust=True)
    got = gb.Cuda(pkg).global_ba(d, iterations=10, robust=True)
    ok, ta, tb = _prefix_equal(got, want)
    assert ok, (ta, tb)
    assert np.array_equal(got["point_included"], want["point_included"])
    ok, worst = gb.close(got["Tcw"], want["Tcw"], d["Tcw"])
    assert ok, worst
    ok, worst = gb.close(got["points"], want["points"], d["points"])
    assert ok, worst


def test_large_map_bit_identical_repeats(pkg):
    """A map of 1,500 keyframes: two calls on the same input give bit-identical outputs (no floating-point atomics)."""
    m = synth_global_ba(n_kf=1500, n_mp=60000, obs_range=(2, 6), seed=21, mono_frac=0.2, pert_deg=0.1, pert_t=0.01)
    d, _, _ = gb.flatten(m)
    opt = pkg.GlobalOptimizer(max_kf=2048, max_mp=262144, max_edges=1 << 21)
    a = opt.BundleAdjustment(d, iterations=5, robust=True)
    b = opt.BundleAdjustment(d, iterations=5, robust=True)
    assert a["n_trials"] >= 5
    for k in ("Tcw", "points", "point_included", "trace"):
        assert np.array_equal(a[k], b[k]), k
    assert a["chi2"] == b["chi2"]


def test_accepted_steps_never_raise_chi2(pkg):
    m = synth_global_ba(n_kf=80, n_mp=4000, seed=31, mono_frac=0.5, outlier_frac=0.05, pert_deg=0.5, pert_t=0.1)
    d, _, _ = gb.flatten(m)
    opt = pkg.GlobalOptimizer(max_kf=128, max_mp=8192, max_edges=1 << 16)
    chi = [opt.BundleAdjustment(d, iterations=i, robust=True)["chi2"] for i in range(0, 7)]
    assert all(chi[i + 1] <= chi[i] for i in range(len(chi) - 1)), chi
    assert chi[-1] < chi[0]


def test_capacity_and_bad_arguments(pkg):
    m = synth_global_ba(n_kf=12, n_mp=300, seed=41)
    d, _, _ = gb.flatten(m)
    small = pkg.GlobalOptimizer(max_kf=8, max_mp=512, max_edges=4096)
    with pytest.raises(pkg.B200SlamError) as e:
        small.BundleAdjustment(d)
    assert e.value.code == pkg.ERR_CAPACITY
    opt = pkg.GlobalOptimizer(max_kf=16, max_mp=512, max_edges=4096)
    for how in ("kf_range", "mp_range", "duplicate", "order"):
        bad = dict(d)
        e2 = d["edges"].copy()
        if how == "kf_range":
            e2["kf"][3] = len(d["Tcw"])
        elif how == "mp_range":
            e2["mp"][-1] = len(d["points"])
        elif how == "duplicate":
            e2[1] = e2[0]
        else:
            e2 = e2[::-1].copy()
        bad["edges"] = e2
        with pytest.raises(pkg.B200SlamError) as e:
            opt.BundleAdjustment(bad)
        assert e.value.code == pkg.ERR_BAD_ARG, how
    with pytest.raises(pkg.B200SlamError) as e:
        pkg.GlobalOptimizer(max_kf=0, max_mp=1, max_edges=1)
    assert e.value.code == pkg.ERR_BAD_ARG


@pytest.mark.skipif(not (os.path.exists(gb.REF_LIB) and os.path.exists(gb.ADP_LIB)),
                    reason="oracle/_ref not built (make -C oracle -f gba.mk gba-ref)")
@pytest.mark.parametrize("kw,its,robust,loop_kf", [
    (dict(n_kf=30, n_mp=1500, seed=10, mono_frac=0.3, n_bad_kf=3, n_bad_mp=25, n_excluded_mp=6, edgeless_kf=True), 10,
     True, 0),
    (dict(n_kf=60, n_mp=3000, seed=6), 10, False, 59),
    (dict(n_kf=2, n_mp=300, obs_range=(2, 2), seed=4, mono_frac=1.0, loop=False, pert_deg=0.3, pert_t=0.03), 20, True, 0)])
def test_global_bundle_adjustment_signature(kw, its, robust, loop_kf):
    """Optimizer::GlobalBundleAdjustemnt(Map*, int, bool*, unsigned long, bool): the drop-in body (gather ->
    b2s_global_ba -> scatter) against the reference's own function on one object graph."""
    ref, adp = ctypes.CDLL(gb.REF_LIB), ctypes.CDLL(gb.ADP_LIB)
    m = synth_global_ba(**kw)
    want = gb.call_map(ref.ref_global_ba, m, its, robust, loop_kf)
    got = gb.call_map(adp.adp_global_ba, m, its, robust, loop_kf)
    for k in ("kf_gba", "mp_gba", "kf_ba_global", "mp_ba_global", "mp_updates"):
        assert np.array_equal(got[k], want[k]), k
    assert gb.close(got["Tcw"], want["Tcw"], m["Tcw"])[0]
    assert gb.close(got["points"], want["points"], m["points"])[0]
