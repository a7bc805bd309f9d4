"""GPU tests of OptimizeSim3 (csrc/sim3opt.cu, pkg.Sim3Optimizer): parity with the CPU restatement on every branch,
the fixed scale, a batch against single calls, bit-identical repeats, the error codes, and the drop-in body
(host/adapters/Optimizer_b200.cc) against the reference on one object graph."""
import ctypes
import os

import numpy as np
import pytest

import sim3_binding as sb
from synth_sim3 import CASES, expand, flatten, synth_sim3
from test_oracle_reference_sim3 import converged_tail

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def opt(pkg):
    o = pkg.Sim3Optimizer(max_matches=2048, max_batch=64)
    yield o
    o.close()


@pytest.mark.parametrize("case", sorted(CASES))
def test_device_matches_oracle(opt, case):
    sc = synth_sim3(**CASES[case])
    d, _ = flatten(sc)
    want = sb.oracle(d)
    got = opt.OptimizeSim3(d)
    assert got["n_inliers"] == want["n_inliers"]
    assert np.array_equal(got["keep"], want["keep"])
    tg, tw = got["trace"][:got["n_trials"]].tolist(), want["trace"][:want["n_trials"]].tolist()
    assert converged_tail(tg, tw), (tg, tw)
    ok, worst = sb.s12_close(got["S12"], want["S12"], sc["S12"], sb.RTOL_DEVICE)
    assert ok, worst


def test_fix_scale_keeps_the_scale(opt):
    sc = synth_sim3(n=300, seed=11, mono=False, outliers=0.1)
    d, _ = flatten(sc)
    d["S12"] = d["S12"].copy()
    d["S12"][7] = 1.0625
    got = opt.OptimizeSim3(d)
    assert got["n_inliers"] > 0
    assert got["S12"][7] == 1.0625
    assert not np.array_equal(got["S12"], d["S12"])


def test_batch_equals_single_calls(opt):
    ds = [flatten(synth_sim3(n=int(n), seed=100 + i, mono=bool(i % 2), outliers=0.2))[0]
          for i, n in enumerate(np.random.default_rng(0).integers(12, 600, 64))]
    batch = opt.OptimizeSim3Batch(ds)
    for d, b in zip(ds, batch):
        s = opt.OptimizeSim3(d)
        for k in ("S12", "keep", "trace"):
            assert np.array_equal(s[k], b[k]), k
        assert (s["n_inliers"], s["n_trials"]) == (b["n_inliers"], b["n_trials"])
    ms, trials = opt.last_ms()
    assert ms > 0 and trials == batch[-1]["n_trials"]


def test_repeats_are_bit_identical(opt):
    d, _ = flatten(synth_sim3(n=1500, seed=12, mono=True, outliers=0.25))
    a, b = opt.OptimizeSim3(d), opt.OptimizeSim3(d)
    assert a["n_trials"] >= 1
    for k in ("S12", "keep", "trace"):
        assert np.array_equal(a[k], b[k]), k
    assert a["n_inliers"] == b["n_inliers"]


def test_capacity_and_bad_arguments(pkg):
    d, _ = flatten(synth_sim3(n=100, seed=13))
    small = pkg.Sim3Optimizer(max_matches=32, max_batch=2)
    with pytest.raises(pkg.B200SlamError) as e:
        small.OptimizeSim3(d)
    assert e.value.code == pkg.ERR_CAPACITY
    ok = flatten(synth_sim3(n=20, seed=14))[0]
    with pytest.raises(pkg.B200SlamError) as e:
        small.OptimizeSim3Batch([ok, ok, ok])
    assert e.value.code == pkg.ERR_CAPACITY
    for th2 in (0.0, -1.0):
        bad = dict(ok, th2=th2)
        with pytest.raises(pkg.B200SlamError) as e:
            small.OptimizeSim3(bad)
        assert e.value.code == pkg.ERR_BAD_ARG
    with pytest.raises(pkg.B200SlamError) as e:
        small.OptimizeSim3Batch([])
    assert e.value.code == pkg.ERR_BAD_ARG
    L = pkg.lib()
    p, r = sb.Problem(), sb.Result()
    p.n, p.th2 = 5, 10.0  # null arrays with n > 0
    assert L.b2s_optimize_sim3(small._h, 1, ctypes.byref(p), ctypes.byref(r)) == pkg.ERR_BAD_ARG
    p.n = -1
    assert L.b2s_optimize_sim3(small._h, 1, ctypes.byref(p), ctypes.byref(r)) == pkg.ERR_BAD_ARG
    with pytest.raises(pkg.B200SlamError) as e:
        pkg.Sim3Optimizer(max_matches=0, max_batch=1)
    assert e.value.code == pkg.ERR_BAD_ARG


@pytest.mark.skipif(not (os.path.exists(sb.REF_LIB) and os.path.exists(sb.ADP_LIB)),
                    reason="oracle/_ref not built (make -C oracle -f sim3opt.mk sim3opt-ref)")
@pytest.mark.parametrize("case", ["mono_400_outliers", "stereo_200_outliers", "mono_12_early"])
def test_optimize_sim3_signature(case):
    """Optimizer::OptimizeSim3(KeyFrame*, KeyFrame*, vector<MapPoint*>&, g2o::Sim3&, const float, const bool): the
    drop-in body (gather -> b2s_optimize_sim3 -> scatter) against the reference's own function on one object graph."""
    sc = synth_sim3(**CASES[case])
    want = sb.call_graph(ctypes.CDLL(sb.REF_LIB).ref_optimize_sim3, sc)
    got = sb.call_graph(ctypes.CDLL(sb.ADP_LIB).adp_optimize_sim3, sc)
    assert got["ret"] == want["ret"]
    assert np.array_equal(got["kept"], want["kept"])
    ok, worst = sb.s12_close(got["S12"], want["S12"], sc["S12"], sb.RTOL)
    assert ok, worst
    # the drop-in body's gather is the Python one
    d, idx = flatten(sc)
    flat = sb.oracle(d)
    assert np.array_equal(expand(sc, flat["keep"], idx), got["kept"])
