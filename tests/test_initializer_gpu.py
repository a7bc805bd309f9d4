"""GPU tests of the monocular initialiser (csrc/initializer.cu, pkg.MonoInitializer): parity with the CPU restatement
on every scene of tests/synth_init.py (bit-identical except the parallax, within 1 ulp), a mixed batch against single
calls, bit-identical repeats and the error codes."""
import numpy as np
import pytest

import init_binding as ib
from synth_init import CASES, synth_init
from test_oracle_init import decisions_clear

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ini(pkg):
    o = pkg.MonoInitializer(max_keys=4096, max_iterations=300, max_batch=64)
    yield o
    o.close()


def ulps(a, b):
    a, b = np.asarray(a, np.float32).view(np.int32).astype(np.int64), np.asarray(b, np.float32).view(np.int32)
    return np.abs(a - b.astype(np.int64))


def bits_equal(a, b):
    """Bit-identical arrays (a NaN parallax, from a cos-parallax just above 1, equals itself)."""
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def same(got, want):
    for k in ("ret", "model", "rt_state", "n_matches", "best_h_iter", "best_f_iter"):
        assert got[k] == want[k], k
    for k in ("SH", "SF", "RH", "n_good", "inliers_h", "inliers_f"):
        assert np.array_equal(got[k], want[k]), k
    assert np.array_equal(got["H21"].ravel(), want["H21"]) and np.array_equal(got["F21"].ravel(), want["F21"])
    gp, wp = got["parallax"], want["parallax"]
    assert len(gp) == len(wp) and ((ulps(gp, wp) <= 1) | (np.isnan(gp) & np.isnan(wp))).all()
    if want["ret"]:
        assert np.array_equal(got["R21"].ravel(), want["R21"]) and np.array_equal(got["t21"], want["t21"])
        assert np.array_equal(got["p3d"], want["p3d"])
        assert np.array_equal(got["triangulated"], want["triangulated"].astype(bool))
    else:
        assert got["p3d"] is None and got["triangulated"] is None


@pytest.mark.parametrize("case", sorted(CASES))
def test_device_matches_oracle(ini, case):
    d = synth_init(**CASES[case])
    same(ini.Initialize(d), ib.oracle(d))


def test_batch_equals_single_calls(ini):
    rng = np.random.default_rng(0)
    kinds = ["planar", "general", "rotation", "ambiguous"]
    ds = [synth_init(n=int(n), seed=200 + i, kind=kinds[i % 4], outliers=float(rng.uniform(0, 0.45)),
                     iterations=int(rng.choice([1, 50, 200, 300])))
          for i, n in enumerate(rng.integers(8, 1200, 64))]
    batch = ini.InitializeBatch(ds)
    assert ini.last_ms() > 0
    for d, b in zip(ds, batch):
        decisions_clear(ib.oracle(d))
        s = ini.Initialize(d)
        for k, v in s.items():
            if v is None:
                assert b[k] is None, k
            else:
                assert bits_equal(v, b[k]), k
        same(b, ib.oracle(d))


def test_repeats_are_bit_identical(ini):
    d = synth_init(**CASES["general_3000"])
    a, b = ini.Initialize(d), ini.Initialize(d)
    assert a["ret"] == 1
    for k, v in a.items():
        assert bits_equal(v, b[k]), k


def test_capacity_and_bad_arguments(pkg):
    small = pkg.MonoInitializer(max_keys=256, max_iterations=50, max_batch=2)
    ok = synth_init(n=100, seed=13, iterations=20)

    def code(ds):
        with pytest.raises(pkg.B200SlamError) as e:
            small.InitializeBatch(ds)
        return e.value.code

    assert code([synth_init(n=300, seed=13, iterations=20)]) == pkg.ERR_CAPACITY  # keypoints
    assert code([dict(ok, sets=np.tile(ok["sets"], (3, 1)))]) == pkg.ERR_CAPACITY  # iterations
    assert code([ok, ok, ok]) == pkg.ERR_CAPACITY  # batch
    assert code([]) == pkg.ERR_BAD_ARG
    assert code([dict(ok, sigma=0.0)]) == pkg.ERR_BAD_ARG
    assert code([dict(ok, sets=ok["sets"][:0])]) == pkg.ERR_BAD_ARG
    few = ok["matches12"].copy()
    few[np.flatnonzero(few >= 0)[7:]] = -1
    assert code([dict(ok, matches12=few, sets=np.arange(8, dtype=np.int32)[None])]) == pkg.ERR_BAD_ARG  # 7 matches
    far = ok["matches12"].copy()
    far[np.flatnonzero(far >= 0)[0]] = len(ok["kp2"])
    assert code([dict(ok, matches12=far)]) == pkg.ERR_BAD_ARG
    for v in (-1, 100):  # 100 matched keypoints: indices 0..99
        sets = ok["sets"].copy()
        sets[3, 2] = v
        assert code([dict(ok, sets=sets)]) == pkg.ERR_BAD_ARG
    sets = ok["sets"].copy()
    sets[5, 7] = sets[5, 0]
    assert code([dict(ok, sets=sets)]) == pkg.ERR_BAD_ARG
    # a bad problem anywhere in the batch: nothing is run
    assert code([ok, dict(ok, sigma=-1.0)]) == pkg.ERR_BAD_ARG
    assert small.Initialize(ok)["n_matches"] == 100
    with pytest.raises(pkg.B200SlamError) as e:
        pkg.MonoInitializer(max_keys=4, max_iterations=1, max_batch=1)
    assert e.value.code == pkg.ERR_BAD_ARG
    small.close()


@pytest.mark.skipif(not (__import__("os").path.exists(ib.REF_LIB) and __import__("os").path.exists(ib.ADP_LIB)),
                    reason="oracle/_ref not built (make -C oracle -f init.mk init-ref)")
@pytest.mark.parametrize("case", sorted(CASES))
def test_drop_in_matches_reference(case):
    """host/adapters/Initializer_b200.cc against the reference's own Initializer on the same Frames after srand(0):
    the same mvSets, return value, R21, t21, vP3D and vbTriangulated, and the same state left on failure."""
    d = synth_init(**CASES[case])
    want = ib.call_initialize(ib.REF_LIB, "ref_initialize", d)
    got = ib.call_initialize(ib.ADP_LIB, "adp_initialize", d)
    assert np.array_equal(got["sets"], want["sets"])
    assert got["ret"] == want["ret"] and got["rt_state"] == want["rt_state"]
    if want["rt_state"] == 1:
        assert np.array_equal(got["R21"], want["R21"]) and np.array_equal(got["t21"], want["t21"])
    assert np.array_equal(got["p3d"], want["p3d"])
    assert np.array_equal(got["triangulated"], want["triangulated"])
