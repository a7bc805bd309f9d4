"""The handle lifecycle the device stages share (b2s::Stage in csrc/common.cuh, _Handle in the package): argument checks
come before device selection, a failed create leaves *out NULL, destroy(NULL) and a query of a NULL handle are safe,
and every Python handle can be closed twice."""
import ctypes

import numpy as np
import pytest

vp = ctypes.c_void_p
# a three-node vocabulary (k = 2, L = 1): parent, leaf flag, descriptor and weight of each node
VOC = [np.array([-1, 0, 0], np.int32), np.array([0, 1, 1], np.uint8), np.zeros((3, 32), np.uint8), np.ones(3)]


def _voc_desc(pkg):
    return ctypes.byref(pkg._VocDesc(2, 1, len(VOC[0]), *[a.ctypes.data for a in VOC]))


# create entry point, good capacities (an entry may be a function of the package), a bad capacity set, destroy, a query
# that takes a NULL handle: last_ms or a count (and whether it takes an lm_trials pointer)
STAGES = [
    ("b2s_extractor_create", (500, 1.2, 8, 20, 7, 640, 480, 1), (500, 1.2, 8, 20, 7, 640, 480, 0),
     "b2s_extractor_destroy", "b2s_extractor_launch_count", False),
    ("b2s_matcher_create", (1000, 1), (0, 1), "b2s_matcher_destroy", "b2s_matcher_launch_count", False),
    ("b2s_vocabulary_create", (_voc_desc,), (None,), "b2s_vocabulary_destroy", "b2s_vocabulary_words", False),
    ("b2s_ba_create", (4, 16, 64, 1), (0, 16, 64, 1), "b2s_ba_destroy", "b2s_ba_last_kernel_ms", True),
    ("b2s_init_create", (64, 10, 1), (7, 10, 1), "b2s_init_destroy", "b2s_init_last_ms", False),
    ("b2s_sim3solver_create", (64, 10, 1), (2, 10, 1), "b2s_sim3solver_destroy", "b2s_sim3solver_last_ms", False),
    ("b2s_pnpsolver_create", (64, 10, 1), (3, 10, 1), "b2s_pnpsolver_destroy", "b2s_pnpsolver_last_ms", False),
    ("b2s_sim3opt_create", (64, 1), (0, 1), "b2s_sim3opt_destroy", "b2s_sim3opt_last_ms", True),
    ("b2s_eg_create", (16, 16, 16), (0, 16, 16), "b2s_eg_destroy", "b2s_eg_last_ms", True),
    ("b2s_gba_create", (16, 16, 16), (16, 0, 16), "b2s_gba_destroy", "b2s_gba_last_ms", True),
    ("b2s_covis_create", (16, 16, 16, 16, 16, 1), (0, 16, 16, 16, 16, 1), "b2s_covis_destroy", "b2s_covis_last_ms",
     False),
    ("b2s_culling_create", (16, 16, 16, 16, 16, 1), (16, 16, 16, 16, 16, 0), "b2s_culling_destroy",
     "b2s_culling_last_ms", False),
    ("b2s_kfdb_create", (100,), (0,), "b2s_kfdb_destroy", "b2s_kfdb_last_query_ms", False),
]
IDS = [s[0][4:-7] for s in STAGES]


def _create(pkg, name, caps, out):  # on device 0, with the signatures lib() declares
    return getattr(pkg.lib(), name)(*[c(pkg) if callable(c) else c for c in caps], 0, ctypes.byref(out))


@pytest.mark.parametrize("stage", STAGES, ids=IDS)
def test_bad_capacity_is_checked_before_the_device(pkg, stage):
    create, _, bad, *_ = stage
    out = vp(1234)
    assert _create(pkg, create, bad, out) == pkg.ERR_BAD_ARG


@pytest.mark.parametrize("stage", STAGES, ids=IDS)
def test_create_without_a_device(pkg, stage):
    if pkg.device_count() > 0:
        pytest.skip("a CUDA device is present")
    create, good, *_ = stage
    out = vp(1234)
    assert _create(pkg, create, good, out) == pkg.ERR_NO_DEVICE
    assert not out.value


@pytest.mark.parametrize("stage", STAGES, ids=IDS)
def test_null_handle(pkg, stage):
    _, _, _, destroy, last_ms, trials = stage
    L = pkg.lib()
    getattr(L, destroy)(None)
    assert getattr(L, last_ms)(*([None, None] if trials else [None])) == 0.0


def _handles(pkg):
    """One small instance of every handle class, with the borrowers of the *Batch handles."""
    rng = np.random.default_rng(0)
    m = pkg.ORBmatcher()
    geom = dict(mnMinX=0.0, mnMinY=0.0, mnMaxX=640.0, mnMaxY=480.0, bf=0.0, scale_factors=1.2 ** np.arange(8))
    e = np.zeros(0, np.float32)
    grid = pkg.FrameGrid(m, e, e, np.zeros(0, np.int32), e, e, np.zeros((0, 32), np.uint8), geom)
    voc = pkg.ORBVocabulary(2, 1, np.array([-1, 0, 0], np.int32), np.array([0, 1, 1], np.uint8),
                            np.zeros((3, 32), np.uint8), np.ones(3))
    X, K = rng.normal(size=(10, 3)).astype(np.float32) + [0, 0, 5], [500.0, 500.0, 320.0, 240.0]
    s3b, pnpb = pkg.Sim3SolverBatch(max_matches=64, max_sets=10, max_batch=2), pkg.PnPsolverBatch(64, 10, 2)
    return [pkg.ORBextractor(500, 1.2, 8, 20, 7, max_width=640, max_height=480), m, grid, voc,
            pkg.KeyFrameDatabase(100), pkg.Optimizer(max_kf=4, max_mp=16, max_edges=64),
            pkg.GlobalOptimizer(16, 16, 64), pkg.EssentialGraphOptimizer(16, 16, 16), pkg.Sim3Optimizer(64, 1),
            pkg.MonoInitializer(64, 10, 1), pkg.Sim3Solver(X, X, np.ones(10), np.ones(10), K, K, max_sets=10),
            s3b.solver(X, X, np.ones(10), np.ones(10), K, K), s3b,
            pkg.PnPsolver(X, X[:, :2], np.ones(10), K, max_sets=10), pnpb.solver(X, X[:, :2], np.ones(10), K), pnpb,
            pkg.Covisibility(16, 16, 16, 16, 16, 1), pkg.KeyFrameCulling(16, 16, 16, 16, 16, 1)]


@pytest.mark.gpu
def test_close_twice(pkg):
    hs = _handles(pkg)
    assert {type(h) for h in hs} == set(pkg._Handle.__subclasses__())
    for h in hs:
        assert h._h
        h.close()
        h.close()
        assert not h._h
    borrowed = [h for h in hs if not h._own]
    assert len(borrowed) == 2
