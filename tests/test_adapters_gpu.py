"""The drop-in adapters with the reference's exact C++ signatures (self_commit_orb-slam2_b200/host/adapters) against the
reference's own functions, on ONE object graph.

oracle/ref_optimizer_glue.cpp builds stand-in KeyFrame / MapPoint / Map / Frame objects (refshim/slam_stubs_optimizer.h)
from a flattened problem and calls `Optimizer::LocalBundleAdjustment(KeyFrame*, bool*, Map*)` /
`Optimizer::PoseOptimization(Frame*)`.  Linked with the reference's src/Optimizer.cc + g2o that is
oracle/_ref/libref_optimizer.so; linked with host/adapters/Optimizer_b200.cc (gather -> b2s_local_ba /
b2s_pose_optimization -> scatter) it is oracle/_ref/libadapter_optimizer.so.  Both are built where /root/reference is
mounted (the adapter includes the reference's own include/Optimizer.h) and travel to the GPU box.

Required: the same keyframe <-> map point observations erased (EraseMapPointMatch / EraseObservation), the same SetPose /
SetWorldPos values within the parity bar, the same mvbOutlier flags and inlier count."""
import ctypes
import os

import numpy as np
import pytest

from oracle_binding import call_local_ba, call_pose_optimization, call_ref_local_ba
from synth import synth_local_ba, synth_pose_problem

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "libref_optimizer.so")
ADP = os.path.join(ROOT, "oracle", "_ref", "libadapter_optimizer.so")
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not (os.path.exists(REF) and os.path.exists(ADP)),
                                                  reason="oracle/_ref not built (make -C oracle ref)")]
RTOL = 1e-5


def _close(got, want, init):
    got, want, init = (np.asarray(a, np.float64) for a in (got, want, init))
    scale = max(np.abs(want - init).max(), 1e-12)
    ulp = np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
    return bool((np.abs(got - want) <= RTOL * scale + ulp).all())


@pytest.fixture(scope="module")
def libs():
    return ctypes.CDLL(REF), ctypes.CDLL(ADP)


@pytest.mark.parametrize("kw", [dict(n_kf=8, n_fixed=2, n_mp=200, obs_per_mp=4, seed=5),
                                dict(n_kf=12, n_fixed=3, n_mp=600, obs_per_mp=5, seed=7, mono_frac=0.4),
                                dict(n_kf=50, n_fixed=10, n_mp=5000, obs_per_mp=6, seed=42),
                                # a free current keyframe; behind the unobserved first keyframe of call_ref_local_ba the
                                # adapter's window has 128 keyframes, 126 of them free, and it grows its handle to 128
                                dict(n_kf=127, n_fixed=1, n_mp=1500, obs_per_mp=4, seed=128, fix_first=False)])
def test_local_bundle_adjustment_signature(libs, kw):
    ref, adp = libs
    d = synth_local_ba(**kw)
    want = call_ref_local_ba(ref.ref_local_ba, d)
    got = call_ref_local_ba(adp.adp_local_ba, d)
    assert np.array_equal(got["outlier"], want["outlier"])  # the same observations are erased
    assert _close(got["Tcw"], want["Tcw"], d["Tcw"][:d["n_local"]])
    assert _close(got["points"], want["points"], d["points"])


def test_local_bundle_adjustment_stop_flag(libs):
    ref, adp = libs
    d = synth_local_ba(n_kf=8, n_fixed=2, n_mp=200, obs_per_mp=4, seed=5)
    stop = np.ones(1, np.uint8)
    assert call_local_ba(ref.ref_local_ba, d, stop) is None
    assert call_local_ba(adp.adp_local_ba, d, stop) is None  # nothing written back (src/Optimizer.cc:858-860)


@pytest.mark.parametrize("seed,kw", [(23, {}), (25, dict(outlier_frac=0.4)), (27, dict(mono_frac=1.0)),
                                     (26, dict(n=12, mp_frac=0.7)), (29, dict(n=40, mp_frac=0.0))])
def test_pose_optimization_signature(libs, seed, kw):
    ref, adp = libs
    d = synth_pose_problem(seed=seed, **kw)
    want = call_pose_optimization(ref.ref_pose_optimization, d)
    got = call_pose_optimization(adp.adp_pose_optimization, d)
    assert got["n_inliers"] == want["n_inliers"]
    assert np.array_equal(got["outlier"], want["outlier"])
    assert _close(got["Tcw"], want["Tcw"], d["Tcw"])
