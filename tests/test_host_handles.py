"""The host layer's handle policy (self_commit_orb-slam2_b200/host/b2s_host.h), which the drop-ins (host/*.cc and
host/adapters/*.cc) share: the grow-on-demand slot against a fake handle, the device choice, the error line, that every
host/*.cc compiles on its own, and that no stage's result depends on the capacity of the handle it runs on (a slot only
grows, so a call may run on a handle larger than the one it needed)."""
import glob
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "self_commit_orb-slam2_b200", "host")
HARNESS = os.path.join(ROOT, "tests", "cpp", "host_slot_harness.cc")


def _gxx():
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("g++ not found")
    return gxx


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("host_slot") / "host_slot_harness")
    out = subprocess.run([_gxx(), "-std=c++14", "-Wall", "-Wextra", "-Werror", "-I", HOST, "-o", exe, HARNESS],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    assert out.returncode == 0, out.stdout.decode()
    return exe


def _run(exe, what, env=None):
    return subprocess.run([exe, what], stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=env, timeout=60)


@pytest.mark.parametrize("scenario", ["first", "reuse", "grow", "alternate", "failed_create", "destroy_once"])
def test_slot_policy(harness, scenario):
    """first get at the floors; reuse within capacity; growth to max(need, cap, floor) in every dimension; two
    alternating shapes regrow once and then never; a failed create returns its code with no handle and no capacity and
    is retried; every replaced handle is destroyed exactly once."""
    r = _run(harness, scenario)
    assert r.returncode == 0 and r.stdout.decode() == "ok\n", r.stdout.decode()


def test_device_follows_environment(harness):
    env = {k: v for k, v in os.environ.items() if k != "B2S_DEVICE"}
    assert _run(harness, "device", env).stdout.decode() == "0\n"
    assert _run(harness, "device", dict(env, B2S_DEVICE="3")).stdout.decode() == "3\n"


def test_report_and_fail(harness):
    r = _run(harness, "report")
    assert r.stderr.decode() == "who: libb200slam error 3: fake error\n"
    r = _run(harness, "fail")
    assert r.stderr.decode() == "who: libb200slam error 3: fake error\n"
    assert r.stdout.decode() == "fake error\n"


@pytest.mark.parametrize("source", sorted(os.path.basename(p) for p in glob.glob(os.path.join(HOST, "*.cc"))))
def test_host_source_compiles(source):
    """Each drop-in under host/ (ORBextractor.cc, ORBVocabulary.cc) compiles warning-free against the C ABI header,
    without OpenCV or the reference's headers."""
    out = subprocess.run([_gxx(), "-std=c++14", "-fsyntax-only", "-Wall", "-Wextra", "-Werror",
                          "-I", os.path.join(ROOT, "include"), os.path.join(HOST, source)],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    assert out.returncode == 0, out.stdout.decode()


# ---- results do not depend on capacity (GPU)

def _assert_bits_equal(a, b, path="out"):
    if isinstance(a, dict):
        assert sorted(a) == sorted(b), path
        for k in a:
            _assert_bits_equal(a[k], b[k], path + "." + k)
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), path
        for i, (x, y) in enumerate(zip(a, b)):
            _assert_bits_equal(x, y, "%s[%d]" % (path, i))
    elif a is None or b is None:
        assert a is None and b is None, path
    else:
        x, y = np.asarray(a), np.asarray(b)
        assert x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes(), path


def _local_ba(pkg):
    from synth import synth_local_ba
    d = synth_local_ba(n_kf=50, n_fixed=10, n_mp=5000, obs_per_mp=6, seed=42, mono_frac=0.3, outlier_frac=0.05)
    caps = [(d["n_kf"], len(d["points"]), len(d["edges"])), (64, 8192, 65536), (128, 8192, 65536)]
    return [pkg.Optimizer(max_kf=k, max_mp=m, max_edges=e).LocalBundleAdjustment(d) for k, m, e in caps]


def _pose(pkg):
    from synth import synth_pose_problem
    d = synth_pose_problem(seed=26, n=800, mp_frac=0.8)
    return [pkg.Optimizer(max_kf=k, max_mp=m, max_edges=e).PoseOptimization(d) for k, m, e in
            [(4, 16, 64), (64, 8192, 65536)]]


def _global_ba(pkg):
    import gba_binding as gb
    from synth_gba import synth_global_ba
    d, _, _ = gb.flatten(synth_global_ba(n_kf=80, n_mp=4000, seed=31, mono_frac=0.5, outlier_frac=0.05, pert_deg=0.5,
                                         pert_t=0.1))
    caps = [(len(d["fixed"]), len(d["points"]), len(d["edges"])), (256, 32768, 262144)]
    return [pkg.GlobalOptimizer(max_kf=k, max_mp=m, max_edges=e).BundleAdjustment(d) for k, m, e in caps]


def _essential(pkg):
    import eg_binding as eb
    from synth_essential import synth_essential
    d, _, _ = eb.flatten(synth_essential(n_kf=300, n_mp=3000, seed=7, mono=True, closures=2, n_bad_kf=3, n_bad_mp=10))
    caps = [(len(d["Siw"]), len(d["edges"]), len(d["points"])), (1024, 16384, 65536)]
    return [pkg.EssentialGraphOptimizer(max_kf=k, max_edges=e, max_mp=m).OptimizeEssentialGraph(d) for k, e, m in caps]


def _sim3opt(pkg):
    from synth_sim3 import flatten, synth_sim3
    d, _ = flatten(synth_sim3(n=300, seed=11, mono=False, outliers=0.1))
    return [pkg.Sim3Optimizer(max_matches=n, max_batch=1).OptimizeSim3(d) for n in (len(d["X1c"]), 4096)]


def _initializer(pkg):
    from synth_init import synth_init
    d = synth_init(n=600, seed=13, iterations=100)
    keys = max(len(d["kp1"]), len(d["kp2"]))
    return [pkg.MonoInitializer(max_keys=k, max_iterations=i, max_batch=1).Initialize(d) for k, i in
            [(keys, len(d["sets"])), (4096, 200)]]


def _sim3solver(pkg):
    import sim3solver_binding as sb
    from synth_sim3solver import CASES, problem, scene
    kw, (p, mi, mx) = CASES["loop_60_free"]
    pr = problem(scene(**kw), mi)
    pr["max_its"] = sb.ransac_max_its(len(pr["X1c"]), p, mi, mx)
    n = len(pr["X1c"])
    rng = np.random.default_rng(5)
    sets = np.array([rng.choice(n, 3, replace=False) for _ in range(pr["max_its"])], np.int32).reshape(-1, 3)
    outs = []
    for cap, k in [(n, len(sets)), (1024, 300)]:
        sv = pkg.Sim3Solver(pr["X1c"], pr["X2c"], pr["sigma2_1"], pr["sigma2_2"], pr["K1"], pr["K2"], pr["fix_scale"],
                            max_matches=cap, max_sets=k)
        sv.min_inliers, sv.max_its = pr["min_inliers"], pr["max_its"]
        outs.append([sv.iterate(5, sets), sv.find(sets), (sv.iterations, sv.best_inliers, sv.R, sv.t, sv.s)])
    return outs


def _pnpsolver(pkg):
    import synth_pnp as sp
    d = sp.case("n200_default", 3)
    n = len(d["P3Dw"])
    rng = np.random.default_rng(3)
    sets = np.array([rng.choice(n, 4, replace=False) for _ in range(d["max_its"])], np.int32).reshape(-1, 4)
    outs = []
    for cap, k in [(n, len(sets)), (1024, 300)]:
        sv = pkg.PnPsolver(d["P3Dw"], d["P2D"], d["sigma2"], d["K"], max_matches=cap, max_sets=k)
        sv.set_ransac_parameters(*d["params"])
        outs.append([sv.iterate(5, sets), sv.find(sets), (sv.iterations, sv.best_inliers, sv.best_Tcw, sv.best_mask)])
    return outs


STAGES = {"local_ba": _local_ba, "pose": _pose, "global_ba": _global_ba, "essential_graph": _essential,
          "sim3_optimization": _sim3opt, "initializer": _initializer, "sim3solver": _sim3solver,
          "pnpsolver": _pnpsolver}


@pytest.mark.gpu
@pytest.mark.parametrize("stage", sorted(STAGES))
def test_results_do_not_depend_on_capacity(pkg, stage):
    """One seeded problem on a handle created at exactly its size and on handles at the host layer's floors (or
    larger): every output — poses, points, outlier flags, traces, inlier masks, solver state — is bit-identical."""
    outs = STAGES[stage](pkg)
    for other in outs[1:]:
        _assert_bits_equal(outs[0], other)
