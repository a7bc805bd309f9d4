"""GPU parity of LocalBundleAdjustment against the CPU oracle: identical LM accept/reject sequence and outlier flags,
pose / landmark deltas within 1e-5 relative (plus one float32 ulp of the written value: both sides cast the FP64
estimate to float like Converter::toCvMat, src/Converter.cc:96-107)."""
import numpy as np
import pytest

from synth import synth_local_ba

pytestmark = pytest.mark.gpu

RTOL = 1e-5


def _close(gpu, ref, init):
    gpu, ref, init = (np.asarray(a, np.float64) for a in (gpu, ref, init))
    delta = np.abs(ref - init)
    scale = max(delta.max(), 1e-12)
    ulp = np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64)
    err = np.abs(gpu - ref)
    ok = err <= RTOL * scale + ulp
    return bool(ok.all()), float((err / scale).max())


def _check(out, ref, d):
    assert ref is not None and out is not None
    tr_g = out["trace"][:out["n_trials"]].tolist()
    tr_o = ref["trace"][:ref["n_trials"]].tolist()
    assert tr_g == tr_o, (tr_g, tr_o)
    assert np.array_equal(out["outlier"], ref["outlier"])
    ok, worst = _close(out["Tcw"], ref["Tcw"], d["Tcw"][:d["n_local"]])
    assert ok, "pose deltas differ: %g" % worst
    ok, worst = _close(out["points"], ref["points"], d["points"])
    assert ok, "landmark deltas differ: %g" % worst
    assert abs(out["chi2"] - ref["chi2"]) <= 1e-7 * abs(ref["chi2"])


def test_local_ba_kitti_window(pkg, oracle):
    d = synth_local_ba(n_kf=50, n_fixed=10, n_mp=5000, obs_per_mp=6, seed=42)
    opt = pkg.Optimizer(max_kf=64, max_mp=8192, max_edges=65536)
    out = opt.LocalBundleAdjustment(d)
    ref = oracle.local_ba(d)
    _check(out, ref, d)
    assert ref["n_trials"] >= 10


def test_local_ba_mixed_mono_stereo(pkg, oracle):
    d = synth_local_ba(n_kf=12, n_fixed=3, n_mp=600, obs_per_mp=5, seed=7, mono_frac=0.4)
    opt = pkg.Optimizer(max_kf=16, max_mp=1024, max_edges=8192)
    _check(opt.LocalBundleAdjustment(d), oracle.local_ba(d), d)


def _hard_problem(sd):
    rng = np.random.RandomState(sd)
    ps, ts = rng.uniform(5, 14), rng.uniform(1, 4)
    d = synth_local_ba(n_kf=10, n_fixed=2, n_mp=300, obs_per_mp=5, seed=3, outlier_frac=0.15)
    d["points"] = (d["points"] + rng.normal(0, ps, d["points"].shape)).astype(np.float32)
    T = d["Tcw"].reshape(-1, 4, 4).copy()
    T[1:d["n_local"], :3, 3] += rng.normal(0, ts, (d["n_local"] - 1, 3)).astype(np.float32)
    d["Tcw"] = T.reshape(-1, 16)
    return d


@pytest.mark.parametrize("sd", [22, 7, 2])
def test_local_ba_rejections(pkg, oracle, sd):
    """Strong perturbations: LM steps get rejected (lambda *= ni, pop/restore), rounds terminate early."""
    d = _hard_problem(sd)
    ref = oracle.local_ba(d)
    if sd in (22, 7):
        tr = "".join(map(str, ref["trace"][:ref["n_trials"]].tolist()))
        assert "01" in tr  # the oracle really exercises reject-then-accept here
    opt = pkg.Optimizer(max_kf=16, max_mp=512, max_edges=4096)
    out = opt.LocalBundleAdjustment(d)
    _check(out, ref, d)


def test_local_ba_stop_flag(pkg, oracle):
    d = synth_local_ba(n_kf=8, n_fixed=2, n_mp=200, obs_per_mp=4, seed=5)
    opt = pkg.Optimizer(max_kf=16, max_mp=512, max_edges=4096)
    stop = np.ones(1, np.uint8)
    assert opt.LocalBundleAdjustment(d, stop=stop) is None  # src/Optimizer.cc:858-860
    assert oracle.local_ba(d, stop=stop) is None
    stop[0] = 0
    _check(opt.LocalBundleAdjustment(d, stop=stop), oracle.local_ba(d, stop=stop), d)


def test_local_ba_batch(pkg, oracle):
    ds = [synth_local_ba(n_kf=10, n_fixed=2, n_mp=300, obs_per_mp=5, seed=11),
          synth_local_ba(n_kf=14, n_fixed=4, n_mp=500, obs_per_mp=6, seed=12, mono_frac=0.2),
          synth_local_ba(n_kf=6, n_fixed=1, n_mp=150, obs_per_mp=4, seed=13)]
    opt = pkg.Optimizer(max_kf=16, max_mp=512, max_edges=4096, max_batch=3)
    outs = opt.LocalBundleAdjustmentBatch(ds)
    for d, out in zip(ds, outs):
        _check(out, oracle.local_ba(d), d)


@pytest.mark.parametrize("budget", [0, 5, 9, 24])
def test_local_ba_batch_sm_budget(pkg, oracle, budget):
    """b2s_ba_set_sm_budget: a batch deals its thread blocks to the windows by estimated cost (1 .. 16 per window); whatever
    the split, every window must reproduce the oracle's LM trace, outlier flags and values."""
    ds = [synth_local_ba(n_kf=12, n_fixed=3, n_mp=400, obs_per_mp=5, seed=21),
          synth_local_ba(n_kf=16, n_fixed=4, n_mp=500, obs_per_mp=7, seed=22, mono_frac=0.2),
          synth_local_ba(n_kf=6, n_fixed=1, n_mp=120, obs_per_mp=4, seed=23),
          synth_local_ba(n_kf=9, n_fixed=2, n_mp=300, obs_per_mp=6, seed=24, outlier_frac=0.05),
          synth_local_ba(n_kf=14, n_fixed=2, n_mp=200, obs_per_mp=4, seed=25)]
    opt = pkg.Optimizer(max_kf=16, max_mp=512, max_edges=4096, max_batch=5)
    opt.set_sm_budget(budget)
    outs = opt.LocalBundleAdjustmentBatch(ds)
    for d, out in zip(ds, outs):
        _check(out, oracle.local_ba(d), d)


def test_local_ba_shuffled_keyframes(pkg, oracle):
    """Keyframe ids permuted: the covisibility pattern of the reduced system is scattered instead of banded, so the
    envelope logic of the Cholesky and the sorted Schur block order see a general structure."""
    d = synth_local_ba(n_kf=30, n_fixed=6, n_mp=1500, obs_per_mp=5, seed=21)
    rng = np.random.RandomState(5)
    nl = d["n_local"]
    perm = np.arange(d["n_kf"])
    perm[1:nl] = 1 + rng.permutation(nl - 1)  # new index -> old index (index 0 stays the fixed origin)
    inv = np.argsort(perm)
    d["Tcw"] = np.ascontiguousarray(d["Tcw"][perm])
    d["fixed"] = np.ascontiguousarray(d["fixed"][perm])
    d["edges"]["kf"] = inv[d["edges"]["kf"]].astype(np.int32)
    opt = pkg.Optimizer(max_kf=32, max_mp=2048, max_edges=8192)
    _check(opt.LocalBundleAdjustment(d), oracle.local_ba(d), d)


def _high_degree_window():
    """High-degree landmarks: the window's covisibility pair list is larger than the initial capacity (8 x max_edges) of
    a handle sized to its edge count."""
    d = synth_local_ba(n_kf=24, n_fixed=2, n_mp=150, obs_per_mp=20, seed=31)
    deg = np.bincount(d["edges"]["mp"][d["fixed"][d["edges"]["kf"]] == 0])
    assert (deg * (deg + 1) // 2).sum() > 8 * len(d["edges"])
    return d


def test_local_ba_pair_list_grows(pkg, oracle):
    """A pair list larger than the initial capacity: the handle grows it on demand."""
    d = _high_degree_window()
    opt = pkg.Optimizer(max_kf=24, max_mp=150, max_edges=len(d["edges"]))
    _check(opt.LocalBundleAdjustment(d), oracle.local_ba(d), d)


def test_local_ba_pair_list_grows_in_reused_handle(pkg, oracle):
    """One handle: the high-degree window alone, then in a batch with two ordinary windows (the per-window stride of the
    grown pair list applies to every window of the batch), then an ordinary window again."""
    hd = _high_degree_window()
    ds = [synth_local_ba(n_kf=10, n_fixed=2, n_mp=150, obs_per_mp=5, seed=11),
          synth_local_ba(n_kf=14, n_fixed=4, n_mp=120, obs_per_mp=6, seed=12, mono_frac=0.2)]
    opt = pkg.Optimizer(max_kf=24, max_mp=150, max_edges=len(hd["edges"]), max_batch=3)
    _check(opt.LocalBundleAdjustment(hd), oracle.local_ba(hd), hd)
    batch = [ds[0], hd, ds[1]]
    for d, out in zip(batch, opt.LocalBundleAdjustmentBatch(batch)):
        _check(out, oracle.local_ba(d), d)
    _check(opt.LocalBundleAdjustment(ds[1]), oracle.local_ba(ds[1]), ds[1])


def _num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _small_windows(n):
    return [synth_local_ba(n_kf=5, n_fixed=1, n_mp=60, obs_per_mp=4, seed=100 + i) for i in range(n)]


def test_local_ba_batch_larger_than_sms(pkg, oracle):
    """More windows than SMs: one CTA per window, consecutive windows packed into ceil(batch / SMs) cooperative
    launches; every window must still reproduce the oracle."""
    ds = _small_windows(_num_sms() + 4)
    opt = pkg.Optimizer(max_kf=8, max_mp=64, max_edges=512, max_batch=len(ds))
    for d, out in zip(ds, opt.LocalBundleAdjustmentBatch(ds)):
        _check(out, oracle.local_ba(d), d)


@pytest.mark.parametrize("batch", ["1", "5", "sms+4"])
def test_local_ba_launch_count(pkg, batch):
    """Five structure kernels, then one cooperative LM launch per group of consecutive windows whose CTAs fit on the
    SMs: one for a batch of at most one window per SM, ceil(batch / SMs) beyond that."""
    sms = _num_sms()
    nb = sms + 4 if batch == "sms+4" else int(batch)
    ds = _small_windows(nb)
    opt = pkg.Optimizer(max_kf=8, max_mp=64, max_edges=512, max_batch=nb)
    before = opt.launch_count()
    opt.LocalBundleAdjustmentBatch(ds)
    assert opt.launch_count() - before == 5 + -(-nb // sms)
