"""One batch of 32 DIFFERENT LocalBA windows (bench.py's set)."""
import sys, time, importlib, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
import importlib.util
spec = importlib.util.spec_from_file_location("bench", os.path.join(ROOT, "bench.py")); b = importlib.util.module_from_spec(spec); spec.loader.exec_module(b)
pkg = importlib.import_module('self_commit_orb-slam2_b200')
ws = b.ba_windows(32)
opt = pkg.Optimizer(max_kf=max(w["n_kf"] for w in ws), max_mp=max(len(w["points"]) for w in ws), max_edges=max(len(w["edges"]) for w in ws), max_batch=32)
for _ in range(2):
    t = time.perf_counter(); out = opt.LocalBundleAdjustmentBatch(ws); dt = time.perf_counter() - t
    print('batch ms', dt * 1e3, 'kernel', opt.last_kernel_ms(), flush=True)
print([(w["n_kf"], w["n_local"]) for w in ws])
