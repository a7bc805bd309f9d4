"""One 32-window LocalBA batch (for ncu captures)."""
import sys, time, importlib, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from synth import synth_local_ba
pkg = importlib.import_module('self_commit_orb-slam2_b200')
d = synth_local_ba()
nb = int(sys.argv[1]) if len(sys.argv) > 1 else 32
opt = pkg.Optimizer(max_kf=64, max_mp=5000, max_edges=30000, max_batch=nb)
for _ in range(int(sys.argv[2]) if len(sys.argv) > 2 else 2):
    t = time.perf_counter(); out = opt.LocalBundleAdjustmentBatch([d] * nb); dt = time.perf_counter() - t
    print('batch', nb, 'ms', dt * 1e3, 'trials', out[0]['n_trials'], flush=True)
