#!/usr/bin/env python3
"""Generates tests/golden/*.npz from the CPU oracle on the deterministic synthetic inputs (tests/synth.py).

The reference ships no golden vectors (SURVEY.md §4) and cannot be built here, so these fixtures freeze the ORACLE
(whose OpenCV-owned stages are pinned to cv2 by tests/test_oracle_cv2.py): they guard against accidental changes of
the oracle and give the GPU box golden data that does not depend on /root/reference.
Run from the repo root:  python tools/make_golden.py
"""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle_binding  # noqa: E402
from synth import synth_descriptors, synth_image, synth_local_ba, synth_projection, synth_projection_map  # noqa: E402

out = os.path.join(ROOT, "tests", "golden")
os.makedirs(out, exist_ok=True)
o = oracle_binding.load()


def sha(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


# extractor, configs[0] (640x480, 1000 features): full arrays
img = synth_image(640, 480, 3)
k, d = o.extractor(1000, 1.2, 8, 20, 7)(img)
np.savez_compressed(os.path.join(out, "extract_640x480_seed3.npz"), kps=k, desc=d, image_sha=sha(img))
# extractor, configs[1] (1241x376, 2000 features): hashes + head
img = synth_image(1241, 376, 3)
k, d = o.extractor(2000, 1.2, 8, 20, 7)(img)
np.savez_compressed(os.path.join(out, "extract_1241x376_seed3.npz"), n=len(k), kps_sha=sha(k), desc_sha=sha(d),
                    kps_head=k[:64], desc_head=d[:64], image_sha=sha(img))
# extractor on uniform noise (dense candidates) at iniThFAST 12 / minThFAST 7: full arrays
from synth import synth_texture  # noqa: E402
img = synth_texture("noise", 640, 480, 3)
k, d = o.extractor(1000, 1.2, 8, 12, 7)(img)
np.savez_compressed(os.path.join(out, "extract_640x480_noise_12_7.npz"), kps=k, desc=d, image_sha=sha(img))
# SearchByBoW
for nodes in (100, 1):
    A, nA, vA, aA, B, nB, aB = synth_descriptors(2000, seed=1234 + nodes, n_nodes=nodes)
    n, m = o.search_by_bow(A, nA, vA, aA, B, nB, aB, nnratio=0.7)
    np.savez_compressed(os.path.join(out, "bow_2000_nodes%d.npz" % nodes), n=n, match=m, input_sha=sha(A, B, nA, nB, aA, aB))
# SearchByProjection
pd = synth_projection(seed=21, cluster=False, th=7.0)
n, m = o.search_by_projection_last(pd["q"], pd["kpx"], pd["kpy"], pd["octave"], pd["angle"], pd["uright"], pd["occupied"],
                                   pd["desc"], pd["geom"], float(pd["th"]), mode=0)
np.savez_compressed(os.path.join(out, "proj_seed21.npz"), n=n, match=m)
# SearchByProjection (local map points)
pm = synth_projection_map(seed=31)
n, m = o.search_by_projection_map(pm["q"], pm["kpx"], pm["kpy"], pm["octave"], pm["uright"], pm["occupied"], pm["desc"],
                                  pm["geom"], th=1.0, nnratio=0.8)
np.savez_compressed(os.path.join(out, "projmap_seed31.npz"), n=n, match=m)
# LocalBA (small window: exact float outputs; KITTI-shaped window: hashes of flags + trace)
ba = synth_local_ba(n_kf=8, n_fixed=2, n_mp=200, obs_per_mp=4, seed=5)
r = o.local_ba(ba)
np.savez_compressed(os.path.join(out, "localba_small_seed5.npz"), Tcw=r["Tcw"], points=r["points"], outlier=r["outlier"],
                    trace=r["trace"], n_trials=r["n_trials"], chi2=r["chi2"])
print("golden fixtures written to", out)
# ComputeStereoMatches (written by tests/test_oracle_stereo.py::_run with the same arguments)
from test_oracle_stereo import _run as _stereo_run  # noqa: E402
_, n, ur, dp = _stereo_run(o, 640, 480, 1000, 9, 0.0)
np.savez_compressed(os.path.join(out, "stereo_640x480_seed9.npz"), n=n, uright=ur, depth=dp)
# search core of Fuse / SearchByProjection(KeyFrame*, Scw, ...)
from synth import synth_windows  # noqa: E402
wout = {}
for name, (chi2, greedy) in dict(fuse=(True, False), fuse_sim3=(False, False), kf_sim3_greedy=(False, True)).items():
    wd = synth_windows(seed=13)
    n, b, bd = o.search_windows(wd["q"], wd["kpx"], wd["kpy"], wd["octave"], wd["uright"], wd["inv_sigma2"],
                                wd["occupied"] if greedy else None, wd["desc"], wd["geom"], chi2=chi2, greedy=greedy)
    wout[name + "_n"], wout[name + "_best"], wout[name + "_dist"] = n, b, bd
np.savez_compressed(os.path.join(out, "windows_seed13.npz"), **wout)
# SearchForTriangulation
from synth import synth_triangulation  # noqa: E402
td = synth_triangulation(seed=117, n_nodes=100)
n, m = o.search_for_triangulation(td["kf1"], td["kf2"], td["F12"], float(td["ex"]), float(td["ey"]), td["scale"], td["sigma2"])
np.savez_compressed(os.path.join(out, "triangulation_seed117.npz"), n=n, match12=m)
# PoseOptimization
from synth import synth_pose_problem  # noqa: E402
pr = o.pose_optimization(synth_pose_problem(seed=23))
np.savez_compressed(os.path.join(out, "poseopt_seed23.npz"), n_inliers=pr["n_inliers"], Tcw=pr["Tcw"], outlier=pr["outlier"],
                    trace=pr["trace"], n_trials=pr["n_trials"])
# DBoW2 transform
from synth import synth_voc_features, synth_vocabulary  # noqa: E402
voc = synth_vocabulary(k=10, L=4, seed=7)
nw, word, w, node = o.bow_transform(voc, synth_voc_features(voc, 2000, 5), 2)
np.savez_compressed(os.path.join(out, "bow_transform_seed7.npz"), nw=nw, word=word, weight=w, node=node)
