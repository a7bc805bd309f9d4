"""Times the device PnPsolver and the reference's own PnPsolver (oracle/_ref/libref_pnpsolver.so, when built) on the
same machine.  One JSON line per configuration: n correspondences, find() at batch 1, and one relocalisation round
(iterate(5) per candidate, Relocalization's parameters) at batch 1, 16 and 64.  Device time is CUDA events around
upload, launches and download (b2s_pnpsolver_last_ms), the median of 20 calls after 3 warm-up calls; the reference time
is the host clock around its calls.  The card's name and power limit are read in the same run."""
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import pnpsolver_binding as pb  # noqa: E402
import synth_pnp as sp  # noqa: E402

pkg = importlib.import_module("self_commit_orb-slam2_b200")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def main():
    dev = card()
    for n in (50, 200, 800):
        for mode, batch in (("find", 1), ("round", 1), ("round", 16), ("round", 64)):
            scenes = [sp.scene(n, 0.5, seed, params=sp.RELOC) for seed in range(batch)]
            handle = pkg.PnPsolverBatch(max_matches=n, max_sets=300, max_batch=batch)
            nit = [d["max_its"] if mode == "find" else 5 for d in scenes]
            rng = np.random.default_rng(n)
            sets = [np.array([rng.choice(n, 4, replace=False) for _ in range(max(k, d["max_its"]))], np.int32)
                    for d, k in zip(scenes, nit)]
            ms = []
            for rep in range(23):
                svs = [handle.solver(d["P3Dw"], d["P2D"], d["sigma2"], d["K"]) for d in scenes]
                for sv, d in zip(svs, scenes):
                    sv.set_ransac_parameters(*d["params"])
                pkg.PnPsolver.iterate_batch(svs, nit, sets, handle=handle)
                if rep >= 3:
                    ms.append(handle.last_ms())
            line = dict(n=n, mode=mode, batch=batch, device_ms=float(np.median(ms)), device=dev)
            if os.path.exists(pb.REF_LIB):
                t = []
                for rep in range(5):
                    refs = [pb.Ref(d) for d in scenes]
                    pb.Ref.srand(rep)
                    t0 = time.perf_counter()
                    for r in refs:
                        r.iterate(None if mode == "find" else 5)
                    t.append((time.perf_counter() - t0) * 1e3)
                line["reference_ms"] = float(np.median(t))
                line["reference"] = "src/PnPsolver.cc, one host thread, solvers in turn"
            print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
