"""Times one keyframe-database query (DetectRelocalizationCandidates, DetectLoopCandidates) on the device against the
reference's own src/KeyFrameDatabase.cc on one CPU thread (oracle/_ref/libref_kfdb.so, built by build() where the
reference's sources are present), on maps of 500, 2,000 and 8,000 keyframes of about 1,200 Zipf-distributed words over
the real vocabulary's 971,814 words.  Both replay the same sequence and their candidate lists are compared in the run.

Per map size and query kind it prints one JSON line: the device time of the query's kernels (CUDA events on the
database's stream), the host wall time of the whole call (covisibility table upload and result download included) and
the reference's wall time, as medians over the timed queries, with the card's name and power limit.

    python tools/kfdb_time.py [--sizes 500,2000,8000] [--queries 40] [--out DIR/kfdb_time.jsonl]"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402

import kfdb_binding as kb  # noqa: E402


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        name, power = [s.strip() for s in out.splitlines()[0].split(",")]
        return name, power
    except Exception as e:  # the numbers are still device events; say where they came from
        return "unknown (%s)" % e, "unknown"


def covis_table(n):
    ids = np.zeros((n, 10), np.uint64)
    cnt = np.zeros(n, np.int32)
    for i in range(n):
        nb = [j for j in (i - 1, i + 1, i - 2, i + 2, i - 3, i + 3, i - 8, i + 8, i - 16, i + 16) if 0 <= j < n]
        cnt[i] = len(nb)
        ids[i, :len(nb)] = nb
    return ids, cnt


def noisy(rng, bow, keep=0.8):
    w, v = bow
    m = rng.random(len(w)) < keep
    v2 = v[m] * (0.5 + rng.random(m.sum()))
    return w[m], v2 / v2.sum()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="500,2000,8000")
    ap.add_argument("--queries", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--words", type=int, default=1200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    pkg = importlib.import_module("self_commit_orb-slam2_b200")
    if pkg.device_count() < 1:
        raise SystemExit("kfdb_time: no CUDA device (the device path has no CPU fallback; nothing was measured)")
    have_ref = os.path.exists(kb.REF_LIB)
    name, power = card()
    lines = []
    for n in [int(s) for s in a.sizes.split(",")]:
        kfs = kb.zipf_map(seed=n, n_kf=n, words_per_kf=a.words)
        covis = covis_table(n)
        db = pkg.KeyFrameDatabase(kb.ORBVOC_WORDS)
        ref = kb.Reference(kb.ORBVOC_WORDS) if have_ref else None
        for i, b in enumerate(kfs):
            db.add(i, *b)
            if ref:
                ref.add(i, *b)
        rng = np.random.default_rng(n + 1)
        res = {"reloc": ([], [], []), "loop": ([], [], [])}
        mismatches = 0
        for q in range(a.warmup + a.queries):
            src = int(rng.integers(0, n))
            for kind in ("reloc", "loop"):
                bow = noisy(rng, kfs[src], 0.8 if kind == "reloc" else 0.9)
                if kind == "reloc":
                    call = lambda d: d.DetectRelocalizationCandidates(10**7 + q, *bow, covis=covis)  # noqa: E731
                else:
                    conn = [src, max(src - 1, 0)]
                    call = lambda d: d.DetectLoopCandidates(n + q, *bow, conn, 0.02, covis=covis)  # noqa: E731
                t0 = time.perf_counter()
                got = call(db)
                t1 = time.perf_counter()
                dev = db.last_query_ms()
                tr = None
                if ref:
                    t2 = time.perf_counter()
                    want = call(ref)
                    tr = (time.perf_counter() - t2) * 1e3
                    mismatches += got != want
                if q >= a.warmup:
                    res[kind][0].append(dev)
                    res[kind][1].append((t1 - t0) * 1e3)
                    if tr is not None:
                        res[kind][2].append(tr)
        words = float(np.mean([len(k[0]) for k in kfs]))
        for kind, (dev, host, cpu) in res.items():
            rec = dict(keyframes=n, query=kind, words_per_keyframe=round(words, 1), queries=a.queries,
                       device_ms=float(np.median(dev)), host_wall_ms=float(np.median(host)),
                       reference_cpu_1thread_ms=float(np.median(cpu)) if cpu else "not measured (libref_kfdb.so absent)",
                       outputs_equal=(mismatches == 0) if ref else "not compared", gpu=name, power_limit=power)
            print(json.dumps(rec), flush=True)
            lines.append(rec)
        db.close()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write("\n".join(json.dumps(r) for r in lines) + "\n")


if __name__ == "__main__":
    main()
