"""ORBVocabulary::score (host/ORBVocabulary.cc; LoopClosing::DetectLoop calls it per covisible keyframe) equals the
reference's vendored DBoW2 score (TemplatedVocabulary::score -> L1Scoring::score, in oracle/_ref/libref_kfdb.so) and the
oracle's, as exact doubles, on random pairs including disjoint and identical vectors.  No GPU: score() is host code."""
import os
import subprocess

import numpy as np
import pytest

import kfdb_binding as kb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def product_score(pkg, tmp_path_factory):
    host = os.path.join(ROOT, "self_commit_orb-slam2_b200", "host")
    so = str(tmp_path_factory.mktemp("voc_score") / "libvoc_score.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-I", host, "-o", so,
                           os.path.join(ROOT, "tests", "cpp", "voc_score_shim.cc"), os.path.join(host, "ORBVocabulary.cc"),
                           pkg.LIB_PATH, "-Wl,-rpath," + os.path.dirname(pkg.LIB_PATH)])
    return kb.l1_score_fn(so, "voc_score")


def pairs():
    rng = np.random.default_rng(11)
    out = []
    for k in range(60):
        n1, n2 = int(rng.integers(0, 400)), int(rng.integers(0, 400))
        w1 = np.unique(rng.integers(0, 3000, n1)).astype(np.uint32)
        w2 = np.unique(rng.integers(0, 3000, n2)).astype(np.uint32)
        v1, v2 = rng.random(len(w1)), rng.random(len(w2))
        if k % 3 == 0 and len(v1):
            v1 /= v1.sum()
        out.append(((w1, v1), (w2, v2)))
    a = (np.arange(0, 500, 2, dtype=np.uint32), rng.random(250))
    out.append((a, (np.arange(1, 500, 2, dtype=np.uint32), rng.random(250))))  # disjoint
    out.append((a, a))                                                           # identical
    out.append((a, (a[0], -a[1])))                                               # opposite signs
    return out


def test_score_equals_oracle(product_score):
    orc = kb.l1_score_fn(kb.ORACLE_LIB, "orc_l1_score")
    for a, b in pairs():
        assert product_score(a, b) == orc(a, b)


@pytest.mark.skipif(not os.path.exists(kb.REF_LIB), reason="oracle/_ref not built (make -C oracle -f kfdb.mk ref)")
def test_score_equals_reference_dbow2(product_score):
    ref = kb.l1_score_fn(kb.REF_LIB, "ref_kfdb_score")
    ps = pairs()
    for a, b in ps:
        assert product_score(a, b) == ref(a, b)
    a = ps[-3][0]
    assert ref(a, ps[-3][1]) == 0.0  # disjoint
    assert abs(ref(a, a) - float(np.abs(a[1]).sum())) < 1e-12  # identical: all of its L1 mass
