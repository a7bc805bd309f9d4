"""The C++ shim classes with the reference's signatures (self_commit_orb-slam2_b200/host) against the oracle."""
import os
import subprocess

import numpy as np
import pytest

from synth import synth_image

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_cpp_extractor_shim(pkg, oracle, tmp_path):
    host = os.path.join(ROOT, "self_commit_orb-slam2_b200", "host")
    exe = str(tmp_path / "test_shim")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "cpp", "test_shim.cc"),
                           os.path.join(host, "ORBextractor.cc"), pkg.LIB_PATH,
                           "-Wl,-rpath," + os.path.dirname(pkg.LIB_PATH)])
    img = synth_image(640, 480, 6)
    raw = str(tmp_path / "img.raw")
    img.tofile(raw)
    out = str(tmp_path / "out.bin")
    subprocess.check_call([exe, raw, "640", "480", out])
    buf = open(out, "rb").read()
    n = int(np.frombuffer(buf[:4], np.int32)[0])
    kps = np.frombuffer(buf[4:4 + 28 * n], pkg.keypoint_dtype)
    desc = np.frombuffer(buf[4 + 28 * n:], np.uint8).reshape(n, 32)
    okps, odesc = oracle.extractor(1000, 1.2, 8, 20, 7)(img)
    assert n == len(okps)
    for f in ("x", "y", "size", "angle", "response", "octave", "class_id"):
        assert np.array_equal(kps[f], okps[f]), f
    assert np.array_equal(desc, odesc)


def test_cpp_vocabulary_shim(pkg, oracle, tmp_path):
    """ORBVocabulary::loadFromTextFile (DBoW2 text format) + transform through the C++ shim against the oracle."""
    from synth import synth_voc_features, synth_vocabulary
    host = os.path.join(ROOT, "self_commit_orb-slam2_b200", "host")
    exe = str(tmp_path / "test_voc")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", host, "-o", exe,
                           os.path.join(ROOT, "tests", "cpp", "test_voc_shim.cc"), os.path.join(host, "ORBVocabulary.cc"),
                           pkg.LIB_PATH, "-Wl,-rpath," + os.path.dirname(pkg.LIB_PATH)])
    voc = synth_vocabulary(k=10, L=3, seed=9)
    txt = str(tmp_path / "voc.txt")
    with open(txt, "w") as f:  # saveToTextFile format: header "k L scoring weighting", then one line per node
        f.write("%d %d 0 0\n" % (voc["k"], voc["L"]))
        for nid in range(1, len(voc["parent"])):
            f.write("%d %d %s %r\n" % (voc["parent"][nid], voc["leaf_flag"][nid],
                                       " ".join(str(int(b)) for b in voc["desc"][nid]), float(voc["weight"][nid])))
    feats = synth_voc_features(voc, n=500, seed=4)
    fb = str(tmp_path / "f.bin")
    feats.tofile(fb)
    out = str(tmp_path / "o.txt")
    subprocess.check_call([exe, txt, fb, "500", out])
    lines = open(out).read().split("\n")
    nwords, nbow, nfv = (int(x) for x in lines[0].split())
    nw, word, w, node = oracle.bow_transform(voc, feats, 2)
    assert nwords == nw
    bow = {}
    for i in range(500):
        if w[i] > 0:
            bow[int(word[i])] = bow.get(int(word[i]), 0.0) + float(w[i])
    norm = sum(abs(bow[k]) for k in sorted(bow))
    got_bow = {int(l.split()[1]): float(l.split()[2]) for l in lines if l.startswith("w ")}
    assert set(got_bow) == set(bow) and nbow == len(bow)
    for k in bow:
        assert abs(got_bow[k] - bow[k] / norm) < 1e-15
    got_fv = {int(l.split()[1]): [int(x) for x in l.split()[2:]] for l in lines if l.startswith("n ")}
    exp_fv = {}
    for i in range(500):
        if w[i] > 0:
            exp_fv.setdefault(int(node[i]), []).append(i)
    assert got_fv == exp_fv and nfv == len(exp_fv)
