"""Pins the oracle's extractor against the REFERENCE'S OWN SOURCE: /root/reference/src/ORBextractor.cc is compiled in place
(oracle/Makefile target `ref`, oracle/_ref/libref_extractor.so) against oracle/refshim — a stand-in for the OpenCV C++
API whose arithmetic is the oracle's cv2-pinned primitives — and must give bit-identical keypoints and descriptors.

The one thing that cannot be reproduced is the allocator: DistributeOctTree breaks ties between equally large nodes by
the heap address of std::list nodes (src/ORBextractor.cc:948).  With a monotonic (bump) allocator the addresses follow
creation order, which is the rule the oracle states; on glibc malloc the same binary gives a different (but equally
valid) selection, which the second test documents."""
import ctypes
import os

import numpy as np
import pytest

from synth import synth_image, synth_stereo, synth_texture

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "oracle", "_ref", "libref_extractor.so")
pytestmark = pytest.mark.skipif(not os.path.exists(LIB), reason="oracle/_ref not built (needs /root/reference: make -C oracle ref)")
FIELDS = ("x", "y", "size", "angle", "response", "octave", "class_id")


def _ref():
    R = ctypes.CDLL(LIB)
    R.ref_extract.argtypes = [ctypes.c_int, ctypes.c_float, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                              ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
    return R


def _run(R, img, nf, sf=1.2, nl=8, ini=20, mn=7):
    img = np.ascontiguousarray(img)
    h, w = img.shape
    cap = nf + 4 * nl + 200
    k = np.zeros((cap, 7), np.float32)
    d = np.zeros((cap, 32), np.uint8)
    n = R.ref_extract(nf, sf, nl, ini, mn, img.ctypes.data, w, h, k.ctypes.data, d.ctypes.data, cap)
    assert n >= 0
    return k[:n], d[:n]


@pytest.mark.parametrize("w,h,nf,seed", [(640, 480, 1000, 3), (1241, 376, 2000, 3), (1241, 376, 2000, 5), (321, 243, 500, 7),
                                         (752, 480, 1200, 9)])
def test_reference_source_equals_oracle(checker, w, h, nf, seed):
    R = _ref()
    R.ref_set_monotonic_allocator(1)
    img = synth_image(w, h, seed) if seed != 5 else synth_stereo(w, h, seed)[1]
    rk, rd = _run(R, img, nf)
    ok, od = checker.extractor(nf, 1.2, 8, 20, 7)(img)  # the oracle (CPU suite) or the CUDA extractor (-m gpu)
    assert len(rk) == len(ok)
    for i, f in enumerate(FIELDS):
        assert np.array_equal(rk[:, i], ok[f].astype(np.float32)), f
    assert np.array_equal(rd, od)


def test_malloc_tie_break_is_the_only_difference(oracle):
    """On the system allocator the reference's largest-first splitting order follows heap addresses: the per-level
    keypoint COUNTS stay within the quota overshoot and almost all keypoints coincide, but the sets are not identical."""
    R = _ref()
    R.ref_set_monotonic_allocator(0)
    img = synth_image(640, 480, 3)
    rk, rd = _run(R, img, 1000)
    R.ref_set_monotonic_allocator(1)
    ok, od = oracle.extractor(1000, 1.2, 8, 20, 7)(img)
    rs = {(float(a), float(b), int(c)) for a, b, c in zip(rk[:, 0], rk[:, 1], rk[:, 5])}
    os_ = {(float(a), float(b), int(c)) for a, b, c in zip(ok["x"], ok["y"], ok["octave"])}
    assert abs(len(rs) - len(os_)) <= 8
    assert len(rs & os_) >= 0.97 * len(os_)
    # descriptors of the common keypoints are identical (same image, same angle)
    rd_by = {(float(a), float(b), int(c)): rd[i].tobytes() for i, (a, b, c) in enumerate(zip(rk[:, 0], rk[:, 1], rk[:, 5]))}
    od_by = {(float(a), float(b), int(c)): od[i].tobytes() for i, (a, b, c) in enumerate(zip(ok["x"], ok["y"], ok["octave"]))}
    assert all(rd_by[p] == od_by[p] for p in rs & os_)


# The parameter, threshold and texture cases of the CUDA sweep (tests/test_extractor_sweep_gpu.py), so the chain
# CUDA -> oracle -> reference source stays closed beyond 1.2 / 8 / 20 / 7.
SWEEP = ([("synth", 800, 600, 1000, (sf, nl, 20, 7)) for sf, nl in [(1.2, 1), (1.2, 2), (1.1, 12), (1.05, 12), (1.44, 6),
                                                                  (2.0, 4)]] +
         [("synth", 640, 480, nf, (1.2, 8, 20, 7)) for nf in (1, 17, 5000)] +
         [("synth", 640, 480, 1000, (1.2, 8, ini, mn)) for ini, mn in [(12, 7), (8, 4), (40, 20), (254, 1)]] +
         [(kind, 640, 480, 1000, p) for kind in ("noise", "saltpepper", "dark", "bright", "checker2", "checker3", "checker5",
                                                 "corner", "fallback", "dense")
          for p in [(1.2, 8, 20, 7), (1.2, 8, 12, 7), (1.44, 6, 8, 4)]] +
         [("noise", 1920, 1080, 2000, (1.2, 8, 20, 7)), ("noise", 3840, 400, 2000, (1.2, 4, 20, 7))])


@pytest.mark.parametrize("kind,w,h,nf,params", SWEEP)
def test_reference_source_equals_oracle_sweep(checker, kind, w, h, nf, params):
    R = _ref()
    R.ref_set_monotonic_allocator(1)
    img = synth_image(w, h, 1) if kind == "synth" else synth_texture(kind, w, h, 1)
    rk, rd = _run(R, img, nf, *params)
    ok, od = checker.extractor(nf, *params)(img)
    assert len(rk) == len(ok)
    for i, f in enumerate(FIELDS):
        assert np.array_equal(rk[:, i], ok[f].astype(np.float32)), f
    assert np.array_equal(rd, od)


def test_noise_golden_equals_reference_source():
    """tests/golden/extract_640x480_noise_12_7.npz (written from the oracle by tools/make_golden.py) is what the
    reference's own source computes."""
    g = np.load(os.path.join(ROOT, "tests", "golden", "extract_640x480_noise_12_7.npz"))
    R = _ref()
    R.ref_set_monotonic_allocator(1)
    rk, rd = _run(R, synth_texture("noise", 640, 480, 3), 1000, 1.2, 8, 12, 7)
    assert len(rk) == len(g["kps"])
    for i, f in enumerate(FIELDS):
        assert np.array_equal(rk[:, i], g["kps"][f].astype(np.float32)), f
    assert np.array_equal(rd, g["desc"])
