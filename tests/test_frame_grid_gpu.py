"""Persistent Frame feature grid (SURVEY §8f rank 4; src/Frame.cc:461-491, 741-852): GetFeaturesInArea on the resident grid
against the oracle's grid (index for index, in the reference's order) and — when oracle/_ref is present — against the
reference's own Frame; the projection matchers on a resident grid must return exactly what the host-buffer calls and the
oracle return."""
import ctypes
import os

import numpy as np
import pytest

from oracle_binding import FrameGeom
from synth import synth_descriptors, synth_projection, synth_projection_map, synth_windows

pytestmark = pytest.mark.gpu
vp, c_i, c_f = ctypes.c_void_p, ctypes.c_int, ctypes.c_float


def _grid(pkg, m, d, is2=None):
    return pkg.FrameGrid(m, d["kpx"], d["kpy"], d["octave"], d["angle"], d["uright"], d["desc"], d["geom"], inv_level_sigma2=is2)


def _queries(rng, d, n):
    for t in range(n):
        if t % 3 == 0:
            j = rng.randint(0, len(d["kpx"]))
            x, y = float(d["kpx"][j]) + rng.uniform(-3, 3), float(d["kpy"][j]) + rng.uniform(-3, 3)
        else:
            x, y = rng.uniform(-60, 1300), rng.uniform(-60, 440)
        r = float(rng.choice([2.5, 7.0, 15.0, 40.0, 120.0, 2000.0]))
        mn, mx = [(-1, -1), (0, 3), (2, -1), (3, 4), (0, 0), (1, 7)][rng.randint(0, 6)]
        yield x, y, r, mn, mx


@pytest.mark.parametrize("cluster", [False, True])
def test_features_in_area_matches_oracle_grid(pkg, oracle, cluster):
    d = synth_projection(nf=2000, nq=10, seed=3, cluster=cluster)
    m = pkg.ORBmatcher(0.9, True)
    gr = _grid(pkg, m, d)
    sf = np.ascontiguousarray(d["geom"]["scale_factors"], np.float32)
    g = FrameGeom(0.0, 0.0, float(d["geom"]["mnMaxX"]), float(d["geom"]["mnMaxY"]), float(d["geom"]["bf"]), sf.ctypes.data, 8)
    L = oracle.L
    L.orc_features_in_area.argtypes = [vp, vp, vp, c_i, vp, c_f, c_f, c_f, c_i, c_i, vp, c_i]
    b = np.zeros(4096, np.int32)
    total = 0
    for x, y, r, mn, mx in _queries(np.random.RandomState(5), d, 400):
        got = gr.GetFeaturesInArea(x, y, r, mn, mx)
        nb = L.orc_features_in_area(d["kpx"].ctypes.data, d["kpy"].ctypes.data, d["octave"].ctypes.data, len(d["kpx"]),
                                    ctypes.byref(g), x, y, r, mn, mx, b.ctypes.data, 4096)
        assert len(got) == nb and np.array_equal(got, b[:nb])
        total += nb
    assert total > 5000


def test_features_in_area_matches_reference_frame(pkg):
    """The grid built from the REFERENCE frame's keypoints answers like the reference's own Frame::GetFeaturesInArea."""
    import test_oracle_reference_frame as T
    if not os.path.exists(T.LIB):
        pytest.skip("oracle/_ref not built")
    from synth import synth_stereo
    imL, imR = synth_stereo(1241, 376, 5)
    F = T.RefFrame(imL, imR, 2000)
    sf = np.array([np.float32(1.0)] * 8, np.float32)
    for i in range(1, 8):
        sf[i] = np.float32(sf[i - 1] * np.float32(1.2))
    geom = dict(mnMinX=np.float32(0), mnMinY=np.float32(0), mnMaxX=np.float32(F.w), mnMaxY=np.float32(F.h), bf=np.float32(T.BF),
                scale_factors=sf)
    m = pkg.ORBmatcher(0.9, True, max_features=4096)
    gr = pkg.FrameGrid(m, F.kpsL["x"], F.kpsL["y"], F.kpsL["octave"], F.kpsL["angle"], F.uright, F.descL, geom)
    a = np.zeros(4096, np.int32)
    d = dict(kpx=np.ascontiguousarray(F.kpsL["x"]), kpy=np.ascontiguousarray(F.kpsL["y"]))
    for x, y, r, mn, mx in _queries(np.random.RandomState(9), d, 300):
        na = F.R.ref_frame_features_in_area(x, y, r, mn, mx, a.ctypes.data, 4096)
        got = gr.GetFeaturesInArea(x, y, r, mn, mx)
        assert len(got) == na and np.array_equal(got, a[:na])


def test_searches_on_resident_grid_equal_host_buffer_calls(pkg, oracle):
    # last-frame projection, three modes on ONE grid
    d = synth_projection(seed=21, cluster=False, th=7.0)
    m = pkg.ORBmatcher(0.9, True)
    gr = _grid(pkg, m, d)
    for mode in (0, 1, 2):
        n, match = gr.SearchByProjection(d["q"], d["occupied"], d["th"], mode=mode)
        on, om = oracle.search_by_projection_last(d["q"], d["kpx"], d["kpy"], d["octave"], d["angle"], d["uright"], d["occupied"],
                                                  d["desc"], d["geom"], float(d["th"]), mode=mode)
        assert n == on and np.array_equal(match, om) and n > 100
    # local-map projection on the same kind of grid, two radii
    d = synth_projection_map(seed=33, cluster=True)
    d["angle"] = np.zeros(len(d["kpx"]), np.float32)
    m8 = pkg.ORBmatcher(0.8, True)
    gr = _grid(pkg, m8, d)
    for th in (1.0, 3.0):
        n, match = gr.SearchByProjectionMap(d["q"], d["occupied"], th=th)
        on, om = oracle.search_by_projection_map(d["q"], d["kpx"], d["kpy"], d["octave"], d["uright"], d["occupied"], d["desc"],
                                                 d["geom"], th=th, nnratio=0.8)
        assert n == on and np.array_equal(match, om) and n > 100
    # window searches (Fuse chi2 / plain / greedy) on one keyframe grid
    d = synth_windows(seed=13)
    d["angle"] = np.zeros(len(d["kpx"]), np.float32)
    gr = _grid(pkg, m8, d, is2=d["inv_sigma2"])
    for chi2, greedy in ((True, False), (False, False), (False, True)):
        occ = d["occupied"] if greedy else None
        n, best, bd = gr.SearchWindows(d["q"], occ, chi2=chi2, greedy=greedy)
        on, ob, obd = oracle.search_windows(d["q"], d["kpx"], d["kpy"], d["octave"], d["uright"], d["inv_sigma2"], occ, d["desc"],
                                            d["geom"], chi2=chi2, greedy=greedy)
        assert n == on and np.array_equal(best, ob) and np.array_equal(bd, obd)


def _launches(m, call):
    before = m.launch_count()
    out = call()
    return out, m.launch_count() - before


def test_host_buffer_searches_equal_their_grid_twins(pkg, oracle):
    """A host-buffer projection search is its resident-grid twin plus a grid build (3 launches) on the same inputs:
    array-for-array identical outputs, and the launch count of every host-buffer matcher call is pinned."""
    d = synth_projection(seed=21, cluster=True, th=7.0)
    m = pkg.ORBmatcher(0.9, True)
    gr = _grid(pkg, m, d)
    for mode in (0, 1, 2):
        (nh, mh), lh = _launches(m, lambda: m.SearchByProjection(d["q"], d["kpx"], d["kpy"], d["octave"], d["angle"], d["uright"],
                                                                 d["occupied"], d["desc"], d["geom"], d["th"], mode=mode))
        (ng, mg), lg = _launches(m, lambda: gr.SearchByProjection(d["q"], d["occupied"], d["th"], mode=mode))
        assert (lh, lg) == (7, 4)
        assert nh == ng > 100 and np.array_equal(mh, mg)
    d = synth_projection_map(seed=33, cluster=True)
    m8 = pkg.ORBmatcher(0.8, True)
    gr = _grid(pkg, m8, d)
    for th in (1.0, 3.0):
        (nh, mh), lh = _launches(m8, lambda: m8.SearchByProjectionMap(d["q"], d["kpx"], d["kpy"], d["octave"], d["uright"],
                                                                      d["occupied"], d["desc"], d["geom"], th=th))
        (ng, mg), lg = _launches(m8, lambda: gr.SearchByProjectionMap(d["q"], d["occupied"], th=th))
        assert (lh, lg) == (6, 3)
        assert nh == ng > 100 and np.array_equal(mh, mg)
    d = synth_windows(seed=13)
    gr = _grid(pkg, m8, d, is2=d["inv_sigma2"])
    for chi2, greedy in ((True, False), (False, False), (False, True)):
        occ = d["occupied"] if greedy else None
        (nh, bh, dh), lh = _launches(m8, lambda: m8.SearchWindows(d["q"], d["kpx"], d["kpy"], d["octave"], d["uright"],
                                                                  d["inv_sigma2"], occ, d["desc"], d["geom"], chi2=chi2,
                                                                  greedy=greedy))
        (ng, bg, dg), lg = _launches(m8, lambda: gr.SearchWindows(d["q"], occ, chi2=chi2, greedy=greedy))
        assert (lh, lg) == (5, 2)
        assert nh == ng > 100 and np.array_equal(bh, bg) and np.array_equal(dh, dg)
    # the two host-buffer matchers without a grid twin: launch counts, and the oracle's answer
    d = synth_projection(nf=1500, nq=1500, seed=41)
    rng = np.random.RandomState(42)
    q = d["q"]
    prev = np.ascontiguousarray(np.stack([q["u"], q["v"]], 1), np.float32)
    oct1 = np.where(rng.randint(0, 100, size=len(q)) < 50, 0, q["octave"]).astype(np.int32)
    oct2 = np.where(rng.randint(0, 100, size=len(d["kpx"])) < 60, 0, d["octave"]).astype(np.int32)
    args = (oct1, q["angle"], q["desc"], d["kpx"], d["kpy"], oct2, d["angle"], d["desc"], d["geom"])
    (n, m12), l = _launches(m, lambda: m.SearchForInitialization(prev.copy(), *args))
    on, om = oracle.search_for_initialization(prev.copy(), *args, nnratio=0.9)
    assert l == 9 and n == on > 100 and np.array_equal(m12, om)
    A, nA, vA, aA, B, nB, aB = synth_descriptors(1000, seed=5)
    (n, mb), l = _launches(m, lambda: m.SearchByBoW(A, nA, vA, aA, B, nB, aB))
    on, om = oracle.search_by_bow(A, nA, vA, aA, B, nB, aB, nnratio=0.9)
    assert l == 5 and n == on > 100 and np.array_equal(mb, om)


def test_grid_from_device_resident_extractor_records(pkg, oracle):
    """b2s_frame_grid_create_device: the extractor's records never leave the device."""
    import torch
    from synth import synth_image
    w, h, nf = 640, 480, 1000
    img = synth_image(w, h, 4)
    ex = pkg.ORBextractor(nf, 1.2, 8, 20, 7, max_width=w, max_height=h, max_batch=1)
    k, dsc = ex.extract_batch([img])[0]
    rec = torch.from_numpy(np.ascontiguousarray(k).view(np.uint8).reshape(len(k), 28)).cuda()
    dd = torch.from_numpy(np.ascontiguousarray(dsc)).cuda()
    sf = np.array([np.float32(1.2) ** 0] * 8, np.float32)
    for i in range(1, 8):
        sf[i] = np.float32(sf[i - 1] * np.float32(1.2))
    geom = dict(mnMinX=np.float32(0), mnMinY=np.float32(0), mnMaxX=np.float32(w), mnMaxY=np.float32(h), bf=np.float32(40.0),
                scale_factors=sf)
    m = pkg.ORBmatcher(0.9, True)
    torch.cuda.synchronize()
    gd = pkg.FrameGrid(m, geom=geom, d_kps_ptr=rec.data_ptr(), d_desc_ptr=dd.data_ptr(), nf=len(k))
    gh = pkg.FrameGrid(m, k["x"], k["y"], k["octave"], k["angle"], np.full(len(k), -1, np.float32), dsc, geom)
    rng = np.random.RandomState(1)
    for _ in range(100):
        x, y, r = rng.uniform(0, w), rng.uniform(0, h), float(rng.choice([5.0, 20.0, 80.0]))
        a, b = gd.GetFeaturesInArea(x, y, r, 0, 3), gh.GetFeaturesInArea(x, y, r, 0, 3)
        assert np.array_equal(a, b)
    # and a search on it: each keypoint's own descriptor finds itself
    q = np.zeros(len(k), pkg.win_query_dtype)
    q["u"], q["v"], q["radius"], q["min_level"], q["max_level"], q["valid"], q["desc"] = k["x"], k["y"], 3.0, k["octave"], k["octave"], 1, dsc
    n, best, bd = gd.SearchWindows(q, None)
    assert n == len(k) and (bd == 0).all()
    same = best == np.arange(len(k))
    assert same.mean() > 0.95  # (duplicates at the same pixel on the same level may tie)


def test_empty_grid_and_bad_arguments(pkg):
    d = synth_projection(nf=50, nq=10, seed=1)
    m = pkg.ORBmatcher(0.9, True)
    g0 = pkg.FrameGrid(m, d["kpx"][:0], d["kpy"][:0], d["octave"][:0], d["angle"][:0], d["uright"][:0], d["desc"][:0], d["geom"])
    assert g0.n == 0 and len(g0.GetFeaturesInArea(10, 10, 50)) == 0
    n, match = g0.SearchByProjection(d["q"], None, 7.0)
    assert n == 0 and len(match) == 0
    other = pkg.ORBmatcher(0.9, True)
    gr = _grid(pkg, m, d)
    gr.matcher = other  # a grid only works with the matcher that owns it
    with pytest.raises(pkg.B200SlamError):
        gr.SearchByProjection(d["q"], None, 7.0)
