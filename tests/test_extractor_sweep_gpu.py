"""Bit-exact parity of the CUDA extractor with the CPU oracle over the input range the C ABI accepts: camera and tile-edge
image shapes, the smallest accepted image, pyramid parameters, feature counts, FAST thresholds, dense and degenerate
textures, handle reuse across sizes and the batch entry points.  Every case compares each pyramid level, each blurred
level, each level's candidate list, every keypoint field and the descriptors, so a failure names its stage."""
import os

import numpy as np
import pytest

from synth import fast_strength, level_sizes, grid_ok, residue_shapes, synth_image, synth_stereo, synth_texture

pytestmark = pytest.mark.gpu

DEFAULT = (1.2, 8, 20, 7)
FIELDS = ("x", "y", "size", "angle", "response", "octave", "class_id")
B2S_ERR_BAD_ARG = 2
_ORACLE = {}  # (image key, nfeatures, params) -> oracle result, shared by the parametrisations of this module


def _image(kind, w, h, seed=1):
    return synth_image(w, h, seed) if kind == "synth" else synth_texture(kind, w, h, seed)


def _oracle_run(oracle, key, img, nf, params):
    k = (key, img.shape, nf, params)
    if k not in _ORACLE:
        sf, nl, ini, mn = params
        oe = oracle.extractor(nf, sf, nl, ini, mn)
        kps, desc = oe(img)
        levels = [(oe.level(l), oe.level(l, blurred=True), oe.candidates(l)) for l in range(nl)]
        _ORACLE[k] = (kps, desc, levels)
    return _ORACLE[k]


def _cmp_kps(a, b, what=""):
    assert len(a) == len(b), "%s: %d vs %d keypoints" % (what, len(a), len(b))
    for f in FIELDS:
        assert np.array_equal(a[f], b[f]), "%s: field %s" % (what, f)


def _check(ex, b, kps, desc, ref, what):
    okps, odesc, levels = ref
    for l, (lv, blurred, cand) in enumerate(levels):
        assert np.array_equal(ex.debug_level(b, l), lv), "%s: pyramid level %d" % (what, l)
        if blurred is not None:
            assert np.array_equal(ex.debug_level(b, l, blurred=True), blurred), "%s: blurred level %d" % (what, l)
        xy, resp = ex.debug_candidates(b, l)
        assert len(xy) == len(cand), "%s: level %d candidates %d vs %d" % (what, l, len(xy), len(cand))
        assert np.array_equal(xy[:, 0], cand["x"].astype(np.int32)) and np.array_equal(xy[:, 1], cand["y"].astype(np.int32)), \
            "%s: level %d candidate positions" % (what, l)
        assert np.array_equal(resp, cand["response"].astype(np.int32)), "%s: level %d candidate responses" % (what, l)
    _cmp_kps(kps, okps, what)
    assert np.array_equal(desc, odesc), "%s: descriptors" % what


def _run_case(pkg, oracle, kind, w, h, nf=1000, params=DEFAULT, seed=1):
    img = _image(kind, w, h, seed)
    sf, nl, ini, mn = params
    ex = pkg.ORBextractor(nf, sf, nl, ini, mn, max_width=w, max_height=h)
    kps, desc = ex(img)
    _check(ex, 0, kps, desc, _oracle_run(oracle, (kind, seed), img, nf, params), "%s %dx%d nf=%d %s" % (kind, w, h, nf, params))
    return kps


# ---------------------------------------------------------------- shapes
@pytest.mark.parametrize("kind,w,h,nf,params", [
    ("synth", 752, 480, 1200, DEFAULT),     # EuRoC
    ("synth", 1226, 370, 2000, DEFAULT),    # KITTI 04-12
    ("synth", 1280, 720, 2000, DEFAULT),
    ("synth", 1920, 1080, 2000, DEFAULT),
    ("noise", 1920, 1080, 2000, DEFAULT),   # level 0 alone holds ~204 k candidates
    ("noise", 3840, 400, 2000, (1.2, 4, 20, 7)),  # > 12 k NMS maxima in one row of cells
    ("noise", 1241, 376, 2000, (1.2, 8, 8, 4)),
])
def test_camera_and_dense_shapes(pkg, oracle, kind, w, h, nf, params):
    _run_case(pkg, oracle, kind, w, h, nf, params)


def test_tile_residue_shapes_cover_every_residue():
    shapes, xs, ys = residue_shapes()
    assert xs == {0, 1, 127} and ys == {0, 1, 31}
    assert len(shapes) <= 8


@pytest.mark.parametrize("wh", residue_shapes()[0])
def test_tile_residue_shapes(pkg, oracle, wh):
    _run_case(pkg, oracle, "synth", wh[0], wh[1], 1000)


@pytest.mark.parametrize("w,h", [(333, 250), (642, 481), (1023, 367), (645, 483)])
def test_widths_not_multiple_of_16(pkg, oracle, w, h):
    _run_case(pkg, oracle, "synth", w, h, 1000)


def test_host_stride_larger_than_width(pkg, oracle):
    w, h, nf = 645, 483, 1000
    big = synth_image(w + 61, h, 1)
    big[:, :w] = synth_image(w, h, 1)
    view = big[:, :w]  # rows of w pixels, stride w + 61
    assert view.strides[0] == w + 61
    ex = pkg.ORBextractor(nf, *DEFAULT, max_width=w, max_height=h)
    kps, desc = ex(view)
    _check(ex, 0, kps, desc, _oracle_run(oracle, ("synth", 1), np.ascontiguousarray(view), nf, DEFAULT), "stride")


def _min_side():
    return min(W for W in range(64, 400) if all(grid_ok(w, h) for w, h in level_sizes(W, W, 1.2, 8)))


def test_smallest_accepted_image(pkg, oracle):
    m = _min_side()
    assert m == 221  # 8 levels at 1.2: level 7 must be >= 62 px (one 30-px cell inside the 16-px border)
    _run_case(pkg, oracle, "noise", m, m, 500)
    ex = pkg.ORBextractor(500, *DEFAULT, max_width=m, max_height=m)
    for w, h in ((m - 1, m), (m, m - 1)):
        with pytest.raises(pkg.B200SlamError) as e:
            ex(synth_texture("noise", w, h, 1))
        assert e.value.code == B2S_ERR_BAD_ARG
        assert "pyramid level 7" in str(e.value) and "too small for the 30-px FAST cell grid" in str(e.value)
    # the refused size leaves no half-built geometry behind: the handle still extracts its last good size
    ex2 = pkg.ORBextractor(500, *DEFAULT, max_width=m, max_height=m)
    img = synth_texture("noise", m, m, 1)
    k1, d1 = ex2(img)
    with pytest.raises(pkg.B200SlamError):
        ex2(synth_texture("noise", m - 1, m, 1))
    k2, d2 = ex2(img)
    assert k1.tobytes() == k2.tobytes() and np.array_equal(d1, d2)


# ---------------------------------------------------------------- pyramid parameters, feature counts, thresholds
@pytest.mark.parametrize("sf,nl", [(1.2, 1), (1.2, 2), (1.1, 12), (1.05, 12), (1.44, 6), (2.0, 4)])
def test_pyramid_parameters(pkg, oracle, sf, nl):
    _run_case(pkg, oracle, "synth", 800, 600, 1000, (sf, nl, 20, 7))  # (2.0, 4): level 3 of 480 rows is too small


def test_many_levels_at_1080p(pkg, oracle):
    """1.05 x 12 levels at 1920x1080 needs 15,696 FAST cells: more than the old 4 x (W/28+2)(H/28+2) allocation."""
    _run_case(pkg, oracle, "synth", 1920, 1080, 2000, (1.05, 12, 20, 7))


@pytest.mark.parametrize("nf", [1, 17, 500, 2000, 5000])
def test_feature_counts(pkg, oracle, nf):
    ex = pkg.ORBextractor(nf, *DEFAULT, max_width=640, max_height=480)
    if nf == 1:
        assert (ex.mnFeaturesPerLevel == 0).sum() == 7  # levels with quota N = 0
    _run_case(pkg, oracle, "synth", 640, 480, nf)


def _largest_admitted_nfeatures(pkg):
    lo, hi = 1, 1 << 16  # lo admitted, hi refused
    while hi - lo > 1:
        mid = (lo + hi) // 2
        try:
            pkg.ORBextractor(mid, *DEFAULT, max_width=64, max_height=64).close()
            lo = mid
        except pkg.B200SlamError as e:
            assert e.code == B2S_ERR_BAD_ARG and "quadtree" in str(e)
            hi = mid
    return lo


def test_largest_nfeatures(pkg, oracle):
    nf = _largest_admitted_nfeatures(pkg)
    assert nf > 5000
    with pytest.raises(pkg.B200SlamError) as e:
        pkg.ORBextractor(nf + 1, *DEFAULT, max_width=1920, max_height=1080)
    assert e.value.code == B2S_ERR_BAD_ARG
    _run_case(pkg, oracle, "noise", 1920, 1080, nf)


@pytest.mark.parametrize("ini,mn", [(20, 7), (12, 7), (8, 4), (40, 20), (254, 1)])
def test_thresholds(pkg, oracle, ini, mn):
    _run_case(pkg, oracle, "synth", 640, 480, 1000, (1.2, 8, ini, mn))


# ---------------------------------------------------------------- textures
TEXTURE_PARAMS = [DEFAULT, (1.2, 8, 12, 7), (1.44, 6, 8, 4)]


@pytest.mark.parametrize("params", TEXTURE_PARAMS)
@pytest.mark.parametrize("kind", ["noise", "saltpepper", "dark", "bright", "checker2", "checker3", "checker4", "checker5",
                                  "checker6", "corner", "fallback", "dense"])
def test_textures(pkg, oracle, kind, params):
    kps = _run_case(pkg, oracle, kind, 640, 480, 1000, params)
    if kind == "corner":
        assert len(kps) >= 1


def test_dense_texture_reaches_the_dense_nms():
    """More than CAND_CAP = 2048 pixels above iniThFAST in a 128 x 32 tile: k_tile's dense NMS branch."""
    img = synth_texture("dense", 640, 480, 1)
    M = fast_strength(img)
    tile = M[64:96, 128:256]  # interior tile (2, 1): inside the FAST band on every side
    assert int((tile > 20).sum()) > 2048
    assert int((tile > 8).sum()) > 2048


# ---------------------------------------------------------------- handle reuse and entry points
def test_handle_reuse_across_sizes(pkg, oracle):
    seq = [("noise", 1920, 1080), ("synth", 321, 243), ("noise", 1241, 376), ("noise", 1920, 1080)]
    ex = pkg.ORBextractor(2000, *DEFAULT, max_width=1920, max_height=1080)
    for kind, w, h in seq:
        img = _image(kind, w, h)
        kps, desc = ex(img)
        fresh = pkg.ORBextractor(2000, *DEFAULT, max_width=w, max_height=h)
        fk, fd = fresh(img)
        assert kps.tobytes() == fk.tobytes() and np.array_equal(desc, fd), (kind, w, h)
        _check(ex, 0, kps, desc, _oracle_run(oracle, (kind, 1), img, 2000, DEFAULT), "reuse %s %dx%d" % (kind, w, h))


def test_chunked_dense_batch(pkg, oracle):
    """>= 16 images: the host-buffer batch is cut into chunks on two streams; dense textures fill the candidate lists."""
    w, h, nf, B = 640, 480, 1000, 16
    kinds = ["noise", "dense", "checker3", "saltpepper"]
    imgs = [synth_texture(kinds[i % 4], w, h, 100 + i) for i in range(B)]
    ex = pkg.ORBextractor(nf, *DEFAULT, max_width=w, max_height=h, max_batch=B)
    res = ex.extract_batch(imgs)
    for i, (k, d) in enumerate(res):
        okps, odesc, _ = _oracle_run(oracle, (kinds[i % 4], 100 + i), imgs[i], nf, DEFAULT)
        _cmp_kps(k, okps, "batch image %d" % i)
        assert np.array_equal(d, odesc), i


def test_device_batch_with_image_pitch(pkg, oracle):
    torch = pytest.importorskip("torch")
    w, h, nf, B, pitch = 645, 483, 1000, 3, 700 * 490
    imgs = [synth_texture("noise", w, h, 7 + i) for i in range(B)]
    host = np.zeros((B, pitch), np.uint8)
    for i, im in enumerate(imgs):
        host[i, :w * h] = im.reshape(-1)
    d_imgs = torch.from_numpy(host).cuda()
    ex = pkg.ORBextractor(nf, *DEFAULT, max_width=w, max_height=h, max_batch=B)
    cap = ex.cap
    d_kps = torch.zeros((B, cap, 7), dtype=torch.float32, device="cuda")
    d_desc = torch.zeros((B, cap, 32), dtype=torch.uint8, device="cuda")
    d_n = torch.zeros(B, dtype=torch.int32, device="cuda")
    ex.extract_batch_device(d_imgs.data_ptr(), pitch, B, w, h, w, d_kps.data_ptr(), d_desc.data_ptr(), d_n.data_ptr(), cap)
    ex.check()
    torch.cuda.synchronize()
    kps_all = d_kps.cpu().numpy().view(pkg.keypoint_dtype).reshape(B, cap)
    desc_all, n = d_desc.cpu().numpy(), d_n.cpu().numpy()
    for i in range(B):
        okps, odesc, _ = _oracle_run(oracle, ("noise", 7 + i), imgs[i], nf, DEFAULT)
        _cmp_kps(kps_all[i, :n[i]], okps, "device image %d" % i)
        assert np.array_equal(desc_all[i, :n[i]], odesc), i


# ---------------------------------------------------------------- stereo on the new shapes
BF = 386.1448


@pytest.mark.parametrize("w,h,nf", [(752, 480, 1200), (1920, 1080, 4000)])
def test_stereo_new_shapes(pkg, oracle, w, h, nf):
    left, right = synth_stereo(w, h, 5)
    ex = pkg.ORBextractor(nf, *DEFAULT, max_width=w, max_height=h, max_batch=2)
    (kL, dL), (kR, dR) = ex.extract_batch([left, right])
    ur, dp, nm = ex.stereo_match(0, 1, 1, BF, 0.0)
    oL, oR = oracle.extractor(nf, *DEFAULT), oracle.extractor(nf, *DEFAULT)
    okL, odL = oL(left)
    okR, odR = oR(right)
    _cmp_kps(kL, okL, "left")
    _cmp_kps(kR, okR, "right")
    n, our, odp = oracle.compute_stereo_matches(oL, oR, okL, odL, okR, odR, BF, 0.0)
    assert n == int(nm[0]) and n > 50
    assert np.array_equal(ur[0, :len(kL)], our) and np.array_equal(dp[0, :len(kL)], odp)


def test_stereo_record_cap_above_limit(pkg):
    """b2s_stereo_match stages at most ST_MAXR = 4096 right keypoints per CTA: a larger record cap is refused."""
    ex = pkg.ORBextractor(4100, *DEFAULT, max_width=640, max_height=480, max_batch=2)
    assert ex.cap > 4096
    img = synth_texture("noise", 640, 480, 3)
    ex.extract_batch([img, img])
    with pytest.raises(pkg.B200SlamError) as e:
        ex.stereo_match(0, 1, 1, BF)
    assert e.value.code == B2S_ERR_BAD_ARG


# ---------------------------------------------------------------- committed golden (no oracle at run time)
def test_noise_golden(pkg):
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "extract_640x480_noise_12_7.npz"))
    ex = pkg.ORBextractor(1000, 1.2, 8, 12, 7, max_width=640, max_height=480)
    k, d = ex(synth_texture("noise", 640, 480, 3))
    assert k.tobytes() == g["kps"].tobytes() and np.array_equal(d, g["desc"])
