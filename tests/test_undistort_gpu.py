"""b2s_undistort_keypoints_device, b2s_stereo_from_depth_device and b2s_undistort_points on the H100, bit for bit:

  * against the cv2-pinned restatement (tests/test_undistort_oracle.py) on real extractor records at 640 x 480 and
    1241 x 376 for every calibration, and against the numpy ComputeStereoFromRGBD;
  * a ragged batch of 32 images with stale records past each count (and one count above cap) equals its single-image
    calls and leaves the padding untouched; repeated calls are bit-identical; k1 == 0 copies the records byte for byte;
  * the chain extract -> undistort -> depth -> frame grid with the computed bounds gives the reference's own RGB-D Frame
    (mvKeysUn, mvuRight, mvDepth, GetFeaturesInArea) where oracle/_ref is built;
  * every refused argument writes nothing."""
import os

import numpy as np
import pytest

import undistort_binding as ub
from synth import synth_image

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
NAMES = ["tum1", "tum1_4", "tum2", "tum2_4", "tum3", "euroc", "euroc_5", "k1zero_p1", "pincushion", "barrel"]
REC = 28  # bytes of one b2s_keypoint record


def _records(t):
    """[..., cap, 28] uint8 device tensor -> numpy keypoint records [..., cap]."""
    a = np.ascontiguousarray(t.cpu().numpy())
    return a.view(ub.kp_dtype).reshape(a.shape[:-1])


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _extract(pkg, imgs, nf):
    """b2s_extract_batch_device on same-sized images; returns (extractor, kps [B, cap, 28] u8, counts [B] i32, cap)."""
    B = len(imgs)
    h, w = imgs[0].shape
    ex = pkg.ORBextractor(nf, 1.2, 8, 20, 7, max_width=w, max_height=h, max_batch=B)
    cap = ex.cap
    d_img = torch.from_numpy(np.stack(imgs)).cuda()
    kps = torch.zeros((B, cap, REC), dtype=torch.uint8, device="cuda")
    desc = torch.zeros((B, cap, 32), dtype=torch.uint8, device="cuda")
    counts = torch.zeros(B, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    ex.extract_batch_device(d_img.data_ptr(), w * h, B, w, h, w, kps.data_ptr(), desc.data_ptr(), counts.data_ptr(), cap)
    ex.check()
    return ex, kps, desc, counts, cap


@pytest.fixture(scope="module", params=[(640, 480, 1500), (1241, 376, 2000)], ids=["640x480", "1241x376"])
def extracted(request, pkg):
    w, h, nf = request.param
    ex, kps, desc, counts, cap = _extract(pkg, [synth_image(w, h, 21)], nf)
    n = int(counts[0])
    assert 1000 <= n <= 2000 + 16
    return ex, kps, desc, counts, cap, w, h


@pytest.mark.parametrize("name", NAMES)
def test_undistort_keypoints_equal_the_restatement(pkg, extracted, name):
    ex, kps, _, counts, cap, w, h = extracted
    K4, dist = ub.calib(name)
    out = torch.full_like(kps, 0xA5)
    ex.undistort_keypoints_device(kps, counts, 1, cap, K4, dist, out)
    ex.check()
    n = int(counts[0])
    src, got = _records(kps)[0, :n], _records(out)[0]
    xy = np.stack([src["x"], src["y"]], 1)
    want = ub.np_undistort(xy, K4, dist) if dist[0] != 0 else xy
    assert np.array_equal(_bits(np.stack([got["x"][:n], got["y"][:n]], 1)), _bits(want))
    for f in ("size", "angle", "response", "octave", "class_id"):
        assert np.array_equal(got[f][:n], src[f]), f
    assert (out[0, n:] == 0xA5).all()  # past the count: untouched
    if dist[0] == 0:  # k1 == 0: the records, byte for byte
        assert torch.equal(out[0, :n], kps[0, :n])
    # the host entry point on the same points
    assert np.array_equal(_bits(ex.undistort_points(xy, K4, dist)), _bits(ub.np_undistort(xy, K4, dist)))


@pytest.mark.parametrize("name", ["tum1", "tum2_4", "euroc", "k1zero_p1"])
def test_stereo_from_depth_equals_the_restatement(pkg, extracted, name):
    ex, kps, _, counts, cap, w, h = extracted
    K4, dist = ub.calib(name)
    un = torch.empty_like(kps)
    ex.undistort_keypoints_device(kps, counts, 1, cap, K4, dist, un)
    depth = ub.depth_image(w, h, seed=NAMES.index(name))
    # a padded row pitch (w + 3 floats)
    dpad = torch.zeros((1, h, w + 3), dtype=torch.float32, device="cuda")
    dpad[0, :, :w] = torch.from_numpy(depth).cuda()
    ur = torch.full((1, cap), 7.0, device="cuda")
    dd = torch.full((1, cap), 7.0, device="cuda")
    torch.cuda.synchronize()
    ex.stereo_from_depth_device(kps, un, counts, 1, cap, dpad[:, :, :w], 40.0, ur, dd)
    ex.check()
    n = int(counts[0])
    want_ur, want_d = ub.np_stereo_from_depth(_records(kps)[0, :n], _records(un)[0, :n], depth, 40.0)
    assert np.array_equal(_bits(ur[0, :n].cpu().numpy()), _bits(want_ur))
    assert np.array_equal(_bits(dd[0, :n].cpu().numpy()), _bits(want_d))
    assert (ur[0, n:] == 7.0).all() and (dd[0, n:] == 7.0).all()
    assert (want_d == -1).any() and np.isposinf(want_d).any()


def test_ragged_batch_equals_single_calls(pkg):
    """32 images of synthetic records with stale entries past each count (counts 0, 1, cap, cap + 5 among them): the
    batch call equals the 32 single-image calls, writes nothing past min(count, cap), and repeats bit for bit."""
    B, cap, w, h = 32, 2000, 640, 480
    ex = pkg.ORBextractor(1000, 1.2, 8, 20, 7, max_width=w, max_height=h, max_batch=1)
    rng = np.random.default_rng(4)
    rec = np.zeros((B, cap), ub.kp_dtype)
    rec["x"] = rng.uniform(0, w - 1e-3, (B, cap))
    rec["y"] = rng.uniform(0, h - 1e-3, (B, cap))
    rec["size"], rec["angle"], rec["response"] = 31.0, rng.uniform(0, 360, (B, cap)), rng.uniform(0, 100, (B, cap))
    rec["octave"], rec["class_id"] = rng.integers(0, 8, (B, cap)), -1
    counts_h = rng.integers(0, cap + 1, B).astype(np.int32)
    counts_h[:4] = [0, 1, cap, cap + 5]
    kps = torch.from_numpy(rec.view(np.uint8).reshape(B, cap, REC)).cuda()
    counts = torch.from_numpy(counts_h).cuda()
    depth = torch.from_numpy(np.stack([ub.depth_image(w, h, seed=100 + b) for b in range(B)])).cuda()
    K4, dist = ub.calib("tum1")
    stale = torch.from_numpy(rng.integers(0, 256, (B, cap, REC), dtype=np.uint8)).cuda()
    stale_f = torch.from_numpy(rng.uniform(-5, 5, (B, cap)).astype(np.float32)).cuda()

    def batch_run():
        un, ur, dd = stale.clone(), stale_f.clone(), stale_f.clone()
        torch.cuda.synchronize()
        ex.undistort_keypoints_device(kps, counts, B, cap, K4, dist, un)
        ex.stereo_from_depth_device(kps, un, counts, B, cap, depth, 40.0, ur, dd)
        ex.check()
        return un, ur, dd

    un, ur, dd = batch_run()
    un2, ur2, dd2 = batch_run()
    assert torch.equal(un, un2) and torch.equal(ur.view(torch.int32), ur2.view(torch.int32))
    assert torch.equal(dd.view(torch.int32), dd2.view(torch.int32))
    s_un, s_ur, s_dd = stale.clone(), stale_f.clone(), stale_f.clone()
    torch.cuda.synchronize()
    for b in range(B):
        ex.undistort_keypoints_device(kps[b], counts[b:b + 1], 1, cap, K4, dist, s_un[b])
        ex.stereo_from_depth_device(kps[b], s_un[b], counts[b:b + 1], 1, cap, depth[b:b + 1], 40.0, s_ur[b], s_dd[b])
    ex.check()
    assert torch.equal(un, s_un)
    assert torch.equal(ur.view(torch.int32), s_ur.view(torch.int32)) and torch.equal(dd.view(torch.int32), s_dd.view(torch.int32))
    for b in range(B):
        n = min(int(counts_h[b]), cap)
        assert torch.equal(un[b, n:], stale[b, n:]) and torch.equal(ur[b, n:], stale_f[b, n:])
        assert torch.equal(dd[b, n:].view(torch.int32), stale_f[b, n:].view(torch.int32))
        r = rec[b, :n]
        want = ub.np_undistort(np.stack([r["x"], r["y"]], 1), K4, dist)
        got = _records(un[b])[:n]
        assert np.array_equal(_bits(np.stack([got["x"], got["y"]], 1)), _bits(want))
        wur, wd = ub.np_stereo_from_depth(r, got, depth[b].cpu().numpy(), 40.0)
        assert np.array_equal(_bits(ur[b, :n].cpu().numpy()), _bits(wur))
        assert np.array_equal(_bits(dd[b, :n].cpu().numpy()), _bits(wd))


@pytest.mark.skipif(not os.path.exists(ub.REF_LIB), reason="oracle/_ref not built")
@pytest.mark.parametrize("name", ["tum1", "euroc_5", "tum2_4", "pincushion"])
def test_rgbd_chain_equals_the_reference_frame(pkg, name):
    """extract -> undistort -> depth -> b2s_frame_grid_create_device over image_bounds(), all on the device, against the
    reference's own RGB-D Frame on the same image, calibration and depth."""
    w, h, nf = 640, 480, 2000
    K4, dist = ub.calib(name)
    img = synth_image(w, h, 31)
    depth = ub.depth_image(w, h, seed=9)
    F = ub.RefMonoFrame(img, K4, dist, depth=depth, nf=nf)
    ex, kps, desc, counts, cap = _extract(pkg, [img], nf)
    n = int(counts[0])
    assert n == F.N
    un = torch.empty_like(kps)
    ur = torch.empty((1, cap), dtype=torch.float32, device="cuda")
    dd = torch.empty((1, cap), dtype=torch.float32, device="cuda")
    ex.undistort_keypoints_device(kps, counts, 1, cap, K4, dist, un)
    ex.stereo_from_depth_device(kps, un, counts, 1, cap, torch.from_numpy(depth)[None].cuda(), 40.0, ur, dd)
    ex.check()
    got = _records(un)[0, :n]
    for f in ("x", "y", "size", "angle", "response"):
        assert np.array_equal(_bits(got[f]), _bits(F.kps_un[f])), f
    assert np.array_equal(got["octave"], F.kps_un["octave"])
    assert np.array_equal(_bits(ur[0, :n].cpu().numpy()), _bits(F.uright))
    assert np.array_equal(_bits(dd[0, :n].cpu().numpy()), _bits(F.depth))
    bounds = ex.image_bounds(w, h, K4, dist)
    assert np.array_equal(_bits([bounds[k] for k in ("mnMinX", "mnMaxX", "mnMinY", "mnMaxY")]), _bits(F.bounds))
    geom = dict(bounds, bf=np.float32(40.0), scale_factors=ex.GetScaleFactors())
    m = pkg.ORBmatcher(0.9, True, max_features=cap)
    grid = pkg.FrameGrid(m, geom=geom, d_kps_ptr=un.data_ptr(), d_desc_ptr=desc.data_ptr(), d_uright_ptr=ur.data_ptr(), nf=n)
    x, y = got["x"], got["y"]
    outside = (x < bounds["mnMinX"]) | (x >= bounds["mnMaxX"]) | (y < bounds["mnMinY"]) | (y >= bounds["mnMaxY"])
    if name == "pincushion":  # keypoints PosInGrid may drop
        assert outside.any()
    rng = np.random.default_rng(5)
    for _ in range(400):
        qx = float(rng.uniform(bounds["mnMinX"] - 40, bounds["mnMaxX"] + 40))
        qy = float(rng.uniform(bounds["mnMinY"] - 40, bounds["mnMaxY"] + 40))
        r = float(rng.choice([3.0, 15.0, 60.0, 200.0]))
        lo, hi = [(-1, -1), (0, 2), (1, -1)][rng.integers(3)]
        assert np.array_equal(grid.GetFeaturesInArea(qx, qy, r, lo, hi), F.features_in_area(qx, qy, r, lo, hi))
    grid.close()


def test_refused_arguments_write_nothing(pkg):
    import ctypes
    L, vp = pkg.lib(), ctypes.c_void_p
    ex = pkg.ORBextractor(500, 1.2, 8, 20, 7, max_width=640, max_height=480)
    cap, B, w, h = 64, 2, 640, 480
    kps = torch.zeros((B, cap, REC), dtype=torch.uint8, device="cuda")
    kps.view(torch.float32)[..., :2] = 10.0
    counts = torch.full((B,), cap, dtype=torch.int32, device="cuda")
    out = torch.full((B, cap, REC), 0x5A, dtype=torch.uint8, device="cuda")
    ur = torch.full((B, cap), 3.0, device="cuda")
    dd = torch.full((B, cap), 3.0, device="cuda")
    depth = torch.ones((B, h, w), device="cuda")
    K4, dist = ub.calib("tum1")
    nan = np.float32(np.nan)
    torch.cuda.synchronize()

    def und(h_=ex._h, k=kps, c=counts, b=B, cp=cap, K=K4, d=dist, nd=None, o=out):
        Kc, dc = np.ascontiguousarray(K, np.float32), np.ascontiguousarray(d, np.float32)
        return L.b2s_undistort_keypoints_device(h_, vp(k.data_ptr()) if k is not None else None,
                                                vp(c.data_ptr()) if c is not None else None, b, cp,
                                                Kc.ctypes.data if K is not None else None,
                                                dc.ctypes.data if d is not None else None, len(dc) if nd is None else nd,
                                                vp(o.data_ptr()) if o is not None else None, None)

    BAD = pkg.ERR_BAD_ARG
    assert und(nd=3) == BAD and und(nd=6) == BAD and und(d=dist[:3]) == BAD
    assert und(d=np.float32([0.1, nan, 0, 0])) == BAD and und(d=np.float32([0.1, 0, 0, np.inf, 0])) == BAD
    assert und(K=np.float32([0, 500, 320, 240])) == BAD and und(K=np.float32([500, 0, 320, 240])) == BAD
    assert und(K=np.float32([nan, 500, 320, 240])) == BAD and und(K=np.float32([500, 500, np.inf, 240])) == BAD
    assert und(b=0) == BAD and und(cp=0) == BAD and und(h_=None) == BAD
    assert und(k=None) == BAD and und(c=None) == BAD and und(o=None) == BAD and und(K=None) == BAD and und(d=None) == BAD

    def dep(h_=ex._h, b=B, cp=cap, pitch=w * 4, ww=w, hh=h, c=counts, o=ur):
        return L.b2s_stereo_from_depth_device(h_, vp(kps.data_ptr()), vp(kps.data_ptr()),
                                              vp(c.data_ptr()) if c is not None else None, b, cp, vp(depth.data_ptr()),
                                              pitch, ww, hh, 40.0, vp(o.data_ptr()) if o is not None else None,
                                              vp(dd.data_ptr()), None)

    assert dep(pitch=w * 4 - 4) == BAD and dep(pitch=w * 4 + 2) == BAD and dep(ww=0) == BAD and dep(hh=0) == BAD
    assert dep(b=0) == BAD and dep(cp=0) == BAD and dep(h_=None) == BAD and dep(c=None) == BAD and dep(o=None) == BAD
    xy = np.float32([[1, 2], [3, 4]])
    xo = np.full_like(xy, 9.0)
    assert L.b2s_undistort_points(ex._h, xy.ctypes.data, 2, K4.ctypes.data, dist.ctypes.data, 3, xo.ctypes.data) == BAD
    assert L.b2s_undistort_points(ex._h, xy.ctypes.data, -1, K4.ctypes.data, dist.ctypes.data, 5, xo.ctypes.data) == BAD
    assert L.b2s_undistort_points(ex._h, None, 2, K4.ctypes.data, dist.ctypes.data, 5, xo.ctypes.data) == BAD
    ex.check()
    assert (out == 0x5A).all() and (ur == 3.0).all() and (dd == 3.0).all() and (xo == 9.0).all()
    # the same handle still works, and n = 0 is a no-op
    assert L.b2s_undistort_points(ex._h, None, 0, K4.ctypes.data, dist.ctypes.data, 5, None) == pkg.OK
    assert und() == pkg.OK and dep() == pkg.OK
    ex.check()
    assert not (out == 0x5A).all() and not (ur == 3.0).all()
