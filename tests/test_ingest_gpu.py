"""b2s_prepare_images_device and b2s_stereo_from_depth_u16_device on the H100, byte for byte:

  * the grey conversion of all 2^24 byte triples for each of RGB2GRAY / BGR2GRAY / RGBA2GRAY / BGRA2GRAY, and every
    remap case of tests/test_ingest_oracle.py (phases, half ties, borders, non-finite coordinates, rectification maps of
    synthetic rigs, a source larger than the output; 1, 3 and 4 channels) equal cv2 and the restatement;
  * a batch of 32 images with padded rows and images at odd pitches equals its single-image calls, leaves the padding
    untouched and repeats bit for bit;
  * the u16 depth call equals the float call fed float32(raw) * float32(1 / DepthMapFactor), raw 0 and 65535 and
    keypoints on the image edges included;
  * prepare -> extract -> stereo match on rectified colour pairs equals the same chain fed cv2-prepared grey images, and
    colour + u16 depth -> prepare -> extract -> undistort -> depth equals the reference's own RGB-D Frame where oracle/_ref
    is built;
  * a StereoStream that ingests colour and rectifies equals one fed the cv2-prepared frames;
  * every refused argument writes nothing."""
import ctypes
import importlib
import os

import numpy as np
import pytest

import ingest_binding as ib
import undistort_binding as ub
from synth import synth_image, synth_stereo

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
cv2 = pytest.importorskip("cv2")
REC = 28


@pytest.fixture(scope="module")
def orc():
    return ib.Oracle()


@pytest.fixture(scope="module")
def ex(pkg):
    return pkg.ORBextractor(500, 1.2, 8, 20, 7, max_width=640, max_height=480)


def _prepare(ex, src, rgb=True, maps=None, out_hw=None):
    """One image (numpy [H, W] or [H, W, C]) through the device; returns the grey output as numpy."""
    h, w = out_hw or src.shape[:2]
    s = torch.from_numpy(np.ascontiguousarray(src)).cuda()[None]
    out = torch.full((1, h, w), 0xA5, dtype=torch.uint8, device="cuda")
    m = None if maps is None else tuple(torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda() for a in maps)
    torch.cuda.synchronize()  # the handle's stream is not ordered after torch's
    n0 = ex.launch_count()
    ex.prepare_images_device(s, out, rgb=rgb, maps=m)
    ex.check()
    assert ex.launch_count() == n0 + 1
    return out[0].cpu().numpy()


@pytest.mark.parametrize("channels,rgb", [(3, True), (3, False), (4, True), (4, False)],
                         ids=["RGB2GRAY", "BGR2GRAY", "RGBA2GRAY", "BGRA2GRAY"])
def test_gray_on_every_triple(ex, orc, channels, rgb):
    img = ib.all_triples(channels, seed=channels)
    want = cv2.cvtColor(img, ib.gray_code(channels, rgb))
    got = _prepare(ex, img, rgb)
    assert np.array_equal(got, want)
    assert np.array_equal(got, orc.gray(img, rgb))


def test_one_channel_without_maps_is_a_copy(ex):
    img = synth_image(641, 479, 3)
    assert np.array_equal(_prepare(ex, img, rgb=False), img)


def _remap_cases():
    (sw, sh) = (200, 120)
    yield "phases", (sw, sh), ib.phase_maps(sw, sh)
    yield "half_ties", (sw, sh), ib.tie_maps(sw, sh)
    yield "borders", (sw, sh), ib.border_maps(sw, sh)
    yield "non_finite", (sw, sh), ib.nonfinite_maps(sw, sh)
    for name in sorted(ib.CALIBS):
        src_size = ib.CALIBS[name][0]
        for side, maps in enumerate(ib.rectify_maps(name)):
            yield "%s_%s" % (name, "LR"[side]), src_size, maps


REMAP = list(_remap_cases())


@pytest.mark.parametrize("case", range(len(REMAP)), ids=[c[0] for c in REMAP])
@pytest.mark.parametrize("channels,rgb", [(1, True), (3, True), (4, False)], ids=["gray", "RGB", "BGRA"])
def test_remap_equals_cv2_and_the_restatement(ex, orc, case, channels, rgb):
    _, (sw, sh), (mx, my) = REMAP[case]
    src = ib.colour_frame(sw, sh, 40 + case, channels)
    with np.errstate(invalid="ignore", over="ignore"):
        want = ib.cv2_prepare(src, rgb, (mx, my))
    got = _prepare(ex, src, rgb, (mx, my), out_hw=mx.shape)
    assert np.array_equal(got, want), int((got != want).sum())
    assert np.array_equal(got, orc.prepare(src, rgb, (mx, my)))


def _strided(buf, shape, strides):
    return torch.as_strided(buf, shape, strides)


@pytest.mark.parametrize("channels,with_maps", [(3, True), (4, False), (1, True)], ids=["RGB_maps", "BGRA", "gray_maps"])
def test_padded_batch_equals_single_calls(ex, orc, channels, with_maps):
    """32 images at odd row and image pitches, output rows and images padded, maps at a pitch that is not a multiple of
    16 bytes: the batch equals 32 single calls and cv2, the padding keeps its bytes, a repeat is bit-identical."""
    B, sw, sh = 32, 331, 197
    w, h = (317, 203) if with_maps else (sw, sh)
    rgb = channels != 4
    srow, simg = sw * channels + 5, (sw * channels + 5) * sh + 7
    orow, oimg = w + 3, (w + 3) * h + 1
    frames = [ib.colour_frame(sw, sh, 60 + b, channels) for b in range(B)]
    sbuf = torch.zeros(B * simg, dtype=torch.uint8, device="cuda")
    src = _strided(sbuf, (B, sh, sw) + ((channels,) if channels > 1 else ()),
                   (simg, srow, channels, 1)[:4 if channels > 1 else 3])
    src.copy_(torch.from_numpy(np.stack(frames)))
    maps = None
    if with_maps:
        rng = np.random.default_rng(7)
        mpitch = w + 5  # floats
        mbuf = torch.from_numpy(rng.uniform(-2.5, max(sw, sh) + 2.5, 2 * h * mpitch).astype(np.float32)).cuda()
        maps = (_strided(mbuf, (h, w), (mpitch, 1)), _strided(mbuf[h * mpitch:], (h, w), (mpitch, 1)))
        maps[0].copy_(torch.from_numpy(rng.uniform(-2.5, sw + 2.5, (h, w)).astype(np.float32)))
        maps[1].copy_(torch.from_numpy(rng.uniform(-2.5, sh + 2.5, (h, w)).astype(np.float32)))
    stale = torch.from_numpy(np.random.default_rng(8).integers(0, 256, B * oimg, dtype=np.uint8)).cuda()

    def run():
        obuf = stale.clone()
        out = _strided(obuf, (B, h, w), (oimg, orow, 1))
        torch.cuda.synchronize()
        ex.prepare_images_device(src, out, rgb=rgb, maps=maps)
        ex.check()
        return obuf, out

    obuf, out = run()
    obuf2, _ = run()
    assert torch.equal(obuf, obuf2)
    single = stale.clone()
    torch.cuda.synchronize()
    for b in range(B):
        sb = _strided(sbuf[b * simg:], src.shape[1:], src.stride()[1:])
        ob = _strided(single[b * oimg:], (1, h, w), (oimg, orow, 1))
        ex.prepare_images_device(sb[None], ob, rgb=rgb, maps=maps)
    ex.check()
    assert torch.equal(obuf, single)
    mask = torch.zeros(B * oimg, dtype=torch.bool, device="cuda")
    _strided(mask, (B, h, w), (oimg, orow, 1)).fill_(True)
    assert torch.equal(obuf[~mask], stale[~mask])
    got = out.cpu().numpy()
    mh = None if maps is None else (maps[0].cpu().numpy(), maps[1].cpu().numpy())
    for b in range(B):
        want = ib.cv2_prepare(frames[b], rgb, mh)
        assert np.array_equal(got[b], want), b
        assert np.array_equal(got[b], orc.prepare(frames[b], rgb, mh)), b


def _edge_records(w, h, cap, seed):
    rng = np.random.default_rng(seed)
    rec = np.zeros(cap, ub.kp_dtype)
    rec["x"], rec["y"] = rng.uniform(0, w - 1e-3, cap), rng.uniform(0, h - 1e-3, cap)
    rec["size"], rec["angle"], rec["octave"], rec["class_id"] = 31.0, rng.uniform(0, 360, cap), rng.integers(0, 8, cap), -1
    edge = [(0, 0), (w - 1e-3, h - 1e-3), (0, h - 1e-3), (w - 1e-3, 0), (-0.5, 3), (3, -0.5), (-1, 5), (5, -1), (w, 5),
            (5, h), (np.float32(w) - np.float32(0.5), 7), (9, np.float32(h) - np.float32(0.25))]
    for i, (x, y) in enumerate(edge):
        rec["x"][i], rec["y"][i] = x, y
    return rec, len(edge)


@pytest.mark.parametrize("factor", [5000.0, 1.0, 1e-6, -1000.0])
def test_depth_u16_equals_the_float_path(pkg, factor):
    B, cap, w, h = 4, 1500, 640, 480
    ex = pkg.ORBextractor(500, 1.2, 8, 20, 7, max_width=w, max_height=h, max_batch=B)
    rng = np.random.default_rng(11)
    raw = rng.integers(0, 65536, (B, h, w), dtype=np.uint16)
    raw[rng.random((B, h, w)) < 0.1] = 0
    raw[rng.random((B, h, w)) < 0.05] = 65535
    raw[:, 0, 0], raw[:, h - 1, w - 1], raw[:, 0, w - 1], raw[:, h - 1, 0] = 0, 65535, 65535, 7
    recs = []
    for b in range(B):
        r, n_edge = _edge_records(w, h, cap, 20 + b)
        recs.append(r)
    rec = np.stack(recs)
    counts_h = np.int32([cap, cap - 3, n_edge, cap + 9])
    kps = torch.from_numpy(rec.view(np.uint8).reshape(B, cap, REC)).cuda()
    counts = torch.from_numpy(counts_h).cuda()
    K4, dist = ub.calib("tum1")
    un = torch.empty_like(kps)
    torch.cuda.synchronize()
    ex.undistort_keypoints_device(kps, counts, B, cap, K4, dist, un)
    dpad = torch.zeros((B, h, w + 3), dtype=torch.int16, device="cuda")  # padded rows; int16 carries the u16 bytes
    dpad[:, :, :w] = torch.from_numpy(raw.view(np.int16)).cuda()
    d16 = dpad[:, :, :w]
    mult = ib.depth_multiplier(factor)
    depth_f = torch.from_numpy(raw.astype(np.float32) * mult).cuda()
    stale = torch.from_numpy(rng.uniform(-5, 5, (B, cap)).astype(np.float32)).cuda()
    ur16, dd16, urf, ddf = stale.clone(), stale.clone(), stale.clone(), stale.clone()
    torch.cuda.synchronize()
    n0 = ex.launch_count()
    ex.stereo_from_depth_u16_device(kps, un, counts, B, cap, d16, factor, 40.0, ur16, dd16)
    ex.check()
    assert ex.launch_count() == n0 + 1
    ex.stereo_from_depth_device(kps, un, counts, B, cap, depth_f, 40.0, urf, ddf)
    ex.check()
    bits = lambda t: t.view(torch.int32)
    assert torch.equal(bits(ur16), bits(urf)) and torch.equal(bits(dd16), bits(ddf))
    for b in range(B):
        n = min(int(counts_h[b]), cap)
        assert torch.equal(bits(ur16[b, n:]), bits(stale[b, n:])) and torch.equal(bits(dd16[b, n:]), bits(stale[b, n:]))
        r = rec[b, :n]
        r_un = np.ascontiguousarray(un[b, :n].cpu().numpy()).view(ub.kp_dtype).reshape(n)
        # one zero row and column past the image: the outside keypoints read 0 there (and are set to -1 below)
        wur, wd = ub.np_stereo_from_depth(r, r_un, np.pad(raw[b].astype(np.float32) * mult, ((0, 1), (0, 1))), 40.0)
        inside = (r["x"] > -1) & (r["x"] < w) & (r["y"] > -1) & (r["y"] < h)
        wur[~inside], wd[~inside] = -1, -1
        assert np.array_equal(ur16[b, :n].cpu().numpy().view(np.uint32), wur.view(np.uint32))
        assert np.array_equal(dd16[b, :n].cpu().numpy().view(np.uint32), wd.view(np.uint32))
    if factor > 0:
        assert (dd16[0, :cap] > 0).any()
        assert float(dd16[2, 1]) == float(np.float32(65535) * mult)  # the corner (w-1, h-1) holds 65535
        assert float(dd16[2, 0]) == -1.0  # raw 0
    else:  # a negative multiplier: no depth anywhere
        for b in range(B):
            assert (dd16[b, :min(int(counts_h[b]), cap)] == -1).all()


def _colour_of(grey, rgb_order):
    """A colour frame whose grey conversion is textured like `grey` and whose channels differ: the same per-pixel map on
    both images of a stereo pair keeps their correspondence."""
    g = grey.astype(np.int32)
    c = np.stack([g, (g * 3 + 17) % 256, 255 - g], -1).astype(np.uint8)
    return c if rgb_order else np.ascontiguousarray(c[..., ::-1])


def _mild_maps(w, h, seed):
    """Rectification maps of one camera of a rig whose cameras differ only in the horizontal centre: rows stay rows."""
    rng = np.random.default_rng(seed)
    K = np.float64([[450, 0, w / 2 + rng.uniform(-3, 3)], [0, 450, h / 2], [0, 0, 1]])
    D = np.float64([-0.05, 0.01, 0, 0])
    mx, my = cv2.initUndistortRectifyMap(K, D, np.eye(3), K, (w, h), cv2.CV_32FC1)
    return mx, my


def _extract_pairs(ex, d_imgs, P, cap):
    w, h = d_imgs.shape[2], d_imgs.shape[1]
    kps = torch.zeros((2 * P, cap, REC), dtype=torch.uint8, device="cuda")
    desc = torch.zeros((2 * P, cap, 32), dtype=torch.uint8, device="cuda")
    counts = torch.zeros(2 * P, dtype=torch.int32, device="cuda")
    ur = torch.zeros((P, cap), dtype=torch.float32, device="cuda")
    dp = torch.zeros((P, cap), dtype=torch.float32, device="cuda")
    nm = torch.zeros(P, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    ex.extract_batch_device(d_imgs.data_ptr(), w * h, 2 * P, w, h, w, kps.data_ptr(), desc.data_ptr(), counts.data_ptr(), cap)
    ex.stereo_match_device(0, P, P, kps.data_ptr(), desc.data_ptr(), counts.data_ptr(), cap, 386.1448, 0.0, ur.data_ptr(),
                           dp.data_ptr(), nm.data_ptr())
    ex.check()
    return kps, desc, counts, ur, dp, nm


def test_rectified_colour_stereo_chain_equals_the_cv2_prepared_chain(pkg):
    P, w, h, nf = 3, 752, 480, 1200
    rgb = False
    pairs = [synth_stereo(w, h, 70 + i) for i in range(P)]
    raw = np.stack([_colour_of(p[0], rgb) for p in pairs] + [_colour_of(p[1], rgb) for p in pairs])
    maps = [_mild_maps(w, h, 1), _mild_maps(w, h, 2)]
    grey = np.stack([ib.cv2_prepare(raw[i], rgb, maps[i // P]) for i in range(2 * P)])
    ex = pkg.ORBextractor(nf, 1.2, 8, 20, 7, max_width=w, max_height=h, max_batch=2 * P)
    cap = ex.cap
    d_raw = torch.from_numpy(raw).cuda()
    d_imgs = torch.empty((2 * P, h, w), dtype=torch.uint8, device="cuda")
    ms = [tuple(torch.from_numpy(a).cuda() for a in maps[side]) for side in range(2)]
    torch.cuda.synchronize()
    for side in range(2):
        ex.prepare_images_device(d_raw[side * P:(side + 1) * P], d_imgs[side * P:(side + 1) * P], rgb=rgb, maps=ms[side])
    ex.check()
    assert np.array_equal(d_imgs.cpu().numpy(), grey)
    a = _extract_pairs(ex, d_imgs, P, cap)
    b = _extract_pairs(ex, torch.from_numpy(grey).cuda(), P, cap)
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.uint8), y.view(torch.uint8))
    assert int(a[5].sum()) > 100  # stereo matches were made


@pytest.mark.skipif(not os.path.exists(ub.REF_LIB), reason="oracle/_ref not built")
@pytest.mark.parametrize("name", ["tum1", "euroc_5"])
def test_rgbd_colour_u16_chain_equals_the_reference_frame(pkg, name):
    """TUM-style input: BGR bytes with Camera.RGB = 1 (the reference follows mbRGB, not the data) and 16-bit depth with
    DepthMapFactor 5000 -> prepare -> extract -> undistort -> u16 depth, against the reference's own RGB-D Frame built on
    GrabImageRGBD's cvtColor and convertTo of the same frame."""
    w, h, nf, factor = 640, 480, 2000, 5000.0
    K4, dist = ub.calib(name)
    colour = ib.colour_frame(w, h, 31, 3)
    raw = np.clip(np.rint(ub.depth_image(w, h, seed=9, special=False) * factor), 0, 65535).astype(np.uint16)
    raw[np.random.default_rng(3).random((h, w)) < 0.05] = 0
    grey = cv2.cvtColor(colour, cv2.COLOR_RGB2GRAY)
    F = ub.RefMonoFrame(grey, K4, dist, depth=raw.astype(np.float32) * ib.depth_multiplier(factor), nf=nf)
    ex = pkg.ORBextractor(nf, 1.2, 8, 20, 7, max_width=w, max_height=h)
    cap = ex.cap
    d_img = torch.empty((1, h, w), dtype=torch.uint8, device="cuda")
    d_col = torch.from_numpy(colour)[None].cuda()
    kps = torch.zeros((1, cap, REC), dtype=torch.uint8, device="cuda")
    desc = torch.zeros((1, cap, 32), dtype=torch.uint8, device="cuda")
    counts = torch.zeros(1, dtype=torch.int32, device="cuda")
    d16 = torch.from_numpy(raw.view(np.int16))[None].cuda()
    torch.cuda.synchronize()  # the handle's stream is not ordered after torch's
    ex.prepare_images_device(d_col, d_img, rgb=True)
    ex.extract_batch_device(d_img.data_ptr(), w * h, 1, w, h, w, kps.data_ptr(), desc.data_ptr(), counts.data_ptr(), cap)
    ex.check()  # synchronises the handle's stream
    assert np.array_equal(d_img[0].cpu().numpy(), grey)
    n = int(counts[0])
    assert n == F.N
    un = torch.empty_like(kps)
    ur = torch.empty((1, cap), dtype=torch.float32, device="cuda")
    dd = torch.empty((1, cap), dtype=torch.float32, device="cuda")
    ex.undistort_keypoints_device(kps, counts, 1, cap, K4, dist, un)
    ex.stereo_from_depth_u16_device(kps, un, counts, 1, cap, d16, factor, 40.0, ur, dd)
    ex.check()
    got = np.ascontiguousarray(un[0, :n].cpu().numpy()).view(ub.kp_dtype).reshape(n)
    for f in ("x", "y", "size", "angle", "response"):
        assert np.array_equal(got[f].view(np.uint32), F.kps_un[f].view(np.uint32)), f
    assert np.array_equal(ur[0, :n].cpu().numpy().view(np.uint32), F.uright.view(np.uint32))
    assert np.array_equal(dd[0, :n].cpu().numpy().view(np.uint32), F.depth.view(np.uint32))
    assert (F.depth > 0).sum() > 100 and (F.depth == -1).any()


def test_stream_with_colour_and_rectification_equals_cv2_prepared_frames(pkg):
    stream_mod = importlib.import_module("self_commit_orb-slam2_b200.stream")
    F, w, h, nf = 3, 752, 480, 1500
    rgb = True
    pairs = [synth_stereo(w, h, 80 + i) for i in range(F)]
    raw = np.stack([_colour_of(p[0], rgb) for p in pairs] + [_colour_of(p[1], rgb) for p in pairs])
    maps = [_mild_maps(w, h, 3), _mild_maps(w, h, 4)]
    grey = np.stack([ib.cv2_prepare(raw[i], rgb, maps[i // F]) for i in range(2 * F)])
    kw = dict(stereo=True, project=True)
    a = stream_mod.StereoStream(F, w, h, nf, source_channels=3, rgb=rgb,
                                rectify=(maps[0][0], maps[0][1], maps[1][0], maps[1][1]), **kw)
    b = stream_mod.StereoStream(F, w, h, nf, **kw)
    assert a.h2d_bytes_per_step() - b.h2d_bytes_per_step() == 2 * F * w * h * 2
    with pytest.raises(ValueError):
        a.step_host(grey)

    def state(s):
        torch.cuda.synchronize()
        s.ex.check()
        return [t.clone() for t in (s.counts, s.kps, s.desc, s.ur, s.dp_all, s.match, s.nmatch, s.pmatch, s.npmatch)]

    a.upload(torch.from_numpy(raw))
    a.step_device()
    b.upload(torch.from_numpy(grey))
    b.step_device()
    sa, sb = state(a), state(b)
    for x, y in zip(sa, sb):
        assert torch.equal(x, y)
    assert int(sa[6].sum()) > 0 and int(sa[8].sum()) > 0 and int((sa[3] >= 0).sum()) > 100
    # load_window from resident raw frames (D = 4, wrapping) == the grey stream's
    D = 4
    extra = [synth_stereo(w, h, 90 + i) for i in range(D - F)]
    allp = pairs + extra
    raw_all = np.stack([np.stack([_colour_of(p[k], rgb) for p in allp]) for k in range(2)])
    grey_all = np.stack([np.stack([ib.cv2_prepare(raw_all[k, i], rgb, maps[k]) for i in range(D)]) for k in range(2)])
    a.load_window(torch.from_numpy(raw_all).cuda(), 2)
    a.step_device()
    b.load_window(torch.from_numpy(grey_all).cuda(), 2)
    b.step_device()
    for x, y in zip(state(a), state(b)):
        assert torch.equal(x, y)


def test_refused_arguments_write_nothing(pkg, ex):
    L, vp = pkg.lib(), ctypes.c_void_p
    B, sw, sh, C = 2, 64, 48, 3
    src = torch.full((B, sh, sw, C), 9, dtype=torch.uint8, device="cuda")
    out = torch.full((B, sh, sw), 0x5A, dtype=torch.uint8, device="cuda")
    mx = torch.zeros((sh, sw), dtype=torch.float32, device="cuda")
    my = torch.zeros((sh, sw), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    BAD = pkg.ERR_BAD_ARG

    def prep(h_=ex._h, s=src, srow=sw * C, simg=sw * C * sh, b=B, w0=sw, h0=sh, c=C, x=None, y=None, mrow=sw * 4, w=sw,
             h=sh, o=out, orow=sw, oimg=sw * sh):
        p = lambda t: vp(t.data_ptr()) if t is not None else None
        return L.b2s_prepare_images_device(h_, p(s), srow, simg, b, w0, h0, c, 1, p(x), p(y), mrow, w, h, p(o), orow, oimg,
                                           None)

    cases = [dict(h_=None), dict(s=None), dict(o=None), dict(x=mx), dict(y=my), dict(b=0), dict(b=65536),
             dict(c=2, srow=sw * 2, simg=sw * 2 * sh), dict(c=0), dict(c=5), dict(w0=0), dict(h0=0), dict(w=0), dict(h=0),
             dict(w0=8193), dict(x=mx, y=my, w=8193), dict(srow=sw * C - 1), dict(simg=sw * C * sh - 1),
             dict(orow=sw - 1), dict(oimg=sw * sh - 1), dict(x=mx, y=my, mrow=sw * 4 - 4), dict(x=mx, y=my, mrow=sw * 4 + 2),
             dict(w=sw - 1, orow=sw - 1, oimg=(sw - 1) * sh), dict(h=sh - 1, oimg=sw * (sh - 1))]
    for kw in cases:
        assert prep(**kw) == BAD, kw

    kps = torch.zeros((B, 8, REC), dtype=torch.uint8, device="cuda")
    counts = torch.full((B,), 8, dtype=torch.int32, device="cuda")
    depth = torch.ones((B, sh, sw), dtype=torch.int16, device="cuda")
    ur = torch.full((B, 8), 3.0, device="cuda")
    dd = torch.full((B, 8), 3.0, device="cuda")

    def dep(h_=ex._h, k=kps, c=counts, b=B, cp=8, d=depth, pitch=sw * 2, w=sw, h=sh, f=5000.0, o=ur):
        p = lambda t: vp(t.data_ptr()) if t is not None else None
        return L.b2s_stereo_from_depth_u16_device(h_, p(k), p(k), p(c), b, cp, p(d), pitch, w, h, f, 40.0, p(o), p(dd), None)

    for kw in [dict(h_=None), dict(k=None), dict(c=None), dict(d=None), dict(o=None), dict(b=0), dict(b=65536), dict(cp=0),
               dict(w=0), dict(h=0), dict(pitch=sw * 2 - 2), dict(pitch=sw * 2 + 1), dict(f=float("nan")),
               dict(f=float("inf")), dict(f=float("-inf"))]:
        assert dep(**kw) == BAD, kw
    ex.check()
    torch.cuda.synchronize()
    assert (out == 0x5A).all() and (ur == 3.0).all() and (dd == 3.0).all()
    # the same handle still works
    assert prep() == pkg.OK and prep(x=mx, y=my) == pkg.OK and dep() == pkg.OK
    ex.check()
    assert not (out == 0x5A).all() and not (dd == 3.0).all()
