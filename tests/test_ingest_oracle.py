"""The frame ingest's CPU restatement (oracle/orb_ingest.cpp) against cv2 4.x, byte for byte, and the Tracking-side rules
it stands for:

  * cvtColor RGB2GRAY / BGR2GRAY / RGBA2GRAY / BGRA2GRAY on all 2^24 byte triples (random alpha), and which of them
    Tracking::GrabImage* picks for each (channels, mbRGB);
  * remap(INTER_LINEAR, CV_32FC1 maps, BORDER_CONSTANT 0) at every sub-pixel phase, on exact half ties of the x32
    rounding, past every border, on NaN / inf / huge coordinates, on initUndistortRectifyMap maps of seeded synthetic rigs
    (one with a source larger than the output), with 1, 3 and 4 channels;
  * remap then grey conversion (the order the stereo examples and GrabImageStereo imply) equals cvtColor(remap(colour)),
    and is not the same as the other order;
  * the 16-bit depth conversion and its multiplier for DepthMapFactor 5000, 1 and 1e-6."""
import numpy as np
import pytest

import ingest_binding as ib

cv2 = pytest.importorskip("cv2")
# the grey coefficients are those of OpenCV 4 (DESIGN.md §2, deviation 9): the restatement is pinned to a 4.x cv2
pytestmark = pytest.mark.skipif(int(cv2.__version__.split(".")[0]) < 4, reason="pinned to OpenCV 4.x")


@pytest.fixture(scope="module")
def orc():
    return ib.Oracle()


@pytest.mark.parametrize("channels,rgb", [(3, True), (3, False), (4, True), (4, False)],
                         ids=["RGB2GRAY", "BGR2GRAY", "RGBA2GRAY", "BGRA2GRAY"])
def test_gray_on_every_triple(orc, channels, rgb):
    img = ib.all_triples(channels, seed=channels)
    want = cv2.cvtColor(img, ib.gray_code(channels, rgb))
    assert np.array_equal(orc.gray(img, rgb), want)
    # the 15-bit formula itself
    c = img.reshape(-1, channels).astype(np.int64)
    r, b = (c[:, 0], c[:, 2]) if rgb else (c[:, 2], c[:, 0])
    assert np.array_equal(((9798 * r + 19235 * c[:, 1] + 3735 * b + 16384) >> 15).astype(np.uint8), want.reshape(-1))


def test_tracking_selects_the_conversion_by_mbRGB(orc):
    """src/Tracking.cc:252-278: the code follows mbRGB, not the data; one channel passes through; alpha never counts."""
    img4 = ib.colour_frame(97, 61, 5, channels=4)
    for channels in (1, 3, 4):
        img = img4[..., 0] if channels == 1 else np.ascontiguousarray(img4[..., :channels])
        for rgb in (True, False):
            code = ib.gray_code(channels, rgb)
            want = img if code is None else cv2.cvtColor(img, code)
            assert np.array_equal(orc.gray(img, rgb), want), (channels, rgb)
    assert not np.array_equal(orc.gray(img4[..., :3].copy(), True), orc.gray(img4[..., :3].copy(), False))
    other_alpha = img4.copy()
    other_alpha[..., 3] ^= 0xFF
    assert np.array_equal(orc.gray(img4, True), orc.gray(other_alpha, True))


def _check_remap(orc, src, mx, my):
    want = cv2.remap(src, mx, my, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
    got = orc.remap(src, mx, my)
    assert got.shape == want.shape
    assert np.array_equal(got, want), int((got != want).sum())
    return want


@pytest.mark.parametrize("channels", [1, 3, 4])
def test_remap_every_phase(orc, channels):
    src = ib.colour_frame(200, 120, 11, channels)
    mx, my = ib.phase_maps(200, 120)
    assert len({(int(round(x * 32)) % 32, int(round(y * 32)) % 32) for x, y in zip(mx[0], my[0])}) == 1024
    _check_remap(orc, src, mx, my)


@pytest.mark.parametrize("channels", [1, 3, 4])
def test_remap_half_ties(orc, channels):
    src = ib.colour_frame(160, 90, 12, channels)
    mx, my = ib.tie_maps(160, 90)
    assert ((mx * 64) % 2 == 1).all() and ((my * 64) % 2 == 1).all()
    _check_remap(orc, src, mx, my)


@pytest.mark.parametrize("channels", [1, 3, 4])
def test_remap_past_every_border(orc, channels):
    src = ib.colour_frame(150, 100, 13, channels)
    mx, my = ib.border_maps(150, 100)
    out = _check_remap(orc, src, mx, my)
    assert (out == 0).any() and (out != 0).any()


@pytest.mark.parametrize("channels", [1, 3, 4])
def test_remap_non_finite_and_huge_coordinates(orc, channels):
    src = ib.colour_frame(120, 80, 14, channels)
    src[src == 0] = 1  # a 0 in the output then means "outside"
    mx, my = ib.nonfinite_maps(120, 80)
    with np.errstate(invalid="ignore", over="ignore"):
        out = _check_remap(orc, src, mx, my)
    for r in range(4):
        assert (out[r, :14] == 0).all()
        assert (out[r, 14:] != 0).all()


@pytest.mark.parametrize("name", sorted(ib.CALIBS))
@pytest.mark.parametrize("channels", [1, 3, 4])
def test_remap_rectification_maps(orc, name, channels):
    (sw, sh), (w, h), _, _ = ib.CALIBS[name]
    for side, (mx, my) in enumerate(ib.rectify_maps(name)):
        assert mx.shape == (h, w)
        src = ib.colour_frame(sw, sh, 20 + side, channels)
        _check_remap(orc, src, mx, my)


@pytest.mark.parametrize("rgb", [True, False])
@pytest.mark.parametrize("channels", [3, 4])
def test_remap_then_gray_is_the_examples_order(orc, channels, rgb):
    (mx, my), _ = ib.rectify_maps("barrel_752x480")
    src = ib.colour_frame(752, 480, 30, channels)
    want = ib.cv2_prepare(src, rgb, (mx, my))
    assert np.array_equal(want, cv2.cvtColor(cv2.remap(src, mx, my, cv2.INTER_LINEAR), ib.gray_code(channels, rgb)))
    assert np.array_equal(orc.prepare(src, rgb, (mx, my)), want)
    other_order = cv2.remap(cv2.cvtColor(src, ib.gray_code(channels, rgb)), mx, my, cv2.INTER_LINEAR)
    assert (other_order != want).sum() > 1000


@pytest.mark.parametrize("factor,mult", [(5000.0, np.float32(1) / np.float32(5000)), (1.0, 1.0), (1e-6, 1.0)])
def test_depth_u16_multiplier_and_conversion(orc, factor, mult):
    raw = np.arange(65536, dtype=np.uint16)
    got, m = orc.depth_u16(raw, factor)
    assert m == np.float32(mult) == ib.depth_multiplier(factor)
    # one rounding of an exact double product: what convertTo gives in float or in double, with or without FMA
    want = (raw.astype(np.float64) * np.float64(np.float32(mult))).astype(np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert np.array_equal(got, raw.astype(np.float32) * np.float32(mult))
    assert got[0] == 0 and got[65535] == np.float32(65535) * np.float32(mult)
