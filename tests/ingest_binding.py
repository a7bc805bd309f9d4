"""Shared pieces of the frame ingest tests: the oracle's orc_gray_from_color / orc_remap_linear / orc_depth_u16
(oracle/liborb_ingest.so, oracle/ingest.mk), the conversion Tracking::GrabImage* selects, seeded synthetic stereo
calibrations and their rectification maps, and colour frames built from tests/synth.py images."""
import ctypes
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_LIB = os.path.join(ROOT, "oracle", "liborb_ingest.so")
vp, c_f, c_i, c_sz = ctypes.c_void_p, ctypes.c_float, ctypes.c_int, ctypes.c_size_t


def gray_code(channels, rgb):
    """The cvtColor code src/Tracking.cc:252-278 (:313-326, :371-384) applies to a `channels`-channel frame with mbRGB =
    rgb; None for one channel (the frame is used as it is)."""
    import cv2
    if channels == 3:
        return cv2.COLOR_RGB2GRAY if rgb else cv2.COLOR_BGR2GRAY
    if channels == 4:
        return cv2.COLOR_RGBA2GRAY if rgb else cv2.COLOR_BGRA2GRAY
    return None


def depth_multiplier(depth_map_factor):
    """mDepthMapFactor of the Tracking constructor (src/Tracking.cc:212-216), in float."""
    f = np.float32(depth_map_factor)
    return np.float32(1) if abs(float(f)) < 1e-5 else np.float32(np.float32(1) / f)


def cv2_prepare(img, rgb, maps=None):
    """What the reference's callers do on the host: the stereo example's cv::remap (per camera), then GrabImage*'s
    cvtColor."""
    import cv2
    if maps is not None:
        img = cv2.remap(img, maps[0], maps[1], cv2.INTER_LINEAR)
    code = gray_code(1 if img.ndim == 2 else img.shape[2], rgb)
    return img if code is None else cv2.cvtColor(img, code)


def all_triples(channels, seed=0):
    """Every (c0, c1, c2) byte triple once, as a 4096 x 4096 image (a random alpha byte for 4 channels)."""
    v = np.arange(1 << 24, dtype=np.uint32)
    img = np.stack([(v >> 16) & 255, (v >> 8) & 255, v & 255], -1).astype(np.uint8)
    if channels == 4:
        a = np.random.default_rng(seed).integers(0, 256, (1 << 24, 1), dtype=np.uint8)
        img = np.concatenate([img, a], -1)
    return img.reshape(4096, 4096, channels)


def colour_frame(w, h, seed, channels=3):
    """A colour frame whose channels are independent synth_image textures, offset so that even their flat patches differ
    (a 4th channel: random alpha)."""
    from synth import synth_image
    ch = [((synth_image(w, h, seed + 7 * k).astype(np.int32) + 71 * k) % 256).astype(np.uint8) for k in range(3)]
    if channels == 4:
        ch.append(np.random.default_rng(seed).integers(0, 256, (h, w), dtype=np.uint8))
    return np.ascontiguousarray(np.stack(ch[:channels], -1)) if channels > 1 else ch[0]


def _rot(rng, deg):
    import cv2
    r = rng.normal(size=3)
    r *= np.deg2rad(deg) / np.linalg.norm(r)
    return cv2.Rodrigues(r)[0]


# Seeded synthetic calibrations (not any real rig's): (source w, h), (output w, h), focal, distortion model
CALIBS = {
    "barrel_752x480": ((752, 480), (752, 480), 458.0, (-0.28, 0.074, 2e-4, 2e-5)),
    "pincushion_640x480": ((640, 480), (640, 480), 520.0, (0.21, -0.12, -1e-3, 6e-4, 0.05)),
    "resized_800x500_to_752x480": ((800, 500), (752, 480), 470.0, (-0.25, 0.06, 1e-4, -3e-4)),
}


def rectify_maps(name, seed=0):
    """initUndistortRectifyMap(K, D, R, P, size, CV_32FC1) for the left (seed) and right (seed + 1) cameras of a synthetic
    rig: K and D jittered from CALIBS[name], R a rotation of about a degree, P a new camera matrix with its own focal and
    centre.  Returns [(mapx, mapy) left, (mapx, mapy) right], float32 [h, w]."""
    import cv2
    (sw, sh), (w, h), f, dist = CALIBS[name]
    out = []
    for cam in range(2):
        rng = np.random.default_rng(1000 * seed + cam)
        K = np.float64([[f * (1 + rng.uniform(-.02, .02)), 0, sw / 2 + rng.uniform(-8, 8)],
                        [0, f * (1 + rng.uniform(-.02, .02)), sh / 2 + rng.uniform(-8, 8)], [0, 0, 1]])
        D = np.float64(dist) * (1 + rng.uniform(-.1, .1, len(dist)))
        R = _rot(rng, 1.0)
        fp = f * 0.95
        P = np.float64([[fp, 0, w / 2 + rng.uniform(-5, 5), 0], [0, fp, h / 2 + rng.uniform(-5, 5), 0], [0, 0, 1, 0]])
        mx, my = cv2.initUndistortRectifyMap(K, D, R, P, (w, h), cv2.CV_32FC1)
        out.append((np.ascontiguousarray(mx), np.ascontiguousarray(my)))
    return out


def phase_maps(sw, sh, rows=8, seed=0):
    """Maps that visit every one of the 1,024 sub-pixel phases (ax, ay) once per row, at random integer bases inside the
    source: [rows, 1024] each."""
    rng = np.random.default_rng(seed)
    ph = np.arange(1024)
    ax, ay = ph % 32, ph // 32
    bx = rng.integers(0, sw - 1, (rows, 1024))
    by = rng.integers(0, sh - 1, (rows, 1024))
    return (bx + ax / 32).astype(np.float32), (by + ay / 32).astype(np.float32)


def tie_maps(sw, sh, rows=8, seed=1):
    """Coordinates on exact half ties of the x32 rounding, (2k + 1) / 64, inside and across every border."""
    rng = np.random.default_rng(seed)
    kx = rng.integers(-3 * 32, (sw + 3) * 32, (rows, 1024))
    ky = rng.integers(-3 * 32, (sh + 3) * 32, (rows, 1024))
    return ((2 * kx + 1) / 64).astype(np.float32), ((2 * ky + 1) / 64).astype(np.float32)


def border_maps(sw, sh, seed=2):
    """Coordinates up to 3 px past each border, and every 1/32 step from -1.5 to 0.5 and across the far edges."""
    rng = np.random.default_rng(seed)
    mx = rng.uniform(-3, sw + 3, (16, 1024)).astype(np.float32)
    my = rng.uniform(-3, sh + 3, (16, 1024)).astype(np.float32)
    steps = np.arange(-48, 17) / 32
    edges_x = np.concatenate([steps, sw - 1 + steps, sw + steps])
    edges_y = np.concatenate([steps, sh - 1 + steps, sh + steps])
    n = len(edges_x)
    mx[0, :n], my[0, :n] = edges_x, rng.uniform(0, sh - 1, n)
    mx[1, :n], my[1, :n] = rng.uniform(0, sw - 1, n), edges_y
    mx[2, :n], my[2, :n] = edges_x, edges_y
    return mx, my


def nonfinite_maps(sw, sh, seed=3):
    """NaN, +-inf, +-1e6, +-1e30 and the largest floats, alone in one coordinate or in both, among ordinary ones."""
    rng = np.random.default_rng(seed)
    mx = rng.uniform(0, sw - 1, (4, 512)).astype(np.float32)
    my = rng.uniform(0, sh - 1, (4, 512)).astype(np.float32)
    bad = np.float32([np.nan, np.inf, -np.inf, 1e6, -1e6, 1e30, -1e30, np.finfo(np.float32).max,
                      -np.finfo(np.float32).max, 2.0 ** 26, -2.0 ** 26, 67108863.0, -1025.0, 1024.5 * 32])
    k = len(bad)
    mx[0, :k] = bad
    my[1, :k] = bad
    mx[2, :k], my[2, :k] = bad, bad[::-1]
    mx[3, :k], my[3, :k] = bad, bad
    return mx, my


class Oracle:
    def __init__(self):
        L = self.L = ctypes.CDLL(ORACLE_LIB)
        L.orc_gray_from_color.argtypes = [vp, c_sz, c_i, c_i, c_i, c_i, vp, c_sz]
        L.orc_gray_from_color.restype = None
        L.orc_remap_linear.argtypes = [vp, c_sz, c_i, c_i, c_i, vp, vp, c_sz, c_i, c_i, vp]
        L.orc_remap_linear.restype = None
        L.orc_depth_u16.argtypes = [vp, c_sz, c_f, vp]
        L.orc_depth_u16.restype = c_f

    def gray(self, img, rgb):
        img = np.ascontiguousarray(img, np.uint8)
        h, w = img.shape[:2]
        c = 1 if img.ndim == 2 else img.shape[2]
        out = np.empty((h, w), np.uint8)
        self.L.orc_gray_from_color(img.ctypes.data, w * c, w, h, c, int(bool(rgb)), out.ctypes.data, w)
        return out

    def remap(self, img, mapx, mapy):
        img = np.ascontiguousarray(img, np.uint8)
        sh, sw = img.shape[:2]
        c = 1 if img.ndim == 2 else img.shape[2]
        mapx, mapy = np.ascontiguousarray(mapx, np.float32), np.ascontiguousarray(mapy, np.float32)
        h, w = mapx.shape
        out = np.empty((h, w) + ((c,) if c > 1 else ()), np.uint8)
        self.L.orc_remap_linear(img.ctypes.data, sw * c, sw, sh, c, mapx.ctypes.data, mapy.ctypes.data, w * 4, w, h,
                                out.ctypes.data)
        return out

    def prepare(self, img, rgb, maps=None):
        if maps is not None:
            img = self.remap(img, *maps)
        return self.gray(img, rgb)

    def depth_u16(self, raw, depth_map_factor):
        raw = np.ascontiguousarray(raw, np.uint16)
        out = np.empty(raw.shape, np.float32)
        m = self.L.orc_depth_u16(raw.ctypes.data, raw.size, float(depth_map_factor), out.ctypes.data)
        return out, np.float32(m)
