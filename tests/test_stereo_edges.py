"""Frame::ComputeStereoMatches (src/Frame.cc:1026-1421) at its decision edges, on hand-made keypoints and images fed
identically to three implementations:

  * the reference's own, unmodified Frame.cc, through ref_frame_stereo_inject (oracle/ref_stereo_glue.cpp: the Frame is
    built on the pair, then its public keypoint / descriptor / baseline members are overwritten and
    ComputeStereoMatches runs again);
  * the CPU oracle (oracle/orb_stereo.cpp), which also reports the decision that settled each left keypoint;
  * the device (k_stereo_match + k_stereo_cull) through b2s_stereo_match_device, on the pyramids the handle extracted
    from the same pair.

Images are a textured base and a right image made of per-row-region integer horizontal shifts of it, so every true
match is known.  Where a case needs an exact SAD of k, exactly k non-centre pixels of the right window are raised by 1;
where it needs dist1 == dist3, the base is mirrored about the keypoint's column.  Keypoint coordinates are exact floats.

Each case asserts, through the oracle's reason codes (and the SAD profile where the branch is a tie), that it reaches its
branch.  Every comparison is on float bits."""
import ctypes
import os

import numpy as np
import pytest

from oracle_binding import kp_dtype

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libref_stereo.so")
need_ref = pytest.mark.skipif(not os.path.exists(REF_LIB), reason="oracle/_ref not built (make -C oracle ref)")
vp, c_f, c_i = ctypes.c_void_p, ctypes.c_float, ctypes.c_int

W, H = 320, 240
PADX = 160  # the base is wider than the image, so that a shifted right image never runs out of texture
NF = 300    # features the reference's constructor extracts (their pyramids are what matters here)
P8, P4 = (1.2, 8), (1.5, 4)  # the device extractor needs a 30-px FAST cell on every level
BF = 40.0   # with MB = 0.5, maxD = bf / mb = 80 exactly
MB = 0.5
MAXR = 4096  # ST_MAXR: right (and left) records per pair on the device
B2S_ERR_BAD_ARG = 2

# ORC_ST_* (oracle/orb_oracle.h)
KEPT, KEPT_ZERO, NO_ROW, MAXU, NO_CAND, HAMMING, WINDOW, EDGE, DELTA, DISPARITY, CULLED = range(11)
NAMES = ["kept", "kept_zero_disparity", "no_row", "maxU<0", "no_candidate", "hamming>=75", "window", "edge_incR",
         "deltaR", "disparity", "culled"]
MATCHED = {KEPT, KEPT_ZERO, CULLED}  # passed every per-keypoint gate
UNMATCHED = {NO_ROW, NO_CAND, HAMMING}
f32 = np.float32


def _tables(sf, nl):
    """mvScaleFactors / mvInvScaleFactors and the level sizes (src/ORBextractor.cc:431-449, :1572-1576), in float."""
    sc = [f32(1.0)]
    for _ in range(1, nl):
        sc.append(f32(sc[-1] * f32(sf)))
    sc = np.array(sc, np.float32)
    isc = (f32(1.0) / sc).astype(np.float32)
    dims = [(int(np.rint(f32(W) * s)), int(np.rint(f32(H) * s))) for s in isc]
    return sc, isc, dims


def _below(y, r, row):
    """largest float y' <= y with floor(y' - r) == row (in float), and the next float up (its floor is row + 1)"""
    y = f32(y)
    while np.floor(f32(y - r)) > row:
        y = np.nextafter(y, f32(-np.inf))
    while np.floor(f32(np.nextafter(y, f32(np.inf)) - r)) == row:
        y = np.nextafter(y, f32(np.inf))
    out = np.nextafter(y, f32(np.inf))
    assert np.floor(f32(y - r)) == row and np.floor(f32(out - r)) == row + 1
    return y, out


def _above(y, r, row):
    """smallest float y' >= y with ceil(y' + r) == row, and the next float down (its ceil is row - 1)"""
    y = f32(y)
    while np.ceil(f32(y + r)) < row:
        y = np.nextafter(y, f32(np.inf))
    while np.ceil(f32(np.nextafter(y, f32(-np.inf)) + r)) == row:
        y = np.nextafter(y, f32(-np.inf))
    out = np.nextafter(y, f32(-np.inf))
    assert np.ceil(f32(y + r)) == row and np.ceil(f32(out + r)) == row - 1
    return y, out


def _x_for_level(target, o, sc, isc, half=False):
    """a float x whose round(x * invScale[o]) is `target` (half: x * invScale[o] == target - 0.5 exactly, so that round
    goes half away from zero to target)"""
    want = f32(target - 0.5) if half else f32(target)
    x0 = f32(want * sc[o])
    x = x0
    for k in range(64):
        for s in (1, -1):
            x = x0
            for _ in range(k):
                x = np.nextafter(x, f32(s * np.inf))
            p = f32(x * isc[o])
            if (p == want) if half else (np.round(p) == target and abs(p - want) < 0.25):
                return float(x)
    raise AssertionError("no float x with x*inv == %r at octave %d" % (want, o))


class Case:
    """One stereo pair with hand-made keypoints.  Rows of the right image default to a noisy shift of d0; a region
    (y0, y1, d, noise, period) overrides whole rows."""

    def __init__(self, name, seed, params=P8, mb=0.0, bf=BF, d0=16):
        self.name, self.params, self.mb, self.bf = name, params, mb, bf
        self.rng = np.random.RandomState(seed)
        self.sc, self.isc, self.dims = _tables(*params)
        b = self.rng.randint(0, 256, (H + 2, W + PADX + 2)).astype(np.float64)
        b = (b[:-2] + 2 * b[1:-1] + b[2:]) / 4
        b = (b[:, :-2] + 2 * b[:, 1:-1] + b[:, 2:]) / 4
        b = (b - b.min()) / (b.max() - b.min()) * 210 + 20
        self.base = np.rint(b).astype(np.int32)
        self.d0 = d0
        self.regions, self.raises = [], []
        self.kl, self.kr, self.dl, self.dr = [], [], [], []
        self.expect, self.facts = {}, []
        self.ref_ok = True
        self.built = None

    # ---- image edits (applied in build(), in this order: periodic rows, mirrors, right image, raises)
    def region(self, y0, y1, d, noise=True, period=None):
        self.regions.append((y0, y1, d, noise, period))

    def mirror(self, x, y, half=16, rows=9):
        """make the base mirror-symmetric about column x on rows y +- rows: then SAD(incR) == SAD(-incR) about the true
        match, so dist1 == dist3 and deltaR == 0"""
        self.facts.append(("mirror", int(x), int(y), half, rows))

    def raise_sad(self, xr, y, k):
        """raise k non-centre pixels of the 11x11 right window centred at (xr, y) by 1 (level 0): SAD k at the true match"""
        self.raises.append((int(xr), int(y), k))

    # ---- keypoints
    def left(self, x, y, o=0, expect=None):
        self.kl.append((x, y, o))
        self.dl.append(self.rng.randint(0, 256, 32).astype(np.uint8))
        if expect is not None:
            self.expect[len(self.kl) - 1] = expect if isinstance(expect, set) else {expect}
        return len(self.kl) - 1

    def right(self, x, y, o=0, near=None, dist=10):
        """a right keypoint; near = a left index: its descriptor is that one's with exactly `dist` bits flipped"""
        if near is None:
            d = self.rng.randint(0, 256, 32).astype(np.uint8)
        else:
            d = self.dl[near].copy()
            for bit in self.rng.choice(256, dist, replace=False):
                d[bit >> 3] ^= np.uint8(1 << (bit & 7))
        self.kr.append((x, y, o))
        self.dr.append(d)
        return len(self.kr) - 1

    def build(self):
        if self.built is not None:
            return self.built
        base = self.base.copy()
        rng = np.random.RandomState(self.rng.randint(1 << 30))
        for (y0, y1, d, noise, period) in self.regions:
            if period:
                pat = rng.randint(20, 236, (y1 - y0, period))
                base[y0:y1] = pat[:, np.arange(base.shape[1]) % period]
        for (kind, x, y, half, rows) in [f for f in self.facts if f[0] == "mirror"]:
            for t in range(1, half + 1):
                base[y - rows:y + rows + 1, x + t] = base[y - rows:y + rows + 1, x - t]
        L = base[:, :W].copy()
        cols = np.arange(W)
        R = base[:, cols + self.d0] + rng.randint(-2, 3, (H, W))
        for (y0, y1, d, noise, period) in self.regions:
            R[y0:y1] = base[y0:y1][:, cols + d]
            if noise and period:
                R[y0:y1] += rng.randint(-2, 3, (y1 - y0, period))[:, (cols + d) % period]
            elif noise:
                R[y0:y1] += rng.randint(-2, 3, (y1 - y0, W))
        for (xr, y, k) in self.raises:
            offs = [(dy, dx) for dy in range(-5, 6) for dx in range(-5, 6) if (dy, dx) != (0, 0)]
            for j in range(k):
                dy, dx = offs[j % 120]
                R[y + dy, xr + dx] += 1
        assert L.min() >= 0 and L.max() <= 255 and R.min() >= 0 and R.max() <= 255
        kl = np.zeros(len(self.kl), kp_dtype)
        kr = np.zeros(len(self.kr), kp_dtype)
        for k, src in ((kl, self.kl), (kr, self.kr)):
            for i, (x, y, o) in enumerate(src):
                k[i]["x"], k[i]["y"], k[i]["octave"] = x, y, o
                k[i]["size"], k[i]["angle"], k[i]["response"], k[i]["class_id"] = 31.0 * self.sc[o], 0.0, 1.0, -1
        dl = np.array(self.dl, np.uint8).reshape(-1, 32)
        dr = np.array(self.dr, np.uint8).reshape(-1, 32)
        self.built = (L.astype(np.uint8), R.astype(np.uint8), kl, dl, kr, dr)
        return self.built


# ------------------------------------------------------------------------------------------------------------- cases
def _companions(c, rows, xs=(90, 170, 250)):
    """noisy matches on the background shift: SAD > 0, so that the median of a case stays above the exact matches"""
    for y in rows:
        for x in xs:
            i = c.left(float(x), float(y), 0, MATCHED)
            c.right(float(x - c.d0), float(y), 0, near=i)


def case_disparity_bound():
    c = Case("disparity_bound", 1, mb=MB)  # maxD = 80, minU = uL - 80
    c.region(31, 50, 80, noise=False)  # disparity exactly maxD: rejected (the test is < maxD)
    c.mirror(200, 40)
    i = c.left(200.0, 40.0, 0, DISPARITY)
    c.right(120.0, 40.0, 0, near=i)
    c.region(61, 80, 79, noise=False)  # maxD - 1: kept
    c.mirror(200, 70)
    i = c.left(200.0, 70.0, 0, KEPT)
    c.right(121.0, 70.0, 0, near=i)
    c.facts += [("d1==d3", 0), ("d1==d3", 1)]
    c.region(91, 110, 77)  # uR == minU: a candidate (inclusive); the block matching finds the true match 3 px right
    i = c.left(200.0, 100.0, 0, KEPT)
    c.right(120.0, 100.0, 0, near=i)
    c.left(-2.0, 100.0, 0, MAXU)  # maxU = uL < 0, with right keypoints in the row
    c.region(121, 140, 3)  # uR == uL == maxU: a candidate (inclusive)
    i = c.left(150.0, 130.0, 0, KEPT)
    c.right(150.0, 130.0, 0, near=i)
    c.region(151, 170, 77)  # uR one float below minU: no candidate
    i = c.left(200.0, 160.0, 0, NO_CAND)
    c.right(float(np.nextafter(f32(120.0), f32(-np.inf))), 160.0, 0, near=i)
    _companions(c, (190, 215))
    return c


def case_zero_disparity():
    c = Case("zero_disparity", 2, mb=MB)
    c.region(50, 71, 0, noise=False)  # right == left: bestuR == uL, disparity 0 -> 0.01, bestuR = uL - 0.01 (double)
    c.mirror(160, 60)
    i = c.left(160.0, 60.0, 0, KEPT_ZERO)
    c.right(160.0, 60.0, 0, near=i)
    c.region(100, 121, 0, noise=False)
    c.mirror(97, 110)
    i = c.left(97.0, 110.0, 0, KEPT_ZERO)
    c.right(97.0, 110.0, 0, near=i)
    c.facts += [("zero", 0), ("zero", 1)]
    _companions(c, (150, 190))
    return c


def case_identical():
    """left == right everywhere: every SAD is 0, the median is 0, thDist is 0 and every match is culled"""
    c = Case("identical", 3, mb=MB, d0=0)
    c.region(0, H, 0, noise=False)
    for j, (x, y) in enumerate([(60, 40), (150, 80), (240, 120), (100, 160), (200, 200)]):
        c.mirror(x, y)
        i = c.left(float(x), float(y), 0, CULLED)
        c.right(float(x), float(y), 0, near=i)
    c.facts.append(("none_matched",))
    return c


def case_subpixel():
    """uR0 off the true match by -6..+6 px: the SAD minimum lands on incR = -off, rejected at +-5 (= L)"""
    c = Case("subpixel_offsets", 4, d0=30)
    for j, off in enumerate(range(-6, 7)):
        y = 20.0 + 15 * j
        i = c.left(150.0, y, 0, EDGE if abs(off) == 5 else (MATCHED if abs(off) < 5 else None))
        c.right(float(150 - 30 + off), y, 0, near=i)
    return c


def case_stripes():
    """periodic rows: equal SAD minima every `period` px; the first (lowest incR) must win"""
    c = Case("stripes", 5, d0=30)
    for j, (period, off, exp) in enumerate([(4, 0, MATCHED), (3, 0, MATCHED), (3, -1, EDGE), (4, 2, MATCHED)]):
        y = 40 + 50 * j
        c.region(y - 12, y + 13, 30, period=period)
        # with off, the true minimum is at incR = -off; its repeats at -off +- period
        i = c.left(150.0, float(y), 0, exp)
        c.right(float(150 - 30 + off), float(y), 0, near=i)
        c.facts.append(("tie", i))
    return c


def case_hamming_gate():
    c = Case("hamming_gate", 6, d0=20)
    for j, (dist, exp) in enumerate([(74, MATCHED), (75, HAMMING), (73, MATCHED), (76, HAMMING)]):
        y = 40.0 + 45 * j
        i = c.left(160.0, y, 0, exp)
        c.right(140.0, y, 0, near=i, dist=dist)
        c.right(100.0, y, 0, near=i, dist=min(dist + 1, 99))
    return c


def case_hamming_ties():
    """4,096 right keypoints; equal best distances at several candidates: the lowest index wins.  The losing
    candidates sit 50 px away, so a wrong pick block-matches somewhere else."""
    c = Case("hamming_ties", 7, d0=20)
    winners = [31, 32, 33, 2047, 4095]
    rows = [30.0, 70.0, 110.0, 150.0, 190.0]
    lefts = [c.left(200.0, y, 0, MATCHED) for y in rows]
    slot = {}
    for k, wi in enumerate(winners):
        slot[wi] = (k, "win")
        if wi != 4095:
            slot[wi + 1000 + k] = (k, "tie")
            slot[wi + 1900 + k] = (k, "tie")
        else:  # the last index: no later tie is possible, so earlier candidates are one bit worse
            slot[100] = (k, "worse")
            slot[1500] = (k, "worse")
    for j in range(MAXR):
        if j in slot:
            k, kind = slot[j]
            y = rows[k]
            if kind == "win":
                c.right(180.0, y, 0, near=lefts[k], dist=20)
            else:
                c.right(130.0 + (j % 7), y, 0, near=lefts[k], dist=20 if kind == "tie" else 21)
        else:  # fillers: random descriptors (~128 bits away), anywhere with their band inside the image
            c.right(float(c.rng.randint(12, 300)), float(c.rng.randint(12, 226)), int(c.rng.randint(0, 3)))
    return c


def case_octave_gate(params, lo):
    """right candidates at levelL-2 .. levelL+2; the two gated-out octaves carry the best descriptors"""
    nl = params[1]
    c = Case("octave_gate_%s_%d" % ("lo" if lo else "hi", nl), 8 + nl + lo, params=params, d0=36)
    oL = 0 if lo else nl - 1
    x, y = 160.0, 120.0
    i = c.left(x, y, oL, MATCHED)
    far = [60.0, 80.0, 100.0, 70.0]
    k = 0
    for do in (-2, -1, 0, 1, 2):
        o = oL + do
        if not 0 <= o < nl:
            continue
        if do == 0:
            c.right(x - 36, y, o, near=i, dist=30)
        else:
            c.right(far[k], y, o, near=i, dist=5 if abs(do) == 2 else 40)
            k += 1
    return c


def case_row_bands():
    """right y whose band [floor(y-r), ceil(y+r)] ends exactly on the left row, and one float past it; left y on and
    off an integer (the row truncates); octave 0 (r = 2) and octaves with non-integer r = 2*scale"""
    c = Case("row_bands", 9, d0=12)
    for g, o in enumerate((0, 1, 3)):
        r = f32(2.0) * c.sc[o]
        x = 60.0 + 90 * g
        for j, frac in enumerate((0.0, 0.75, 0.0, 0.75)):
            yl = 30 + 44 * j
            vL = f32(yl + frac)
            row = int(vL)
            if j < 2:
                y_in, y_out = _below(row + 1 + r, r, row)
            else:
                y_in, y_out = _above(row - 1 - r, r, row)
            i = c.left(x, float(vL), o, MATCHED)
            c.right(x - 12, float(y_in), o, near=i)
            i = c.left(x + 30, float(vL), o, UNMATCHED)
            c.right(x + 30 - 12, float(y_out), o, near=i)
    return c


def case_levels(params):
    """a keypoint on every octave; x with x*invScale an exact .5 (round goes half away from zero); the right window
    at scaleduR0 + 11 == level width (rejected) and == width - 1, and at cxR0 - 10 == 0 (accepted)"""
    nl = params[1]
    c = Case("levels_%d" % nl, 20 + nl, params=params, d0=24)
    sc, isc, dims = c.sc, c.isc, c.dims
    for o in range(nl):
        y = 120.0
        x = _x_for_level(int(np.round(150 * isc[o])) + 1, o, sc, isc, half=True)
        i = c.left(x, y, o)
        xr = _x_for_level(int(np.round((x - 24) * isc[o])) + 1, o, sc, isc, half=True)
        c.right(xr, y, o, near=i)
        c.facts.append(("half", i, o))
    for k, o in enumerate((0, 2)):
        lw = dims[o][0]
        for j, (su, exp) in enumerate(((lw - 11, WINDOW), (lw - 12, MATCHED))):
            y = 30.0 + 40 * (2 * k + j)
            c.region(int(y) - 20, int(y) + 21, 4 if o == 0 else 6)
            xr = _x_for_level(su, o, sc, isc)
            xl = _x_for_level(lw - 7, o, sc, isc)
            i = c.left(xl, y, o, exp)
            c.right(xr, y, o, near=i)
    c.region(185, 226, 20)  # cxR0 - 10 == 0: the leftmost right window column is 0
    i = c.left(30.0, 205.0, 0, MATCHED)
    c.right(10.0, 205.0, 0, near=i)
    return c


def case_cull(name, sads, seed, expect):
    """M matches with exact SADs (k raised pixels each) and nothing else"""
    c = Case(name, seed, d0=20)
    n = len(sads)
    for j, k in enumerate(sads):
        y = 20 + (200 // max(n, 1)) * j + 10
        x = 60 + 37 * (j % 6)
        c.region(y - 9, y + 10, 20, noise=False)
        c.raise_sad(x - 20, y, k)
        i = c.left(float(x), float(y), 0, expect[j])
        c.right(float(x - 20), float(y), 0, near=i)
        c.facts.append(("sad", i, k))
    return c


def cull_cases():
    K, C = KEPT, CULLED
    p = f32(1.5) * f32(1.4)
    assert f32(p * f32(10)) == 21 and f32(p * f32(30)) < 63 and f32(p * f32(50)) < 105
    return [
        case_cull("cull_m1", [7], 30, [K]),
        case_cull("cull_m1_zero", [0], 31, [C]),
        case_cull("cull_m2", [10, 4], 32, [K, K]),             # median = sorted[1] = 10, th 21
        case_cull("cull_m3", [13, 3, 6], 33, [C, K, K]),       # median 6, th 12.6
        case_cull("cull_m4", [9, 2, 30, 4], 34, [K, K, C, K]),  # median = sorted[2] = 9, th 18.9
        case_cull("cull_tie", [8, 20, 8, 5, 8], 35, [K, C, K, K, K]),  # ties at the median index
        case_cull("cull_tie_all", [8, 8, 8, 8], 36, [K] * 4),
        case_cull("cull_exact_21", [1, 10, 21, 10], 37, [K, K, C, K]),    # 2.1f*10 == 21.0f exactly: SAD 21 culled
        case_cull("cull_exact_42", [41, 20, 42, 1, 20], 38, [K, K, C, K, K]),
        case_cull("cull_below_63", [30, 63, 1, 62, 30], 39, [K, C, K, K, K]),  # 62.999996f
        case_cull("cull_below_105", [50, 1, 105, 104, 50], 40, [K, K, C, K, K]),
    ]


def refused_cases():
    """input on which the reference is undefined: run on the device and the oracle only"""
    out = []
    c = Case("window_left_of_level", 50, d0=20)  # cxR0 - 10 == -1: the iniu test passes, column -1 would be read
    c.region(90, 131, 20)
    i = c.left(29.0, 110.0, 0, WINDOW)
    c.right(9.0, 110.0, 0, near=i)
    _companions(c, (40, 180))
    out.append(c)
    c = Case("window_above_level", 51, d0=20)  # the left window's rows leave level 0
    i = c.left(100.0, 3.0, 0, WINDOW)
    c.right(80.0, 3.0, 0, near=i)
    _companions(c, (60, 180))
    out.append(c)
    c = Case("band_outside_image", 52, d0=20)  # a right band reaching row -1 and one reaching row H
    i = c.left(100.0, 60.0, 0)
    c.right(80.0, 1.0, 0, near=i)
    c.right(200.0, 238.5, 0)
    _companions(c, (100, 160))
    out.append(c)
    c = Case("no_left_keypoints", 53, d0=20)  # N == 0
    c.right(80.0, 60.0, 0)
    c.right(180.0, 120.0, 0)
    out.append(c)
    for c in out:
        c.ref_ok = False
    return out


def all_cases():
    cs = [case_disparity_bound(), case_zero_disparity(), case_identical(), case_subpixel(), case_stripes(),
          case_hamming_gate(), case_hamming_ties(), case_row_bands(), case_levels(P8), case_levels(P4),
          case_octave_gate(P8, True), case_octave_gate(P8, False), case_octave_gate(P4, True),
          case_octave_gate(P4, False)]
    return cs + cull_cases() + refused_cases()


_CASES = []


def cases():
    if not _CASES:
        _CASES.extend(all_cases())
    return _CASES


# ------------------------------------------------------------------------------------------------------ checkers
class OracleRun:
    """the oracle on a case, with the pyramids of an oracle extractor run on each image"""

    def __init__(self, oracle, c):
        L, R, kl, dl, kr, dr = c.build()
        sf, nl = c.params
        self.exL, self.exR = oracle.extractor(NF, sf, nl, 20, 7), oracle.extractor(NF, sf, nl, 20, 7)
        self.exL(L)
        self.exR(R)
        self.reason = np.full(len(kl), -1, np.int32)
        self.n, self.ur, self.dp = oracle.compute_stereo_matches(self.exL, self.exR, kl, dl, kr, dr, c.bf, c.mb,
                                                                 self.reason if len(kl) else None)
        self.levels = ([self.exL.level(l) for l in range(nl)], [self.exR.level(l) for l in range(nl)])


def sad_profile(run, c, iL, iR):
    """the 11 SADs of the block matching of left keypoint iL around right keypoint iR (integers)"""
    kl, kr = c.build()[2], c.build()[4]
    o = int(kl[iL]["octave"])
    inv = c.isc[o]
    cy, cxL = int(np.round(f32(kl[iL]["y"] * inv))), int(np.round(f32(kl[iL]["x"] * inv)))
    cxR0 = int(np.round(f32(kr[iR]["x"] * inv)))
    IL, IR = (a.astype(np.int64) for a in (run.levels[0][o], run.levels[1][o]))
    wl = IL[cy - 5:cy + 6, cxL - 5:cxL + 6] - IL[cy, cxL]
    out = []
    for inc in range(-5, 6):
        wr = IR[cy - 5:cy + 6, cxR0 + inc - 5:cxR0 + inc + 6] - IR[cy, cxR0 + inc]
        out.append(int(np.abs(wl - wr).sum()))
    return out


_REF = []


def ref_lib():
    if not _REF:
        R = ctypes.CDLL(REF_LIB)
        R.ref_frame_stereo_inject.argtypes = [vp, vp, c_i, c_i, c_i, c_f, c_i, c_i, c_i, vp, vp, c_i, vp, vp, c_i, c_f, c_f,
                                              vp, vp]
        _REF.append(R)
    return _REF[0]


def _flat(k):
    a = np.zeros((len(k), 7), np.float32)
    for j, f in enumerate(("x", "y", "size", "angle", "response", "octave", "class_id")):
        a[:, j] = k[f]
    return np.ascontiguousarray(a)


def ref_run(c):
    """(rc, mvuRight, mvDepth) of the reference's own ComputeStereoMatches on the case"""
    L, R, kl, dl, kr, dr = c.build()
    sf, nl = c.params
    a, b = _flat(kl), _flat(kr)
    dl, dr = np.ascontiguousarray(dl), np.ascontiguousarray(dr)
    ur, dp = np.full(max(len(kl), 1), -2, np.float32), np.full(max(len(kl), 1), -2, np.float32)
    rc = ref_lib().ref_frame_stereo_inject(L.ctypes.data, R.ctypes.data, W, H, NF, sf, nl, 20, 7, a.ctypes.data, dl.ctypes.data,
                                           len(kl), b.ctypes.data, dr.ctypes.data, len(kr), c.bf, c.mb, ur.ctypes.data,
                                           dp.ctypes.data)
    return rc, ur[:len(kl)], dp[:len(kl)]


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


# ---------------------------------------------------------------------------------------------------- CPU tests
def test_cases_reach_every_branch(oracle):
    counts = np.zeros(len(NAMES), np.int64)
    for c in cases():
        run = OracleRun(oracle, c)
        kl = c.build()[2]
        assert run.n == int((run.ur >= 0).sum()), c.name
        assert (run.reason >= 0).all()
        for iL, want in c.expect.items():
            assert run.reason[iL] in want, "%s: left %d ended in %s, expected %s" % (
                c.name, iL, NAMES[run.reason[iL]], [NAMES[w] for w in want])
        for f in c.facts:
            if f[0] == "d1==d3":  # deltaR == 0 exactly: an integer bestuR
                prof = sad_profile(run, c, f[1], f[1])
                b = int(np.argmin(prof))
                assert 0 < b < 10 and prof[b - 1] == prof[b + 1], (c.name, prof)
            elif f[0] == "zero":
                i = f[1]
                assert run.reason[i] == KEPT_ZERO
                assert bits(run.ur[i]) == bits(f32(np.float64(kl[i]["x"]) - 0.01))
                assert bits(run.dp[i]) == bits(f32(c.bf) / f32(0.01))
            elif f[0] == "none_matched":
                assert run.n == 0 and (run.ur == -1).all()
            elif f[0] == "tie":  # the SAD minimum occurs more than once inside the search range
                prof = sad_profile(run, c, f[1], f[1])
                assert prof.count(min(prof)) >= 2, (c.name, prof)
            elif f[0] == "sad":
                prof = sad_profile(run, c, f[1], f[1])
                assert min(prof) == f[2] and prof.index(min(prof)) == 5, (c.name, prof)
            elif f[0] == "half":
                i, o = f[1], f[2]
                p = f32(kl[i]["x"] * c.isc[o])
                assert p - np.floor(p) == 0.5
        counts += np.bincount(run.reason, minlength=len(NAMES))
    print("\nstereo edge cases, left keypoints per decision:")
    for k, n in enumerate(NAMES):
        print("  %-22s %6d" % (n, counts[k]))
    # With a strict first minimum dist1 > dist2 <= dist3, so |deltaR| <= 1/2 and the deltaR gate can never fire.
    assert counts[DELTA] == 0
    assert all(counts[k] > 0 for k in range(len(NAMES)) if k != DELTA), dict(zip(NAMES, counts.tolist()))


def test_zero_disparity_substitution_in_float_equals_double():
    """bestuR = uL - 0.01 is a double subtraction rounded to float.  For every float uL in [0.125, 8192) it equals the
    float subtraction uL - 0.01f, and an accepted match has uL >= scale * (cxR0 + bestincR - 1/2) >= 5.5, so no input
    can tell the two apart: the zero-disparity cases pin the value, and this pins why a float slip cannot show."""
    for m in range(-3, 13):
        u = (np.int64(f32(2.0 ** m).view(np.int32)) + np.arange(1 << 23, dtype=np.int64)).astype(np.int32).view(np.float32)
        assert np.array_equal((u.astype(np.float64) - 0.01).astype(np.float32), u - f32(0.01)), m
    u = f32(0.0625)  # below 1/8 they differ
    assert f32(np.float64(u) - 0.01) != u - f32(0.01)


@need_ref
def test_oracle_equals_reference(oracle):
    seen = 0
    for c in cases():
        rc, ur, dp = ref_run(c)
        if not c.ref_ok:
            assert rc < 0, "%s: the reference entry must refuse this input" % c.name
            continue
        assert rc == 0, "%s: refused (%d)" % (c.name, rc)
        run = OracleRun(oracle, c)
        assert np.array_equal(bits(run.ur), bits(ur)), c.name
        assert np.array_equal(bits(run.dp), bits(dp)), c.name
        seen += 1
    assert seen >= 20


# ---------------------------------------------------------------------------------------------------- GPU tests
def _device_groups():
    g = {}
    for c in cases():
        g.setdefault(c.params, []).append(c)
    return g


def _device_run(pkg, group, cap=MAXR, singles=False):
    """extract every left image then every right image of the group in one batch; stereo-match all pairs in one call
    (or each pair alone); returns per case (uright, depth, n_matched)"""
    import torch
    n = len(group)
    sf, nl = group[0].params
    ex = pkg.ORBextractor(NF, sf, nl, 20, 7, max_width=W, max_height=H, max_batch=2 * n)
    ex.extract_batch([c.build()[0] for c in group] + [c.build()[1] for c in group])
    kps = np.zeros((2 * n, cap), kp_dtype)
    desc = np.zeros((2 * n, cap, 32), np.uint8)
    cnt = np.zeros(2 * n, np.int32)
    for p, c in enumerate(group):
        _, _, kl, dl, kr, dr = c.build()
        kps[p, :len(kl)], desc[p, :len(kl)], cnt[p] = kl, dl, len(kl)
        kps[n + p, :len(kr)], desc[n + p, :len(kr)], cnt[n + p] = kr, dr, len(kr)
    d_kps = torch.from_numpy(kps.view(np.uint8).reshape(2 * n, cap, 28)).cuda()
    d_desc, d_cnt = torch.from_numpy(desc).cuda(), torch.from_numpy(cnt).cuda()
    ur = torch.full((n, cap), -2.0, dtype=torch.float32, device="cuda")
    dp = torch.full((n, cap), -2.0, dtype=torch.float32, device="cuda")
    nm = torch.full((n,), -2, dtype=torch.int32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    torch.cuda.synchronize()
    bf, mb = group[0].bf, group[0].mb
    assert all(c.bf == bf for c in group)
    if singles:
        for p, c in enumerate(group):
            ex.stereo_match_device(p, n + p, 1, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), cap, c.bf, c.mb,
                                   ur[p].data_ptr(), dp[p].data_ptr(), nm[p:].data_ptr(), stream=st)
    else:
        mbs = {c.mb for c in group}
        for m in mbs:  # one call per baseline (bf / mb is one scalar per call)
            idx = [p for p, c in enumerate(group) if c.mb == m]
            sub = [group[p] for p in idx]
            assert idx == list(range(idx[0], idx[0] + len(idx))), "group the cases by baseline"
            p0 = idx[0]
            ex.stereo_match_device(p0, n + p0, len(sub), d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), cap, bf, m,
                                   ur[p0].data_ptr(), dp[p0].data_ptr(), nm[p0:].data_ptr(), stream=st)
    torch.cuda.synchronize()
    return ur.cpu().numpy(), dp.cpu().numpy(), nm.cpu().numpy()


def _sorted_group(group):
    return sorted(group, key=lambda c: c.mb)


@pytest.mark.gpu
@pytest.mark.parametrize("params", [P8, P4], ids=["1.2x8", "1.5x4"])
def test_device_equals_oracle(pkg, oracle, params):
    """every case, including those the reference refuses (windows outside the level, bands outside the image, N = 0)"""
    group = _sorted_group(_device_groups()[params])
    ur, dp, nm = _device_run(pkg, group)
    for p, c in enumerate(group):
        N = len(c.build()[2])
        run = OracleRun(oracle, c)
        assert np.array_equal(bits(ur[p, :N]), bits(run.ur)), c.name
        assert np.array_equal(bits(dp[p, :N]), bits(run.dp)), c.name
        assert (ur[p, N:] == -1).all() and (dp[p, N:] == -1).all(), c.name
        assert int(nm[p]) == int((ur[p, :N] >= 0).sum()) == run.n, c.name


@pytest.mark.gpu
@need_ref
@pytest.mark.parametrize("params", [P8, P4], ids=["1.2x8", "1.5x4"])
def test_device_equals_reference(pkg, params):
    group = _sorted_group(_device_groups()[params])
    ur, dp, nm = _device_run(pkg, group)
    seen = 0
    for p, c in enumerate(group):
        N = len(c.build()[2])
        rc, rur, rdp = ref_run(c)
        if not c.ref_ok:
            assert rc < 0, c.name
            continue
        assert rc == 0, c.name
        assert np.array_equal(bits(ur[p, :N]), bits(rur)), c.name
        assert np.array_equal(bits(dp[p, :N]), bits(rdp)), c.name
        assert int(nm[p]) == int((rur >= 0).sum()), c.name
        seen += 1
    assert seen == sum(c.ref_ok for c in group) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("params", [P8, P4], ids=["1.2x8", "1.5x4"])
def test_device_batch_equals_single_pairs(pkg, params):
    group = _sorted_group(_device_groups()[params])
    a = _device_run(pkg, group)
    b = _device_run(pkg, group, singles=True)
    for x, y in zip(a, b):
        assert np.array_equal(np.ascontiguousarray(x).view(np.uint32), np.ascontiguousarray(y).view(np.uint32))


def capacity_case():
    """4,096 left and 4,096 right records, every left keypoint with its match"""
    c = Case("capacity", 60, d0=8)
    for j in range(MAXR):
        x = 20.0 + 4.375 * (j % 64)
        y = 20.0 + 3.125 * (j // 64)
        c.left(x, y, 0)
    for j in range(MAXR):
        c.right(c.kl[j][0] - 8.0, c.kl[j][1], 0, near=j, dist=int(j % 90))
    return c


@need_ref
def test_capacity_case_oracle_equals_reference(oracle):
    c = capacity_case()
    rc, rur, rdp = ref_run(c)
    assert rc == 0
    run = OracleRun(oracle, c)
    assert np.array_equal(bits(run.ur), bits(rur)) and np.array_equal(bits(run.dp), bits(rdp))
    assert run.n > 1000 and (run.reason == HAMMING).sum() > 0  # descriptor distances 0..89


@pytest.mark.gpu
def test_device_capacity(pkg, oracle):
    """the device on the capacity case equals the oracle (which equals the reference on it, above)"""
    import torch
    c = capacity_case()
    run = OracleRun(oracle, c)
    ur, dp, nm = _device_run(pkg, [c], cap=MAXR)
    assert np.array_equal(bits(ur[0]), bits(run.ur)) and np.array_equal(bits(dp[0]), bits(run.dp))
    assert int(nm[0]) == int((run.ur >= 0).sum()) == run.n > 1000
    # one record more than a CTA stages: refused, and nothing is written
    ex = pkg.ORBextractor(NF, 1.2, 8, 20, 7, max_width=W, max_height=H, max_batch=2)
    ex.extract_batch([c.build()[0], c.build()[1]])
    cap = MAXR + 1
    d_kps = torch.zeros((2, cap, 28), dtype=torch.uint8, device="cuda")
    d_desc = torch.zeros((2, cap, 32), dtype=torch.uint8, device="cuda")
    d_cnt = torch.tensor([10, 10], dtype=torch.int32, device="cuda")
    u = torch.full((1, cap), -2.0, dtype=torch.float32, device="cuda")
    d = torch.full((1, cap), -2.0, dtype=torch.float32, device="cuda")
    m = torch.full((1,), -2, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    with pytest.raises(pkg.B200SlamError) as e:
        ex.stereo_match_device(0, 1, 1, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), cap, BF, 0.0, u.data_ptr(),
                               d.data_ptr(), m.data_ptr(), stream=torch.cuda.current_stream().cuda_stream)
    assert e.value.code == B2S_ERR_BAD_ARG
    torch.cuda.synchronize()
    assert (u == -2).all() and (d == -2).all() and (m == -2).all()


@pytest.mark.gpu
def test_host_path_capacity(pkg):
    """b2s_stereo_match after extract_batch: an extractor whose record capacity is exactly 4,096 works, one whose
    capacity is 4,097 is refused"""
    c = case_subpixel()
    L, R = c.build()[:2]
    nl = 8
    ok = pkg.ORBextractor(MAXR - 4 * nl - 16, 1.2, nl, 20, 7, max_width=W, max_height=H, max_batch=2)
    assert ok.cap == MAXR
    ok.extract_batch([L, R])
    ur, dp, nm = ok.stereo_match(0, 1, 1, BF, 0.0)
    assert ur.shape == (1, MAXR) and int(nm[0]) == int((ur[0] >= 0).sum()) > 0
    big = pkg.ORBextractor(MAXR - 4 * nl - 15, 1.2, nl, 20, 7, max_width=W, max_height=H, max_batch=2)
    assert big.cap == MAXR + 1
    big.extract_batch([L, R])
    with pytest.raises(pkg.B200SlamError) as e:
        big.stereo_match(0, 1, 1, BF, 0.0)
    assert e.value.code == B2S_ERR_BAD_ARG
