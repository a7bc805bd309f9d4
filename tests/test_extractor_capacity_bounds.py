"""Host-only check (no GPU) that every extractor buffer covers its worst case for each shape and parameter set of the
extractor sweep (tests/test_extractor_sweep_gpu.py), whatever the image content.  The bounds are restated here from the
geometry of src/ORBextractor.cc; the allocations come from b2s_debug_extractor_plan, which runs the same sizing code as
b2s_extractor_create / build_geometry without touching a device.

  * candidates of a level: the cell NMS keeps strict 3x3 maxima inside each cell's detectable area, at most one per 2x2
    block of that area, so a level holds at most sum over cells of ceil(cw/2) * ceil(ch/2);
  * k_cells: one CTA collects the maxima of cellsPerCta cells of one row of cells in a list of CL_CAP entries;
  * k_fast_cells_list: one cell's maxima in a list of 1024 entries;
  * FAST cells, NMS bitmap words (4 x 32 words per 128 x 32 tile)."""
import ctypes

import numpy as np
import pytest

from synth import level_sizes, residue_shapes

CASES = [(w, h, 2000, 1.2, 8) for (w, h) in [(640, 480), (1241, 376), (752, 480), (1226, 370), (1280, 720), (1920, 1080),
                                            (321, 243), (221, 221), (333, 250), (642, 481), (1023, 367), (645, 483),
                                            (8192, 8192), (8192, 221)]]
CASES += [(3840, 400, 2000, 1.2, 4)]
CASES += [(w, h, 1000, 1.2, 8) for (w, h) in residue_shapes()[0]]
CASES += [(w, h, 1000, sf, nl) for (w, h) in [(800, 600), (1920, 1080), (1280, 720)]
          for sf, nl in [(1.2, 1), (1.2, 2), (1.1, 12), (1.05, 12), (1.44, 6), (2.0, 4)]]
CASES += [(640, 480, nf, 1.2, 8) for nf in (1, 17, 500, 5000)]


def _plan(pkg, nf, sf, nl, max_w, max_h, w, h):
    L = ctypes.CDLL(pkg.LIB_PATH)
    L.b2s_debug_extractor_plan.argtypes = [ctypes.c_int, ctypes.c_float] + [ctypes.c_int] * 5 + [ctypes.c_void_p]
    L.b2s_last_error.restype = ctypes.c_char_p
    out = np.zeros(8 + 8 * 12, np.int64)
    rc = L.b2s_debug_extractor_plan(nf, sf, nl, max_w, max_h, w, h, out.ctypes.data)
    head = dict(zip(("cand_alloc", "cand_total", "cell_alloc", "cells", "bm_alloc", "cl_cap", "cl_maxcols", "fast_cell_cap"),
                    (int(v) for v in out[:8])))
    lv = [dict(zip(("w", "h", "nCols", "nRows", "wCell", "hCell", "candCap", "cellsPerCta"), (int(v) for v in out[8 + 8 * l:16 + 8 * l])))
          for l in range(nl)]
    return rc, head, lv, L.b2s_last_error().decode()


def _grid(w, h):
    width, height = np.float32(w - 32), np.float32(h - 32)
    nc, nr = int(width / np.float32(30)), int(height / np.float32(30))
    return nc, nr, int(np.ceil(width / np.float32(nc))), int(np.ceil(height / np.float32(nr)))


def _spans(n, cell, maxb, margin):
    """detectable extents of the cells of one grid row / column (:1089-1120); skipped cells omitted"""
    out = []
    for j in range(n):
        ini = 16 + j * cell
        if ini >= maxb - margin:
            break
        mx = min(ini + cell + 6, maxb)
        if mx - ini >= 7:
            out.append(mx - ini - 6)
    return out


def _bounds(w, h):
    nc, nr, wc, hc = _grid(w, h)
    cols = _spans(nc, wc, w - 16, 6)
    rows = _spans(nr, hc, h - 16, 3)
    half = lambda s: sum((d + 1) // 2 for d in s)  # noqa: E731
    return dict(nCols=nc, nRows=nr, wCell=wc, hCell=hc, cand=half(cols) * half(rows), cols=cols, rows=rows,
                cell_max=max((c + 1) // 2 * ((r + 1) // 2) for c in cols for r in rows))


@pytest.mark.parametrize("w,h,nf,sf,nl", CASES)
def test_allocations_cover_worst_case(pkg, w, h, nf, sf, nl):
    rc, head, lv, err = _plan(pkg, nf, sf, nl, w, h, w, h)
    assert rc == 0, err
    sizes = level_sizes(w, h, sf, nl)
    cand_total = cells = bm = 0
    for l, (lw, lh) in enumerate(sizes):
        g, b = lv[l], _bounds(lw, lh)
        assert (g["w"], g["h"]) == (lw, lh), l
        assert (g["nCols"], g["nRows"], g["wCell"], g["hCell"]) == (b["nCols"], b["nRows"], b["wCell"], b["hCell"]), l
        assert g["candCap"] >= b["cand"], "level %d: candidate capacity %d < worst case %d" % (l, g["candCap"], b["cand"])
        # k_cells: the cells one CTA owns can never overflow its list, nor its per-cell counters
        cpc = g["cellsPerCta"]
        assert 1 <= cpc <= head["cl_maxcols"]
        worst = max(sum((c + 1) // 2 for c in b["cols"][j:j + cpc]) for j in range(0, len(b["cols"]), cpc)) * \
            max((r + 1) // 2 for r in b["rows"])
        assert worst <= head["cl_cap"], "level %d: %d maxima per k_cells CTA > %d" % (l, worst, head["cl_cap"])
        assert b["cell_max"] <= head["fast_cell_cap"]
        cand_total += -(-b["cand"] // 64) * 64
        cells += b["nCols"] * b["nRows"]
        bm += -(-lw // 128) * 4 * (-(-lh // 32) * 32)
    assert head["cand_total"] >= cand_total and head["cand_alloc"] >= head["cand_total"]
    assert head["cells"] == cells and head["cell_alloc"] >= cells
    assert head["bm_alloc"] >= bm


@pytest.mark.parametrize("w,h,nf,sf,nl", [c for c in CASES if c[0] <= 1920 and c[1] <= 1080][::3])
def test_smaller_images_fit_the_handle(pkg, w, h, nf, sf, nl):
    """Buffers are sized once for max_width x max_height: every smaller image must plan within them."""
    for dw, dh in [(0, 0), (-1, 0), (0, -1), (-37, -11), (-w // 3, -h // 4)]:
        rc, head, lv, err = _plan(pkg, nf, sf, nl, w, h, w + dw, h + dh)
        if rc != 0:
            assert "too small for the 30-px FAST cell grid" in err or "portrait" in err, err
            continue
        assert head["cand_alloc"] >= head["cand_total"] and head["cell_alloc"] >= head["cells"]


def test_old_heuristics_were_short():
    """What the sizing replaced: min(65535, max(1024, w*h/10)) candidates per level and 4 (W/28+2)(H/28+2) + 64 cells
    are below the worst case for dense 1080p frames and for 1.05 x 12 levels."""
    lw, lh = level_sizes(1920, 1080, 1.2, 8)[0]
    assert min(65535, max(1024, lw * lh // 10)) < _bounds(lw, lh)["cand"]
    cells = sum(_bounds(a, b)["nCols"] * _bounds(a, b)["nRows"] for a, b in level_sizes(1920, 1080, 1.05, 12))
    assert (-(-1920 // 28) + 2) * (-(-1080 // 28) + 2) * 4 + 64 < cells


def test_refused_geometry_message(pkg):
    rc, _, _, err = _plan(pkg, 500, 1.2, 8, 221, 221, 220, 221)
    assert rc == 2 and "pyramid level 7 (61x62) is too small for the 30-px FAST cell grid" in err
    rc, _, _, err = _plan(pkg, 500, 1.2, 8, 221, 221, 221, 221)
    assert rc == 0, err
