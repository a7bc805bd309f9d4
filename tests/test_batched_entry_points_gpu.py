"""Batched entry points, member by member: every member of a ragged batch against the CPU oracle on its own unpadded slice
and, bit for bit, against the single-pair call of the same entry point.

The stream's step calls the kernels with up to 160 stereo pairs, records strided by a capacity, counts read from device
memory, records past each count left over from earlier steps, and handles reused across steps and batch sizes.  The
batches here look like that:
  - per-member counts sit on the kernels' tile edges: 0, 1, 31-33 (warps), 127-129 (BI_ROWS of k_bow_topk_imma), about
    1000 and the capacity itself;
  - every slot past a count holds real records of the same member ("stale padding": the member's own features that the
    count leaves out, with their descriptors, vocabulary node, valid flag and coordinates), so a kernel that reads past a
    count finds candidates there and changes its matches;
  - one run per entry point zeroes the padding instead, and must give the same result.
Each member is one independent CTA or warp with a fixed reduction order, so a batched result is bit-identical to the
single call, not merely close to it."""
import ctypes
import importlib

import numpy as np
import pytest

from synth import synth_descriptors, synth_local_ba, synth_pose_problem, synth_projection, synth_stereo

pytestmark = pytest.mark.gpu

W, H, NFEAT = 1241, 376, 2000
FX, FY, CX, CY, BF = 718.856, 718.856, 607.1928, 185.2157, 386.1448
RAGGED = (0, 1, 31, 32, 33, 127, 128, 129, 1000, None)  # None: the member's capacity
_vp = ctypes.c_void_p


def ragged_counts(B, cap, shift, avail=None):
    """B per-member counts taken round-robin from RAGGED, starting at `shift`, clamped to cap (and to `avail`)."""
    n = np.array([cap if RAGGED[(k + shift) % len(RAGGED)] is None else RAGGED[(k + shift) % len(RAGGED)]
                  for k in range(B)], np.int32)
    n = np.minimum(n, cap)
    if avail is not None:
        n = np.minimum(n, np.asarray(avail, np.int32))
    return np.ascontiguousarray(n, np.int32)


def zero_padded(a, n):
    """Copy of the batch array a [B, cap, ...] with every slot past n[b] zeroed."""
    z = np.array(a, copy=True)
    for b, k in enumerate(n):
        z[b, k:] = 0
    return z


def _p(a):
    return None if a is None else a.ctypes.data_as(_vp)


def extract_full(pkg, ex, imgs):
    """b2s_extract_batch on a host batch; full record arrays [B, cap] (slots past a count keep what they held: zeros)."""
    B = len(imgs)
    imgs = np.ascontiguousarray(np.stack(imgs))
    kps = np.zeros((B, ex.cap), pkg.keypoint_dtype)
    desc = np.zeros((B, ex.cap, 32), np.uint8)
    n = np.zeros(B, np.int32)
    ptrs = (_vp * B)(*[imgs[b].ctypes.data for b in range(B)])
    pkg._check(pkg.lib().b2s_extract_batch(ex._h, ctypes.cast(ptrs, _vp), B, imgs.shape[2], imgs.shape[1], imgs.shape[2],
                                           _p(kps), _p(desc), ex.cap, _p(n)))
    return kps, desc, n


def dense_images(seed0, count):
    """`count` ordinary images (left and right images of 8 synth_stereo pairs, repeated)."""
    pairs = [synth_stereo(W, H, seed0 + j) for j in range(8)]
    return [pairs[i % 8][i // 8 % 2] for i in range(count)]


def blank_image(value=128):
    return np.full((H, W), value, np.uint8)


def low_texture_pair(seed, n_blobs=6, disparity=23):
    """A flat grey pair with a few bright squares (a handful of FAST corners), shifted by one disparity in the right."""
    rng = np.random.RandomState(seed)
    left, right = blank_image(90), blank_image(90)
    for _ in range(n_blobs):
        x, y = int(rng.randint(80, W - 80)), int(rng.randint(40, H - 40))
        s, v = int(rng.randint(6, 14)), int(rng.randint(170, 250))
        left[y:y + s, x:x + s] = v
        right[y:y + s, x - disparity:x - disparity + s] = v
    return left, right


# ================================================================================================ 1. SearchByBoW
def bow_members(B, capA, capB, n_nodes, seed, shift):
    """B members of SearchByBoW inputs: every slot of [B, cap] holds a real record of the member; the counts cut them."""
    n = max(capA, capB)
    d = {k: [] for k in ("descA", "nodeA", "validA", "angA", "descB", "nodeB", "validB", "angB")}
    for b in range(B):
        A, nA, vA, aA, Bd, nB, aB = synth_descriptors(n, seed=seed + b, n_nodes=n_nodes)
        vB = (np.random.RandomState(seed + b + 7).randint(0, 100, size=n) < 93).astype(np.uint8)
        for k, v, c in (("descA", A, capA), ("nodeA", nA, capA), ("validA", vA, capA), ("angA", aA, capA),
                        ("descB", Bd, capB), ("nodeB", nB, capB), ("validB", vB, capB), ("angB", aB, capB)):
            d[k].append(v[:c])
    d = {k: np.ascontiguousarray(np.stack(v)) for k, v in d.items()}
    d["nA"] = ragged_counts(B, capA, shift)
    d["nB"] = ragged_counts(B, capB, shift + 4)
    return d


def bow_batch(pkg, m, d, nA, nB, cfg, zero=False):
    """b2s_search_by_bow_batch, as stream.step_host calls it."""
    g = (lambda k, n: zero_padded(d[k], n)) if zero else (lambda k, n: d[k])
    B, capA = d["nodeA"].shape
    capB = d["nodeB"].shape[1]
    keep = [g("descA", nA), g("nodeA", nA), g("validA", nA) if cfg["validA"] else None, g("angA", nA),
            g("descB", nB), g("nodeB", nB), g("validB", nB) if cfg["validB"] else None, g("angB", nB)]
    nA, nB = np.ascontiguousarray(nA, np.int32), np.ascontiguousarray(nB, np.int32)
    match = np.full((B, capB), 7, np.int32)  # the call writes every slot
    nm = np.full(B, -5, np.int32)
    pkg._check(pkg.lib().b2s_search_by_bow_batch(m._h, B, _p(keep[0]), _p(keep[1]), _p(keep[2]), _p(keep[3]), _p(nA), capA,
                                                 _p(keep[4]), _p(keep[5]), _p(keep[6]), _p(keep[7]), _p(nB), capB,
                                                 cfg["th_low"], float(np.float32(cfg["nnratio"])), int(cfg["strict_lt"]),
                                                 int(cfg["check_ori"]), _p(match), _p(nm)))
    return nm, match


def bow_device(pkg, m, d, nA_dev, nB_dev, cfg, stream):
    """b2s_search_by_bow_device on device copies of the inputs, counts read from device memory, on `stream`."""
    import torch
    t = {k: torch.from_numpy(d[k]).cuda() for k in ("descA", "nodeA", "validA", "angA", "descB", "nodeB", "validB", "angB")}
    B, capA = d["nodeA"].shape
    capB = d["nodeB"].shape[1]
    nA, nB = torch.from_numpy(np.asarray(nA_dev, np.int32)).cuda(), torch.from_numpy(np.asarray(nB_dev, np.int32)).cuda()
    match = torch.full((B, capB), 7, dtype=torch.int32, device="cuda")
    nm = torch.full((B,), -5, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    pkg._check(pkg.lib().b2s_search_by_bow_device(
        m._h, B, _vp(t["descA"].data_ptr()), _vp(t["nodeA"].data_ptr()),
        _vp(t["validA"].data_ptr()) if cfg["validA"] else None, _vp(t["angA"].data_ptr()), _vp(nA.data_ptr()), capA,
        _vp(t["descB"].data_ptr()), _vp(t["nodeB"].data_ptr()), _vp(t["validB"].data_ptr()) if cfg["validB"] else None,
        _vp(t["angB"].data_ptr()), _vp(nB.data_ptr()), capB, cfg["th_low"], float(np.float32(cfg["nnratio"])),
        int(cfg["strict_lt"]), int(cfg["check_ori"]), _vp(match.data_ptr()), _vp(nm.data_ptr()), _vp(stream.cuda_stream)))
    stream.synchronize()
    return nm.cpu().numpy(), match.cpu().numpy()


def check_bow_members(pkg, oracle, d, nA, nB, cfg, nm, match, with_oracle=True):
    """Every member: slots past nB stay -1, the single-pair call is bit-identical, the oracle agrees on the slice."""
    capB = d["nodeB"].shape[1]
    single = pkg.ORBmatcher(cfg["nnratio"], cfg["check_ori"], max_features=max(d["nodeA"].shape[1], capB))
    for b in range(len(nA)):
        a, n = int(nA[b]), int(nB[b])
        assert (match[b, n:] == -1).all(), b
        s = lambda k, c: np.ascontiguousarray(d[k][b, :c])
        vA = s("validA", a) if cfg["validA"] else None
        vB = s("validB", n) if cfg["validB"] else None
        n1, m1 = single.SearchByBoW(s("descA", a), s("nodeA", a), vA, s("angA", a), s("descB", n), s("nodeB", n),
                                    s("angB", n), validB=vB, strict_lt=cfg["strict_lt"], th_low=cfg["th_low"])
        assert n1 == nm[b] and np.array_equal(m1, match[b, :n]), (b, a, n)
        if with_oracle:
            on, om = oracle.search_by_bow(s("descA", a), s("nodeA", a), vA if vA is not None else np.ones(a, np.uint8),
                                          s("angA", a), s("descB", n), s("nodeB", n), s("angB", n), validB=vB,
                                          th_low=cfg["th_low"], nnratio=cfg["nnratio"], strict_lt=cfg["strict_lt"],
                                          check_ori=cfg["check_ori"])
            assert on == nm[b] and np.array_equal(om, match[b, :n]), (b, a, n)


def _cfg(validA=True, validB=True, strict_lt=False, check_ori=True, nnratio=0.7, th_low=50):
    return dict(validA=validA, validB=validB, strict_lt=strict_lt, check_ori=check_ori, nnratio=nnratio, th_low=th_low)


# (capA, capB, vocabulary nodes, batch, shift of the ragged counts, options): every value of every option appears, capA < capB
# and capA > capB both appear, and over the configurations every RAGGED count lands on both sides
BOW_CASES = [
    (1100, 1300, 1, 5, 0, _cfg()),
    (1300, 1100, 7, 5, 5, _cfg(validA=False, strict_lt=True, check_ori=False, nnratio=0.6, th_low=100)),
    (1100, 1300, 100, 5, 2, _cfg(validB=False, nnratio=0.9, th_low=100)),
    (1300, 1100, 1, 5, 7, _cfg(validA=False, validB=False, strict_lt=True, nnratio=0.9)),
    (1300, 1100, 100, 5, 1, _cfg(check_ori=False, nnratio=0.6)),
    (1100, 1300, 7, 5, 6, _cfg(validB=False, strict_lt=True, th_low=100)),
    (1300, 1100, 7, 1, 9, _cfg()),
    (1100, 1300, 100, 1, 8, _cfg(validA=False, nnratio=0.6)),
]


@pytest.mark.parametrize("case", range(len(BOW_CASES)))
def test_search_by_bow_batch_ragged(pkg, oracle, case):
    capA, capB, nodes, B, shift, cfg = BOW_CASES[case]
    d = bow_members(B, capA, capB, nodes, seed=300 + 17 * case, shift=shift)
    nA, nB = d["nA"], d["nB"]
    m = pkg.ORBmatcher(cfg["nnratio"], cfg["check_ori"], max_features=max(capA, capB), max_batch=B)
    nm, match = bow_batch(pkg, m, d, nA, nB, cfg)
    check_bow_members(pkg, oracle, d, nA, nB, cfg, nm, match)
    assert nm.sum() > 0
    nz, mz = bow_batch(pkg, m, d, nA, nB, cfg, zero=True)  # stale padding == zero padding
    assert np.array_equal(nz, nm) and np.array_equal(mz, match)


def test_search_by_bow_device_stream_and_clamped_counts(pkg):
    """Device entry on an explicit stream == host-buffer batch; device counts above the capacity act as the capacity."""
    import torch
    capA, capB, cfg = 1100, 1300, _cfg(nnratio=0.9, th_low=100)
    d = bow_members(5, capA, capB, 7, seed=911, shift=0)
    nA = np.array([capA, 33, 0, capA, 1000], np.int32)
    nB = np.array([129, capB, capB, 1, capB], np.int32)
    nA_dev = np.array([capA + 1, 33, 0, 1 << 30, 1000], np.int32)
    nB_dev = np.array([129, capB + 64, 65535, 1, (1 << 31) - 1], np.int32)
    m = pkg.ORBmatcher(cfg["nnratio"], cfg["check_ori"], max_features=max(capA, capB), max_batch=5)
    nm, match = bow_batch(pkg, m, d, nA, nB, cfg)
    check_bow_members(pkg, None, d, nA, nB, cfg, nm, match, with_oracle=False)
    st = torch.cuda.Stream()
    nm_d, match_d = bow_device(pkg, m, d, nA_dev, nB_dev, cfg, st)
    assert np.array_equal(nm_d, nm) and np.array_equal(match_d, match)
    nm_d, match_d = bow_device(pkg, m, d, nA, nB, cfg, st)
    assert np.array_equal(nm_d, nm) and np.array_equal(match_d, match)


@pytest.fixture(scope="module")
def bench_records(pkg):
    """Device extraction of 160 synth_stereo pairs at the benchmark's size: left records [160, cap] (A side), right records
    (B side), their counts; one vocabulary node, as the stream's temporal matcher."""
    F = 160
    pairs = [synth_stereo(W, H, 700 + i) for i in range(F)]
    ex = pkg.ORBextractor(NFEAT, 1.2, 8, 20, 7, max_width=W, max_height=H, max_batch=2 * F)
    kps, desc, n = extract_full(pkg, ex, [p[0] for p in pairs] + [p[1] for p in pairs])
    ex.close()
    cap = kps.shape[1]
    d = dict(descA=desc[:F], nodeA=np.zeros((F, cap), np.int32), validA=np.ones((F, cap), np.uint8),
             angA=np.ascontiguousarray(kps["angle"][:F]), descB=desc[F:], nodeB=np.zeros((F, cap), np.int32),
             validB=np.ones((F, cap), np.uint8), angB=np.ascontiguousarray(kps["angle"][F:]))
    d = {k: np.ascontiguousarray(v) for k, v in d.items()}
    return d, n[:F].copy(), n[F:].copy()


BENCH_CFG = _cfg(validB=False)  # stream.py: validA present, validB absent, TH_LOW, ratio 0.7, orientation check


def _narrow(d, capB):
    e = dict(d)
    for k in ("descB", "nodeB", "validB", "angB"):
        e[k] = np.ascontiguousarray(d[k][:, :capB])
    return e


def test_search_by_bow_bench_batch(pkg, oracle, bench_records):
    """160 pairs of 2000 x 2000 features in one node: the bench's shape with its own counts, then ragged counts whose
    padding is the rest of each member's extracted records."""
    d, nA_full, nB_full = bench_records
    F, cap = d["nodeA"].shape
    assert nA_full.min() > 1500 and nB_full.min() > 1500
    m = pkg.ORBmatcher(0.7, True, max_features=cap, max_batch=F)
    nm, match = bow_batch(pkg, m, d, nA_full, nB_full, BENCH_CFG)
    check_bow_members(pkg, oracle, d, nA_full, nB_full, BENCH_CFG, nm, match)
    assert (nm > 0).all() and nm.mean() > 100
    nA, nB = ragged_counts(F, cap, 0, nA_full), ragged_counts(F, cap, 3, nB_full)
    nm_r, match_r = bow_batch(pkg, m, d, nA, nB, BENCH_CFG)
    check_bow_members(pkg, oracle, d, nA, nB, BENCH_CFG, nm_r, match_r)
    nz, mz = bow_batch(pkg, m, d, nA, nB, BENCH_CFG, zero=True)
    assert np.array_equal(nz, nm_r) and np.array_equal(mz, match_r)


def test_search_by_bow_handle_reuse(pkg, bench_records):
    """One handle for batches 160 -> 3 -> 160 with different capacities == fresh handles."""
    d, nA_full, nB_full = bench_records
    F, cap = d["nodeA"].shape
    capB2 = 1500
    d2 = _narrow(d, capB2)
    nA2, nB2 = ragged_counts(F, cap, 6, nA_full), ragged_counts(F, capB2, 2, nB_full)
    small = bow_members(3, 1300, 1100, 7, seed=77, shift=3)
    cfg_small = _cfg(nnratio=0.9, th_low=100)
    runs = [(d, nA_full, nB_full, BENCH_CFG), (small, small["nA"], small["nB"], cfg_small), (d2, nA2, nB2, BENCH_CFG),
            (small, small["nA"], small["nB"], cfg_small)]
    fresh = []
    for dd, a, b, cfg in runs:
        fm = pkg.ORBmatcher(cfg["nnratio"], cfg["check_ori"], max_features=cap, max_batch=len(a))
        fresh.append(bow_batch(pkg, fm, dd, a, b, cfg))
        fm.close()
    m = pkg.ORBmatcher(0.7, True, max_features=cap, max_batch=F)
    for (dd, a, b, cfg), (nm0, match0) in zip(runs, fresh):
        nm, match = bow_batch(pkg, m, dd, a, b, cfg)
        assert np.array_equal(nm, nm0) and np.array_equal(match, match0)


# ================================================================================================ 2. stereo
STEREO_F = 160
STEREO_MB = (0.0, BF / 30.0)


@pytest.fixture(scope="module")
def stereo_batch(pkg):
    """Pairs: 0 blank left, 1 blank right, 2-4 low texture, the rest ordinary.  One extractor handle (max_batch = 2F)
    first extracts a dense batch, then this one, so the records past each count are stale."""
    F = STEREO_F
    pairs = [(blank_image(), synth_stereo(W, H, 900)[1]), (synth_stereo(W, H, 901)[0], blank_image(60))]
    pairs += [low_texture_pair(902 + i, n_blobs=3 + 2 * i) for i in range(3)]
    pairs += [synth_stereo(W, H, 905 + i) for i in range(F - len(pairs))]
    dense = dense_images(1200, 2 * F)
    ex = pkg.ORBextractor(NFEAT, 1.2, 8, 20, 7, max_width=W, max_height=H, max_batch=2 * F)
    _, _, n_dense = extract_full(pkg, ex, dense)
    assert n_dense.min() > 1500
    left, right = [p[0] for p in pairs], [p[1] for p in pairs]
    return ex, left, right


def test_stereo_match_batch_stale_records(pkg, oracle, stereo_batch):
    ex, left, right = stereo_batch
    F = len(left)
    extract_full(pkg, ex, dense_images(1300, 2 * F))
    kps, desc, n = extract_full(pkg, ex, left + right)  # stale dense records past every count on the device
    assert n[0] == 0 and n[F + 1] == 0 and 0 < n[2] < 200 and 0 < n[F + 2] < 200 and n[5:F].min() > 1500
    cap = ex.cap
    for mb in STEREO_MB:
        ur, dp, nm = ex.stereo_match(0, F, F, BF, mb)
        assert nm[0] == 0 and nm[1] == 0 and (nm[5:] > 0).all() and nm[5:].mean() > 100
        for i in range(F):
            u1, d1, n1 = ex.stereo_match(i, F + i, 1, BF, mb)
            assert n1[0] == nm[i] and np.array_equal(u1[0], ur[i]) and np.array_equal(d1[0], dp[i]), (mb, i)
            assert (ur[i, n[i]:] == -1).all() and (dp[i, n[i]:] == -1).all()
        for i in (0, 1, 2, 4, F - 1):  # the oracle is pinned to the reference in test_stereo_gpu / test_oracle_reference_frame
            oL, oR = oracle.extractor(NFEAT, 1.2, 8, 20, 7), oracle.extractor(NFEAT, 1.2, 8, 20, 7)
            okL, odL = oL(left[i])
            okR, odR = oR(right[i])
            assert len(okL) == n[i] and len(okR) == n[F + i]
            on, our, odp = oracle.compute_stereo_matches(oL, oR, okL, odL, okR, odR, BF, mb)
            assert on == nm[i] and np.array_equal(our, ur[i, :n[i]]) and np.array_equal(odp, dp[i, :n[i]]), (mb, i)
        # right images first in the batch
        extract_full(pkg, ex, right + left)
        ur2, dp2, nm2 = ex.stereo_match(F, 0, F, BF, mb)
        assert np.array_equal(nm2, nm) and np.array_equal(ur2, ur) and np.array_equal(dp2, dp)
        extract_full(pkg, ex, left + right)


def test_stereo_match_device_stale_records(pkg, stereo_batch):
    """b2s_extract_batch_device + b2s_stereo_match_device into record buffers that hold a dense batch's records, on an
    explicit stream == the host-buffer path."""
    import torch
    ex, left, right = stereo_batch
    F, cap = len(left), ex.cap
    dense = np.stack(dense_images(1400, 2 * F))
    imgs = np.stack(left + right)
    st = torch.cuda.Stream()
    d_kps = torch.zeros((2 * F, cap, pkg.keypoint_dtype.itemsize), dtype=torch.uint8, device="cuda")
    d_desc = torch.zeros((2 * F, cap, 32), dtype=torch.uint8, device="cuda")
    d_n = torch.zeros(2 * F, dtype=torch.int32, device="cuda")
    d_ur = torch.full((F, cap), 5.0, dtype=torch.float32, device="cuda")
    d_dp = torch.full((F, cap), 5.0, dtype=torch.float32, device="cuda")
    d_nm = torch.full((F,), -3, dtype=torch.int32, device="cuda")
    for batch in (dense, imgs):
        d_img = torch.from_numpy(batch).cuda()
        torch.cuda.synchronize()
        ex.extract_batch_device(d_img.data_ptr(), W * H, 2 * F, W, H, W, d_kps.data_ptr(), d_desc.data_ptr(), d_n.data_ptr(),
                                cap, stream=st.cuda_stream)
        st.synchronize()
    ex.check()
    kps, desc, n = extract_full(pkg, ex, left + right)
    assert np.array_equal(d_n.cpu().numpy(), n)
    for mb in STEREO_MB:
        ex.stereo_match_device(0, F, F, d_kps.data_ptr(), d_desc.data_ptr(), d_n.data_ptr(), cap, BF, mb, d_ur.data_ptr(),
                               d_dp.data_ptr(), d_nm.data_ptr(), stream=st.cuda_stream)
        st.synchronize()
        ur, dp, nm = ex.stereo_match(0, F, F, BF, mb)
        assert np.array_equal(d_nm.cpu().numpy(), nm)
        assert np.array_equal(d_ur.cpu().numpy(), ur) and np.array_equal(d_dp.cpu().numpy(), dp)


# ================================================================================================ 3. SearchByProjection
PROJ_TH = 7.0


def _geom():
    return dict(mnMinX=0.0, mnMinY=0.0, mnMaxX=float(W), mnMaxY=float(H), bf=BF,
                scale_factors=np.array([np.float32(1.2) ** i for i in range(8)], np.float32))


def proj_members(pkg, B, capQ, capF, seed, shift):
    """B SearchByProjection(Cur, Last) members from synth_projection; every slot holds a real query / feature."""
    q = np.zeros((B, capQ), pkg.proj_query_dtype)
    kps = np.zeros((B, capF), pkg.keypoint_dtype)
    ur = np.zeros((B, capF), np.float32)
    desc = np.zeros((B, capF, 32), np.uint8)
    for b in range(B):
        s = synth_projection(nf=capF, nq=capQ, seed=seed + b)
        for f in pkg.proj_query_dtype.names:
            q[b][f] = s["q"][f]
        kps[b]["x"], kps[b]["y"], kps[b]["octave"], kps[b]["angle"] = s["kpx"], s["kpy"], s["octave"], s["angle"]
        kps[b]["size"], kps[b]["response"] = 31.0, 1.0
        ur[b], desc[b] = s["uright"], s["desc"]
    return dict(q=q, kps=kps, ur=ur, desc=desc, nq=ragged_counts(B, capQ, shift), nf=ragged_counts(B, capF, shift + 5))


def tcl_for(mode, b=0):
    """Relative pose Tcl (3 x 4) whose motion takes the reference's branch `mode` (0 / 1 forward / 2 backward)."""
    a = 0.004 * (b + 1)
    t = {0: (0.05, 0.0, -0.1), 1: (0.02, 0.0, -0.8), 2: (0.0, 0.01, 0.9)}[mode]
    return np.array([[np.cos(a), 0, np.sin(a), t[0]], [0, 1, 0, t[1]], [-np.sin(a), 0, np.cos(a), t[2]]], np.float32)


def proj_chain(pkg, B, cap, seed, mode, counts):
    """Frames 0..B of a sequence (records, descriptors, stereo depth; uright of frames 1..B): frame b + 1 sees the live
    stereo points of frame b moved by Tcl[b] (jittered, a few descriptor bits flipped) plus new features, shuffled."""
    stream_mod = importlib.import_module("self_commit_orb-slam2_b200.stream")
    rng = np.random.RandomState(seed)
    f32 = np.float32
    kps = np.zeros((B + 1, cap), pkg.keypoint_dtype)
    desc = np.zeros((B + 1, cap, 32), np.uint8)
    depth = np.zeros((B + 1, cap), np.float32)
    Tcl = np.stack([tcl_for(mode, b).reshape(12) for b in range(B)]).astype(np.float32)

    def fresh(k):
        return dict(x=rng.uniform(10, W - 10, k).astype(f32), y=rng.uniform(10, H - 10, k).astype(f32),
                    octave=rng.randint(0, 8, k).astype(np.int32), angle=rng.uniform(0, 360, k).astype(f32),
                    desc=rng.randint(0, 256, (k, 32)).astype(np.uint8), depth=rng.uniform(4, 40, k).astype(f32))

    def put(b, fr):
        for k in ("x", "y", "octave", "angle"):
            kps[b][k] = fr[k]
        kps[b]["size"], kps[b]["response"] = 31.0, 1.0
        desc[b], depth[b] = fr["desc"], fr["depth"]
        depth[b][rng.uniform(size=cap) < 0.15] = -1.0  # monocular features

    put(0, fresh(cap))
    for b in range(B):
        q = stream_mod.StereoStream.track_queries_host(kps[b:b + 1], desc[b:b + 1], depth[b:b + 1], counts[b:b + 1],
                                                       Tcl[b:b + 1], FX, FY, CX, CY)[0]
        seen = np.nonzero((q["invz"] > 0) & (q["u"] > 8) & (q["u"] < W - 8) & (q["v"] > 8) & (q["v"] < H - 8))[0][:cap]
        fr = fresh(cap)
        k = len(seen)
        fr["x"][:k] = q["u"][seen] + rng.uniform(-1.5, 1.5, k).astype(f32)
        fr["y"][:k] = q["v"][seen] + rng.uniform(-1.5, 1.5, k).astype(f32)
        fr["octave"][:k] = q["octave"][seen]
        fr["angle"][:k] = np.mod(q["angle"][seen] + rng.uniform(-5, 5, k), 360).astype(f32)
        fr["depth"][:k] = (f32(1) / q["invz"][seen]).astype(f32)
        dd = q["desc"][seen].copy()
        for i in range(k):
            for bit in rng.choice(256, size=int(rng.randint(0, 20)), replace=False):
                dd[i, bit >> 3] ^= np.uint8(1 << (bit & 7))
        fr["desc"][:k] = dd
        perm = rng.permutation(cap)
        put(b + 1, {kk: v[perm] for kk, v in fr.items()})
    uright = np.where(depth[1:] > 0, kps["x"][1:] - f32(BF) / np.where(depth[1:] > 0, depth[1:], f32(1)), f32(-1))
    return dict(kps=kps, desc=desc, depth=depth, uright=np.ascontiguousarray(uright, np.float32), n=counts, Tcl=Tcl)


def check_proj_member(pkg, oracle, m1, q, kps, ur, desc, nq, nf, mode, nm, match):
    """One member: slots past nf stay -1; the single-pair call and the oracle give the same matches."""
    assert (match[nf:] == -1).all()
    k = kps[:nf]
    args = (np.ascontiguousarray(q[:nq]), k["x"].copy(), k["y"].copy(), k["octave"].copy(), k["angle"].copy(),
            np.ascontiguousarray(ur[:nf]), None, np.ascontiguousarray(desc[:nf]), _geom(), PROJ_TH)
    n1, m_1 = m1.SearchByProjection(*args, mode=mode)
    assert n1 == nm and np.array_equal(m_1, match[:nf])
    if oracle is not None:
        no, mo = oracle.search_by_projection_last(*args, mode=mode)
        assert no == nm and np.array_equal(mo, match[:nf])


def proj_batch(m, d, zero=False):
    g = (lambda k, n: zero_padded(d[k], n)) if zero else (lambda k, n: d[k])
    return m.SearchByProjectionBatch(g("q", d["nq"]), d["nq"], g("kps", d["nf"]), g("ur", d["nf"]), g("desc", d["nf"]),
                                     d["nf"], _geom(), PROJ_TH, mode=d["mode"])


def proj_sequence(m, c, zero=False):
    n = c["n"]
    g = (lambda k, cnt: zero_padded(c[k], cnt)) if zero else (lambda k, cnt: c[k])
    return m.SearchByProjectionSequence(g("kps", n), g("desc", n), g("depth", n), g("uright", n[1:]), n, c["Tcl"], FX, FY, CX,
                                        CY, _geom(), PROJ_TH, mode=c["mode"])


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("capQ,capF", [(1100, 1400), (1400, 1100)])
def test_search_by_projection_batch_ragged(pkg, oracle, mode, capQ, capF):
    import torch
    B = 10
    d = proj_members(pkg, B, capQ, capF, seed=500 + 31 * mode + capQ, shift=mode)
    d["mode"] = mode
    m = pkg.ORBmatcher(0.9, True, max_features=max(capQ, capF), max_batch=B)
    nm, match = proj_batch(m, d)
    m1 = pkg.ORBmatcher(0.9, True, max_features=max(capQ, capF))
    for b in range(B):
        check_proj_member(pkg, oracle, m1, d["q"][b], d["kps"][b], d["ur"][b], d["desc"][b], d["nq"][b], d["nf"][b], mode,
                          nm[b], match[b])
    assert nm.sum() > 20
    nz, mz = proj_batch(m, d, zero=True)
    assert np.array_equal(nz, nm) and np.array_equal(mz, match)
    # device entry, counts and records in device memory, explicit stream
    st = torch.cuda.Stream()
    t = {k: torch.from_numpy(np.ascontiguousarray(d[k]).view(np.uint8) if k in ("q", "kps") else d[k]).cuda()
         for k in ("q", "kps", "ur", "desc", "nq", "nf")}
    d_match = torch.full((B, capF), 9, dtype=torch.int32, device="cuda")
    d_nm = torch.full((B,), -4, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    m.search_by_projection_last_device(B, t["q"].data_ptr(), t["nq"].data_ptr(), capQ, t["kps"].data_ptr(), t["ur"].data_ptr(),
                                       t["desc"].data_ptr(), t["nf"].data_ptr(), capF, _geom(), PROJ_TH, mode,
                                       d_match.data_ptr(), d_nm.data_ptr(), stream=st.cuda_stream)
    st.synchronize()
    assert np.array_equal(d_nm.cpu().numpy(), nm) and np.array_equal(d_match.cpu().numpy(), match)


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_search_by_projection_sequence_ragged(pkg, oracle, mode):
    import torch
    stream_mod = importlib.import_module("self_commit_orb-slam2_b200.stream")
    B, cap = 10, 1300
    n = ragged_counts(B + 1, cap, 8 + mode)
    c = proj_chain(pkg, B, cap, seed=610 + mode, mode=mode, counts=n)
    c["mode"] = mode
    m = pkg.ORBmatcher(0.9, True, max_features=cap, max_batch=B)
    nm, match = proj_sequence(m, c)
    q = stream_mod.StereoStream.track_queries_host(c["kps"][:B], c["desc"][:B], c["depth"][:B], n[:B], c["Tcl"], FX, FY, CX,
                                                   CY)
    m1 = pkg.ORBmatcher(0.9, True, max_features=cap)
    for b in range(B):
        check_proj_member(pkg, oracle, m1, q[b], c["kps"][b + 1], c["uright"][b], c["desc"][b + 1], n[b], n[b + 1], mode,
                          nm[b], match[b])
    assert nm.sum() > 200
    nz, mz = proj_sequence(m, c, zero=True)
    assert np.array_equal(nz, nm) and np.array_equal(mz, match)
    # the device projection on its own: queries bit-identical to the numpy restatement, counts = the last frames' counts
    st = torch.cuda.Stream()
    kd = torch.from_numpy(np.ascontiguousarray(c["kps"][:B]).view(np.uint8)).cuda()
    dd = torch.from_numpy(np.ascontiguousarray(c["desc"][:B])).cuda()
    zd = torch.from_numpy(np.ascontiguousarray(c["depth"][:B])).cuda()
    nd = torch.from_numpy(np.ascontiguousarray(n[:B])).cuda()
    Td = torch.from_numpy(c["Tcl"]).cuda()
    qd = torch.zeros((B, cap, pkg.proj_query_dtype.itemsize), dtype=torch.uint8, device="cuda")
    nqd = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    m.track_queries_device(B, kd.data_ptr(), dd.data_ptr(), zd.data_ptr(), nd.data_ptr(), cap, Td.data_ptr(), FX, FY, CX, CY, 1,
                           qd.data_ptr(), nqd.data_ptr(), stream=st.cuda_stream)
    st.synchronize()
    q_dev = qd.cpu().numpy().view(pkg.proj_query_dtype).reshape(B, cap)
    assert np.array_equal(nqd.cpu().numpy(), n[:B])
    for b in range(B):
        assert q_dev[b, :n[b]].tobytes() == q[b, :n[b]].tobytes()


def test_search_by_projection_sequence_and_batch_share_one_handle(pkg):
    """SearchByProjectionSequence and SearchByProjectionBatch share the record staging of a handle; called alternately
    with growing sizes they give what fresh handles give."""
    runs = []
    for i, (kind, B, c1, c2) in enumerate([("seq", 2, 600, 0), ("batch", 3, 700, 900), ("seq", 5, 1200, 0),
                                           ("batch", 8, 1500, 1800), ("seq", 8, 2000, 0), ("batch", 3, 700, 900),
                                           ("seq", 2, 600, 0)]):
        mode = i % 3
        if kind == "seq":
            c = proj_chain(pkg, B, c1, seed=700 + i, mode=mode, counts=ragged_counts(B + 1, c1, i))
            c["mode"] = mode
            runs.append((proj_sequence, c))
        else:
            d = proj_members(pkg, B, c1, c2, seed=720 + 13 * i, shift=i)
            d["mode"] = mode
            runs.append((proj_batch, d))
    fresh = [fn(pkg.ORBmatcher(0.9, True, max_features=2048, max_batch=8), d) for fn, d in runs]
    m = pkg.ORBmatcher(0.9, True, max_features=2048, max_batch=8)
    for (fn, d), (nm0, match0) in zip(runs, fresh):
        nm, match = fn(m, d)
        assert np.array_equal(nm, nm0) and np.array_equal(match, match0)
    assert sum(int(r[0].sum()) for r in fresh) > 0


# ================================================================================================ 4. PoseOptimization
RTOL = 1e-5


def _check(out, ref, d):
    """The bar of test_poseopt_gpu: same flags and inliers, pose within 1e-5 relative, the first 8 LM trials identical."""
    assert out["n_inliers"] == ref["n_inliers"]
    assert np.array_equal(out["outlier"], ref["outlier"])
    g, r, i0 = (np.asarray(a, np.float64) for a in (out["Tcw"], ref["Tcw"], d["Tcw"]))
    scale = max(np.abs(r - i0).max(), 1e-12)
    ulp = np.spacing(np.abs(r).astype(np.float32)).astype(np.float64)
    assert (np.abs(g - r) <= RTOL * scale + ulp).all(), float((np.abs(g - r) / scale).max())
    tg = out["trace"][:out["n_trials"]].tolist()
    tr = ref["trace"][:ref["n_trials"]].tolist()
    k = min(len(tg), len(tr), 8)
    assert tg[:k] == tr[:k]


def bench_pose_problems(n, seed0=0):
    """The benchmark's PoseOptimization problems: 2000 features per frame, 50-70 % with a map point, 5-20 % gross outliers."""
    out = []
    for i in range(n):
        rng = np.random.RandomState(11000 + seed0 + i)
        out.append(synth_pose_problem(n=2000, seed=13000 + seed0 + i, mp_frac=float(rng.uniform(0.5, 0.7)), mono_frac=0.2,
                                      outlier_frac=float(rng.uniform(0.05, 0.2)), pert_t=float(rng.uniform(0.02, 0.15)),
                                      pert_deg=float(rng.uniform(0.2, 1.5))))
    return out


def pose_with_edges(k, seed):
    """A problem with exactly k correspondences (features with a map point)."""
    n = max(2 * k, 40)
    d = synth_pose_problem(n=n, seed=seed, mp_frac=1.0)
    has = np.zeros(n, np.uint8)
    has[np.random.RandomState(seed).choice(n, k, replace=False)] = 1
    d["has_mp"] = has
    return d


def with_camera(d, s, dx, dy):
    """The same problem seen by a camera with intrinsics scaled by s and the principal point moved by (dx, dy): pixel
    observations follow, inv_sigma2 is scaled so that every chi2 stays what it was."""
    f = np.float32
    e = dict(d)
    e["fx"], e["fy"] = f(float(d["fx"]) * s), f(float(d["fy"]) * s)
    e["cx"], e["cy"], e["bf"] = f(float(d["cx"]) * s + dx), f(float(d["cy"]) * s + dy), f(float(d["bf"]) * s)
    e["kpx"] = (d["kpx"].astype(np.float64) * s + dx).astype(f)
    e["kpy"] = (d["kpy"].astype(np.float64) * s + dy).astype(f)
    ur = d["uright"].astype(np.float64)
    e["uright"] = np.where(ur < 0, ur, ur * s + dx).astype(f)
    e["inv_sigma2"] = (d["inv_sigma2"].astype(np.float64) / (s * s)).astype(f)
    return e


EDGE_COUNTS = (0, 2, 3, 9, 10, 11, 255, 256, 257, 5000)  # the < 3 and < 10 rules, the PO_T = 256 stride, a large frame


@pytest.fixture(scope="module")
def pose_batch():
    ds = bench_pose_problems(160) + [pose_with_edges(k, 4000 + k) for k in EDGE_COUNTS]
    rng = np.random.RandomState(99)
    ds = [with_camera(d, float(rng.uniform(0.8, 1.25)), float(rng.uniform(-20, 20)), float(rng.uniform(-10, 10)))
          for d in ds]
    return [ds[i] for i in rng.permutation(len(ds))]


def _same_pose(a, b):
    assert a["n_inliers"] == b["n_inliers"] and a["n_trials"] == b["n_trials"]
    assert np.array_equal(a["Tcw"], b["Tcw"]) and np.array_equal(a["outlier"], b["outlier"])
    assert np.array_equal(a["trace"], b["trace"])


def test_pose_optimization_bench_batch(pkg, oracle, pose_batch):
    ds = pose_batch
    assert len({float(d["fx"]) for d in ds}) == len(ds)  # every member has its own camera
    opt = pkg.Optimizer(max_kf=4, max_mp=16, max_edges=64, max_batch=len(ds))
    outs = opt.PoseOptimizationBatch(ds)
    for d, out in zip(ds, outs):
        _check(out, oracle.pose_optimization(d), d)
    one = pkg.Optimizer(max_kf=4, max_mp=16, max_edges=64)
    for d, out in zip(ds, outs):
        _same_pose(one.PoseOptimization(d), out)
    # the stream's path: prepared problem arrays, no trace
    prep = opt.prepare_pose_batch(ds)
    ress = opt.run_prepared_pose(prep)
    for i, out in enumerate(outs):
        Tcw, outl = prep["keep"][i][1]
        n = len(ds[i]["has_mp"])
        assert ress[i].n_inliers == out["n_inliers"] and ress[i].n_trials == out["n_trials"]
        assert np.array_equal(Tcw, out["Tcw"]) and np.array_equal(outl[:n], out["outlier"])


def test_pose_optimization_handle_reuse(pkg, pose_batch):
    """One handle for batches of 1 -> 160 -> 7 -> 300 frames (its scratch regrows in frames and in edges) == fresh
    handles."""
    ds = pose_batch
    sizes = (1, 160, 7, 300)
    batches, k = [], 0
    for s in sizes:
        batches.append([ds[(k + i) % len(ds)] for i in range(s)])
        k += 37
    opt = pkg.Optimizer(max_kf=4, max_mp=16, max_edges=64)
    for b in batches:
        got = opt.PoseOptimizationBatch(b)
        ref = pkg.Optimizer(max_kf=4, max_mp=16, max_edges=64).PoseOptimizationBatch(b)
        for x, y in zip(got, ref):
            _same_pose(x, y)
    big = [d for d in ds if len(d["has_mp"]) >= 10000]
    small = [d for d in ds if int(d["has_mp"].sum()) < 3]
    got = opt.PoseOptimizationBatch(small + big)  # after the 300-frame batch: few frames, the largest edge list
    for x, d in zip(got, small + big):
        _same_pose(x, pkg.Optimizer(max_kf=4, max_mp=16, max_edges=64).PoseOptimization(d))


# ================================================================================================ 5. the stream across steps
def test_stream_lanes_across_steps(pkg, oracle):
    """Two StereoStream lanes take the steps in turn, frames fed by load_window from a resident set of D < 2F frames (the
    window wraps); some frames are blank or low-texture, so the ring holds stale records past the counts.  After each step
    every frame's outputs equal the single-pair entry points on that step's own records; after finish() the solvers'
    latest outputs equal direct calls on the same problems."""
    import torch
    stream_mod = importlib.import_module("self_commit_orb-slam2_b200.stream")
    F, D = 6, 9
    frames = [synth_stereo(W, H, 60 + i) for i in range(6)]
    frames += [(blank_image(), synth_stereo(W, H, 66)[1]), low_texture_pair(67), (synth_stereo(W, H, 68)[0], blank_image(40))]
    d_all = torch.from_numpy(np.stack([np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames])])).cuda()
    windows = [synth_local_ba(n_kf=8, n_fixed=2, n_mp=200, obs_per_mp=4, seed=5 + k) for k in range(3)]
    poses = [synth_pose_problem(n=300 + 40 * k, seed=60 + k) for k in range(8)]
    kw = dict(ba_problems=windows, pose_problems=poses, stereo=True, project=True, bf=BF, intrinsics=(FX, FY, CX, CY))
    lanes = [stream_mod.StereoStream(F, W, H, NFEAT, **kw) for _ in range(2)]
    cap = lanes[0].cap
    ex = pkg.ORBextractor(NFEAT, 1.2, 8, 20, 7, max_width=W, max_height=H, max_batch=2 * F)
    bow1 = pkg.ORBmatcher(0.7, True, max_features=cap)
    proj1 = pkg.ORBmatcher(0.9, True, max_features=cap)
    for step in range(6):
        ss = lanes[step % 2]
        start = (step * F) % D
        ss.load_window(d_all, start)
        ss.step_device(pipelined=True)
        torch.cuda.synchronize()
        ss.ex.check()
        idx = [(start + i) % D for i in range(F)]
        imgs = [frames[i][0] for i in idx] + [frames[i][1] for i in idx]
        kps_r, desc_r, n_r = extract_full(pkg, ex, imgs)
        counts = ss.counts.cpu().numpy()
        kps = ss.kps.cpu().numpy().view(pkg.keypoint_dtype).reshape(1 + 2 * F, cap)
        desc = ss.desc.cpu().numpy()
        assert np.array_equal(counts[1:], n_r) and counts[0] == counts[F]
        for b in range(2 * F):
            assert np.array_equal(kps[1 + b, :n_r[b]], kps_r[b, :n_r[b]]) and np.array_equal(desc[1 + b, :n_r[b]],
                                                                                               desc_r[b, :n_r[b]])
        if 6 in idx:
            assert counts[1 + idx.index(6)] == 0
        # BoW: pair f matches left image f-1 (slot f; slot 0 = this step's left image F-1) against left image f
        nm, match = ss.nmatch.cpu().numpy(), ss.match.cpu().numpy()
        for f in range(F):
            a, nb = int(counts[f]), int(counts[1 + f])
            n1, m1 = bow1.SearchByBoW(desc[f, :a].copy(), np.zeros(a, np.int32), np.ones(a, np.uint8),
                                      kps[f, :a]["angle"].copy(), desc[1 + f, :nb].copy(), np.zeros(nb, np.int32),
                                      kps[1 + f, :nb]["angle"].copy())
            assert n1 == nm[f] and np.array_equal(m1, match[f, :nb]) and (match[f, nb:] == -1).all(), (step, f)
        # stereo, pair by pair
        ur, dp_all, ns = ss.ur.cpu().numpy(), ss.dp_all.cpu().numpy(), ss.nstereo.cpu().numpy()
        assert np.array_equal(dp_all[0], dp_all[F])
        for f in range(F):
            ur1, dp1, ns1 = ex.stereo_match(f, F + f, 1, BF, 0.0)
            assert ns1[0] == ns[f] and np.array_equal(ur1[0], ur[f]) and np.array_equal(dp1[0], dp_all[1 + f]), (step, f)
        # projection: pair f = last (slot f, its depth) -> current (slot f + 1)
        q = ss.track_queries_host(kps[:F], desc[:F], dp_all[:F], counts[:F], np.tile(ss.motion.reshape(1, 12), (F, 1)), ss.fx,
                                  ss.fy, ss.cx, ss.cy, 1)
        npm, pm = ss.npmatch.cpu().numpy(), ss.pmatch.cpu().numpy()
        for f in range(F):
            nl, nc = int(counts[f]), int(counts[1 + f])
            k = kps[1 + f, :nc]
            n1, m1 = proj1.SearchByProjection(np.ascontiguousarray(q[f, :nl]), k["x"].copy(), k["y"].copy(), k["octave"].copy(),
                                              k["angle"].copy(), ur[f, :nc].copy(), None, desc[1 + f, :nc].copy(), ss.geom,
                                              ss.proj_th, mode=ss.proj_mode)
            assert n1 == npm[f] and np.array_equal(m1, pm[f, :nc]) and (pm[f, nc:] == -1).all(), (step, f)
        assert npm.sum() > 0 and nm.sum() > 0
    for ss in lanes:
        ss.finish()
        step = ss._step_no - 1  # a lane counts its own steps: pose problems and windows go round-robin over them
        ps, prep = ss.last_solved["pose"]
        assert ps == step
        direct = pkg.Optimizer(max_kf=4, max_mp=16, max_edges=64, max_batch=F).PoseOptimizationBatch(ss._step_poses(step))
        for i, out in enumerate(direct):
            Tcw, outl = prep["keep"][i][1]
            assert prep["ress"][i].n_inliers == out["n_inliers"]
            assert np.array_equal(Tcw, out["Tcw"]) and np.array_equal(outl[:len(out["outlier"])], out["outlier"])
        bs, ba = ss.last_solved["ba"]
        assert bs == step
        wins = ss._step_windows(step)
        opt = pkg.Optimizer(max_kf=16, max_mp=max(16, max(len(w["points"]) for w in wins)),
                            max_edges=max(64, max(len(w["edges"]) for w in wins)), max_batch=len(wins))
        opt.set_sm_budget(64)
        for out, ref in zip(ba, opt.LocalBundleAdjustmentBatch(wins)):
            assert out["n_trials"] == ref["n_trials"] and out["chi2"] == ref["chi2"]
            for k in ("Tcw", "points", "outlier", "trace"):
                assert np.array_equal(out[k], ref[k]), k
        ref_ba = oracle.local_ba(wins[0])
        assert ba[0]["n_trials"] == ref_ba["n_trials"] and np.array_equal(ba[0]["outlier"], ref_ba["outlier"])
