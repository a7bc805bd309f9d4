"""GPU parity of the matchers against the CPU oracle: bit-exact match pairs and counts."""
import numpy as np
import pytest

from synth import CROWD_F, CROWD_Q, synth_descriptors, synth_projection, synth_projection_map, synth_triangulation, synth_windows

pytestmark = pytest.mark.gpu


def test_descriptor_distance(pkg, oracle):
    rng = np.random.RandomState(0)
    a = rng.randint(0, 256, size=(3000, 32)).astype(np.uint8)
    b = rng.randint(0, 256, size=(3000, 32)).astype(np.uint8)
    b[:10] = a[:10]
    b[10:20] = ~a[10:20]
    m = pkg.ORBmatcher()
    d = m.DescriptorDistance(a, b)
    ref = np.array([oracle.descriptor_distance(a[i], b[i]) for i in range(len(a))])
    assert np.array_equal(d, ref)
    assert d[0] == 0 and d[10] == 256


@pytest.mark.parametrize("n_nodes", [100, 1, 17])
@pytest.mark.parametrize("nnratio,strict,checkori", [(0.7, False, True), (0.75, True, True), (0.9, False, False)])
def test_search_by_bow(pkg, oracle, n_nodes, nnratio, strict, checkori):
    A, nA, vA, aA, B, nB, aB = synth_descriptors(2000, seed=1234 + n_nodes, n_nodes=n_nodes)
    vB = None
    if strict:  # KF-KF variant needs MapPoints on both sides
        vB = (np.random.RandomState(3).randint(0, 100, size=len(B)) < 90).astype(np.uint8)
    m = pkg.ORBmatcher(nnratio, checkori)
    n, match = m.SearchByBoW(A, nA, vA, aA, B, nB, aB, validB=vB, strict_lt=strict)
    on, omatch = oracle.search_by_bow(A, nA, vA, aA, B, nB, aB, validB=vB, nnratio=nnratio, strict_lt=strict,
                                      check_ori=checkori)
    assert n == on
    assert np.array_equal(match, omatch)
    assert n > 500


def test_search_by_bow_contention(pkg, oracle):
    """Near-duplicate descriptors in one node: many rows want the same frame feature -> K-lists run dry (rescan path)."""
    rng = np.random.RandomState(9)
    n = 600
    base = rng.randint(0, 256, size=(3, 32)).astype(np.uint8)

    def noisy(k):
        d = base[rng.randint(0, 3, size=k)].copy()
        for i in range(k):
            for b in rng.choice(256, size=int(rng.randint(0, 10)), replace=False):
                d[i, b >> 3] ^= np.uint8(1 << (b & 7))
        return d

    A, B = noisy(n), noisy(n)
    nodeA = np.zeros(n, np.int32)
    nodeB = np.zeros(n, np.int32)
    vA = np.ones(n, np.uint8)
    aA = np.zeros(n, np.float32)
    aB = np.zeros(n, np.float32)
    m = pkg.ORBmatcher(0.99, False)
    cnt, match = m.SearchByBoW(A, nodeA, vA, aA, B, nodeB, aB)
    on, omatch = oracle.search_by_bow(A, nodeA, vA, aA, B, nodeB, aB, nnratio=0.99, check_ori=False)
    assert cnt == on and np.array_equal(match, omatch)


@pytest.mark.parametrize("nnratio,th_low", [(0.7, 50), (0.6, 50), (0.9, 50), (0.75, 100), (0.3, 50), (1.5, 50)])
def test_search_by_bow_distance_cut_boundaries(pkg, oracle, nnratio, th_low):
    """The K-list stage only lists candidates closer than cut = floor(TH_LOW / ratio) + 2 (bow_distance_cut): rows whose best /
    second-best distances sit on and around TH_LOW, ratio * second and the cut itself, with 0, 1, 2 and > 8 candidates below
    the cut, plus rows that compete for the same frame feature, must still match the oracle exactly."""
    rng = np.random.RandomState(int(nnratio * 100) + th_low)
    cut = max(int(np.floor(th_low / nnratio)) + 2, th_low + 2)

    def flipped(d, k):
        o = d.copy()
        for b in rng.choice(256, size=k, replace=False):
            o[b >> 3] ^= np.uint8(1 << (b & 7))
        return o
    A, B, nodeA, nodeB = [], [], [], []
    dists = sorted(set([0, 1, th_low - 1, th_low, th_low + 1, cut - 2, cut - 1, cut, cut + 1, int(th_low * nnratio), 255, 256]))
    dists = [d for d in dists if 0 <= d <= 256]
    node = 0
    for d1 in dists:
        for d2 in dists:
            if d2 < d1:
                continue
            a = rng.randint(0, 256, size=32).astype(np.uint8)
            A.append(a)
            nodeA.append(node)
            B += [flipped(a, d1), flipped(a, d2)]
            nodeB += [node, node]
            node += 1
    # a crowded node: 12 candidates below the cut for each of 6 rows that share them (K-list overflow + contention)
    c = rng.randint(0, 256, size=32).astype(np.uint8)
    for r in range(6):
        A.append(flipped(c, r))
        nodeA.append(node)
    for k in range(12):
        B.append(flipped(c, min(max(cut - 14 + k, 0), 256)))
        nodeB.append(node)
    A, B = np.array(A, np.uint8), np.array(B, np.uint8)
    nodeA, nodeB = np.array(nodeA, np.int32), np.array(nodeB, np.int32)
    vA = np.ones(len(A), np.uint8)
    aA, aB = np.zeros(len(A), np.float32), np.zeros(len(B), np.float32)
    for strict in (False, True):
        m = pkg.ORBmatcher(nnratio, False)
        n, match = m.SearchByBoW(A, nodeA, vA, aA, B, nodeB, aB, strict_lt=strict, th_low=th_low)
        on, omatch = oracle.search_by_bow(A, nodeA, vA, aA, B, nodeB, aB, nnratio=nnratio, strict_lt=strict, check_ori=False,
                                          th_low=th_low)
        assert n == on and np.array_equal(match, omatch)
        assert n > 0


def test_search_by_bow_ragged(pkg, oracle):
    m = pkg.ORBmatcher(0.7, True)
    A, nA, vA, aA, B, nB, aB = synth_descriptors(333, seed=5, n_nodes=7)
    n, match = m.SearchByBoW(A, nA, vA, aA, B[:57], nB[:57], aB[:57])
    on, om = oracle.search_by_bow(A, nA, vA, aA, B[:57], nB[:57], aB[:57])
    assert n == on and np.array_equal(match, om)
    n, match = m.SearchByBoW(A[:0], nA[:0], vA[:0], aA[:0], B, nB, aB)
    assert n == 0 and (match == -1).all()
    vz = np.zeros_like(vA)
    n, match = m.SearchByBoW(A, nA, vz, aA, B, nB, aB)
    assert n == 0 and (match == -1).all()


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("cluster,th", [(False, 7.0), (False, 15.0), (True, 15.0), ("crowd", 7.0)])
def test_search_by_projection(pkg, oracle, mode, cluster, th):
    """cluster = "crowd": the crowded window of synth_projection, whose last queries reach the exact rescan."""
    d = synth_projection(seed=21 + mode, cluster=cluster is True, th=th, crowd=cluster == "crowd")
    m = pkg.ORBmatcher(0.9, True)
    n, match = m.SearchByProjection(d["q"], d["kpx"], d["kpy"], d["octave"], d["angle"], d["uright"], d["occupied"],
                                    d["desc"], d["geom"], d["th"], mode=mode)
    on, om = oracle.search_by_projection_last(d["q"], d["kpx"], d["kpy"], d["octave"], d["angle"], d["uright"],
                                              d["occupied"], d["desc"], d["geom"], float(d["th"]), mode=mode)
    assert n == on
    assert np.array_equal(match, om)
    assert n > 100
    if cluster == "crowd":
        assert (match[CROWD_F] >= 0).all()  # features 9..12 of the crowd are only found by the rescan
        # the batched form (no occupancy on entry) on the same pair
        kps = np.zeros((1, len(d["kpx"])), pkg.keypoint_dtype)
        kps["x"][0], kps["y"][0], kps["octave"][0], kps["angle"][0] = d["kpx"], d["kpy"], d["octave"], d["angle"]
        nb, mb = m.SearchByProjectionBatch(d["q"][None], np.array([len(d["q"])]), kps, d["uright"][None], d["desc"][None],
                                           np.array([len(d["kpx"])]), d["geom"], d["th"], mode=mode)
        on, om = oracle.search_by_projection_last(d["q"], d["kpx"], d["kpy"], d["octave"], d["angle"], d["uright"], None,
                                                  d["desc"], d["geom"], float(d["th"]), mode=mode)
        assert nb[0] == on and np.array_equal(mb[0], om)
        assert (mb[0][CROWD_F] >= 0).all()


def test_against_committed_golden(pkg):
    import os
    G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    m = pkg.ORBmatcher(0.7, True)
    for nodes in (100, 1):
        g = np.load(os.path.join(G, "bow_2000_nodes%d.npz" % nodes))
        A, nA, vA, aA, B, nB, aB = synth_descriptors(2000, seed=1234 + nodes, n_nodes=nodes)
        n, match = m.SearchByBoW(A, nA, vA, aA, B, nB, aB)
        assert n == int(g["n"]) and np.array_equal(match, g["match"])
    g = np.load(os.path.join(G, "proj_seed21.npz"))
    d = synth_projection(seed=21, cluster=False, th=7.0)
    m9 = pkg.ORBmatcher(0.9, True)
    n, match = m9.SearchByProjection(d["q"], d["kpx"], d["kpy"], d["octave"], d["angle"], d["uright"], d["occupied"],
                                     d["desc"], d["geom"], d["th"], mode=0)
    assert n == int(g["n"]) and np.array_equal(match, g["match"])


@pytest.mark.parametrize("th", [1.0, 3.0])
@pytest.mark.parametrize("cluster", [False, True, "crowd"])
@pytest.mark.parametrize("nnratio", [0.8, 0.6])
def test_search_by_projection_map(pkg, oracle, th, cluster, nnratio):
    """SearchByProjection(Frame&, vector<MapPoint*>&, th) (src/ORBmatcher.cc:70-175): bit-exact match array and count,
    including the level-gated ratio test, the dynamic occupancy and K-list exhaustion (clustered descriptors, and the
    crowded window of synth_projection, whose queries from the eighth on reach the exact rescan)."""
    d = synth_projection_map(seed=31 + int(th), cluster=cluster is True, crowd=cluster == "crowd")
    m = pkg.ORBmatcher(nnratio, True)
    n, match = m.SearchByProjectionMap(d["q"], d["kpx"], d["kpy"], d["octave"], d["uright"], d["occupied"], d["desc"],
                                       d["geom"], th=th)
    on, om = oracle.search_by_projection_map(d["q"], d["kpx"], d["kpy"], d["octave"], d["uright"], d["occupied"],
                                             d["desc"], d["geom"], th=th, nnratio=nnratio)
    assert n == on
    assert np.array_equal(match, om)
    assert n > 100
    if cluster == "crowd":
        assert (match[CROWD_F] >= 0).all()


def test_search_by_projection_map_edge_cases(pkg, oracle):
    d = synth_projection_map(seed=5)
    m = pkg.ORBmatcher(0.8, True)
    n, match = m.SearchByProjectionMap(d["q"][:0], d["kpx"], d["kpy"], d["octave"], d["uright"], d["occupied"], d["desc"],
                                       d["geom"])
    assert n == 0 and (match == -1).all()
    q = d["q"].copy()
    q["in_view"] = 0  # nothing in view: no match
    n, match = m.SearchByProjectionMap(q, d["kpx"], d["kpy"], d["octave"], d["uright"], d["occupied"], d["desc"], d["geom"])
    assert n == 0 and (match == -1).all()
    occ = np.ones_like(d["occupied"])  # every feature already holds a map point
    n, match = m.SearchByProjectionMap(d["q"], d["kpx"], d["kpy"], d["octave"], d["uright"], occ, d["desc"], d["geom"])
    assert n == 0 and (match == -1).all()
    n, match = m.SearchByProjectionMap(d["q"], d["kpx"], d["kpy"], d["octave"], d["uright"], None, d["desc"], d["geom"])
    on, om = oracle.search_by_projection_map(d["q"], d["kpx"], d["kpy"], d["octave"], d["uright"], None, d["desc"],
                                             d["geom"], nnratio=0.8)
    assert n == on and np.array_equal(match, om)


@pytest.mark.parametrize("chi2,greedy", [(True, False), (False, False), (False, True), (True, True)])
@pytest.mark.parametrize("cluster", [False, True, "crowd"])
def test_search_windows(pkg, oracle, chi2, greedy, cluster):
    """Search core of Fuse (src/ORBmatcher.cc:1020-1174 with the chi-square gate, :1179-1310 without) and of
    SearchByProjection(KeyFrame*, Scw, vpPoints, vpMatched, th) (:388-512, greedy occupancy): identical best feature per
    map point, distance and accepted count.  cluster = "crowd": the crowded window of synth_projection."""
    d = synth_windows(seed=13 + int(chi2) + 2 * int(greedy), th=3.0 if not cluster else 6.0, cluster=cluster is True,
                      crowd=cluster == "crowd")
    occ = d["occupied"] if greedy else None
    m = pkg.ORBmatcher(0.8, True)
    n, best, bd = m.SearchWindows(d["q"], d["kpx"], d["kpy"], d["octave"], d["uright"], d["inv_sigma2"], occ, d["desc"],
                                  d["geom"], chi2=chi2, greedy=greedy)
    on, obest, obd = oracle.search_windows(d["q"], d["kpx"], d["kpy"], d["octave"], d["uright"], d["inv_sigma2"], occ,
                                           d["desc"], d["geom"], chi2=chi2, greedy=greedy)
    assert n == on
    assert np.array_equal(best, obest)
    assert np.array_equal(bd, obd)
    assert n > 100
    if greedy:  # every feature is given to at most one map point
        used = best[best >= 0]
        assert len(np.unique(used)) == len(used)
        if cluster == "crowd":  # the greedy search hands the whole crowd out, the last four through the rescan
            assert set(CROWD_F) <= set(best[CROWD_Q])


@pytest.mark.parametrize("only_stereo", [False, True])
@pytest.mark.parametrize("n_nodes", [100, 7])
def test_search_for_triangulation(pkg, oracle, only_stereo, n_nodes):
    """ORBmatcher::SearchForTriangulation (src/ORBmatcher.cc:810-1009): identical vMatches12 and count (greedy per node,
    last-minimum tie rule, epipole and epipolar-line gates, rotation consistency)."""
    d = synth_triangulation(seed=17 + n_nodes, n_nodes=n_nodes)
    m = pkg.ORBmatcher(0.6, True)
    n, m12 = m.SearchForTriangulation(d["kf1"], d["kf2"], d["F12"], d["ex"], d["ey"], d["scale"], d["sigma2"],
                                      only_stereo=only_stereo)
    on, om12 = oracle.search_for_triangulation(d["kf1"], d["kf2"], d["F12"], float(d["ex"]), float(d["ey"]), d["scale"],
                                               d["sigma2"], only_stereo=only_stereo)
    assert n == on
    assert np.array_equal(m12, om12)
    assert n > 100
    used = m12[m12 >= 0]
    assert len(np.unique(used)) == len(used)


def test_search_by_sim3_directions(pkg, oracle):
    """SearchBySim3 (src/ORBmatcher.cc:1314-1555) = two window searches with th_dist = TH_HIGH and no flags, followed by
    the mutual-consistency loop; both directions must agree with the oracle and the composition must be symmetric."""
    d12 = synth_windows(seed=51, th=7.5)
    d21 = synth_windows(seed=52, th=7.5)
    m = pkg.ORBmatcher(0.8, True)
    res = []
    for d in (d12, d21):
        n, best, bd = m.SearchWindows(d["q"], d["kpx"], d["kpy"], d["octave"], d["uright"], None, None, d["desc"], d["geom"],
                                      th_dist=100)
        on, obest, obd = oracle.search_windows(d["q"], d["kpx"], d["kpy"], d["octave"], d["uright"], None, None, d["desc"],
                                               d["geom"], th_dist=100)
        assert n == on and np.array_equal(best, obest) and np.array_equal(bd, obd)
        assert (bd[best >= 0] <= 100).all() and n > 200
        res.append(best)


def test_distinctive_descriptors(pkg, oracle):
    """MapPoint::ComputeDistinctiveDescriptors (src/MapPoint.cc:359-440): same representative descriptor per map point
    (median of the distance rows, first minimum), including points with 0, 1, 2 and >32 observations and ties."""
    rng = np.random.RandomState(8)
    counts = np.concatenate([[0, 1, 2, 2, 3, 40, 97], rng.randint(1, 25, size=3000)]).astype(np.int32)
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    desc = np.zeros((offsets[-1], 32), np.uint8)
    for p in range(len(counts)):
        base = rng.randint(0, 256, 32).astype(np.uint8)
        for i in range(counts[p]):
            d = base.copy()
            for b in rng.choice(256, size=int(rng.randint(0, 30)), replace=False):
                d[b >> 3] ^= np.uint8(1 << (b & 7))
            desc[offsets[p] + i] = d
        if counts[p] >= 3 and p % 7 == 0:  # exact duplicates -> ties between medians
            desc[offsets[p] + 1] = desc[offsets[p]]
    m = pkg.ORBmatcher(0.6, True)
    best = m.DistinctiveDescriptors(desc, offsets)
    obest = oracle.distinctive_descriptors(desc, offsets)
    assert np.array_equal(best, obest)
    assert best[0] == -1 and best[1] == 0


def _flip(d, bits):
    o = d.copy()
    for b in bits:
        o[b >> 3] ^= np.uint8(1 << (b & 7))
    return o


_GEOM = dict(mnMinX=np.float32(0), mnMinY=np.float32(0), mnMaxX=np.float32(640), mnMaxY=np.float32(480),
             bf=np.float32(0), scale_factors=np.array([np.float32(1.2) ** i for i in range(8)], np.float32))


@pytest.mark.parametrize("check_ori", [False, True])
def test_search_for_initialization_crowded(pkg, oracle, check_ori):
    """SearchForInitialization (src/ORBmatcher.cc:515-643) on one crowded window.  Twelve features, each 20 bits from a
    base descriptor B on bits of its own, are claimed at distance 0 by the first twelve keypoints.  The later keypoints
    carry B: their eight nearest features are claimed ones (vMatchedDistance 0 <= 20), and the window holds 15 candidates,
    so they are decided by the exact rescan, which finds the three unclaimed features at 30, 40 and 45 bits from B."""
    rng = np.random.RandomState(3)
    base = rng.randint(0, 256, 32).astype(np.uint8)
    bits = rng.permutation(256)
    claimed = [_flip(base, bits[20 * k:20 * k + 20]) for k in range(12)]
    free = [_flip(base, bits[240:256].tolist() + bits[:n - 16].tolist()) for n in (30, 40, 45)]
    desc2 = np.array(claimed + free, np.uint8)
    n2 = len(desc2)
    kpx2 = (np.float32(320) + (np.arange(n2) % 5 - 2) * np.float32(1.5)).astype(np.float32)
    kpy2 = (np.float32(240) + (np.arange(n2) // 5 - 1) * np.float32(1.5)).astype(np.float32)
    desc1 = np.array(claimed + [base] * 5, np.uint8)
    n1 = len(desc1)
    prev = np.tile(np.array([[320.0, 240.0]], np.float32), (n1, 1))
    oct1, oct2 = np.zeros(n1, np.int32), np.zeros(n2, np.int32)
    ang1 = np.full(n1, 10.0, np.float32)
    ang2 = np.full(n2, 9.0, np.float32)
    m = pkg.ORBmatcher(0.9, check_ori)
    n, m12 = m.SearchForInitialization(prev.copy(), oct1, ang1, desc1, kpx2, kpy2, oct2, ang2, desc2, _GEOM, window=10)
    on, om = oracle.search_for_initialization(prev.copy(), oct1, ang1, desc1, kpx2, kpy2, oct2, ang2, desc2, _GEOM,
                                              window=10, nnratio=0.9, check_ori=check_ori)
    assert n == on and np.array_equal(m12, om)
    assert np.array_equal(m12[:12], np.arange(12))
    assert m12[12] >= 12  # only the rescan reaches the unclaimed features


# (bin: pairs) of a rotation histogram, and the matches ComputeThreeMaxima (src/ORBmatcher.cc:1866-1908) keeps
ROT_HISTS = [
    ({2: 10, 9: 1, 17: 1}, 12),         # second and third at exactly a tenth of the first: kept
    ({2: 11, 9: 1, 17: 1}, 11),         # just below a tenth: dropped
    ({4: 5, 11: 5, 20: 5, 25: 5}, 15),  # four equal bins: the earlier three win
    ({2: 10, 9: 10, 17: 1, 25: 1}, 21),  # a tie for third at a tenth: the earlier bin wins
]


@pytest.mark.parametrize("search", ["bow", "proj", "init"])
@pytest.mark.parametrize("bins,kept", ROT_HISTS)
def test_rotation_three_maxima(pkg, oracle, search, bins, kept):
    """The rotation culls of SearchByBoW, SearchByProjection and SearchForInitialization at ComputeThreeMaxima's edges: one
    unambiguous match per pair (equal descriptors, one candidate), its rotation put in the bin asked for."""
    rot = np.concatenate([np.full(c, 12.0 * b + 3.0) for b, c in bins.items()]).astype(np.float32)
    n = len(rot)
    rng = np.random.RandomState(n)
    desc = rng.randint(0, 256, size=(n, 32)).astype(np.uint8)
    zero = np.zeros(n, np.float32)
    m = pkg.ORBmatcher(0.9, True)
    if search == "bow":
        node, valid = np.arange(n, dtype=np.int32), np.ones(n, np.uint8)
        got = m.SearchByBoW(desc, node, valid, rot, desc, node, zero)
        ref = oracle.search_by_bow(desc, node, valid, rot, desc, node, zero, nnratio=0.9, check_ori=True)
    else:
        x = (np.float32(40) + np.float32(40) * (np.arange(n) % 14)).astype(np.float32)
        y = (np.float32(40) + np.float32(40) * (np.arange(n) // 14)).astype(np.float32)
        octave = np.zeros(n, np.int32)
        if search == "proj":
            q = np.zeros(n, pkg.proj_query_dtype)
            q["u"], q["v"], q["invz"], q["angle"], q["has_obs"], q["desc"] = x, y, np.float32(0.1), rot, 1, desc
            args = (q, x, y, octave, zero, np.full(n, -1, np.float32), None, desc, _GEOM, np.float32(7))
            got = m.SearchByProjection(*args)
            ref = oracle.search_by_projection_last(*args[:-1], 7.0)
        else:
            prev = np.stack([x, y], 1)
            args = (octave, rot, desc, x, y, octave, zero, desc, _GEOM)
            got = m.SearchForInitialization(prev.copy(), *args, window=10)
            ref = oracle.search_for_initialization(prev.copy(), *args, window=10, nnratio=0.9, check_ori=True)
    assert got[0] == ref[0] == kept
    assert np.array_equal(got[1], ref[1])
