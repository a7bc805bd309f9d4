"""Pins keyframe culling (oracle: oracle/culling.cpp; cuda: csrc/culling.cu behind pkg.KeyFrameCulling) against the
REFERENCE'S OWN LocalMapping::KeyFrameCulling (src/LocalMapping.cc, src/KeyFrame.cc and src/MapPoint.cc compiled in place
-> oracle/_ref/libref_localmapping.so, oracle/ref_culling_glue.cpp), which runs the real KeyFrame::SetBadFlag and
MapPoint::EraseObservation / SetBadFlag.  Compared after each call: the verdicts in list order (the reference's culls in
the order SetBadFlag made them), and every point's bad flag, nObs, observers and the local keyframes' slots.  Everything
is an integer or one double compare: the bar is equality."""
import os

import numpy as np
import pytest

import culling_binding as cb

pytestmark = pytest.mark.skipif(not os.path.exists(cb.REF_LIB),
                                reason="oracle/_ref not built (needs the reference's sources: make -C oracle -f "
                                       "culling.mk culling-ref REF=...)")
REF = None
ORC = None


@pytest.fixture(params=["oracle", pytest.param("cuda", marks=pytest.mark.gpu)])
def subject(request):
    """The implementation under test: `oracle` (CPU) or the CUDA path (-m gpu)."""
    global REF, ORC
    REF = REF or cb.Reference()
    ORC = ORC or cb.Oracle()
    if request.param == "oracle":
        return ORC
    return request.getfixturevalue("pkg").KeyFrameCulling(max_kf=1024, max_mp=1 << 17, max_obs=1 << 20,
                                                          max_local=512, max_slots=1 << 18, max_batch=64)


def check(subject, w, cur, local, mono):
    """One call on the reference and on the subject; compares and returns the subject's result."""
    d = w.problem(local, monocular=mono)
    want, got = REF(w, d, cur), subject(d)
    cb.same(want, got, counts=False)
    assert [local[i] for i in range(len(local)) if got["verdict"][i] == cb.pkg.VERDICT_CULLED] == want["erased"]
    if subject is not ORC:  # the counts the reference does not report
        cb.same(ORC(d), got)
    return got


@pytest.mark.parametrize("mono", [False, True])
def test_trajectory_with_revisits(subject, mono):
    """A 160-keyframe path that comes back over itself; the current keyframe is on the revisit, so its local list
    spans both passes.  Several current keyframes along the path."""
    w = cb.trajectory(seed=11 + mono, n_kf=160, stereo=not mono, revisit=110)
    culled = 0
    for cur in (40, 120, 159):
        got = check(subject, w, cur, w.covisible(cur), mono)
        culled += got["n_culled"]
    assert culled > 0


def _cascades(mono):
    """Seeds of small worlds where an earlier cull flips a later verdict: kept at entry but culled, and the reverse."""
    rng = np.random.default_rng(5 + mono)
    orc = cb.Oracle()
    found = {}
    for seed in range(400):
        w = cb.random_world(1000 + seed, 24, slots_per_kf=40, stereo=not mono, odd=0.02)
        cur = int(rng.integers(1, 24))
        local = cb.local_list(w, rng, cur, size=23)
        d = w.problem(local, monocular=mono)
        entry, now = cb.entry_verdicts(orc, d), orc(d)["verdict"].tolist()
        for e, v in zip(entry, now):
            if e == cb.pkg.VERDICT_KEPT and v == cb.pkg.VERDICT_CULLED:
                found.setdefault("to_culled", (w, cur, local))
            if e == cb.pkg.VERDICT_CULLED and v == cb.pkg.VERDICT_KEPT:
                found.setdefault("to_kept", (w, cur, local))
        if len(found) == 2:
            break
    return found


@pytest.mark.parametrize("mono", [False, True])
def test_cascade_flips_later_verdicts(subject, mono):
    """An earlier cull turns a later keyframe from kept to culled (its points turn bad and leave nMPs) and from culled
    to kept (its points lose the observers that made them redundant)."""
    found = _cascades(mono)
    assert set(found) == {"to_culled", "to_kept"}
    for w, cur, local in found.values():
        check(subject, w, cur, local, mono)


def boundary_world():
    """Hand-built keyframes, each probing one rule; witnesses 1-4 observe at octave 0 and are in the list last, so the
    slot nulling of the earlier culls shows in their rows.  Returns (w, cur, local, probes)."""
    probes = [(10, 9), (10, 10), (20, 18), (20, 19), (30, 27), (30, 28), (100, 90), (100, 91), (11, 10), (0, 0)]
    n = 1 + 4 + len(probes) + 5 + 1
    w = cb.World(np.arange(n) * 2)
    W = [1, 2, 3, 4]
    k = 5
    for nm, nr in probes:  # nMPs = nm, nRedundant = nr
        for j in range(nm):
            m = w.add_point()
            w.add_slot(k, m, 0, j % 2 == 0, 1.0)
            for x in (W[:3] if j < nr else W[:1]):
                w.add_slot(x, m, 0, False, 1.0)
        if nm == 0:  # only NULL slots and a bad point
            w.add_slot(k, -1)
            m = w.add_point(bad=1)
            w.add_slot(k, m)
        k += 1
    # nObs exactly 3 with a stereo observation: not redundant; culling the stereo observer makes it bad
    S = k
    for j in range(6):
        m = w.add_point()
        w.add_slot(S, m, 0, True, 1.0)
        w.add_slot(W[0], m, 0, False, 1.0)
    k += 1
    # octave: observers at own + 1 count, at own + 2 do not
    O1, O2 = k, k + 1
    for kk, dlt in ((O1, 1), (O2, 2)):
        for j in range(10):
            m = w.add_point()
            w.add_slot(kk, m, 1, False, 1.0)
            for x in W[:3]:
                w.add_slot(x, m, 1 + dlt, False, 1.0)
    k += 2
    # depth exactly mThDepth and NaN (counted, not redundant), negative (skipped, redundant), 9 redundant
    D = k
    w.th_depth[D] = 4.0
    for z, red in [(1.0, True)] * 9 + [(4.0, False), (np.nan, False), (-1.0, True)]:
        m = w.add_point()
        w.add_slot(D, m, 0, True, z)
        for x in (W[:3] if red else W[:1]):
            w.add_slot(x, m, 0, False, 1.0)
    k += 1
    # a deferred one: redundant, mbNotErase
    N = k
    w.not_erase[N] = 1
    for j in range(10):
        m = w.add_point()
        w.add_slot(N, m, 0, False, 1.0)
        for x in W[:3]:
            w.add_slot(x, m, 0, False, 1.0)
    k += 1
    w.count_nobs()
    for m, o in enumerate(w.obs):  # the nObs-3 points of S
        if S in o:
            w.nobs[m] = 3
    cur = n - 1
    local = list(range(5, cur)) + [0] + W
    return w, cur, local, dict(S=S, O1=O1, O2=O2, D=D, N=N, probes=probes)


@pytest.mark.parametrize("mono", [False, True])
def test_boundaries(subject, mono):
    """The 90 % boundary at multiples of 10 (9/10 and 18/20 kept, 10/10 and 19/20 culled, 10/11 culled), nMPs = 0,
    nObs exactly 3 with a stereo observer, octave + 1 against + 2, depths exactly mThDepth / negative / NaN, mbNotErase
    and mnId 0 in the list."""
    w, cur, local, pr = boundary_world()
    got = check(subject, w, cur, local, mono)
    V = dict(zip(local, got["verdict"].tolist()))
    K, C, D_, S_ = cb.pkg.VERDICT_KEPT, cb.pkg.VERDICT_CULLED, cb.pkg.VERDICT_DEFERRED, cb.pkg.VERDICT_SKIPPED
    for i, (nm, nr) in enumerate(pr["probes"]):
        assert V[5 + i] == (C if nr > 0.9 * nm else K), (nm, nr)
    assert V[0] == S_ and V[pr["N"]] == D_
    assert V[pr["O1"]] == C and V[pr["O2"]] == K
    o = ORC(w.problem(local, monocular=mono))
    i = local.index(pr["D"])
    # stereo: 9 redundant of 11 counted (the negative depth is skipped, NaN and mThDepth are not); monocular: all 12
    assert (o["n_mps"][i], o["n_redundant"][i]) == ((12, 10) if mono else (11, 9)) and V[pr["D"]] == K


def test_inconsistent_graphs(subject):
    """Duplicate slots, slots whose point does not list the keyframe, observations whose slot holds another point, bad
    points with observers and nObs off by one, at a high rate."""
    rng = np.random.default_rng(3)
    for seed in range(6):
        mono = seed % 2 == 1
        w = cb.random_world(200 + seed, 50, slots_per_kf=60, stereo=not mono, odd=0.2)
        cur = int(rng.integers(1, 50))
        check(subject, w, cur, cb.local_list(w, rng, cur, size=49), mono)


def test_20_random_maps(subject):
    """20 seeded maps, stereo and monocular, with mbNotErase keyframes and mnId 0 in the lists; the maps reach every
    verdict."""
    rng = np.random.default_rng(1)
    seen = np.zeros(4, int)
    for seed in range(20):
        mono = seed % 3 == 0
        n = int(rng.integers(10, 70))
        w = cb.random_world(seed, n, stereo=not mono)
        cur = int(rng.integers(1, n))
        local = cb.local_list(w, rng, cur)
        if 0 not in local and rng.random() < 0.5:
            local.insert(int(rng.integers(0, len(local) + 1)), 0)
        seen += np.bincount(check(subject, w, cur, local, mono)["verdict"], minlength=4)
    assert np.all(seen > 0), seen
