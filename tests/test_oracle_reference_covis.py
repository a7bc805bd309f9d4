"""Pins the covisibility update (oracle: oracle/covis.cpp; cuda: csrc/covis.cu behind pkg.Covisibility) against the
REFERENCE'S OWN src/KeyFrame.cc (compiled in place -> oracle/_ref/libref_keyframe.so, oracle/ref_covis_glue.cpp).  Every
batch runs on both; after every batch the full state of every keyframe must be identical (connection map, ordered list and
weights, parent, children, mbFirstConnection), and so must each call's reads: GetVectorCovisibleKeyFrames() just before
it and the connection map just after it.  Everything is an integer: the bar is equality."""
import copy
import os

import numpy as np
import pytest

import covis_binding as cb

pytestmark = pytest.mark.skipif(not os.path.exists(cb.REF_LIB),
                                reason="oracle/_ref not built (needs the reference's sources: make -C oracle -f covis.mk "
                                       "covis-ref REF=...)")
REF = None


@pytest.fixture(params=["oracle", pytest.param("cuda", marks=pytest.mark.gpu)])
def subject(request):
    """The implementation under test: `oracle` (CPU) or the CUDA path (-m gpu)."""
    global REF
    REF = REF or cb.Reference()
    if request.param == "oracle":
        return cb.Oracle()
    pkg = request.getfixturevalue("pkg")
    return pkg.Covisibility(max_kf=2048, max_mp=1 << 18, max_obs=1 << 21, max_slots=1 << 18, max_conn=1 << 21,
                            max_batch=1024)


def run(w, subject, members):
    """One batch on the reference and on the subject; compares, then carries the reference's state into w."""
    d = w.problem(members)
    want = REF.UpdateConnections(d)
    got = subject.UpdateConnections(d)
    cb.same(want, got, len(w.ids))
    children = [set(c) for c in w.children]
    for p, c in got["pairs"]:
        children[p].add(int(c))
    assert want["children"] == children
    w.apply(want)
    return d, want, got


def test_trajectory_300(subject):
    """300 keyframes along a path that comes back to its start (revisits), one call per new keyframe after its
    observations join the map (LocalMapping::ProcessNewKeyFrame)."""
    w = cb.trajectory(seed=1, n_kf=300, revisit=150)
    n_parent = 0
    for i in range(300):
        cb.observe(w, i)
        d, want, got = run(w, subject, [i])
        n_parent += len(got["pairs"])
    assert n_parent > 250


def test_loop_correction(subject):
    """A map built keyframe by keyframe, then LoopClosing::CorrectLoop: fusion rewires observations (a point of the
    current keyframe's neighbourhood replaced by a loop-side point, the old one bad), then the step 2.2 batch (the
    connected keyframes in CorrectedSim3 key order: ascending index) and the step 5 batch (mvpCurrentConnectedKFs)."""
    rng = np.random.default_rng(3)
    w = cb.trajectory(seed=2, n_kf=160, revisit=120)
    for i in range(160):
        cb.observe(w, i)
        run(w, subject, [i])
    cur = 159
    for rnd in range(2):
        conn = sorted(set(w.ordKf[cur]) | {cur})
        # SearchAndFuse / ReplaceMapPoint: points seen around the current keyframe take over loop-side points
        for k in conn:
            for j, p in enumerate(w.slots[k]):
                if p < 0 or w.mp_bad[p] or rng.random() > 0.15:
                    continue
                loop_kf = int(rng.integers(0, 40))
                q = w.add_point(w.obs[p] + [loop_kf])
                w.mp_bad[p] = 1
                for o in w.obs[q]:
                    w.slots[o] = [q if s == p else s for s in w.slots[o]]
                    if p not in w.slots[o] and q not in w.slots[o]:
                        w.slots[o].append(q)
        run(w, subject, conn)                                   # step 2.2
        current_connected = w.ordKf[cur] + [cur]
        d, want, got = run(w, subject, current_connected)      # step 5
        assert len(got["start_off"]) == len(current_connected) + 1
        cur = 158


def test_initial_map_pair(subject):
    """Tracking::CreateInitialMapMonocular (Tracking.cc:1074-1075): the first two keyframes, ids 0 and 1, each call in
    turn.  Keyframe 0 never takes a parent."""
    w = cb.World([0, 1])
    for _ in range(300):
        w.slots[0].append(w.add_point([0, 1]))
    w.slots[1] = list(reversed(w.slots[0]))
    run(w, subject, [0])
    d, want, got = run(w, subject, [1])
    assert w.parent[0] == -1 and w.first[0] == 1
    assert w.parent[1] == 0 and w.first[1] == 0 and w.children[0] == {1}


@pytest.mark.parametrize("seed", range(20))
def test_random_maps(subject, seed):
    """Random maps of 100-1,000 keyframes with Zipf observation counts, bad keyframes and bad points, NULL slots: a
    batch of every keyframe, then random batches with repeated members."""
    rng = np.random.default_rng(100 + seed)
    n = int(rng.integers(100, 1001))
    w = cb.random_map(seed=seed, n_kf=n, slots_per_kf=int(rng.integers(40, 160)))
    run(w, subject, list(rng.permutation(n)))
    for _ in range(2):
        run(w, subject, rng.integers(0, n, int(rng.integers(1, 65))).tolist())


def test_batch_equals_sequential(subject):
    """A batch equals its members run one at a time with the state passed from each call to the next."""
    rng = np.random.default_rng(9)
    w = cb.random_map(seed=50, n_kf=300, slots_per_kf=120)
    run(w, subject, list(range(300)))
    members = rng.integers(0, 300, 40).tolist() + [5, 5, 6, 5]
    w1, w2 = copy.deepcopy(w), copy.deepcopy(w)
    s = subject.UpdateConnections(w1.problem(members))
    w1.apply(s)
    for i, m in enumerate(members):
        one = subject.UpdateConnections(w2.problem([m]))
        assert np.array_equal(one["start_kf"], s["start_kf"][s["start_off"][i]:s["start_off"][i + 1]])
        assert np.array_equal(one["after_kf"], s["after_kf"][s["after_off"][i]:s["after_off"][i + 1]])
        w2.apply(one)
    assert w1.conn == w2.conn and w1.ordKf == w2.ordKf and w1.ordW == w2.ordW and w1.children == w2.children
    assert np.array_equal(w1.parent, w2.parent) and np.array_equal(w1.first, w2.first)
    # a partner whose own call ran last keeps a strong-only list beside weak map entries
    assert any(len(w1.ordKf[i]) < len(w1.conn[i]) for i in range(300))


def targeted_world():
    """Keyframes built so that each case of the reference's logic happens once (see test_targeted_cases)."""
    w = cb.World([0, 4, 7, 9, 12, 20, 21, 30, 31])
    def pts(n, obs):
        return [w.add_point(obs) for _ in range(n)]
    # K1 (index 1): partners 2 and 3 at 10 each (a tie below 15: fallback to the first, index 2), NULL and bad slots
    w.slots[1] = pts(10, [1, 2]) + pts(10, [1, 3]) + [-1, -1]
    bad = pts(30, [1, 4])
    for p in bad:
        w.mp_bad[p] = 1
    w.slots[1] += bad
    # K5 (index 5): partners 6 and 7 at 20 each (equal weights: larger id first), 8 at 3 (weak), 6 is a bad keyframe
    w.slots[5] = pts(20, [5, 6]) + pts(20, [5, 7]) + pts(3, [5, 8])
    w.kf_bad[6] = 1
    # K6 and K7 see each other (members that are each other's partners) and K5
    w.slots[6] = [s for s in w.slots[5] if 6 in w.obs[s]] + pts(16, [6, 7])
    w.slots[7] = [s for s in w.slots[5] if 7 in w.obs[s]] + w.slots[6][20:]
    # K8: no observation besides itself (empty counter); K0 (id 0) sees K1 strongly
    w.slots[8] = pts(5, [8])
    w.slots[0] = pts(18, [0, 1])
    for p in w.slots[0]:
        w.slots[1].append(p)
    return w


def test_targeted_cases(subject):
    """Each case of UpdateConnections, asserted to occur: fallback with a tie for nmax, an empty counter, mnId 0 never
    gets a parent, the parent set only once, equal weights ordered larger id first, NULL slots and bad points, a bad observer keyframe still counted, a repeated member, members that are each other's partners."""
    w = targeted_world()
    d, want, got = run(w, subject, [1, 8, 0, 5, 6, 7, 5, 1])
    c = cb.counters(d)
    assert c[0] == {0: 18, 2: 10, 3: 10}                      # K1: strong K0, weak tie 2 / 3
    assert c[1] == {}                                         # empty counter: K8 unchanged, no parent
    assert w.parent[8] == -1 and w.first[8] == 1 and not w.conn[8]
    assert w.parent[0] == -1 and w.first[0] == 1              # id 0: no parent
    assert 6 in c[3] and c[3][6] == 20 and c[3][7] == 20      # bad keyframe 6 counted; equal weights
    assert got["start_kf"][got["start_off"][6]:got["start_off"][7]].tolist()[:2] == [7, 6]  # K5's second call: 7 first
    assert w.parent[5] == 7                                    # set by the first call, kept by the second
    assert w.ordW[5] == [20, 20] and w.conn[5][8] == 3         # strong-only list, weak partner in the map
    # the fallback with a tie: K1's second call in the same batch keeps K0 (18 >= 15) strong
    w2 = targeted_world()
    w2.slots[1] = w2.slots[1][:22]                              # only the tie 2 / 3 at 10, plus NULL slots
    d, want, got = run(w2, subject, [1])
    assert w2.ordKf[1] == [2] and w2.ordW[1] == [10] and w2.parent[1] == 2
    assert sorted(w2.conn[1].items()) == [(2, 10), (3, 10)]
    assert w2.ordKf[2] == [1]                                   # AddConnection on the fallback partner only
