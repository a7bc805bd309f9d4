"""Pins the keyframe database (oracle: oracle/kfdb.cpp; cuda: csrc/kfdb.cu behind pkg.KeyFrameDatabase) against the
REFERENCE'S OWN src/KeyFrameDatabase.cc (compiled in place -> oracle/_ref/libref_kfdb.so, oracle/ref_kfdb_glue.cpp) with
the vendored DBoW2 as ORBVocabulary.  Seeded sequences of add / erase / clear / loop query / relocalisation query are
replayed on both; after every query the candidate lists must be identical, order included, and so must the six query
fields (mnLoopQuery, mnLoopWords, mLoopScore, mnRelocQuery, mnRelocWords, mRelocScore) of every keyframe id."""
import os

import numpy as np
import pytest

import kfdb_binding as kb

pytestmark = pytest.mark.skipif(not os.path.exists(kb.REF_LIB),
                                reason="oracle/_ref not built (needs the reference's sources: make -C oracle -f kfdb.mk ref REF=...)")


@pytest.fixture(params=["oracle", pytest.param("cuda", marks=pytest.mark.gpu)])
def make_db(request):
    """`oracle` (CPU) or the CUDA path (-m gpu), constructed from the vocabulary size."""
    if request.param == "oracle":
        return kb.Oracle
    pkg = request.getfixturevalue("pkg")
    return pkg.KeyFrameDatabase


class Replay:
    """Runs the same operations on the reference and on the implementation under test and compares after every query."""

    def __init__(self, make_db, n_words):
        self.ref, self.db, self.orc = kb.Reference(n_words), make_db(n_words), kb.Oracle(n_words)
        self.ids = set()
        self.n_queries = self.n_nonempty = 0

    def add(self, i, bow):
        for d in (self.ref, self.db, self.orc):
            d.add(i, *bow)
        self.ids.add(i)

    def erase(self, i):
        for d in (self.ref, self.db, self.orc):
            d.erase(i)

    def clear(self):
        for d in (self.ref, self.db, self.orc):
            d.clear()

    def _compare(self, want, got, what, state_ids):
        assert got == want, what
        for i in state_ids:
            assert self.db.keyframe_state(i) == self.ref.keyframe_state(i), (what, i)
        self.n_queries += 1
        self.n_nonempty += bool(want)
        return want

    def loop(self, qid, bow, connected, min_score, covis, state_ids=None):
        r = [d.DetectLoopCandidates(qid, bow[0], bow[1], connected, min_score, covis=covis) for d in (self.ref, self.db, self.orc)]
        assert r[2] == r[0]
        return self._compare(r[0], r[1], ("loop", qid), sorted(self.ids) if state_ids is None else state_ids)

    def reloc(self, fid, bow, covis, state_ids=None):
        r = [d.DetectRelocalizationCandidates(fid, bow[0], bow[1], covis=covis) for d in (self.ref, self.db, self.orc)]
        assert r[2] == r[0]
        return self._compare(r[0], r[1], ("reloc", fid), sorted(self.ids) if state_ids is None else state_ids)


def noisy(rng, bow, keep=0.8):
    w, v = bow
    m = rng.random(len(w)) < keep
    v2 = v[m] * (0.5 + rng.random(m.sum()))
    return w[m], v2 / v2.sum()


def test_trajectory_with_revisits(make_db):
    """300 keyframes along a trajectory that revisits its 40 places, loop queries before adding each third keyframe
    (LoopClosing::DetectLoop: the query keyframe is not in the database yet, its connected keyframes are its last ones)
    and relocalisation queries with noisy copies of earlier keyframes, interleaved.  Includes query id 0, repeated frame ids,
    the query keyframe itself in the database, duplicated BowVectors (equal scores) and neighbours outside the database."""
    m = kb.MapModel(seed=1)
    rng = np.random.default_rng(2)
    R = Replay(make_db, m.n_words)
    stale0 = R.ref.stale_reads()[1]
    covis = m.covis(310)
    bows, fid = [], 1
    for i in range(300):
        bow = bows[-1] if i % 37 == 36 else m.keyframe(i)  # an exact copy: equal scores
        bows.append(bow)
        if i % 3 == 0 and i > 5:
            qid = 0 if i == 12 else i
            conn = [j for j in range(max(0, i - 6), i) if rng.random() < 0.8]
            R.loop(qid, bow, conn, float(rng.uniform(0.0, 0.04)), covis)
        R.add(i, bow)
        if i % 50 == 49:  # the query keyframe itself in the database
            R.loop(i, bow, [i - 1, i - 2], 0.01, covis)
        if i % 4 == 1 and i > 5:
            src = int(rng.integers(0, i))
            f = 0 if i == 9 else fid
            R.reloc(f, noisy(rng, bows[src]), covis)
            if i % 20 == 1:  # a repeated frame id
                R.reloc(f, noisy(rng, bows[int(rng.integers(0, i))]), covis)
            fid += 1
    assert R.n_nonempty > 40
    assert R.ref.stale_reads()[1] > stale0          # the stale mRelocScore read fired
    assert R.orc.counters()[0] > 0 and R.orc.counters()[1] > 0  # and the dedupe path was taken


def test_culling_churn(make_db):
    """Keyframes are culled (erased, 40 %) while the map grows, some culled ids are added again (with a new add sequence
    number, so a new place in every inverted list), queries in between."""
    m = kb.MapModel(seed=3, n_places=25)
    rng = np.random.default_rng(4)
    R = Replay(make_db, m.n_words)
    covis = m.covis(420)
    alive, erased, bows, fid = [], [], {}, 1000
    for i in range(400):
        bows[i] = m.keyframe(i)
        R.add(i, bows[i])
        alive.append(i)
        if rng.random() < 0.4 and len(alive) > 5:
            j = alive.pop(int(rng.integers(0, len(alive))))
            R.erase(j)
            erased.append(j)
        if erased and rng.random() < 0.1:
            j = erased.pop(int(rng.integers(0, len(erased))))
            bows[j] = m.keyframe(j) if rng.random() < 0.5 else bows[j]
            R.add(j, bows[j])
            alive.append(j)
        R.erase(10**6)  # not in the database: no effect
        if i % 7 == 3:
            R.reloc(fid, noisy(rng, bows[int(rng.integers(0, i + 1))]), covis)
            fid += 1
        if i % 9 == 5:
            R.loop(i + 1, m.keyframe(i + 1), alive[-4:], float(rng.uniform(0.0, 0.03)), covis)
    assert R.n_nonempty > 20


def test_clear_with_reused_ids(make_db):
    """clear() (Tracking::Reset): every keyframe is deleted and ids restart at 0 with fresh objects and fresh state."""
    m = kb.MapModel(seed=5, n_places=15)
    rng = np.random.default_rng(6)
    R = Replay(make_db, m.n_words)
    covis = m.covis(130)
    for rnd in range(3):
        bows = []
        for i in range(60 + 30 * rnd):
            bows.append(m.keyframe(i + 7 * rnd))
            R.add(i, bows[-1])
            if i % 6 == 5:
                R.reloc(i // 6 + 1, noisy(rng, bows[int(rng.integers(0, i + 1))]), covis)
                R.loop(i + 1, m.keyframe(i + 1), [i, i - 1], 0.005, covis)
        R.clear()
        assert R.db.size() == 0
        R.reloc(1, noisy(rng, bows[3]), covis)  # empty database
        R.ids = set(range(130))
    assert R.n_nonempty > 10


def test_zipf_map_3000(make_db):
    """3,000 keyframes of about 1,000 Zipf-distributed words each over the real vocabulary's 971,814 words."""
    kfs = kb.zipf_map(seed=7, n_kf=3000, words_per_kf=1000)
    rng = np.random.default_rng(8)
    R = Replay(make_db, kb.ORBVOC_WORDS)
    ids = np.zeros((3000, 10), np.uint64)
    n = np.zeros(3000, np.int32)
    for i in range(3000):
        nb = [j for j in (i - 1, i + 1, i - 2, i + 2, i - 3, i + 3, i - 8, i + 8, i - 16, i + 16) if 0 <= j < 3000]
        n[i] = len(nb)
        ids[i, :len(nb)] = nb
    for i, b in enumerate(kfs):
        R.add(i, b)
    check_ids = sorted(set(rng.integers(0, 3000, 300).tolist()))
    for q in range(8):
        src = int(rng.integers(0, 3000))
        got = R.reloc(5000 + q, noisy(rng, kfs[src]), (ids, n), state_ids=check_ids)
        assert got
        R.loop(3000 + q, noisy(rng, kfs[src], 0.9), [src, max(src - 1, 0)], 0.02, (ids, n), state_ids=check_ids)


def test_edge_cases(make_db):
    """Empty database, empty query, no shared word, every score below minScore, query id 0 on untouched keyframes
    (their mnLoopQuery / mnRelocQuery is already 0: nothing is listed, the counts still grow), neighbours outside the
    database, and no covisibility table at all."""
    R = Replay(make_db, 1000)
    w = np.array([1, 5, 9, 40], np.uint32)
    v = np.array([0.1, 0.2, 0.3, 0.4])
    assert R.reloc(1, (w, v), None) == []                     # empty database
    R.add(3, (w, v))
    R.add(4, (np.array([5, 9, 41], np.uint32), np.array([0.5, 0.25, 0.25])))
    R.add(7, (np.array([2, 600], np.uint32), np.array([0.5, 0.5])))
    covis = (np.array([[0] * 10] * 3 + [[4, 7, 900] + [0] * 7, [3, 900] + [0] * 8] + [[0] * 10] * 3, np.uint64),
             np.array([0, 0, 0, 3, 2, 0, 0, 0], np.int32))
    assert R.reloc(2, (np.zeros(0, np.uint32), np.zeros(0)), covis) == []   # empty query
    assert R.reloc(3, (np.array([100, 200], np.uint32), np.array([0.5, 0.5])), covis) == []  # no shared word
    assert R.loop(10, (w, v), [], 2.0, covis) == []          # everything below minScore
    assert R.reloc(0, (w, v), covis) == []                   # query id 0: untouched keyframes are not listed
    R.loop(0, (w, v), [], 0.0, covis)
    assert R.reloc(11, (w, v), covis)                        # neighbour 900 was never in the database
    assert R.reloc(12, (w, v), None)
    R.loop(12, (w, v), [4], 0.0, covis)                      # 4 connected: reset and never listed
    R.loop(12, (w, v), [], 0.0, covis)                       # the same id again: nothing new is listed
    with pytest.raises(Exception):
        R.db.add(3, w, v)                                    # a live id again
