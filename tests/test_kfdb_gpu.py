"""The device keyframe database (csrc/kfdb.cu, pkg.KeyFrameDatabase): BowVector pool growth and compaction under churn,
the capacity and duplicate-add errors, and the drop-in adapter (host/adapters/KeyFrameDatabase_b200.cc) against the
reference's own src/KeyFrameDatabase.cc on one object graph (oracle/ref_kfdb_glue.cpp drives both)."""
import os

import numpy as np
import pytest

import kfdb_binding as kb

pytestmark = pytest.mark.gpu


def test_pool_churn_beyond_initial_capacity(pkg):
    """More than 1.3 M BowVector entries pass through a pool that starts at 65,536 and is compacted as erased vectors pile
    up; the database keeps answering like the oracle."""
    m = kb.MapModel(seed=21, n_places=30, place_words=900, noise=200)
    rng = np.random.default_rng(22)
    db, orc = pkg.KeyFrameDatabase(m.n_words), kb.Oracle(m.n_words)
    covis = m.covis(4000)
    alive, bows, total = [], {}, 0
    for i in range(4000):
        bows[i] = m.keyframe(i)
        total += len(bows[i][0])
        for d in (db, orc):
            d.add(i, *bows[i])
        alive.append(i)
        if len(alive) > 150:  # a sliding map: old keyframes are culled
            j = alive.pop(int(rng.integers(0, 100)))
            for d in (db, orc):
                d.erase(j)
        if i % 250 == 249:
            q = bows[alive[int(rng.integers(0, len(alive)))]]
            assert db.DetectRelocalizationCandidates(i, *q, covis=covis) == orc.DetectRelocalizationCandidates(i, *q, covis=covis)
            assert db.DetectLoopCandidates(i + 1, *q, alive[-3:], 0.01, covis=covis) == \
                orc.DetectLoopCandidates(i + 1, *q, alive[-3:], 0.01, covis=covis)
            for k in alive[-20:]:
                assert db.keyframe_state(k) == orc.keyframe_state(k)
    assert total > 20 * 65536 and db.size() == orc.size() == 150


def test_overlong_vector_is_a_capacity_error(pkg):
    db = pkg.KeyFrameDatabase(100000)
    w = np.arange(8193, dtype=np.uint32)
    v = np.full(8193, 1.0 / 8193)
    with pytest.raises(pkg.B200SlamError) as e:
        db.add(1, w, v)
    assert e.value.code == pkg.ERR_CAPACITY
    with pytest.raises(pkg.B200SlamError) as e:
        db.DetectRelocalizationCandidates(1, w, v)
    assert e.value.code == pkg.ERR_CAPACITY
    db.add(1, w[:8192], v[:8192])  # the longest accepted
    assert db.DetectRelocalizationCandidates(2, w[:8192], v[:8192]) == [1]


def test_adding_a_live_id_again_is_an_error(pkg):
    db = pkg.KeyFrameDatabase(1000)
    w, v = np.array([1, 2, 3], np.uint32), np.array([0.2, 0.3, 0.5])
    db.add(5, w, v)
    with pytest.raises(pkg.B200SlamError) as e:
        db.add(5, w, v)
    assert e.value.code == pkg.ERR_BAD_ARG
    db.erase(5)
    db.add(5, w, v)  # erased ids may come back
    assert db.size() == 1
    with pytest.raises(pkg.B200SlamError):
        db.add(6, np.array([3, 2], np.uint32), np.array([0.5, 0.5]))  # not in word order


@pytest.mark.skipif(not (os.path.exists(kb.REF_LIB) and os.path.exists(kb.ADP_LIB)),
                    reason="oracle/_ref not built (make -C oracle -f kfdb.mk ref)")
def test_adapter_matches_reference_on_one_object_graph():
    """The same stand-in KeyFrame / Frame objects, covisibility and connected sets go to the reference's
    KeyFrameDatabase and to the drop-in; both must return the same vector<KeyFrame*> (as ids)."""
    m = kb.MapModel(seed=31, n_places=20)
    rng = np.random.default_rng(32)
    ref, adp = kb.Reference(m.n_words), kb.Reference(m.n_words, adapter=True)
    covis = m.covis(260)
    bows, n_nonempty = {}, 0
    for i in range(250):
        bows[i] = m.keyframe(i)
        if i % 4 == 0 and i > 4:
            conn = [j for j in range(i - 5, i) if rng.random() < 0.7]
            a = ref.DetectLoopCandidates(i, *bows[i], conn, 0.01, covis=covis)
            assert adp.DetectLoopCandidates(i, *bows[i], conn, 0.01, covis=covis) == a
            n_nonempty += bool(a)
        for d in (ref, adp):
            d.add(i, *bows[i])
        if i % 5 == 2:
            q = bows[int(rng.integers(0, i + 1))]
            a = ref.DetectRelocalizationCandidates(i, *q, covis=covis)
            assert adp.DetectRelocalizationCandidates(i, *q, covis=covis) == a
            n_nonempty += bool(a)
        if i % 11 == 10:
            for d in (ref, adp):
                d.erase(i - 7)
        if i == 150:
            for d in (ref, adp):
                d.clear()
    assert n_nonempty > 20
