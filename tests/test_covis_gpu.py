"""The CUDA covisibility update (csrc/covis.cu behind pkg.Covisibility) at size, its error codes, and the drop-in
host/adapters/Covisibility_b200.cc against the reference's sequential KeyFrame::UpdateConnections on one object graph."""
import os

import numpy as np
import pytest

import covis_binding as cb

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def covis(pkg):
    return pkg.Covisibility(max_kf=8192, max_mp=1 << 19, max_obs=1 << 22, max_slots=1 << 19, max_conn=1 << 22,
                            max_batch=1024)


def test_8000_keyframes_batch_256_vs_oracle(covis):
    """8,000 keyframes, a batch of every keyframe (in 256-call batches) and then random batches of 256 with repeats:
    every keyframe's state, the pairs, the reads and the changed flags equal the oracle's."""
    rng = np.random.default_rng(1)
    w = cb.random_map(seed=77, n_kf=8000, slots_per_kf=120)
    orc = cb.Oracle()
    order = rng.permutation(8000).tolist()
    batches = [order[i:i + 256] for i in range(0, 8000, 256)] + [rng.integers(0, 8000, 256).tolist() for _ in range(3)]
    for members in batches:
        d = w.problem(members)
        want, got = orc.UpdateConnections(d), covis.UpdateConnections(d)
        cb.same(want, got, 8000)
        assert np.array_equal(want["pairs"], got["pairs"]) and np.array_equal(want["changed"], got["changed"])
        w.apply(want)
    assert covis.last_ms() > 0


def test_repeat_bit_identical(covis):
    w = cb.random_map(seed=5, n_kf=600, slots_per_kf=150)
    d = w.problem(list(range(600)) + list(range(0, 600, 7)))
    r0 = covis.raw(d)
    for _ in range(3):
        r = covis.raw(d)
        assert r[0] == r0[0] == 0
        for k in r0[1]:
            assert np.array_equal(np.asarray(r0[1][k]), np.asarray(r[1][k])), k


def _untouched(o):
    return all(not np.any(v) for k, v in o.items() if isinstance(v, np.ndarray))


def test_error_codes(pkg, covis):
    """Every error code; nothing is written on BAD_ARG, only the *_need fields on a caller-capacity error."""
    w = cb.random_map(seed=6, n_kf=200, slots_per_kf=80)
    base = w.problem(list(range(50)))
    BAD, CAP = pkg.ERR_BAD_ARG, pkg.ERR_CAPACITY

    def bad(**kw):
        d = dict(base)
        d.update(kw)
        rc, o = covis.raw(d)
        assert rc == BAD, kw.keys()
        assert _untouched(o) and o["need"] == (0, 0, 0, 0)

    bad(member=np.zeros(0, np.int32), slot_off=np.zeros(1, np.int32))           # batch < 1
    bad(member=np.array([200] + [0] * 49, np.int32))                            # member out of range
    ids = base["kf_id"].copy(); ids[5] = ids[4]
    bad(kf_id=ids)                                                              # ids not ascending
    ok = base["obs_kf"].copy(); o0 = base["obs_off"]
    r = next(i for i in range(len(o0) - 1) if o0[i + 1] - o0[i] >= 2)
    ok[o0[r] + 1] = ok[o0[r]]
    bad(obs_kf=ok)                                                              # observer repeated
    ok = base["obs_kf"].copy(); ok[o0[r]], ok[o0[r] + 1] = ok[o0[r] + 1], ok[o0[r]]
    bad(obs_kf=ok)                                                              # observers not ascending
    ok = base["obs_kf"].copy(); ok[0] = 200
    bad(obs_kf=ok)                                                              # observer missing from the table
    sm = base["slot_mp"].copy(); sm[0] = len(base["mp_bad"])
    bad(slot_mp=sm)                                                             # slot out of range
    par = base["parent"].copy(); par[3] = 200
    bad(parent=par)                                                             # parent out of range
    mo = base["slot_off"].copy(); mo[3] = mo[2] - 1
    bad(slot_off=mo)                                                            # offsets that are not a CSR
    # the caller's capacities: the need is reported, nothing else written
    rc, o = covis.raw(base, cap=1)
    assert rc == CAP and o["need"][0] > 1 and not np.any(o["map_kf"]) and not np.any(o["changed"])
    # the handle's capacities
    small = pkg.Covisibility(max_kf=100, max_mp=1 << 16, max_obs=1 << 20, max_slots=1 << 16, max_conn=1 << 16,
                             max_batch=8)
    rc, o = small.raw(base)
    assert rc == CAP and _untouched(o)
    rc, o = small.raw(w.problem(list(range(9))))
    assert rc == CAP
    tiny = pkg.Covisibility(max_kf=256, max_mp=1 << 16, max_obs=1 << 20, max_slots=1 << 16, max_conn=64, max_batch=64)
    rc, o = tiny.raw(cb.random_map(seed=7, n_kf=50, slots_per_kf=40).problem(list(range(50))))
    assert rc == CAP and _untouched(o)                                          # the output areas
    # the handle stays usable
    rc, o = covis.raw(base)
    assert rc == 0


@pytest.mark.skipif(not os.path.exists(cb.ADP_LIB), reason="oracle/_ref/libadapter_covis.so not built")
def test_adapter_vs_reference():
    """libadapter_covis.so (one device call per batch through b200::UpdateConnections) against the reference's own
    UpdateConnections called one keyframe at a time, on one object graph: new keyframes, then a loop correction's
    step 2.2 and step 5 batches."""
    ref, adp = cb.Reference(), cb.Reference(adapter=True)
    w = cb.trajectory(seed=4, n_kf=120, revisit=90)
    for i in range(120):
        cb.observe(w, i)
        d = w.problem([i])
        want, got = ref.UpdateConnections(d), adp.UpdateConnections(d)
        cb.same(want, got, 120)
        assert want["children"] == got["children"]
        w.apply(want)
    cur = 119
    for members in (sorted(set(w.ordKf[cur]) | {cur}), w.ordKf[cur] + [cur]):
        d = w.problem(members)
        want, got = ref.UpdateConnections(d), adp.UpdateConnections(d)
        cb.same(want, got, 120)
        assert want["children"] == got["children"]
        w.apply(want)
