"""The CUDA keyframe insertion and UpdateNormalAndDepth (csrc/mappoint.cu behind pkg.ORBmatcher) against the CPU
restatement bit for bit, batches against their problems run one by one, repeated calls, the argument errors, and the
drop-in host/adapters/LocalMapping_b200.cc against the reference's own ProcessNewKeyFrame + MapPointCulling on one object
graph."""
import os

import numpy as np
import pytest

import kfinsert_binding as kb
from test_oracle_reference_kfinsert import SCENES

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def matcher(pkg):
    return pkg.ORBmatcher(max_features=64)


@pytest.fixture(scope="module")
def orc():
    return kb.Oracle()


@pytest.mark.parametrize("name", sorted(SCENES))
def test_device_equals_restatement(matcher, orc, name):
    d = kb.scene(**SCENES[name])
    want = orc(d)
    got = matcher.ProcessNewKeyFrame(d)
    kb.same(want, got)
    kb.same(got, matcher.ProcessNewKeyFrame(d))  # repeated calls are bit-identical


@pytest.mark.parametrize("seed", range(8))
def test_random_scenes(matcher, orc, seed):
    d = kb.scene(200 + seed, n_kf=int(5 + 9 * seed), n_slots=int(50 + 250 * seed), mono=seed % 2 == 0)
    kb.same(orc(d), matcher.ProcessNewKeyFrame(d))


def test_ragged_batch_equals_single_calls(matcher, orc):
    rng = np.random.default_rng(5)
    ds = [kb.scene(300 + i, n_kf=int(rng.integers(3, 80)), n_slots=int(rng.integers(1, 2000)), mono=bool(i % 2),
                   n_recent=int(rng.integers(0, 400))) for i in range(32)]
    before = matcher.launch_count()
    outs = matcher.ProcessNewKeyFrame(ds)
    assert matcher.launch_count() - before == 2  # one list pass and one point pass for the whole batch
    for d, o in zip(ds, outs):
        kb.same(o, matcher.ProcessNewKeyFrame(d))
        kb.same(o, orc(d))


def _broken(d):
    """Copies of d with one malformed field each."""
    out = []
    for k, v in [("cur", len(d["kf_center"])), ("cur", -1), ("mp_ref", None), ("obs_octave", 8), ("slot_mp", -2),
                 ("recent", len(d["mp_bad"])), ("obs_kf", None), ("scale_factors", np.zeros(0, np.float32))]:
        e = {key: (val.copy() if isinstance(val, np.ndarray) else val) for key, val in d.items()}
        if k == "mp_ref":  # a point to associate whose reference keyframe is not an observer
            first = next(m for m in e["slot_mp"].tolist() if m >= 0 and not e["mp_bad"][m] and
                         d["cur"] not in e["obs_kf"][e["obs_off"][m]:e["obs_off"][m + 1]].tolist())
            e["mp_ref"][first] = d["cur"]
        elif k == "obs_kf":  # a row not strictly ascending
            m = int(np.argmax(np.diff(e["obs_off"]) >= 2))
            a = e["obs_off"][m]
            e["obs_kf"][a + 1] = e["obs_kf"][a]
        elif isinstance(v, np.ndarray) or k == "cur":
            e[k] = v
        else:
            e[k][0] = v
        out.append(e)
    return out


def test_bad_arguments_write_nothing(matcher, pkg):
    good = kb.scene(11, n_slots=200)
    for bad in _broken(good):
        rc, outs = matcher.raw_kfinsert([good, bad])
        assert rc == 2  # B2S_ERR_BAD_ARG
        for o in outs:
            for k in kb.OUT_KEYS[:-2]:
                assert not np.asarray(o[k]).any(), k
            assert o["n_list"] == 0 and o["n_culled"] == 0


@pytest.mark.parametrize("n_mp", [10000, 100000])
def test_normal_and_depth_equals_restatement(matcher, orc, n_mp):
    d = kb.normal_depth_scene(n_mp, n_mp=n_mp, n_kf=300)
    want, got = orc.normal_and_depth(d), matcher.UpdateNormalAndDepth(d)
    assert np.array_equal(want["updated"], got["updated"])
    for k in ("normal", "min_dist", "max_dist"):
        assert np.array_equal(kb.bits(want[k]), kb.bits(got[k])), k
    again = matcher.UpdateNormalAndDepth(d)
    assert all(np.array_equal(kb.bits(again[k]), kb.bits(got[k])) for k in ("normal", "min_dist", "max_dist"))


def test_normal_and_depth_rejects_a_foreign_reference(matcher, pkg):
    d = kb.normal_depth_scene(1, n_mp=100, n_kf=50)
    m = int(np.argmax(np.diff(d["obs_off"]) > 0))
    row = d["obs_kf"][d["obs_off"][m]:d["obs_off"][m + 1]].tolist()
    d["mp_ref"][m] = next(k for k in range(50) if k not in row)
    with pytest.raises(pkg.B200SlamError):
        matcher.UpdateNormalAndDepth(d)


@pytest.mark.skipif(not os.path.exists(kb.ADP_LIB), reason="oracle/_ref/libadapter_kfinsert.so not built")
@pytest.mark.parametrize("name", ["stereo", "mono", "stereo_listed", "duplicates", "bad_points_and_keyframes"])
def test_drop_in_equals_reference(name):
    d = kb.scene(**SCENES[name])
    want, got = kb.Reference()(d), kb.Reference(adapter=True)(d)
    for k in ("mp_nobs", "mp_bad", "obs_alive", "cur_idx", "desc", "slot_mp"):
        assert np.array_equal(want[k], got[k]), k
    for k in ("normal", "min_dist", "max_dist"):
        assert np.array_equal(kb.bits(want[k]), kb.bits(got[k])), k
    assert want["recent"] == got["recent"] and want["erased"] == got["erased"] and want["conn"] == got["conn"]
