"""Pins the keyframe insertion's CPU restatement (oracle/kfinsert.cpp) against the REFERENCE'S OWN
LocalMapping::ProcessNewKeyFrame + MapPointCulling and MapPoint::UpdateNormalAndDepth (src/LocalMapping.cc,
src/KeyFrame.cc and src/MapPoint.cc compiled in place -> oracle/_ref/libref_kfinsert.so, oracle/ref_kfinsert_glue.cpp).
Integers, lists and descriptors must be identical and every float bit-identical."""
import os

import numpy as np
import pytest

import kfinsert_binding as kb

pytestmark = pytest.mark.skipif(not os.path.exists(kb.REF_LIB),
                                reason="oracle/_ref not built (needs the reference's sources: make -C oracle -f "
                                       "kfinsert.mk kfinsert-ref REF=...)")

SCENES = {
    "stereo": dict(seed=1),
    "mono": dict(seed=2, mono=True),
    "stereo_listed": dict(seed=3, p_listed=0.5),
    "duplicates": dict(seed=4, p_dup=0.2, n_recent=600),
    "bad_points_and_keyframes": dict(seed=5, p_bad=0.2, p_kf_bad=0.3),
    "one_observer": dict(seed=6, max_obs=1),
    "two_hundred_observers": dict(seed=7, n_kf=220, n_slots=120, big_obs=4),
    "wrapping_ids": dict(seed=8, cur_id=(1 << 32) + 1),
    "mono_2000_slots": dict(seed=9, mono=True, n_slots=2000, n_kf=60),
}


@pytest.fixture(scope="module")
def ref():
    return kb.Reference()


@pytest.fixture(scope="module")
def orc():
    return kb.Oracle()


@pytest.mark.parametrize("name", sorted(SCENES))
def test_restatement_equals_reference(ref, orc, name):
    d = kb.scene(**SCENES[name])
    o = orc(d)
    kb.same_as_reference(d, ref(d), o)
    # the scene reaches the cases it is named for
    assert o["mp_updated"].any() and o["n_list"] > 0


def test_every_culling_rule_is_reached(orc):
    seen = set()
    for seed in range(10):
        seen |= set(orc(kb.scene(seed, n_slots=300)).get("list_verdict").tolist())
    assert seen == {kb.pkg.KFI_KEPT, kb.pkg.KFI_BAD, kb.pkg.KFI_CULLED_RATIO, kb.pkg.KFI_CULLED_OBS,
                    kb.pkg.KFI_RETIRED}


@pytest.mark.parametrize("seed", range(12))
def test_random_scenes(ref, orc, seed):
    d = kb.scene(100 + seed, n_kf=int(5 + 7 * seed), n_slots=int(50 + 40 * seed), mono=seed % 3 == 0)
    kb.same_as_reference(d, ref(d), orc(d))


def test_normal_and_depth_equals_reference(ref, orc):
    d = kb.normal_depth_scene(3, n_mp=10000)
    a, b = orc.normal_and_depth(d), ref.normal_and_depth(d)
    assert np.array_equal(a["updated"], b["updated"])
    u = a["updated"] != 0
    assert u.sum() > 9000
    for k in ("normal", "min_dist", "max_dist"):
        assert np.array_equal(kb.bits(a[k])[u], kb.bits(b[k])[u]), k
