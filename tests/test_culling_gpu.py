"""The CUDA keyframe culling (csrc/culling.cu behind pkg.KeyFrameCulling) at size against the CPU restatement, batches
against their problems run one by one, repeated calls, its error codes, and the drop-in host/adapters/LocalMapping_b200.cc
against the reference's own KeyFrameCulling on one object graph."""
import os
import subprocess
import sys

import numpy as np
import pytest

import culling_binding as cb

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def culling(pkg):
    return pkg.KeyFrameCulling(max_kf=512, max_mp=1 << 16, max_obs=1 << 19, max_local=320, max_slots=1 << 18,
                               max_batch=256)


@pytest.fixture(scope="module")
def big_batch():
    """256 problems over four 320-keyframe paths with revisits (two stereo, two monocular): local lists of 1-300
    keyframes in covisibility order, random order, or with mnId 0 and mbNotErase keyframes."""
    rng = np.random.default_rng(2)
    worlds = []
    for i in range(4):
        w = cb.trajectory(seed=40 + i, n_kf=320, pts_per_kf=40, stereo=i < 2, revisit=200)
        w.not_erase[rng.random(320) < 0.05] = 1
        worlds.append((w, i >= 2))
    ds = []
    for j in range(256):
        w, mono = worlds[j % 4]
        cur = int(rng.integers(1, 320))
        size = int(rng.choice([1, 2, 31, 32, 33, 100, 299, 300])) if j < 64 else int(rng.integers(1, 301))
        if j % 3 == 0:
            local = cb.local_list(w, rng, cur, size=size)
        else:
            local = [k for k in rng.permutation(320).tolist() if k != cur][:size]
        ds.append(w.problem(local, monocular=mono))
    return ds


def test_batch_256_vs_oracle(culling, big_batch):
    """Every output of every problem equals the restatement's; the batch reaches every verdict."""
    want, got = cb.Oracle()(big_batch), culling(big_batch)
    seen = np.zeros(4, int)
    for a, b in zip(want, got):
        cb.same(a, b)
        seen += np.bincount(b["verdict"], minlength=4)
    assert np.all(seen > 0), seen
    assert culling.last_ms() > 0


def test_batch_equals_one_by_one(culling, big_batch):
    ds = big_batch[:40]
    whole = culling(ds)
    for d, a in zip(ds, whole):
        cb.same(a, culling([d])[0])


def test_repeat_bit_identical(culling, big_batch):
    r0 = culling(big_batch)
    for _ in range(3):
        r = culling(big_batch)
        for a, b in zip(r0, r):
            cb.same(a, b)


def _untouched(outs):
    return all(not np.any(v) for o in outs for v in o.values() if isinstance(v, np.ndarray))


def test_error_codes(pkg, culling):
    """Every error code; nothing is written unless every problem is valid."""
    w = cb.random_world(9, 60, slots_per_kf=40)
    base = w.problem(list(range(1, 40)))
    good = w.problem(list(range(40, 60)))
    BAD, CAP = pkg.ERR_BAD_ARG, pkg.ERR_CAPACITY

    def rc_of(h, **kw):
        d = dict(base)
        d.update(kw)
        rc, outs = h.raw([good, d])
        assert _untouched(outs) and all(o["n_culled"] == 0 for o in outs), kw.keys()
        return rc

    assert culling.raw([])[0] == BAD                                            # batch < 1
    oo = base["obs_off"].copy(); oo[3] = oo[2] - 1
    assert rc_of(culling, obs_off=oo) == BAD                                    # offsets that are not a CSR
    so = base["slot_off"].copy(); so[0] = 1
    assert rc_of(culling, slot_off=so) == BAD
    lk = base["local_kf"].copy(); lk[2] = 60
    assert rc_of(culling, local_kf=lk) == BAD                                   # local keyframe out of range
    lk = base["local_kf"].copy(); lk[2] = lk[1]
    assert rc_of(culling, local_kf=lk) == BAD                                   # local keyframe repeated
    ok, o0 = base["obs_kf"].copy(), base["obs_off"]
    r = next(i for i in range(len(o0) - 1) if o0[i + 1] - o0[i] >= 2)
    ok[o0[r] + 1] = ok[o0[r]]
    assert rc_of(culling, obs_kf=ok) == BAD                                     # observer repeated
    ok = base["obs_kf"].copy(); ok[0] = 60
    assert rc_of(culling, obs_kf=ok) == BAD                                     # observer out of range
    sm = base["slot_mp"].copy(); sm[0] = len(base["mp_bad"])
    assert rc_of(culling, slot_mp=sm) == BAD                                    # slot out of range
    oi = base["obs_idx"].copy(); oi[0] = -1
    assert rc_of(culling, obs_idx=oi) == BAD                                    # negative obs_idx
    loc = {int(k): l for l, k in enumerate(base["local_kf"])}
    o = next(i for i in range(len(base["obs_kf"])) if int(base["obs_kf"][i]) in loc)
    l = loc[int(base["obs_kf"][o])]
    oi = base["obs_idx"].copy(); oi[o] = base["slot_off"][l + 1] - base["slot_off"][l]
    assert rc_of(culling, obs_idx=oi) == BAD                                    # beyond a local observer's slots
    small = pkg.KeyFrameCulling(max_kf=59, max_mp=1 << 16, max_obs=1 << 19, max_local=320, max_slots=1 << 18,
                                max_batch=4)
    assert rc_of(small) == CAP                                                  # n_kf
    small = pkg.KeyFrameCulling(max_kf=512, max_mp=1 << 16, max_obs=1 << 19, max_local=320, max_slots=100,
                                max_batch=4)
    assert rc_of(small) == CAP                                                  # slots
    small = pkg.KeyFrameCulling(max_kf=512, max_mp=1 << 16, max_obs=1 << 19, max_local=320, max_slots=1 << 18,
                                max_batch=1)
    assert rc_of(small) == CAP                                                  # batch
    assert culling.raw([good, base])[0] == 0                                    # the handle stays usable
    code = ("import importlib, sys; sys.path.insert(0, %r); pkg = importlib.import_module('self_commit_orb-slam2_b200')\n"
            "try:\n    pkg.KeyFrameCulling()\nexcept pkg.B200SlamError as e:\n    print(e.code)\n") % cb.ROOT
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=300)
    assert out.stdout.strip() == str(pkg.ERR_NO_DEVICE), out.stderr              # no device


@pytest.mark.skipif(not os.path.exists(cb.ADP_LIB), reason="oracle/_ref/libadapter_culling.so not built")
@pytest.mark.parametrize("mono", [False, True])
def test_adapter_vs_reference(mono):
    """libadapter_culling.so (one device call, then the reference's SetBadFlag on the culled and deferred keyframes)
    against the reference's own KeyFrameCulling on one object graph: the culled set and order, every keyframe's bad and
    to-be-erased flags, connections, parent and children, and every point's state."""
    ref, adp = cb.Reference(), cb.Reference(adapter=True)
    rng = np.random.default_rng(8 + mono)
    w = cb.trajectory(seed=21 + mono, n_kf=140, stereo=not mono, revisit=100)
    w.not_erase[rng.random(140) < 0.1] = 1
    culled = 0
    for cur in (60, 139):
        d = w.problem(w.covisible(cur), monocular=mono)
        want, got = ref(w, d, cur), adp(w, d, cur)
        cb.same(want, got, counts=False)
        for k in ("kf_bad", "to_be_erased", "parent"):
            assert np.array_equal(want[k], got[k]), k
        assert want["erased"] == got["erased"] and want["conn"] == got["conn"] and want["children"] == got["children"]
        culled += len(want["erased"])
    w2 = cb.random_world(31 + mono, 60, stereo=not mono, odd=0.1)
    local = cb.local_list(w2, rng, 59, size=59)
    d = w2.problem(local, monocular=mono)
    want, got = ref(w2, d, 59), adp(w2, d, 59)
    cb.same(want, got, counts=False)
    for k in ("kf_bad", "to_be_erased", "parent"):
        assert np.array_equal(want[k], got[k]), k
    assert want["erased"] == got["erased"] and want["conn"] == got["conn"] and want["children"] == got["children"]
    assert culled + len(want["erased"]) > 0
