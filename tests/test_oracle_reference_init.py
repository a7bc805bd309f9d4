"""The CPU restatement of Initializer::Initialize (oracle/init.cpp) against the reference's own src/Initializer.cc,
compiled in place against refshim/refshim_cv_init.h (oracle/_ref/libref_init.so), bit for bit on every scene of
tests/synth_init.py: FindHomography / FindFundamental (score, best matrix, inlier flags), ReconstructH / ReconstructF on
the restatement's best hypotheses (return value, R21, t21, vP3D, vbTriangulated, the state left on failure), and the
end-to-end Initialize with the reference object's own mvSets (drawn by DUtils::Random after srand(0))."""
import numpy as np
import pytest

import init_binding as ib
from synth_init import CASES, synth_init

pytestmark = pytest.mark.skipif(not __import__("os").path.exists(ib.REF_LIB),
                                reason="oracle/_ref not built (make -C oracle -f init.mk init-ref)")


def same_outputs(ref, orc):
    """ref: the glue's view of the reference's arguments; orc: the restatement's result."""
    assert ref["ret"] == orc["ret"]
    assert ref["rt_state"] == orc["rt_state"]
    if orc["rt_state"] == 1:
        assert np.array_equal(ref["R21"], orc["R21"]) and np.array_equal(ref["t21"], orc["t21"])
    if orc["ret"]:
        assert np.array_equal(ref["p3d"], orc["p3d"])
        assert np.array_equal(ref["triangulated"].astype(bool), orc["triangulated"].astype(bool))
    else:  # vP3D / vbTriangulated untouched
        assert (ref["p3d"] == ib.UNTOUCHED).all() and ref["triangulated"].all()


@pytest.mark.parametrize("case", sorted(CASES))
def test_find_matches_reference(case):
    d = synth_init(**CASES[case])
    for homography in (True, False):
        score, X, inl = ib.ref_find(d, homography)
        best, oscore, oX, oinl = ib.find(d, homography)
        assert score == oscore
        assert np.array_equal(X, oX)
        assert np.array_equal(inl, oinl)


@pytest.mark.parametrize("case", sorted(CASES))
def test_reconstruct_matches_reference(case):
    d = synth_init(**CASES[case])
    for homography in (True, False):
        best, _, X, inl = ib.find(d, homography)
        if best < 0:
            continue
        same_outputs(ib.ref_reconstruct(d, homography, inl, X), ib.reconstruct(d, homography, inl, X))


@pytest.mark.parametrize("case", sorted(CASES))
def test_initialize_matches_reference(case):
    d = synth_init(**CASES[case])
    ref = ib.call_initialize(ib.REF_LIB, "ref_initialize", d)
    # the reference's draws are sets of 8 distinct indices into the compacted matches
    n = int((d["matches12"] >= 0).sum())
    assert ref["sets"].min() >= 0 and ref["sets"].max() < n
    assert all(len(set(s)) == 8 for s in ref["sets"].tolist())
    orc = ib.oracle(dict(d, sets=ref["sets"]))
    same_outputs(ref, orc)
    assert abs(float(orc["RH"]) - 0.40) > 1e-6
    assert not (np.abs(orc["parallax"].astype(np.float64) - 1.0) <= 1e-4).any()
