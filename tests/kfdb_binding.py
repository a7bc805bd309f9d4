"""ctypes bindings of the keyframe-database checkers, with the method names of pkg.KeyFrameDatabase:

  Oracle()      oracle/liborb_kfdb.so, the CPU restatement (oracle/kfdb.cpp)
  Reference()   oracle/_ref/libref_kfdb.so, the reference's own src/KeyFrameDatabase.cc on stand-in objects
  Reference(adapter=True)  oracle/_ref/libadapter_kfdb.so, the product's drop-in KeyFrameDatabase_b200.cc on the same glue

and the seeded map / query sequences the tests and tools/kfdb_time.py replay."""
import ctypes
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_LIB = os.path.join(ROOT, "oracle", "liborb_kfdb.so")
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libref_kfdb.so")
ADP_LIB = os.path.join(ROOT, "oracle", "_ref", "libadapter_kfdb.so")
ORBVOC_WORDS = 971814  # words of Vocabulary/ORBvoc.txt
vp = ctypes.c_void_p
state_dtype = np.dtype([("loop_query", "<u8"), ("loop_words", "<i4"), ("loop_score", "<f4"), ("reloc_query", "<u8"),
                        ("reloc_words", "<i4"), ("reloc_score", "<f4")])


def _p(a):
    return a.ctypes.data_as(vp)


class _CKfdb:
    def __init__(self, path, prefix, n_words):
        self.h = None
        L = ctypes.CDLL(path)
        self.L, self.pre = L, prefix
        f = self._f
        f("create").restype = vp
        f("create").argtypes = [ctypes.c_int]
        f("destroy").argtypes = [vp]
        f("add").argtypes = [vp, ctypes.c_uint64, vp, vp, ctypes.c_int]
        f("erase").argtypes = [vp, ctypes.c_uint64]
        f("clear").argtypes = [vp]
        f("size").argtypes = [vp]
        f("detect_loop").argtypes = [vp, ctypes.c_uint64, vp, vp, ctypes.c_int, vp, ctypes.c_int, ctypes.c_float, vp, vp,
                                     ctypes.c_int, vp, ctypes.c_int]
        f("detect_reloc").argtypes = [vp, ctypes.c_uint64, vp, vp, ctypes.c_int, vp, vp, ctypes.c_int, vp, ctypes.c_int]
        f("state").argtypes = [vp, ctypes.c_uint64, vp]
        self.h = f("create")(int(n_words))

    def _f(self, name):
        return getattr(self.L, self.pre + name)

    def close(self):
        if self.h:
            self._f("destroy")(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def add(self, kf_id, words, values):
        w, v = np.ascontiguousarray(words, np.uint32), np.ascontiguousarray(values, np.float64)
        if self._f("add")(self.h, int(kf_id), _p(w), _p(v), len(w)) != 0:
            raise ValueError("keyframe %d is already in the database" % kf_id)

    def erase(self, kf_id):
        self._f("erase")(self.h, int(kf_id))

    def clear(self):
        self._f("clear")(self.h)

    def size(self):
        return self._f("size")(self.h)

    @staticmethod
    def _covis(covis):
        if covis is None:
            return np.zeros((0, 10), np.uint64), np.zeros(0, np.int32)
        return np.ascontiguousarray(covis[0], np.uint64).reshape(-1, 10), np.ascontiguousarray(covis[1], np.int32)

    def _run(self, call):
        cap = self.size() + 1
        out = np.zeros(cap, np.uint64)
        n = call(out, cap)
        assert n <= cap
        return out[:n].tolist()

    def DetectLoopCandidates(self, kf_id, words, values, connected, min_score, covis=None):
        w, v = np.ascontiguousarray(words, np.uint32), np.ascontiguousarray(values, np.float64)
        conn = np.ascontiguousarray(list(connected), np.uint64)
        ci, cn = self._covis(covis)
        return self._run(lambda out, cap: self._f("detect_loop")(self.h, int(kf_id), _p(w), _p(v), len(w), _p(conn), len(conn),
                                                               float(min_score), _p(ci), _p(cn), len(cn), _p(out), cap))

    def DetectRelocalizationCandidates(self, frame_id, words, values, covis=None):
        w, v = np.ascontiguousarray(words, np.uint32), np.ascontiguousarray(values, np.float64)
        ci, cn = self._covis(covis)
        return self._run(lambda out, cap: self._f("detect_reloc")(self.h, int(frame_id), _p(w), _p(v), len(w), _p(ci), _p(cn),
                                                                len(cn), _p(out), cap))

    def keyframe_state(self, kf_id):
        s = np.zeros(1, state_dtype)
        self._f("state")(self.h, int(kf_id), _p(s))
        s = s[0]
        return (int(s["loop_query"]), int(s["loop_words"]), float(s["loop_score"]), int(s["reloc_query"]),
                int(s["reloc_words"]), float(s["reloc_score"]))


class Oracle(_CKfdb):
    def __init__(self, n_words):
        super().__init__(ORACLE_LIB, "orc_kfdb_", n_words)
        self.L.orc_kfdb_counters.argtypes = [vp, vp, vp]

    def counters(self):
        """(covisibility neighbours whose score this query had not written, best keyframes dropped by the dedupe)"""
        a, b = ctypes.c_longlong(0), ctypes.c_longlong(0)
        self.L.orc_kfdb_counters(self.h, ctypes.byref(a), ctypes.byref(b))
        return a.value, b.value


class Reference(_CKfdb):
    def __init__(self, n_words, adapter=False):
        super().__init__(ADP_LIB if adapter else REF_LIB, "adp_kfdb_" if adapter else "ref_kfdb_", n_words)
        self._f("counters").argtypes = [vp, vp]

    def stale_reads(self):
        """(reads of mLoopScore, of mRelocScore) that the running query had not written, since the library was loaded"""
        a, b = ctypes.c_longlong(0), ctypes.c_longlong(0)
        self._f("counters")(ctypes.byref(a), ctypes.byref(b))
        return a.value, b.value


def l1_score_fn(path, name):
    L = ctypes.CDLL(path)
    f = getattr(L, name)
    f.restype = ctypes.c_double
    f.argtypes = [vp, vp, ctypes.c_int, vp, vp, ctypes.c_int]

    def score(a, b):
        aw, av = np.ascontiguousarray(a[0], np.uint32), np.ascontiguousarray(a[1], np.float64)
        bw, bv = np.ascontiguousarray(b[0], np.uint32), np.ascontiguousarray(b[1], np.float64)
        return f(_p(aw), _p(av), len(aw), _p(bw), _p(bv), len(bw))
    return score


# ------------------------------------------------------------------------------------------------ seeded sequences
def _normalised(rng, words):
    v = rng.random(len(words)) + 0.05
    return words.astype(np.uint32), v / v.sum()


class MapModel:
    """A trajectory through `n_places` places that comes back to them (revisits): keyframe i sees place i % n_places with
    70 % of that place's words plus noise words, word ids Zipf-distributed over `n_words`.  Keyframe ids are consecutive.
    The covisibility of keyframe i is up to 10 of its trajectory neighbours i +- 1, +- 2 ... and its previous visit of the
    place, whatever their state (erased, not added yet: neighbours outside the database)."""

    def __init__(self, seed, n_words=20000, n_places=40, place_words=300, noise=60, zipf_shift=10.0):
        self.rng = np.random.default_rng(seed)
        self.n_words, self.n_places, self.noise = n_words, n_places, noise
        p = 1.0 / (np.arange(n_words) + zipf_shift)
        self.pz = p / p.sum()
        self.places = [np.unique(self.rng.choice(n_words, place_words, p=self.pz)) for _ in range(n_places)]

    def keyframe(self, i):
        pw = self.places[i % self.n_places]
        keep = pw[self.rng.random(len(pw)) < 0.7]
        words = np.unique(np.concatenate([keep, self.rng.choice(self.n_words, self.noise, p=self.pz)]))
        return _normalised(self.rng, words)

    def covis(self, n_rows, n_neigh=None):
        ids = np.zeros((n_rows, 10), np.uint64)
        n = np.zeros(n_rows, np.int32)
        for i in range(n_rows):
            cand = []
            for d in range(1, 8):
                cand += [i - d, i + d]
            cand.insert(3, i - self.n_places)
            cand = [c for c in cand if c >= 0][:10 if n_neigh is None else n_neigh]
            k = int(self.rng.integers(0, len(cand) + 1)) if n_neigh is None else len(cand)
            n[i] = k
            ids[i, :k] = cand[:k]
        return ids, n


def zipf_map(seed, n_kf, words_per_kf, n_words=ORBVOC_WORDS, n_places=None):
    """Keyframes of about `words_per_kf` distinct Zipf-distributed words over a vocabulary of `n_words` (the real one's
    size by default), grouped in places of consecutive keyframes that share most of their words."""
    rng = np.random.default_rng(seed)
    p = 1.0 / (np.arange(n_words) + 50.0)
    p /= p.sum()
    n_places = n_places or max(1, n_kf // 8)
    kfs = []
    place = None
    for i in range(n_kf):
        if i % (n_kf // n_places or 1) == 0:
            place = np.unique(rng.choice(n_words, int(words_per_kf * 1.3), p=p))
        keep = place[rng.random(len(place)) < 0.75]
        words = np.unique(np.concatenate([keep, rng.choice(n_words, words_per_kf // 5, p=p)]))
        kfs.append(_normalised(rng, words))
    return kfs
