"""Direct tests of csrc/chol.cuh, the tiled envelope Cholesky, substitutions, tile envelope and deterministic sums that the
global BA (gba.cu, 6-scalar blocks) and the essential graph (essential.cu, 7-scalar Sim3 blocks) solve their reduced
systems with.  The solvers' own tests only see it through an LM loop, which rejects a bad step and carries on, so here
it is driven through a test-only harness (tests/cpp/chol_harness.cu) and held to a high-precision reference.

The harness is compiled twice with the product's flags (build.py): as gba.o is, with FMA contraction, and as essential.o
is, with --fmad=false.  Every GPU test runs against both builds.  The envelope tests are host code and need nvcc only.

Error bars (u = 2^-53, the unit roundoff of FP64):
- Factor (backward) error.  Every entry of L L^T is a dot product of at most n terms, and the textbook Cholesky bound
  is |L^ L^T - H| <= gamma_{n+1} |L^| |L^T|, with gamma_k = k u / (1 - k u).  For a positive definite H, |L^| |L^T| is at
  most ||H||_max entrywise (Cauchy-Schwarz on the rows of L), so ||L^ L^T - H||_max / ||H||_max <= 4 n u keeps a
  factor of about 4 for the DMMA accumulation order and the explicit diagonal inverses.  L^'s diagonal tiles are
  Linv_KK^-1, formed in long double: the panel L_IK = A_IK Linv_KK^T uses Linv, so this is the factor the solve uses.
- Forward error.  A backward error of 4 n u ||H|| gives ||x^ - x*|| / ||x*|| <= 4 n kappa(H) u to first order, with
  kappa = kappa_inf(H) = ||H||_inf ||H^-1||_inf.  In the well-conditioned cases this bar is at most 1e-10, so one FP32
  operation (about 1e-7 relative) anywhere in the chain fails it.
- The reference x* is a float64 Cholesky solve (scipy) refined twice with the residual b - H x formed in long double, so
  it is accurate to about kappa u^2 + u_longdouble, far below these bars.

The ill-conditioned cases (pose graphs with a weak scale column or a weak gauge, kappa 1e6 to 1e13) are held to the
same forward bar; their backward error is printed (run pytest with -s) next to kappa(L_KK) n u, which is what the
explicit-inverse panel can add to it."""
import ctypes
import importlib.util
import math
import os
import shutil
import subprocess
import zlib

import numpy as np
import pytest
import scipy.linalg as sla
import scipy.sparse as sps
import scipy.sparse.linalg as spla

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG_DIR = os.path.join(ROOT, "self_commit_orb-slam2_b200")
HARNESS = os.path.join(ROOT, "tests", "cpp", "chol_harness.cu")
TS = 64
U = 2.0 ** -53
FLAG_POISON, FLAG_KEEP_FAIL = 1, 2
GBA_CAP, EG_CAP = (2048, 6), (4096, 7)  # poses x block size of the two solvers' largest systems
# the harness is built with the flags of each including object: gba.o contracts FMAs, essential.o does not (NO_FMAD)
BUILDS = {"gba": "gba.cu", "essential": "essential.cu"}


def _product_build():
    spec = importlib.util.spec_from_file_location("_chol_product_build", os.path.join(PKG_DIR, "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _nvcc():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    return nvcc if os.path.exists(nvcc) else shutil.which("nvcc")


# ================================================================================================ harness binding
class Harness:
    def __init__(self, path, name):
        self.name = name
        lib = self.lib = ctypes.CDLL(path)
        P, I, LL = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong
        lib.chol_envelope.restype = LL
        lib.chol_envelope.argtypes = [P, I, I, P, P, P, P, LL, P]
        lib.chol_ctx_create.restype = P
        lib.chol_ctx_create.argtypes = [LL, I]
        lib.chol_ctx_destroy.restype = None
        lib.chol_ctx_destroy.argtypes = [P]
        lib.chol_ctx_solve.restype = I
        lib.chol_ctx_solve.argtypes = [P, I, I, P, LL, P, P, P, P, I, P, P, P, P]
        lib.chol_reduce.restype = I
        lib.chol_reduce.argtypes = [I, P, LL, P]

    def envelope(self, env_blk, B):
        env_blk = np.ascontiguousarray(env_blk, dtype=np.int32)
        nT = -(-len(env_blk) * B // TS)
        envT, off = np.zeros(nT, np.int32), np.zeros(nT + 1, np.int64)
        row_off, n_rows = np.zeros(nT + 1, np.int32), ctypes.c_longlong(0)
        cap = nT * (nT - 1) // 2
        rows = np.zeros(max(cap, 1), np.int32)
        n_tiles = self.lib.chol_envelope(env_blk.ctypes.data, len(env_blk), B, envT.ctypes.data, off.ctypes.data,
                                         row_off.ctypes.data, rows.ctypes.data, cap, ctypes.byref(n_rows))
        assert n_tiles >= 0
        return n_tiles, envT, off, row_off, rows[:n_rows.value]

    def reduce(self, op, v):
        v = np.ascontiguousarray(v, dtype=np.float64)
        out = np.zeros(1)
        assert self.lib.chol_reduce(op, v.ctypes.data, len(v), out.ctypes.data) == 0
        return out[0]

    def context(self, max_tiles, max_np_pad):
        return Context(self, max_tiles, max_np_pad)


class Context:
    def __init__(self, h, max_tiles, max_np_pad):
        self.h = h
        self.p = h.lib.chol_ctx_create(max_tiles, max_np_pad)
        assert self.p, "chol_ctx_create failed"

    def close(self):
        if self.p:
            self.h.lib.chol_ctx_destroy(self.p)
            self.p = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def solve_raw(self, s, b, flags=0, env_blk=None, readback=True):
        """(return code, x_out, fail, tiles, linv) for System s, optionally over a different declared envelope."""
        env = np.ascontiguousarray(s.env_blk if env_blk is None else env_blk, dtype=np.int32)
        n_tiles, envT, _, _, _ = self.h.envelope(env, s.B)
        nT = len(envT)
        x = np.zeros(nT * TS)
        fail = np.zeros(1, np.int32)
        tiles = np.zeros((n_tiles, TS, TS)) if readback else None
        linv = np.zeros((nT, TS, TS)) if readback else None
        rc = self.h.lib.chol_ctx_solve(self.p, s.n_blk, s.B, env.ctypes.data, len(s.row), s.row.ctypes.data,
                                       s.col.ctypes.data, s.val.ctypes.data, np.ascontiguousarray(b).ctypes.data, flags,
                                       x.ctypes.data, fail.ctypes.data, tiles.ctypes.data if readback else None,
                                       linv.ctypes.data if readback else None)
        return rc, x, int(fail[0]), tiles, linv

    def solve(self, s, b, flags=0, env_blk=None, readback=True):
        rc, x, fail, tiles, linv = self.solve_raw(s, b, flags, env_blk, readback)
        assert rc == 0, "chol_ctx_solve returned %d" % rc
        return x, fail, tiles, linv


@pytest.fixture(scope="module")
def harness_libs(tmp_path_factory):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    bld = _product_build()
    out = tmp_path_factory.mktemp("chol_harness")
    procs = {}
    for name in BUILDS:
        so = str(out / ("libchol_%s.so" % name))
        cmd = [nvcc] + bld.NVCC_FLAGS + (["--fmad=false"] if BUILDS[name] in bld.NO_FMAD else []) + [
            "-shared", "-I", os.path.join(PKG_DIR, "csrc"), "-o", so, HARNESS]
        procs[name] = (so, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT))
    libs = {}
    for name, (so, p) in procs.items():
        log, _ = p.communicate()
        assert p.returncode == 0, log.decode()
        libs[name] = so
    return libs


@pytest.fixture(scope="module")
def host_harness(harness_libs):
    return Harness(harness_libs["gba"], "gba")


@pytest.fixture(scope="module", params=[pytest.param(b, marks=pytest.mark.gpu) for b in BUILDS])
def chol(request, harness_libs):
    return Harness(harness_libs[request.param], request.param)


# ================================================================================================ tile envelope
def envelope_restated(env_blk, B):
    """tile_envelope's comment, restated: envT[T] is the first tile column any scalar row of tile row T reaches, off is
    the prefix count of stored tiles, and rows[rowOff[K]:rowOff[K+1]] are the tile rows I > K with envT[I] <= K."""
    env_blk = np.asarray(env_blk, np.int64)
    n = len(env_blk) * B
    nT = -(-n // TS)
    first_col = np.repeat(env_blk * B, B)  # per scalar row
    envT = np.array([first_col[T * TS:min(n, (T + 1) * TS)].min() // TS for T in range(nT)], np.int64)
    off = np.concatenate([[0], np.cumsum(np.arange(nT) - envT + 1)])
    rows = [[I for I in range(K + 1, nT) if envT[I] <= K] for K in range(nT)]
    row_off = np.concatenate([[0], np.cumsum([len(r) for r in rows])])
    return envT, off, row_off, np.array([I for r in rows for I in r], np.int64)


def boundary_profile(n_blk, B, rng):
    """Block rows reaching back to a block that starts exactly at a tile boundary, or to the block holding the scalar
    just before one."""
    targets = set()
    for k in range(1, -(-n_blk * B // TS)):
        targets.add(-(-k * TS // B))         # first block starting at or after the boundary
        targets.add((k * TS - 1) // B)       # block holding the last scalar before it
    targets = sorted(t for t in targets if t < n_blk) or [0]
    env = np.arange(n_blk)
    for i in range(n_blk):
        ok = [t for t in targets if t <= i]
        if ok and rng.random() < 0.5:
            env[i] = ok[int(rng.integers(len(ok)))]
    return env


def envelope_cases():
    rng = np.random.default_rng(1)
    cases = []
    for B in (1, 3, 6, 7, 9, 64, 100):
        for n_blk in sorted({1, 2, 3, max(1, TS // B), TS // B + 1, 2 * TS // B + 1, 11, 50, 200}):
            cases.append((B, "random", np.array([int(rng.integers(0, i + 1)) for i in range(n_blk)])))
            cases.append((B, "boundary", boundary_profile(n_blk, B, rng)))
            cases.append((B, "diagonal", np.arange(n_blk)))
    for n_blk, B in (GBA_CAP, EG_CAP):
        chain = np.maximum(np.arange(n_blk) - 1, 0)
        for i in rng.choice(n_blk, 4, replace=False):
            chain[i] = 0 if rng.random() < 0.5 else int(rng.integers(0, i + 1))
        cases.append((B, "capacity-pose-graph", chain))
        cases.append((B, "capacity-boundary", boundary_profile(n_blk, B, rng)))
    return cases


def test_tile_envelope_matches_its_definition(host_harness):
    for B, kind, env in envelope_cases():
        n_tiles, envT, off, row_off, rows = host_harness.envelope(env, B)
        want = envelope_restated(env, B)
        what = "B=%d n_blk=%d %s" % (B, len(env), kind)
        assert np.array_equal(envT, want[0]), what
        assert np.array_equal(off, want[1]) and n_tiles == want[1][-1], what
        assert np.array_equal(row_off, want[2]), what
        assert np.array_equal(rows, want[3]), what


def test_tile_envelope_straddling_blocks(host_harness):
    """A block that straddles a tile boundary pulls the next tile row's envelope back: B = 6, block 10 holds scalars
    60..65, so only its reach decides tile row 1."""
    env = np.arange(22)
    env[10] = 0
    _, envT, _, _, _ = host_harness.envelope(env, 6)
    assert envT.tolist() == [0, 0, 1]  # block 21 (scalars 126..131) starts in tile column 1
    env = np.arange(22)
    env[11] = 0  # block 11 starts at scalar 66: tile row 1 only
    _, envT, _, row_off, rows = host_harness.envelope(env, 6)
    assert envT.tolist() == [0, 0, 1] and rows.tolist() == [1, 2] and row_off.tolist() == [0, 1, 2, 2]


# ================================================================================================ test systems
class System:
    """A symmetric positive definite (or deliberately not) system over nBlk blocks of B scalars: the lower-triangle COO
    entries that go to the harness, H as a scipy CSR matrix, and the block envelope."""

    def __init__(self, B, n_blk, H, env_blk):
        self.B, self.n_blk, self.n = B, n_blk, B * n_blk
        self.H = sps.csr_matrix(H)
        self.env_blk = np.asarray(env_blk, np.int32)
        low = sps.tril(self.H).tocoo()
        self.row, self.col = low.row.astype(np.int32), low.col.astype(np.int32)
        self.val = np.ascontiguousarray(low.data, dtype=np.float64)

    def dense(self):
        return self.H.toarray()

    def first_col(self):
        """per scalar row: first column holding a nonzero of H (its own index for an empty row)"""
        low = sps.tril(self.H).tocsr()
        first = np.arange(self.n)
        for r in range(self.n):
            cols = low.indices[low.indptr[r]:low.indptr[r + 1]]
            cols = cols[low.data[low.indptr[r]:low.indptr[r + 1]] != 0]
            if len(cols):
                first[r] = cols.min()
        return first


def shape_edges(shape, n_blk, rng):
    """(i, j), i > j, block pairs of one envelope shape"""
    chain = [(i, i - 1) for i in range(1, n_blk)]
    if shape == "blockdiag":
        return []
    if shape == "chain":
        return chain
    if shape == "loops":  # odometry band plus 1-3 closures to block 0 and to mid-map blocks
        e = list(chain)
        for k in range(int(rng.integers(1, 4))):
            i = int(rng.integers(max(2, n_blk // 2), n_blk)) if n_blk > 2 else n_blk - 1
            j = 0 if k == 0 else int(rng.integers(0, max(1, i // 2)))
            if i > j:
                e.append((i, j))
        return e
    if shape == "posegraph":  # band of short covisibility links, three closures to block 0 and two to mid-map blocks
        e = list(chain) + [(i, i - int(rng.integers(2, 6))) for i in range(6, n_blk) if rng.random() < 0.3]
        for i in rng.choice(np.arange(n_blk // 2, n_blk), 3, replace=False):
            e.append((int(i), 0))
        for i in rng.choice(np.arange(n_blk // 2, n_blk), 2, replace=False):
            e.append((int(i), int(rng.integers(n_blk // 4, n_blk // 2))))
        return e
    if shape == "arrow":
        return chain + [(i, 0) for i in range(2, n_blk)]
    if shape == "dense":
        return [(i, j) for i in range(n_blk) for j in range(i)]
    if shape == "random":
        e = []
        for i in range(1, n_blk):
            j = int(rng.integers(0, i + 1))
            if j < i:
                e.append((i, j))
        return e
    raise ValueError(shape)


def env_of(edges, n_blk):
    env = np.arange(n_blk)
    for i, j in edges:
        env[i] = min(env[i], j)
    return env


def assemble(B, n_blk, edges, jac, unary):
    """H = sum over edges of J_e^T J_e with J_e = [jac_i, jac_j] on blocks (i, j), plus unary J^T J per block"""
    n = B * n_blk
    rows, cols, vals = [], [], []
    bi = np.arange(B)

    def put(I, J, M):
        rows.append(np.repeat(I * B + bi, B))
        cols.append(np.tile(J * B + bi, B))
        vals.append(M.ravel())
    for (i, j) in edges:
        Ji, Jj = jac()
        put(i, i, Ji.T @ Ji)
        put(j, j, Jj.T @ Jj)
        put(i, j, Ji.T @ Jj)
        put(j, i, Jj.T @ Ji)
    for i, A in unary:
        put(i, i, A.T @ A)
    if not rows:
        return sps.csr_matrix((n, n))
    return sps.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(n, n))


def well_conditioned(B, n_blk, shape, seed):
    """H = sum J_e^T J_e + unary terms + a diagonal that makes H strictly diagonally dominant with a margin sized so that
    4 n kappa_inf u <= 1e-10 (Varah: ||H^-1||_inf <= 1 / min_i (h_ii - sum_j!=i |h_ij|))"""
    rng = np.random.default_rng(seed)
    edges = shape_edges(shape, n_blk, rng)
    G = assemble(B, n_blk, edges, lambda: (rng.normal(size=(B, B)), rng.normal(size=(B, B))),
                 [(i, rng.normal(size=(B, B))) for i in range(n_blk)])
    n = B * n_blk
    R = np.asarray(abs(G).sum(axis=1)).ravel()
    kappa_target = min(1e3, 1e-10 / (4 * n * U))
    beta = 2.0 / (kappa_target - 1)  # kappa_inf <= (2 Rmax + c) / c with c = beta Rmax
    H = G + sps.diags(R + beta * R.max())
    return System(B, n_blk, H, env_of(edges, n_blk))


def pose_graph(B, n_blk, shape, seed, eps=1.0, anchor=1.0, lam=1e-16):
    """Relative-pose edges r = A (x_j - x_i) with a well-conditioned A and the last column scaled by eps (the weak
    scale of a Sim3 pose graph), an anchor of strength `anchor` on block 0 (the gauge), and LM's lambda on the
    diagonal"""
    rng = np.random.default_rng(seed)
    S = np.ones(B)
    S[-1] = eps

    def orth():
        q, _ = np.linalg.qr(rng.normal(size=(B, B)))
        return q * rng.uniform(1, 2, B)

    def jac():
        A = orth() * S
        return -A, A
    edges = shape_edges(shape, n_blk, rng)
    G = assemble(B, n_blk, edges, jac, [(0, orth() * S * anchor)])
    H = G + lam * sps.identity(B * n_blk)
    return System(B, n_blk, H, env_of(edges, n_blk))


# ================================================================================================ reference
def kappa_inf(s):
    if s.n <= 4500:
        Hd = s.dense()
        return float(np.linalg.norm(Hd, np.inf) * np.linalg.norm(np.linalg.inv(Hd), np.inf))
    # Varah's bound for the diagonally dominant large cases
    A = abs(s.H)
    d = A.diagonal()
    margin = 2 * d - np.asarray(A.sum(axis=1)).ravel()
    assert margin.min() > 0
    return float(np.asarray(A.sum(axis=1)).max() / margin.min())


def residual_ld(s, x):
    """b - H x is formed by the caller; this is H x in long double, row by row over the CSR rows"""
    H = s.H
    prod = H.data.astype(np.longdouble) * np.asarray(x, np.longdouble)[H.indices]
    out = np.zeros(s.n, np.longdouble)
    nz = np.diff(H.indptr) > 0
    out[nz] = np.add.reduceat(prod, H.indptr[:-1][nz])
    return out


def reference_solve(s, b):
    """x* in long double: a float64 Cholesky (dense) or LU (sparse, large) solve, refined twice with long-double
    residuals"""
    if s.n <= 4500:
        fac = sla.cho_factor(s.dense(), lower=True)
        solve = lambda r: sla.cho_solve(fac, r)
    else:
        lu = spla.splu(s.H.tocsc())
        solve = lu.solve
    x = solve(b).astype(np.longdouble)
    bl = b.astype(np.longdouble)
    for _ in range(2):
        r = bl - residual_ld(s, x)
        x = x + solve(r.astype(np.float64)).astype(np.longdouble)
    return x


def tri_inv_ld(Li):
    """inverse of a lower-triangular tile in long double (column-vectorised forward substitution)"""
    Li = Li.astype(np.longdouble)
    m = Li.shape[0]
    X = np.zeros((m, m), np.longdouble)
    for r in range(m):
        acc = -(Li[r, :r] @ X[:r, :])
        acc[r] += 1
        X[r, :] = acc / Li[r, r]
    return X


def factor_tiles_ld(s, envT, off, tiles, linv):
    """L^ as a dict (I, K) -> 64 x 64 long-double tile over the stored envelope, padding rows / columns removed by the
    caller's mask: off-diagonal tiles as stored, diagonal tiles Linv^-1"""
    L = {}
    for I in range(len(envT)):
        for K in range(envT[I], I + 1):
            L[(I, K)] = tri_inv_ld(linv[K]) if K == I else tiles[off[I] + K - envT[I]].astype(np.longdouble)
    return L


def tile_products(envT):
    return sum(J - max(envT[I], envT[J]) + 1 for I in range(len(envT)) for J in range(envT[I], I + 1))


def backward_error(s, envT, off, tiles, linv):
    """||L^ L^T - H||_max / ||H||_max over the lower stored envelope (tile products in long double), and
    max_K kappa_2(L^_KK)"""
    nT = len(envT)
    L = factor_tiles_ld(s, envT, off, tiles, linv)
    Hd = s.H.tocsr()
    worst = 0.0
    for I in range(nT):
        r0, r1 = I * TS, min(s.n, (I + 1) * TS)
        for J in range(envT[I], I + 1):
            c0, c1 = J * TS, min(s.n, (J + 1) * TS)
            acc = np.zeros((TS, TS), np.longdouble)
            for K in range(max(envT[I], envT[J]), J + 1):
                acc += L[(I, K)] @ L[(J, K)].T
            E = acc[:r1 - r0, :c1 - c0] - Hd[r0:r1, c0:c1].toarray().astype(np.longdouble)
            if I == J:
                E = np.tril(E)
            worst = max(worst, float(abs(E).max()))
    hmax = float(abs(s.H).max())
    kL = 0.0
    for K in range(nT):
        m = min(s.n, (K + 1) * TS) - K * TS
        kL = max(kL, float(np.linalg.cond(L[(K, K)][:m, :m].astype(np.float64))))
    return worst / hmax, kL


def check_exact_zeros(s, envT, off, tiles, x):
    """stored tiles are exactly 0 left of each scalar row's first nonzero of H (fill-in stays inside the row profile;
    on diagonal tiles the stored Schur complement obeys the same rule), the padded rows of off-diagonal tiles stay 0,
    and x_out is 0 past n"""
    first = s.first_col()
    nT = len(envT)
    for I in range(nT):
        for K in range(envT[I], I + 1):
            t = tiles[off[I] + K - envT[I]]
            r = np.arange(I * TS, (I + 1) * TS)
            c = np.arange(K * TS, (K + 1) * TS)
            real = r < s.n
            left = c[None, :] < np.where(real, first[np.minimum(r, s.n - 1)], 0)[:, None]
            assert not t[left].any(), "tile (%d, %d): nonzero left of the row profile" % (I, K)
            if K < I:
                assert not t[~real].any(), "tile (%d, %d): nonzero padding row" % (I, K)
    assert not x[s.n:].any(), "x_out past n"


# ================================================================================================ factor / solve cases
# (id, builder): every shape at and around tile boundaries, exact tile multiples and the two solvers' capacities.
WELL = [
    ("B6-n6-one-block", lambda: well_conditioned(6, 1, "blockdiag", 1)),
    ("B7-n7-one-block", lambda: well_conditioned(7, 1, "blockdiag", 2)),
    ("B6-n60-chain", lambda: well_conditioned(6, 10, "chain", 3)),
    ("B7-n63-chain", lambda: well_conditioned(7, 9, "chain", 4)),
    ("B6-n66-loops", lambda: well_conditioned(6, 11, "loops", 5)),
    ("B7-n70-dense", lambda: well_conditioned(7, 10, "dense", 6)),
    ("B6-n126-arrow", lambda: well_conditioned(6, 21, "arrow", 7)),
    ("B7-n126-random", lambda: well_conditioned(7, 18, "random", 8)),
    ("B6-n132-random", lambda: well_conditioned(6, 22, "random", 9)),
    ("B6-n132-loops", lambda: well_conditioned(6, 22, "loops", 10)),
    ("B6-n192-dense", lambda: well_conditioned(6, 32, "dense", 11)),
    ("B6-n192-blockdiag", lambda: well_conditioned(6, 32, "blockdiag", 12)),
    ("B6-n384-loops", lambda: well_conditioned(6, 64, "loops", 13)),
    ("B6-n384-chain", lambda: well_conditioned(6, 64, "chain", 14)),
    ("B7-n448-loops", lambda: well_conditioned(7, 64, "loops", 15)),
    ("B7-n448-dense", lambda: well_conditioned(7, 64, "dense", 16)),
    ("B7-n448-blockdiag", lambda: well_conditioned(7, 64, "blockdiag", 17)),
    ("B1-n130-random", lambda: well_conditioned(1, 130, "random", 18)),
    ("B64-n192-dense", lambda: well_conditioned(64, 3, "dense", 19)),
    ("B7-n4095-arrow", lambda: well_conditioned(7, 585, "arrow", 20)),
    ("B6-n12288-posegraph", lambda: well_conditioned(6, GBA_CAP[0], "posegraph", 21)),
    ("B7-n28672-posegraph", lambda: well_conditioned(7, EG_CAP[0], "posegraph", 22)),
]
ILL = [
    ("B7-n126-loops-scale1e-2", lambda: pose_graph(7, 18, "loops", 31, eps=1e-2)),
    ("B7-n448-loops-scale1e-3", lambda: pose_graph(7, 64, "loops", 32, eps=1e-3)),
    ("B7-n448-chain-scale1e-4", lambda: pose_graph(7, 64, "chain", 33, eps=1e-4)),
    ("B7-n448-loops-scale1e-2-gauge1e-3", lambda: pose_graph(7, 64, "loops", 34, eps=1e-2, anchor=1e-3)),
    ("B6-n384-loops-gauge1e-4", lambda: pose_graph(6, 64, "loops", 35, anchor=1e-4)),
    ("B7-n196-posegraph-scale1e-3", lambda: pose_graph(7, 28, "posegraph", 36, eps=1e-3)),
]
BACKWARD_MAX_PRODUCTS = 3000  # the long-double factor check costs about 1 ms per 64 x 64 tile product; skipped above

_cache = {}


def case(cid, builder):
    """System, right-hand side, x*, kappa: built once per module, shared by both builds"""
    if cid not in _cache:
        s = builder()
        b = np.random.default_rng(zlib.crc32(cid.encode())).normal(size=s.n)
        _cache[cid] = (s, b, reference_solve(s, b), kappa_inf(s))
    return _cache[cid]


def context_for(chol, s):
    n_tiles, envT, _, _, _ = chol.envelope(s.env_blk, s.B)
    return chol.context(n_tiles, len(envT) * TS)


def run_case(chol, cid, builder, well):
    s, b, xs, kappa = case(cid, builder)
    with context_for(chol, s) as ctx:
        x, fail, tiles, linv = ctx.solve(s, b)
    assert fail == 0, cid
    n_tiles, envT, off, _, _ = chol.envelope(s.env_blk, s.B)
    check_exact_zeros(s, envT, off, tiles, x)
    fwd = float(np.max(abs(x[:s.n].astype(np.longdouble) - xs)) / np.max(abs(xs)))
    bar_f = 4 * s.n * kappa * U
    checked = tile_products(envT) <= BACKWARD_MAX_PRODUCTS
    bwd, kL = backward_error(s, envT, off, tiles, linv) if checked else (float("nan"), float("nan"))
    print("CHOLROW | %s | %s | n=%d | B=%d | kappa=%.2e | factor=%.2e | factor bar=%.2e | kappa(L_KK)=%.2e | forward=%.2e | "
          "forward bar=%.2e" % (chol.name, cid, s.n, s.B, kappa, bwd, 4 * s.n * U, kL, fwd, bar_f))
    if well:
        assert bar_f <= 1e-10, (cid, bar_f)
        if checked:
            assert bwd <= 4 * s.n * U, (cid, bwd)
    assert fwd <= bar_f, (cid, fwd, bar_f)
    return s, b, x, tiles, linv


@pytest.mark.parametrize("cid,builder", WELL, ids=[c[0] for c in WELL])
def test_factor_solve_well_conditioned(chol, cid, builder):
    run_case(chol, cid, builder, well=True)


@pytest.mark.parametrize("cid,builder", ILL, ids=[c[0] for c in ILL])
def test_factor_solve_ill_conditioned(chol, cid, builder):
    s, _, _, kappa = case(cid, builder)
    assert 1e6 <= kappa <= 1e14, kappa
    run_case(chol, cid, builder, well=False)


@pytest.mark.parametrize("cid", ["B6-n132-loops", "B7-n448-loops", "B6-n192-blockdiag"])
def test_wider_envelope_gives_the_same_answer(chol, cid):
    """Lowering envBlk entries without changing H adds tiles and tile columns that hold only zeros: they stay exactly 0
    in L (check_exact_zeros reads the profile from H, not from the envelope) and x does not change by a bit."""
    builder = dict(WELL)[cid]
    s, b, xs, kappa = case(cid, builder)
    rng = np.random.default_rng(5)
    wide = s.env_blk.copy()
    for i in rng.choice(s.n_blk, max(1, s.n_blk // 4), replace=False):
        wide[i] = int(rng.integers(0, wide[i] + 1))
    wide[-1] = 0
    assert (wide < s.env_blk).any()
    n_tiles, envT, off, _, _ = chol.envelope(wide, s.B)
    with chol.context(n_tiles, len(envT) * TS) as ctx:
        x_n, f_n, _, _ = ctx.solve(s, b)
        x_w, f_w, tiles, _ = ctx.solve(s, b, env_blk=wide)
    assert f_n == 0 and f_w == 0
    check_exact_zeros(s, envT, off, tiles, x_w)
    fwd = float(np.max(abs(x_w[:s.n].astype(np.longdouble) - xs)) / np.max(abs(xs)))
    assert fwd <= 4 * s.n * kappa * U
    assert np.array_equal(x_w, x_n)


# ================================================================================================ determinism and state
def test_repeat_and_poison_are_bit_identical(chol):
    s, b, _, _ = case("B7-n448-loops", dict(WELL)["B7-n448-loops"])
    with context_for(chol, s) as ctx:
        first = ctx.solve(s, b)
        again = ctx.solve(s, b)
        poisoned = ctx.solve(s, b, flags=FLAG_POISON)
    for other in (again, poisoned):
        assert other[1] == 0
        for k in (0, 2, 3):  # x_out, tiles, linv
            assert np.array_equal(first[k], other[k])


def test_large_then_small_matches_a_fresh_context(chol):
    big, bb, _, _ = case("B6-n384-loops", dict(WELL)["B6-n384-loops"])
    small, sb, _, _ = case("B6-n66-loops", dict(WELL)["B6-n66-loops"])
    with context_for(chol, small) as fresh:
        want = fresh.solve(small, sb)
    with context_for(chol, big) as ctx:
        ctx.solve(big, bb)
        got = ctx.solve(small, sb)
    for k in (0, 2, 3):
        assert np.array_equal(want[k], got[k])


def test_entries_outside_the_envelope_are_rejected_on_the_host(chol):
    s, b, _, _ = case("B6-n384-chain", dict(WELL)["B6-n384-chain"])
    with context_for(chol, s) as ctx:
        bad = System(s.B, s.n_blk, s.H, s.env_blk)
        assert chol.envelope(s.env_blk, s.B)[1][2] > 0  # tile row 2 does not reach tile column 0
        bad.row = np.append(bad.row, np.int32(2 * TS)).astype(np.int32)
        bad.col = np.append(bad.col, np.int32(0)).astype(np.int32)
        bad.val = np.append(bad.val, 1.0)
        assert ctx.solve_raw(bad, b)[0] == 1
        up = System(s.B, s.n_blk, s.H, s.env_blk)
        up.row, up.col = up.col.copy(), up.row.copy()  # upper triangle
        assert ctx.solve_raw(up, b)[0] == 1
        assert ctx.solve(s, b)[1] == 0  # the context is still usable


# ================================================================================================ failure
def numpy_says_indefinite(Hd):
    try:
        L = np.linalg.cholesky(Hd)
    except np.linalg.LinAlgError:
        return True
    return not np.all(np.isfinite(L))


def failing_systems():
    base = well_conditioned(6, 22, "loops", 41)  # n = 132: three tiles, block 10 straddles rows 60..65
    Hd = base.dense()
    out = []

    def with_diag(r, v):
        H = Hd.copy()
        H[r, r] = v
        return H
    out.append(("negative pivot, first tile", with_diag(3, -1.0)))
    out.append(("negative pivot, block straddling a tile boundary", with_diag(65, -Hd[65, 65])))
    out.append(("negative pivot, last real row", with_diag(base.n - 1, -1e-3)))
    H = Hd.copy()
    H[70, :] = 0
    H[:, 70] = 0
    out.append(("zero row", H))
    H = Hd.copy()
    r = 64 + int(np.argmax(Hd[64:128, 0:64].any(axis=1)))
    c = int(np.flatnonzero(Hd[r, :64])[0])
    H[r, c] = H[c, r] = np.nan
    out.append(("NaN in an off-diagonal tile", H))
    sys_ = [(name, System(base.B, base.n_blk, M, base.env_blk)) for name, M in out]
    # Schur complement indefinite: [[A, C], [C^T, D]] with A = 2 I (tile 0), C = 3 Q (Q orthonormal columns) and
    # D = C^T A^-1 C + M: D is positive definite (eigenvalues 3.5 .. 5.5), its Schur complement M has eigenvalue -1
    rng = np.random.default_rng(42)
    m = 62
    Q, _ = np.linalg.qr(rng.normal(size=(64, m)))
    R, _ = np.linalg.qr(rng.normal(size=(m, m)))
    M = R.T @ np.diag(np.linspace(-1.0, 1.0, m)) @ R
    C = 3 * Q
    H = np.block([[2 * np.eye(64), C], [C.T, C.T @ C / 2 + M]])
    assert np.linalg.eigvalsh(H[64:, 64:]).min() > 3 and np.linalg.eigvalsh(M).min() <= -1e-3 * abs(H).max()
    assert not numpy_says_indefinite(H[:64, :64]) and not numpy_says_indefinite(H[64:, 64:])
    sys_.append(("indefinite Schur complement", System(2, 63, H, np.zeros(63, np.int32))))
    return sys_


def test_failures_set_fail_and_the_context_recovers(chol):
    good, gb, _, _ = case("B6-n132-random", dict(WELL)["B6-n132-random"])
    with context_for(chol, good) as fresh:
        want = fresh.solve(good, gb)
    cases = failing_systems()
    cap = max(chol.envelope(s.env_blk, s.B)[0] for _, s in cases + [("", good)])
    with chol.context(cap, 3 * TS) as ctx:
        for name, s in cases:
            assert numpy_says_indefinite(s.dense()), name
            x, fail, _, _ = ctx.solve(s, np.ones(s.n), readback=False)
            assert fail == 1, name
            # fail is sticky: solving again without resetting it runs no kernel past the flag (x keeps the poison)
            x, fail, _, _ = ctx.solve(s, np.ones(s.n), flags=FLAG_POISON | FLAG_KEEP_FAIL, readback=False)
            assert fail == 1 and np.isnan(x).all(), name
            got = ctx.solve(good, gb)
            assert got[1] == 0, name
            for k in (0, 2, 3):
                assert np.array_equal(want[k], got[k]), name


# ================================================================================================ deterministic sums
def reduce0_restated(v):
    """reduce<0>: 256 fixed chunks of ceil(n / 256); per thread a sequential strided sum from 0; per warp an
    xor-butterfly over o = 16, 8, 4, 2, 1 read at lane 0; the 8 warp sums left to right; then the same over the 256
    partials (each thread starting from its partial)"""
    n = len(v)
    chunk = -(-n // 256)
    steps = -(-chunk // 256)  # strided loads per thread
    flat = np.zeros(256 * chunk)
    flat[:n] = v  # zeros past n add nothing: s + 0 == s
    blocks = np.zeros((256, steps * 256))
    blocks[:, :chunk] = flat.reshape(256, chunk)
    s = np.zeros((256, 256))
    for k in range(steps):
        s = s + blocks[:, k * 256:(k + 1) * 256]
    return block_tree(block_tree(s)[None, :])[0]


def block_tree(s):
    """(rows, 256) thread values -> (rows,) block results of the butterfly + warp-sum order"""
    w = s.reshape(-1, 8, 32)
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        w = w + w[:, :, lanes ^ o]
    r = w[:, 0, 0]
    for i in range(1, 8):
        r = r + w[:, i, 0]
    return r


def sum_inputs():
    rng = np.random.default_rng(17)
    out = []
    for n in (0, 1, 31, 255, 256, 257, 65537, 3000017):
        a = rng.normal(size=n) * 10.0 ** rng.integers(-8, 9, size=n)
        half = n // 2
        a[half:2 * half] = -a[:half][rng.permutation(half)] * (1 + 1e-12 * rng.normal(size=half))  # near-cancelling
        out.append(a)
    return out


def test_reduce_sum_bit_exact_order_and_accuracy(chol):
    for v in sum_inputs():
        got = chol.reduce(0, v)
        assert got == reduce0_restated(v), len(v)
        assert abs(got - math.fsum(v)) <= len(v) * U * float(np.abs(v).sum()), len(v)
    assert chol.reduce(0, np.array([])) == 0.0


def test_reduce_max_abs_exact(chol):
    for v in sum_inputs():
        want = float(np.abs(v).max()) if len(v) else 0.0
        assert chol.reduce(1, v) == want, len(v)
    v = np.zeros(70000)
    v[69999] = -3.5  # the last element, in the last chunk
    assert chol.reduce(1, v) == 3.5
