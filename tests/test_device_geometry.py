"""Direct tests of the device geometry shared by the solvers: csrc/jacobi.cuh (OpenCV's one-sided Jacobi SVD, float in
initializer.cu and double in pnpsolver.cu), csrc/sim3.cuh (g2o's Sim3: product, inverse, map, exp, log) and
csrc/ba_math.cuh (Eigen's quaternion conversions, SE3Quat's normalisation and exp-update, Converter's Tcw conversions,
the Huber kernel and linearizeOplus of the mono and stereo edges).  The solvers' own tests only see this code through
LM loops that reject a bad step and carry on, so here each function runs one thread per case through a test-only
harness (tests/cpp/geom_harness.cu) and is held to a high-precision reference.

The harness is built once per flag set an includer of the header is built with (build.py's NVCC_FLAGS and NO_FMAD):
ba_math.cuh with FMA contraction (localba.o, gba.o) and without (essential.o, sim3opt.o); sim3.cuh and jacobi.cuh
without only.  Every ba_math case runs against both builds.

The Jacobi SVD is compared bit for bit with cv2.SVDecomp, which runs the same JacobiSVDImpl_, at every shape the callers
instantiate.  The double instantiation uses only + - * / sqrt, so it must agree exactly.  The float one calls CUDA's
double hypot (documented error up to 2 ulp) where OpenCV uses lapack.cpp's template; a difference reaches the output
only if it moves the float rounding of a rotation's c or s, and the test counts the cases where any bit differs and
requires none (it was none of 2,408 when the test was written: random, rank-deficient, zero-column, all-zero and
repeated-singular-value matrices and the initialiser's normalised 8-point H and F systems).  The float SVD is also
checked as an SVD against float64, independently of cv2.

Everything else is compared with a restatement of the reference's own formulas (g2o's sim3.h, se3quat.h and
types_six_dof_expmap.cpp, quirks included: R = I + Omega + Omega^2 below theta = 1e-5, and the small-theta
B = ((sigma^2/2 - sigma + 1) s) / sigma^3 without the - 1), evaluated at 60 digits with mpmath.  Each branch is chosen
from the float64 value of the reference's own predicate, evaluated in the device's order, so both sides take the same
branch; the case lists keep every computed predicate far (relative 2^-20 or more) from its threshold, and the direct
inputs of quat_from_R and huber sit exactly on theirs (m11 = m00, m22 = m11, e = delta^2).  Each GPU test asserts that
its case list reaches every branch it names and prints the per-branch counts (pytest -s).

Error bars: Higham's running error analysis.  A value RE carries the exact value x (mpmath) of the restated formula on
the exact float64 inputs, the plain float64 value f of the same evaluation (used for the branch predicates only) and a
bound e on |float64 evaluation - x|.  With u = 2^-53:
- a correctly rounded + - * / sqrt adds u (|x| + p), where p is the propagated bound: |a|e_b + |b|e_a + e_a e_b for a
  product, e_a + e_b for a sum, (e_a + |x| e_b) / (|b| - e_b) for a quotient;
- a libm call (sin, cos, exp, log, acos: CUDA documents at most 2 ulp, and 2 ulp <= 4u |x|) adds 4u (|x| + p), and p
  is the exact spread of the function over [a - e_a, a + e_a] (|a - b| for sin and cos, which are 1-Lipschitz);
- a rounding to float32 adds 2^-24 (|x| + e).
A device output passes when |device - x| <= 2 e.  FMA contraction only removes roundings, and the factor 2 absorbs the
device's different but equivalent evaluation order where it has one (edge_jacobians forms 1/z once, the reference
divides by z and z^2 in every entry).  Where the formula is badly conditioned the bound grows and the test still holds:
(1 - cos theta)/theta^2 just above 1e-5 carries an error near 1e-6, theta/(2 sqrt(1 - d^2)) near theta = pi far more.
One float32 rounding anywhere in a chain (about 6e-8 relative), a swapped operand, a wrong branch or a wrong constant
lands far outside these bars.

The reference itself is checked on the CPU: where g2o's formulas are exact they must agree with the matrix exponential
(scipy.linalg.expm and mpmath's expm of the 4 x 4 sim3 / se3 generator) to 1e-25 and log(exp(u)) must give u back;
in the approximate branches the departure must stay under the truncation bound; and the running bound must hold for
the plain float64 evaluation on a few thousand random inputs."""
import ctypes
import importlib.util
import math
import os
import re
import shutil
import subprocess
from collections import Counter

import mpmath
import numpy as np
import pytest
import scipy.linalg as sla

from synth_init import synth_init

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG_DIR = os.path.join(ROOT, "self_commit_orb-slam2_b200")
CSRC = os.path.join(PKG_DIR, "csrc")
HARNESS = os.path.join(ROOT, "tests", "cpp", "geom_harness.cu")
HEADERS = ("ba_math.cuh", "sim3.cuh", "jacobi.cuh")
MACRO = {"sim3.cuh": "GEOM_SIM3", "jacobi.cuh": "GEOM_JACOBI"}  # ba_math.cuh is in every build

MP = mpmath.MPContext()
MP.dps = 60
U = 2.0 ** -53
UF = 2.0 ** -24
EPS = 0.00001  # g2o's branch threshold in sim3.h and se3quat.h
CAM = (520.0, 515.0, 40.0)  # fx, fy, bf


# ================================================================================================ running error
class RE:
    """Exact value x, float64 value f and a bound e on |float64 evaluation - x| (module docstring)."""
    __slots__ = ("x", "f", "e")

    def __init__(self, x, f, e):
        self.x, self.f, self.e = x, f, e

    @staticmethod
    def c(v):
        v = float(v)
        return RE(MP.mpf(v), v, MP.zero)

    @staticmethod
    def _r(x, f, p, k=1):
        return RE(x, f, p + k * U * (abs(x) + p))

    def __add__(a, b):
        b = lift(b)
        return RE._r(a.x + b.x, a.f + b.f, a.e + b.e)

    __radd__ = __add__

    def __sub__(a, b):
        b = lift(b)
        return RE._r(a.x - b.x, a.f - b.f, a.e + b.e)

    def __rsub__(a, b):
        return lift(b) - a

    def __neg__(a):
        return RE(-a.x, -a.f, a.e)

    def __abs__(a):
        return RE(abs(a.x), abs(a.f), a.e)

    def __mul__(a, b):
        b = lift(b)
        return RE._r(a.x * b.x, a.f * b.f, abs(a.x) * b.e + abs(b.x) * a.e + a.e * b.e)

    __rmul__ = __mul__

    def __truediv__(a, b):
        b = lift(b)
        x = a.x / b.x
        d = abs(b.x) - b.e
        p = (a.e + abs(x) * b.e) / d if d > 0 else MP.inf
        return RE._r(x, a.f / b.f, p)

    def __rtruediv__(a, b):
        return lift(b) / a

    def f32(a):
        return RE(a.x, float(np.float32(a.f)), a.e + UF * (abs(a.x) + a.e))


def lift(v):
    return v if isinstance(v, RE) else RE.c(v)


def _monotone(a, fx, ff, k, lo=None, hi=None):
    x = fx(a.x)
    ends = [a.x - a.e, a.x + a.e]
    if lo is not None:
        ends = [max(t, lo) for t in ends]
    if hi is not None:
        ends = [min(t, hi) for t in ends]
    p = max(abs(fx(t) - x) for t in ends)
    return RE._r(x, ff(a.f), p, k)


def r_sqrt(a):
    return _monotone(a, MP.sqrt, math.sqrt, 1, lo=MP.zero)


def r_exp(a):
    return _monotone(a, MP.exp, math.exp, 4)


def r_log(a):
    assert a.x - a.e > 0
    return _monotone(a, MP.log, math.log, 4)


def r_acos(a):
    return _monotone(a, MP.acos, math.acos, 4, lo=-MP.one, hi=MP.one)


def r_sin(a):
    return RE._r(MP.sin(a.x), math.sin(a.f), a.e, 4)


def r_cos(a):
    return RE._r(MP.cos(a.x), math.cos(a.f), a.e, 4)


def _re_vec(vals):
    return [RE.c(v) for v in np.asarray(vals, np.float64).ravel()]


# ================================================================================================ restatements
def cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def quat_rotate(q, v):
    """Eigen's q * v: uv = 2 (q.vec x v); v + w uv + q.vec x uv."""
    uv = cross(q[:3], v)
    uv = [t + t for t in uv]
    c = cross(q[:3], uv)
    return [(v[i] + q[3] * uv[i]) + c[i] for i in range(3)]


def quat_to_R(q):
    """Eigen's toRotationMatrix, row-major 3 x 3 list of lists."""
    tx, ty, tz = 2 * q[0], 2 * q[1], 2 * q[2]
    twx, twy, twz = tx * q[3], ty * q[3], tz * q[3]
    txx, txy, txz = tx * q[0], ty * q[0], tz * q[0]
    tyy, tyz, tzz = ty * q[1], tz * q[1], tz * q[2]
    return [[1 - (tyy + tzz), txy - twz, txz + twy],
            [txy + twz, 1 - (txx + tzz), tyz - twx],
            [txz - twy, tyz + twx, 1 - (txx + tyy)]]


def quat_from_R(m):
    """Eigen's Quaterniond(Matrix3d); returns (q, branch) with branch 'trace' or 'pivot0' / 'pivot1' / 'pivot2'."""
    t = (m[0][0] + m[1][1]) + m[2][2]
    if t.f > 0.0:
        t = r_sqrt(t + 1.0)
        w = 0.5 * t
        t = 0.5 / t
        return [(m[2][1] - m[1][2]) * t, (m[0][2] - m[2][0]) * t, (m[1][0] - m[0][1]) * t, w], "trace"
    i = 0
    if m[1][1].f > m[0][0].f:
        i = 1
    if m[2][2].f > m[i][i].f:
        i = 2
    j, k = (i + 1) % 3, (i + 2) % 3
    t = r_sqrt(((m[i][i] - m[j][j]) - m[k][k]) + 1.0)
    v = [None] * 3
    v[i] = 0.5 * t
    t = 0.5 / t
    w = (m[k][j] - m[j][k]) * t
    v[j] = (m[j][i] + m[i][j]) * t
    v[k] = (m[k][i] + m[i][k]) * t
    return v + [w], "pivot%d" % i


def normalize_rot(q):
    """SE3Quat::normalizeRotation: flip to w >= 0, then divide by the norm.  Returns (q, flipped)."""
    flip = q[3].f < 0
    if flip:
        q = [-t for t in q]
    n = r_sqrt(((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]) + q[3] * q[3])
    return [t / n for t in q], flip


def skew(w):
    z = RE.c(0.0)
    return [[z, -w[2], w[1]], [w[2], z, -w[0]], [-w[1], w[0], z]]


def mat_mul3(A, B):
    return [[(A[i][0] * B[0][j] + A[i][1] * B[1][j]) + A[i][2] * B[2][j] for j in range(3)] for i in range(3)]


def eye(i, j):
    return 1.0 if i == j else 0.0


def s3_mul(a, b):
    rt = quat_rotate(a, b[4:7])
    q = [a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1],
         a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2],
         a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0],
         a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2]]
    return q + [a[7] * rt[i] + a[4 + i] for i in range(3)] + [a[7] * b[7]]


def s3_inv(a):
    c = [-a[0], -a[1], -a[2], a[3]]
    k = -1.0 / a[7]
    return c + quat_rotate(c, [k * a[4], k * a[5], k * a[6]]) + [1.0 / a[7]]


def s3_map(a, X):
    rt = quat_rotate(a, X)
    return [a[7] * rt[i] + a[4 + i] for i in range(3)]


def _sim3_ABC(sigma, s, theta, small_sigma, small_theta):
    """A, B, C of sim3.h's exp (and log, given theta); theta is None when small_theta."""
    if small_sigma:
        C = RE.c(1.0)
        if small_theta:
            return RE.c(0.5), RE.c(1.0 / 6.0), C
        th2 = theta * theta
        return (1 - r_cos(theta)) / th2, (theta - r_sin(theta)) / (th2 * theta), C
    C = (s - 1) / sigma
    if small_theta:
        sg2 = sigma * sigma
        return ((sigma - 1) * s + 1) / sg2, ((0.5 * sg2 - sigma + 1) * s) / (sg2 * sigma), C
    a, b = s * r_sin(theta), s * r_cos(theta)
    th2, sg2 = theta * theta, sigma * sigma
    c = th2 + sg2
    A = (a * sigma + (1 - b) * theta) / (theta * c)
    B = (C - ((b - 1) * sigma + a * theta) / c) * 1.0 / th2
    return A, B, C


def s3_exp(u):
    """Sim3(const Vector7d&); returns (sim3 of 8, branch 'sigma{0,1}_theta{0,1}', 1 = small)."""
    w = u[:3]
    sigma = u[6]
    theta = r_sqrt((w[0] * w[0] + w[1] * w[1]) + w[2] * w[2])
    O = skew(w)
    s = r_exp(sigma)
    O2 = mat_mul3(O, O)
    small_s, small_t = abs(sigma.f) < EPS, theta.f < EPS
    A, B, C = _sim3_ABC(sigma, s, theta, small_s, small_t)
    if small_t:
        Rm = [[(eye(i, j) + O[i][j]) + O2[i][j] for j in range(3)] for i in range(3)]
    else:
        k1 = r_sin(theta) / theta
        k2 = (1 - r_cos(theta)) / (theta * theta)
        Rm = [[(eye(i, j) + k1 * O[i][j]) + k2 * O2[i][j] for j in range(3)] for i in range(3)]
    q, _ = quat_from_R(Rm)
    W = [[(A * O[i][j] + B * O2[i][j]) + C * eye(i, j) for j in range(3)] for i in range(3)]
    t = [(W[i][0] * u[3] + W[i][1] * u[4]) + W[i][2] * u[5] for i in range(3)]
    return q + t + [s], "sigma%d_theta%d" % (small_s, small_t)


def lu_solve(W, b):
    """Eigen's PartialPivLU solve, pivots from the float64 values (first largest |entry| on ties).  Returns (x, perm)."""
    W = [row[:] for row in W]
    perm = [0, 1, 2]
    for k in range(3):
        p, best = k, abs(W[k][k].f)
        for i in range(k + 1, 3):
            if abs(W[i][k].f) > best:
                best, p = abs(W[i][k].f), i
        if p != k:
            W[k], W[p] = W[p], W[k]
            perm[k], perm[p] = perm[p], perm[k]
        if W[k][k].f == 0.0:
            continue
        for i in range(k + 1, 3):
            W[i][k] = W[i][k] / W[k][k]
            for j in range(k + 1, 3):
                W[i][j] = W[i][j] - W[i][k] * W[k][j]
    x = [None] * 3
    for i in range(3):
        v = b[perm[i]]
        for k in range(i):
            v = v - W[i][k] * x[k]
        x[i] = v
    for i in (2, 1, 0):
        v = x[i]
        for k in range(i + 1, 3):
            v = v - W[i][k] * x[k]
        x[i] = v / W[i][i]
    return x, tuple(perm)


def s3_log(a):
    """Sim3::log(); returns (u of 7, branch 'sigma{0,1}_d{0,1}' with 1 = small sigma / d > 1 - eps, LU permutation)."""
    s = a[7]
    sigma = r_log(s)
    Rm = quat_to_R(a)
    d = 0.5 * (((Rm[0][0] + Rm[1][1]) + Rm[2][2]) - 1)
    dR = [Rm[2][1] - Rm[1][2], Rm[0][2] - Rm[2][0], Rm[1][0] - Rm[0][1]]
    small_s, small_d = abs(sigma.f) < EPS, d.f > 1 - EPS
    if small_d:
        omega = [0.5 * t for t in dR]
        A, B, C = _sim3_ABC(sigma, s, None, small_s, True)
    else:
        theta = r_acos(d)
        k = theta / (2 * r_sqrt(1 - d * d))
        omega = [k * t for t in dR]
        A, B, C = _sim3_ABC(sigma, s, theta, small_s, False)
    O = skew(omega)
    BOO = mat_mul3([[B * O[i][j] for j in range(3)] for i in range(3)], O)
    W = [[(A * O[i][j] + BOO[i][j]) + C * eye(i, j) for j in range(3)] for i in range(3)]
    x, perm = lu_solve(W, a[4:7])
    return omega + x + [sigma], "sigma%d_d%d" % (small_s, small_d), perm


def pose_oplus(P, upd):
    """SE3Quat::exp(update) * estimate; returns (pose of 7, branch 'small' / 'large', whether a normalisation flipped)."""
    w = upd[:3]
    theta = r_sqrt((w[0] * w[0] + w[1] * w[1]) + w[2] * w[2])
    O = skew(w)
    O2 = mat_mul3(O, O)
    small = theta.f < EPS
    if small:
        Rm = [[(eye(i, j) + O[i][j]) + O2[i][j] for j in range(3)] for i in range(3)]
        V = Rm
    else:
        a = r_sin(theta) / theta
        bb = (1 - r_cos(theta)) / (theta * theta)
        c = (theta - r_sin(theta)) / ((theta * theta) * theta)
        Rm = [[(eye(i, j) + a * O[i][j]) + bb * O2[i][j] for j in range(3)] for i in range(3)]
        V = [[(eye(i, j) + bb * O[i][j]) + c * O2[i][j] for j in range(3)] for i in range(3)]
    eq, _ = quat_from_R(Rm)
    eq, f1 = normalize_rot(eq)
    et = [(V[i][0] * upd[3] + V[i][1] * upd[4]) + V[i][2] * upd[5] for i in range(3)]
    rt = quat_rotate(eq, P[4:7])
    a, b = eq, P
    r = [a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1],
         a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2],
         a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0],
         a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2]]
    r, f2 = normalize_rot(r)
    return r + [et[i] + rt[i] for i in range(3)], ("small" if small else "large"), f1 or f2


def se3quat_from_Tcw(T):
    m = [[RE.c(T[4 * i + j]) for j in range(3)] for i in range(3)]
    q, br = quat_from_R(m)
    q, flip = normalize_rot(q)
    return q + [RE.c(T[3]), RE.c(T[7]), RE.c(T[11]), RE.c(0.0)], br, flip


def se3quat_to_Tcw(P):
    Rm = quat_to_R(P)
    out = []
    for r in range(3):
        out += [Rm[r][c].f32() for c in range(3)] + [P[4 + r].f32()]
    return out + [RE.c(0.0), RE.c(0.0), RE.c(0.0), RE.c(1.0)]


def huber(e, delta):
    dsqr = delta * delta
    if e.f <= dsqr.f:
        return [e, RE.c(1.0)], "quadratic"
    s = r_sqrt(e)
    return [(2 * s) * delta - dsqr, delta / s], "linear"


def edge_jacobians(P, X, stereo, fx, fy, bf):
    """linearizeOplus as types_six_dof_expmap.cpp writes it (divisions by z and z^2 in every entry).  Returns the 30
    outputs in the harness order: Xc 3, A 3 x 3, B 3 x 6 (a monocular edge's third rows are exact zeros)."""
    Xc = [quat_rotate(P, X)[i] + P[4 + i] for i in range(3)]
    Rm = quat_to_R(P)
    x, y, z = Xc
    z2 = z * z
    zero = RE.c(0.0)
    if stereo:
        A = [[-fx * Rm[0][c] / z + fx * x * Rm[2][c] / z2 for c in range(3)],
             [-fy * Rm[1][c] / z + fy * y * Rm[2][c] / z2 for c in range(3)]]
        A.append([A[0][c] - bf * Rm[2][c] / z2 for c in range(3)])
    else:
        tmp = [[RE.c(fx), zero, -x / z * fx], [zero, RE.c(fy), -y / z * fy]]
        M = [[(-1.0 / z) * t for t in row] for row in tmp]
        A = [[(M[r][0] * Rm[0][c] + M[r][1] * Rm[1][c]) + M[r][2] * Rm[2][c] for c in range(3)] for r in range(2)]
        A.append([zero] * 3)
    B = [[x * y / z2 * fx, -(1 + (x * x / z2)) * fx, y / z * fx, -1.0 / z * fx, zero, x / z2 * fx],
         [(1 + y * y / z2) * fy, -x * y / z2 * fy, -x / z * fy, zero, -1.0 / z * fy, y / z2 * fy]]
    if stereo:
        B.append([B[0][0] - bf * y / z2, B[0][1] + bf * x / z2, B[0][2], B[0][3], zero, B[0][5] - bf / z2])
    else:
        B.append([zero] * 6)
    return Xc + [t for row in A for t in row] + [t for row in B for t in row]


# ================================================================================================ first principles
def sim3_generator(u):
    """4 x 4 generator [[Omega + sigma I, upsilon], [0, 0]] whose exponential is [[s R, t], [0, 1]] (mpmath)."""
    w, ups, sg = [MP.mpf(float(v)) for v in u[:3]], [MP.mpf(float(v)) for v in u[3:6]], MP.mpf(float(u[6]))
    G = MP.zeros(4, 4)
    O = [[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]]
    for i in range(3):
        for j in range(3):
            G[i, j] = O[i][j] + (sg if i == j else 0)
        G[i, 3] = ups[i]
    return G


def R_of(q):
    return [[t.x for t in row] for row in quat_to_R([RE(v, 0.0, MP.zero) for v in q])]


# ================================================================================================ harness
def _product_build():
    spec = importlib.util.spec_from_file_location("_geom_product_build", os.path.join(PKG_DIR, "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _nvcc():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    return nvcc if os.path.exists(nvcc) else shutil.which("nvcc")


def header_flag_sets(no_fmad):
    """{header: {False (FMA contraction) / True (--fmad=false)}}: the flag sets of every csrc/*.cu that includes the
    header, directly or through another header."""
    inc = {}
    for f in os.listdir(CSRC):
        if f.endswith((".cu", ".cuh")):
            with open(os.path.join(CSRC, f)) as fh:
                inc[f] = set(re.findall(r'#include\s+"([^"]+)"', fh.read()))

    def reaches(f, h, seen=()):
        return any(g == h or (g in inc and g not in seen and reaches(g, h, seen + (g,))) for g in inc.get(f, ()))

    return {h: {f in no_fmad for f in inc if f.endswith(".cu") and reaches(f, h)} for h in HEADERS}


def harness_builds():
    """{build name: (nvcc flags, headers it covers)}: one build per flag set, covering the headers whose includers use
    it."""
    bld = _product_build()
    sets = header_flag_sets(bld.NO_FMAD)
    builds = {}
    for nofma in (False, True):
        hs = [h for h in HEADERS if nofma in sets[h]]
        if hs:
            flags = bld.NVCC_FLAGS + (["--fmad=false"] if nofma else []) + ["-D%s" % MACRO[h] for h in hs if h in MACRO]
            builds["nofma" if nofma else "fma"] = (flags, hs)
    return builds


def compile_harness(out_dir):
    nvcc = _nvcc()
    procs = {}
    for name, (flags, hs) in harness_builds().items():
        so = os.path.join(str(out_dir), "libgeom_%s.so" % name)
        cmd = [nvcc] + flags + ["-shared", "-I", CSRC, "-o", so, HARNESS]
        procs[name] = (so, hs, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT))
    libs = {}
    for name, (so, hs, p) in procs.items():
        log, _ = p.communicate()
        assert p.returncode == 0, log.decode()
        libs[name] = (so, hs)
    return libs


class Harness:
    def __init__(self, path, name, headers):
        self.name, self.headers = name, headers
        self.lib = ctypes.CDLL(path)

    def call(self, fn, n, *arrays):
        f = getattr(self.lib, "geom_" + fn)
        f.restype = ctypes.c_int
        rc = f(ctypes.c_int(n), *[a.ctypes.data_as(ctypes.c_void_p) for a in arrays])
        assert rc == 0, "geom_%s returned %d" % (fn, rc)

    def jacobi(self, dtype, At, m, n, n1):
        """At: (count, max(n, n1), m) in place; returns (At, W, Vt)."""
        At = np.ascontiguousarray(At, dtype)
        count = At.shape[0]
        W, Vt = np.zeros((count, n), dtype), np.zeros((count, n, n), dtype)
        f = self.lib.geom_jacobi_f32 if dtype == np.float32 else self.lib.geom_jacobi_f64
        f.restype = ctypes.c_int
        P = ctypes.c_void_p
        rc = f(count, m, n, n1, At.ctypes.data_as(P), W.ctypes.data_as(P), Vt.ctypes.data_as(P))
        assert rc == 0, "jacobi returned %d" % rc
        return At, W, Vt


@pytest.fixture(scope="module")
def harness_libs(tmp_path_factory):
    if _nvcc() is None:
        pytest.skip("nvcc not found")
    return compile_harness(tmp_path_factory.mktemp("geom_harness"))


@pytest.fixture(scope="module")
def device(harness_libs):
    n = ctypes.c_int(0)
    lib = ctypes.CDLL(harness_libs["fma"][0])
    if lib.geom_device_count(ctypes.byref(n)) != 0 or n.value < 1:
        pytest.skip("no CUDA device")


def _libs_with(header):
    return [n for n, (_, hs) in harness_builds().items() if header in hs]


@pytest.fixture(scope="module", params=[pytest.param(b, marks=pytest.mark.gpu) for b in _libs_with("ba_math.cuh")])
def ba(request, harness_libs, device):
    so, hs = harness_libs[request.param]
    return Harness(so, request.param, hs)


@pytest.fixture(scope="module")
def nofma(harness_libs, device):
    so, hs = harness_libs["nofma"]
    return Harness(so, "nofma", hs)


# ================================================================================================ comparison
def assert_within(name, dev, refs, ids=None):
    """Every device value within twice its running bound of the exact value; prints the worst ratio."""
    dev = np.asarray(dev, np.float64).reshape(len(refs), -1)
    worst, bad = 0.0, []
    for c, row in enumerate(refs):
        assert dev.shape[1] == len(row)
        for k, r in enumerate(row):
            d = dev[c, k]
            if not math.isfinite(d):
                bad.append((c, k, d, float(r.x), float(r.e)))
                continue
            err = abs(MP.mpf(d) - r.x)
            bar = 2 * r.e
            ratio = float(err / bar) if bar > 0 else (0.0 if err == 0 else math.inf)
            worst = max(worst, ratio)
            if ratio > 1:
                bad.append((ids[c] if ids else c, k, d, float(r.x), float(r.e)))
    print("%s: %d cases, worst |dev - exact| / (2 e) = %.3g" % (name, len(refs), worst))
    assert not bad, "%s: %d outputs outside the bar, first: %s" % (name, len(bad), bad[:5])


def report_branches(name, branches, required):
    cnt = Counter(branches)
    print("%s branches: %s" % (name, dict(sorted(cnt.items(), key=str))))
    missing = set(required) - set(cnt)
    assert not missing, "%s: no case reached %s" % (name, sorted(missing, key=str))


# ================================================================================================ case lists
def rand_axis(rng):
    a = rng.normal(size=3)
    return a / np.linalg.norm(a)


def rand_quat(rng, theta=None):
    th = rng.uniform(0, math.pi) if theta is None else theta
    ax = rand_axis(rng)
    q = np.concatenate([math.sin(th / 2) * ax, [math.cos(th / 2)]])
    return q / np.linalg.norm(q)


def quat_of_axis_angle(ax, th):
    ax = np.asarray(ax, np.float64) / np.linalg.norm(ax)
    return np.concatenate([math.sin(th / 2) * ax, [math.cos(th / 2)]])


def s3_exp_cases():
    rng = np.random.default_rng(71)
    b = 1e-5
    sigmas = [0.0] + [sg * v for sg in (1, -1) for v in (b * (1 + 2.0 ** -20), b * (1 - 2.0 ** -20), 1e-3, 0.5, 3.0)]
    thetas = [0.0, b * (1 + 2.0 ** -20), b * (1 - 2.0 ** -20), 4.47e-3, 1.0, math.pi - 1e-6, 3.0]
    out = []
    for sg in sigmas:
        for th in thetas:
            w = rand_axis(rng) * th
            t = rng.normal(size=3) * 10.0 ** rng.uniform(-2, 3)
            out.append(np.concatenate([w, t, [sg]]))
    return np.array(out)


def s3_log_cases():
    """Sim3 inputs: d = cos theta straddles 1 - 1e-5 (theta = acos(1 - 1e-5 (1 -+ 2^-10))), theta near pi,
    s = 1 and exp(+-1e-5 (1 +- 2^-20)), and translations whose W takes or does not take a row swap."""
    rng = np.random.default_rng(72)
    th_edge = [math.acos(1 - 1e-5 * (1 + k * 2.0 ** -10)) for k in (-1, 1)]
    thetas = [0.0, 1e-7, th_edge[0], th_edge[1], 0.3, 1.5, 2.5, math.pi - 1e-4, math.pi - 1e-7]
    scales = [1.0, math.exp(1e-5 * (1 + 2.0 ** -20)), math.exp(1e-5 * (1 - 2.0 ** -20)),
              math.exp(-1e-5 * (1 + 2.0 ** -20)), math.exp(-1e-5 * (1 - 2.0 ** -20)), 0.2, 3.0]
    out = []
    for th in thetas:
        for s in scales:
            for _ in range(2):
                q = rand_quat(rng, th)
                t = rng.normal(size=3) * 10.0 ** rng.uniform(-2, 2)
                out.append(np.concatenate([q, t, [s]]))
    # theta about a coordinate axis with a large sigma: W's off-diagonal dominates the diagonal -> a row swap
    for ax in np.eye(3):
        for th in (2.0, 2.8):
            out.append(np.concatenate([quat_of_axis_angle(ax, th), rng.normal(size=3), [0.05]]))
    return np.array(out)


def sim3_operands(rng, k):
    out = []
    for s in (1e-3, 1.0, 1e3):
        for _ in range(k):
            out.append(np.concatenate([rand_quat(rng), rng.normal(size=3) * 10.0 ** rng.uniform(-2, 3), [s]]))
    return np.array(out)


def pose_oplus_cases():
    """(poses, updates).  theta straddling 1e-5, theta near pi, and products whose w comes out negative."""
    rng = np.random.default_rng(73)
    P, D = [], []
    thetas = [0.0, 1e-5 * (1 - 2.0 ** -20), 1e-5 * (1 + 2.0 ** -20), 1e-3, 0.5, 2.0, math.pi - 1e-6]
    for th in thetas:
        for _ in range(4):
            q = rand_quat(rng)
            P.append(np.concatenate([q, rng.normal(size=3) * 5, [0.0]]))
            D.append(np.concatenate([rand_axis(rng) * th, rng.normal(size=3) * 10.0 ** rng.uniform(-3, 1)]))
    # the current rotation near pi with w > 0 and an update that carries it past pi: the product's w is negative
    for _ in range(4):
        ax = rand_axis(rng)
        P.append(np.concatenate([quat_of_axis_angle(ax, math.pi - 0.01), rng.normal(size=3), [0.0]]))
        D.append(np.concatenate([ax * 0.05, rng.normal(size=3) * 0.1]))
    return np.array(P), np.array(D)


def rot_matrix(ax, th):
    ax = np.asarray(ax, np.float64) / np.linalg.norm(ax)
    S = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    return np.eye(3) + math.sin(th) * S + (1 - math.cos(th)) * S @ S


def quat_from_R_cases():
    rng = np.random.default_rng(74)
    out = []
    for _ in range(8):
        out.append(rot_matrix(rand_axis(rng), rng.uniform(0, 1.5)))  # trace > 0
    # trace <= 0 with each diagonal pivot: large rotations about axes near x, y, z
    for i in range(3):
        for _ in range(4):
            ax = np.eye(3)[i] + rng.normal(size=3) * 0.2
            out.append(rot_matrix(ax, rng.uniform(2.3, 3.1)))
    for i in range(3):  # pi about each axis: w = 0
        out.append(np.diag([1.0 if k == i else -1.0 for k in range(3)]))
    out.append(np.array([[0.0, 1, 0], [1, 0, 0], [0, 0, -1]]))  # pi about (1, 1, 0): m11 == m00 keeps pivot 0
    out.append(np.array([[-1.0, 0, 0], [0, 0, 1], [0, 1, 0]]))  # pi about (0, 1, 1): m22 == m11 keeps pivot 1
    out.append(rot_matrix([1, 1, 1], 2 * math.pi / 3))  # trace exactly 0 (a cyclic permutation)
    out.append(np.array([[0.0, 0, 1], [1, 0, 0], [0, 1, 0]]))
    return np.array(out)


def synth_systems(n_sets=64):
    """The initialiser's 8-point systems, float32: ComputeH21's 16 x 9 and ComputeF21's 8 x 9 over Normalize'd
    keypoints of tests/synth_init.py scenes."""
    H, F = [], []
    for seed, kind in ((1, "planar"), (4, "general"), (9, "ambiguous")):
        sc = synth_init(200, seed, kind=kind, iterations=n_sets)
        pn = []
        for kp in (sc["kp1"], sc["kp2"]):
            mean = kp.astype(np.float64).mean(0).astype(np.float32)
            dev = np.abs(kp - mean).astype(np.float64).mean(0).astype(np.float32)
            sxy = (1.0 / dev.astype(np.float64)).astype(np.float32)
            pn.append(((kp - mean) * sxy).astype(np.float32))
        m = np.nonzero(sc["matches12"] >= 0)[0]
        pairs = np.stack([m, sc["matches12"][m]], 1)
        for st in sc["sets"]:
            p1, p2 = pn[0][pairs[st, 0]], pn[1][pairs[st, 1]]
            u1, v1, u2, v2 = p1[:, 0], p1[:, 1], p2[:, 0], p2[:, 1]
            z, o = np.zeros(8, np.float32), np.ones(8, np.float32)
            A = np.zeros((16, 9), np.float32)
            A[0::2] = np.stack([z, z, z, -u1, -v1, -o, v2 * u1, v2 * v1, v2], 1)
            A[1::2] = np.stack([u1, v1, o, z, z, z, -u2 * u1, -u2 * v1, -u2], 1)
            H.append(A)
            F.append(np.stack([u2 * u1, u2 * v1, u2, v2 * u1, v2 * v1, v2, u1, v1, o], 1).astype(np.float32))
    return H, F


def svd_families(rng, rows, cols, k, dtype):
    """Random, rank 2, rank 1, a zero column, all zero, repeated singular values."""
    out = []
    for _ in range(k):
        out.append(rng.normal(size=(rows, cols)) * 10.0 ** rng.uniform(-2, 2))
    for r in (2, 1):
        for _ in range(max(k // 4, 2)):
            out.append(rng.normal(size=(rows, r)) @ rng.normal(size=(r, cols)))
    for c in range(min(cols, 3)):
        A = rng.normal(size=(rows, cols))
        A[:, c] = 0
        out.append(A)
    out.append(np.zeros((rows, cols)))
    n = min(rows, cols)
    for _ in range(3):
        Qa = np.linalg.qr(rng.normal(size=(rows, rows)))[0][:, :n]
        Qb = np.linalg.qr(rng.normal(size=(cols, cols)))[0][:n]
        out.append(Qa @ np.diag([2.0] * (n // 2) + [1.0] * (n - n // 2)) @ Qb)
    out.append(np.eye(rows, cols) * 3.0)
    return [np.asarray(A, dtype) for A in out]


# ---- cv2's JacobiSVD mapped to the harness's (At, W, Vt): SVD::compute transposes a wide input
def harness_input(A, m, n, n1):
    rows = max(n, n1)
    At = np.zeros((rows, m), A.dtype)
    At[:n] = A if A.shape[0] < A.shape[1] else A.T
    return At


def cv2_expected(A, n1):
    """(At, W, Vt) the way SVD::compute leaves JacobiSVD's buffers, or None for At when n1 = 0 (At is then UW)."""
    import cv2
    wide = A.shape[0] < A.shape[1]
    w, u, vt = cv2.SVDecomp(A.copy(), flags=cv2.SVD_FULL_UV if wide else 0)
    if wide:  # JacobiSVD(A) of the 9 x 8 transpose: At holds vt (completed to 9 rows), Vt holds u^T
        return vt, w.ravel(), u.T
    return (u.T if n1 else None), w.ravel(), vt


F32_SHAPES = [(3, 3, 3), (4, 4, 0), (16, 9, 0), (9, 8, 9)]  # (m, n, n1) as initializer.cu instantiates them
F64_SHAPES = [(3, 3, 3), (12, 12, 12), (6, 3, 3), (6, 4, 4), (6, 5, 5)]  # pnpsolver.cu


def matrix_shape(m, n, n1):
    return (n, m) if n1 > n else (m, n)  # ComputeF21 passes the 8 x 9 system itself


# ================================================================================================ CPU: the reference
def test_harness_flag_sets_follow_build():
    """One harness build per flag set that really includes each header, and the ones the headers are documented with."""
    sets = header_flag_sets(_product_build().NO_FMAD)
    assert sets == {"ba_math.cuh": {False, True}, "sim3.cuh": {True}, "jacobi.cuh": {True}}
    b = harness_builds()
    assert set(b) == {"fma", "nofma"}
    assert b["fma"][1] == ["ba_math.cuh"] and "--fmad=false" not in b["fma"][0]
    assert b["nofma"][1] == list(HEADERS) and "--fmad=false" in b["nofma"][0]


def test_harness_compiles(tmp_path):
    if _nvcc() is None:
        pytest.skip("nvcc not found")
    libs = compile_harness(tmp_path)
    for name, (so, hs) in libs.items():
        syms = subprocess.run(["nm", "-D", so], capture_output=True, text=True).stdout
        assert "geom_pose_oplus" in syms
        assert ("geom_s3_log" in syms) == ("sim3.cuh" in hs)
        assert ("geom_jacobi_f32" in syms) == ("jacobi.cuh" in hs)


def test_running_error_bounds_float64():
    """The bound e holds for the plain float64 evaluation (f) of every restated function on random inputs."""
    rng = np.random.default_rng(5)
    checked = 0

    def chk(outs):
        nonlocal checked
        for r in outs:
            assert abs(MP.mpf(r.f) - r.x) <= r.e, (r.f, r.x, r.e)
            checked += 1

    for _ in range(150):
        u = np.concatenate([rand_axis(rng) * 10.0 ** rng.uniform(-7, 0.4), rng.normal(size=3) * 100,
                            [rng.choice([0.0, 1e-6, -0.3, 2.0]) * rng.uniform(0.5, 1)]])
        chk(s3_exp(_re_vec(u))[0])
        a = np.concatenate([rand_quat(rng), rng.normal(size=3) * 10, [10.0 ** rng.uniform(-2, 2)]])
        chk(s3_log(_re_vec(a))[0])
        chk(s3_mul(_re_vec(a), _re_vec(np.concatenate([rand_quat(rng), rng.normal(size=3), [2.0]]))))
        chk(s3_inv(_re_vec(a)))
        P = np.concatenate([rand_quat(rng), rng.normal(size=3), [0.0]])
        d = np.concatenate([rand_axis(rng) * 10.0 ** rng.uniform(-7, 0.4), rng.normal(size=3)])
        chk(pose_oplus(_re_vec(P), _re_vec(d))[0])
        X = rng.normal(size=3) * 2 + [0, 0, 6]
        chk(edge_jacobians(_re_vec(P), _re_vec(X), bool(rng.integers(2)), *CAM))
    assert checked > 5000


def _close(a, b, tol):
    return all(abs(MP.mpf(x) - MP.mpf(y)) <= tol for x, y in zip(a, b))


def test_sim3_exp_matches_matrix_exponential():
    """In the exact branches sim3.h's closed forms are exp of the 4 x 4 generator (mpmath to 1e-25, scipy to 1e-13);
    below theta = 1e-5 R = I + Omega + Omega^2 departs from exp(Omega) by at most theta^2 / 2 + theta^3."""
    rng = np.random.default_rng(6)
    n_exact = n_approx = 0
    for u in s3_exp_cases():
        out, br = s3_exp(_re_vec(u))
        q, t, s = [r.x for r in out[:4]], [r.x for r in out[4:7]], out[7].x
        E = MP.expm(sim3_generator(u))
        Rq = R_of(q)
        sR = [[s * Rq[i][j] for j in range(3)] for i in range(3)]
        theta = float(np.linalg.norm(u[:3]))
        if br.endswith("theta0"):  # R's closed form is exact; A, B, C too unless C = 1 stands in for (s - 1)/sigma
            assert _close([sR[i][j] for i in range(3) for j in range(3)], [E[i, j] for i in range(3) for j in range(3)],
                          MP.mpf("1e-25") * (1 + abs(s)))
            Es = sla.expm(np.array(sim3_generator(u).tolist(), dtype=float))
            assert np.allclose(Es[:3, :3], np.array(sR, float), rtol=1e-12, atol=1e-13 * float(s))
            if br.startswith("sigma1") and u[6] != 0.0:
                continue
            assert _close(t, [E[i, 3] for i in range(3)], MP.mpf("1e-25") * (1 + float(np.abs(u[3:6]).max())) * (1 + abs(s)))
            assert np.allclose(Es[:3, 3], np.array(t, float), rtol=1e-11, atol=1e-11 * float(np.abs(u[3:6]).max()))
            n_exact += 1
        else:
            Er = MP.expm(MP.matrix([[0, -u[2], u[1]], [u[2], 0, -u[0]], [-u[1], u[0], 0]]))
            dev = max(abs(Rq[i][j] - Er[i, j]) for i in range(3) for j in range(3))
            assert dev <= theta ** 2 / 2 + theta ** 3 + 1e-30
            n_approx += 1
        assert abs(s - MP.exp(MP.mpf(float(u[6])))) <= MP.mpf("1e-50")
    assert n_exact and n_approx


def test_se3_exp_matches_matrix_exponential():
    rng = np.random.default_rng(7)
    n = 0
    for _ in range(40):
        th = 10.0 ** rng.uniform(-4, 0.45)
        d = np.concatenate([rand_axis(rng) * th, rng.normal(size=3)])
        ident = np.array([0, 0, 0, 1.0, 0, 0, 0, 0])
        out, br, _ = pose_oplus(_re_vec(ident), _re_vec(d))
        assert br == "large"
        E = MP.expm(sim3_generator(np.concatenate([d, [0.0]])))
        Rq = R_of([r.x for r in out[:4]])
        assert _close([Rq[i][j] for i in range(3) for j in range(3)], [E[i, j] for i in range(3) for j in range(3)],
                      MP.mpf("1e-25"))
        assert _close([r.x for r in out[4:7]], [E[i, 3] for i in range(3)], MP.mpf("1e-25") * 10)
        n += 1
    assert n


def test_sim3_log_inverts_exp():
    """log(exp(u)) = u at 60 digits wherever both take exact branches (theta in (4.5e-3, pi), |sigma| >= 1e-5)."""
    rng = np.random.default_rng(8)
    for _ in range(40):
        th, sg = rng.uniform(0.01, 3.0), rng.choice([-1, 1]) * 10.0 ** rng.uniform(-4, 0.3)
        u = np.concatenate([rand_axis(rng) * th, rng.normal(size=3) * 5, [sg]])
        for usg in (sg, 0.0):
            uu = u.copy()
            uu[6] = usg
            e, br = s3_exp(_re_vec(uu))
            assert br == "sigma%d_theta0" % (usg == 0.0)
            back, br2, _ = s3_log([RE(r.x, float(r.x), MP.zero) for r in e])
            assert br2 == "sigma%d_d0" % (usg == 0.0)
            assert _close([r.x for r in back], [MP.mpf(float(v)) for v in uu], MP.mpf("1e-25") * 10)


def test_sim3_group_ops_match_matrices():
    """s3_mul / s3_inv / s3_map restated agree with the 4 x 4 similarity matrices (to 1e-13: a float64 quaternion is
    unit only to about 1e-16, and Eigen's q * v and toRotationMatrix agree exactly for unit quaternions only)."""
    rng = np.random.default_rng(9)
    ops = sim3_operands(rng, 3)

    def mat(a):
        Rq = R_of([MP.mpf(float(v)) for v in a[:4]])
        M = MP.eye(4)
        for i in range(3):
            for j in range(3):
                M[i, j] = MP.mpf(float(a[7])) * Rq[i][j]
            M[i, 3] = MP.mpf(float(a[4 + i]))
        return M

    def mat_x(o):
        Rq = R_of([r.x for r in o[:4]])
        M = MP.eye(4)
        for i in range(3):
            for j in range(3):
                M[i, j] = o[7].x * Rq[i][j]
            M[i, 3] = o[4 + i].x
        return M

    for a in ops:
        for b in ops[::2]:
            prod = mat_x(s3_mul(_re_vec(a), _re_vec(b)))
            assert MP.mnorm(prod - mat(a) * mat(b), 1) <= 1e-13 * MP.mnorm(mat(a), 1) * MP.mnorm(mat(b), 1)
        inv = mat_x(s3_inv(_re_vec(a)))
        assert MP.mnorm(inv * mat(a) - MP.eye(4), 1) <= 1e-13 * MP.mnorm(mat(a), 1) * MP.mnorm(inv, 1)
        X = rng.normal(size=3)
        y = s3_map(_re_vec(a), _re_vec(X))
        Y = mat(a) * MP.matrix([MP.mpf(float(v)) for v in X] + [1])
        assert _close([r.x for r in y], [Y[i] for i in range(3)], 1e-13 * MP.mnorm(mat(a), 1) * 10)


def test_quat_from_R_inverts_quat_to_R():
    """Eigen's Quaterniond(Matrix3d) restated, on every branch: toRotationMatrix of the result gives R back."""
    brs = []
    for Rm in quat_from_R_cases():
        q, br = quat_from_R([[RE.c(v) for v in row] for row in Rm])
        brs.append(br)
        back = R_of([r.x for r in q])
        assert max(abs(back[i][j] - Rm[i][j]) for i in range(3) for j in range(3)) < 1e-14
    report_branches("quat_from_R (reference)", brs, ["trace", "pivot0", "pivot1", "pivot2"])


def test_edge_jacobians_reference_against_central_differences():
    """The restated linearizeOplus is the derivative of the reprojection error: error = obs - proj(exp(d) T X)."""
    rng = np.random.default_rng(10)
    fx, fy, bf = CAM
    for st in (False, True):
        for _ in range(5):
            P = np.concatenate([rand_quat(rng), rng.normal(size=3), [0.0]])
            X = rng.normal(size=3) + [0, 0, 5]
            out = np.array([float(r.x) for r in edge_jacobians(_re_vec(P), _re_vec(X), st, fx, fy, bf)])
            Xc = out[:3]
            A, B = out[3:12].reshape(3, 3), out[12:].reshape(3, 6)
            Rm = np.array(R_of([MP.mpf(v) for v in P[:4]]), float)

            def err(xc):
                u = fx * xc[0] / xc[2]
                v = fy * xc[1] / xc[2]
                return -np.array([u, v, u - bf / xc[2]] if st else [u, v, 0.0])

            h = 1e-6
            for c in range(3):
                dX = np.eye(3)[c] * h
                fd = (err(Rm @ (X + dX) + P[4:7]) - err(Rm @ (X - dX) + P[4:7])) / (2 * h)
                assert np.allclose(A[:, c], fd, rtol=1e-6, atol=1e-6)
            for c in range(6):
                d = np.eye(6)[c] * h
                plus = Xc + np.cross(d[:3], Xc) + d[3:]  # exp(d) Xc to first order
                minus = Xc - np.cross(d[:3], Xc) - d[3:]
                fd = (err(plus) - err(minus)) / (2 * h)
                assert np.allclose(B[:, c], fd, rtol=1e-5, atol=1e-5)


# ================================================================================================ GPU: Jacobi SVD
@pytest.mark.gpu
def test_jacobi_double_bit_identical_to_cv2(nofma):
    rng = np.random.default_rng(21)
    for m, n, n1 in F64_SHAPES:
        rows, cols = matrix_shape(m, n, n1)
        mats = svd_families(rng, rows, cols, 60, np.float64)
        At, W, Vt = nofma.jacobi(np.float64, np.stack([harness_input(A, m, n, n1) for A in mats]), m, n, n1)
        diff = 0
        for c, A in enumerate(mats):
            eAt, eW, eVt = cv2_expected(A, n1)
            diff += not (np.array_equal(At[c], eAt) and np.array_equal(W[c], eW) and np.array_equal(Vt[c], eVt))
        print("jacobi f64 %dx%d n1=%d: %d cases, %d differ from cv2" % (m, n, n1, len(mats), diff))
        assert diff == 0


def _f32_cases(rng, m, n, n1):
    rows, cols = matrix_shape(m, n, n1)
    mats = svd_families(rng, rows, cols, 300, np.float32)
    H, F = synth_systems()
    if (rows, cols) == (16, 9):
        mats += H
    if (rows, cols) == (8, 9):
        mats += F
    if (rows, cols) == (3, 3):  # ComputeF21's Fpre: the null vector of each 8 x 9 system, as a 3 x 3
        import cv2
        mats += [cv2.SVDecomp(A.copy(), flags=cv2.SVD_FULL_UV)[2][8].reshape(3, 3).copy() for A in F]
    return mats


@pytest.mark.gpu
def test_jacobi_float_bit_identical_to_cv2(nofma):
    rng = np.random.default_rng(22)
    total = 0
    for m, n, n1 in F32_SHAPES:
        mats = _f32_cases(rng, m, n, n1)
        At, W, Vt = nofma.jacobi(np.float32, np.stack([harness_input(A, m, n, n1) for A in mats]), m, n, n1)
        diff = 0
        for c, A in enumerate(mats):
            eAt, eW, eVt = cv2_expected(A, n1)
            same = np.array_equal(W[c], eW) and np.array_equal(Vt[c], eVt)
            if eAt is not None:
                same = same and np.array_equal(At[c], eAt)
            diff += not same
        total += diff
        print("jacobi f32 %dx%d n1=%d: %d cases, %d differ from cv2 in some bit" % (m, n, n1, len(mats), diff))
    assert total == 0


@pytest.mark.gpu
def test_jacobi_float_is_an_svd(nofma):
    """Independently of cv2: W sorted, Vt orthonormal to 8 n u_f, and ||A - U W Vt|| <= 8 n u_f ||A|| (UW itself when
    n1 = 0), W within 8 n u_f ||A|| of a float64 SVD's singular values."""
    rng = np.random.default_rng(23)
    for m, n, n1 in F32_SHAPES:
        mats = _f32_cases(rng, m, n, n1)
        Ain = np.stack([harness_input(A, m, n, n1) for A in mats])
        At, W, Vt = nofma.jacobi(np.float32, Ain.copy(), m, n, n1)
        tol = 8 * n * UF
        for c, A in enumerate(mats):
            w, V, Ut = W[c].astype(float), Vt[c].astype(float), At[c, :n].astype(float)
            nA = np.linalg.norm(A.astype(float))
            assert np.all(np.diff(w) <= 0)
            assert np.abs(V @ V.T - np.eye(n)).max() <= tol
            M = Ain[c, :n].astype(float).T  # the m x n matrix JacobiSVD decomposes
            rec = Ut.T @ np.diag(w) @ V if n1 else Ut.T @ V
            assert np.linalg.norm(M - rec) <= tol * max(nA, 1e-30) + 1e-37
            sv = np.linalg.svd(M.astype(float), compute_uv=False)
            assert np.abs(np.sort(w)[::-1] - sv).max() <= tol * max(nA, 1e-30) + 1e-37


# ================================================================================================ GPU: sim3.cuh
@pytest.mark.gpu
def test_s3_exp(nofma):
    U7 = s3_exp_cases()
    out = np.zeros((len(U7), 8))
    nofma.call("s3_exp", len(U7), np.ascontiguousarray(U7), out)
    refs, brs = zip(*[s3_exp(_re_vec(u)) for u in U7])
    report_branches("s3_exp", brs, ["sigma%d_theta%d" % (a, b) for a in (0, 1) for b in (0, 1)])
    assert_within("s3_exp", out, refs)


@pytest.mark.gpu
def test_s3_log(nofma):
    A = s3_log_cases()
    out = np.zeros((len(A), 7))
    nofma.call("s3_log", len(A), np.ascontiguousarray(A), out)
    refs, brs, perms = zip(*[s3_log(_re_vec(a)) for a in A])
    report_branches("s3_log", brs, ["sigma%d_d%d" % (a, b) for a in (0, 1) for b in (0, 1)])
    cnt = Counter(perms)
    print("s3_log LU pivot paths: %s" % dict(cnt))
    assert len(cnt) == 6  # every row order W.lu() can choose, the identity included
    assert_within("s3_log", out, refs)


@pytest.mark.gpu
def test_s3_mul_inv_map(nofma):
    rng = np.random.default_rng(24)
    a = sim3_operands(rng, 6)
    b = a[rng.permutation(len(a))]
    X = rng.normal(size=(len(a), 3)) * 10
    o = np.zeros((len(a), 8))
    nofma.call("s3_mul", len(a), a, b, o)
    assert_within("s3_mul", o, [s3_mul(_re_vec(x), _re_vec(y)) for x, y in zip(a, b)])
    nofma.call("s3_inv", len(a), a, o)
    assert_within("s3_inv", o, [s3_inv(_re_vec(x)) for x in a])
    o3 = np.zeros((len(a), 3))
    nofma.call("s3_map", len(a), a, np.ascontiguousarray(X), o3)
    assert_within("s3_map", o3, [s3_map(_re_vec(x), _re_vec(y)) for x, y in zip(a, X)])


# ================================================================================================ GPU: ba_math.cuh
def test_pose_oplus(ba):
    P, D = pose_oplus_cases()
    out = np.ascontiguousarray(P.copy())
    ba.call("pose_oplus", len(P), out, np.ascontiguousarray(D))
    refs, brs, flips = zip(*[pose_oplus(_re_vec(p), _re_vec(d)) for p, d in zip(P, D)])
    report_branches("pose_oplus[%s]" % ba.name, list(brs) + ["flip" for f in flips if f], ["small", "large", "flip"])
    assert_within("pose_oplus[%s]" % ba.name, out[:, :7], refs)
    assert np.all(out[:, 7] == P[:, 7])


def test_quat_from_R_and_normalize(ba):
    Rs = quat_from_R_cases()
    q = np.zeros((len(Rs), 4))
    ba.call("quat_from_R", len(Rs), np.ascontiguousarray(Rs.reshape(-1, 9)), q)
    refs, brs = zip(*[quat_from_R([[RE.c(v) for v in row] for row in Rm]) for Rm in Rs])
    report_branches("quat_from_R[%s]" % ba.name, brs, ["trace", "pivot0", "pivot1", "pivot2"])
    assert_within("quat_from_R[%s]" % ba.name, q, refs)
    rng = np.random.default_rng(25)
    Q = rng.normal(size=(16, 4)) * 10.0 ** rng.uniform(-3, 3, size=(16, 1))
    Q[:4, 3] = np.abs(Q[:4, 3])
    Q[4:8, 3] = -np.abs(Q[4:8, 3])
    Q[8, 3] = 0.0
    out = np.ascontiguousarray(Q.copy())
    ba.call("normalize_rot", len(Q), out)
    refs, flips = zip(*[normalize_rot(_re_vec(v)) for v in Q])
    report_branches("normalize_rot[%s]" % ba.name, ["flip" if f else "keep" for f in flips], ["flip", "keep"])
    assert_within("normalize_rot[%s]" % ba.name, out, refs)


def test_se3quat_tcw_conversions(ba):
    """Converter's toSE3Quat on float Tcw that is not exactly orthonormal, toCvMat back, and the round trip."""
    rng = np.random.default_rng(26)
    Ts = []
    for Rm in quat_from_R_cases():
        T = np.eye(4)
        T[:3, :3] = Rm + rng.normal(size=(3, 3)) * 1e-6
        T[:3, 3] = rng.normal(size=3) * 10
        Ts.append(T.astype(np.float32))
    Ts = np.ascontiguousarray(np.array(Ts).reshape(-1, 16))
    P = np.zeros((len(Ts), 8))
    ba.call("se3quat_from_Tcw", len(Ts), Ts, P)
    refs, brs, _ = zip(*[se3quat_from_Tcw(T.astype(np.float64)) for T in Ts])
    report_branches("se3quat_from_Tcw[%s]" % ba.name, brs, ["trace", "pivot0", "pivot1", "pivot2"])
    assert_within("se3quat_from_Tcw[%s]" % ba.name, P, refs)
    T2 = np.zeros((len(Ts), 16), np.float32)
    ba.call("se3quat_to_Tcw", len(Ts), P, T2)
    assert_within("se3quat_to_Tcw[%s]" % ba.name, T2, [se3quat_to_Tcw(_re_vec(p)) for p in P])
    # round trip: the orthonormalised rotation comes back within a few float ulps of the input's
    assert np.abs(T2 - Ts).max() <= 1e-5 * max(1.0, np.abs(Ts).max())


def test_huber(ba):
    deltas = [math.sqrt(5.991), math.sqrt(7.815), 0.1, 1.0]
    E = []
    for d in deltas:
        d2 = d * d
        E += [(0.0, d), (d2, d), (np.nextafter(d2, math.inf), d), (d2 * 0.5, d), (d2 * 4, d), (1e6, d)]
    E = np.ascontiguousarray(np.array(E))
    rho = np.zeros((len(E), 2))
    ba.call("huber", len(E), E, rho)
    refs, brs = zip(*[huber(RE.c(e), RE.c(d)) for e, d in E])
    report_branches("huber[%s]" % ba.name, brs, ["quadratic", "linear"])
    # e = delta^2 is quadratic, its successor linear
    assert [brs[6 * k + 1] for k in range(len(deltas))] == ["quadratic"] * len(deltas)
    assert [brs[6 * k + 2] for k in range(len(deltas))] == ["linear"] * len(deltas)
    assert_within("huber[%s]" % ba.name, rho, refs)


def edge_cases():
    rng = np.random.default_rng(27)
    P, X = [], []
    for z in (1e-3, 0.1, 1.0, 100.0, 1e4, -2.0):
        for ratio in (0.0, 0.3, 3.0, 10.0):
            q = rand_quat(rng)
            t = rng.normal(size=3)
            xc = np.array([ratio * z * rng.choice([-1, 1]), ratio * z * rng.uniform(-1, 1), z])
            Rm = np.array(R_of([MP.mpf(v) for v in q]), float)
            X.append(Rm.T @ (xc - t))
            P.append(np.concatenate([q, t, [0.0]]))
    return np.array(P), np.array(X)


def test_edge_jacobians(ba):
    P, X = edge_cases()
    n = len(P)
    fx, fy, bf = CAM
    for st in (0.0, 1.0):
        arg = np.ascontiguousarray(np.concatenate([X, np.tile([fx, fy, bf, st], (n, 1))], 1))
        out = np.zeros((n, 30))
        ba.call("edge_jacobians", n, np.ascontiguousarray(P), arg, out)
        refs = [edge_jacobians(_re_vec(p), _re_vec(x), bool(st), fx, fy, bf) for p, x in zip(P, X)]
        assert_within("edge_jacobians[%s, %s]" % (ba.name, "stereo" if st else "mono"), out, refs)
