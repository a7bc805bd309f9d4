"""Direct tests of csrc/levenberg.cuh, the Levenberg-Marquardt step control that LocalBA, PoseOptimization, the global
bundle adjustment and the essential graph share.  The solvers' own tests only see it through the trials their problems
happen to take, so here it is driven through a test-only harness (tests/cpp/levenberg_harness.cu, host code) with
scripted (solved, tempChi, scale) trials.

Every expectation is derived from the reference's g2o (Thirdparty/g2o/g2o/core/optimization_algorithm_levenberg.cpp):
  :47-51    tau = 1e-5, good-step scale factors 2/3 (upper) and 1/3 (lower), at most 10 trials per iteration
  :93-97    on the first iteration lambda = computeLambdaInit(), ni = 2, nBad = 0
  :127-133  tempChi = DBL_MAX on a failed solve; rho = (currentChi - tempChi) / (computeScale() + 1e-3)
  :135-148  accept when rho > 0 and tempChi is finite: lambda *= max(1/3, min(1 - (2 rho - 1)^3, 2/3)), ni = 2;
            reject: lambda *= ni, ni *= 2
  :149      another trial while rho < 0, fewer than 10 trials and no stop request
  :151-161  the optimisation ends after 10 trials or rho == 0, and after three iterations in a row that lower chi2 by
            less than 1e-3 of its initial value
The library's own additions: a failed solve has rho = -1 (its x is undefined, so computeScale is not used), and each
trial appends 1 (accepted) / 0 to a trace of at most 255 entries while counting every trial."""
import ctypes
import importlib.util
import math
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG_DIR = os.path.join(ROOT, "self_commit_orb-slam2_b200")
HARNESS = os.path.join(ROOT, "tests", "cpp", "levenberg_harness.cu")
DBL_MAX = sys.float_info.max


class _State(ctypes.Structure):
    _fields_ = [("lam", ctypes.c_double), ("ni", ctypes.c_double), ("currentChi", ctypes.c_double),
                ("iniChi", ctypes.c_double), ("rho", ctypes.c_double), ("qmax", ctypes.c_int), ("nBad", ctypes.c_int),
                ("nTrials", ctypes.c_int)]


def _nvcc():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    return nvcc if os.path.exists(nvcc) else shutil.which("nvcc")


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    spec = importlib.util.spec_from_file_location("_lm_product_build", os.path.join(PKG_DIR, "build.py"))
    bld = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bld)
    so = str(tmp_path_factory.mktemp("levenberg_harness") / "liblevenberg.so")
    out = subprocess.run([nvcc] + bld.NVCC_FLAGS + ["-shared", "-I", os.path.join(PKG_DIR, "csrc"), "-o", so, HARNESS],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    assert out.returncode == 0, out.stdout.decode()
    L = ctypes.CDLL(so)
    P, I, D = ctypes.c_void_p, ctypes.c_int, ctypes.c_double
    L.lm_state_size.restype = I
    L.lm_init_lambda.argtypes = [P, D]
    L.lm_init_lambda.restype = None
    L.lm_begin.argtypes = [P, D]
    L.lm_begin.restype = None
    L.lm_trial.argtypes = [P, I, D, D, P]
    L.lm_trial.restype = I
    L.lm_retry.argtypes = [P, I]
    L.lm_retry.restype = I
    L.lm_end_iteration.argtypes = [P]
    L.lm_end_iteration.restype = I
    return L


class Lm:
    """The controller behind the harness, with a 256-entry trace (filled with 7 so untouched entries show)."""

    def __init__(self, L, lam0):
        self.L, self.s = L, _State()
        self.trace = np.full(256, 7, np.int32)
        L.lm_init_lambda(ctypes.byref(self.s), lam0)

    def begin(self, chi):
        self.L.lm_begin(ctypes.byref(self.s), chi)

    def trial(self, solved, temp, scale):
        return bool(self.L.lm_trial(ctypes.byref(self.s), int(solved), temp, scale, self.trace.ctypes.data))

    def retry(self, stop=False):
        return bool(self.L.lm_retry(ctypes.byref(self.s), int(stop)))

    def end_iteration(self):
        return bool(self.L.lm_end_iteration(ctypes.byref(self.s)))

    def __getattr__(self, k):
        return getattr(self.s, k)


def rho_of(cur, temp, scale):
    return (cur - temp) / (scale + 1e-3)  # :130-133


def good_factor(rho):
    return max(1 / 3, min(1 - (2 * rho - 1) ** 3, 2 / 3))  # :136-139


def test_state_layout(lib):
    assert lib.lm_state_size() == ctypes.sizeof(_State)


def test_accept_reaches_the_upper_cap_and_the_lower_floor(lib):
    lm = Lm(lib, 1.0)
    assert (lm.ni, lm.nBad, lm.nTrials) == (2, 0, 0)
    lm.begin(100.0)
    assert (lm.currentChi, lm.iniChi, lm.rho, lm.qmax) == (100.0, 100.0, 0.0, 0)
    scale = 100.0 - 1e-3  # rho ~ 0.5: 1 - (2 rho - 1)^3 ~ 1, cut to 2/3
    assert lm.trial(True, 50.0, scale)
    assert lm.rho == rho_of(100.0, 50.0, scale) and abs(lm.rho - 0.5) < 1e-12
    assert lm.lam == 2 / 3 and lm.ni == 2 and lm.currentChi == 50.0 and lm.qmax == 1
    assert not lm.retry()
    assert not lm.end_iteration()  # a large gain: nBad stays 0
    assert lm.nBad == 0

    lm.begin(50.0)
    assert lm.trial(True, 0.0, 50.0 - 1e-3)  # rho ~ 1: 1 - 1 = 0, raised to 1/3
    assert lm.lam == (2 / 3) * (1 / 3)
    lm.begin(10.0)
    lam = lm.lam
    assert lm.trial(True, 1.0, 10.0 - 1e-3)  # rho ~ 0.9: between the bounds
    r = rho_of(10.0, 1.0, 10.0 - 1e-3)
    assert 1 / 3 < 1 - (2 * r - 1) ** 3 < 2 / 3
    assert lm.lam == lam * good_factor(r)
    assert lm.trace[:4].tolist() == [1, 1, 1, 7] and lm.nTrials == 3


def test_reject_then_accept(lib):
    lm = Lm(lib, 1e-3)
    lm.begin(10.0)
    assert not lm.trial(True, 12.0, 1.0)
    assert lm.lam == 2e-3 and lm.ni == 4 and lm.currentChi == 10.0 and lm.rho < 0
    assert lm.retry()
    assert lm.trial(True, 5.0, 10.0)
    assert lm.lam == 2e-3 * good_factor(rho_of(10.0, 5.0, 10.0)) and lm.ni == 2 and lm.currentChi == 5.0
    assert not lm.retry()
    assert (lm.qmax, lm.nTrials) == (2, 2) and lm.trace[:3].tolist() == [0, 1, 7]
    assert not lm.end_iteration() and lm.nBad == 0


def test_failed_solve_is_a_rejection(lib):
    lm = Lm(lib, 1.0)
    lm.begin(10.0)
    assert not lm.trial(False, 1.0, 5.0)  # a smaller chi2, but the solve failed
    assert lm.rho == -1 and lm.lam == 2 and lm.ni == 4 and lm.currentChi == 10.0
    assert lm.retry() and lm.trace[0] == 0


def test_non_finite_trial_chi2(lib):
    lm = Lm(lib, 1.0)
    lm.begin(10.0)
    assert not lm.trial(True, math.inf, 1.0)  # rho = -inf: rejected, tried again
    assert lm.rho == -math.inf and lm.retry() and lm.lam == 2
    assert not lm.trial(True, -math.inf, 1.0)  # rho = +inf > 0, but tempChi is not finite
    assert lm.rho == math.inf and lm.lam == 8 and lm.currentChi == 10.0
    assert not lm.retry()  # rho > 0: no further trial
    assert not lm.end_iteration() and lm.nBad == 1  # no gain: a bad iteration
    lm.begin(10.0)
    assert not lm.trial(True, math.nan, 1.0)  # rho = NaN: neither accepted nor retried
    assert math.isnan(lm.rho) and not lm.retry() and lm.currentChi == 10.0
    assert not lm.end_iteration() and lm.nBad == 2
    assert lm.trace[:4].tolist() == [0, 0, 0, 7]


def test_ten_rejections_end_the_optimisation(lib):
    lm = Lm(lib, 1.0)
    lm.begin(10.0)
    n = 0
    while True:
        assert not lm.trial(True, 11.0, 1.0)
        n += 1
        if not lm.retry():
            break
    assert n == 10 and lm.qmax == 10
    assert lm.lam == 2.0 ** sum(range(1, 11)) and lm.ni == 2.0 ** 11
    assert lm.end_iteration()
    assert lm.trace[:11].tolist() == [0] * 10 + [7]


def test_zero_gain_ends_the_optimisation(lib):
    lm = Lm(lib, 1.0)
    lm.begin(10.0)
    assert not lm.trial(True, 10.0, 1.0)  # rho == 0: rejected, not retried
    assert lm.rho == 0 and lm.lam == 2 and not lm.retry()
    assert lm.end_iteration()


def small_gain_iteration(lm, chi, accept_to):
    lm.begin(chi)
    assert lm.trial(True, accept_to, 1.0)
    assert not lm.retry()
    return lm.end_iteration()


def test_three_small_gains_in_a_row_end_the_optimisation(lib):
    lm = Lm(lib, 1.0)
    assert not small_gain_iteration(lm, 1000.0, 999.5) and lm.nBad == 1  # (1000 - 999.5) * 1e3 < 1000
    assert not small_gain_iteration(lm, 999.5, 999.4) and lm.nBad == 2
    assert small_gain_iteration(lm, 999.4, 999.3) and lm.nBad == 3


def test_a_good_iteration_resets_the_small_gain_count(lib):
    lm = Lm(lib, 1.0)
    assert not small_gain_iteration(lm, 1000.0, 999.9)
    assert not small_gain_iteration(lm, 999.9, 999.8) and lm.nBad == 2
    assert not small_gain_iteration(lm, 999.8, 500.0) and lm.nBad == 0  # (999.8 - 500) * 1e3 >= 999.8
    assert not small_gain_iteration(lm, 500.0, 499.9)
    assert not small_gain_iteration(lm, 499.9, 499.8) and lm.nBad == 2
    assert small_gain_iteration(lm, 499.8, 499.7)


def test_stop_flag_cuts_the_retries(lib):
    lm = Lm(lib, 1.0)
    lm.begin(10.0)
    assert not lm.trial(True, 11.0, 1.0)
    assert lm.retry(stop=False)
    assert not lm.retry(stop=True)
    assert not lm.end_iteration()  # the stop request, not the policy, ends the loop


def test_trace_is_capped_at_255_entries(lib):
    lm = Lm(lib, 1.0)
    want = []
    for k in range(300):
        lm.begin(10.0)
        good = k % 3 == 0
        assert lm.trial(True, 9.0 if good else 11.0, 1.0) == good
        want.append(int(good))
    assert lm.nTrials == 300
    assert lm.trace[:255].tolist() == want[:255]
    assert lm.trace[255] == 7  # never written: the caller puts the -1 terminator at min(nTrials, 255)
