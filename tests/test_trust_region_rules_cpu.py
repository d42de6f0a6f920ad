"""The trust-region rules of csrc/pxr_lm.cuh, which the BA driver runs on the host and the KA and QBA kernels run on the
device, compiled for the host and checked bit for bit:
- StepEvaluator against the oracle's restatement of ceres' TrustRegionStepEvaluator (oracle/orc_trust_region.h);
- TrustRegion's radius, decrease factor, invalid-step count and stop codes against the minimizer's rules in
  orc_trust_region.h, restated below;
- on monotonic solves with min_relative_decrease >= 0, the shared evaluator against the shortcut form the KA and QBA
  kernels used before (quality = relative decrease alone, no bookkeeping on acceptance)."""
import ctypes
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "pixel-perfect-sfm_b200", "csrc")
ORACLE = os.path.join(ROOT, "oracle")
CUDA_INCLUDE = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
DBL_MAX = 1.7976931348623157e308

SHIM = r"""
#include "pxr_lm.cuh"
#include "orc_trust_region.h"

extern "C" {

// A sequence of steps: the quality of each from both evaluators, then StepAccepted where accept[i] is set.
void ev_sequence(double c0, int max_nm, int n, const double* cost, const double* mcc, const int* accept,
                 double* q_pxr, double* q_orc) {
  pxr::StepEvaluator e; e.init(c0, max_nm);
  orc::StepEvaluator r(c0, max_nm);
  for (int i = 0; i < n; ++i) {
    q_pxr[i] = e.quality(cost[i], mcc[i]);
    q_orc[i] = r.StepQuality(cost[i], mcc[i]);
    if (accept[i]) { e.accepted(cost[i], mcc[i]); r.StepAccepted(cost[i], mcc[i]); }
  }
}

// A scripted solve.  Per iteration i: the stop test at (iteration[i], gmax[i]); valid[i] == 0 is an invalid step,
// otherwise the tolerance test, then the step quality and accept or reject.  Every rule runs whatever the previous one
// returned, so that each is exercised on many states.  rec[i] = {radius, decrease_factor, relative decrease},
// codes[i] = {stop, invalid_step, tolerance, successful, num_invalid}.
void tr_script(const double* od, const int* oi, double c0, int n, const int* iteration, int max_iteration,
               const double* gmax, const int* valid, const double* step_norm, const double* x_norm, const double* cost,
               const double* mcc, double* rec, int* codes) {
  pxr::TrustRegionOptions o;
  o.max_consecutive_invalid_steps = oi[0]; o.max_nonmonotonic = oi[1];
  o.initial_radius = od[0]; o.max_radius = od[1]; o.min_radius = od[2]; o.gradient_tolerance = od[3];
  o.parameter_tolerance = od[4]; o.function_tolerance = od[5]; o.min_relative_decrease = od[6];
  pxr::TrustRegion tr; tr.init(o, c0);
  double x_cost = c0;
  for (int i = 0; i < n; ++i) {
    int* c = codes + 5 * i;
    double rel = 0.0;
    c[0] = tr.stop(iteration[i], max_iteration, gmax[i]);
    c[1] = c[2] = c[3] = 0;
    if (!valid[i]) {
      c[1] = tr.invalid_step() ? 1 : 0;
    } else {
      tr.num_invalid = 0;
      c[2] = tr.tolerance(step_norm[i], x_norm[i], x_cost - cost[i], x_cost);
      rel = tr.ev.quality(cost[i], mcc[i]);
      c[3] = tr.successful(rel) ? 1 : 0;
      if (c[3]) { tr.accept(rel, cost[i], mcc[i]); x_cost = cost[i]; } else tr.reject();
    }
    c[4] = tr.num_invalid;
    rec[3 * i] = tr.radius; rec[3 * i + 1] = tr.decrease_factor; rec[3 * i + 2] = rel;
  }
}

}
"""


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    gxx = shutil.which("g++")
    if gxx is None or not os.path.exists(os.path.join(CUDA_INCLUDE, "cuda_runtime.h")):
        pytest.skip("needs g++ and the CUDA headers")
    d = tmp_path_factory.mktemp("trust_region")
    src, lib = d / "shim.cc", d / "libshim.so"
    src.write_text(SHIM)
    subprocess.check_call([gxx, "-O2", "-std=c++17", "-shared", "-fPIC", "-I" + CUDA_INCLUDE, "-I" + CSRC,
                           "-I" + ORACLE, str(src), "-o", str(lib)])
    return ctypes.CDLL(str(lib))


def _p(a, t=ctypes.c_double):
    return a.ctypes.data_as(ctypes.POINTER(t))


def _bits(a):
    return np.asarray(a, np.float64).view(np.uint64)


def _steps(rng, n, c0):
    """Costs around a decreasing trajectory, with increases, equal costs and non-finite trial costs mixed in."""
    cost = np.empty(n)
    c = c0
    for i in range(n):
        u = rng.random()
        if u < 0.05:
            cost[i] = DBL_MAX                     # a trial cost that was not finite
        elif u < 0.1:
            cost[i] = c                           # no change
        else:
            cost[i] = c * (1.0 + rng.normal(-0.05, 0.1))
            if rng.random() < 0.7:
                c = cost[i]
    mcc = np.abs(rng.normal(0.05, 0.05, n)) * c0 + 1e-300
    return cost, mcc


def _ev_sequence(shim, c0, max_nm, cost, mcc, accept):
    n = len(cost)
    q1, q2 = np.zeros(n), np.zeros(n)
    acc = np.ascontiguousarray(accept, np.int32)
    shim.ev_sequence(ctypes.c_double(c0), max_nm, n, _p(cost), _p(mcc), _p(acc, ctypes.c_int), _p(q1), _p(q2))
    return q1, q2


@pytest.mark.parametrize("max_nm", [0, 1, 3, 5])
@pytest.mark.parametrize("seed", range(4))
def test_step_evaluator_matches_oracle(shim, max_nm, seed):
    rng = np.random.default_rng(seed)
    cost, mcc = _steps(rng, 400, 10.0)
    accept = (rng.random(400) < 0.6) & (cost < DBL_MAX)
    q_pxr, q_orc = _ev_sequence(shim, 10.0, max_nm, cost, mcc, accept)
    assert np.array_equal(_bits(q_pxr), _bits(q_orc))


# ---- orc_trust_region.h's minimizer rules, restated
class _OrcEvaluator:
    def __init__(self, c0, max_nm):
        self.max_nm, self.n_nm = max_nm, 0
        self.minimum = self.current = self.reference = self.candidate = c0
        self.acc_ref = self.acc_cand = 0.0

    def quality(self, cost, mcc):
        if cost >= DBL_MAX:
            return -DBL_MAX
        r1 = (self.current - cost) / mcc
        r2 = (self.reference - cost) / (self.acc_ref + mcc)
        return r2 if r1 < r2 else r1              # std::max

    def accepted(self, cost, mcc):
        self.current = cost
        self.acc_cand += mcc
        self.acc_ref += mcc
        if cost < self.minimum:
            self.minimum, self.n_nm, self.candidate, self.acc_cand = cost, 0, cost, 0.0
        else:
            self.n_nm += 1
            if cost > self.candidate:
                self.candidate, self.acc_cand = cost, 0.0
        if self.n_nm == self.max_nm:
            self.reference, self.acc_ref = self.candidate, self.acc_cand


def _orc_script(o, c0, iteration, max_iteration, gmax, valid, step_norm, x_norm, cost, mcc):
    (radius0, max_radius, min_radius, gtol, ptol, ftol, min_rel), (max_invalid, max_nm) = o
    radius, decf, n_invalid, x_cost = radius0, 2.0, 0, c0
    ev = _OrcEvaluator(c0, max_nm)
    rec, codes = [], []
    for i in range(len(cost)):
        if iteration[i] >= max_iteration:
            stop = 1
        elif gmax[i] <= gtol:
            stop = 2
        elif radius < min_radius:
            stop = 3
        else:
            stop = 0
        inv = tol = ok = 0
        rel = 0.0
        if not valid[i]:
            n_invalid += 1
            if n_invalid >= max_invalid:
                inv = 1
            else:
                radius, decf = radius / decf, decf * 2.0
        else:
            n_invalid = 0
            if step_norm[i] <= ptol * (x_norm[i] + ptol):
                tol = 4
            elif abs(x_cost - cost[i]) <= ftol * x_cost:
                tol = 5
            rel = ev.quality(cost[i], mcc[i])
            ok = 1 if rel > min_rel else 0
            if ok:
                shrink = 1.0 - math.pow(2.0 * rel - 1.0, 3.0)
                radius = radius / (shrink if 1.0 / 3.0 < shrink else 1.0 / 3.0)
                radius = radius if radius < max_radius else max_radius
                decf = 2.0
                ev.accepted(cost[i], mcc[i])
                x_cost = cost[i]
            else:
                radius, decf = radius / decf, decf * 2.0
        rec.append((radius, decf, rel))
        codes.append((stop, inv, tol, ok, n_invalid))
    return np.array(rec), np.array(codes, np.int32)


@pytest.mark.parametrize("max_nm", [0, 2])
@pytest.mark.parametrize("seed", range(6))
def test_trust_region_matches_oracle_rules(shim, max_nm, seed):
    rng = np.random.default_rng(100 + seed)
    n = 300
    c0 = 5.0
    cost, mcc = _steps(rng, n, c0)
    od = np.array([1e4, 1e6 if seed % 2 else 1e16, 1e-3 if seed % 3 == 0 else 1e-32, 1e-4, 1e-3, 1e-4,
                   -0.5 if seed == 5 else 1e-3])
    oi = np.array([3, max_nm], np.int32)
    iteration = rng.integers(0, 60, n).astype(np.int32)
    gmax = 10.0 ** rng.uniform(-6, 2, n)
    valid = (rng.random(n) < 0.65).astype(np.int32)
    step_norm = 10.0 ** rng.uniform(-5, 0, n)
    x_norm = 10.0 ** rng.uniform(-1, 2, n)
    rec, codes = np.zeros((n, 3)), np.zeros((n, 5), np.int32)
    shim.tr_script(_p(od), _p(oi, ctypes.c_int), ctypes.c_double(c0), n, _p(iteration, ctypes.c_int), 50, _p(gmax),
                   _p(valid, ctypes.c_int), _p(step_norm), _p(x_norm), _p(cost), _p(mcc), _p(rec), _p(codes, ctypes.c_int))
    want_rec, want_codes = _orc_script(((*od,), (3, max_nm)), c0, iteration, 50, gmax, valid, step_norm, x_norm, cost, mcc)
    assert np.array_equal(codes, want_codes)
    assert np.array_equal(_bits(rec), _bits(want_rec))
    assert set(codes[:, 0]) >= {0, 1, 2} and codes[:, 1].any() and codes[:, 3].any() and not codes[:, 3].all()


def test_trust_region_thresholds(shim):
    """Every test on its threshold, in exactly representable numbers: the iteration limit, the gradient tolerance, the
    minimum radius, the parameter and function tolerances, min_relative_decrease and the invalid-step limit."""
    c0 = 2.0
    od = np.array([1.0, 1e16, 0.25, 1e-4, 0.5, 0.125, 0.25])    # radius0, max, min, gtol, ptol, ftol, min_rel
    oi = np.array([3, 0], np.int32)
    # row 0: iteration == max_iteration; cost_change == ftol * x_cost; quality == min_relative_decrease (rejected)
    # row 1: gmax == gradient_tolerance; step_norm == ptol * (x_norm + ptol); quality 0.5 (accepted, radius unchanged)
    # row 2: an invalid step;  row 3: radius == min_radius, invalid;  row 4: radius < min_radius, the third invalid step
    iteration = np.array([5, 4, 0, 0, 0], np.int32)
    gmax = np.array([1.0, 1e-4, 1.0, 1.0, 1.0])
    valid = np.array([1, 1, 0, 0, 0], np.int32)
    step_norm = np.array([10.0, 0.75, 0, 0, 0])
    x_norm = np.array([1.0, 1.0, 0, 0, 0])
    cost = np.array([1.75, 1.5, 0, 0, 0])
    mcc = np.array([1.0, 1.0, 0, 0, 0])
    n = len(cost)
    rec, codes = np.zeros((n, 3)), np.zeros((n, 5), np.int32)
    shim.tr_script(_p(od), _p(oi, ctypes.c_int), ctypes.c_double(c0), n, _p(iteration, ctypes.c_int), 5, _p(gmax),
                   _p(valid, ctypes.c_int), _p(step_norm), _p(x_norm), _p(cost), _p(mcc), _p(rec), _p(codes, ctypes.c_int))
    # {stop, invalid_step ends the solve, tolerance, successful, num_invalid}
    assert codes.tolist() == [[1, 0, 5, 0, 0], [2, 0, 4, 1, 0], [0, 0, 0, 0, 1], [0, 0, 0, 0, 2], [3, 1, 0, 0, 3]]
    assert rec.tolist() == [[0.5, 4.0, 0.25], [0.5, 2.0, 0.5], [0.25, 4.0, 0.0], [0.0625, 8.0, 0.0], [0.0625, 8.0, 0.0]]
    want_rec, want_codes = _orc_script(((*od,), (3, 0)), c0, iteration, 5, gmax, valid, step_norm, x_norm, cost, mcc)
    assert np.array_equal(codes, want_codes) and np.array_equal(_bits(rec), _bits(want_rec))


class _OldDeviceEvaluator:
    """The evaluator the KA and QBA kernels carried before they shared the host's: in monotonic mode the quality is the
    relative decrease alone (fmax with the historical one otherwise) and an acceptance only moves current_cost."""

    def __init__(self, c0, max_nm):
        self.e = _OrcEvaluator(c0, max_nm)

    def quality(self, cost, mcc):
        e = self.e
        if cost >= DBL_MAX:
            return -DBL_MAX
        rel = (e.current - cost) / mcc
        if e.max_nm > 0:
            rel = float(np.fmax(rel, (e.reference - cost) / (e.acc_ref + mcc)))
        return rel

    def accepted(self, cost, mcc):
        if self.e.max_nm == 0:
            self.e.current = cost
        else:
            self.e.accepted(cost, mcc)


@pytest.mark.parametrize("min_rel", [0.0, 1e-3, 0.25])
@pytest.mark.parametrize("seed", range(4))
def test_monotonic_shortcut_equals_shared_evaluator(shim, min_rel, seed):
    """KA and QBA accept a step when its quality exceeds min_relative_decrease; with min_relative_decrease >= 0 and
    monotonic steps the shared evaluator's qualities, and so every accept decision, are those of the old shortcut."""
    rng = np.random.default_rng(200 + seed)
    cost, mcc = _steps(rng, 400, 3.0)
    old = _OldDeviceEvaluator(3.0, 0)
    q_old, accept = np.zeros(len(cost)), np.zeros(len(cost), bool)
    for i in range(len(cost)):
        q_old[i] = old.quality(cost[i], mcc[i])
        accept[i] = q_old[i] > min_rel
        if accept[i]:
            old.accepted(cost[i], mcc[i])
    assert accept.any() and not accept.all()
    q_new, _ = _ev_sequence(shim, 3.0, 0, cost, mcc, accept)
    assert np.array_equal(_bits(q_new), _bits(q_old))
