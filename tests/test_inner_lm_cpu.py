"""The per-point Levenberg-Marquardt rules of the inner iterations (csrc/pxr_lm.cuh: inner_start, inner_judge,
inner_propose), compiled for the host and driven on seeded three-parameter least-squares problems:
- bit for bit against the rules the step kernel carried before they moved to pxr_lm.cuh (copied below): every
  candidate, accept / reject, radius, decrease factor and the final point;
- against the oracle's TrustRegionMinimizer (oracle/orc_trust_region.h) under default TROptions: the same accept /
  reject / invalid sequence and stop reason, and the final point to 1e-10 relative (not to the bit: the oracle forms
  D² as c/(radius·s·s), the gradient norm through Plus and the model cost change from J and r);
- on the edge cases: a non-finite start cost, an indefinite H, a vanishing gradient at the start, the iteration cap,
  and every tolerance and limit exactly on its threshold."""
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

# stop reasons: pxr_lm.cuh's TR_* codes; -1 is a start cost that is not finite
CONTINUE, MAX_ITERATIONS, GRADIENT_TOLERANCE, MIN_RADIUS, PARAMETER_TOLERANCE, FUNCTION_TOLERANCE, INVALID_STEPS = range(7)
START_NOT_FINITE = -1

SHIM = r"""
#include <cstring>
#include <limits>
#include <string>
#include "pxr_lm.cuh"
#include "orc_trust_region.h"

using pxr::InnerState;

namespace {

// ---- the rules as pxr_inner.cuh's inner_propose and inner_step_point held them, before they moved to pxr_lm.cuh
// (only the evaluation and the parameter-set writes are left out of old_step)
bool old_propose(InnerState& s) {
  // ceres Solver::Options defaults (CoordinateDescentMinimizer::Solve)
  const int max_iter = 50, max_invalid = 5;
  const double gtol = 1e-10, min_radius = 1e-32, min_diag = 1e-6, max_diag = 1e32;
  for (;;) {
    s.iter += 1;
    if (s.iter - 1 >= max_iter) return false;
    if (s.gmax <= gtol) return false;
    if (s.radius < min_radius) return false;
    const double diag[3] = {s.H[0], s.H[3], s.H[5]};
    double D2[3];
    for (int k = 0; k < 3; ++k) {
      const double s2 = s.sc[k] * s.sc[k];
      D2[k] = fmin(fmax(diag[k] * s2, min_diag), max_diag) / (s.radius * s2);
    }
    const double Hf[9] = {s.H[0], s.H[1], s.H[2], s.H[1], s.H[3], s.H[4], s.H[2], s.H[4], s.H[5]};
    double inv[9];
    bool valid = pxr::inv3_sym(Hf, D2, inv);
    double d[3] = {0, 0, 0}, mcc = 0;
    if (valid) {
      for (int k = 0; k < 3; ++k) d[k] = -(inv[k * 3] * s.g[0] + inv[k * 3 + 1] * s.g[1] + inv[k * 3 + 2] * s.g[2]);
      double gd = 0, dHd = 0;
      for (int k = 0; k < 3; ++k) {
        gd += s.g[k] * d[k];
        dHd += d[k] * (Hf[k * 3] * d[0] + Hf[k * 3 + 1] * d[1] + Hf[k * 3 + 2] * d[2]);
      }
      mcc = -gd - 0.5 * dHd;
      valid = std::isfinite(d[0]) && std::isfinite(d[1]) && std::isfinite(d[2]) && mcc > 0.0;
    }
    if (!valid) {
      if (++s.invalid >= max_invalid) return false;
      s.radius /= s.decf; s.decf *= 2.0;
      continue;
    }
    s.invalid = 0;
    s.mcc = mcc;
    for (int k = 0; k < 3; ++k) s.cand[k] = s.x[k] + d[k];
    return true;
  }
}

bool old_step(InnerState& s, int phase, double cost, const double* H, const double* g) {
  if (phase == 0) { s.iter = 0; s.invalid = 0; }
  const double ftol = 1e-6, ptol = 1e-8, min_rel_dec = 1e-3, max_radius = 1e16;
  bool go = true;
  if (phase == 0) {
    if (!std::isfinite(cost)) go = false;
    s.cost = s.current_cost = cost;
    for (int k = 0; k < 6; ++k) s.H[k] = H[k];
    for (int k = 0; k < 3; ++k) s.g[k] = g[k];
    s.sc[0] = 1.0 / (1.0 + sqrt(H[0])); s.sc[1] = 1.0 / (1.0 + sqrt(H[3])); s.sc[2] = 1.0 / (1.0 + sqrt(H[5]));
    s.radius = 1e4; s.decf = 2.0;
    s.xnorm = sqrt(s.x[0] * s.x[0] + s.x[1] * s.x[1] + s.x[2] * s.x[2]);
    s.gmax = fmax(fabs(g[0]), fmax(fabs(g[1]), fabs(g[2])));
  } else {
    const double candidate_cost = std::isfinite(cost) ? cost : 1.7976931348623157e308;
    const double dx = s.cand[0] - s.x[0], dy = s.cand[1] - s.x[1], dz = s.cand[2] - s.x[2];
    const double step_norm = sqrt(dx * dx + dy * dy + dz * dz);
    if (step_norm <= ptol * (s.xnorm + ptol)) go = false;                      // parameter tolerance
    else if (fabs(s.cost - candidate_cost) <= ftol * s.cost) go = false;       // function tolerance
    else {
      const double rel = (s.current_cost - candidate_cost) / s.mcc;
      if (rel > min_rel_dec) {
        for (int k = 0; k < 3; ++k) { s.x[k] = s.cand[k]; s.g[k] = g[k]; }
        for (int k = 0; k < 6; ++k) s.H[k] = H[k];
        s.xnorm = sqrt(s.x[0] * s.x[0] + s.x[1] * s.x[1] + s.x[2] * s.x[2]);
        s.cost = cost; s.current_cost = candidate_cost;
        s.gmax = fmax(fabs(g[0]), fmax(fabs(g[1]), fabs(g[2])));
        s.radius = s.radius / fmax(1.0 / 3.0, 1.0 - pow(2.0 * rel - 1.0, 3.0));
        s.radius = fmin(max_radius, s.radius);
        s.decf = 2.0;
      } else {
        s.radius /= s.decf; s.decf *= 2.0;
      }
    }
  }
  if (go) go = old_propose(s);
  return go;
}

// ---- the rules as the step kernel calls them (inner_step_point)
bool new_step(InnerState& s, int phase, double cost, const double* H, const double* g, int* why) {
  *why = phase == 0 ? (pxr::inner_start(s, cost, H, g) ? 0 : -1) : pxr::inner_judge(s, cost, H, g);
  if (*why == 0) *why = pxr::inner_propose(s);
  return *why == 0;
}

// ---- the problems.  p = {kind, n, hscale, ...}
//   kind 0: residuals r_i = |x - a_i| - d_i for n anchors (p[3 + 3i ..] = a_i, p[3 + 3n + i] = d_i): J^T J, J^T r;
//   kind 1: cost = x^T Q x / 2 + b^T x + c (p[3..11] = Q, p[12..14] = b, p[15] = c) with the model H = hscale * Q.
struct Problem {
  const double* p;
  int kind() const { return (int)p[0]; }
  int n() const { return (int)p[1]; }
  // cost, H (6 uniques), g; and, for kind 0, the residuals and the Jacobian
  double eval(const double* x, double* H, double* g, double* r = nullptr, double* J = nullptr) const {
    for (int k = 0; k < 6; ++k) H[k] = 0.0;
    for (int k = 0; k < 3; ++k) g[k] = 0.0;
    double cost = 0.0;
    if (kind() == 0) {
      for (int i = 0; i < n(); ++i) {
        const double* a = p + 3 + 3 * i;
        const double dx = x[0] - a[0], dy = x[1] - a[1], dz = x[2] - a[2];
        const double dist = sqrt(dx * dx + dy * dy + dz * dz);
        const double ri = dist - p[3 + 3 * n() + i];
        const double j[3] = {dx / dist, dy / dist, dz / dist};
        cost += 0.5 * ri * ri;
        H[0] += j[0] * j[0]; H[1] += j[0] * j[1]; H[2] += j[0] * j[2];
        H[3] += j[1] * j[1]; H[4] += j[1] * j[2]; H[5] += j[2] * j[2];
        for (int k = 0; k < 3; ++k) g[k] += j[k] * ri;
        if (r) r[i] = ri;
        if (J) for (int k = 0; k < 3; ++k) J[3 * i + k] = j[k];
      }
      for (int k = 0; k < 6; ++k) H[k] *= p[2];
    } else {
      const double* Q = p + 3;
      const double* b = p + 12;
      for (int i = 0; i < 3; ++i) {
        double qx = 0.0;
        for (int k = 0; k < 3; ++k) qx += Q[3 * i + k] * x[k];
        cost += 0.5 * x[i] * qx + b[i] * x[i];
        g[i] = qx + b[i];
      }
      cost += p[15];
      H[0] = p[2] * Q[0]; H[1] = p[2] * Q[1]; H[2] = p[2] * Q[2]; H[3] = p[2] * Q[4]; H[4] = p[2] * Q[5]; H[5] = p[2] * Q[8];
    }
    return cost;
  }
};

// the oracle's view of the same problem
struct Evaluator : orc::TREvaluator {
  Problem P;
  double H[6], g[3], r[64], J[192];
  explicit Evaluator(const double* p) { P.p = p; }
  int NumParameters() const override { return 3; }
  int NumLocal() const override { return 3; }
  bool Evaluate(const double* x, double* cost, bool with_jacobian) override {
    double h[6], gg[3], rr[64], jj[192];
    *cost = P.eval(x, h, gg, rr, jj);
    if (with_jacobian) {
      std::memcpy(H, h, sizeof(H)); std::memcpy(g, gg, sizeof(g));
      std::memcpy(r, rr, sizeof(r)); std::memcpy(J, jj, sizeof(J));
    }
    return std::isfinite(*cost);
  }
  void Gradient(double* out) const override { for (int k = 0; k < 3; ++k) out[k] = g[k]; }
  void SquaredColumnNorm(double* d) const override { d[0] = H[0]; d[1] = H[3]; d[2] = H[5]; }
  bool SolveDamped(const double* D2, double* delta, int* iters) override {
    *iters = 1;
    const double Hf[9] = {H[0], H[1], H[2], H[1], H[3], H[4], H[2], H[4], H[5]};
    double inv[9];
    if (!pxr::inv3_sym(Hf, D2, inv)) return false;
    for (int k = 0; k < 3; ++k) delta[k] = -(inv[3 * k] * g[0] + inv[3 * k + 1] * g[1] + inv[3 * k + 2] * g[2]);
    return true;
  }
  double ModelCostChange(const double* d) const override {
    if (P.kind() == 0 && P.p[2] == 1.0) {     // -(J d)^T (r + J d / 2)
      double m = 0.0;
      for (int i = 0; i < P.n(); ++i) {
        const double jd = J[3 * i] * d[0] + J[3 * i + 1] * d[1] + J[3 * i + 2] * d[2];
        m -= jd * (r[i] + 0.5 * jd);
      }
      return m;
    }
    const double Hf[9] = {H[0], H[1], H[2], H[1], H[3], H[4], H[2], H[4], H[5]};
    double m = 0.0;
    for (int i = 0; i < 3; ++i) m -= d[i] * (g[i] + 0.5 * (Hf[3 * i] * d[0] + Hf[3 * i + 1] * d[1] + Hf[3 * i + 2] * d[2]));
    return m;
  }
  void Plus(const double* x, const double* d, double* out) const override { for (int k = 0; k < 3; ++k) out[k] = x[k] + d[k]; }
};

}  // namespace

extern "C" {

int inner_state_size() { return (int)sizeof(InnerState); }

// One point's solve, as the rounds run it: the start evaluation, then one evaluated candidate per round.  Both rule sets
// run in lockstep; states_new / states_old get the state after every round (at most cap), go_* whether it stays active.
// seq gets 'A' (accepted), 'R' (rejected) and 'I' (invalid) per iteration of the new rules; returns the number of rounds.
int lockstep(const double* p, const double* x0, int cap, InnerState* states_new, InnerState* states_old, int* go_new,
             int* go_old, char* seq, int* why) {
  Problem P{p};
  InnerState sn, so;
  std::memset(&sn, 0, sizeof(sn)); std::memset(&so, 0, sizeof(so));
  for (int k = 0; k < 3; ++k) sn.x[k] = so.x[k] = x0[k];
  sn.active = so.active = 1;
  int n = 0, ns = 0;
  for (int round = 0; round < cap; ++round) {
    double H[6], g[3], Ho[6], go[3];
    const double cost = P.eval(round == 0 ? sn.x : sn.cand, H, g);
    const double cost_o = P.eval(round == 0 ? so.x : so.cand, Ho, go);
    // the new rules as new_step runs them, taken apart to read the sequence
    int w = round == 0 ? (pxr::inner_start(sn, cost, H, g) ? 0 : -1) : pxr::inner_judge(sn, cost, H, g);
    if (round > 0 && w == 0) seq[ns++] = sn.decf == 2.0 ? 'A' : 'R';     // a rejection leaves decf >= 4
    if (w == 0) {
      const int iter0 = sn.iter;
      w = pxr::inner_propose(sn);
      for (int k = iter0 + 1; k < sn.iter; ++k) seq[ns++] = 'I';       // the last iteration proposed or stopped
    }
    *why = w;
    const bool gn = w == 0;
    const bool gold = old_step(so, round == 0 ? 0 : 1, cost_o, Ho, go);
    if (!gn) sn.active = 0;
    if (!gold) so.active = 0;
    states_new[n] = sn; states_old[n] = so; go_new[n] = gn; go_old[n] = gold;
    ++n;
    if (!gn || !gold) break;
  }
  seq[ns] = 0;
  return n;
}

// The oracle's TrustRegionMinimizer on the same problem from x0 (default TROptions): the final point, the sequence in
// the same letters, and the stop reason in pxr_lm.cuh's codes.
void oracle_solve(const double* p, double* x, char* seq, int* why) {
  Evaluator ev(p);
  orc::TrustRegionMinimizer m{orc::TROptions()};
  orc::TRSummary sum;
  m.Minimize(&ev, x, &sum);
  int ns = 0;
  for (size_t i = 1; i < sum.iterations.size(); ++i)
    seq[ns++] = !sum.iterations[i].step_is_valid ? 'I' : sum.iterations[i].step_is_successful ? 'A' : 'R';
  seq[ns] = 0;
  const std::string& msg = sum.message;
  *why = msg == "initial evaluation failed" ? -1 : msg == "Maximum number of iterations reached." ? 1
       : msg == "Gradient tolerance reached." ? 2 : msg == "Minimum trust region radius reached." ? 3
       : msg == "Parameter tolerance reached." ? 4 : msg == "Function tolerance reached." ? 5
       : msg.rfind("Number of consecutive invalid steps", 0) == 0 ? 6 : 99;
}

// One step of both rule sets from a given state: phase 0 takes (cost, H, g) as the start evaluation, phase 1 as the
// candidate's; phase 2 only proposes.  Returns the new rules' stop reason.
int step_from(const InnerState* in, int phase, double cost, const double* H, const double* g, InnerState* out_new,
              InnerState* out_old, int* go_old) {
  *out_new = *in; *out_old = *in;
  int why;
  if (phase == 2) {
    why = pxr::inner_propose(*out_new);
    *go_old = old_propose(*out_old);
  } else {
    new_step(*out_new, phase, cost, H, g, &why);
    *go_old = old_step(*out_old, phase, cost, H, g);
  }
  return why;
}

}
"""


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    gxx = shutil.which("g++")
    if gxx is None or not os.path.exists(os.path.join(CUDA_INCLUDE, "cuda_runtime.h")):
        pytest.skip("needs g++ and the CUDA headers")
    d = tmp_path_factory.mktemp("inner_lm")
    src, lib = d / "shim.cc", d / "libshim.so"
    src.write_text(SHIM)
    subprocess.check_call([gxx, "-O2", "-std=c++17", "-shared", "-fPIC", "-I" + CUDA_INCLUDE, "-I" + CSRC,
                           "-I" + ORACLE, str(src), "-o", str(lib)])
    lib = ctypes.CDLL(str(lib))
    assert lib.inner_state_size() == STATE.itemsize
    return lib


STATE = np.dtype([("x", "3f8"), ("cand", "3f8"), ("cost", "f8"), ("current_cost", "f8"), ("H", "6f8"), ("g", "3f8"),
                  ("sc", "3f8"), ("radius", "f8"), ("decf", "f8"), ("xnorm", "f8"), ("gmax", "f8"), ("mcc", "f8"),
                  ("iter", "i4"), ("invalid", "i4"), ("active", "i4")], align=True)


def _p(a, t=ctypes.c_double):
    return a.ctypes.data_as(ctypes.POINTER(t))


def _same_bits(a, b):
    """every field of two InnerState arrays, bit for bit (the padding is not compared)"""
    for name in STATE.names:
        x, y = np.ascontiguousarray(a[name]), np.ascontiguousarray(b[name])
        if not np.array_equal(x.view(np.uint8), y.view(np.uint8)):
            return False
    return True


def _anchors(rng, n, noise, hscale=1.0):
    """a point located by its distances to n anchors; returns (problem, start point)"""
    x_true = rng.normal(0, 2, 3)
    a = x_true + rng.normal(0, 5, (n, 3))
    d = np.linalg.norm(a - x_true, axis=1) + rng.normal(0, noise, n)
    x0 = x_true + rng.normal(0, 1.5, 3)
    return np.concatenate([[0, n, hscale], a.ravel(), d]), x0


def _quadratic(Q, b, c, hscale=1.0):
    return np.concatenate([[1, 0, hscale], np.asarray(Q, float).ravel(), b, [c]])


def _lockstep(shim, p, x0, cap=200):
    sn, so = np.zeros(cap, STATE), np.zeros(cap, STATE)
    gn, go = np.zeros(cap, np.int32), np.zeros(cap, np.int32)
    seq = ctypes.create_string_buffer(4096)
    why = ctypes.c_int()
    n = shim.lockstep(_p(p), _p(np.asarray(x0, float)), cap, sn.ctypes.data_as(ctypes.c_void_p),
                      so.ctypes.data_as(ctypes.c_void_p), _p(gn, ctypes.c_int), _p(go, ctypes.c_int), seq, ctypes.byref(why))
    assert n < cap
    return sn[:n], so[:n], gn[:n], go[:n], seq.value.decode(), why.value


def _oracle(shim, p, x0):
    x = np.array(x0, float)
    seq = ctypes.create_string_buffer(4096)
    why = ctypes.c_int()
    shim.oracle_solve(_p(p), _p(x), seq, ctypes.byref(why))
    return x, seq.value.decode(), why.value


def _check(shim, p, x0):
    """both rule sets bit for bit, and the new ones against the oracle; returns (sequence, stop reason, final point)"""
    sn, so, gn, go, seq, why = _lockstep(shim, p, x0)
    assert np.array_equal(gn, go)
    assert _same_bits(sn, so)
    assert not gn[-1] and sn[-1]["active"] == 0
    x_final = sn[-1]["x"]
    x_orc, seq_orc, why_orc = _oracle(shim, p, x0)
    assert (seq, why) == (seq_orc, why_orc)
    assert np.linalg.norm(x_final - x_orc) <= 1e-10 * np.linalg.norm(x_orc)
    return seq, why, x_final


@pytest.mark.parametrize("seed", range(12))
def test_anchor_problems(shim, seed):
    rng = np.random.default_rng(seed)
    p, x0 = _anchors(rng, 3 + seed % 6, [0.0, 1e-3, 0.05, 0.5][seed % 4])
    seq, why, x = _check(shim, p, x0)
    assert "A" in seq and why in (GRADIENT_TOLERANCE, PARAMETER_TOLERANCE, FUNCTION_TOLERANCE)


def test_anchor_problems_cover_rejections_and_every_tolerance(shim):
    """across more seeds, with larger start errors, rejected steps and each way a converging solve stops"""
    reasons, rejected = set(), False
    for seed in range(40):
        rng = np.random.default_rng(1000 + seed)
        p, x0 = _anchors(rng, 3 + seed % 4, [0.0, 0.02, 0.3][seed % 3])
        x0 = x0 + rng.normal(0, 4.0, 3)
        seq, why, _ = _check(shim, p, x0)
        reasons.add(why)
        rejected |= "R" in seq
    assert rejected and reasons >= {GRADIENT_TOLERANCE, PARAMETER_TOLERANCE, FUNCTION_TOLERANCE}


def test_start_cost_not_finite(shim):
    p, x0 = _anchors(np.random.default_rng(7), 4, 0.01)
    p[3 + 3 * 4] = np.nan                   # d_0
    seq, why, x = _check(shim, p, x0)
    assert (seq, why) == ("", START_NOT_FINITE) and np.array_equal(x, x0)


def test_indefinite_h_stops_at_the_fifth_invalid_step(shim):
    # H has eigenvalues -1, 1, 3; the damping 1/radius stays below 1 over five radius halvings
    p = _quadratic([[1, 2, 0], [2, 1, 0], [0, 0, 1]], [0.3, -0.2, 0.5], 2.0)
    seq, why, x = _check(shim, p, [0.1, 0.2, 0.3])
    assert (seq, why) == ("IIII", INVALID_STEPS) and np.array_equal(x, [0.1, 0.2, 0.3])


def test_gradient_vanishes_at_the_start(shim):
    rng = np.random.default_rng(3)
    x0 = rng.normal(0, 2, 3)
    a = x0 + rng.normal(0, 5, (4, 3))
    # the distances exactly as the shim computes them, so that every residual and the gradient are 0
    d = [math.sqrt((x0[0] - ai[0]) * (x0[0] - ai[0]) + (x0[1] - ai[1]) * (x0[1] - ai[1]) + (x0[2] - ai[2]) * (x0[2] - ai[2]))
         for ai in a]
    p = np.concatenate([[0, 4, 1.0], a.ravel(), d])
    seq, why, x = _check(shim, p, x0)
    assert (seq, why) == ("", GRADIENT_TOLERANCE) and np.array_equal(x, x0)


def test_iteration_cap(shim):
    # the model's curvature is 100 times the cost's: every step goes about 1 % of the way and is accepted
    p = _quadratic(np.diag([1.0, 2.0, 0.5]), [0.0, 0.0, 0.0], 0.0, hscale=100.0)
    seq, why, x = _check(shim, p, [1.0, -2.0, 3.0])
    assert (seq, why) == ("A" * 50, MAX_ITERATIONS)


# ---- every test on its threshold, from a given state
def _state(**kw):
    s = np.zeros(1, STATE)
    s["x"] = [1.0, 2.0, 3.0]
    s["cand"] = [1.5, 2.0, 3.0]
    s["cost"] = s["current_cost"] = 1e6
    s["H"] = [4.0, 0.5, 0.25, 3.0, 0.5, 2.0]
    s["g"] = [1.0, -2.0, 0.5]
    s["sc"] = [1 / 3, 1 / (1 + math.sqrt(3.0)), 1 / (1 + math.sqrt(2.0))]
    s["radius"], s["decf"], s["xnorm"], s["gmax"], s["mcc"] = 1e4, 2.0, math.sqrt(14.0), 2.0, 1e6
    s["active"] = 1
    for k, v in kw.items():
        s[k] = v
    return s


def _step(shim, s, phase, cost=0.0, H=(4.0, 0.5, 0.25, 3.0, 0.5, 2.0), g=(1.0, -2.0, 0.5)):
    out_new, out_old = np.zeros(1, STATE), np.zeros(1, STATE)
    go_old = ctypes.c_int()
    why = shim.step_from(s.ctypes.data_as(ctypes.c_void_p), phase, ctypes.c_double(cost), _p(np.array(H, float)),
                         _p(np.array(g, float)), out_new.ctypes.data_as(ctypes.c_void_p),
                         out_old.ctypes.data_as(ctypes.c_void_p), ctypes.byref(go_old))
    assert _same_bits(out_new, out_old) and bool(go_old.value) == (why == CONTINUE)
    return why, out_new[0]


def test_parameter_tolerance_on_its_threshold(shim):
    t = 1e-8 * (0.0 + 1e-8)                      # ptol * (|x| + ptol) at x = 0
    why, _ = _step(shim, _state(x=[0, 0, 0], xnorm=0.0, cand=[t, 0, 0]), 1, cost=5e5)
    assert why == PARAMETER_TOLERANCE
    why, s = _step(shim, _state(x=[0, 0, 0], xnorm=0.0, cand=[np.nextafter(t, 1), 0, 0]), 1, cost=5e5)
    assert why == CONTINUE and s["decf"] == 2.0   # accepted, and a new candidate proposed


def test_function_tolerance_on_its_threshold(shim):
    assert 1e-6 * 1e6 == 1.0 and 1e6 - 999999.0 == 1.0
    why, _ = _step(shim, _state(), 1, cost=999999.0)
    assert why == FUNCTION_TOLERANCE
    why, _ = _step(shim, _state(), 1, cost=np.nextafter(999999.0, 0))
    assert why == CONTINUE


def test_min_relative_decrease_on_its_threshold(shim):
    assert (1e6 - 999000.0) / 1e6 == 1e-3
    why, s = _step(shim, _state(), 1, cost=999000.0)
    assert why == CONTINUE and s["decf"] == 4.0 and np.array_equal(s["x"], [1.0, 2.0, 3.0])       # rejected
    why, s = _step(shim, _state(), 1, cost=np.nextafter(999000.0, 0))
    assert why == CONTINUE and s["decf"] == 2.0 and np.array_equal(s["x"], [1.5, 2.0, 3.0])       # accepted


def test_gradient_tolerance_on_its_threshold(shim):
    assert _step(shim, _state(gmax=1e-10), 2)[0] == GRADIENT_TOLERANCE
    assert _step(shim, _state(gmax=np.nextafter(1e-10, 1)), 2)[0] == CONTINUE


def test_min_radius_on_its_threshold(shim):
    assert _step(shim, _state(radius=np.nextafter(1e-32, 0)), 2)[0] == MIN_RADIUS
    why, s = _step(shim, _state(radius=1e-32), 2)
    assert why == CONTINUE and s["iter"] == 1


def test_iteration_limit_on_its_threshold(shim):
    assert _step(shim, _state(iter=50), 2)[0] == MAX_ITERATIONS
    why, s = _step(shim, _state(iter=49), 2)
    assert why == CONTINUE and s["iter"] == 50


def test_invalid_step_limit(shim):
    H = (1.0, 2.0, 0.0, 1.0, 0.0, 1.0)           # indefinite
    why, s = _step(shim, _state(H=H, invalid=3), 2)
    assert why == INVALID_STEPS and s["iter"] == 2 and s["invalid"] == 5 and s["radius"] == 5e3 and s["decf"] == 4.0
    why, s = _step(shim, _state(H=H, invalid=4), 2)
    assert why == INVALID_STEPS and s["iter"] == 1 and s["radius"] == 1e4


def test_start_state(shim):
    """inner_start against the old phase 0, on a finite and a non-finite start cost"""
    for cost, want in ((3.5, CONTINUE), (np.inf, START_NOT_FINITE), (np.nan, START_NOT_FINITE)):
        why, s = _step(shim, _state(iter=7, invalid=2, radius=3.0, decf=16.0), 0, cost=cost)
        assert why == want and s["radius"] == 1e4 and s["decf"] == 2.0 and s["invalid"] == 0
        assert s["iter"] == (0 if want == START_NOT_FINITE else 1)
