// pxr_lm.cuh — the trust-region rules of ceres' TrustRegionMinimizer + LevenbergMarquardtStrategy (Ceres 2.1,
// DESIGN §4), shared by the BA driver on the host (pxr_ba.cu), the one-CTA-per-problem solvers on the device
// (pxr_ka.cu, pxr_qba.cu) and the per-point inner iterations (pxr_inner.cuh).  Every expression keeps one shape on
// both sides: the host results and nvcc's FMA contraction depend on it.
#pragma once
#include <cuda_runtime.h>
#include <math.h>

namespace pxr {

// ceres::internal::TrustRegionStepEvaluator (Conn, Gould & Toint, algorithm 10.1.2), as
// oracle/orc_trust_region.h::StepEvaluator; max_nonmonotonic == 0 is the monotonic minimizer.
struct StepEvaluator {
  int max_nonmonotonic, num_consecutive_nonmonotonic_steps;
  double minimum_cost, current_cost, reference_cost, candidate_cost, acc_reference, acc_candidate;
  __host__ __device__ __forceinline__ void init(double cost, int max_nm) {
    max_nonmonotonic = max_nm; num_consecutive_nonmonotonic_steps = 0;
    minimum_cost = current_cost = reference_cost = candidate_cost = cost;
    acc_reference = acc_candidate = 0.0;
  }
  __host__ __device__ __forceinline__ double quality(double cost, double model_cost_change) const {
    if (cost >= 1.7976931348623157e308) return -1.7976931348623157e308;
    const double relative = (current_cost - cost) / model_cost_change;
    const double historical = (reference_cost - cost) / (acc_reference + model_cost_change);
    return relative < historical ? historical : relative;     // std::max: a NaN relative decrease propagates
  }
  __host__ __device__ __forceinline__ void accepted(double cost, double model_cost_change) {
    current_cost = cost; acc_candidate += model_cost_change; acc_reference += model_cost_change;
    if (cost < minimum_cost) {
      minimum_cost = cost; num_consecutive_nonmonotonic_steps = 0; candidate_cost = cost; acc_candidate = 0.0;
    } else {
      ++num_consecutive_nonmonotonic_steps;
      if (cost > candidate_cost) { candidate_cost = cost; acc_candidate = 0.0; }
    }
    if (num_consecutive_nonmonotonic_steps == max_nonmonotonic) { reference_cost = candidate_cost; acc_reference = acc_candidate; }
  }
};

// The options the rules read: the host fills them from pxr_solver_options, the kernels from their arguments.
struct TrustRegionOptions {
  int max_consecutive_invalid_steps, max_nonmonotonic;    // max_nonmonotonic: 0 unless use_nonmonotonic_steps
  double initial_radius, max_radius, min_radius;
  double gradient_tolerance, parameter_tolerance, function_tolerance, min_relative_decrease;
};

// Why a solve stops (tr_stop and tr_tolerance); 0 lets it go on.  TR_MAX_ITERATIONS is termination 1 (NO_CONVERGENCE),
// the others 0 (CONVERGENCE); too many invalid steps (tr_invalid_stop; TR_INVALID_STEPS where a code reports it) is 2
// (FAILURE).
enum { TR_CONTINUE = 0, TR_MAX_ITERATIONS, TR_GRADIENT_TOLERANCE, TR_MIN_RADIUS, TR_PARAMETER_TOLERANCE, TR_FUNCTION_TOLERANCE,
       TR_INVALID_STEPS };

// The rules on a radius and decrease factor held anywhere: in TrustRegion below, or in CTA control slots that one
// thread updates (ka_solve_kernel).
// FinalizeIterationAndCheckIfMinimizerCanContinue, before the next step
__host__ __device__ __forceinline__ int tr_stop(const TrustRegionOptions& o, double radius, int iteration, int max_iteration,
                                                double gradient_max_norm) {
  if (iteration >= max_iteration) return TR_MAX_ITERATIONS;
  if (gradient_max_norm <= o.gradient_tolerance) return TR_GRADIENT_TOLERANCE;
  if (radius < o.min_radius) return TR_MIN_RADIUS;
  return TR_CONTINUE;
}
// HandleInvalidStep: true when this invalid step ends the solve; otherwise the caller applies tr_reject
__host__ __device__ __forceinline__ bool tr_invalid_stop(const TrustRegionOptions& o, int& num_invalid) {
  return ++num_invalid >= o.max_consecutive_invalid_steps;
}
// ParameterToleranceReached, then FunctionToleranceReached; the step is not applied when either is
__host__ __device__ __forceinline__ int tr_tolerance(const TrustRegionOptions& o, double step_norm, double x_norm,
                                                     double cost_change, double x_cost) {
  if (step_norm <= o.parameter_tolerance * (x_norm + o.parameter_tolerance)) return TR_PARAMETER_TOLERANCE;
  if (fabs(cost_change) <= o.function_tolerance * x_cost) return TR_FUNCTION_TOLERANCE;
  return TR_CONTINUE;
}
__host__ __device__ __forceinline__ bool tr_successful(const TrustRegionOptions& o, double relative_decrease) {
  return relative_decrease > o.min_relative_decrease;
}
// LevenbergMarquardtStrategy::StepAccepted.  The comparisons are std::max(1/3, ·) and std::min(max_radius, ·): a NaN
// right operand gives the left one, as fmax / fmin do.
__host__ __device__ __forceinline__ void tr_accept(const TrustRegionOptions& o, double& radius, double& decrease_factor,
                                                   double relative_decrease) {
  const double shrink = 1.0 - pow(2.0 * relative_decrease - 1.0, 3.0);
  radius = radius / (1.0 / 3.0 < shrink ? shrink : 1.0 / 3.0);
  radius = radius < o.max_radius ? radius : o.max_radius;
  decrease_factor = 2.0;
}
// LevenbergMarquardtStrategy::StepRejected (StepIsInvalid too)
__host__ __device__ __forceinline__ void tr_reject(double& radius, double& decrease_factor) {
  radius /= decrease_factor;
  decrease_factor *= 2.0;
}

// LevenbergMarquardtStrategy's radius, the invalid-step count and the step evaluator of one solve, with the rules above.
struct TrustRegion {
  TrustRegionOptions o;
  double radius, decrease_factor;
  int num_invalid;
  StepEvaluator ev;
  __host__ __device__ __forceinline__ void init(const TrustRegionOptions& opts, double cost) {
    o = opts; radius = o.initial_radius; decrease_factor = 2.0; num_invalid = 0;
    ev.init(cost, o.max_nonmonotonic);
  }
  __host__ __device__ __forceinline__ int stop(int iteration, int max_iteration, double gradient_max_norm) const {
    return tr_stop(o, radius, iteration, max_iteration, gradient_max_norm);
  }
  // true when the solve stops; otherwise the radius shrinks
  __host__ __device__ __forceinline__ bool invalid_step() {
    if (tr_invalid_stop(o, num_invalid)) return true;
    reject();
    return false;
  }
  __host__ __device__ __forceinline__ int tolerance(double step_norm, double x_norm, double cost_change, double x_cost) const {
    return tr_tolerance(o, step_norm, x_norm, cost_change, x_cost);
  }
  __host__ __device__ __forceinline__ bool successful(double relative_decrease) const { return tr_successful(o, relative_decrease); }
  __host__ __device__ __forceinline__ void accept(double relative_decrease, double cost, double model_cost_change) {
    tr_accept(o, radius, decrease_factor, relative_decrease);
    ev.accepted(cost, model_cost_change);
  }
  __host__ __device__ __forceinline__ void reject() { tr_reject(radius, decrease_factor); }
};

// Jacobi scaling of one column, 1/(1+sqrt(diag(J^T J))), at the first linearisation (ceres trust_region_minimizer.cc)
__host__ __device__ __forceinline__ double jacobi_scale(double diag) { return 1.0 / (1.0 + sqrt(diag)); }
// LevenbergMarquardtStrategy's damping of one column in the unscaled variables: clamp(diag·s², lo, hi) / (radius·s²)
__host__ __device__ __forceinline__ double lm_damping(double diag, double scale, double radius, double lo, double hi) {
  const double s2 = scale * scale;
  return fmin(fmax(diag * s2, lo), hi) / (radius * s2);
}

// (H + diag(D2))^-1 of a symmetric 3x3 H (row-major, the lower triangle is read) through its Cholesky factor; false
// when H + diag(D2) is not positive definite
__host__ __device__ __forceinline__ bool inv3_sym(const double* H, const double* D2, double inv[9]) {
  const double a = H[0] + D2[0], b = H[1], c = H[2], dd = H[4] + D2[1], e = H[5], f = H[8] + D2[2];
  if (!(a > 0.0)) return false;
  const double l00 = sqrt(a), l10 = b / l00, l20 = c / l00;
  const double t11 = dd - l10 * l10;
  if (!(t11 > 0.0)) return false;
  const double l11 = sqrt(t11), l21 = (e - l20 * l10) / l11;
  const double t22 = f - l20 * l20 - l21 * l21;
  if (!(t22 > 0.0)) return false;
  const double l22 = sqrt(t22);
  const double i00 = 1.0 / l00, i11 = 1.0 / l11, i22 = 1.0 / l22;
  const double i10 = -l10 * i00 * i11;
  const double i21 = -l21 * i11 * i22;
  const double i20 = -(l20 * i00 + l21 * i10) * i22;
  inv[0] = i00 * i00 + i10 * i10 + i20 * i20;
  inv[1] = inv[3] = i10 * i11 + i20 * i21;
  inv[2] = inv[6] = i20 * i22;
  inv[4] = i11 * i11 + i21 * i21;
  inv[5] = inv[7] = i21 * i22;
  inv[8] = i22 * i22;
  return true;
}

// ---- inner iterations: ceres' CoordinateDescentMinimizer solves each 3D point alone, with everything else fixed, by a
// TrustRegionMinimizer under the default Solver::Options (CoordinateDescentMinimizer::Solve builds its
// Minimizer::Options from defaults): monotonic steps and Jacobi scaling.  Those defaults, the same values as the
// oracle's TROptions defaults:
struct InnerOptions {
  TrustRegionOptions tr;
  int max_iterations;
  double min_diagonal, max_diagonal;     // min_lm_diagonal, max_lm_diagonal
};
__host__ __device__ constexpr InnerOptions inner_options() {
  return {{/*max_consecutive_invalid_steps*/ 5, /*max_nonmonotonic*/ 0, /*initial_radius*/ 1e4, /*max_radius*/ 1e16,
           /*min_radius*/ 1e-32, /*gradient_tolerance*/ 1e-10, /*parameter_tolerance*/ 1e-8, /*function_tolerance*/ 1e-6,
           /*min_relative_decrease*/ 1e-3},
          50, 1e-6, 1e32};
}

// One point's solve between evaluations (pxr_inner.cuh keeps one per point and evaluates the candidates).  Evaluations
// give the cost, J^T J (6 uniques: 00 01 02 11 12 22) and J^T r of the point.
struct InnerState {
  double x[3];        // last accepted point
  double cand[3];     // candidate being evaluated (also written to the parameter set)
  double cost, current_cost, H[6], g[3], sc[3];
  double radius, decf, xnorm, gmax, mcc;
  int iter, invalid, active;
};

__host__ __device__ __forceinline__ double inner_gmax(const double g[3]) { return fmax(fabs(g[0]), fmax(fabs(g[1]), fabs(g[2]))); }

// The evaluation at the start point s.x; false when its cost is not finite and the point stays where it is.
__host__ __device__ __forceinline__ bool inner_start(InnerState& s, double cost, const double H[6], const double g[3]) {
  constexpr InnerOptions o = inner_options();
  s.iter = 0; s.invalid = 0;
  s.cost = s.current_cost = cost;
#pragma unroll
  for (int k = 0; k < 6; ++k) s.H[k] = H[k];
#pragma unroll
  for (int k = 0; k < 3; ++k) s.g[k] = g[k];
  s.sc[0] = jacobi_scale(H[0]); s.sc[1] = jacobi_scale(H[3]); s.sc[2] = jacobi_scale(H[5]);
  s.radius = o.tr.initial_radius; s.decf = 2.0;
  s.xnorm = sqrt(s.x[0] * s.x[0] + s.x[1] * s.x[1] + s.x[2] * s.x[2]);
  s.gmax = inner_gmax(g);
  return isfinite(cost);
}

// Judges the evaluated candidate s.cand: accepts or rejects it, or returns the tolerance (TR_PARAMETER_TOLERANCE,
// TR_FUNCTION_TOLERANCE) that ends the solve without applying it.
// The step quality is the relative decrease (current − candidate) / model cost change alone, without a StepEvaluator
// in InnerState (its 56 bytes would be loaded and stored by every round's step kernel): with monotonic steps and
// min_relative_decrease >= 0 that decides every step as ceres' evaluator does (test_trust_region_rules_cpu.py).
__host__ __device__ __forceinline__ int inner_judge(InnerState& s, double cost, const double H[6], const double g[3]) {
  constexpr InnerOptions o = inner_options();
  const double candidate_cost = isfinite(cost) ? cost : 1.7976931348623157e308;
  const double dx = s.cand[0] - s.x[0], dy = s.cand[1] - s.x[1], dz = s.cand[2] - s.x[2];
  const double step_norm = sqrt(dx * dx + dy * dy + dz * dz);
  if (const int tol = tr_tolerance(o.tr, step_norm, s.xnorm, s.cost - candidate_cost, s.cost)) return tol;
  const double rel = (s.current_cost - candidate_cost) / s.mcc;
  if (tr_successful(o.tr, rel)) {
#pragma unroll
    for (int k = 0; k < 3; ++k) { s.x[k] = s.cand[k]; s.g[k] = g[k]; }
#pragma unroll
    for (int k = 0; k < 6; ++k) s.H[k] = H[k];
    s.xnorm = sqrt(s.x[0] * s.x[0] + s.x[1] * s.x[1] + s.x[2] * s.x[2]);
    s.cost = cost; s.current_cost = candidate_cost;
    s.gmax = inner_gmax(g);
    tr_accept(o.tr, s.radius, s.decf, rel);
  } else {
    tr_reject(s.radius, s.decf);
  }
  return TR_CONTINUE;
}

// Proposes the next candidate s.cand from the last accepted point, taking invalid steps in passing; returns TR_CONTINUE,
// or why the solve stops: a tr_stop code, or TR_INVALID_STEPS.
__host__ __device__ __forceinline__ int inner_propose(InnerState& s) {
  constexpr InnerOptions o = inner_options();
  for (;;) {
    s.iter += 1;
    if (const int stop = tr_stop(o.tr, s.radius, s.iter - 1, o.max_iterations, s.gmax)) return stop;
    const double diag[3] = {s.H[0], s.H[3], s.H[5]};
    double D2[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) D2[k] = lm_damping(diag[k], s.sc[k], s.radius, o.min_diagonal, o.max_diagonal);
    const double Hf[9] = {s.H[0], s.H[1], s.H[2], s.H[1], s.H[3], s.H[4], s.H[2], s.H[4], s.H[5]};
    double inv[9];
    bool valid = inv3_sym(Hf, D2, inv);
    double d[3] = {0, 0, 0}, mcc = 0;
    if (valid) {
#pragma unroll
      for (int k = 0; k < 3; ++k) d[k] = -(inv[k * 3] * s.g[0] + inv[k * 3 + 1] * s.g[1] + inv[k * 3 + 2] * s.g[2]);
      double gd = 0, dHd = 0;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        gd += s.g[k] * d[k];
        dHd += d[k] * (Hf[k * 3] * d[0] + Hf[k * 3 + 1] * d[1] + Hf[k * 3 + 2] * d[2]);
      }
      mcc = -gd - 0.5 * dHd;
      valid = isfinite(d[0]) && isfinite(d[1]) && isfinite(d[2]) && mcc > 0.0;
    }
    if (!valid) {
      if (tr_invalid_stop(o.tr, s.invalid)) return TR_INVALID_STEPS;
      tr_reject(s.radius, s.decf);
      continue;
    }
    s.invalid = 0;
    s.mcc = mcc;
#pragma unroll
    for (int k = 0; k < 3; ++k) s.cand[k] = s.x[k] + d[k];
    return TR_CONTINUE;
  }
}

}  // namespace pxr
