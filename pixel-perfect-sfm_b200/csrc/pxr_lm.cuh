// pxr_lm.cuh — the trust-region rules of ceres' TrustRegionMinimizer + LevenbergMarquardtStrategy (Ceres 2.1,
// DESIGN §4), shared by the BA driver on the host (pxr_ba.cu) and the one-CTA-per-problem solvers on the device
// (pxr_ka.cu, pxr_qba.cu).  Every expression keeps one shape on both sides: the host results and nvcc's FMA
// contraction depend on it.
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
// the others 0 (CONVERGENCE); too many invalid steps (tr_invalid_stop) is 2 (FAILURE).
enum { TR_CONTINUE = 0, TR_MAX_ITERATIONS, TR_GRADIENT_TOLERANCE, TR_MIN_RADIUS, TR_PARAMETER_TOLERANCE, TR_FUNCTION_TOLERANCE };

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

}  // namespace pxr
