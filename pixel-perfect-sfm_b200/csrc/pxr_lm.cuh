// pxr_lm.cuh — Levenberg-Marquardt pieces shared by the one-CTA-per-problem solvers (pxr_ka.cu, pxr_qba.cu).
#pragma once
#include <cuda_runtime.h>

namespace pxr {

// ceres::internal::TrustRegionStepEvaluator (Conn, Gould & Toint, algorithm 10.1.2) on chip.  Every input is a
// CTA-uniform value, so each thread may hold its own copy.  max_nonmonotonic == 0 is the monotonic minimizer, whose
// quality is (current_cost - cost) / model_cost_change alone (the host StepEvaluator's second term then equals the
// first).  Same arithmetic as the host StepEvaluator in pxr_ba_host.h.
struct DevStepEvaluator {
  int max_nonmonotonic, num_consecutive_nonmonotonic_steps;
  double minimum_cost, current_cost, reference_cost, candidate_cost, acc_reference, acc_candidate;
  __device__ __forceinline__ void init(double cost, int max_nm) {
    max_nonmonotonic = max_nm; num_consecutive_nonmonotonic_steps = 0;
    minimum_cost = current_cost = reference_cost = candidate_cost = cost;
    acc_reference = acc_candidate = 0.0;
  }
  __device__ __forceinline__ double quality(double cost, double model_cost_change) const {
    if (cost >= 1.7976931348623157e308) return -1.7976931348623157e308;
    double rel = (current_cost - cost) / model_cost_change;
    if (max_nonmonotonic > 0) rel = fmax(rel, (reference_cost - cost) / (acc_reference + model_cost_change));
    return rel;
  }
  __device__ __forceinline__ void accepted(double cost, double model_cost_change) {
    current_cost = cost;
    if (max_nonmonotonic == 0) return;
    acc_candidate += model_cost_change; acc_reference += model_cost_change;
    if (cost < minimum_cost) {
      minimum_cost = cost; num_consecutive_nonmonotonic_steps = 0; candidate_cost = cost; acc_candidate = 0.0;
    } else {
      ++num_consecutive_nonmonotonic_steps;
      if (cost > candidate_cost) { candidate_cost = cost; acc_candidate = 0.0; }
    }
    if (num_consecutive_nonmonotonic_steps == max_nonmonotonic) { reference_cost = candidate_cost; acc_reference = acc_candidate; }
  }
};

}  // namespace pxr
