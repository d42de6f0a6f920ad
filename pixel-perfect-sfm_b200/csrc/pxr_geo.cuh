// K1g: geometric (reprojection-error) evaluation — the residual of classic bundle adjustment.
//
// Reference: GeometricBundleOptimizer::AddResiduals (bundle_adjustment/src/geometric_bundle_optimizer.h:36-83) adds
// colmap::BundleAdjustmentCostFunction / ...ConstantPoseCostFunction (residuals/src/geometric.h:16-41):
//   r = WorldToImage(camera, R(q) X + t) - point2D.XY()          (2 residuals, image pixels)
// On a geometric handle K0 runs with the identity patch frame (scale 1, corner 0, upsampling 1), so its Jacobian
// record is d(xy)/d(theta) exactly, and it writes the projection itself to `xy` (its `uv` is xy - 0.5 and is not
// read).  The residual is formed here from that `xy` with one subtraction: no rounding beyond the projection's own.
// With G = d r / d(xy) = I the record K1 writes for a featuremetric observation becomes
//   out[o*8 + 0..5] = (||r||^2, r_x, r_y, 1, 0, 1)
// so everything downstream of K1 (builds, Schur walks, solves, inner iterations, cost reduction) is shared.
// One thread per item; item_index / end_dev as in fm_eval_small_kernel (the batched inner-iteration rounds drive it
// through a device-counted list).
#pragma once
#include "pxr_device.cuh"

namespace pxr {

struct GeoEvalArgs {
  const double* xy;            // [n_obs][2] projection (K0's xy output)
  const double* target;        // [n_obs][2] observed keypoint, image pixels
  int64_t begin, end;          // item range
  const int64_t* item_index;   // optional indirection: item k is observation item_index[k]
  const unsigned long long* end_dev = nullptr;   // optional: item count on the device (end = begin + *end_dev)
  double* out;                 // [n_obs][8]: s, r_x, r_y, 1, 0, 1 (MODE 1) / only s (MODE 0)
  double* residuals = nullptr; // optional [n_obs][2]
  double* grad = nullptr;      // optional [n_obs][2][2]: d r / d x, d r / d y (the identity; MODE 1)
};

// grid-stride, so a list whose length lives on the device gets a grid bounded by the SM count (as K0 does)
template <int MODE>
static __global__ void __launch_bounds__(128) geo_eval_kernel(GeoEvalArgs a) {
  const int64_t end = a.end_dev ? a.begin + (int64_t)*a.end_dev : a.end;
  for (int64_t k = a.begin + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < end; k += (int64_t)gridDim.x * blockDim.x) {
    const int64_t o = a.item_index ? a.item_index[k] : k;
    const double rx = a.xy[2 * o] - a.target[2 * o];
    const double ry = a.xy[2 * o + 1] - a.target[2 * o + 1];
    if (a.residuals) { a.residuals[2 * o] = rx; a.residuals[2 * o + 1] = ry; }
    if (MODE == 1 && a.grad) {
      double* g = a.grad + o * 4;
      g[0] = 1.0; g[1] = 0.0; g[2] = 0.0; g[3] = 1.0;
    }
    double* op = a.out + o * 8;
    op[0] = __dadd_rn(__dmul_rn(rx, rx), __dmul_rn(ry, ry));     // no contraction: the CPU restatement's sum, bit for bit
    if (MODE == 1) { op[1] = rx; op[2] = ry; op[3] = 1.0; op[4] = 0.0; op[5] = 1.0; }
  }
}

}  // namespace pxr
