// pxr_device.cuh — device-side math shared by the featuremetric kernels (sm_90a).
//
//  * cubic Hermite splines with the SAME operation order as the reference's AVX2 header
//    (reference pixsfm/base/src/cubic_hermite_spline_simd.h:56-192): IEEE fmaf/fma are
//    deterministic, so the horizontal (fp32) and vertical (fp64) passes reproduce the
//    reference's per-channel values bit for bit; only reduction orders differ.
//  * WorldToPixel (reference pixsfm/base/src/projection.h:60-75) with hand-derived analytic
//    Jacobians replacing ceres::Jet autodiff (feature_reference.h:87-96).
//  * ceres loss functions rho(s) (reference bundle_adjustment_options.h:49).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace pxr {

// ------------------------------------------------------------------ splines
// f16/f32-in overload (:123-192), one channel. Intrinsics forbid re-association/contraction.
struct SplineCoefF32 {
  float x2s, fourx, xhalf, onefivex2;
  __device__ __forceinline__ explicit SplineCoefF32(double x) {
    x2s = (float)(x * x);
    fourx = (float)(4.0 * x);
    xhalf = (float)(x * 0.5);
    onefivex2 = __fmul_rn(1.5f, x2s);
  }
};
template <bool DERIV>
__device__ __forceinline__ void spline_f32(float p0, float p1, float p2, float p3,
                                           const SplineCoefF32& c, float& f, float& d) {
  const float t1 = __fmaf_rn(3.0f, p1, -p0);
  const float t2 = __fmaf_rn(3.0f, p2, -p3);
  const float t4 = __fmaf_rn(4.0f, p2, -p3);
  const float t5 = __fmaf_rn(2.5f, p1, -p0);
  const float t6 = __fmaf_rn(-1.0f, p0, p2);
  const float t3 = __fsub_rn(t1, t2);
  const float b = __fmaf_rn(0.5f, t4, -t5);
  const float t7 = __fmaf_rn(c.xhalf, t6, p1);
  const float t8 = __fmaf_rn(c.xhalf, t3, b);
  f = __fmaf_rn(c.x2s, t8, t7);
  if (DERIV) {
    const float t9 = __fmaf_rn(c.fourx, b, t6);
    const float t10 = __fmul_rn(c.onefivex2, t3);
    d = __fmaf_rn(0.5f, t9, t10);
  }
}

// f64-in overload (:56-121)
struct SplineCoefF64 {
  double x2s, fourx, xhalf, onefivex2;
  __device__ __forceinline__ explicit SplineCoefF64(double x) {
    x2s = __dmul_rn(x, x);
    fourx = __dmul_rn(4.0, x);
    xhalf = __dmul_rn(x, 0.5);
    onefivex2 = __dmul_rn(1.5, x2s);
  }
};
template <bool VALUE, bool DERIV>
__device__ __forceinline__ void spline_f64(double p0, double p1, double p2, double p3,
                                           const SplineCoefF64& c, double& f, double& d) {
  const double t1 = __fma_rn(3.0, p1, -p0);
  const double t2 = __fma_rn(3.0, p2, -p3);
  const double t4 = __fma_rn(4.0, p2, -p3);
  const double t5 = __fma_rn(2.5, p1, -p0);
  const double t6 = __fma_rn(-1.0, p0, p2);
  const double t3 = __dsub_rn(t1, t2);
  const double b = __fma_rn(0.5, t4, -t5);
  if (VALUE) {
    const double t7 = __fma_rn(c.xhalf, t6, p1);
    const double t8 = __fma_rn(c.xhalf, t3, b);
    f = __fma_rn(c.x2s, t8, t7);
  }
  if (DERIV) {
    const double t9 = __fma_rn(c.fourx, b, t6);
    const double t10 = __dmul_rn(c.onefivex2, t3);
    d = __fma_rn(0.5, t9, t10);
  }
}

// (ceres) CubicHermiteSpline in double — the reference's path when C < 8 (interpolation.h:224-262)
template <bool DERIV>
__device__ __forceinline__ void spline_ceres(double p0, double p1, double p2, double p3, double x,
                                             double& f, double& d) {
  const double a = __dmul_rn(0.5, __dadd_rn(__dsub_rn(__dadd_rn(-p0, __dmul_rn(3.0, p1)), __dmul_rn(3.0, p2)), p3));
  const double b = __dmul_rn(0.5, __dsub_rn(__dadd_rn(__dsub_rn(__dmul_rn(2.0, p0), __dmul_rn(5.0, p1)), __dmul_rn(4.0, p2)), p3));
  const double c = __dmul_rn(0.5, __dadd_rn(-p0, p2));
  f = __dadd_rn(p1, __dmul_rn(x, __dadd_rn(c, __dmul_rn(x, __dadd_rn(b, __dmul_rn(x, a))))));
  if (DERIV) d = __dadd_rn(c, __dmul_rn(x, __dadd_rn(__dmul_rn(2.0, b), __dmul_rn(__dmul_rn(3.0, a), x))));
}

// ------------------------------------------------------------------ loss
struct LossParams {
  int type;     // pxr_loss_type
  double a;
};
// rho[0..2] (ceres internal/ceres/loss_function.cc); weight = ScaledLoss factor
__device__ __forceinline__ void loss_eval(const LossParams& L, double weight, double s, double rho[3]) {
  const double kMin = 2.2250738585072014e-308;
  switch (L.type) {
    case 1: {
      const double b = L.a * L.a, c = 1.0 / b;
      const double sum = 1.0 + s * c, inv = 1.0 / sum;
      rho[0] = b * log(sum); rho[1] = fmax(kMin, inv); rho[2] = -c * (inv * inv);
    } break;
    case 2: {
      const double b = L.a * L.a;
      if (s > b) { const double r = sqrt(s); rho[0] = 2.0 * L.a * r - b; rho[1] = fmax(kMin, L.a / r); rho[2] = -rho[1] / (2.0 * s); }
      else { rho[0] = s; rho[1] = 1.0; rho[2] = 0.0; }
    } break;
    case 3: {
      const double b = L.a * L.a, c = 1.0 / b;
      const double sum = 1.0 + s * c, tmp = sqrt(sum);
      rho[0] = 2.0 * b * (tmp - 1.0); rho[1] = fmax(kMin, 1.0 / tmp); rho[2] = -(c * rho[1]) / (2.0 * sum);
    } break;
    case 4: {
      const double b = 1.0 / (L.a * L.a);
      const double sum = 1.0 + s * s * b, inv = 1.0 / sum;
      rho[0] = L.a * atan2(s, L.a); rho[1] = fmax(kMin, inv); rho[2] = -2.0 * s * b * (inv * inv);
    } break;
    default: rho[0] = s; rho[1] = 1.0; rho[2] = 0.0;
  }
  rho[0] *= weight; rho[1] *= weight; rho[2] *= weight;
}
// All supported losses have rho'' <= 0, for which the ceres Corrector (internal/ceres/corrector.cc)
// reduces to J <- sqrt(rho') J, r <- sqrt(rho') r, i.e. J^T J and J^T r scale by rho'.

// ------------------------------------------------------------------ cameras
__host__ __device__ __forceinline__ int cam_num_params(int model) {
  switch (model) {
    case 0: return 3; case 1: return 4; case 2: return 4; case 3: return 5;
    case 4: return 8; case 5: return 8; case 6: return 12; default: return 0;
  }
}

constexpr int kMaxK = 12;  // PXR_MAX_CAM_PARAMS

// the mean of a model's focal lengths (COLMAP's MeanFocalLength): pixel thresholds over it are normalised-plane ones
__device__ __forceinline__ double mean_focal(int model, const double* p) {
  return (model == 0 || model == 2 || model == 3) ? p[0] : 0.5 * (p[0] + p[1]);
}

// normalised unit quaternion (w, x, y, z) -> rotation matrix (row-major)
__device__ __forceinline__ void quat_to_rot(const double* qv, double* R) {
  const double s = 1.0 / sqrt(qv[0] * qv[0] + qv[1] * qv[1] + qv[2] * qv[2] + qv[3] * qv[3]);
  const double w = qv[0] * s, a = qv[1] * s, b = qv[2] * s, c = qv[3] * s;
  R[0] = 1.0 - 2.0 * (b * b + c * c); R[1] = 2.0 * (a * b - w * c); R[2] = 2.0 * (a * c + w * b);
  R[3] = 2.0 * (a * b + w * c); R[4] = 1.0 - 2.0 * (a * a + c * c); R[5] = 2.0 * (b * c - w * a);
  R[6] = 2.0 * (a * c - w * b); R[7] = 2.0 * (b * c + w * a); R[8] = 1.0 - 2.0 * (a * a + b * b);
}

// the counter-based stream of the RANSAC samplers (include/pxr.h states it); integer code, so every translation unit
// draws the same words whatever its floating-point flags
__host__ __device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
  uint64_t z = x + 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// (colmap 3.8 camera_models.h) WorldToImage + derivatives.
// Dm = d(x,y)/d(u,v) row-major 2x2; Jk[0][k] = dx/dp_k, Jk[1][k] = dy/dp_k.
template <bool JAC>
__device__ __forceinline__ void cam_world_to_image(int model, const double* __restrict__ p, double u, double v,
                                                   double& x, double& y, double Dm[4], double Jk[2][kMaxK]) {
  if (JAC) {
#pragma unroll
    for (int k = 0; k < kMaxK; ++k) { Jk[0][k] = 0.0; Jk[1][k] = 0.0; }
  }
  switch (model) {
    case 0: {  // SIMPLE_PINHOLE f cx cy
      x = p[0] * u + p[1]; y = p[0] * v + p[2];
      if (JAC) { Dm[0] = p[0]; Dm[1] = 0; Dm[2] = 0; Dm[3] = p[0];
        Jk[0][0] = u; Jk[1][0] = v; Jk[0][1] = 1.0; Jk[1][2] = 1.0; }
    } break;
    case 1: {  // PINHOLE fx fy cx cy
      x = p[0] * u + p[2]; y = p[1] * v + p[3];
      if (JAC) { Dm[0] = p[0]; Dm[1] = 0; Dm[2] = 0; Dm[3] = p[1];
        Jk[0][0] = u; Jk[1][1] = v; Jk[0][2] = 1.0; Jk[1][3] = 1.0; }
    } break;
    case 2: {  // SIMPLE_RADIAL f cx cy k
      const double r2 = u * u + v * v;
      const double radial = p[3] * r2;
      const double du = u * radial, dv = v * radial;
      x = p[0] * (u + du) + p[1]; y = p[0] * (v + dv) + p[2];
      if (JAC) {
        const double rp = p[3];
        Dm[0] = p[0] * (1.0 + radial + 2.0 * u * u * rp); Dm[1] = p[0] * (2.0 * u * v * rp);
        Dm[2] = Dm[1]; Dm[3] = p[0] * (1.0 + radial + 2.0 * v * v * rp);
        Jk[0][0] = u + du; Jk[1][0] = v + dv; Jk[0][1] = 1.0; Jk[1][2] = 1.0;
        Jk[0][3] = p[0] * u * r2; Jk[1][3] = p[0] * v * r2;
      }
    } break;
    case 3: {  // RADIAL f cx cy k1 k2
      const double r2 = u * u + v * v;
      const double radial = p[3] * r2 + p[4] * r2 * r2;
      const double du = u * radial, dv = v * radial;
      x = p[0] * (u + du) + p[1]; y = p[0] * (v + dv) + p[2];
      if (JAC) {
        const double rp = p[3] + 2.0 * p[4] * r2;
        Dm[0] = p[0] * (1.0 + radial + 2.0 * u * u * rp); Dm[1] = p[0] * (2.0 * u * v * rp);
        Dm[2] = Dm[1]; Dm[3] = p[0] * (1.0 + radial + 2.0 * v * v * rp);
        Jk[0][0] = u + du; Jk[1][0] = v + dv; Jk[0][1] = 1.0; Jk[1][2] = 1.0;
        Jk[0][3] = p[0] * u * r2; Jk[1][3] = p[0] * v * r2;
        Jk[0][4] = p[0] * u * r2 * r2; Jk[1][4] = p[0] * v * r2 * r2;
      }
    } break;
    case 4: {  // OPENCV fx fy cx cy k1 k2 p1 p2
      const double u2 = u * u, uv = u * v, v2 = v * v;
      const double r2 = u2 + v2;
      const double radial = p[4] * r2 + p[5] * r2 * r2;
      const double du = u * radial + 2.0 * p[6] * uv + p[7] * (r2 + 2.0 * u2);
      const double dv = v * radial + 2.0 * p[7] * uv + p[6] * (r2 + 2.0 * v2);
      x = p[0] * (u + du) + p[2]; y = p[1] * (v + dv) + p[3];
      if (JAC) {
        const double rp = p[4] + 2.0 * p[5] * r2;
        const double duu = radial + 2.0 * u2 * rp + 2.0 * p[6] * v + 6.0 * p[7] * u;
        const double duv = 2.0 * uv * rp + 2.0 * p[6] * u + 2.0 * p[7] * v;
        const double dvu = 2.0 * uv * rp + 2.0 * p[7] * v + 2.0 * p[6] * u;
        const double dvv = radial + 2.0 * v2 * rp + 2.0 * p[7] * u + 6.0 * p[6] * v;
        Dm[0] = p[0] * (1.0 + duu); Dm[1] = p[0] * duv; Dm[2] = p[1] * dvu; Dm[3] = p[1] * (1.0 + dvv);
        Jk[0][0] = u + du; Jk[1][1] = v + dv; Jk[0][2] = 1.0; Jk[1][3] = 1.0;
        Jk[0][4] = p[0] * u * r2; Jk[1][4] = p[1] * v * r2;
        Jk[0][5] = p[0] * u * r2 * r2; Jk[1][5] = p[1] * v * r2 * r2;
        Jk[0][6] = p[0] * 2.0 * uv; Jk[1][6] = p[1] * (r2 + 2.0 * v2);
        Jk[0][7] = p[0] * (r2 + 2.0 * u2); Jk[1][7] = p[1] * 2.0 * uv;
      }
    } break;
    case 5: {  // OPENCV_FISHEYE fx fy cx cy k1 k2 k3 k4
      const double r = sqrt(u * u + v * v);
      double du = 0.0, dv = 0.0;
      if (r > 2.220446049250313e-16) {
        const double th = atan(r);
        const double t2 = th * th, t4 = t2 * t2, t6 = t4 * t2, t8 = t4 * t4;
        const double thd = th * (1.0 + p[4] * t2 + p[5] * t4 + p[6] * t6 + p[7] * t8);
        const double s = thd / r;
        du = u * s - u; dv = v * s - v;
        if (JAC) {
          const double thp = 1.0 / (1.0 + r * r);
          const double thdp = 1.0 + 3.0 * p[4] * t2 + 5.0 * p[5] * t4 + 7.0 * p[6] * t6 + 9.0 * p[7] * t8;
          const double dsdr = (thdp * thp * r - thd) / (r * r);
          const double su = dsdr * u / r, sv = dsdr * v / r;
          Dm[0] = p[0] * (s + u * su); Dm[1] = p[0] * (u * sv);
          Dm[2] = p[1] * (v * su); Dm[3] = p[1] * (s + v * sv);
          const double t3 = th * t2, t5 = th * t4, t7 = th * t6, t9 = th * t8;
          Jk[0][4] = p[0] * u * t3 / r; Jk[1][4] = p[1] * v * t3 / r;
          Jk[0][5] = p[0] * u * t5 / r; Jk[1][5] = p[1] * v * t5 / r;
          Jk[0][6] = p[0] * u * t7 / r; Jk[1][6] = p[1] * v * t7 / r;
          Jk[0][7] = p[0] * u * t9 / r; Jk[1][7] = p[1] * v * t9 / r;
        }
      } else if (JAC) { Dm[0] = p[0]; Dm[1] = 0; Dm[2] = 0; Dm[3] = p[1]; }
      x = p[0] * (u + du) + p[2]; y = p[1] * (v + dv) + p[3];
      if (JAC) { Jk[0][0] = u + du; Jk[1][1] = v + dv; Jk[0][2] = 1.0; Jk[1][3] = 1.0; }
    } break;
    case 6: {  // FULL_OPENCV fx fy cx cy k1 k2 p1 p2 k3 k4 k5 k6
      const double u2 = u * u, uv = u * v, v2 = v * v;
      const double r2 = u2 + v2, r4 = r2 * r2, r6 = r4 * r2;
      const double N = 1.0 + p[4] * r2 + p[5] * r4 + p[8] * r6;
      const double D = 1.0 + p[9] * r2 + p[10] * r4 + p[11] * r6;
      const double radial = N / D;
      const double du = u * radial + 2.0 * p[6] * uv + p[7] * (r2 + 2.0 * u2) - u;
      const double dv = v * radial + 2.0 * p[7] * uv + p[6] * (r2 + 2.0 * v2) - v;
      x = p[0] * (u + du) + p[2]; y = p[1] * (v + dv) + p[3];
      if (JAC) {
        const double Np = p[4] + 2.0 * p[5] * r2 + 3.0 * p[8] * r4;
        const double Dp = p[9] + 2.0 * p[10] * r2 + 3.0 * p[11] * r4;
        const double rp = (Np * D - N * Dp) / (D * D);
        const double xu = radial + 2.0 * u2 * rp + 2.0 * p[6] * v + 6.0 * p[7] * u;  // d(u+du)/du
        const double xv = 2.0 * uv * rp + 2.0 * p[6] * u + 2.0 * p[7] * v;
        const double yu = 2.0 * uv * rp + 2.0 * p[7] * v + 2.0 * p[6] * u;
        const double yv = radial + 2.0 * v2 * rp + 2.0 * p[7] * u + 6.0 * p[6] * v;
        Dm[0] = p[0] * xu; Dm[1] = p[0] * xv; Dm[2] = p[1] * yu; Dm[3] = p[1] * yv;
        Jk[0][0] = u + du; Jk[1][1] = v + dv; Jk[0][2] = 1.0; Jk[1][3] = 1.0;
        Jk[0][4] = p[0] * u * r2 / D; Jk[1][4] = p[1] * v * r2 / D;
        Jk[0][5] = p[0] * u * r4 / D; Jk[1][5] = p[1] * v * r4 / D;
        Jk[0][6] = p[0] * 2.0 * uv; Jk[1][6] = p[1] * (r2 + 2.0 * v2);
        Jk[0][7] = p[0] * (r2 + 2.0 * u2); Jk[1][7] = p[1] * 2.0 * uv;
        Jk[0][8] = p[0] * u * r6 / D; Jk[1][8] = p[1] * v * r6 / D;
        const double nd2 = -N / (D * D);
        Jk[0][9] = p[0] * u * nd2 * r2; Jk[1][9] = p[1] * v * nd2 * r2;
        Jk[0][10] = p[0] * u * nd2 * r4; Jk[1][10] = p[1] * v * nd2 * r4;
        Jk[0][11] = p[0] * u * nd2 * r6; Jk[1][11] = p[1] * v * nd2 * r6;
      }
    } break;
    default: x = u; y = v; if (JAC) { Dm[0] = 1; Dm[1] = 0; Dm[2] = 0; Dm[3] = 1; }
  }
}

// (colmap 3.8 camera_models.h) ImageToWorld: pixel (x, y) -> normalised image point (u, v), the inverse of
// cam_world_to_image.  The principal point and focal lengths are removed, then the distortion is undone by Newton steps
// on the forward map (at most 100, until the squared step norm falls below 1e-28): COLMAP's IterativeUndistortion with
// the analytic Jacobian Dm in place of central differences, so the inverse round-trips to the last bits.
// OPENCV_FISHEYE solves its theta mapping theta_d = theta (1 + k1 theta^2 + ... + k4 theta^8) for theta instead.
__device__ __forceinline__ void cam_image_to_world(int model, const double* __restrict__ p, double x, double y, double& u,
                                                   double& v) {
  const bool one_f = model == 0 || model == 2 || model == 3;
  const double fx = p[0], fy = one_f ? p[0] : p[1];
  const double cx = one_f ? p[1] : p[2], cy = one_f ? p[2] : p[3];
  const double ud = (x - cx) / fx, vd = (y - cy) / fy;
  u = ud; v = vd;
  if (model == 0 || model == 1) return;
  if (model == 5) {
    const double thd = sqrt(ud * ud + vd * vd);
    if (!(thd > 2.220446049250313e-16)) return;
    double th = thd;
    for (int it = 0; it < 100; ++it) {
      const double t2 = th * th, t4 = t2 * t2, t6 = t4 * t2, t8 = t4 * t4;
      const double f = th * (1.0 + p[4] * t2 + p[5] * t4 + p[6] * t6 + p[7] * t8) - thd;
      const double fp = 1.0 + 3.0 * p[4] * t2 + 5.0 * p[5] * t4 + 7.0 * p[6] * t6 + 9.0 * p[7] * t8;
      const double step = f / fp;
      th -= step;
      if (step * step < 1e-28) break;
    }
    const double s = tan(th) / thd;
    u = ud * s; v = vd * s;
    return;
  }
  double Jk[2][kMaxK], Dm[4];
  for (int it = 0; it < 100; ++it) {
    double px, py;
    cam_world_to_image<true>(model, p, u, v, px, py, Dm, Jk);
    const double rx = px - x, ry = py - y;
    const double det = Dm[0] * Dm[3] - Dm[1] * Dm[2];
    const double su = (Dm[3] * rx - Dm[1] * ry) / det, sv = (Dm[0] * ry - Dm[2] * rx) / det;
    u -= su; v -= sv;
    if (!(su * su + sv * sv >= 1e-28)) break;      // converged, or a NaN step
  }
}

// WorldToPixel (projection.h:60-75) = ceres::QuaternionRotatePoint (normalising) + t, perspective
// divide, camera model.  With JAC, returns d(xy)/d(local pose: 3 rot (QuaternionManifold
// tangent, left-multiplicative) + 3 t), d(xy)/dX, d(xy)/d(cam params).
template <bool JAC>
__device__ __forceinline__ void world_to_pixel(int model, const double* __restrict__ cam,
                                               const double* __restrict__ q, const double* __restrict__ t,
                                               const double* __restrict__ X, double xy[2],
                                               double Jpose[2][6], double Jpt[2][3], double Jk[2][kMaxK]) {
  const double scale = 1.0 / sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  const double w = scale * q[0], a = scale * q[1], b = scale * q[2], c = scale * q[3];
  // UnitQuaternionRotatePoint (ceres rotation.h @2.1)
  double uv0 = b * X[2] - c * X[1];
  double uv1 = c * X[0] - a * X[2];
  double uv2 = a * X[1] - b * X[0];
  uv0 += uv0; uv1 += uv1; uv2 += uv2;
  double y0 = X[0] + w * uv0, y1 = X[1] + w * uv1, y2 = X[2] + w * uv2;
  y0 += b * uv2 - c * uv1;
  y1 += c * uv0 - a * uv2;
  y2 += a * uv1 - b * uv0;
  const double px = y0 + t[0], py = y1 + t[1], pz = y2 + t[2];
  const double un = px / pz, vn = py / pz;
  double Dm[4];
  cam_world_to_image<JAC>(model, cam, un, vn, xy[0], xy[1], Dm, Jk);
  if (JAC) {
    const double iz = 1.0 / pz;
    // M = Dm * d(un,vn)/d(pc)   (2x3)
    double M[2][3];
    M[0][0] = Dm[0] * iz; M[0][1] = Dm[1] * iz; M[0][2] = -(Dm[0] * un + Dm[1] * vn) * iz;
    M[1][0] = Dm[2] * iz; M[1][1] = Dm[3] * iz; M[1][2] = -(Dm[2] * un + Dm[3] * vn) * iz;
    // rotation matrix of the unit quaternion
    const double R00 = 1.0 - 2.0 * (b * b + c * c), R01 = 2.0 * (a * b - w * c), R02 = 2.0 * (a * c + w * b);
    const double R10 = 2.0 * (a * b + w * c), R11 = 1.0 - 2.0 * (a * a + c * c), R12 = 2.0 * (b * c - w * a);
    const double R20 = 2.0 * (a * c - w * b), R21 = 2.0 * (b * c + w * a), R22 = 1.0 - 2.0 * (a * a + b * b);
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      Jpt[r][0] = M[r][0] * R00 + M[r][1] * R10 + M[r][2] * R20;
      Jpt[r][1] = M[r][0] * R01 + M[r][1] * R11 + M[r][2] * R21;
      Jpt[r][2] = M[r][0] * R02 + M[r][1] * R12 + M[r][2] * R22;
      // d(pc)/d(delta) = -2 [y]_x  (y = R X):  [y]_x = [[0,-y2,y1],[y2,0,-y0],[-y1,y0,0]]
      Jpose[r][0] = -2.0 * (M[r][1] * y2 - M[r][2] * y1);
      Jpose[r][1] = -2.0 * (-M[r][0] * y2 + M[r][2] * y0);
      Jpose[r][2] = -2.0 * (M[r][0] * y1 - M[r][1] * y0);
      Jpose[r][3] = M[r][0]; Jpose[r][4] = M[r][1]; Jpose[r][5] = M[r][2];
    }
  }
}

// (ceres) QuaternionManifold::Plus: q_delta (x) q
__device__ __forceinline__ void quaternion_plus(const double* x, const double* d, double* out) {
  const double sq = d[0] * d[0] + d[1] * d[1] + d[2] * d[2];
  if (sq == 0.0) { out[0] = x[0]; out[1] = x[1]; out[2] = x[2]; out[3] = x[3]; return; }
  const double nd = sqrt(sq);
  const double s = sin(nd) / nd;
  const double z0 = cos(nd), z1 = s * d[0], z2 = s * d[1], z3 = s * d[2];
  out[0] = z0 * x[0] - z1 * x[1] - z2 * x[2] - z3 * x[3];
  out[1] = z0 * x[1] + z1 * x[0] + z2 * x[3] - z3 * x[2];
  out[2] = z0 * x[2] - z1 * x[3] + z2 * x[0] + z3 * x[1];
  out[3] = z0 * x[3] + z1 * x[2] - z2 * x[1] + z3 * x[0];
}

// ------------------------------------------------------------------ mbarrier / bulk-copy (TMA) PTX
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// cp.async.bulk global -> shared (TMA bulk copy engine; SASS: UBLKCP). 16-byte aligned, size % 16 == 0.
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// ------------------------------------------------------------------ warp reductions (fp64)
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}


// Transposed reduction of 8 per-lane doubles over the warp: 9 double shuffles instead of 40.
// On return lane L holds the total of value index ((L>>4)&1)*4 + ((L>>3)&1)*2 + ((L>>2)&1).
__device__ __forceinline__ double warp_reduce8_transposed(const double v[8], int lane) {
  const bool b4 = lane & 16, b3 = lane & 8, b2 = lane & 4;
  double a[4], b[2];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const double keep = b4 ? v[4 + j] : v[j];
    const double send = b4 ? v[j] : v[4 + j];
    a[j] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
  }
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const double keep = b3 ? a[2 + j] : a[j];
    const double send = b3 ? a[j] : a[2 + j];
    b[j] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
  }
  const double keep = b2 ? b[1] : b[0];
  const double send = b2 ? b[0] : b[1];
  double c = keep + __shfl_xor_sync(0xffffffffu, send, 4);
  c += __shfl_xor_sync(0xffffffffu, c, 2);
  c += __shfl_xor_sync(0xffffffffu, c, 1);
  return c;
}

}  // namespace pxr
