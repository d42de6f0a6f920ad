// pxr_pnp.cu — batched absolute pose estimation: pycolmap 0.4's absolute_pose_estimation for many queries at once.
//
//   RANSAC kernel  one CTA per query.  The query's 2D points go once to the normalised plane (cam_image_to_world) and,
//                  with the 3D points, into shared memory when they fit (kPCorrSmem bytes), else into a global
//                  workspace.  Per round the first PXR_PNP_ROUND_TRIALS threads draw one sample each and solve P3P
//                  (Lambda Twist); the warps then score every hypothesis against every correspondence (one warp per
//                  hypothesis, lanes over the correspondences, butterfly sums), warp 0 picks the round's best and, when
//                  it improves the query's best, the CTA runs local optimisation.  The specification of the sample
//                  stream, the support measure and the stopping rule is include/pxr.h's; tests/pnp_reference.py
//                  restates it.
//   refinement     one CTA per query through qba_lm_solve (pxr_qba_lm.cuh), the LM loop of query bundle adjustment,
//                  with a reprojection evaluation: Cauchy-robust pixel residuals over the RANSAC inliers, the pose on
//                  the quaternion manifold, focal length / extra parameters free only when asked (COLMAP 3.8
//                  RefineAbsolutePose).  The inliers of the refined pose are then recounted.
// This file is compiled without fused multiply-add (build.py), so P3P and the residuals evaluate exactly as written and
// a host restatement in IEEE double reproduces them bit for bit.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <vector>

#include "pxr_qba_lm.cuh"
#include "pxr_waves.h"

namespace pxr {

constexpr int kPThreads = kQThreads;                 // both kernels: 8 warps
constexpr int kPWarps = kPThreads / 32;
constexpr int kPTrials = PXR_PNP_ROUND_TRIALS;
constexpr int kPHyp = 4 * kPTrials;                  // hypotheses of one round: 4 P3P solutions per trial
constexpr int kPPose = 12;                           // R (row-major) | t
constexpr int kLOSteps = 3;
constexpr int kCorrBytes = 40;                       // u, v, X, Y, Z
constexpr size_t kPCorrSmem = 96 * 1024;             // a query's correspondences stay on chip up to 2457 of them
constexpr double kDblEps = 2.220446049250313e-16;

// the three indices trial t draws (include/pxr.h); false when 64 draws give fewer than three distinct ones
__device__ __forceinline__ bool draw_sample(uint64_t s0, int64_t t, int64_t n, int idx[3]) {
  int k = 0;
  for (int d = 0; d < 64 && k < 3; ++d) {
    const uint64_t w = splitmix64(s0 ^ ((uint64_t)t << 8) ^ (uint64_t)d);
    const int i = (int)(((w >> 32) * (uint64_t)n) >> 32);
    if ((k > 0 && idx[0] == i) || (k > 1 && idx[1] == i)) continue;
    idx[k++] = i;
  }
  return k == 3;
}

// ---- Lambda Twist P3P (Persson & Nordberg, "Lambda Twist: An Accurate Fast Robust Perspective Three Point (P3P)
// Solver", ECCV 2018)
__device__ __forceinline__ void root2real(double b, double c, double& r1, double& r2) {
  const double v = b * b - 4.0 * c;
  if (v < 0.0) { r1 = r2 = 0.5 * b; return; }
  const double y = sqrt(v);
  r1 = b < 0.0 ? 0.5 * (-b + y) : 0.5 * (-b - y);
  r2 = r1 != 0.0 ? c / r1 : INFINITY;
}

// a real root of x^3 + b x^2 + c x + d: a start on the correct side of the stationary points, then Newton
static __device__ double cubick(double b, double c, double d) {
  double r0;
  if (b * b >= 3.0 * c) {
    const double v = sqrt(b * b - 3.0 * c);
    const double t1 = (-b - v) / 3.0;
    double k = ((t1 + b) * t1 + c) * t1 + d;
    if (k > 0.0) {
      r0 = t1 - sqrt(-k / (3.0 * t1 + b));
    } else {
      const double t2 = (-b + v) / 3.0;
      k = ((t2 + b) * t2 + c) * t2 + d;
      r0 = t2 + sqrt(-k / (3.0 * t2 + b));
    }
  } else {
    r0 = -b / 3.0;
    if (fabs((3.0 * r0 + 2.0 * b) * r0 + c) < 1e-4) r0 += 1.0;
  }
  for (int i = 0; i < 50; ++i) {
    const double fx = ((r0 + b) * r0 + c) * r0 + d;
    if (i >= 7 && fabs(fx) <= kDblEps) break;
    const double fpx = (3.0 * r0 + 2.0 * b) * r0 + c;
    r0 = r0 - fx / fpx;
  }
  return r0;
}

// eigenvectors V (row-major, columns) and eigenvalues of the symmetric x (row-major) whose third eigenvalue is 0
static __device__ void eig_known0(const double x[9], double V[9], double L[3]) {
  double v3[3] = {x[3] * x[7] - x[6] * x[4], x[6] * x[1] - x[7] * x[0], x[4] * x[0] - x[3] * x[1]};
  const double n3 = sqrt(v3[0] * v3[0] + v3[1] * v3[1] + v3[2] * v3[2]);
  v3[0] = v3[0] / n3; v3[1] = v3[1] / n3; v3[2] = v3[2] / n3;
  const double x01_squared = x[1] * x[1];
  const double b = -x[0] - x[4] - x[8];
  const double c = -x01_squared - x[2] * x[2] - x[5] * x[5] + x[0] * (x[4] + x[8]) + x[4] * x[8];
  double e1, e2;
  root2real(b, c, e1, e2);
  if (fabs(e1) < fabs(e2)) { const double s = e1; e1 = e2; e2 = s; }
  const double mx0011 = -x[0] * x[4];
  const double prec_0 = x[1] * x[5] - x[2] * x[4];
  const double prec_1 = x[1] * x[2] - x[0] * x[5];
  double vs[2][3];
  for (int k = 0; k < 2; ++k) {
    const double e = k == 0 ? e1 : e2;
    const double tmp = 1.0 / (e * (x[0] + x[4]) + mx0011 - e * e + x01_squared);
    const double a1 = -(e * x[2] + prec_0) * tmp;
    const double a2 = -(e * x[5] + prec_1) * tmp;
    const double rnorm = 1.0 / sqrt(a1 * a1 + a2 * a2 + 1.0);
    vs[k][0] = a1 * rnorm; vs[k][1] = a2 * rnorm; vs[k][2] = rnorm;
  }
  for (int r = 0; r < 3; ++r) { V[3 * r] = vs[0][r]; V[3 * r + 1] = vs[1][r]; V[3 * r + 2] = v3[r]; }
  L[0] = e1; L[1] = e2; L[2] = 0.0;
}

// Gauss-Newton on the three depth equations, kept while the residual falls
static __device__ void refine_lambda(double& l1, double& l2, double& l3, double a12, double a13, double a23, double b12,
                              double b13, double b23) {
  for (int it = 0; it < 5; ++it) {
    const double r1 = l1 * l1 + l2 * l2 + b12 * l1 * l2 - a12;
    const double r2 = l1 * l1 + l3 * l3 + b13 * l1 * l3 - a13;
    const double r3 = l2 * l2 + l3 * l3 + b23 * l2 * l3 - a23;
    const double e0 = fabs(r1) + fabs(r2) + fabs(r3);
    if (!(e0 > 0.0)) break;
    const double a = 2.0 * l1 + b12 * l2, b = 2.0 * l2 + b12 * l1;
    const double c = 2.0 * l1 + b13 * l3, e = 2.0 * l3 + b13 * l1;
    const double f = 2.0 * l2 + b23 * l3, g = 2.0 * l3 + b23 * l2;
    const double idet = 1.0 / (-a * e * f - b * c * g);
    const double d1 = (-e * f * r1 - b * g * r2 + b * e * r3) * idet;
    const double d2 = (-c * g * r1 + a * g * r2 - a * e * r3) * idet;
    const double d3 = (c * f * r1 - a * f * r2 - b * c * r3) * idet;
    const double m1 = l1 - d1, m2 = l2 - d2, m3 = l3 - d3;
    const double s1 = m1 * m1 + m2 * m2 + b12 * m1 * m2 - a12;
    const double s2 = m1 * m1 + m3 * m3 + b13 * m1 * m3 - a13;
    const double s3 = m2 * m2 + m3 * m3 + b23 * m2 * m3 - a23;
    if (!(fabs(s1) + fabs(s2) + fabs(s3) < e0)) break;
    l1 = m1; l2 = m2; l3 = m3;
  }
}

// x [3][2] normalised image points, X [3][3] world points -> up to 4 poses P [k][12] = R (row-major) | t, world->camera
static __device__ int p3p_lambda_twist(const double x[3][2], const double X[3][3], double* P) {
  double y[3][3];
  for (int k = 0; k < 3; ++k) {
    const double nrm = sqrt(x[k][0] * x[k][0] + x[k][1] * x[k][1] + 1.0);
    y[k][0] = x[k][0] / nrm; y[k][1] = x[k][1] / nrm; y[k][2] = 1.0 / nrm;
  }
  auto dot = [](const double* p, const double* q) { return p[0] * q[0] + p[1] * q[1] + p[2] * q[2]; };
  const double b12 = -2.0 * dot(y[0], y[1]), b13 = -2.0 * dot(y[0], y[2]), b23 = -2.0 * dot(y[1], y[2]);
  double d12[3], d13[3], d23[3], d12xd13[3];
  for (int k = 0; k < 3; ++k) { d12[k] = X[0][k] - X[1][k]; d13[k] = X[0][k] - X[2][k]; d23[k] = X[1][k] - X[2][k]; }
  d12xd13[0] = d12[1] * d13[2] - d12[2] * d13[1];
  d12xd13[1] = d12[2] * d13[0] - d12[0] * d13[2];
  d12xd13[2] = d12[0] * d13[1] - d12[1] * d13[0];
  const double a12 = dot(d12, d12), a13 = dot(d13, d13), a23 = dot(d23, d23);
  const double c31 = -0.5 * b13, c23 = -0.5 * b23, c12 = -0.5 * b12;
  const double blob = c12 * c23 * c31 - 1.0;
  const double s31_squared = 1.0 - c31 * c31, s23_squared = 1.0 - c23 * c23, s12_squared = 1.0 - c12 * c12;
  const double p3 = a13 * (a23 * s31_squared - a13 * s23_squared);
  const double p2 = 2.0 * blob * a23 * a13 + a13 * (2.0 * a12 + a13) * s23_squared + a23 * (a23 - a12) * s31_squared;
  const double p1 = a23 * (a13 - a23) * s12_squared - a12 * a12 * s23_squared - 2.0 * a12 * (blob * a23 + a13 * s23_squared);
  const double p0 = a12 * (a12 * s23_squared - a23 * s12_squared);
  if (!(p3 != 0.0)) return 0;
  const double ip3 = 1.0 / p3;
  const double g = cubick(p2 * ip3, p1 * ip3, p0 * ip3);
  double A[9];
  A[0] = a23 * (1.0 - g); A[1] = (a23 * b12) * 0.5; A[2] = (a23 * b13 * g) * (-0.5);
  A[4] = a23 - a12 + a13 * g; A[5] = b23 * (a13 * g - a12) * 0.5; A[8] = g * (a13 - a23) - a12;
  A[3] = A[1]; A[6] = A[2]; A[7] = A[5];
  double V[9], L[3];
  eig_known0(A, V, L);
  const double v = sqrt(fmax(0.0, -L[1] / L[0]));
  double Ls[4][3];
  int nl = 0;
  for (int sgn = 0; sgn < 2; ++sgn) {
    const double s = sgn == 0 ? v : -v;
    const double w2 = 1.0 / (s * V[1] - V[0]);
    const double w0 = (V[3] - s * V[4]) * w2;
    const double w1 = (V[6] - s * V[7]) * w2;
    const double a = 1.0 / ((a13 - a12) * w1 * w1 - a12 * b13 * w1 - a12);
    const double b = (a13 * b12 * w1 - a12 * b13 * w0 - 2.0 * w0 * w1 * (a12 - a13)) * a;
    const double c = ((a13 - a12) * w0 * w0 + a13 * b12 * w0 + a13) * a;
    if (b * b - 4.0 * c >= 0.0) {
      double tau[2];
      root2real(b, c, tau[0], tau[1]);
      for (int k = 0; k < 2; ++k) {
        if (!(tau[k] > 0.0)) continue;
        const double d = a23 / (tau[k] * (b23 + tau[k]) + 1.0);
        if (!(d > 0.0)) continue;
        const double l2 = sqrt(d);
        const double l3 = tau[k] * l2;
        const double l1 = w0 * l2 + w1 * l3;
        if (l1 >= 0.0) { Ls[nl][0] = l1; Ls[nl][1] = l2; Ls[nl][2] = l3; ++nl; }
      }
    }
  }
  // inverse of the matrix with columns d12, d13, d12 x d13 (adjugate / determinant)
  const double M[3][3] = {{d12[0], d13[0], d12xd13[0]}, {d12[1], d13[1], d12xd13[1]}, {d12[2], d13[2], d12xd13[2]}};
  const double det = M[0][0] * (M[1][1] * M[2][2] - M[1][2] * M[2][1]) - M[0][1] * (M[1][0] * M[2][2] - M[1][2] * M[2][0]) +
                     M[0][2] * (M[1][0] * M[2][1] - M[1][1] * M[2][0]);
  if (!(det != 0.0) || !isfinite(det)) return 0;
  const double idet = 1.0 / det;
  const double Xi[3][3] = {
      {(M[1][1] * M[2][2] - M[1][2] * M[2][1]) * idet, (M[0][2] * M[2][1] - M[0][1] * M[2][2]) * idet,
       (M[0][1] * M[1][2] - M[0][2] * M[1][1]) * idet},
      {(M[1][2] * M[2][0] - M[1][0] * M[2][2]) * idet, (M[0][0] * M[2][2] - M[0][2] * M[2][0]) * idet,
       (M[0][2] * M[1][0] - M[0][0] * M[1][2]) * idet},
      {(M[1][0] * M[2][1] - M[1][1] * M[2][0]) * idet, (M[0][1] * M[2][0] - M[0][0] * M[2][1]) * idet,
       (M[0][0] * M[1][1] - M[0][1] * M[1][0]) * idet}};
  int ns = 0;
  for (int k = 0; k < nl; ++k) {
    double l1 = Ls[k][0], l2 = Ls[k][1], l3 = Ls[k][2];
    refine_lambda(l1, l2, l3, a12, a13, a23, b12, b13, b23);
    double ry1[3], e1[3], e2[3], e3[3];
    for (int j = 0; j < 3; ++j) {
      ry1[j] = y[0][j] * l1;
      e1[j] = ry1[j] - y[1][j] * l2;
      e2[j] = ry1[j] - y[2][j] * l3;
    }
    e3[0] = e1[1] * e2[2] - e1[2] * e2[1];
    e3[1] = e1[2] * e2[0] - e1[0] * e2[2];
    e3[2] = e1[0] * e2[1] - e1[1] * e2[0];
    const double Y[3][3] = {{e1[0], e2[0], e3[0]}, {e1[1], e2[1], e3[1]}, {e1[2], e2[2], e3[2]}};
    double* out = P + ns * kPPose;
    bool finite = true;
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        out[3 * i + j] = Y[i][0] * Xi[0][j] + Y[i][1] * Xi[1][j] + Y[i][2] * Xi[2][j];
        finite = finite && isfinite(out[3 * i + j]);
      }
    for (int i = 0; i < 3; ++i) {
      out[9 + i] = ry1[i] - (out[3 * i] * X[0][0] + out[3 * i + 1] * X[0][1] + out[3 * i + 2] * X[0][2]);
      finite = finite && isfinite(out[9 + i]);
    }
    if (finite) ++ns;
  }
  return ns;
}

// rotation matrix -> unit quaternion (w, x, y, z), w >= 0
static __device__ void rot_to_quat(const double* R, double* q) {
  const double tr = R[0] + R[4] + R[8];
  if (tr > 0.0) {
    const double s = sqrt(tr + 1.0) * 2.0;
    q[0] = 0.25 * s; q[1] = (R[7] - R[5]) / s; q[2] = (R[2] - R[6]) / s; q[3] = (R[3] - R[1]) / s;
  } else if (R[0] > R[4] && R[0] > R[8]) {
    const double s = sqrt(1.0 + R[0] - R[4] - R[8]) * 2.0;
    q[0] = (R[7] - R[5]) / s; q[1] = 0.25 * s; q[2] = (R[1] + R[3]) / s; q[3] = (R[2] + R[6]) / s;
  } else if (R[4] > R[8]) {
    const double s = sqrt(1.0 + R[4] - R[0] - R[8]) * 2.0;
    q[0] = (R[2] - R[6]) / s; q[1] = (R[1] + R[3]) / s; q[2] = 0.25 * s; q[3] = (R[5] + R[7]) / s;
  } else {
    const double s = sqrt(1.0 + R[8] - R[0] - R[4]) * 2.0;
    q[0] = (R[3] - R[1]) / s; q[1] = (R[2] + R[6]) / s; q[2] = (R[5] + R[7]) / s; q[3] = 0.25 * s;
  }
  const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  const double sg = q[0] < 0.0 ? -1.0 : 1.0;
  for (int k = 0; k < 4; ++k) q[k] = sg * (q[k] / n);
}

// the squared normalised-plane error of one correspondence; false when the point is not in front of the camera
__device__ __forceinline__ bool pnp_residual(const double* P, double u, double v, double X, double Y, double Z, double& r) {
  const double x = P[0] * X + P[1] * Y + P[2] * Z + P[9];
  const double y = P[3] * X + P[4] * Y + P[5] * Z + P[10];
  const double z = P[6] * X + P[7] * Y + P[8] * Z + P[11];
  const double iz = 1.0 / z;
  const double du = x * iz - u, dv = y * iz - v;
  r = du * du + dv * dv;
  return z > kDblEps;
}

struct Support { int cnt; double sum; int idx; };
__device__ __forceinline__ bool better(const Support& a, const Support& b) {     // strict, ties to the lower index
  return a.cnt > b.cnt || (a.cnt == b.cnt && (a.sum < b.sum || (a.sum == b.sum && a.idx < b.idx)));
}

struct PnPArgs {
  int n_queries;
  const int64_t* corr_begin;           // [nq+1]
  const double* p2d; const double* p3d;   // [n_corr][2], [n_corr][3]
  const int32_t* cam_model; const uint64_t* seed;
  double* params;                      // [nq][kQParams] cam | qvec | tvec: the RANSAC pose is written here
  double* work;                        // [5][n_corr] u, v, X, Y, Z of queries that do not fit on chip
  double* in_xyz; double* in_xy;       // [n_corr][3], [n_corr][2]: the winner's inliers, at the front of each query's range
  int32_t* n_refine;                   // [nq] inliers handed to the refinement (0: none)
  int64_t n_corr;
  double max_error, min_inlier_ratio, confidence, multiplier;
  int min_trials, max_trials, refine;
  int corr_cap;                        // correspondences a query may keep in shared memory
  pxr_pnp_result* results;
};

// CTA-wide sums of 28 doubles (the LO normal equations) in a fixed order: lanes by butterfly, warps in order
static __device__ void block_sum(double* v, int m, double* sred, double* out) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int k = 0; k < m; ++k) {
    const double s = warp_sum(v[k]);
    if (lane == 0) sred[warp * 28 + k] = s;
  }
  __syncthreads();
  if (threadIdx.x < m) {
    double s = 0.0;
    for (int w = 0; w < kPWarps; ++w) s += sred[w * 28 + threadIdx.x];
    out[threadIdx.x] = s;
  }
  __syncthreads();
}

__global__ void __launch_bounds__(kPThreads) pnp_ransac_kernel(PnPArgs a) {
  extern __shared__ __align__(16) double psm[];
  double* spose = psm;                                  // [kPHyp][12]
  double* ssum = spose + kPHyp * kPPose;                // [kPHyp]
  double* scorr = ssum + kPHyp;                         // [5][corr_cap]
  int* scnt = reinterpret_cast<int*>(scorr + 5 * (size_t)a.corr_cap);   // [kPHyp], -1: no hypothesis
  __shared__ int snsol[kPTrials];
  __shared__ double sbest[kPPose], slo[kPPose], sred[kPWarps * 28], ssys[28];
  __shared__ Support sbs;
  __shared__ int sflag[3];                              // run LO, stop, LO solve failed
  __shared__ int slo_won, sn_run;
  const int q = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (q >= a.n_queries) return;
  const int64_t ob = a.corr_begin[q];
  const int64_t n = a.corr_begin[q + 1] - ob;
  const int model = a.cam_model[q];
  const double* cam = a.params + (int64_t)q * kQParams;
  pxr_pnp_result* res = a.results + q;
  // ---- the correspondences in the normalised plane
  const bool on_chip = n <= a.corr_cap;
  const int64_t stride = on_chip ? a.corr_cap : a.n_corr;
  double* cu = on_chip ? scorr : a.work + ob;
  double* cv = cu + stride;
  double* cX = cv + stride;
  double* cY = cX + stride;
  double* cZ = cY + stride;
  for (int64_t i = tid; i < n; i += kPThreads) {
    double u, v;
    cam_image_to_world(model, cam, a.p2d[2 * (ob + i)], a.p2d[2 * (ob + i) + 1], u, v);
    cu[i] = u; cv[i] = v;
    cX[i] = a.p3d[3 * (ob + i)]; cY[i] = a.p3d[3 * (ob + i) + 1]; cZ[i] = a.p3d[3 * (ob + i) + 2];
  }
  const double thr = a.max_error / mean_focal(model, cam);
  const double thr2 = thr * thr;
  const uint64_t s0 = splitmix64(a.seed[q]);
  if (tid == 0) { sbs.cnt = -1; sbs.sum = INFINITY; sbs.idx = -1; slo_won = 0; sn_run = 0; }
  __syncthreads();
  for (int round = 0; n >= 3; ++round) {
    // ---- draw and solve
    if (tid < kPTrials) {
      const int64_t t = (int64_t)round * kPTrials + tid;
      int ns = 0, idx[3];
      if (t < a.max_trials && draw_sample(s0, t, n, idx)) {
        double x[3][2], X[3][3];
        for (int k = 0; k < 3; ++k) {
          x[k][0] = cu[idx[k]]; x[k][1] = cv[idx[k]];
          X[k][0] = cX[idx[k]]; X[k][1] = cY[idx[k]]; X[k][2] = cZ[idx[k]];
        }
        ns = p3p_lambda_twist(x, X, spose + (size_t)tid * 4 * kPPose);
      }
      snsol[tid] = ns;
    }
    __syncthreads();
    // ---- score: one warp per hypothesis
    for (int h = warp; h < kPHyp; h += kPWarps) {
      if ((h & 3) >= snsol[h >> 2]) { if (lane == 0) scnt[h] = -1; continue; }
      double P[kPPose];
#pragma unroll
      for (int k = 0; k < kPPose; ++k) P[k] = spose[h * kPPose + k];
      int cnt = 0;
      double sum = 0.0;
      for (int64_t i = lane; i < n; i += 32) {
        double r;
        if (pnp_residual(P, cu[i], cv[i], cX[i], cY[i], cZ[i], r) && r <= thr2) { ++cnt; sum += r; }
      }
      cnt = __reduce_add_sync(0xffffffffu, cnt);
      sum = warp_sum(sum);
      if (lane == 0) { scnt[h] = cnt; ssum[h] = sum; }
    }
    __syncthreads();
    // ---- the round's best (warp 0), and the query's
    if (warp == 0) {
      Support b{-1, INFINITY, 0x7fffffff};
      for (int h = lane * (kPHyp / 32); h < (lane + 1) * (kPHyp / 32); ++h) {
        const Support c{scnt[h], ssum[h], h};
        if (c.cnt >= 0 && better(c, b)) b = c;
      }
      for (int off = 16; off > 0; off >>= 1) {
        const Support o{__shfl_xor_sync(0xffffffffu, b.cnt, off), __shfl_xor_sync(0xffffffffu, b.sum, off),
                        __shfl_xor_sync(0xffffffffu, b.idx, off)};
        if (better(o, b)) b = o;
      }
      const Support cur = sbs;
      const bool improved = b.cnt >= 0 && (b.cnt > cur.cnt || (b.cnt == cur.cnt && b.sum < cur.sum));
      if (improved && lane < kPPose) sbest[lane] = spose[b.idx * kPPose + lane];
      __syncwarp();
      if (lane == 0) {
        if (improved) {
          sbs = Support{b.cnt, b.sum, round * kPHyp + b.idx};
          slo_won = 0;
        }
        sflag[0] = improved && b.cnt > 3; sflag[2] = 0;
      }
    }
    __syncthreads();
    // ---- local optimisation: Gauss-Newton over the new best's inliers, when they are more than a minimal sample
    if (sflag[0]) {
      double P0[kPPose], P[kPPose];
      for (int k = 0; k < kPPose; ++k) P0[k] = P[k] = sbest[k];
      for (int step = 0; step < kLOSteps; ++step) {
        double acc[28];
        for (int k = 0; k < 27; ++k) acc[k] = 0.0;
        for (int64_t i = tid; i < n; i += kPThreads) {
          double r;
          if (!(pnp_residual(P0, cu[i], cv[i], cX[i], cY[i], cZ[i], r) && r <= thr2)) continue;
          const double X = cX[i], Y = cY[i], Z = cZ[i];
          const double p0 = P[0] * X + P[1] * Y + P[2] * Z, p1 = P[3] * X + P[4] * Y + P[5] * Z,
                       p2 = P[6] * X + P[7] * Y + P[8] * Z;
          const double x = p0 + P[9], y = p1 + P[10], z = p2 + P[11];
          const double iz = 1.0 / z;
          const double res[2] = {x * iz - cu[i], y * iz - cv[i]};
          const double av[2][3] = {{iz, 0.0, -x * iz * iz}, {0.0, iz, -y * iz * iz}};
          double J[2][6];
          for (int rr = 0; rr < 2; ++rr) {
            const double* A = av[rr];
            J[rr][0] = -A[1] * p2 + A[2] * p1; J[rr][1] = A[0] * p2 - A[2] * p0; J[rr][2] = -A[0] * p1 + A[1] * p0;
            J[rr][3] = A[0]; J[rr][4] = A[1]; J[rr][5] = A[2];
          }
          int k = 0;
          for (int r0 = 0; r0 < 6; ++r0)
            for (int c0 = 0; c0 <= r0; ++c0) acc[k++] += J[0][r0] * J[0][c0] + J[1][r0] * J[1][c0];
          for (int r0 = 0; r0 < 6; ++r0) acc[21 + r0] += J[0][r0] * res[0] + J[1][r0] * res[1];
        }
        block_sum(acc, 27, sred, ssys);
        if (tid == 0) {
          double Lc[21], d[6];
          bool ok = true;
          for (int k = 0; k < 21; ++k) Lc[k] = ssys[k];
          for (int j = 0; j < 6 && ok; ++j) {
            double djj = Lc[qtri(j, j)];
            for (int k = 0; k < j; ++k) djj -= Lc[qtri(j, k)] * Lc[qtri(j, k)];
            if (!(djj > 0.0) || !isfinite(djj)) { ok = false; break; }
            const double ljj = sqrt(djj);
            Lc[qtri(j, j)] = ljj;
            for (int i = j + 1; i < 6; ++i) {
              double v = Lc[qtri(i, j)];
              for (int k = 0; k < j; ++k) v -= Lc[qtri(i, k)] * Lc[qtri(j, k)];
              Lc[qtri(i, j)] = v / ljj;
            }
          }
          if (ok) {
            for (int i = 0; i < 6; ++i) {
              double v = -ssys[21 + i];
              for (int k = 0; k < i; ++k) v -= Lc[qtri(i, k)] * d[k];
              d[i] = v / Lc[qtri(i, i)];
            }
            for (int i = 5; i >= 0; --i) {
              double v = d[i];
              for (int k = i + 1; k < 6; ++k) v -= Lc[qtri(k, i)] * d[k];
              d[i] = v / Lc[qtri(i, i)];
            }
            // R <- Exp(w) R, t <- t + dt
            const double th = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
            double E[9] = {0.0, -d[2], d[1], d[2], 0.0, -d[0], -d[1], d[0], 0.0};
            double Rx[9];
            if (th < 1e-12) {
              for (int k = 0; k < 9; ++k) Rx[k] = E[k] + ((k % 4) == 0 ? 1.0 : 0.0);
            } else {
              for (int k = 0; k < 9; ++k) E[k] = E[k] / th;
              const double sn = sin(th), cs = 1.0 - cos(th);
              for (int i = 0; i < 3; ++i)
                for (int j = 0; j < 3; ++j) {
                  const double e2 = E[3 * i] * E[j] + E[3 * i + 1] * E[3 + j] + E[3 * i + 2] * E[6 + j];
                  Rx[3 * i + j] = (i == j ? 1.0 : 0.0) + sn * E[3 * i + j] + cs * e2;
                }
            }
            for (int i = 0; i < 3; ++i)
              for (int j = 0; j < 3; ++j)
                slo[3 * i + j] = Rx[3 * i] * P[j] + Rx[3 * i + 1] * P[3 + j] + Rx[3 * i + 2] * P[6 + j];
            for (int i = 0; i < 3; ++i) slo[9 + i] = P[9 + i] + d[3 + i];
          }
          sflag[2] = !ok;
        }
        __syncthreads();
        if (sflag[2]) break;
        for (int k = 0; k < kPPose; ++k) P[k] = slo[k];
        __syncthreads();
      }
      // the support of the optimised pose
      double acc[2] = {0.0, 0.0};
      bool finite = true;
      for (int k = 0; k < kPPose; ++k) finite = finite && isfinite(P[k]);
      for (int64_t i = tid; i < n && finite; i += kPThreads) {
        double r;
        if (pnp_residual(P, cu[i], cv[i], cX[i], cY[i], cZ[i], r) && r <= thr2) { acc[0] += 1.0; acc[1] += r; }
      }
      block_sum(acc, 2, sred, ssys);
      if (tid == 0 && finite) {
        const int c = (int)ssys[0];
        if (c > sbs.cnt || (c == sbs.cnt && ssys[1] < sbs.sum)) {
          sbs.cnt = c; sbs.sum = ssys[1]; slo_won = 1;
          for (int k = 0; k < kPPose; ++k) sbest[k] = P[k];
        }
      }
    }
    // ---- COLMAP's dynamic trial count
    if (tid == 0) {
      const int64_t run = std::min<int64_t>((int64_t)(round + 1) * kPTrials, a.max_trials);
      double req = (double)a.max_trials;
      if (sbs.cnt > 0) {
        const double ratio = (double)sbs.cnt / (double)n;
        const double nom = 1.0 - a.confidence;
        if (nom > 0.0) {
          const double denom = 1.0 - ratio * ratio * ratio;
          if (denom <= 0.0) req = 1.0;
          else if (denom != 1.0) req = ceil(log(nom) / log(denom) * a.multiplier);
        }
      }
      req = fmin(fmax(req, (double)a.min_trials), (double)a.max_trials);
      sn_run = (int)run;
      sflag[1] = (double)run >= req;
    }
    __syncthreads();
    if (sflag[1]) break;
  }
  // ---- report; the winner's inliers go to the refinement, compacted in order
  const Support best = sbs;
  const bool success = n >= 3 && best.cnt >= 3 && (double)best.cnt / (double)n >= a.min_inlier_ratio;
  double P[kPPose];
  for (int k = 0; k < kPPose; ++k) P[k] = sbest[k];
  int64_t kept = 0;
  if (success) {
    for (int64_t base = 0; base < n; base += kPThreads) {
      const int64_t i = base + tid;
      double r;
      const bool inl = i < n && pnp_residual(P, cu[i], cv[i], cX[i], cY[i], cZ[i], r) && r <= thr2;
      const unsigned bal = __ballot_sync(0xffffffffu, inl);
      if (lane == 0) snsol[warp] = __popc(bal);
      __syncthreads();
      int64_t off = kept;
      for (int w = 0; w < warp; ++w) off += snsol[w];
      off += __popc(bal & ((1u << lane) - 1u));
      if (inl) {
        const int64_t o = ob + i, d = ob + off;
        a.in_xyz[3 * d] = a.p3d[3 * o]; a.in_xyz[3 * d + 1] = a.p3d[3 * o + 1]; a.in_xyz[3 * d + 2] = a.p3d[3 * o + 2];
        a.in_xy[2 * d] = a.p2d[2 * o]; a.in_xy[2 * d + 1] = a.p2d[2 * o + 1];
      }
      for (int w = 0; w < kPWarps; ++w) kept += snsol[w];
      __syncthreads();
    }
  }
  if (tid == 0) {
    res->status = PXR_OK;
    res->success = success;
    res->num_inliers = success ? best.cnt : 0;
    res->num_trials = sn_run;
    res->best_trial = best.idx >= 0 ? best.idx >> 2 : -1;
    res->best_solution = best.idx >= 0 ? best.idx & 3 : -1;
    res->local_optimized = best.idx >= 0 ? slo_won : 0;
    res->num_iterations = 0; res->termination_type = 0;
    res->initial_cost = 0.0; res->final_cost = 0.0;
    a.n_refine[q] = success && a.refine ? (int32_t)kept : 0;
    if (success) {
      double* prm = a.params + (int64_t)q * kQParams;
      rot_to_quat(P, prm + kMaxK);
      for (int k = 0; k < 3; ++k) prm[kMaxK + 4 + k] = P[9 + k];
    }
  }
}

// Linearisation of the refinement at prm (whole CTA), in qba_evaluate's layout: every lane projects one inlier into its
// shared row [rho' rx, rho' ry, rho, rho', Ju(n), Jv(n)], then each lane accumulates its entries of J^T J / J^T r over
// the warp's rows in order; the warps' partials are summed in warp order.
static __device__ double pnp_evaluate(const QBAArgs& a, const double* obs, const double* prm, int model, uint32_t mask, int n,
                               double* H, double* g, double* rows, double* part, int64_t ob, int64_t oe) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int RS = a.row_stride;
  double* wrow = rows + (size_t)warp * 32 * RS;
  const int ntri = n * (n + 1) / 2, nent = ntri + n;
  int ea[kQEntries], eb[kQEntries];
#pragma unroll
  for (int i = 0; i < kQEntries; ++i) {
    const int k = lane + 32 * i;
    ea[i] = -1; eb[i] = -1;
    if (k < ntri) { int r = 0; while ((r + 1) * (r + 2) / 2 <= k) ++r; ea[i] = r; eb[i] = k - r * (r + 1) / 2; }
    else if (k < nent) ea[i] = k - ntri;
  }
  double acc[kQEntries];
#pragma unroll
  for (int i = 0; i < kQEntries; ++i) acc[i] = 0.0;
  double cost = 0.0;
  const int Kc = cam_num_params(model);
  for (int64_t b0 = ob + (int64_t)warp * 32; b0 < oe; b0 += kQWarps * 32) {
    __syncwarp();
    const int64_t o = b0 + lane;
    if (o < oe) {
      double X[3], xy[2], Jpose[2][6], Jpt[2][3], Jk[2][kMaxK];
      for (int k = 0; k < 3; ++k) X[k] = a.xyz[3 * o + k];
      world_to_pixel<true>(model, prm, prm + kMaxK, prm + kMaxK + 4, X, xy, Jpose, Jpt, Jk);
      const double rx = xy[0] - obs[2 * o], ry = xy[1] - obs[2 * o + 1];
      double rho[3];
      loss_eval(a.loss, 1.0, rx * rx + ry * ry, rho);
      double* r = wrow + lane * RS;
      r[0] = rho[1] * rx; r[1] = rho[1] * ry; r[2] = rho[0]; r[3] = rho[1];
      for (int k = 0; k < 6; ++k) { r[4 + k] = Jpose[0][k]; r[4 + n + k] = Jpose[1][k]; }
      int c = 6;
      for (int k = 0; k < kMaxK; ++k)
        if (k < Kc && !((mask >> k) & 1u)) { r[4 + c] = Jk[0][k]; r[4 + n + c] = Jk[1][k]; ++c; }
    }
    __syncwarp();
    const int nb = (int)min((int64_t)32, oe - b0);
    for (int j = 0; j < nb; ++j) {
      const double* r = wrow + j * RS;
      const double w = r[3];
      const double* Ju = r + 4;
      const double* Jv = r + 4 + n;
      cost += 0.5 * r[2];
#pragma unroll
      for (int i = 0; i < kQEntries; ++i) {
        const int ia = ea[i], ib = eb[i];
        if (ia < 0) continue;
        if (ib >= 0) acc[i] += w * (Ju[ia] * Ju[ib] + Jv[ia] * Jv[ib]);
        else acc[i] += Ju[ia] * r[0] + Jv[ia] * r[1];
      }
    }
  }
  double* mine = part + warp * kQPart;
#pragma unroll
  for (int i = 0; i < kQEntries; ++i)
    if (ea[i] >= 0) mine[lane + 32 * i] = acc[i];
  if (lane == 0) mine[nent] = cost;
  __syncthreads();
  for (int k = threadIdx.x; k <= nent; k += kQThreads) {
    double s = 0.0;
    for (int wi = 0; wi < kQWarps; ++wi) s += part[wi * kQPart + k];
    if (k < ntri) H[k] = s;
    else if (k < nent) g[k - ntri] = s;
    else part[kQWarps * kQPart] = s;
  }
  __syncthreads();
  const double total = part[kQWarps * kQPart];
  __syncthreads();
  return total;
}

struct PnPRefineArgs {
  const int64_t* corr_begin;
  const int32_t* n_refine;
  const double* in_xy;
  const double* p2d; const double* p3d;
  uint8_t* mask;
  double max_error;
  pxr_pnp_result* results;
};

__global__ void __launch_bounds__(kQThreads) pnp_refine_kernel(QBAArgs a, PnPRefineArgs r) {
  extern __shared__ __align__(16) double prows[];
  __shared__ double spart[kQWarps * kQPart + 1];
  __shared__ int sok;
  const int q = blockIdx.x, tid = threadIdx.x;
  if (q >= a.n_queries) return;
  const int64_t ob = r.corr_begin[q], n = r.corr_begin[q + 1] - ob;
  const int64_t oe = ob + r.n_refine[q];
  qba_lm_solve(a, q, ob, oe, [&](const double* prm, int model, uint32_t mask, int nt, double* H, double* g) {
    return pnp_evaluate(a, r.in_xy, prm, model, mask, nt, H, g, prows, spart, ob, oe);
  });
  __syncthreads();
  if (tid == 0) {
    pxr_pnp_result* res = r.results + q;
    const pxr_qba_result& lm = a.results[q];
    if (lm.status != PXR_OK) { res->status = lm.status; res->success = 0; }
    res->num_iterations = lm.num_iterations; res->termination_type = lm.termination_type;
    res->initial_cost = lm.initial_cost; res->final_cost = lm.final_cost;
    sok = res->success;
  }
  __syncthreads();
  // the inliers of the returned pose, with the returned intrinsics
  const double* prm = a.params + (int64_t)q * kQParams;
  const int model = a.cam_model[q];
  double P[kPPose];
  quat_to_rot(prm + kMaxK, P);
  for (int k = 0; k < 3; ++k) P[9 + k] = prm[kMaxK + 4 + k];
  const double thr = r.max_error / mean_focal(model, prm);
  const double thr2 = thr * thr;
  int count = 0;
  for (int64_t base = 0; base < n; base += kQThreads) {
    const int64_t i = base + tid;
    bool inl = false;
    if (i < n && sok) {
      const int64_t o = ob + i;
      double u, v, res2;
      cam_image_to_world(model, prm, r.p2d[2 * o], r.p2d[2 * o + 1], u, v);
      inl = pnp_residual(P, u, v, r.p3d[3 * o], r.p3d[3 * o + 1], r.p3d[3 * o + 2], res2) && res2 <= thr2;
    }
    if (i < n) r.mask[ob + i] = inl ? 1 : 0;
    count += __syncthreads_count(inl);
  }
  if (tid == 0) r.results[q].num_inliers = sok ? count : 0;
}

__global__ void pnp_image_to_world_kernel(int model, const double* params, int64_t n, const double* xy, double* out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) cam_image_to_world(model, params, xy[2 * i], xy[2 * i + 1], out[2 * i], out[2 * i + 1]);
}

__global__ void pnp_p3p_kernel(int64_t n, const double* x, const double* X, double* poses, int32_t* n_sol) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double xx[3][2], XX[3][3], P[4 * kPPose];
  for (int k = 0; k < 3; ++k) {
    xx[k][0] = x[6 * i + 2 * k]; xx[k][1] = x[6 * i + 2 * k + 1];
    for (int j = 0; j < 3; ++j) XX[k][j] = X[9 * i + 3 * k + j];
  }
  const int ns = p3p_lambda_twist(xx, XX, P);
  n_sol[i] = ns;
  for (int s = 0; s < 4; ++s) {
    double* out = poses + (i * 4 + s) * 7;
    if (s < ns) {
      rot_to_quat(P + s * kPPose, out);
      for (int k = 0; k < 3; ++k) out[4 + k] = P[s * kPPose + 9 + k];
    } else {
      for (int k = 0; k < 7; ++k) out[k] = 0.0;
    }
  }
}

// ---- host side --------------------------------------------------------------------------------------------------
static int check_pnp(const pxr_pnp_desc* d, const pxr_pnp_options* o) {
  if (!d) return fail(PXR_ERR_INVALID_ARGUMENT, "desc is NULL");
  if (!o) return fail(PXR_ERR_INVALID_ARGUMENT, "options is NULL");
  if (d->n_queries < 0) return fail(PXR_ERR_INVALID_ARGUMENT, "n_queries < 0");
  if (o->estimate_focal_length)
    return fail(PXR_ERR_UNSUPPORTED, "estimate_focal_length is not supported: RANSAC estimates the pose only");
  if (!(o->max_error > 0.0)) return fail(PXR_ERR_INVALID_ARGUMENT, "max_error must be > 0");
  if (!(o->confidence >= 0.0 && o->confidence <= 1.0)) return fail(PXR_ERR_INVALID_ARGUMENT, "confidence must be in [0, 1]");
  if (o->min_num_trials < 0 || o->max_num_trials < 1 || o->min_num_trials > o->max_num_trials)
    return fail(PXR_ERR_INVALID_ARGUMENT, "need 0 <= min_num_trials <= max_num_trials, max_num_trials >= 1");
  if (!(o->dyn_num_trials_multiplier > 0.0)) return fail(PXR_ERR_INVALID_ARGUMENT, "dyn_num_trials_multiplier must be > 0");
  if (o->refine && (o->max_num_iterations < 0 || !(o->loss_function_scale > 0.0) || !(o->gradient_tolerance >= 0.0) ||
                    !(o->function_tolerance >= 0.0) || !(o->parameter_tolerance >= 0.0)))
    return fail(PXR_ERR_INVALID_ARGUMENT, "bad refinement options");
  if (d->n_queries == 0) return PXR_OK;
  if (!d->corr_begin || !d->cam_model || !d->cam_params || !d->seed || !d->qvec || !d->tvec)
    return fail(PXR_ERR_INVALID_ARGUMENT, "a required array is NULL");
  if (d->corr_begin[0] != 0) return fail(PXR_ERR_INVALID_ARGUMENT, "corr_begin[0] must be 0");
  for (int q = 0; q < d->n_queries; ++q) {
    if (d->corr_begin[q + 1] < d->corr_begin[q]) return fail(PXR_ERR_INVALID_ARGUMENT, "corr_begin must be non-decreasing");
    if (d->corr_begin[q + 1] - d->corr_begin[q] > INT32_MAX)
      return fail(PXR_ERR_INVALID_ARGUMENT, "query %d has more than 2^31 - 1 correspondences", q);
    if (cam_num_params(d->cam_model[q]) == 0) return fail(PXR_ERR_UNSUPPORTED, "unsupported camera model id %d", d->cam_model[q]);
  }
  if (d->corr_begin[d->n_queries] > 0 && (!d->points2D || !d->points3D || !d->inlier_mask))
    return fail(PXR_ERR_INVALID_ARGUMENT, "a required array is NULL");
  return PXR_OK;
}

// principal point always constant; focal length and extra parameters as the options ask (RefineAbsolutePose)
static uint32_t refine_const_mask(int model, const pxr_pnp_options* o) {
  const int K = cam_num_params(model);
  const int nf = (model == 0 || model == 2 || model == 3) ? 1 : 2;
  uint32_t m = 0;
  for (int k = 0; k < K; ++k) {
    const bool free_ = (k < nf && o->refine_focal_length) || (k >= nf + 2 && o->refine_extra_params);
    if (!free_) m |= 1u << k;
  }
  return m;
}

}  // namespace pxr

using namespace pxr;

extern "C" void pxr_default_pnp_options(pxr_pnp_options* o) {
  if (!o) return;
  std::memset(o, 0, sizeof(*o));
  o->max_error = 12.0; o->min_inlier_ratio = 0.01; o->min_num_trials = 1000; o->max_num_trials = 100000;
  o->confidence = 0.9999; o->dyn_num_trials_multiplier = 3.0; o->estimate_focal_length = 0;
  o->refine = 1; o->gradient_tolerance = 1.0; o->max_num_iterations = 100; o->loss_function_scale = 1.0;
  o->refine_focal_length = 0; o->refine_extra_params = 0;
  o->function_tolerance = 1e-6; o->parameter_tolerance = 1e-8;
}

// One launch of each kernel for the whole batch: the upload is 40 bytes per correspondence and the device workspace
// another 80 (normalised points for queries that do not fit on chip, the compacted inliers), so a million
// correspondences take 120 MB; unlike the featuremetric solvers there are no patches whose size calls for waves.
extern "C" int pxr_pnp_run(pxr_ctx* ctx, const pxr_pnp_desc* d, const pxr_pnp_options* opt, pxr_pnp_result* results,
                           pxr_summary* total) {
  const auto t0 = std::chrono::steady_clock::now();
  PXR_TRY(check_pnp(d, opt));
  if (!results && d->n_queries > 0) return fail(PXR_ERR_INVALID_ARGUMENT, "results is NULL");
  PXR_TRY(require_ctx(ctx));
  const int nq = d->n_queries;
  const int64_t nc = nq ? d->corr_begin[nq] : 0;
  double kernel_ms = 0.0, h2d = 0.0;
  const int64_t launches0 = ctx->launches;
  if (nq > 0) {
    PXR_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    int64_t max_n = 0;
    for (int q = 0; q < nq; ++q) max_n = std::max<int64_t>(max_n, d->corr_begin[q + 1] - d->corr_begin[q]);
    // per query: params, corr_begin, model, const mask, seed; per correspondence: points, workspace, inliers, mask
    std::vector<double> params((size_t)nq * kQParams, 0.0);
    std::vector<uint32_t> cmask(nq);
    for (int q = 0; q < nq; ++q) {
      std::memcpy(params.data() + (size_t)q * kQParams, d->cam_params + (size_t)q * kMaxK, kMaxK * 8);
      params[(size_t)q * kQParams + kMaxK] = 1.0;
      cmask[q] = refine_const_mask(d->cam_model[q], opt);
    }
    DevBuf<double> dparams, dp2d, dp3d, dwork, din_xyz, din_xy;
    DevBuf<int64_t> dbegin;
    DevBuf<int32_t> dmodel, dnref;
    DevBuf<uint32_t> dcmask;
    DevBuf<uint64_t> dseed;
    DevBuf<uint8_t> dmask;
    DevBuf<pxr_pnp_result> dres;
    DevBuf<pxr_qba_result> dlm;
    PXR_TRY(dparams.upload(params.data(), params.size(), s));
    PXR_TRY(dbegin.upload(d->corr_begin, (size_t)nq + 1, s));
    PXR_TRY(dmodel.upload(d->cam_model, nq, s));
    PXR_TRY(dcmask.upload(cmask.data(), nq, s));
    PXR_TRY(dseed.upload(d->seed, nq, s));
    PXR_TRY(dp2d.upload(d->points2D, (size_t)nc * 2, s));
    PXR_TRY(dp3d.upload(d->points3D, (size_t)nc * 3, s));
    h2d = (double)nq * (kQParams * 8 + 8 + 4 + 4 + 8) + 8.0 + (double)nc * kCorrBytes;
    const int cap = (int)std::min<int64_t>(max_n, (int64_t)(kPCorrSmem / kCorrBytes));
    const bool spill = max_n > cap;
    PXR_TRY(dwork.alloc(spill ? (size_t)nc * 5 : 1));
    PXR_TRY(din_xyz.alloc((size_t)std::max<int64_t>(nc, 1) * 3));
    PXR_TRY(din_xy.alloc((size_t)std::max<int64_t>(nc, 1) * 2));
    PXR_TRY(dnref.alloc(nq));
    PXR_TRY(dmask.alloc((size_t)std::max<int64_t>(nc, 1)));
    PXR_TRY(dres.alloc(nq));
    PXR_TRY(dlm.alloc(nq));
    PnPArgs pa;
    std::memset(&pa, 0, sizeof(pa));
    pa.n_queries = nq; pa.corr_begin = dbegin.p; pa.p2d = dp2d.p; pa.p3d = dp3d.p; pa.cam_model = dmodel.p;
    pa.seed = dseed.p; pa.params = dparams.p; pa.work = dwork.p; pa.in_xyz = din_xyz.p; pa.in_xy = din_xy.p;
    pa.n_refine = dnref.p; pa.n_corr = nc; pa.max_error = opt->max_error; pa.min_inlier_ratio = opt->min_inlier_ratio;
    pa.confidence = opt->confidence; pa.multiplier = opt->dyn_num_trials_multiplier;
    pa.min_trials = opt->min_num_trials; pa.max_trials = opt->max_num_trials; pa.refine = opt->refine;
    pa.corr_cap = cap; pa.results = dres.p;
    const size_t smem_r = (size_t)kPHyp * kPPose * 8 + (size_t)kPHyp * 8 + (size_t)cap * kCorrBytes + (size_t)kPHyp * 4;
    // ceres' defaults where COLMAP's RefineAbsolutePose leaves them
    QBAArgs la;
    std::memset(&la, 0, sizeof(la));
    la.n_queries = nq; la.cam_model = dmodel.p; la.cam_mask = dcmask.p; la.params = dparams.p; la.xyz = din_xyz.p;
    la.loss.type = PXR_LOSS_CAUCHY; la.loss.a = opt->loss_function_scale;
    la.max_iter = opt->max_num_iterations; la.max_invalid = 5; la.max_nonmonotonic = 0; la.jacobi_scaling = 1;
    la.ftol = opt->function_tolerance; la.gtol = opt->gradient_tolerance; la.ptol = opt->parameter_tolerance; la.min_rel_dec = 1e-3;
    la.radius0 = 1e4; la.max_radius = 1e16; la.min_radius = 1e-32; la.min_diag = 1e-6; la.max_diag = 1e32;
    int nmax = 6;
    for (int q = 0; q < nq; ++q) {
      int nt = 6;
      for (int k = 0; k < cam_num_params(d->cam_model[q]); ++k) nt += ((cmask[q] >> k) & 1u) ? 0 : 1;
      nmax = std::max(nmax, nt);
    }
    la.row_stride = (4 + 2 * nmax) | 1;
    la.results = dlm.p;
    PnPRefineArgs ra;
    ra.corr_begin = dbegin.p; ra.n_refine = dnref.p; ra.in_xy = din_xy.p; ra.p2d = dp2d.p; ra.p3d = dp3d.p;
    ra.mask = dmask.p; ra.max_error = opt->max_error; ra.results = dres.p;
    const size_t smem_f = (size_t)kQWarps * 32 * la.row_stride * sizeof(double);
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    struct Events { cudaEvent_t* a; cudaEvent_t* b; ~Events() { if (*a) cudaEventDestroy(*a); if (*b) cudaEventDestroy(*b); } } guard{&e0, &e1};
    PXR_CUDA(cudaEventCreate(&e0));
    PXR_CUDA(cudaEventCreate(&e1));
    PXR_CUDA(cudaFuncSetAttribute(pnp_ransac_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_r));
    PXR_CUDA(cudaFuncSetAttribute(pnp_refine_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_f));
    PXR_CUDA(cudaEventRecord(e0, s));
    PXR_LAUNCH(ctx, pnp_ransac_kernel, nq, kPThreads, smem_r, pa);
    PXR_CUDA(cudaGetLastError());
    PXR_LAUNCH(ctx, pnp_refine_kernel, nq, kQThreads, smem_f, la, ra);
    PXR_CUDA(cudaGetLastError());
    PXR_CUDA(cudaEventRecord(e1, s));
    std::vector<pxr_pnp_result> hres(nq);
    PXR_CUDA(cudaMemcpyAsync(params.data(), dparams.p, params.size() * 8, cudaMemcpyDeviceToHost, s));
    PXR_CUDA(cudaMemcpyAsync(hres.data(), dres.p, (size_t)nq * sizeof(pxr_pnp_result), cudaMemcpyDeviceToHost, s));
    if (nc) PXR_CUDA(cudaMemcpyAsync(d->inlier_mask, dmask.p, (size_t)nc, cudaMemcpyDeviceToHost, s));
    PXR_CUDA(cudaStreamSynchronize(s));
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, e0, e1) == cudaSuccess) kernel_ms = ms;
    const bool intrinsics = opt->refine && (opt->refine_focal_length || opt->refine_extra_params);
    for (int q = 0; q < nq; ++q) {
      results[q] = hres[q];
      if (!hres[q].success) continue;
      const double* p = params.data() + (size_t)q * kQParams;
      std::memcpy(d->qvec + (size_t)q * 4, p + kMaxK, 32);
      std::memcpy(d->tvec + (size_t)q * 3, p + kMaxK + 4, 24);
      if (intrinsics) std::memcpy(d->cam_params + (size_t)q * kMaxK, p, kMaxK * 8);
    }
  }
  if (total) {
    const int cap_it = total->iterations_capacity;
    pxr_iteration_summary* keep = total->iterations;
    std::memset(total, 0, sizeof(*total));
    total->iterations_capacity = cap_it; total->iterations = keep;
    total->h2d_bytes = h2d;
    total->kernel_launches = ctx->launches - launches0;
    total->total_time_s = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    total->solve_time_s = kernel_ms * 1e-3;
    std::snprintf(total->message, sizeof(total->message), "%d queries, %lld correspondences, kernels %.3f ms", nq,
                  (long long)nc, kernel_ms);
  }
  return PXR_OK;
}

extern "C" int pxr_pnp_debug_image_to_world(pxr_ctx* ctx, int32_t model, const double* params, int64_t n, const double* xy,
                                            double* out) {
  if (cam_num_params(model) == 0) return fail(PXR_ERR_UNSUPPORTED, "unsupported camera model id %d", model);
  if (n < 0 || !params || (n > 0 && (!xy || !out))) return fail(PXR_ERR_INVALID_ARGUMENT, "bad arguments");
  PXR_TRY(require_ctx(ctx));
  if (n == 0) return PXR_OK;
  PXR_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  DevBuf<double> dp, dxy, dout;
  PXR_TRY(dp.upload(params, kMaxK, s));
  PXR_TRY(dxy.upload(xy, (size_t)n * 2, s));
  PXR_TRY(dout.alloc((size_t)n * 2));
  PXR_LAUNCH(ctx, pnp_image_to_world_kernel, (unsigned)cdiv(n, 128), 128, 0, model, dp.p, n, dxy.p, dout.p);
  PXR_CUDA(cudaGetLastError());
  PXR_CUDA(cudaMemcpyAsync(out, dout.p, (size_t)n * 16, cudaMemcpyDeviceToHost, s));
  PXR_CUDA(cudaStreamSynchronize(s));
  return PXR_OK;
}

extern "C" int pxr_pnp_debug_p3p(pxr_ctx* ctx, int64_t n, const double* x, const double* X, double* poses, int32_t* n_sol) {
  if (n < 0 || (n > 0 && (!x || !X || !poses || !n_sol))) return fail(PXR_ERR_INVALID_ARGUMENT, "bad arguments");
  PXR_TRY(require_ctx(ctx));
  if (n == 0) return PXR_OK;
  PXR_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  DevBuf<double> dx, dX, dposes;
  DevBuf<int32_t> dn;
  PXR_TRY(dx.upload(x, (size_t)n * 6, s));
  PXR_TRY(dX.upload(X, (size_t)n * 9, s));
  PXR_TRY(dposes.alloc((size_t)n * 28));
  PXR_TRY(dn.alloc(n));
  PXR_LAUNCH(ctx, pnp_p3p_kernel, (unsigned)cdiv(n, 128), 128, 0, n, dx.p, dX.p, dposes.p, dn.p);
  PXR_CUDA(cudaGetLastError());
  PXR_CUDA(cudaMemcpyAsync(poses, dposes.p, (size_t)n * 28 * 8, cudaMemcpyDeviceToHost, s));
  PXR_CUDA(cudaMemcpyAsync(n_sol, dn.p, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
  PXR_CUDA(cudaStreamSynchronize(s));
  return PXR_OK;
}
