// pxr_ka.cu — featuremetric keypoint adjustment on the device.
//
// Replaces _keypoint_adjustment.FeatureMetricKeypointOptimizer.run (reference
// pixsfm/keypoint_adjustment/src/featuremetric_keypoint_optimizer.h:50-202): thousands of small
// independent non-linear least-squares problems (<= max_kps_per_problem keypoints each,
// base/src/parallel_optimizer.h:77-211).  One CTA solves one problem end to end:
//   residual  FeatureMetric2DCostFunctor (residuals/src/featuremetric.h:24-69):
//             r = interp(patch1, kp1) - interp(patch2, kp2), J = [G1 s1 | -G2 s2]
//   loss      ceres::ScaledLoss(Cauchy, similarity) (featuremetric_keypoint_optimizer.h:191-196)
//   bounds    KeypointOptimizerBase::ParameterizeKeypoints (keypoint_optimizer.h:110-157)
//   solve     ceres::Solve: bounded Levenberg-Marquardt with projected Armijo line search
//             (TrustRegionMinimizer::DoLineSearch), Cholesky per connected component of the problem (the
//             reference's SPARSE_NORMAL_CHOLESKY is an exact factorization too); the workspace lives in shared
//             memory, or in global memory for a problem whose workspace does not fit there.
// Feature windows are re-read from L2 on every evaluation: after first touch a problem's working
// set (<= 50 windows x 4 KiB) is cache resident, so KA is compute/L2 bound, not HBM bound.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <unordered_map>
#include <vector>

#include "pxr_fm_eval.cuh"
#include "pxr_internal.h"
#include "pxr_lm.cuh"
#include "pxr_waves.h"

namespace pxr {

struct KAArgs {
  // problems
  int n_problems;
  const int64_t* prob_edge_begin;   // [P+1]
  const int32_t* prob_var_begin;    // [P+1] offsets into var arrays
  // edges (sorted by problem)
  const int64_t* e_k1; const int64_t* e_k2;   // global keypoint ids
  const int32_t* e_v1; const int32_t* e_v2;   // local variable index inside the problem or -1
  const double* e_w;                          // ScaledLoss weight
  // variables
  const int64_t* var_kp;            // [n_var] global keypoint id
  const double* var_lower; const double* var_upper;  // [n_var][2]
  // keypoints / patches
  double* keypoints;                // [n_kp][2] in/out
  const int64_t* kp_patch;          // or null
  const uint8_t* patches; int ph, pw;
  const int32_t* corner; const double* scale; double ups;
  // options
  LossParams loss; int l2_normalize; int constrained;
  int max_iter, max_invalid;
  double ftol, gtol, ptol, min_rel_dec, radius0, max_radius, min_radius, min_diag, max_diag;
  int jacobi_scaling;
  int max_nonmonotonic;             // 0: monotonic steps; > 0: use_nonmonotonic_steps with this many consecutive ones
  // outputs per problem: initial cost, final cost, iterations, successful, unsuccessful, termination
  double* prob_out;                 // [P][6]
  // query mode (REF): every edge is (keypoint e_k1, fixed descriptor ref_desc[e_k2]); block-diagonal normal equations,
  // workspace in global memory so that a problem may hold any number of keypoints
  // dense mode: the normal equations are block diagonal over the connected components of the problem's edge graph
  // (tracks packed into one problem do not couple); per variable the scalar range [lo, hi) of its component and the
  // offset of the component's packed lower triangle inside the problem's H and L
  const int32_t* var_blk_lo; const int32_t* var_blk_hi; const int32_t* var_blk_off;   // [n_var]
  const double* ref_desc;           // [n_ref][C]
  // per problem: its workspace (2 m + 10 n doubles, m = matrix size) at workspace + ws_off[p], or in shared memory
  // where ws_off is NULL or ws_off[p] < 0
  double* workspace; const int64_t* ws_off;
};

constexpr int kKAThreads = 256;
constexpr int kKAWarps = kKAThreads / 32;

__device__ __forceinline__ int tri(int i, int j) { return i * (i + 1) / 2 + j; }  // i >= j

// L2 normalisation of one descriptor (PixelInterpolator::Evaluate, interpolation.h:648-666)
template <int CPL, bool DERIV>
__device__ __forceinline__ void l2_normalize_desc(bool active, double f[CPL], double fr[CPL], double fc[CPL]) {
  double n2 = 0.0;
  if (active) {
#pragma unroll
    for (int k = 0; k < CPL; ++k) n2 += f[k] * f[k];
  }
  n2 = warp_sum(n2);
  const double ninv = 1.0 / sqrt(n2);
  double dc = 0.0, dr = 0.0;
#pragma unroll
  for (int k = 0; k < CPL; ++k) {
    f[k] *= ninv;
    if (DERIV) { fc[k] *= ninv; fr[k] *= ninv; if (active) { dc += f[k] * fc[k]; dr += f[k] * fr[k]; } }
  }
  if (DERIV) {
    dc = warp_sum(dc); dr = warp_sum(dr);
#pragma unroll
    for (int k = 0; k < CPL; ++k) { fc[k] -= dc * f[k]; fr[k] -= dr * f[k]; }
  }
}

template <typename T, int C>
__device__ __forceinline__ GlobalWindow make_window(const KAArgs& a, int64_t kp, const double* xy, double& xc, double& xr,
                                                    double& sx, double& sy) {
  constexpr int TAP_BYTES = C * (int)sizeof(T);
  const int64_t pi = a.kp_patch ? a.kp_patch[kp] : kp;
  sx = a.scale[2 * pi] * a.ups; sy = a.scale[2 * pi + 1] * a.ups;
  const double u = (xy[0] * a.scale[2 * pi] - 0.5 - (double)a.corner[2 * pi]) * a.ups;
  const double v = (xy[1] * a.scale[2 * pi + 1] - 0.5 - (double)a.corner[2 * pi + 1]) * a.ups;
  const double fu = floor(u), fv = floor(v);
  const int col = (int)fmin(fmax(fu, -4.0), (double)a.pw + 4.0);
  const int row = (int)fmin(fmax(fv, -4.0), (double)a.ph + 4.0);
  xc = u - fu; xr = v - fv;
  const uint8_t* src = a.patches + pi * (int64_t)a.ph * a.pw * TAP_BYTES;
  GlobalWindow w;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int rr = min(max(row - 1 + i, 0), a.ph - 1);
    w.rowp[i] = src + (int64_t)rr * a.pw * TAP_BYTES;
    w.coff[i] = min(max(col - 1 + i, 0), a.pw - 1) * TAP_BYTES;
  }
  return w;
}

// Workspace of one problem: shared memory, or global memory for a problem too large for it
struct KAWork {
  int m;          // doubles per matrix
  const int32_t* blo; const int32_t* boff;   // the problem's var_blk_lo / var_blk_off
  double* H;      // per component packed lower: J^T J at x (REF: h00, h10, h11 per keypoint)
  double* L;      // per component packed lower: factor of H + D
  double* g;      // J^T r at x
  double* gq;     // gradient at a line-search trial point
  double* x; double* cand; double* delta; double* scale; double* D2; double* lo; double* hi; double* tmp;
  double* wcost;  // [kKAWarps]
  double* ctrl;   // scalars shared between thread 0 and the CTA
};

// mode 0: cost, 1: cost + gradient (into gout), 2: cost + gradient + J^T J (into H, gout)
// REF: block-diagonal mode, H holds (h00, h10, h11) per keypoint
template <typename T, int C, bool FS, bool REF>
__device__ double ka_evaluate(const KAArgs& a, const KAWork& w, int64_t eb, int64_t ee, int n, const double* xv, int mode,
                              double* gout) {
  constexpr int CPL = C >= 32 ? C / 32 : 1;
  constexpr int ACTIVE = C / CPL;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool active = lane < ACTIVE;
  __syncthreads();
  if (mode >= 1) for (int i = threadIdx.x; i < n; i += kKAThreads) gout[i] = 0.0;
  if (mode == 2) for (int i = threadIdx.x; i < w.m; i += kKAThreads) w.H[i] = 0.0;
  __syncthreads();
  double cost = 0.0;
  for (int64_t e = eb + warp; e < ee; e += kKAWarps) {
    const int64_t k1 = a.e_k1[e], k2 = a.e_k2[e];
    if (!REF && k1 == k2) continue;  // "Avoid optimizing a keypoint to itself" (topological_keypoint_optimizer.h:139-143)
    const int v1 = a.e_v1[e], v2 = REF ? -1 : a.e_v2[e];
    // J^T J of the edge goes into its component's triangle (both variable endpoints lie in one component); the
    // offsets are read here, where their latency hides behind the interpolation
    int r0 = 0, hoff = 0;
    if (!REF && mode == 2) { const int cv = v1 >= 0 ? v1 : v2; if (cv >= 0) { r0 = w.blo[cv]; hoff = w.boff[cv]; } }
    double p1[2], p2[2] = {0.0, 0.0};
    if (v1 >= 0) { p1[0] = xv[2 * v1]; p1[1] = xv[2 * v1 + 1]; } else { p1[0] = a.keypoints[2 * k1]; p1[1] = a.keypoints[2 * k1 + 1]; }
    if (!REF) { if (v2 >= 0) { p2[0] = xv[2 * v2]; p2[1] = xv[2 * v2 + 1]; } else { p2[0] = a.keypoints[2 * k2]; p2[1] = a.keypoints[2 * k2 + 1]; } }
    double xc1, xr1, xc2 = 0, xr2 = 0, sx1, sy1, sx2 = 0, sy2 = 0;
    const GlobalWindow w1 = make_window<T, C>(a, k1, p1, xc1, xr1, sx1, sy1);
    GlobalWindow w2 = w1;
    if (!REF) w2 = make_window<T, C>(a, k2, p2, xc2, xr2, sx2, sy2);
    double f1[CPL], r1[CPL], c1[CPL], f2[CPL], r2[CPL], c2[CPL];
#pragma unroll
    for (int k = 0; k < CPL; ++k) { f1[k] = r1[k] = c1[k] = f2[k] = r2[k] = c2[k] = 0.0; }
    double s;
    double red[14];
    if (mode == 0) {
      if (active) { bicubic_window<T, C, CPL, false, FS>(w1, lane, xc1, xr1, f1, r1, c1); if (!REF) bicubic_window<T, C, CPL, false, FS>(w2, lane, xc2, xr2, f2, r2, c2); }
      if (a.l2_normalize) { l2_normalize_desc<CPL, false>(active, f1, r1, c1); if (!REF) l2_normalize_desc<CPL, false>(active, f2, r2, c2); }
      if (REF && active) {
#pragma unroll
        for (int k = 0; k < CPL; ++k) f2[k] = a.ref_desc[k2 * C + lane * CPL + k];   // the fixed reference descriptor
      }
      double ss = 0.0;
      if (active) {
#pragma unroll
        for (int k = 0; k < CPL; ++k) { const double d = f1[k] - f2[k]; ss += d * d; }
      }
      s = warp_sum(ss);
    } else {
      if (active) { bicubic_window<T, C, CPL, true, FS>(w1, lane, xc1, xr1, f1, r1, c1); if (!REF) bicubic_window<T, C, CPL, true, FS>(w2, lane, xc2, xr2, f2, r2, c2); }
      if (a.l2_normalize) { l2_normalize_desc<CPL, true>(active, f1, r1, c1); if (!REF) l2_normalize_desc<CPL, true>(active, f2, r2, c2); }
      if (REF && active) {
#pragma unroll
        for (int k = 0; k < CPL; ++k) f2[k] = a.ref_desc[k2 * C + lane * CPL + k];   // r2 = c2 = 0: no derivative
      }
      double v[15];
#pragma unroll
      for (int k = 0; k < 15; ++k) v[k] = 0.0;
      if (active) {
#pragma unroll
        for (int k = 0; k < CPL; ++k) {
          const double d = f1[k] - f2[k];
          v[0] += d * d;
          v[1] += c1[k] * d; v[2] += r1[k] * d; v[3] += c2[k] * d; v[4] += r2[k] * d;   // G^T r (u = col, v = row)
          if (mode == 2) {
            v[5] += c1[k] * c1[k]; v[6] += c1[k] * r1[k]; v[7] += r1[k] * r1[k];
            v[8] += c2[k] * c2[k]; v[9] += c2[k] * r2[k]; v[10] += r2[k] * r2[k];
            v[11] += c1[k] * c2[k]; v[12] += c1[k] * r2[k]; v[13] += r1[k] * c2[k]; v[14] += r1[k] * r2[k];
          }
        }
      }
      s = warp_sum(v[0]);
      const int nred = mode == 2 ? 14 : 4;
#pragma unroll
      for (int k = 0; k < 14; ++k) red[k] = k < nred ? warp_sum(v[k + 1]) : 0.0;
    }
    if (lane == 0) {
      double rho[3];
      loss_eval(a.loss, a.e_w ? a.e_w[e] : 1.0, s, rho);
      cost += 0.5 * rho[0];
      if (mode >= 1) {
        // J columns: [d/dx1, d/dy1, d/dx2, d/dy2] = [sx1 G1u, sy1 G1v, -sx2 G2u, -sy2 G2v]
        const double cf[4] = {sx1, sy1, -sx2, -sy2};
        const int col[4] = {v1 >= 0 ? 2 * v1 : -1, v1 >= 0 ? 2 * v1 + 1 : -1, v2 >= 0 ? 2 * v2 : -1, v2 >= 0 ? 2 * v2 + 1 : -1};
        for (int q = 0; q < 4; ++q)
          if (col[q] >= 0) atomicAdd(&gout[col[q]], rho[1] * cf[q] * red[q]);
        if (mode == 2) {
          // dot(Ga, Gb) for the 4 columns
          const double dd[4][4] = {{red[4], red[5], red[10], red[11]}, {red[5], red[6], red[12], red[13]},
                                   {red[10], red[12], red[7], red[8]}, {red[11], red[13], red[8], red[9]}};
          if (REF) {
            if (v1 >= 0) {
              atomicAdd(&w.H[3 * v1 + 0], rho[1] * cf[0] * cf[0] * dd[0][0]);
              atomicAdd(&w.H[3 * v1 + 1], rho[1] * cf[1] * cf[0] * dd[1][0]);
              atomicAdd(&w.H[3 * v1 + 2], rho[1] * cf[1] * cf[1] * dd[1][1]);
            }
          } else {
          double* Hc = w.H + hoff;
          for (int q = 0; q < 4; ++q)
            for (int t = 0; t < 4; ++t) {
              if (col[q] < 0 || col[t] < 0 || col[q] < col[t]) continue;
              if (col[q] == col[t] && q != t) continue;
              atomicAdd(&Hc[tri(col[q] - r0, col[t] - r0)], rho[1] * cf[q] * cf[t] * dd[q][t]);
            }
          }
        }
      }
    }
  }
  if (lane == 0) w.wcost[warp] = cost;
  __syncthreads();
  double total = 0.0;
  for (int k = 0; k < kKAWarps; ++k) total += w.wcost[k];
  __syncthreads();
  return total;
}

// Block-diagonal variants: one warp per connected component [r0, r1) of the matrix, whose packed lower triangle starts
// at boff.  The components of a packed KA problem are its tracks (a handful of keypoints each), so this replaces an
// O(n^3) factorisation of the whole problem by many tiny ones that run in parallel; a component holds at most 160
// scalars.
__device__ bool ka_cholesky_blocks(double* L, int n, const int32_t* bhi, const int32_t* boff, double* ctrl_flag) {
  if (threadIdx.x == 0) *ctrl_flag = 0.0;
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int r0 = 0; r0 < n;) {
    const int r1 = bhi[r0 >> 1];
    // every warp walks the same block list; the block starting at variable v belongs to warp v % kKAWarps
    if (((r0 >> 1) % kKAWarps) == warp) {
      double* Lc = L + boff[r0 >> 1];
      const int nb = r1 - r0;
      for (int j = 0; j < nb; ++j) {
        double d = Lc[tri(j, j)];
        if (!(d > 0.0) || !isfinite(d)) { if (lane == 0) *ctrl_flag = 1.0; d = 1.0; }
        const double dj = sqrt(d);
        __syncwarp();
        if (lane == 0) Lc[tri(j, j)] = dj;
        for (int i = j + 1 + lane; i < nb; i += 32) Lc[tri(i, j)] /= dj;
        __syncwarp();
        const int m = nb - (j + 1);
        for (int e = lane; e < m * m; e += 32) {
          const int i = j + 1 + e / m, k = j + 1 + e % m;
          if (k <= i) Lc[tri(i, k)] -= Lc[tri(i, j)] * Lc[tri(k, j)];
        }
        __syncwarp();
      }
    }
    r0 = r1;
  }
  __syncthreads();
  return *ctrl_flag == 0.0;
}
__device__ void ka_chol_solve_blocks(const double* L, int n, const int32_t* bhi, const int32_t* boff, double* b) {
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int r0 = 0; r0 < n;) {
    const int r1 = bhi[r0 >> 1];
    if (((r0 >> 1) % kKAWarps) == warp) {
      const double* Lc = L + boff[r0 >> 1];
      double* bc = b + r0;
      const int nb = r1 - r0;
      for (int i = 0; i < nb; ++i) {
        double sacc = 0.0;
        for (int k = lane; k < i; k += 32) sacc += Lc[tri(i, k)] * bc[k];
        sacc = warp_sum(sacc);
        if (lane == 0) bc[i] = (bc[i] - sacc) / Lc[tri(i, i)];
        __syncwarp();
      }
      for (int i = nb - 1; i >= 0; --i) {
        double sacc = 0.0;
        for (int k = i + 1 + lane; k < nb; k += 32) sacc += Lc[tri(k, i)] * bc[k];
        sacc = warp_sum(sacc);
        if (lane == 0) bc[i] = (bc[i] - sacc) / Lc[tri(i, i)];
        __syncwarp();
      }
    }
    r0 = r1;
  }
  __syncthreads();
}

// ---- polynomial interpolation for the Armijo line search (ceres internal/ceres/polynomial.cc,
// MinimizeInterpolatingPolynomial); executed by one thread.
struct KASample { double x, value, gradient; int value_valid, gradient_valid; };
__device__ double ka_poly_eval(const double* p, int deg, double x) { double v = 0; for (int i = 0; i <= deg; ++i) v = v * x + p[i]; return v; }
__device__ bool ka_solve_dense(int n, double* A, double* b) {
  for (int k = 0; k < n; ++k) {
    int p = k; double m = fabs(A[k * n + k]);
    for (int i = k + 1; i < n; ++i) if (fabs(A[i * n + k]) > m) { m = fabs(A[i * n + k]); p = i; }
    if (m == 0.0) return false;
    if (p != k) { for (int j = 0; j < n; ++j) { const double t = A[k * n + j]; A[k * n + j] = A[p * n + j]; A[p * n + j] = t; } const double t = b[k]; b[k] = b[p]; b[p] = t; }
    for (int i = k + 1; i < n; ++i) {
      const double f = A[i * n + k] / A[k * n + k];
      for (int j = k; j < n; ++j) A[i * n + j] -= f * A[k * n + j];
      b[i] -= f * b[k];
    }
  }
  for (int i = n - 1; i >= 0; --i) {
    double s = b[i];
    for (int j = i + 1; j < n; ++j) s -= A[i * n + j] * b[j];
    b[i] = s / A[i * n + i];
  }
  return true;
}
__device__ double ka_min_interp_poly(const KASample* smp, int ns, double xmin, double xmax) {
  int n = 0;
  for (int i = 0; i < ns; ++i) { n += smp[i].value_valid; n += smp[i].gradient_valid; }
  double A[36], b[6];
  for (int i = 0; i < n * n; ++i) A[i] = 0.0;
  const int deg = n - 1;
  int row = 0;
  for (int i = 0; i < ns; ++i) {
    if (smp[i].value_valid) { for (int j = 0; j <= deg; ++j) A[row * n + j] = pow(smp[i].x, (double)(deg - j)); b[row++] = smp[i].value; }
    if (smp[i].gradient_valid) { for (int j = 0; j < deg; ++j) A[row * n + j] = (deg - j) * pow(smp[i].x, (double)(deg - j - 1)); b[row++] = smp[i].gradient; }
  }
  double best_x = (xmin + xmax) / 2.0;
  if (!ka_solve_dense(n, A, b)) return best_x;
  double best = 1.7976931348623157e308;
  { const double v = ka_poly_eval(b, deg, xmin); if (v < best) { best = v; best_x = xmin; } }
  { const double v = ka_poly_eval(b, deg, xmax); if (v < best) { best = v; best_x = xmax; } }
  double d[6];
  for (int j = 0; j < deg; ++j) d[j] = (deg - j) * b[j];
  const int kGrid = 512;
  double xp = xmin, fp = ka_poly_eval(d, deg - 1, xmin);
  for (int i = 1; i <= kGrid; ++i) {
    const double x = xmin + (xmax - xmin) * i / kGrid, f = ka_poly_eval(d, deg - 1, x);
    double root = 0; bool have = false;
    if (fp == 0.0) { root = xp; have = true; }
    else if ((fp < 0) != (f < 0) && f != 0.0) {
      double lo = xp, hi = x, fa = fp;
      for (int it = 0; it < 200; ++it) {
        const double m = 0.5 * (lo + hi), fm = ka_poly_eval(d, deg - 1, m);
        if ((fa < 0) != (fm < 0)) hi = m; else { lo = m; fa = fm; }
      }
      root = 0.5 * (lo + hi); have = true;
    }
    if (have) { const double v = ka_poly_eval(b, deg, root); if (v < best) { best = v; best_x = root; } }
    xp = x; fp = f;
  }
  if (fp == 0.0) { const double v = ka_poly_eval(b, deg, xp); if (v < best) { best = v; best_x = xp; } }
  return best_x;
}

enum { C_STOP = 0, C_RADIUS, C_DECF, C_XCOST, C_CURCOST, C_XNORM, C_GMAX, C_MCC, C_CAND, C_TMP, C_TMP2, C_FLAG, C_N };
constexpr size_t kKACtrlBytes = (kKAWarps + C_N) * sizeof(double);   // wcost + ctrl: on chip in every launch

// GWS: the launch over the problems whose workspace is in global memory (ws_off[p] >= 0; query mode: all of them); the
// other launch takes the rest, with its workspace in shared memory.  Two instances keep the on-chip one's accesses in
// the shared state space.
template <typename T, int C, bool FS, bool REF, bool GWS = REF>
__global__ void __launch_bounds__(kKAThreads) ka_solve_kernel(KAArgs a) {
  extern __shared__ __align__(16) double sm[];
  const int p = blockIdx.x;
  if (p >= a.n_problems) return;
  const int64_t wo = a.ws_off ? a.ws_off[p] : -1;
  if (GWS != (wo >= 0)) return;
  const int64_t eb = a.prob_edge_begin[p], ee = a.prob_edge_begin[p + 1];
  const int vb = a.prob_var_begin[p];
  const int nv = a.prob_var_begin[p + 1] - vb;
  const int n = 2 * nv;
  auto hdiag = [&](int i) {
    if (REF) return 3 * (i >> 1) + ((i & 1) ? 2 : 0);
    const int v = vb + (i >> 1), l = i - a.var_blk_lo[v];
    return a.var_blk_off[v] + tri(l, l);
  };
  KAWork w;
  w.m = 3 * nv;                    // REF: (h00, h10, h11) per keypoint; dense: the components' triangles back to back
  if (!REF && nv > 0) {
    const int v = vb + nv - 1, nb = a.var_blk_hi[v] - a.var_blk_lo[v];
    w.m = a.var_blk_off[v] + nb * (nb + 1) / 2;
  }
  w.blo = a.var_blk_lo + vb; w.boff = a.var_blk_off + vb;
  w.wcost = sm; w.ctrl = sm + kKAWarps;
  {
    double* q = GWS ? a.workspace + wo : sm + kKAWarps + C_N;
    w.H = q; q += w.m; w.L = q; q += w.m;
    w.g = q; q += n; w.gq = q; q += n; w.x = q; q += n; w.cand = q; q += n; w.delta = q; q += n;
    w.scale = q; q += n; w.D2 = q; q += n; w.lo = q; q += n; w.hi = q; q += n; w.tmp = q; q += n;
  }
  const int tid = threadIdx.x;
  double* out = a.prob_out + (int64_t)p * 6;
  if (n == 0) {
    const double c = ka_evaluate<T, C, FS, REF>(a, w, eb, ee, 0, w.x, 0, w.g);
    if (tid == 0) { out[0] = c; out[1] = c; out[2] = 0; out[3] = 0; out[4] = 0; out[5] = 0; }
    return;
  }
  const bool constrained = a.constrained != 0;
  for (int i = tid; i < n; i += kKAThreads) {
    const int64_t kp = a.var_kp[vb + i / 2];
    w.lo[i] = constrained ? a.var_lower[2 * (int64_t)(vb + i / 2) + (i & 1)] : -1.7976931348623157e308;
    w.hi[i] = constrained ? a.var_upper[2 * (int64_t)(vb + i / 2) + (i & 1)] : 1.7976931348623157e308;
    double v = a.keypoints[2 * kp + (i & 1)];
    if (constrained) v = fmin(fmax(v, w.lo[i]), w.hi[i]);  // IterationZero: x = Plus(x, 0)
    w.x[i] = v;
  }
  double x_cost = ka_evaluate<T, C, FS, REF>(a, w, eb, ee, n, w.x, 2, w.g);
  auto reduce_max_proj_grad = [&]() {  // ||x - Plus(x, -g)||_inf, result in ctrl[C_TMP]
    __syncthreads();
    double m = 0.0;
    for (int i = tid; i < n; i += kKAThreads) m = fmax(m, fabs(w.x[i] - fmin(fmax(w.x[i] - w.g[i], w.lo[i]), w.hi[i])));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((tid & 31) == 0) w.wcost[tid >> 5] = m;
    __syncthreads();
    if (tid == 0) { double t = 0; for (int k = 0; k < kKAWarps; ++k) t = fmax(t, w.wcost[k]); w.ctrl[C_TMP] = t; }
    __syncthreads();
  };
  auto block_sum = [&](double v) -> double {  // deterministic sum over the CTA
    __syncthreads();
    v = warp_sum(v);
    if ((tid & 31) == 0) w.wcost[tid >> 5] = v;
    __syncthreads();
    double t = 0; for (int k = 0; k < kKAWarps; ++k) t += w.wcost[k];
    __syncthreads();
    return t;
  };
  for (int i = tid; i < n; i += kKAThreads) w.scale[i] = a.jacobi_scaling ? jacobi_scale(w.H[hdiag(i)]) : 1.0;
  { double v = 0; for (int i = tid; i < n; i += kKAThreads) v += w.x[i] * w.x[i]; const double t = block_sum(v); if (tid == 0) w.ctrl[C_XNORM] = sqrt(t); }
  reduce_max_proj_grad();
  if (tid == 0) {
    w.ctrl[C_RADIUS] = a.radius0; w.ctrl[C_DECF] = 2.0; w.ctrl[C_XCOST] = x_cost; w.ctrl[C_CURCOST] = x_cost;
    w.ctrl[C_GMAX] = w.ctrl[C_TMP]; w.ctrl[C_STOP] = isfinite(x_cost) ? 0.0 : 1.0;
    out[0] = x_cost;
  }
  __syncthreads();
  int iter = 0, invalid = 0, n_succ = 0, n_unsucc = 0, term = 1;
  // the trust-region rules of pxr_lm.cuh: thread 0 keeps radius and decrease factor in the C_RADIUS / C_DECF slots (a
  // per-thread copy costs registers); every input of the decisions is a block-wide reduction, so each thread takes them,
  // counts invalid steps and holds a step evaluator itself
  const TrustRegionOptions o = {a.max_invalid, a.max_nonmonotonic, a.radius0, a.max_radius, a.min_radius, a.gtol, a.ptol,
                                a.ftol, a.min_rel_dec};
  StepEvaluator ev;
  ev.init(x_cost, a.max_nonmonotonic);
  double minimum_cost = x_cost;     // ceres keeps the lowest-cost iterate in the user's parameter blocks
  while (true) {
    // FinalizeIterationAndCheckIfMinimizerCanContinue
    if (w.ctrl[C_STOP] != 0.0) { term = 2; break; }
    if (const int stop = tr_stop(o, w.ctrl[C_RADIUS], iter, a.max_iter, w.ctrl[C_GMAX])) {
      term = stop == TR_MAX_ITERATIONS ? 1 : 0;
      break;
    }
    ++iter;
    const double radius = w.ctrl[C_RADIUS];
    // ---- LM step: (H + D) delta = -g
    for (int i = tid; i < n; i += kKAThreads) {
      w.D2[i] = lm_damping(w.H[hdiag(i)], w.scale[i], radius, a.min_diag, a.max_diag);
      w.delta[i] = -w.g[i];
    }
    __syncthreads();
    bool valid;
    double mcc = 0.0;
    if (REF) {
      // block-diagonal system: one 2x2 Cholesky + solve per keypoint
      if (tid == 0) w.ctrl[C_FLAG] = 0.0;
      __syncthreads();
      double part = 0.0;
      for (int v = tid; v < nv; v += kKAThreads) {
        const double h00 = w.H[3 * v], h10 = w.H[3 * v + 1], h11 = w.H[3 * v + 2];
        const double a00 = h00 + w.D2[2 * v], a11 = h11 + w.D2[2 * v + 1];
        bool ok = a00 > 0.0 && isfinite(a00);
        const double l00 = sqrt(ok ? a00 : 1.0), l10 = h10 / l00;
        const double s11 = a11 - l10 * l10;
        ok = ok && s11 > 0.0 && isfinite(s11);
        const double l11 = sqrt(ok ? s11 : 1.0);
        if (!ok) w.ctrl[C_FLAG] = 1.0;
        const double y0 = w.delta[2 * v] / l00, y1 = (w.delta[2 * v + 1] - l10 * y0) / l11;
        const double d1 = y1 / l11, d0 = (y0 - l10 * d1) / l00;
        w.delta[2 * v] = d0; w.delta[2 * v + 1] = d1;
        const double hd0 = h00 * d0 + h10 * d1, hd1 = h10 * d0 + h11 * d1;
        part += w.g[2 * v] * d0 + 0.5 * d0 * hd0 + w.g[2 * v + 1] * d1 + 0.5 * d1 * hd1;
        if (!isfinite(d0) || !isfinite(d1)) part = nan("");
      }
      mcc = -block_sum(part);
      valid = w.ctrl[C_FLAG] == 0.0 && isfinite(mcc) && mcc > 0.0;
    } else {
    const int32_t* blo = a.var_blk_lo + vb;
    const int32_t* bhi = a.var_blk_hi + vb;
    const int32_t* boff = a.var_blk_off + vb;
    for (int i = tid; i < w.m; i += kKAThreads) w.L[i] = w.H[i];
    __syncthreads();
    for (int i = tid; i < n; i += kKAThreads) w.L[hdiag(i)] += w.D2[i];
    __syncthreads();
    valid = ka_cholesky_blocks(w.L, n, bhi, boff, &w.ctrl[C_FLAG]);
    if (valid) {
      ka_chol_solve_blocks(w.L, n, bhi, boff, w.delta);
      // model cost change = -g.d - d^T H d / 2 (H is block diagonal over the components)
      double part = 0.0;
      for (int i = tid; i < n; i += kKAThreads) {
        double hd = 0.0;
        const int r0 = blo[i >> 1];
        const double* Hc = w.H + boff[i >> 1];
        for (int j = r0; j < bhi[i >> 1]; ++j) hd += (i >= j ? Hc[tri(i - r0, j - r0)] : Hc[tri(j - r0, i - r0)]) * w.delta[j];
        part += w.g[i] * w.delta[i] + 0.5 * w.delta[i] * hd;
        if (!isfinite(w.delta[i])) part = nan("");
      }
      mcc = -block_sum(part);
      valid = isfinite(mcc) && mcc > 0.0;
    }
    }
    if (!valid) {
      if (tr_invalid_stop(o, invalid)) { term = 2; break; }
      __syncthreads();
      if (tid == 0) tr_reject(w.ctrl[C_RADIUS], w.ctrl[C_DECF]);
      __syncthreads();
      continue;
    }
    invalid = 0;
    double candidate_cost;
    if (constrained) {
      // ---- TrustRegionMinimizer::DoLineSearch / ArmijoLineSearch (CUBIC interpolation)
      double ig = 0.0, dmx = 0.0;
      { double v = 0; for (int i = tid; i < n; i += kKAThreads) v += w.g[i] * w.delta[i]; ig = block_sum(v); }
      { double m = 0; for (int i = tid; i < n; i += kKAThreads) m = fmax(m, fabs(w.delta[i]));
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
        __syncthreads(); if ((tid & 31) == 0) w.wcost[tid >> 5] = m; __syncthreads();
        for (int k = 0; k < kKAWarps; ++k) dmx = fmax(dmx, w.wcost[k]); __syncthreads(); }
      KASample initial = {0.0, x_cost, ig, 1, 1}, previous = {0, 0, 0, 0, 0}, current = {0, 0, 0, 0, 0};
      auto ls_eval = [&](double alpha, KASample& s) {
        for (int i = tid; i < n; i += kKAThreads) w.cand[i] = fmin(fmax(w.x[i] + alpha * w.delta[i], w.lo[i]), w.hi[i]);
        const double c = ka_evaluate<T, C, FS, REF>(a, w, eb, ee, n, w.cand, 1, w.gq);
        double v = 0; for (int i = tid; i < n; i += kKAThreads) v += w.gq[i] * w.delta[i];
        const double gd = block_sum(v);
        s.x = alpha; s.value = c; s.value_valid = isfinite(c) ? 1 : 0; s.gradient = gd; s.gradient_valid = (s.value_valid && isfinite(gd)) ? 1 : 0;
      };
      ls_eval(1.0, current);
      const KASample first = current;
      int ls_iters = 0; bool success = true;
      while (!current.value_valid || current.value > x_cost + 1e-4 * ig * current.x) {
        ++ls_iters;
        if (ls_iters >= 20) { success = false; break; }
        __syncthreads();
        if (tid == 0) {
          double step;
          if (!current.value_valid) step = 0.5 * (1e-3 * current.x + 0.6 * current.x);
          else {
            KASample smp[3]; int ns = 0;
            smp[ns++] = initial; smp[ns++] = current; if (previous.value_valid) smp[ns++] = previous;
            step = ka_min_interp_poly(smp, ns, 1e-3 * current.x, 0.6 * current.x);
          }
          w.ctrl[C_TMP2] = step;
        }
        __syncthreads();
        const double step = w.ctrl[C_TMP2];
        if (step * dmx < 1e-9) { success = false; break; }
        previous = current;
        ls_eval(step, current);
      }
      if (success) {
        __syncthreads();
        for (int i = tid; i < n; i += kKAThreads) w.delta[i] *= current.x;
        __syncthreads();
        for (int i = tid; i < n; i += kKAThreads) w.cand[i] = fmin(fmax(w.x[i] + w.delta[i], w.lo[i]), w.hi[i]);
        candidate_cost = current.value;   // Plus(x, delta) is the accepted line-search point
      } else {
        __syncthreads();
        for (int i = tid; i < n; i += kKAThreads) w.cand[i] = fmin(fmax(w.x[i] + w.delta[i], w.lo[i]), w.hi[i]);
        candidate_cost = first.value_valid ? first.value : 1.7976931348623157e308;
      }
      __syncthreads();
    } else {
      for (int i = tid; i < n; i += kKAThreads) w.cand[i] = w.x[i] + w.delta[i];
      candidate_cost = ka_evaluate<T, C, FS, REF>(a, w, eb, ee, n, w.cand, 0, w.gq);
      if (!isfinite(candidate_cost)) candidate_cost = 1.7976931348623157e308;
    }
    // ---- tolerances and step acceptance
    double sn = 0; { double v = 0; for (int i = tid; i < n; i += kKAThreads) { const double d = w.x[i] - w.cand[i]; v += d * d; } sn = sqrt(block_sum(v)); }
    if (tr_tolerance(o, sn, w.ctrl[C_XNORM], x_cost - candidate_cost, x_cost)) { term = 0; break; }   // step not applied
    const double rel = ev.quality(candidate_cost, mcc);
    if (tr_successful(o, rel)) {
      __syncthreads();
      for (int i = tid; i < n; i += kKAThreads) w.x[i] = w.cand[i];
      x_cost = ka_evaluate<T, C, FS, REF>(a, w, eb, ee, n, w.x, 2, w.g);
      { double v = 0; for (int i = tid; i < n; i += kKAThreads) v += w.x[i] * w.x[i]; const double t = block_sum(v); if (tid == 0) w.ctrl[C_XNORM] = sqrt(t); }
      reduce_max_proj_grad();
      if (tid == 0) {
        w.ctrl[C_GMAX] = w.ctrl[C_TMP];
        tr_accept(o, w.ctrl[C_RADIUS], w.ctrl[C_DECF], rel);
        w.ctrl[C_XCOST] = x_cost;
      }
      ++n_succ;
      ev.accepted(candidate_cost, mcc);
      if (a.max_nonmonotonic > 0 && x_cost < minimum_cost) {    // new best iterate: it goes to the output right away
        minimum_cost = x_cost;
        for (int i = tid; i < n; i += kKAThreads) a.keypoints[2 * a.var_kp[vb + i / 2] + (i & 1)] = w.x[i];
      }
    } else {
      __syncthreads();
      if (tid == 0) tr_reject(w.ctrl[C_RADIUS], w.ctrl[C_DECF]);
      ++n_unsucc;
    }
    __syncthreads();
  }
  __syncthreads();
  if (a.max_nonmonotonic == 0) {   // monotonic: the last accepted iterate is the best one
    for (int i = tid; i < n; i += kKAThreads) a.keypoints[2 * a.var_kp[vb + i / 2] + (i & 1)] = w.x[i];
  } else x_cost = minimum_cost;
  if (tid == 0) { out[1] = x_cost; out[2] = iter; out[3] = n_succ; out[4] = n_unsucc; out[5] = term; }
}

template <typename T, int C>
static int launch_ka(pxr_ctx* ctx, bool fs, bool ref, const KAArgs& a, size_t smem) {
  if (ref) {
    if (fs) return fail(PXR_ERR_UNSUPPORTED, "use_float_simd is not built for the query (reference-descriptor) mode");
    PXR_LAUNCH(ctx, (ka_solve_kernel<T, C, false, true>), a.n_problems, kKAThreads, smem, a);
  } else if (fs) {
    PXR_CUDA(cudaFuncSetAttribute(ka_solve_kernel<T, C, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    PXR_LAUNCH(ctx, (ka_solve_kernel<T, C, true, false>), a.n_problems, kKAThreads, smem, a);
    if (a.ws_off) PXR_LAUNCH(ctx, (ka_solve_kernel<T, C, true, false, true>), a.n_problems, kKAThreads, kKACtrlBytes, a);
  } else {
    PXR_CUDA(cudaFuncSetAttribute(ka_solve_kernel<T, C, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    PXR_LAUNCH(ctx, (ka_solve_kernel<T, C, false, false>), a.n_problems, kKAThreads, smem, a);
    if (a.ws_off) PXR_LAUNCH(ctx, (ka_solve_kernel<T, C, false, false, true>), a.n_problems, kKAThreads, kKACtrlBytes, a);
  }
  PXR_CUDA(cudaGetLastError());
  return PXR_OK;
}


// the (dtype, channels) pairs of the PXR_KA_CASE dispatch
static bool ka_supported(int dtype, int C) {
  return (dtype == PXR_F16 && (C == 128 || C == 64 || C == 32 || C == 16 || C == 8)) ||
         (dtype == PXR_F32 && (C == 128 || C == 16)) || (dtype == PXR_F64 && (C == 128 || C == 16));
}

// A buffer that only grows: the batched solve reuses its wave buffers across waves.  A wave larger than every earlier one
// on the same buffer set still reallocates, and that cudaFree / cudaMalloc waits for the wave in flight.
template <typename T>
static int grow(DevBuf<T>& b, size_t count) { return (b.p && b.n >= count) ? (int)PXR_OK : b.alloc(count); }
template <typename T>
static int put(DevBuf<T>& b, const T* host, size_t count, cudaStream_t s) {
  PXR_TRY(grow(b, count));
  if (count) PXR_CUDA(cudaMemcpyAsync(b.p, host, count * sizeof(T), cudaMemcpyHostToDevice, s));
  return PXR_OK;
}

// One pxr_ka_desc on the device: the host-side problem structure, its uploads and the kernel arguments.  pxr_ka_run
// solves one; pxr_qka_run solves one per wave of queries (a query is one problem), so both make the same decisions.
struct KASolve {
  int P = 0, n_offchip = 0;
  double h2d = 0;
  std::vector<int64_t> peb, var_kp, wso;
  std::vector<int32_t> pvb, ev1, ev2, vblo, vbhi, vboff;
  std::vector<double> vlo, vhi;
  DevBuf<int64_t> d_peb, d_k1, d_k2, d_varkp, d_kppatch, d_wsoff;
  DevBuf<int32_t> d_pvb, d_v1, d_v2, d_corner, d_vblo, d_vbhi, d_vboff;
  DevBuf<double> d_w, d_lo, d_hi, d_kp, d_scale, d_out, d_ref, d_ws;
  DevBuf<uint8_t> d_patches;
  KAArgs a;
  size_t smem = 0;
};

// Host set-up of every problem of `d` (reference: TopologicalKeypointOptimizer::SetUp + ParameterizeKeypoints) and the
// uploads, enqueued on stream s.  d->ref_desc != NULL selects query mode.
static int ka_prepare(pxr_ctx* ctx, const pxr_ka_desc* d, const pxr_interp_config& ic, const pxr_solver_options& so,
                      cudaStream_t s, KASolve& k) {
  const int P = std::max(1, d->n_problems);
  k.P = P;
  const bool refmode = d->ref_desc != nullptr;
  const int C = d->channels;
  // ---- host-side problem structure (reference: TopologicalKeypointOptimizer::SetUp + ParameterizeKeypoints)
  std::vector<int64_t>& peb = k.peb;
  peb.assign(P + 1, 0);
  for (int64_t e = 0; e < d->n_edges; ++e) {
    const int pl = d->edge_problem ? d->edge_problem[e] : 0;
    if (pl < 0 || pl >= P) return fail(PXR_ERR_INVALID_ARGUMENT, "edge_problem out of range");
    if (e && d->edge_problem && d->edge_problem[e] < d->edge_problem[e - 1]) return fail(PXR_ERR_INVALID_ARGUMENT, "edges must be sorted by problem label");
    if (d->edge_src[e] < 0 || d->edge_src[e] >= d->n_keypoints || d->edge_dst[e] < 0 ||
        d->edge_dst[e] >= (refmode ? d->n_ref_desc : d->n_keypoints))
      return fail(PXR_ERR_INVALID_ARGUMENT, "edge endpoint out of range");
    peb[pl + 1]++;
  }
  for (int p = 0; p < P; ++p) peb[p + 1] += peb[p];
  std::vector<int32_t>& pvb = k.pvb; std::vector<int32_t>& ev1 = k.ev1; std::vector<int32_t>& ev2 = k.ev2;
  std::vector<int64_t>& var_kp = k.var_kp;
  std::vector<double>& vlo = k.vlo; std::vector<double>& vhi = k.vhi;
  pvb.assign(P + 1, 0); ev1.assign(d->n_edges, 0); ev2.assign(d->n_edges, 0);
  var_kp.clear(); vlo.clear(); vhi.clear();
  const bool constrained = d->bound > 0.0 || d->patches_are_sparse;
  int max_comp = 0;                     // variable keypoints of the largest component (dense mode)
  std::vector<int64_t> owner(d->n_keypoints, -1);
  // per variable: scalar range of its connected component and the offset of the component's packed triangle in the
  // problem's matrices (dense mode); per problem: doubles per matrix
  std::vector<int32_t>& vblo = k.vblo; std::vector<int32_t>& vbhi = k.vbhi; std::vector<int32_t>& vboff = k.vboff;
  vblo.clear(); vbhi.clear(); vboff.clear();
  std::vector<int64_t> pm(P, 0);
  for (int p = 0; p < P; ++p) {
    std::unordered_map<int64_t, int> idx;
    const size_t v0 = var_kp.size();
    pvb[p] = (int32_t)v0;
    std::vector<double> lo_p, hi_p;
    for (int64_t e = peb[p]; e < peb[p + 1]; ++e) {
      const int64_t ks[2] = {d->edge_src[e], refmode ? -1 : d->edge_dst[e]};
      int v[2] = {-1, -1};
      if (ks[0] != ks[1]) {
        for (int q = 0; q < (refmode ? 1 : 2); ++q) {
          if (d->kp_const[ks[q]]) continue;
          auto it = idx.find(ks[q]);
          if (it == idx.end()) {
            if (owner[ks[q]] >= 0 && owner[ks[q]] != p) return fail(PXR_ERR_INVALID_ARGUMENT, "keypoint %lld is variable in two problems", (long long)ks[q]);
            owner[ks[q]] = p;
            v[q] = (int)idx.size(); idx.emplace(ks[q], v[q]); var_kp.push_back(ks[q]);
            const int64_t pi = d->kp_patch ? d->kp_patch[ks[q]] : ks[q];
            const double sx = d->scale[2 * pi], sy = d->scale[2 * pi + 1];
            const double* k = d->keypoints + 2 * ks[q];
            double lox = (d->corner[2 * pi] + 0.5) / sx, loy = (d->corner[2 * pi + 1] + 0.5) / sy;
            double hix = lox + d->pw / sx, hiy = loy + d->ph / sy;
            if (d->bound > 0.0) {
              hix = std::min(k[0] + d->bound / sx, hix); hiy = std::min(k[1] + d->bound / sy, hiy);
              lox = std::max(k[0] - d->bound / sx, lox); loy = std::max(k[1] - d->bound / sy, loy);
            }
            lo_p.push_back(lox); lo_p.push_back(loy); hi_p.push_back(hix); hi_p.push_back(hiy);
          } else v[q] = it->second;
        }
      }
      ev1[e] = v[0]; ev2[e] = v[1];
    }
    const int nvp = (int)idx.size();
    // connected components of the variables (union-find over edges with two variable endpoints), then a stable
    // reordering that makes every component contiguous: J^T J is block diagonal over them
    std::vector<int> parent(nvp), order(nvp), newidx(nvp);
    for (int i = 0; i < nvp; ++i) parent[i] = i;
    auto find = [&](int x) { while (parent[x] != x) { parent[x] = parent[parent[x]]; x = parent[x]; } return x; };
    if (!refmode)
      for (int64_t e = peb[p]; e < peb[p + 1]; ++e)
        if (ev1[e] >= 0 && ev2[e] >= 0) { const int ra = find(ev1[e]), rb = find(ev2[e]); if (ra != rb) parent[std::max(ra, rb)] = std::min(ra, rb); }
    for (int i = 0; i < nvp; ++i) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](int x, int y) { return find(x) < find(y); });
    for (int i = 0; i < nvp; ++i) newidx[order[i]] = i;
    std::vector<int64_t> kp_p(var_kp.begin() + v0, var_kp.end());
    for (int i = 0; i < nvp; ++i) {
      var_kp[v0 + i] = kp_p[order[i]];
      vlo.push_back(lo_p[2 * order[i]]); vlo.push_back(lo_p[2 * order[i] + 1]);
      vhi.push_back(hi_p[2 * order[i]]); vhi.push_back(hi_p[2 * order[i] + 1]);
    }
    for (int64_t e = peb[p]; e < peb[p + 1]; ++e) {
      if (ev1[e] >= 0) ev1[e] = newidx[ev1[e]];
      if (ev2[e] >= 0) ev2[e] = newidx[ev2[e]];
    }
    int64_t m = 0;
    for (int i = 0; i < nvp;) {
      int jn = i + 1;
      while (jn < nvp && find(order[jn]) == find(order[i])) ++jn;
      for (int q = i; q < jn; ++q) { vblo.push_back(2 * i); vbhi.push_back(2 * jn); vboff.push_back((int32_t)m); }
      const int64_t nb = 2 * (jn - i);
      m += nb * (nb + 1) / 2;
      max_comp = std::max(max_comp, jn - i);
      if (m > INT32_MAX) return fail(PXR_ERR_UNSUPPORTED, "a KA problem's normal equations exceed 2^31 entries");
      i = jn;
    }
    pm[p] = refmode ? 3 * (int64_t)nvp : m;
  }
  pvb[P] = (int32_t)var_kp.size();
  // one warp factors one component (ka_cholesky_blocks)
  if (!refmode && max_comp > 80)
    return fail(PXR_ERR_UNSUPPORTED, "a KA problem has a connected component of %d variable keypoints (> 80 supported per component)", max_comp);
  // placement: a problem whose workspace fits the opt-in shared memory of one block runs on chip, any other one gets
  // its workspace in global memory (query mode: every problem, its size is not bounded)
  int smem_optin = 0;
  PXR_CUDA(cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, ctx->device));
  std::vector<int64_t>& wso = k.wso;
  wso.assign(P, -1);
  int64_t ws_words = 0, smem_words = 0;
  int& n_offchip = k.n_offchip;
  n_offchip = 0;
  for (int p = 0; p < P; ++p) {
    const int64_t words = 2 * pm[p] + 10 * 2 * (int64_t)(pvb[p + 1] - pvb[p]);
    if (!refmode && (kKAWarps + C_N + words) * (int64_t)sizeof(double) <= smem_optin) smem_words = std::max(smem_words, words);
    else { wso[p] = ws_words; ws_words += words; ++n_offchip; }
  }
  // ---- upload
  double& h2d = k.h2d;
  h2d = 0;
  PXR_TRY(put(k.d_peb, peb.data(), peb.size(), s)); PXR_TRY(put(k.d_pvb, pvb.data(), pvb.size(), s));
  PXR_TRY(put(k.d_k1, d->edge_src, d->n_edges, s)); PXR_TRY(put(k.d_k2, d->edge_dst, d->n_edges, s));
  PXR_TRY(put(k.d_v1, ev1.data(), ev1.size(), s)); PXR_TRY(put(k.d_v2, ev2.data(), ev2.size(), s));
  if (d->edge_weight) PXR_TRY(put(k.d_w, d->edge_weight, d->n_edges, s));
  PXR_TRY(put(k.d_varkp, var_kp.data(), var_kp.size(), s));
  PXR_TRY(put(k.d_lo, vlo.data(), vlo.size(), s)); PXR_TRY(put(k.d_hi, vhi.data(), vhi.size(), s));
  PXR_TRY(put(k.d_vblo, vblo.data(), vblo.size(), s)); PXR_TRY(put(k.d_vbhi, vbhi.data(), vbhi.size(), s));
  PXR_TRY(put(k.d_vboff, vboff.data(), vboff.size(), s));
  PXR_TRY(put(k.d_kp, d->keypoints, (size_t)d->n_keypoints * 2, s));
  if (d->kp_patch) PXR_TRY(put(k.d_kppatch, d->kp_patch, d->n_keypoints, s));
  const int64_t n_patches = d->kp_patch ? d->n_patches : std::max(d->n_patches, d->n_keypoints);
  PXR_TRY(put(k.d_corner, d->corner, (size_t)n_patches * 2, s)); PXR_TRY(put(k.d_scale, d->scale, (size_t)n_patches * 2, s));
  PXR_TRY(grow(k.d_out, (size_t)P * 6));
  const size_t esz = d->patch_dtype == PXR_F16 ? 2 : (d->patch_dtype == PXR_F32 ? 4 : 8);
  const size_t pbytes = (size_t)n_patches * d->ph * d->pw * C * esz;
  const uint8_t* dp = nullptr;
  if (d->n_patch_blocks > 0) {
    if (!d->patch_block_ptrs || !d->patch_block_counts) return fail(PXR_ERR_INVALID_ARGUMENT, "patch block arrays are NULL");
    int64_t tot = 0;
    for (int b = 0; b < d->n_patch_blocks; ++b) tot += d->patch_block_counts[b];
    if (tot < n_patches) return fail(PXR_ERR_INVALID_ARGUMENT, "patch blocks hold %lld patches, %lld needed", (long long)tot, (long long)n_patches);
    const size_t per = (size_t)d->ph * d->pw * C * esz;
    PXR_TRY(grow(k.d_patches, (size_t)tot * per));
    std::vector<size_t> seg_bytes((size_t)d->n_patch_blocks);
    for (int b = 0; b < d->n_patch_blocks; ++b) seg_bytes[b] = (size_t)d->patch_block_counts[b] * per;
    PXR_TRY(upload_segments(ctx, k.d_patches.p, d->patch_block_ptrs, seg_bytes.data(), d->n_patch_blocks, &h2d, s));
    dp = k.d_patches.p;
  } else if (d->patches_on_device) dp = (const uint8_t*)d->patches;
  else { PXR_TRY(grow(k.d_patches, pbytes)); PXR_TRY(upload_bytes(ctx, k.d_patches.p, d->patches, pbytes, nullptr, s)); dp = k.d_patches.p; h2d += pbytes; }
  h2d += d->n_edges * 40.0 + d->n_keypoints * 24.0;
  KAArgs& a = k.a;
  a.n_problems = P; a.prob_edge_begin = k.d_peb.p; a.prob_var_begin = k.d_pvb.p;
  a.e_k1 = k.d_k1.p; a.e_k2 = k.d_k2.p; a.e_v1 = k.d_v1.p; a.e_v2 = k.d_v2.p; a.e_w = d->edge_weight ? k.d_w.p : nullptr;
  a.var_kp = k.d_varkp.p; a.var_lower = k.d_lo.p; a.var_upper = k.d_hi.p;
  a.var_blk_lo = k.d_vblo.p; a.var_blk_hi = k.d_vbhi.p; a.var_blk_off = k.d_vboff.p;
  a.keypoints = k.d_kp.p; a.kp_patch = d->kp_patch ? k.d_kppatch.p : nullptr;
  a.patches = dp; a.ph = d->ph; a.pw = d->pw; a.corner = k.d_corner.p; a.scale = k.d_scale.p; a.ups = d->upsampling_factor;
  a.loss.type = so.loss_type; a.loss.a = so.loss_scale; a.l2_normalize = ic.l2_normalize; a.constrained = constrained ? 1 : 0;
  a.max_iter = so.max_num_iterations; a.max_invalid = so.max_num_consecutive_invalid_steps;
  a.ftol = so.function_tolerance; a.gtol = so.gradient_tolerance; a.ptol = so.parameter_tolerance;
  a.min_rel_dec = so.min_relative_decrease; a.radius0 = so.initial_trust_region_radius; a.max_radius = so.max_trust_region_radius;
  a.min_radius = so.min_trust_region_radius; a.min_diag = so.min_lm_diagonal; a.max_diag = so.max_lm_diagonal;
  a.jacobi_scaling = so.jacobi_scaling; a.prob_out = k.d_out.p;
  a.max_nonmonotonic = so.use_nonmonotonic_steps ? std::max(0, so.max_consecutive_nonmonotonic_steps) : 0;
  a.ref_desc = nullptr; a.workspace = nullptr; a.ws_off = nullptr;
  if (refmode) {
    PXR_TRY(put(k.d_ref, d->ref_desc, (size_t)d->n_ref_desc * C, s));
    a.ref_desc = k.d_ref.p;
    h2d += (double)d->n_ref_desc * C * 8;
  }
  if (n_offchip > 0) {
    PXR_TRY(put(k.d_wsoff, wso.data(), wso.size(), s));
    PXR_TRY(grow(k.d_ws, (size_t)std::max<int64_t>(ws_words, 1)));
    a.workspace = k.d_ws.p; a.ws_off = k.d_wsoff.p;
  }
  k.smem = (size_t)(kKAWarps + C_N + smem_words) * sizeof(double);
  return PXR_OK;
}

// ka_solve_kernel over the prepared problems, on ctx->stream
static int ka_launch(pxr_ctx* ctx, const pxr_ka_desc* d, bool fs, KASolve& k) {
  const int C = d->channels;
  const bool refmode = d->ref_desc != nullptr;
  int rc = PXR_ERR_UNSUPPORTED;
#define PXR_KA_CASE(T, CC) if (C == CC) rc = launch_ka<T, CC>(ctx, fs, refmode, k.a, k.smem);
  if (d->patch_dtype == PXR_F16) { PXR_KA_CASE(__half, 128) PXR_KA_CASE(__half, 64) PXR_KA_CASE(__half, 32) PXR_KA_CASE(__half, 16) PXR_KA_CASE(__half, 8) }
  else if (d->patch_dtype == PXR_F32) { PXR_KA_CASE(float, 128) PXR_KA_CASE(float, 16) }
  else { PXR_KA_CASE(double, 128) PXR_KA_CASE(double, 16) }
#undef PXR_KA_CASE
  return rc;
}

}  // namespace pxr

using namespace pxr;

extern "C" int pxr_ka_run(pxr_ctx* ctx, const pxr_ka_desc* d, const pxr_interp_config* interp_in,
                          const pxr_solver_options* opt_in, pxr_summary* summary) {
  const auto t0 = std::chrono::steady_clock::now();
  if (!ctx || !d) return fail(PXR_ERR_INVALID_ARGUMENT, "NULL argument");
  if (d->n_keypoints < 0 || d->n_edges < 0 || !d->keypoints || !d->kp_const || (d->n_edges && (!d->edge_src || !d->edge_dst)) ||
      (!d->patches && d->n_patch_blocks <= 0) || !d->corner || !d->scale || d->n_problems < 0)
    return fail(PXR_ERR_INVALID_ARGUMENT, "a required array is NULL");
  pxr_interp_config ic; if (interp_in) ic = *interp_in; else pxr_default_interp_config(&ic);
  pxr_solver_options so; if (opt_in) so = *opt_in; else pxr_default_ka_options(&so);
  const bool refmode = d->ref_desc != nullptr;
  if (refmode && d->n_ref_desc <= 0) return fail(PXR_ERR_INVALID_ARGUMENT, "ref_desc without n_ref_desc");
  const int C = d->channels;
  if (!ka_supported(d->patch_dtype, C)) return fail(PXR_ERR_UNSUPPORTED, "Unsupported dimensions (CHANNELS=%d, dtype=%d, N_NODES=1).", C, d->patch_dtype);
  PXR_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  const int64_t launches0 = ctx->launches;
  KASolve k;
  PXR_TRY(ka_prepare(ctx, d, ic, so, s, k));
  const int P = k.P;
  const bool fs = ic.use_float_simd != 0;
  cudaEvent_t tev0 = nullptr, tev1 = nullptr;
  cudaEventCreate(&tev0); cudaEventCreate(&tev1);
  cudaEventRecord(tev0, s);
  const int rc = ka_launch(ctx, d, fs, k);
  cudaEventRecord(tev1, s);
  if (rc != PXR_OK) { cudaEventDestroy(tev0); cudaEventDestroy(tev1); return rc; }
  std::vector<double> out((size_t)P * 6);
  PXR_CUDA(cudaMemcpyAsync(out.data(), k.d_out.p, out.size() * 8, cudaMemcpyDeviceToHost, s));
  PXR_CUDA(cudaMemcpyAsync(d->keypoints, k.d_kp.p, (size_t)d->n_keypoints * 16, cudaMemcpyDeviceToHost, s));
  PXR_CUDA(cudaStreamSynchronize(s));
  if (summary) {
    double ic0 = 0, fc = 0; int ns = 0, nu = 0, iters = 0;
    for (int p = 0; p < P; ++p) { ic0 += out[p * 6]; fc += out[p * 6 + 1]; iters = std::max(iters, (int)out[p * 6 + 2]); ns += (int)out[p * 6 + 3]; nu += (int)out[p * 6 + 4]; }
    summary->initial_cost = ic0; summary->final_cost = fc;
    summary->num_residual_blocks = (int32_t)d->n_edges; summary->num_residuals = d->n_edges * d->channels;
    summary->num_successful_steps = ns; summary->num_unsuccessful_steps = nu; summary->num_inner_iteration_steps = 0;
    summary->termination_type = 0; summary->num_iterations = 0;
    summary->h2d_bytes = k.h2d; summary->d2h_bytes = d->n_keypoints * 16.0 + P * 48.0;
    summary->kernel_launches = ctx->launches - launches0;
    summary->solve_time_s = summary->total_time_s = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    float kms = 0.f;
    cudaEventElapsedTime(&kms, tev0, tev1);
    std::snprintf(summary->message, sizeof(summary->message),
                  "%d problems, max %d LM iterations, solve kernel %.3f ms, %d with an off-chip workspace", P, iters, kms,
                  k.n_offchip);
  }
  cudaEventDestroy(tev0); cudaEventDestroy(tev1);
  return PXR_OK;
}

// ---- batched query keypoint adjustment: one query = one problem of the query mode, solved wave by wave
namespace pxr {

static int check_qka(const pxr_qka_desc* d, const pxr_interp_config* ic) {
  if (!d) return fail(PXR_ERR_INVALID_ARGUMENT, "desc is NULL");
  if (d->n_queries < 0) return fail(PXR_ERR_INVALID_ARGUMENT, "n_queries < 0");
  if (d->n_queries > 0 && (!d->kp_begin || !d->patch_blocks || !d->patch_counts || !d->patches_are_sparse))
    return fail(PXR_ERR_INVALID_ARGUMENT, "a required array is NULL");
  if (ic && ic->check_bounds) return fail(PXR_ERR_UNSUPPORTED, "check_bounds=true is not supported on this path");
  if (ic && ic->use_float_simd) return fail(PXR_ERR_UNSUPPORTED, "use_float_simd is not built for the query (reference-descriptor) mode");
  if (!ka_supported(d->patch_dtype, d->channels))
    return fail(PXR_ERR_UNSUPPORTED, "Unsupported dimensions (CHANNELS=%d, dtype=%d, N_NODES=1).", d->channels, d->patch_dtype);
  if (d->ph < 1 || d->pw < 1) return fail(PXR_ERR_INVALID_ARGUMENT, "bad patch size");
  if (!(d->upsampling_factor > 0.0)) return fail(PXR_ERR_INVALID_ARGUMENT, "upsampling_factor must be > 0");
  if (d->n_queries == 0) return PXR_OK;
  if (d->kp_begin[0] != 0) return fail(PXR_ERR_INVALID_ARGUMENT, "kp_begin[0] must be 0");
  int64_t n_patches = 0;
  for (int q = 0; q < d->n_queries; ++q) {
    if (d->kp_begin[q + 1] < d->kp_begin[q]) return fail(PXR_ERR_INVALID_ARGUMENT, "kp_begin must be non-decreasing");
    if (d->patch_counts[q] < 0) return fail(PXR_ERR_INVALID_ARGUMENT, "patch_counts[%d] < 0", q);
    if (d->patch_counts[q] > 0 && !d->patch_blocks[q]) return fail(PXR_ERR_INVALID_ARGUMENT, "patch block %d is NULL", q);
    n_patches += d->patch_counts[q];
  }
  const int64_t n_kp = d->kp_begin[d->n_queries];
  if (n_kp > 0 && (!d->keypoints || !d->kp_patch || !d->desc_begin)) return fail(PXR_ERR_INVALID_ARGUMENT, "a required array is NULL");
  if (n_patches > 0 && (!d->corner || !d->scale)) return fail(PXR_ERR_INVALID_ARGUMENT, "a required array is NULL");
  if (n_kp == 0) return PXR_OK;
  if (d->desc_begin[0] != 0) return fail(PXR_ERR_INVALID_ARGUMENT, "desc_begin[0] must be 0");
  for (int64_t k = 0; k < n_kp; ++k)
    if (d->desc_begin[k + 1] < d->desc_begin[k]) return fail(PXR_ERR_INVALID_ARGUMENT, "desc_begin must be non-decreasing");
  if (d->desc_begin[n_kp] > 0 && !d->descs) return fail(PXR_ERR_INVALID_ARGUMENT, "a required array is NULL");
  for (int q = 0; q < d->n_queries; ++q)
    for (int64_t k = d->kp_begin[q]; k < d->kp_begin[q + 1]; ++k)
      if (d->kp_patch[k] < 0 || d->kp_patch[k] >= d->patch_counts[q])
        return fail(PXR_ERR_INVALID_ARGUMENT, "kp_patch[%lld] is not a patch of query %d", (long long)k, q);
  return PXR_OK;
}

static bool qka_constrained(const pxr_qka_desc* d, int q) { return d->bound > 0.0 || d->patches_are_sparse[q]; }
static int64_t qka_blocks(const pxr_qka_desc* d, int q) {
  return d->desc_begin[d->kp_begin[q + 1]] - d->desc_begin[d->kp_begin[q]];
}

// device bytes of query q in a wave: its patches (host or device: both are copied into the wave's slab), corners and
// scales, per keypoint the keypoint, patch index, variable state and off-chip workspace (26 doubles), per residual
// block its descriptor and edge, and the problem's offsets and outputs
static double qka_query_bytes(const pxr_qka_desc* d, int q) {
  const double patch = (double)d->ph * d->pw * d->channels * dtype_bytes(d->patch_dtype);
  const double nk = (double)(d->kp_begin[q + 1] - d->kp_begin[q]);
  return d->patch_counts[q] * (patch + 24.0) + nk * (16.0 + 8.0 + 8.0 + 32.0 + 12.0 + 26.0 * 8.0 + 1.0) +
         (double)qka_blocks(d, q) * (d->channels * 8.0 + 24.0) + (8.0 + 4.0 + 48.0 + 8.0);
}

static void qka_plan(const pxr_qka_desc* d, double budget, WavePlan* p) {
  plan_waves(d->n_queries, d->patch_blocks, d->patch_counts, 12.0 /* closing problem offsets */, budget,
             [d](int q, bool) { return qka_query_bytes(d, q); }, p,
             [d](int q) { return qka_constrained(d, q) != qka_constrained(d, q - 1); });
}

// the pxr_ka_desc of one wave: its queries as the problems of one query-mode call (host arrays kept alive here)
struct QKAWave {
  int q0 = 0, nq = 0;
  int64_t k0 = 0, nk = 0, p0 = 0;
  std::vector<int64_t> es, ed, kp_patch;
  std::vector<int32_t> ep;
  std::vector<uint8_t> kp_const;
  std::vector<const void*> blocks;
  pxr_ka_desc desc;
};

static void qka_wave(const pxr_qka_desc* d, const WavePlan& plan, int w, QKAWave& v) {
  static const double kNoDesc = 0.0;
  static const uint8_t kNoPatch = 0;
  v.q0 = plan.begin[w]; v.nq = plan.begin[w + 1] - v.q0;
  v.k0 = d->kp_begin[v.q0]; v.nk = d->kp_begin[v.q0 + v.nq] - v.k0;
  v.p0 = 0; for (int q = 0; q < v.q0; ++q) v.p0 += d->patch_counts[q];
  const int64_t db0 = v.nk ? d->desc_begin[v.k0] : 0;
  v.es.clear(); v.ed.clear(); v.ep.clear(); v.kp_patch.assign((size_t)v.nk, 0); v.kp_const.assign((size_t)std::max<int64_t>(v.nk, 1), 0);
  v.blocks.assign((size_t)v.nq, &kNoPatch);
  int64_t poff = 0;
  for (int i = 0; i < v.nq; ++i) {
    const int q = v.q0 + i;
    if (d->patch_counts[q] > 0) v.blocks[i] = d->patch_blocks[q];
    for (int64_t k = d->kp_begin[q]; k < d->kp_begin[q + 1]; ++k) {
      v.kp_patch[k - v.k0] = poff + d->kp_patch[k];
      for (int64_t j = d->desc_begin[k]; j < d->desc_begin[k + 1]; ++j) { v.es.push_back(k - v.k0); v.ed.push_back(j - db0); v.ep.push_back(i); }
    }
    poff += d->patch_counts[q];
  }
  pxr_ka_desc& a = v.desc;
  std::memset(&a, 0, sizeof(a));
  a.n_keypoints = v.nk; a.keypoints = d->keypoints ? d->keypoints + 2 * v.k0 : nullptr; a.kp_const = v.kp_const.data();
  a.kp_patch = v.kp_patch.data();
  a.n_edges = (int64_t)v.es.size(); a.edge_src = v.es.data(); a.edge_dst = v.ed.data(); a.edge_weight = nullptr;
  a.edge_problem = v.ep.data(); a.n_problems = v.nq;
  a.n_patches = poff; a.patches = nullptr; a.patches_on_device = 0;
  a.patch_dtype = d->patch_dtype; a.ph = d->ph; a.pw = d->pw; a.channels = d->channels;
  a.corner = d->corner ? d->corner + 2 * v.p0 : nullptr; a.scale = d->scale ? d->scale + 2 * v.p0 : nullptr;
  a.upsampling_factor = d->upsampling_factor; a.bound = d->bound; a.patches_are_sparse = d->patches_are_sparse[v.q0];
  a.n_patch_blocks = v.nq; a.patch_block_ptrs = v.blocks.data(); a.patch_block_counts = d->patch_counts + v.q0;
  a.ref_desc = (d->descs && v.nk) ? d->descs + db0 * d->channels : &kNoDesc;
  a.n_ref_desc = v.nk ? d->desc_begin[v.k0 + v.nk] - db0 : 0;
}

}  // namespace pxr

extern "C" int pxr_qka_run(pxr_ctx* ctx, const pxr_qka_desc* d, const pxr_interp_config* interp_in,
                           const pxr_solver_options* opt_in, pxr_qka_result* results, int32_t* n_waves_out,
                           pxr_summary* total) {
  const auto t0 = std::chrono::steady_clock::now();
  PXR_TRY(check_qka(d, interp_in));
  PXR_TRY(require_ctx(ctx));
  if (!results && d->n_queries > 0) return fail(PXR_ERR_INVALID_ARGUMENT, "results is NULL");
  pxr_interp_config ic; if (interp_in) ic = *interp_in; else pxr_default_interp_config(&ic);
  pxr_solver_options so; if (opt_in) so = *opt_in; else pxr_default_ka_options(&so);
  PXR_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  cudaStream_t us = nullptr;
  PXR_TRY(upload_stream(ctx, &us));
  const int64_t launches0 = ctx->launches;
  double budget = 0.0;
  PXR_TRY(wave_budget(d->max_wave_bytes, &budget));
  WavePlan plan;
  qka_plan(d, budget, &plan);
  const int nw = (int)plan.bytes.size();
  double max_bytes = 0.0; int64_t max_out = 1;
  for (int w = 0; w < nw; ++w) {
    max_bytes = std::max(max_bytes, plan.bytes[w]);
    const int nq = plan.begin[w + 1] - plan.begin[w];
    const int64_t nk = d->kp_begin[plan.begin[w + 1]] - d->kp_begin[plan.begin[w]];
    max_out = std::max<int64_t>(max_out, (int64_t)nq * 6 + nk * 2);
  }
  int nsets = 1;
  PXR_TRY(wave_sets(nw, (size_t)max_bytes, &nsets));
  KASolve ks[2];
  QKAWave wv[2];
  // per buffer set, the pinned host copy of a wave's outputs: per-problem results | keypoints
  struct Pinned { void* p = nullptr; ~Pinned() { if (p) cudaFreeHost(p); } } hout[2];
  for (int k = 0; k < nsets; ++k) PXR_CUDA(cudaMallocHost(&hout[k].p, (size_t)max_out * 8));
  cudaEvent_t kt0 = nullptr, kt1 = nullptr;
  struct Events { cudaEvent_t* a; cudaEvent_t* b; ~Events() { if (*a) cudaEventDestroy(*a); if (*b) cudaEventDestroy(*b); } } guard{&kt0, &kt1};
  PXR_CUDA(cudaEventCreate(&kt0));
  PXR_CUDA(cudaEventCreate(&kt1));
  double h2d = 0.0, kernel_ms = 0.0, ic0 = 0.0, fc = 0.0;
  int ns = 0, nu = 0;
  WaveSteps steps;
  steps.upload = [&](int w, int set) {
    qka_wave(d, plan, w, wv[set]);
    PXR_TRY(ka_prepare(ctx, &wv[set].desc, ic, so, us, ks[set]));
    h2d += ks[set].h2d;
    return (int)PXR_OK;
  };
  steps.launch = [&](int, int set) {
    const QKAWave& v = wv[set];
    PXR_CUDA(cudaEventRecord(kt0, s));
    PXR_TRY(ka_launch(ctx, &v.desc, false, ks[set]));
    PXR_CUDA(cudaEventRecord(kt1, s));
    double* ho = static_cast<double*>(hout[set].p);
    PXR_CUDA(cudaMemcpyAsync(ho, ks[set].d_out.p, (size_t)v.nq * 6 * 8, cudaMemcpyDeviceToHost, s));
    if (v.nk) PXR_CUDA(cudaMemcpyAsync(ho + (size_t)v.nq * 6, ks[set].d_kp.p, (size_t)v.nk * 16, cudaMemcpyDeviceToHost, s));
    return (int)PXR_OK;
  };
  steps.finish = [&](int w, int set) {
    // the wave's bounds from the plan: with one buffer set wv[set] already describes the next wave
    const int q0 = plan.begin[w], nq = plan.begin[w + 1] - q0;
    const int64_t k0 = d->kp_begin[q0];
    const double* ho = static_cast<const double*>(hout[set].p);
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, kt0, kt1) == cudaSuccess) kernel_ms += ms;
    for (int i = 0; i < nq; ++i) {
      const int q = q0 + i;
      const double* o = ho + (size_t)i * 6;
      pxr_qka_result& r = results[q];
      r.num_residual_blocks = (int32_t)qka_blocks(d, q);
      r.initial_cost = o[0]; r.final_cost = o[1]; r.num_iterations = (int32_t)o[2];
      r.num_successful_steps = (int32_t)o[3]; r.num_unsuccessful_steps = (int32_t)o[4]; r.termination_type = (int32_t)o[5];
      r.status = std::isfinite(o[0]) ? PXR_OK : PXR_ERR_NUMERIC;
      if (r.num_residual_blocks == 0) continue;   // keypoints untouched
      // written back whatever the status: pxr_ka_run writes what the kernel leaves for such a query too
      const int64_t kb = d->kp_begin[q], ke = d->kp_begin[q + 1];
      std::memcpy(d->keypoints + 2 * kb, ho + (size_t)nq * 6 + 2 * (kb - k0), (size_t)(ke - kb) * 16);
      if (r.status != PXR_OK) continue;
      ic0 += r.initial_cost; fc += r.final_cost; ns += r.num_successful_steps; nu += r.num_unsuccessful_steps;
    }
    return (int)PXR_OK;
  };
  int done = 0;
  const int rc = run_waves(ctx, nw, nsets, us, steps, &done);
  if (n_waves_out) *n_waves_out = done;
  if (rc != PXR_OK) return rc;
  if (total) {
    const int cap = total->iterations_capacity;
    pxr_iteration_summary* keep = total->iterations;
    std::memset(total, 0, sizeof(*total));
    total->iterations_capacity = cap; total->iterations = keep;
    total->initial_cost = ic0; total->final_cost = fc;
    int64_t nb = 0; for (int q = 0; q < d->n_queries; ++q) nb += qka_blocks(d, q);
    total->num_residual_blocks = (int32_t)nb;
    total->num_residuals = nb * d->channels;
    total->num_successful_steps = ns; total->num_unsuccessful_steps = nu;
    total->h2d_bytes = h2d;
    total->kernel_launches = ctx->launches - launches0;
    total->total_time_s = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    total->solve_time_s = kernel_ms * 1e-3;
    std::snprintf(total->message, sizeof(total->message), "%d queries in %d waves, solve kernels %.3f ms", d->n_queries, nw,
                  kernel_ms);
  }
  return PXR_OK;
}
