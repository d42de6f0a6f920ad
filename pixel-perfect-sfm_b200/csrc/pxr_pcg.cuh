// pxr_pcg.cuh — ITERATIVE_SCHUR: preconditioned conjugate gradients on the explicit reduced camera system
// with the SCHUR_JACOBI preconditioner (block diagonal of S), the reference's choice above 1000 images
// (pixsfm/bundle_adjustment/src/bundle_optimizer.h:188-190).  Restates ceres' ConjugateGradientsSolver
// (internal/ceres/conjugate_gradients_solver.cc @2.1): Q-based termination zeta = k (Q1 - Q0) / Q1 < eta,
// residual refresh every 10 iterations, x0 = 0.  All scalar logic lives in a device-side state so that the
// host only polls a flag every few iterations.
#pragma once
#include "pxr_device.cuh"

namespace pxr {

struct CGState {
  double rho, last_rho, alpha, beta, Q0, pq, rz, xbr;   // pq / rz / xbr double as atomic accumulators of the multi-CTA path
  int it, done, failed, max_iter;
  double q_tol;
};

// full symmetric copy of the lower-stored S
static __global__ void cg_mirror_kernel(double* S, int n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)n * n) return;
  const int r = (int)(i / n), c = (int)(i % n);
  if (c > r) S[i] = S[(int64_t)c * n + r];
}

// inverse of every diagonal block (dim <= 12), one thread per block; Minv row-wise [n][12].  A non-positive pivot sets
// *fail and leaves the block's rows unwritten: the CG init kernels then end the solve before its first iteration.
static __global__ void cg_block_inverse_kernel(const double* S, int n, const int32_t* blk_off, const int32_t* blk_dim, int nblk,
                                               double* Minv, int* fail) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= nblk) return;
  const int o = blk_off[b], d = blk_dim[b];
  double A[12][24];
  for (int i = 0; i < d; ++i) { for (int j = 0; j < d; ++j) { A[i][j] = S[(int64_t)(o + i) * n + o + j]; A[i][d + j] = i == j ? 1.0 : 0.0; } }
  for (int k = 0; k < d; ++k) {
    const double pv = A[k][k];
    if (!(pv > 0.0)) { *fail = 1; return; }
    for (int j = 0; j < 2 * d; ++j) A[k][j] /= pv;
    for (int i = 0; i < d; ++i) {
      if (i == k) continue;
      const double f = A[i][k];
      for (int j = 0; j < 2 * d; ++j) A[i][j] -= f * A[k][j];
    }
  }
  for (int i = 0; i < d; ++i)
    for (int j = 0; j < d; ++j) Minv[(int64_t)(o + i) * 12 + j] = A[i][d + j];
}

// out = S v (S full, row-major), one warp per row
static __global__ void __launch_bounds__(256) cg_gemv_kernel(const double* __restrict__ S, const double* __restrict__ v, double* out, int n,
                                                             const CGState* st) {
  if (st && st->done) return;
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= n) return;
  const double* r = S + (int64_t)row * n;
  double s = 0.0;
  for (int j = lane; j < n; j += 32) s += r[j] * v[j];
  s = warp_sum(s);
  if (lane == 0) out[row] = s;
}

// single-CTA vector kernels (n is the reduced system size, at most a few 10^4)
__device__ __forceinline__ double cta_sum(double v) {
  __shared__ double sh[32];
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0.0;
  for (int k = 0; k < (int)(blockDim.x >> 5); ++k) t += sh[k];
  return t;
}

// init: x = 0, r = b, state.  A failed preconditioner (*precond_fail, set by the block inverse) ends the solve here with
// 0 iterations, as ceres' ConjugateGradientsSolver stops when the preconditioner update fails.
static __global__ void __launch_bounds__(1024) cg_init_kernel(const double* b, double* x, double* r, int n, CGState* st, int max_iter, double q_tol,
                                                              const int* precond_fail) {
  double nb = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) { x[i] = 0.0; r[i] = b[i]; nb += b[i] * b[i]; }
  nb = cta_sum(nb);
  if (threadIdx.x == 0) {
    const int failed = *precond_fail != 0;
    st->rho = 1.0; st->last_rho = 1.0; st->alpha = 0; st->beta = 0; st->Q0 = 0.0; st->it = 0; st->failed = failed;
    st->done = (failed || nb == 0.0) ? 1 : 0; st->max_iter = max_iter; st->q_tol = q_tol;
  }
}

// z = M^-1 r ; rho = r.z ; p = z (+ beta p)
static __global__ void __launch_bounds__(1024) cg_precond_kernel(const double* Minv, const int32_t* row_off, const int32_t* row_dim, const double* r,
                                                                 double* z, double* p, int n, CGState* st) {
  if (st->done) return;
  double rz = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    double s = 0.0;
    const int o = row_off[i], d = row_dim[i];
    for (int j = 0; j < d; ++j) s += Minv[(int64_t)i * 12 + j] * r[o + j];
    z[i] = s; rz += r[i] * s;
  }
  rz = cta_sum(rz);
  __shared__ double beta_s; __shared__ int stop;
  if (threadIdx.x == 0) {
    st->it += 1;
    st->last_rho = st->rho; st->rho = rz;
    stop = 0;
    if (rz == 0.0 || !isfinite(rz)) { st->failed = 1; st->done = 1; stop = 1; }
    double beta = 0.0;
    if (st->it > 1) { beta = rz / st->last_rho; if (beta == 0.0 || !isfinite(beta)) { st->failed = 1; st->done = 1; stop = 1; } }
    st->beta = beta; beta_s = beta;
  }
  __syncthreads();
  if (stop) return;
  const double beta = beta_s;
  const bool first = st->it == 1;
  for (int i = threadIdx.x; i < n; i += blockDim.x) p[i] = first ? z[i] : z[i] + beta * p[i];
}

// alpha = rho / p.q ; x += alpha p ; r -= alpha q (or flagged for refresh) ; Q test
static __global__ void __launch_bounds__(1024) cg_update_kernel(const double* b, const double* p, const double* q, double* x, double* r, int n, CGState* st) {
  if (st->done) return;
  double pq = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) pq += p[i] * q[i];
  pq = cta_sum(pq);
  __shared__ double alpha_s; __shared__ int stop;
  if (threadIdx.x == 0) {
    stop = 0;
    if (pq <= 0.0 || !isfinite(pq)) { st->done = 1; stop = 1; }          // matrix not positive definite along p: keep x
    const double alpha = st->rho / pq;
    if (!stop && !isfinite(alpha)) { st->failed = 1; st->done = 1; stop = 1; }
    st->alpha = alpha; alpha_s = alpha;
  }
  __syncthreads();
  if (stop) return;
  const double alpha = alpha_s;
  const bool refresh = (st->it % 10) == 0;   // residual_reset_period: r = b - S x is recomputed by the caller's next launches
  for (int i = threadIdx.x; i < n; i += blockDim.x) { x[i] += alpha * p[i]; if (!refresh) r[i] -= alpha * q[i]; }
}

// after an optional residual refresh: Q1 = -0.5 x.(b + r), zeta test, iteration cap
static __global__ void __launch_bounds__(1024) cg_check_kernel(const double* b, const double* x, const double* r, int n, CGState* st) {
  if (st->done) return;
  double xbr = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) xbr += x[i] * (b[i] + r[i]);
  xbr = cta_sum(xbr);
  if (threadIdx.x == 0) {
    const double Q1 = -0.5 * xbr;
    const double zeta = st->it * (Q1 - st->Q0) / Q1;
    if (zeta < st->q_tol) st->done = 1;
    st->Q0 = Q1;
    if (st->it >= st->max_iter) st->done = 1;
  }
}

// r = b - tmp (only on refresh iterations)
static __global__ void __launch_bounds__(1024) cg_refresh_kernel(const double* b, const double* Sx, double* r, int n, const CGState* st) {
  if (st->done || (st->it % 10) != 0) return;
  for (int i = threadIdx.x; i < n; i += blockDim.x) r[i] = b[i] - Sx[i];
}

// ---------------------------------------------------------------------------------------------------------------
// Multi-CTA variants for large reduced systems (n >= 4096: the single-CTA kernels above then
// dominate a CG iteration).  Vector work is spread over the grid; every dot product is a two-stage FIXED-ORDER
// reduction (one partial per CTA, summed by one warp of the scalar kernel that needs it), so the solve is a
// deterministic function of (S, b): ranks that run it redundantly on the same all-reduced system stay bit-identical.
// Same arithmetic and termination rule as the single-CTA kernels.  `part` holds 3 * gridDim.x doubles (rz | pq | xbr).
__device__ __forceinline__ double det_sum_warp(const double* part, int n) {   // one full warp, fixed order
  double v = 0.0;
  for (int i = threadIdx.x & 31; i < n; i += 32) v += part[i];
  return warp_sum(v);
}
static __global__ void __launch_bounds__(256) cgm_init_kernel(const double* b, double* x, double* r, int n, CGState* st, double* part) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double nb = 0.0;
  if (i < n) { x[i] = 0.0; r[i] = b[i]; nb = b[i] * b[i]; }
  nb = cta_sum(nb);
  if (threadIdx.x == 0) part[2 * gridDim.x + blockIdx.x] = nb;
}
static __global__ void cgm_init_state_kernel(CGState* st, int max_iter, double q_tol, const int* precond_fail) {   // before cgm_init_kernel
  const int failed = *precond_fail != 0;         // failed preconditioner: done before the first iteration, as cg_init_kernel
  st->rho = 1.0; st->last_rho = 1.0; st->alpha = 0; st->beta = 0; st->Q0 = 0.0; st->it = 0; st->failed = failed; st->done = failed;
  st->max_iter = max_iter; st->q_tol = q_tol; st->pq = 0.0; st->rz = 0.0; st->xbr = 0.0;
}
static __global__ void __launch_bounds__(32) cgm_init_done_kernel(CGState* st, const double* part, int g) {   // b == 0
  const double nb = det_sum_warp(part + 2 * g, g);
  if (threadIdx.x == 0 && nb == 0.0) st->done = 1;
}

// z = M^-1 r ; rz partial
static __global__ void __launch_bounds__(256) cgm_precond_kernel(const double* Minv, const int32_t* row_off, const int32_t* row_dim,
                                                                 const double* r, double* z, int n, CGState* st, double* part) {
  if (st->done) return;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double rz = 0.0;
  if (i < n) {
    double sacc = 0.0;
    const int o = row_off[i], d = row_dim[i];
    for (int j = 0; j < d; ++j) sacc += Minv[(int64_t)i * 12 + j] * r[o + j];
    z[i] = sacc; rz = r[i] * sacc;
  }
  rz = cta_sum(rz);
  if (threadIdx.x == 0) part[blockIdx.x] = rz;
}
static __global__ void __launch_bounds__(32) cgm_beta_kernel(CGState* st, const double* part, int g) {
  if (st->done) return;
  const double rz = det_sum_warp(part, g);
  if (threadIdx.x != 0) return;
  st->it += 1;
  st->last_rho = st->rho; st->rho = rz;
  if (rz == 0.0 || !isfinite(rz)) { st->failed = 1; st->done = 1; return; }
  double beta = 0.0;
  if (st->it > 1) { beta = rz / st->last_rho; if (beta == 0.0 || !isfinite(beta)) { st->failed = 1; st->done = 1; } }
  st->beta = beta;
}
// p = z (+ beta p)
static __global__ void __launch_bounds__(256) cgm_dir_kernel(const double* z, double* p, int n, const CGState* st) {
  if (st->done) return;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = st->it == 1 ? z[i] : z[i] + st->beta * p[i];
}
// pq partial
static __global__ void __launch_bounds__(256) cgm_pq_kernel(const double* p, const double* q, int n, CGState* st, double* part) {
  if (st->done) return;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double v = i < n ? p[i] * q[i] : 0.0;
  v = cta_sum(v);
  if (threadIdx.x == 0) part[gridDim.x + blockIdx.x] = v;
}
static __global__ void __launch_bounds__(32) cgm_alpha_kernel(CGState* st, const double* part, int g) {
  if (st->done) return;
  const double pq = det_sum_warp(part + g, g);
  if (threadIdx.x != 0) return;
  if (pq <= 0.0 || !isfinite(pq)) { st->done = 1; st->alpha = 0.0; return; }   // not positive definite along p: keep x
  const double alpha = st->rho / pq;
  if (!isfinite(alpha)) { st->failed = 1; st->done = 1; st->alpha = 0.0; return; }
  st->alpha = alpha;
}
// x += alpha p ; r -= alpha q (unless this is a refresh iteration) ; xbr partial = x.(b + r) when no refresh follows
static __global__ void __launch_bounds__(256) cgm_update_kernel(const double* b, const double* p, const double* q, double* x, double* r,
                                                                int n, CGState* st, double* part) {
  if (st->done) return;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool refresh = (st->it % 10) == 0;
  const double alpha = st->alpha;
  double v = 0.0;
  if (i < n) {
    const double xi = x[i] + alpha * p[i];
    x[i] = xi;
    if (!refresh) { const double ri = r[i] - alpha * q[i]; r[i] = ri; v = xi * (b[i] + ri); }
  }
  if (!refresh) { v = cta_sum(v); if (threadIdx.x == 0) part[2 * gridDim.x + blockIdx.x] = v; }
}
// refresh iterations: r = b - S x ; xbr partial
static __global__ void __launch_bounds__(256) cgm_refresh_kernel(const double* b, const double* Sx, const double* x, double* r, int n, CGState* st,
                                                                 double* part) {
  if (st->done || (st->it % 10) != 0) return;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double v = 0.0;
  if (i < n) { const double ri = b[i] - Sx[i]; r[i] = ri; v = x[i] * (b[i] + ri); }
  v = cta_sum(v);
  if (threadIdx.x == 0) part[2 * gridDim.x + blockIdx.x] = v;
}
static __global__ void __launch_bounds__(32) cgm_check_kernel(CGState* st, const double* part, int g) {
  if (st->done) return;
  const double xbr = det_sum_warp(part + 2 * g, g);
  if (threadIdx.x != 0) return;
  const double Q1 = -0.5 * xbr;
  const double zeta = st->it * (Q1 - st->Q0) / Q1;
  if (zeta < st->q_tol) st->done = 1;
  st->Q0 = Q1;
  if (st->it >= st->max_iter) st->done = 1;
}

}  // namespace pxr
