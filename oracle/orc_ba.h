// oracle/orc_ba.h — TEST INFRASTRUCTURE ONLY.
//
// CPU restatement of the reference's featuremetric bundle adjustment:
//   residual blocks  : FeatureReferenceCostFunctor / ...ConstantPose...
//                      (pixsfm/residuals/src/feature_reference.h:71-207) evaluated with
//                      forward-mode Jets exactly as ceres::AutoDiffCostFunction does
//   parameterisation : BundleOptimizer::Parameterize{Points,Images,Cameras}
//                      (pixsfm/bundle_adjustment/src/bundle_optimizer.h:335-442), already
//                      resolved to masks in pxr_ba_desc
//   solve            : ceres::Solve with DENSE_SCHUR/SPARSE_SCHUR (exact Schur complement)
//                      (bundle_optimizer.h:172-245) -> orc_trust_region.h
//   inner iterations : ceres CoordinateDescentMinimizer over the 3D points
//                      (bundle_optimizer.h:131-134,350-355)
// The full C x p Jacobian of every block is formed (no rank-2 shortcut), so the CUDA
// path's 2x2 reduction is validated against un-shortcut arithmetic.
#pragma once
#include <omp.h>

#include <cstdio>
#include <cstdlib>
#include <memory>
#include <vector>

#include "../include/pxr.h"
#include "orc_core.h"
#include "orc_trust_region.h"

namespace orc {

inline int Popcount(uint32_t v) { return __builtin_popcount(v); }

// (ceres) QuaternionManifold::Plus / PlusJacobian, include/ceres/manifold.h @2.1
inline void QuaternionPlus(const double* x, const double* d, double* out) {
  const double sq = d[0] * d[0] + d[1] * d[1] + d[2] * d[2];
  if (sq == 0.0) { for (int i = 0; i < 4; ++i) out[i] = x[i]; return; }
  const double nd = std::sqrt(sq);
  const double s = std::sin(nd) / nd;
  const double z[4] = {std::cos(nd), s * d[0], s * d[1], s * d[2]};
  out[0] = z[0] * x[0] - z[1] * x[1] - z[2] * x[2] - z[3] * x[3];
  out[1] = z[0] * x[1] + z[1] * x[0] + z[2] * x[3] - z[3] * x[2];
  out[2] = z[0] * x[2] - z[1] * x[3] + z[2] * x[0] + z[3] * x[1];
  out[3] = z[0] * x[3] + z[1] * x[2] - z[2] * x[1] + z[3] * x[0];
}
inline void QuaternionPlusJacobian(const double* x, double* J /*4x3 row-major*/) {
  J[0] = -x[1]; J[1] = -x[2]; J[2] = -x[3];
  J[3] = x[0];  J[4] = x[3];  J[5] = -x[2];
  J[6] = -x[3]; J[7] = x[0];  J[8] = x[1];
  J[9] = x[2];  J[10] = -x[1]; J[11] = x[0];
}

inline bool CholeskySolveInPlace(int n, std::vector<double>& A, std::vector<double>& b) {
  // A row-major symmetric (lower used); overwritten by L.  Blocked right-looking factorization:
  // three parallel regions per 64-wide panel (what a threaded LAPACK dpotrf does).
  const int NB = 64;
  bool ok = true;
  for (int k0 = 0; k0 < n && ok; k0 += NB) {
    const int kb = std::min(NB, n - k0);
    // diagonal block (serial)
    for (int j = k0; j < k0 + kb; ++j) {
      double d = A[(size_t)j * n + j];
      for (int k = k0; k < j; ++k) d -= A[(size_t)j * n + k] * A[(size_t)j * n + k];
      if (!(d > 0.0) || !std::isfinite(d)) { ok = false; break; }
      d = std::sqrt(d);
      A[(size_t)j * n + j] = d;
      for (int i = j + 1; i < k0 + kb; ++i) {
        double s = A[(size_t)i * n + j];
        for (int k = k0; k < j; ++k) s -= A[(size_t)i * n + k] * A[(size_t)j * n + k];
        A[(size_t)i * n + j] = s / d;
      }
    }
    if (!ok) break;
    const int r0 = k0 + kb;
    // panel: rows below, X L_kk^T = A_ik
#pragma omp parallel for schedule(static) if (n - r0 > 128)
    for (int i = r0; i < n; ++i) {
      double* ai = &A[(size_t)i * n];
      for (int j = k0; j < k0 + kb; ++j) {
        double s = ai[j];
        const double* aj = &A[(size_t)j * n];
        for (int k = k0; k < j; ++k) s -= ai[k] * aj[k];
        ai[j] = s / aj[j];
      }
    }
    // trailing update: A_ij -= L_ik L_jk^T, i >= j >= r0
#pragma omp parallel for schedule(dynamic, 8) if (n - r0 > 128)
    for (int i = r0; i < n; ++i) {
      double* ai = &A[(size_t)i * n];
      for (int j = r0; j <= i; ++j) {
        const double* aj = &A[(size_t)j * n];
        double s = 0;
        for (int k = k0; k < k0 + kb; ++k) s += ai[k] * aj[k];
        ai[j] -= s;
      }
    }
  }
  if (!ok) return false;
  for (int i = 0; i < n; ++i) {
    double s = b[i];
    for (int k = 0; k < i; ++k) s -= A[(size_t)i * n + k] * b[k];
    b[i] = s / A[(size_t)i * n + i];
  }
  for (int i = n - 1; i >= 0; --i) {
    double s = b[i];
    for (int k = i + 1; k < n; ++k) s -= A[(size_t)k * n + i] * b[k];
    b[i] = s / A[(size_t)i * n + i];
  }
  return true;
}

inline bool Invert3x3Sym(const double* H, double* inv) {
  // Cholesky-based inverse of a 3x3 SPD matrix (ceres InvertPSDMatrix, llt path)
  const double a = H[0], b = H[1], c = H[2], d = H[4], e = H[5], f = H[8];
  if (!(a > 0)) return false;
  const double l00 = std::sqrt(a), l10 = b / l00, l20 = c / l00;
  const double t11 = d - l10 * l10; if (!(t11 > 0)) return false;
  const double l11 = std::sqrt(t11), l21 = (e - l20 * l10) / l11;
  const double t22 = f - l20 * l20 - l21 * l21; if (!(t22 > 0)) return false;
  const double l22 = std::sqrt(t22);
  // inv(L)
  const double i00 = 1.0 / l00, i11 = 1.0 / l11, i22 = 1.0 / l22;
  const double i10 = -l10 * i00 * i11;
  const double i21 = -l21 * i11 * i22;
  const double i20 = -(l20 * i00 + l21 * i10) * i22;
  // inv = inv(L)^T inv(L)
  inv[0] = i00 * i00 + i10 * i10 + i20 * i20;
  inv[1] = inv[3] = i10 * i11 + i20 * i21;
  inv[2] = inv[6] = i20 * i22;
  inv[4] = i11 * i11 + i21 * i21;
  inv[5] = inv[7] = i21 * i22;
  inv[8] = i22 * i22;
  return true;
}

struct BALayout {
  int n_cam_local = 0;  // reduced camera system size
  int n_local = 0;
  int n_ambient = 0;
  std::vector<int> pose_off, pose_dim, intr_off, intr_dim;
  std::vector<int64_t> point_off;     // local offset or -1
  std::vector<int64_t> pt_begin;      // CSR over obs, size n_points+1
  int64_t off_cam = 0, off_q = 0, off_t = 0, off_xyz = 0;
};

inline BALayout MakeLayout(const pxr_ba_desc& d) {
  BALayout L;
  L.pose_off.assign(d.n_images, -1); L.pose_dim.assign(d.n_images, 0);
  L.intr_off.assign(d.n_cameras, -1); L.intr_dim.assign(d.n_cameras, 0);
  int off = 0;
  for (int i = 0; i < d.n_images; ++i) {
    if (d.pose_const[i]) continue;
    L.pose_off[i] = off;
    L.pose_dim[i] = 3 + (3 - Popcount(d.tvec_const_mask[i] & 7u));
    off += L.pose_dim[i];
  }
  for (int c = 0; c < d.n_cameras; ++c) {
    const int k = CameraNumParams(d.cam_model[c]);
    const uint32_t full = (1u << k) - 1u;
    const uint32_t m = d.cam_const_mask[c] & full;
    if (m == full) continue;
    L.intr_off[c] = off;
    L.intr_dim[c] = k - Popcount(m);
    off += L.intr_dim[c];
  }
  L.n_cam_local = off;
  L.point_off.assign(d.n_points, -1);
  int64_t po = off;
  for (int64_t p = 0; p < d.n_points; ++p) if (!d.point_const[p]) { L.point_off[p] = po; po += 3; }
  L.n_local = (int)po;
  L.off_cam = 0;
  L.off_q = (int64_t)d.n_cameras * PXR_MAX_CAM_PARAMS;
  L.off_t = L.off_q + (int64_t)d.n_images * 4;
  L.off_xyz = L.off_t + (int64_t)d.n_images * 3;
  L.n_ambient = (int)(L.off_xyz + d.n_points * 3);
  L.pt_begin.assign(d.n_points + 1, 0);
  for (int64_t o = 0; o < d.n_obs; ++o) L.pt_begin[d.obs_pt[o] + 1]++;
  for (int64_t p = 0; p < d.n_points; ++p) L.pt_begin[p + 1] += L.pt_begin[p];
  return L;
}

inline Patch MakePatch(const pxr_ba_desc& d, int64_t o) {
  const int64_t pi = d.obs_patch ? d.obs_patch[o] : o;
  Patch p;
  const size_t esz = d.patch_dtype == PXR_F16 ? 2 : (d.patch_dtype == PXR_F32 ? 4 : 8);
  if (d.n_patch_blocks > 0) {
    int64_t local = pi;
    int b = 0;
    while (b < d.n_patch_blocks - 1 && local >= d.patch_block_counts[b]) { local -= d.patch_block_counts[b]; ++b; }
    p.data = (const char*)d.patch_block_ptrs[b] + (size_t)local * d.ph * d.pw * d.channels * esz;
  } else {
    p.data = (const char*)d.patches + (size_t)pi * d.ph * d.pw * d.channels * esz;
  }
  p.dtype = d.patch_dtype; p.h = d.ph; p.w = d.pw; p.c = d.channels;
  p.corner[0] = d.corner[2 * pi]; p.corner[1] = d.corner[2 * pi + 1];
  p.scale[0] = d.scale[2 * pi]; p.scale[1] = d.scale[2 * pi + 1];
  p.upsampling = d.upsampling_factor;
  return p;
}

// One residual block: r (C) and the ambient Jacobian columns [q(4) t(3) X(3) cam(K)]
// via Jets — FeatureReferenceCostFunctor::operator()<Jet> (feature_reference.h:98-137)
// + Interpolator::Evaluate<JetT> (interpolation.h:130-140).
// Jq/Jt may be null (constant-pose functor, feature_reference.h:157-207).
template <int K, bool POSE>
inline void EvalBlockJets(int model, const double* cam, const double* q, const double* t,
                          const double* X, const Patch& patch, const InterpConfig& icfg,
                          const double* ref, double* r, double* J /*C x (POSE?7:0)+3+K*/,
                          double* xy_out, std::vector<double>& scratch) {
  constexpr int N = (POSE ? 7 : 0) + 3 + K;
  typedef Jet<N> JT;
  JT jq[4], jt[3], jX[3], jc[K > 0 ? K : 1];
  int k = 0;
  if (POSE) { for (int i = 0; i < 4; ++i) jq[i] = JT(q[i], k++); for (int i = 0; i < 3; ++i) jt[i] = JT(t[i], k++); }
  else { for (int i = 0; i < 4; ++i) jq[i] = JT(q[i]); for (int i = 0; i < 3; ++i) jt[i] = JT(t[i]); }
  for (int i = 0; i < 3; ++i) jX[i] = JT(X[i], k++);
  for (int i = 0; i < K; ++i) jc[i] = JT(cam[i], k++);
  JT xy[2], uv[2];
  WorldToPixel<JT>(model, jc, jq, jt, jX, xy);
  ToPixelCoordinates<JT>(patch, xy, uv);
  const int C = patch.c;
  scratch.resize(3 * C);
  double* f = scratch.data(); double* dfdr = f + C; double* dfdc = f + 2 * C;
  PixelInterp(patch, icfg, uv[1].a, uv[0].a, f, dfdr, dfdc);
  for (int i = 0; i < C; ++i) {
    r[i] = ref ? f[i] - ref[i] : f[i];
    if (J) for (int n = 0; n < N; ++n) J[i * N + n] = dfdr[i] * uv[1].v[n] + dfdc[i] * uv[0].v[n];
  }
  if (xy_out) { xy_out[0] = xy[0].a; xy_out[1] = xy[1].a; }
}

typedef void (*EvalBlockFn)(int, const double*, const double*, const double*, const double*,
                            const Patch&, const InterpConfig&, const double*, double*, double*,
                            double*, std::vector<double>&);
template <bool POSE>
inline EvalBlockFn SelectEval(int model) {
  switch (CameraNumParams(model)) {
    case 3: return &EvalBlockJets<3, POSE>;
    case 4: return &EvalBlockJets<4, POSE>;
    case 5: return &EvalBlockJets<5, POSE>;
    case 8: return &EvalBlockJets<8, POSE>;
    case 12: return &EvalBlockJets<12, POSE>;
  }
  return nullptr;
}

struct BAEvalOptions {
  InterpConfig interp;
  Loss loss;
  bool iterative_schur = false;     // ITERATIVE_SCHUR + SCHUR_JACOBI (bundle_optimizer.h:188-190)
  int max_linear_solver_iterations = 200;
  double eta = 0.1;                 // ceres Solver::Options::eta -> CG q_tolerance
  TROptions inner;  // defaults = ceres Solver::Options defaults (CoordinateDescentMinimizer::Solve)
};

// (ceres) ConjugateGradientsSolver::Solve (internal/ceres/conjugate_gradients_solver.cc @2.1) on the explicit
// damped Schur complement S (symmetric, full storage) with the SCHUR_JACOBI preconditioner = inverse of the
// diagonal blocks of S (one block per camera-side parameter block).  x starts at 0.  stop_out (optional) tells why it
// ended: PCGStop below.
enum PCGStop { kPCGZeta = 0, kPCGNonPositiveCurvature = 1, kPCGMaxIterations = 2, kPCGFailure = 3 };
inline bool SchurJacobiPCG(int n, const std::vector<double>& S, const std::vector<double>& b,
                           const std::vector<std::pair<int, int>>& blocks, int max_iter, double q_tolerance,
                           std::vector<double>* xout, int* iters_out, int* stop_out = nullptr) {
  int stop_dummy = 0;
  int& stop = stop_out ? *stop_out : stop_dummy;
  stop = kPCGFailure;
  std::vector<double> Minv((size_t)n * 12, 0.0);  // row-wise storage of the block inverses (block dim <= 12)
  for (auto& bk : blocks) {
    const int o = bk.first, d = bk.second;
    // invert the SPD block by Gauss-Jordan on [B | I]
    std::vector<double> A((size_t)d * 2 * d, 0.0);
    for (int i = 0; i < d; ++i) { for (int j = 0; j < d; ++j) A[(size_t)i * 2 * d + j] = S[(size_t)(o + i) * n + o + j]; A[(size_t)i * 2 * d + d + i] = 1.0; }
    for (int k = 0; k < d; ++k) {
      const double pv = A[(size_t)k * 2 * d + k];
      if (!(pv > 0.0)) return false;
      for (int j = 0; j < 2 * d; ++j) A[(size_t)k * 2 * d + j] /= pv;
      for (int i = 0; i < d; ++i) {
        if (i == k) continue;
        const double f = A[(size_t)i * 2 * d + k];
        for (int j = 0; j < 2 * d; ++j) A[(size_t)i * 2 * d + j] -= f * A[(size_t)k * 2 * d + j];
      }
    }
    for (int i = 0; i < d; ++i) for (int j = 0; j < d; ++j) Minv[(size_t)(o + i) * 12 + j] = A[(size_t)i * 2 * d + d + j];
  }
  std::vector<int> blk_of(n, 0), blk_off(n, 0), blk_dim(n, 0);
  for (auto& bk : blocks) for (int i = 0; i < bk.second; ++i) { blk_off[bk.first + i] = bk.first; blk_dim[bk.first + i] = bk.second; }
  auto apply_M = [&](const std::vector<double>& r, std::vector<double>& z) {
    for (int i = 0; i < n; ++i) { double s = 0; for (int j = 0; j < blk_dim[i]; ++j) s += Minv[(size_t)i * 12 + j] * r[blk_off[i] + j]; z[i] = s; }
  };
  auto mul = [&](const std::vector<double>& v, std::vector<double>& out) {
#pragma omp parallel for schedule(static) if (n > 512)
    for (int i = 0; i < n; ++i) { double s = 0; const double* row = &S[(size_t)i * n]; for (int j = 0; j < n; ++j) s += row[j] * v[j]; out[i] = s; }
  };
  auto dot = [&](const std::vector<double>& a, const std::vector<double>& c) { double s = 0; for (int i = 0; i < n; ++i) s += a[i] * c[i]; return s; };
  std::vector<double>& x = *xout;
  x.assign(n, 0.0);
  *iters_out = 0;
  const double norm_b = std::sqrt(dot(b, b));
  if (norm_b == 0.0) { stop = kPCGZeta; return true; }
  std::vector<double> r(b), z(n), p(n), q(n), tmp(n);
  double rho = 1.0, Q0 = 0.0;  // -0.5 * x.(b + r) with x = 0
  for (int it = 1;; ++it) {
    apply_M(r, z);
    const double last_rho = rho;
    rho = dot(r, z);
    if (rho == 0.0 || !std::isfinite(rho)) return false;
    if (it == 1) p = z;
    else { const double beta = rho / last_rho; if (beta == 0.0 || !std::isfinite(beta)) return false; for (int i = 0; i < n; ++i) p[i] = z[i] + beta * p[i]; }
    mul(p, q);
    const double pq = dot(p, q);
    if (pq <= 0.0 || !std::isfinite(pq)) { *iters_out = it; stop = kPCGNonPositiveCurvature; break; }
    const double alpha = rho / pq;
    if (!std::isfinite(alpha)) return false;
    for (int i = 0; i < n; ++i) x[i] += alpha * p[i];
    if (it % 10 == 0) { mul(x, tmp); for (int i = 0; i < n; ++i) r[i] = b[i] - tmp[i]; }   // residual_reset_period
    else for (int i = 0; i < n; ++i) r[i] -= alpha * q[i];
    double xbr = 0; for (int i = 0; i < n; ++i) xbr += x[i] * (b[i] + r[i]);
    const double Q1 = -0.5 * xbr;
    const double zeta = it * (Q1 - Q0) / Q1;
    *iters_out = it;
    if (zeta < q_tolerance) { stop = kPCGZeta; break; }
    Q0 = Q1;
    if (it >= max_iter) { stop = kPCGMaxIterations; break; }
  }
  return true;
}

// wall-clock split of a solve (bench.py prints it next to the CPU number): 0 residual+Jacobian evaluation,
// 1 cost-only evaluation, 2 Schur elimination, 3 reduced solve, 4 back-substitution, 5 inner iterations
struct StageClock {
  double t[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  struct Scope {
    double* acc; double t0;
    explicit Scope(double* a) : acc(a), t0(omp_get_wtime()) {}
    ~Scope() { *acc += omp_get_wtime() - t0; }
  };
};
inline StageClock& GlobalStageClock() { static StageClock c; return c; }

class BAEvaluator : public TREvaluator {
 public:
  const pxr_ba_desc& d;
  BALayout L;
  BAEvalOptions eo;
  static constexpr int kMaxDc = 6 + PXR_MAX_CAM_PARAMS;
  // linearisation
  std::vector<double> Hcc, gc, Hpp, gp, W;
  std::vector<int> Wcols, Wdc;
  std::vector<double> obs_sq_norm;  // last evaluation: uncorrected ||r||^2 per block

  BAEvaluator(const pxr_ba_desc& desc, const BAEvalOptions& o) : d(desc), L(MakeLayout(desc)), eo(o) {
    Hcc.assign((size_t)L.n_cam_local * L.n_cam_local, 0.0);
    gc.assign(L.n_cam_local, 0.0);
    Hpp.assign((size_t)d.n_points * 9, 0.0);
    gp.assign((size_t)d.n_points * 3, 0.0);
    W.assign((size_t)d.n_obs * kMaxDc * 3, 0.0);
    Wcols.assign((size_t)d.n_obs * kMaxDc, -1);
    Wdc.assign(d.n_obs, 0);
    obs_sq_norm.assign(d.n_obs, 0.0);
  }
  void PackParameters(double* x) const {
    for (int64_t i = 0; i < (int64_t)d.n_cameras * PXR_MAX_CAM_PARAMS; ++i) x[L.off_cam + i] = d.cam_params[i];
    for (int64_t i = 0; i < (int64_t)d.n_images * 4; ++i) x[L.off_q + i] = d.qvec[i];
    for (int64_t i = 0; i < (int64_t)d.n_images * 3; ++i) x[L.off_t + i] = d.tvec[i];
    for (int64_t i = 0; i < d.n_points * 3; ++i) x[L.off_xyz + i] = d.xyz[i];
  }
  void UnpackParameters(const double* x) const {
    for (int64_t i = 0; i < (int64_t)d.n_cameras * PXR_MAX_CAM_PARAMS; ++i) d.cam_params[i] = x[L.off_cam + i];
    for (int64_t i = 0; i < (int64_t)d.n_images * 4; ++i) d.qvec[i] = x[L.off_q + i];
    for (int64_t i = 0; i < (int64_t)d.n_images * 3; ++i) d.tvec[i] = x[L.off_t + i];
    for (int64_t i = 0; i < d.n_points * 3; ++i) d.xyz[i] = x[L.off_xyz + i];
  }
  int NumParameters() const override { return L.n_ambient; }
  int NumLocal() const override { return L.n_local; }

  // Local, loss-corrected Jacobian of one block: Jc (C x dc) with column ids, Jp (C x 3), r (C)
  // Returns cost contribution 0.5*rho(s).
  double LinearizeBlock(const double* x, int64_t o, bool with_jac, std::vector<double>& r,
                        std::vector<double>& Jc, int* cols, int* dc_out, std::vector<double>& Jp,
                        std::vector<double>& Jamb, std::vector<double>& scratch, double* sq_norm_out,
                        double* xy_out = nullptr, const double* X_override = nullptr) const {
    const int img = d.obs_img[o];
    const int64_t pt = d.obs_pt[o];
    const int cam = d.img_cam[img];
    const int model = d.cam_model[cam];
    const int K = CameraNumParams(model);
    const int C = d.channels;
    const bool pose_var = L.pose_off[img] >= 0;
    const double* q = x + L.off_q + 4 * img;
    const double* t = x + L.off_t + 3 * img;
    const double* X = X_override ? X_override : x + L.off_xyz + 3 * pt;
    const double* cp = x + L.off_cam + (int64_t)PXR_MAX_CAM_PARAMS * cam;
    const Patch patch = MakePatch(d, o);
    const double* ref = d.refs ? d.refs + (size_t)pt * C : nullptr;
    const int N = (pose_var ? 7 : 0) + 3 + K;
    r.resize(C);
    Jamb.resize((size_t)C * N);
    EvalBlockFn fn = pose_var ? SelectEval<true>(model) : SelectEval<false>(model);
    fn(model, cp, q, t, X, patch, eo.interp, ref, r.data(), with_jac ? Jamb.data() : nullptr, xy_out, scratch);
    double s = 0;
    for (int i = 0; i < C; ++i) s += r[i] * r[i];
    if (sq_norm_out) *sq_norm_out = s;
    double rho[3];
    eo.loss.Evaluate(s, rho);
    if (!with_jac) return 0.5 * rho[0];
    // local parameterisation (ResidualBlock::Evaluate multiplies by the manifold's PlusJacobian)
    int dc = 0;
    const int xoff = pose_var ? 7 : 0;
    Jc.assign((size_t)C * kMaxDc, 0.0);
    if (pose_var) {
      double PJ[12];
      QuaternionPlusJacobian(q, PJ);
      for (int i = 0; i < C; ++i)
        for (int a = 0; a < 3; ++a) {
          double v = 0;
          for (int b = 0; b < 4; ++b) v += Jamb[(size_t)i * N + b] * PJ[b * 3 + a];
          Jc[(size_t)i * kMaxDc + a] = v;
        }
      for (int a = 0; a < 3; ++a) cols[dc++] = L.pose_off[img] + a;
      int la = 3;
      for (int b = 0; b < 3; ++b) {
        if (d.tvec_const_mask[img] & (1u << b)) continue;
        for (int i = 0; i < C; ++i) Jc[(size_t)i * kMaxDc + dc] = Jamb[(size_t)i * N + 4 + b];
        cols[dc++] = L.pose_off[img] + la++;
      }
    }
    if (L.intr_off[cam] >= 0) {
      int la = 0;
      for (int b = 0; b < K; ++b) {
        if (d.cam_const_mask[cam] & (1u << b)) continue;
        for (int i = 0; i < C; ++i) Jc[(size_t)i * kMaxDc + dc] = Jamb[(size_t)i * N + xoff + 3 + b];
        cols[dc++] = L.intr_off[cam] + la++;
      }
    }
    *dc_out = dc;
    Jp.resize((size_t)C * 3);
    for (int i = 0; i < C; ++i)
      for (int a = 0; a < 3; ++a) Jp[(size_t)i * 3 + a] = Jamb[(size_t)i * N + xoff + a];
    Corrector corr(s, rho);
    corr.CorrectJacobian(C, kMaxDc, r.data(), Jc.data());
    corr.CorrectJacobian(C, 3, r.data(), Jp.data());
    corr.CorrectResiduals(C, r.data());
    return 0.5 * rho[0];
  }

  // An observation's camera columns are the columns of its image (pose block, then the intrinsics block of the image's
  // camera), so J_c^T J_c lands in ONE (dc x dc) block per image: every thread accumulates its own [n_images] blocks and
  // the blocks are summed and scattered into Hcc once (what ceres' SchurEliminator does with per-thread buffers).
  bool Evaluate(const double* x, double* cost, bool with_jac) override {
    StageClock::Scope clk(&GlobalStageClock().t[with_jac ? 0 : 1]);
    const int nc = L.n_cam_local;
    const int nthreads = omp_get_max_threads();
    const int BD = kMaxDc;
    double total = 0;
    if (with_jac) {
      std::fill(Hcc.begin(), Hcc.end(), 0.0);
      std::fill(gc.begin(), gc.end(), 0.0);
      std::fill(Hpp.begin(), Hpp.end(), 0.0);
      std::fill(gp.begin(), gp.end(), 0.0);
    }
    std::vector<std::vector<double>> tH(with_jac ? nthreads : 0), tg(with_jac ? nthreads : 0);
    std::vector<int> img_dc(d.n_images, 0), img_cols((size_t)d.n_images * BD, -1);
    for (int i = 0; i < d.n_images; ++i) {       // [pose block | intrinsics block], the order LinearizeBlock emits
      int dc = 0;
      for (int a = 0; a < L.pose_dim[i]; ++a) img_cols[(size_t)i * BD + dc++] = L.pose_off[i] + a;
      const int cam = d.img_cam[i];
      for (int a = 0; a < L.intr_dim[cam]; ++a) img_cols[(size_t)i * BD + dc++] = L.intr_off[cam] + a;
      img_dc[i] = dc;
    }
#pragma omp parallel reduction(+ : total)
    {
      const int tid = omp_get_thread_num();
      std::vector<double> r, Jc, Jp, Jamb, scratch;
      int cols[kMaxDc];
      if (with_jac) { tH[tid].assign((size_t)d.n_images * BD * BD, 0.0); tg[tid].assign((size_t)d.n_images * BD, 0.0); }
#pragma omp for schedule(dynamic, 16)
      for (int64_t p = 0; p < d.n_points; ++p) {
        for (int64_t o = L.pt_begin[p]; o < L.pt_begin[p + 1]; ++o) {
          int dc = 0;
          double s;
          total += LinearizeBlock(x, o, with_jac, r, Jc, cols, &dc, Jp, Jamb, scratch, &s);
          obs_sq_norm[o] = s;
          if (!with_jac) continue;
          const int C = d.channels;
          const bool pvar = L.point_off[p] >= 0;
          const int img = d.obs_img[o];
          double* Hb = &tH[tid][(size_t)img * BD * BD];
          double* gb = &tg[tid][(size_t)img * BD];
          // rank-1 accumulation per residual row: the inner loops run over contiguous columns (vectorisable)
          for (int i = 0; i < C; ++i) {
            const double* row = &Jc[(size_t)i * kMaxDc];
            const double ri = r[i];
            for (int a = 0; a < dc; ++a) {
              const double ja = row[a];
              gb[a] += ja * ri;
              double* ha = Hb + a * BD;
              for (int b = 0; b < dc; ++b) ha[b] += ja * row[b];
            }
          }
          Wdc[o] = dc;
          for (int a = 0; a < dc; ++a) Wcols[(size_t)o * kMaxDc + a] = cols[a];
          if (pvar) {
            double hp[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, gpa[3] = {0, 0, 0};
            double* Wo = &W[(size_t)o * kMaxDc * 3];
            for (int k = 0; k < dc * 3; ++k) Wo[k] = 0.0;
            for (int i = 0; i < C; ++i) {
              const double* jp = &Jp[(size_t)i * 3];
              const double* row = &Jc[(size_t)i * kMaxDc];
              const double ri = r[i];
              for (int a = 0; a < 3; ++a) { gpa[a] += jp[a] * ri; for (int b = 0; b < 3; ++b) hp[a * 3 + b] += jp[a] * jp[b]; }
              for (int a = 0; a < dc; ++a) { const double ja = row[a]; Wo[a * 3] += ja * jp[0]; Wo[a * 3 + 1] += ja * jp[1]; Wo[a * 3 + 2] += ja * jp[2]; }
            }
            for (int a = 0; a < 3; ++a) gp[(size_t)p * 3 + a] += gpa[a];
            for (int k = 0; k < 9; ++k) Hpp[(size_t)p * 9 + k] += hp[k];
          }
        }
      }
    }
    if (with_jac) {
      // sum the threads' image blocks (parallel over images), then scatter every image's block into Hcc / gc
      std::vector<double>& H0 = tH[0];
      std::vector<double>& g0 = tg[0];
#pragma omp parallel for schedule(static)
      for (int img = 0; img < d.n_images; ++img)
        for (int t = 1; t < nthreads; ++t) {
          if (tH[t].empty()) continue;
          const double* hs = &tH[t][(size_t)img * BD * BD]; double* hd = &H0[(size_t)img * BD * BD];
          for (int k = 0; k < BD * BD; ++k) hd[k] += hs[k];
          const double* gs = &tg[t][(size_t)img * BD]; double* gd = &g0[(size_t)img * BD];
          for (int k = 0; k < BD; ++k) gd[k] += gs[k];
        }
      for (int img = 0; img < d.n_images; ++img) {
        const int dc = img_dc[img];
        const int* cl = &img_cols[(size_t)img * BD];
        for (int a = 0; a < dc; ++a) {
          gc[cl[a]] += g0[(size_t)img * BD + a];
          for (int b = 0; b < dc; ++b) Hcc[(size_t)cl[a] * nc + cl[b]] += H0[((size_t)img * BD + a) * BD + b];
        }
      }
    }
    *cost = total;
    return std::isfinite(total);
  }

  void Gradient(double* g) const override {
    for (int i = 0; i < L.n_cam_local; ++i) g[i] = gc[i];
    for (int64_t p = 0; p < d.n_points; ++p)
      if (L.point_off[p] >= 0) for (int a = 0; a < 3; ++a) g[L.point_off[p] + a] = gp[(size_t)p * 3 + a];
  }
  void SquaredColumnNorm(double* dd) const override {
    const int nc = L.n_cam_local;
    for (int i = 0; i < nc; ++i) dd[i] = Hcc[(size_t)i * nc + i];
    for (int64_t p = 0; p < d.n_points; ++p)
      if (L.point_off[p] >= 0) for (int a = 0; a < 3; ++a) dd[L.point_off[p] + a] = Hpp[(size_t)p * 9 + a * 4];
  }

  // Exact Schur complement solve (DENSE_SCHUR / SPARSE_SCHUR are both exact factorizations).
  // Also exposes S and rhs for parity tests.
  std::vector<double> S_last, rhs_last;
  bool SolveDamped(const double* D2, double* delta, int* iters) override {
    const int nc = L.n_cam_local;
    std::vector<double> S(Hcc), rhs(nc);
    for (int i = 0; i < nc; ++i) { S[(size_t)i * nc + i] += D2[i]; rhs[i] = -gc[i]; }
    std::vector<double> inv((size_t)d.n_points * 9, 0.0);
    std::vector<double> T((size_t)d.n_obs * kMaxDc * 3, 0.0);
    bool ok = true;
    {
      StageClock::Scope clk(&GlobalStageClock().t[2]);
      // (H_pp + D)^-1 and T = W (H_pp + D)^-1 per observation: independent per point
#pragma omp parallel for schedule(static) reduction(&& : ok)
      for (int64_t p = 0; p < d.n_points; ++p) {
        if (L.point_off[p] < 0) continue;
        double H[9];
        for (int k = 0; k < 9; ++k) H[k] = Hpp[(size_t)p * 9 + k];
        for (int a = 0; a < 3; ++a) H[a * 4] += D2[L.point_off[p] + a];
        double* iv = &inv[(size_t)p * 9];
        if (!Invert3x3Sym(H, iv)) { ok = false; continue; }
        for (int64_t oi = L.pt_begin[p]; oi < L.pt_begin[p + 1]; ++oi)
          for (int a = 0; a < Wdc[oi]; ++a)
            for (int b = 0; b < 3; ++b) {
              double v = 0;
              for (int k = 0; k < 3; ++k) v += W[((size_t)oi * kMaxDc + a) * 3 + k] * iv[k * 3 + b];
              T[((size_t)oi * kMaxDc + a) * 3 + b] = v;
            }
      }
      if (ok && nc > 0) {
        // S -= sum_p sum_{i,j} T_i W_j^T, rhs += sum T_i g_p.  Every thread owns a contiguous range of ROWS of S and
        // visits all observation pairs, keeping only the block rows whose column id falls in its range: no locks, no
        // atomics, and a fixed summation order per entry (ceres' SchurEliminator is threaded over point chunks with
        // per-block locks; the arithmetic per pair is the same).
#pragma omp parallel
        {
          const int nt = omp_get_num_threads(), tid = omp_get_thread_num();
          const int r0 = (int)((int64_t)nc * tid / nt), r1 = (int)((int64_t)nc * (tid + 1) / nt);
          for (int64_t p = 0; p < d.n_points; ++p) {
            if (L.point_off[p] < 0) continue;
            const double* g = &gp[(size_t)p * 3];
            for (int64_t oi = L.pt_begin[p]; oi < L.pt_begin[p + 1]; ++oi) {
              const int dci = Wdc[oi];
              const int* ci = &Wcols[(size_t)oi * kMaxDc];
              // an observation's columns are ascending: [pose block | intrinsics block]; skip it when none is mine
              bool mine = false;
              for (int a = 0; a < dci; ++a) if (ci[a] >= r0 && ci[a] < r1) { mine = true; break; }
              if (!mine) continue;
              const double* Ti = &T[(size_t)oi * kMaxDc * 3];
              for (int a = 0; a < dci; ++a) {
                const int ca = ci[a];
                if (ca < r0 || ca >= r1) continue;
                rhs[ca] += Ti[a * 3 + 0] * g[0] + Ti[a * 3 + 1] * g[1] + Ti[a * 3 + 2] * g[2];
                double* Srow = &S[(size_t)ca * nc];
                for (int64_t oj = L.pt_begin[p]; oj < L.pt_begin[p + 1]; ++oj) {
                  const int dcj = Wdc[oj];
                  const int* cj = &Wcols[(size_t)oj * kMaxDc];
                  const double* Wj = &W[(size_t)oj * kMaxDc * 3];
                  for (int b = 0; b < dcj; ++b)
                    Srow[cj[b]] -= Ti[a * 3] * Wj[b * 3] + Ti[a * 3 + 1] * Wj[b * 3 + 1] + Ti[a * 3 + 2] * Wj[b * 3 + 2];
                }
              }
            }
          }
        }
      }
    }
    if (!ok) return false;
    S_last = S; rhs_last = rhs;
    int lin_iters = 1;
    {
      StageClock::Scope clk(&GlobalStageClock().t[3]);
      if (eo.iterative_schur && nc > 0) {
        std::vector<std::pair<int, int>> blocks;
        for (int i = 0; i < d.n_images; ++i) if (L.pose_off[i] >= 0) blocks.push_back({L.pose_off[i], L.pose_dim[i]});
        for (int c = 0; c < d.n_cameras; ++c) if (L.intr_off[c] >= 0) blocks.push_back({L.intr_off[c], L.intr_dim[c]});
        std::vector<double> xs;
        if (!SchurJacobiPCG(nc, S, rhs, blocks, eo.max_linear_solver_iterations, eo.eta, &xs, &lin_iters)) return false;
        rhs = xs;
      } else if (nc > 0 && !CholeskySolveInPlace(nc, S, rhs)) return false;
    }
    StageClock::Scope clk(&GlobalStageClock().t[4]);
    for (int i = 0; i < nc; ++i) delta[i] = rhs[i];
#pragma omp parallel for schedule(static)
    for (int64_t p = 0; p < d.n_points; ++p) {
      if (L.point_off[p] < 0) continue;
      double v[3] = {-gp[(size_t)p * 3], -gp[(size_t)p * 3 + 1], -gp[(size_t)p * 3 + 2]};
      for (int64_t o = L.pt_begin[p]; o < L.pt_begin[p + 1]; ++o)
        for (int a = 0; a < Wdc[o]; ++a) {
          const double dca = delta[Wcols[(size_t)o * kMaxDc + a]];
          for (int k = 0; k < 3; ++k) v[k] -= W[((size_t)o * kMaxDc + a) * 3 + k] * dca;
        }
      const double* iv = &inv[(size_t)p * 9];
      for (int a = 0; a < 3; ++a)
        delta[L.point_off[p] + a] = iv[a * 3] * v[0] + iv[a * 3 + 1] * v[1] + iv[a * 3 + 2] * v[2];
    }
    *iters = lin_iters;
    return true;
  }

  double ModelCostChange(const double* delta) const override {
    // -(J d)^T (r + J d / 2) = -g^T d - d^T H d / 2, H = J^T J (undamped)
    StageClock::Scope clk(&GlobalStageClock().t[4]);
    const int nc = L.n_cam_local;
    double gd = 0, dHd = 0;
#pragma omp parallel for schedule(static) reduction(+ : gd, dHd)
    for (int i = 0; i < nc; ++i) {
      gd += gc[i] * delta[i];
      double row = 0;
      for (int j = 0; j < nc; ++j) row += Hcc[(size_t)i * nc + j] * delta[j];
      dHd += delta[i] * row;
    }
#pragma omp parallel for schedule(static) reduction(+ : gd, dHd)
    for (int64_t p = 0; p < d.n_points; ++p) {
      if (L.point_off[p] < 0) continue;
      const double* dp = delta + L.point_off[p];
      for (int a = 0; a < 3; ++a) {
        gd += gp[(size_t)p * 3 + a] * dp[a];
        for (int b = 0; b < 3; ++b) dHd += dp[a] * Hpp[(size_t)p * 9 + a * 3 + b] * dp[b];
      }
      for (int64_t o = L.pt_begin[p]; o < L.pt_begin[p + 1]; ++o)
        for (int a = 0; a < Wdc[o]; ++a) {
          const double dca = delta[Wcols[(size_t)o * kMaxDc + a]];
          for (int k = 0; k < 3; ++k) dHd += 2.0 * dca * W[((size_t)o * kMaxDc + a) * 3 + k] * dp[k];
        }
    }
    return -gd - 0.5 * dHd;
  }

  void Plus(const double* x, const double* delta, double* xp) const override {
    for (int i = 0; i < L.n_ambient; ++i) xp[i] = x[i];
    for (int i = 0; i < d.n_images; ++i) {
      if (L.pose_off[i] < 0) continue;
      const double* dl = delta + L.pose_off[i];
      QuaternionPlus(x + L.off_q + 4 * i, dl, xp + L.off_q + 4 * i);
      int la = 3;
      for (int b = 0; b < 3; ++b) {
        if (d.tvec_const_mask[i] & (1u << b)) continue;
        xp[L.off_t + 3 * i + b] = x[L.off_t + 3 * i + b] + dl[la++];
      }
    }
    for (int c = 0; c < d.n_cameras; ++c) {
      if (L.intr_off[c] < 0) continue;
      const int K = CameraNumParams(d.cam_model[c]);
      int la = 0;
      for (int b = 0; b < K; ++b) {
        if (d.cam_const_mask[c] & (1u << b)) continue;
        xp[L.off_cam + (int64_t)PXR_MAX_CAM_PARAMS * c + b] += delta[L.intr_off[c] + la++];
      }
    }
    for (int64_t p = 0; p < d.n_points; ++p)
      if (L.point_off[p] >= 0)
        for (int a = 0; a < 3; ++a) xp[L.off_xyz + 3 * p + a] += delta[L.point_off[p] + a];
  }

  void InnerIterations(double* x) override;
};

// One 3D point with everything else fixed: the inner_program of
// CoordinateDescentMinimizer::Minimize (ceres internal/ceres/coordinate_descent_minimizer.cc).
class PointEvaluator : public TREvaluator {
 public:
  const BAEvaluator& ba;
  const double* xfull;
  int64_t p;
  double H[9], g[3];
  PointEvaluator(const BAEvaluator& b, const double* x, int64_t pt) : ba(b), xfull(x), p(pt) {}
  int NumParameters() const override { return 3; }
  int NumLocal() const override { return 3; }
  bool Evaluate(const double* x, double* cost, bool with_jac) override {
    std::vector<double> r, Jc, Jp, Jamb, scratch;
    int cols[BAEvaluator::kMaxDc], dc;
    double total = 0;
    if (with_jac) { for (int k = 0; k < 9; ++k) H[k] = 0; g[0] = g[1] = g[2] = 0; }
    const int C = ba.d.channels;
    for (int64_t o = ba.L.pt_begin[p]; o < ba.L.pt_begin[p + 1]; ++o) {
      total += ba.LinearizeBlock(xfull, o, with_jac, r, Jc, cols, &dc, Jp, Jamb, scratch, nullptr, nullptr, x);
      if (!with_jac) continue;
      for (int a = 0; a < 3; ++a) {
        for (int i = 0; i < C; ++i) g[a] += Jp[(size_t)i * 3 + a] * r[i];
        for (int b = 0; b < 3; ++b)
          for (int i = 0; i < C; ++i) H[a * 3 + b] += Jp[(size_t)i * 3 + a] * Jp[(size_t)i * 3 + b];
      }
    }
    *cost = total;
    return std::isfinite(total);
  }
  void Gradient(double* gg) const override { for (int a = 0; a < 3; ++a) gg[a] = g[a]; }
  void SquaredColumnNorm(double* dd) const override { for (int a = 0; a < 3; ++a) dd[a] = H[a * 4]; }
  bool SolveDamped(const double* D2, double* delta, int* iters) override {
    double Hd[9], inv[9];
    for (int k = 0; k < 9; ++k) Hd[k] = H[k];
    for (int a = 0; a < 3; ++a) Hd[a * 4] += D2[a];
    if (!Invert3x3Sym(Hd, inv)) return false;
    for (int a = 0; a < 3; ++a) delta[a] = -(inv[a * 3] * g[0] + inv[a * 3 + 1] * g[1] + inv[a * 3 + 2] * g[2]);
    *iters = 1;
    return true;
  }
  double ModelCostChange(const double* dl) const override {
    double gd = 0, dHd = 0;
    for (int a = 0; a < 3; ++a) { gd += g[a] * dl[a]; for (int b = 0; b < 3; ++b) dHd += dl[a] * H[a * 3 + b] * dl[b]; }
    return -gd - 0.5 * dHd;
  }
  void Plus(const double* x, const double* dl, double* xp) const override { for (int a = 0; a < 3; ++a) xp[a] = x[a] + dl[a]; }
};

inline void BAEvaluator::InnerIterations(double* x) {
  StageClock::Scope clk(&GlobalStageClock().t[5]);
  std::vector<double> xin(x, x + L.n_ambient);
#pragma omp parallel for schedule(dynamic, 8)
  for (int64_t p = 0; p < d.n_points; ++p) {
    if (L.point_off[p] < 0) continue;
    PointEvaluator pe(*this, xin.data(), p);
    TrustRegionMinimizer tr(eo.inner);
    TRSummary s;
    double xp[3] = {xin[L.off_xyz + 3 * p], xin[L.off_xyz + 3 * p + 1], xin[L.off_xyz + 3 * p + 2]};
    tr.Minimize(&pe, xp, &s);
    for (int a = 0; a < 3; ++a) x[L.off_xyz + 3 * p + a] = xp[a];
  }
}

inline TROptions ToTROptions(const pxr_solver_options& o) {
  TROptions t;
  t.max_num_iterations = o.max_num_iterations;
  t.function_tolerance = o.function_tolerance;
  t.gradient_tolerance = o.gradient_tolerance;
  t.parameter_tolerance = o.parameter_tolerance;
  t.min_relative_decrease = o.min_relative_decrease;
  t.initial_trust_region_radius = o.initial_trust_region_radius;
  t.max_trust_region_radius = o.max_trust_region_radius;
  t.min_trust_region_radius = o.min_trust_region_radius;
  t.min_lm_diagonal = o.min_lm_diagonal;
  t.max_lm_diagonal = o.max_lm_diagonal;
  t.jacobi_scaling = o.jacobi_scaling != 0;
  t.max_num_consecutive_invalid_steps = o.max_num_consecutive_invalid_steps;
  t.use_inner_iterations = o.use_inner_iterations != 0;
  t.inner_iteration_tolerance = o.inner_iteration_tolerance;
  t.use_nonmonotonic_steps = o.use_nonmonotonic_steps != 0;
  t.max_consecutive_nonmonotonic_steps = o.max_consecutive_nonmonotonic_steps;
  return t;
}

}  // namespace orc
