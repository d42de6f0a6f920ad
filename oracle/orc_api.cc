// oracle/orc_api.cc — TEST INFRASTRUCTURE ONLY: C entry points of the CPU oracle
// (liboracle.so), loaded with ctypes by tests/, __graft_entry__.smoke() and
// bench.py's cpu_baseline / --impl reference legs.  Never linked into libpxr.so.
#include <dlfcn.h>

#include <chrono>
#include <cstring>

#include "orc_ba.h"
#include "orc_refs_graph.h"
#include "orc_ka.h"
#include "orc_costmap.h"

using namespace orc;

static InterpConfig ToInterp(const pxr_interp_config* c) {
  InterpConfig ic;
  ic.l2_normalize = c ? c->l2_normalize != 0 : true;
  ic.use_float_simd = c ? c->use_float_simd != 0 : false;
  return ic;
}

extern "C" {

int orc_num_threads() { return omp_get_max_threads(); }

// The reference's own AVX2 spline as the inner kernel of every bicubic evaluation (see orc_core.h::RefSpline):
// path = oracle/_ref/libpxref.so.  Returns 0 when all three entry points resolved; enable = 0 switches back.
int orc_use_reference_spline(const char* path, int enable) {
  RefSpline& R = GlobalRefSpline();
  if (!enable) { R = RefSpline(); return 0; }
  void* h = dlopen(path, RTLD_NOW | RTLD_LOCAL);
  if (!h) return 1;
  RefSpline r;
  r.f16 = (decltype(r.f16))dlsym(h, "ref_spline_f16");
  r.f32 = (decltype(r.f32))dlsym(h, "ref_spline_f32");
  r.f64 = (decltype(r.f64))dlsym(h, "ref_spline_f64");
  if (!r.f16 || !r.f32 || !r.f64) return 2;
  R = r;
  return 0;
}

// wall-clock split of the solves since the last reset (orc_ba.h::StageClock): evaluation with Jacobians, cost-only
// evaluation, Schur elimination, reduced solve, back-substitution + model cost, inner iterations
void orc_stage_seconds(double* out6, int reset) {
  StageClock& c = GlobalStageClock();
  if (out6) for (int i = 0; i < 6; ++i) out6[i] = c.t[i];
  if (reset) c = StageClock();
}

// CPU counterpart of pxr_synth_patches_device (pixel-perfect-sfm_b200/csrc/pxr_synth.cu): the same counter-based hash,
// field model and noise, so that bench.py's reference arm can build its workload WITHOUT the CUDA library.  (libm's
// logf / cosf / 1/sqrtf stand in for the device's fast-math intrinsics: same distribution, last bits differ.)
static inline uint64_t Mix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
static inline float NormalFrom(uint64_t key) {
  const uint64_t h = Mix64(key);
  const float u1 = ((uint32_t)(h >> 40) + 1.0f) * (1.0f / 16777217.0f);
  const float u2 = (uint32_t)(h & 0xFFFFFF) * (1.0f / 16777216.0f);
  return std::sqrt(-2.0f * std::log(u1)) * std::cos(6.2831853f * u2);
}
int orc_synth_patches(uint16_t* out, int64_t n_patches, int ps, int C, const double* uv0, const int64_t* field,
                      uint64_t seed, double noise_sigma) {
  if (!out || !uv0 || !field || n_patches < 1 || ps < 1 || C < 2 || (C & 1) || C > 1024) return 1;
  const float noise = (float)noise_sigma;
  const int npx = ps * ps;
#pragma omp parallel
  {
    std::vector<float> coef((size_t)4 * C), vals(C), nz(C);
    std::vector<uint64_t> keys(C);
#pragma omp for schedule(static)
    for (int64_t pi = 0; pi < n_patches; ++pi) {
      const int64_t fid = field[pi];
      for (int i = 0; i < 4 * C; ++i) {
        const int k = i / C, c = i % C;
        const float sd = k == 0 ? 1.0f : 0.15f;
        coef[i] = sd * NormalFrom(seed ^ Mix64((uint64_t)fid * 4099ull + (uint64_t)k * 1000003ull + (uint64_t)c * 7919ull + 17ull));
      }
      for (int px = 0; px < npx; ++px) {
        const int row = px / ps, col = px % ps;
        const float du = (float)((double)col - uv0[2 * pi]);
        const float dv = (float)((double)row - uv0[2 * pi + 1]);
        const float dudv = du * dv;
        float n2 = 0.f;
        for (int c = 0; c < C; ++c) {
          const float f = coef[c] + coef[C + c] * du + coef[2 * C + c] * dv + coef[3 * C + c] * dudv;
          vals[c] = f; n2 += f * f;
        }
        const float ninv = 1.0f / std::sqrt(n2);
        if (noise > 0.f) {
          const uint64_t key0 = seed * 0x100000001B3ull + ((uint64_t)pi * npx + px) * (uint64_t)C;
          for (int c = 0; c < C; ++c) {           // hash, then Box-Muller: a plain loop the compiler can vectorise
            const uint64_t h = Mix64(key0 + c);
            const float u1 = ((uint32_t)(h >> 40) + 1.0f) * (1.0f / 16777217.0f);
            const float u2 = (uint32_t)(h & 0xFFFFFF) * (1.0f / 16777216.0f);
            nz[c] = std::sqrt(-2.0f * std::log(u1)) * std::cos(6.2831853f * u2);
          }
          for (int c = 0; c < C; ++c) vals[c] = vals[c] * ninv + noise * nz[c];
        } else {
          for (int c = 0; c < C; ++c) vals[c] *= ninv;
        }
        half_t* dst = reinterpret_cast<half_t*>(out) + ((size_t)pi * npx + px) * C;
        for (int c = 0; c < C; ++c) dst[c] = (half_t)vals[c];
      }
    }
  }
  return 0;
}
void orc_set_num_threads(int n) { if (n > 0) omp_set_num_threads(n); }

// a1 — single spline evaluations (pin against oracle/_ref)
void orc_spline_f16(const uint16_t* p, double x, float* f, float* dfdx) {
  half_t h[4];
  std::memcpy(h, p, 8);
  CubicHermiteF32<half_t>(h[0], h[1], h[2], h[3], x, f, dfdx);
}
void orc_spline_f32(const float* p, double x, float* f, float* dfdx) {
  CubicHermiteF32<float>(p[0], p[1], p[2], p[3], x, f, dfdx);
}
void orc_spline_f64(const double* p, double x, double* f, double* dfdx) {
  CubicHermiteF64(p[0], p[1], p[2], p[3], x, f, dfdx);
}
void orc_spline_ceres(const double* p, double x, double* f, double* dfdx) {
  CubicHermiteCeres(p[0], p[1], p[2], p[3], x, f, dfdx);
}

// a3/a4 — PixelInterpolator::Evaluate on a raw grid (rows r, cols c)
void orc_pixel_interp(const void* data, int dtype, int h, int w, int c, double r, double col,
                      int l2_normalize, int use_float_simd, double* f, double* dfdr, double* dfdc) {
  Patch g{data, dtype, h, w, c, {0, 0}, {1.0, 1.0}, 1.0};
  InterpConfig ic; ic.l2_normalize = l2_normalize != 0; ic.use_float_simd = use_float_simd != 0;
  PixelInterp(g, ic, r, col, f, dfdr, dfdc);
}
void orc_bicubic_ceres(const void* data, int dtype, int h, int w, int c, double r, double col,
                       double* f, double* dfdr, double* dfdc) {
  Patch g{data, dtype, h, w, c, {0, 0}, {1.0, 1.0}, 1.0};
  BiCubicCeres(g, r, col, f, dfdr, dfdc);
}

// a6 — WorldToPixel
void orc_world_to_pixel(int model, const double* cam, const double* q, const double* t,
                        const double* X, double* xy) {
  WorldToPixel<double>(model, cam, q, t, X, xy);
}
int orc_camera_num_params(int model) { return CameraNumParams(model); }
void orc_camera_param_groups(int model, uint32_t* focal, uint32_t* pp, uint32_t* extra) {
  CameraParamGroups(model, focal, pp, extra);
}
void orc_quaternion_plus(const double* x, const double* d, double* out) { QuaternionPlus(x, d, out); }

void orc_loss(int type, double a, double weight, double s, double* rho) {
  Loss l; l.type = type; l.a = a; l.weight = weight;
  l.Evaluate(s, rho);
}

static BAEvalOptions MakeEO(const pxr_interp_config* ic, const pxr_solver_options* so) {
  BAEvalOptions eo;
  eo.interp = ToInterp(ic);
  eo.loss.type = so->loss_type; eo.loss.a = so->loss_scale; eo.loss.weight = 1.0;
  eo.iterative_schur = so->linear_solver == PXR_SOLVER_ITERATIVE_SCHUR;
  eo.max_linear_solver_iterations = so->max_linear_solver_iterations;
  return eo;
}

// a7 — every residual block at the current parameters (same outputs as pxr_ba_evaluate)
int orc_ba_evaluate(const pxr_ba_desc* d, const pxr_interp_config* ic, const pxr_solver_options* so,
                    double* sq_norm, double* gtr, double* gtg, double* xy, double* residuals,
                    double* cost) {
  BAEvalOptions eo = MakeEO(ic, so);
  const int C = d->channels;
  double total = 0;
#pragma omp parallel for reduction(+ : total) schedule(dynamic, 64)
  for (int64_t o = 0; o < d->n_obs; ++o) {
    const int img = d->obs_img[o];
    const int64_t pt = d->obs_pt[o];
    const int cam = d->img_cam[img];
    double pxy[2], uv[2];
    WorldToPixel<double>(d->cam_model[cam], d->cam_params + (size_t)cam * PXR_MAX_CAM_PARAMS,
                         d->qvec + 4 * img, d->tvec + 3 * img, d->xyz + 3 * pt, pxy);
    const Patch patch = MakePatch(*d, o);
    ToPixelCoordinates<double>(patch, pxy, uv);
    std::vector<double> f(C), dfdr(C), dfdc(C);
    PixelInterp(patch, eo.interp, uv[1], uv[0], f.data(), dfdr.data(), dfdc.data());
    double s = 0, gr0 = 0, gr1 = 0, g00 = 0, g01 = 0, g11 = 0;
    for (int i = 0; i < C; ++i) {
      const double r = d->refs ? f[i] - d->refs[(size_t)pt * C + i] : f[i];
      if (residuals) residuals[(size_t)o * C + i] = r;
      s += r * r;
      gr0 += dfdc[i] * r; gr1 += dfdr[i] * r;
      g00 += dfdc[i] * dfdc[i]; g01 += dfdc[i] * dfdr[i]; g11 += dfdr[i] * dfdr[i];
    }
    if (sq_norm) sq_norm[o] = s;
    if (gtr) { gtr[2 * o] = gr0; gtr[2 * o + 1] = gr1; }
    if (gtg) { gtg[3 * o] = g00; gtg[3 * o + 1] = g01; gtg[3 * o + 2] = g11; }
    if (xy) { xy[2 * o] = pxy[0]; xy[2 * o + 1] = pxy[1]; }
    double rho[3];
    eo.loss.Evaluate(s, rho);
    total += 0.5 * rho[0];
  }
  if (cost) *cost = total;
  return 0;
}

// The reference's cost functors as ceres would evaluate them (residuals/src/feature_reference.h:98-137 through
// AutoDiffCostFunction): per block r [C] and the AMBIENT Jacobian, columns [q(4) t(3) X(3) cam(K of the block's model)],
// row-major C x (10 + PXR_MAX_CAM_PARAMS) with the unused camera columns zero.  Checks pxr_ba_evaluate_jacobians
// and the `_residuals` mirror.
int orc_ba_block_jacobians(const pxr_ba_desc* d, const pxr_interp_config* ic, double* residuals, double* J) {
  pxr_solver_options so; std::memset(&so, 0, sizeof(so));
  BAEvalOptions eo = MakeEO(ic, &so);
  const int C = d->channels;
  const int W = 10 + PXR_MAX_CAM_PARAMS;
  int bad = 0;
#pragma omp parallel for schedule(dynamic, 64)
  for (int64_t o = 0; o < d->n_obs; ++o) {
    const int img = d->obs_img[o];
    const int64_t pt = d->obs_pt[o];
    const int cam = d->img_cam[img];
    const int model = d->cam_model[cam];
    const int K = CameraNumParams(model);
    EvalBlockFn fn = SelectEval<true>(model);
    if (!fn) { bad = 1; continue; }
    const Patch patch = MakePatch(*d, o);
    std::vector<double> r(C), Jb((size_t)C * (10 + K)), scratch;
    fn(model, d->cam_params + (size_t)cam * PXR_MAX_CAM_PARAMS, d->qvec + 4 * img, d->tvec + 3 * img, d->xyz + 3 * pt,
       patch, eo.interp, d->refs ? d->refs + (size_t)pt * C : nullptr, r.data(), Jb.data(), nullptr, scratch);
    for (int i = 0; i < C; ++i) {
      if (residuals) residuals[(size_t)o * C + i] = r[i];
      if (J) {
        double* row = J + ((size_t)o * C + i) * W;
        for (int n = 0; n < W; ++n) row[n] = n < 10 + K ? Jb[(size_t)i * (10 + K) + n] : 0.0;
      }
    }
  }
  return bad;
}

int orc_ba_layout(const pxr_ba_desc* d, int* n_cam_local, int* n_local, int* pose_off, int* intr_off,
                  int64_t* point_off) {
  BALayout L = MakeLayout(*d);
  *n_cam_local = L.n_cam_local; *n_local = L.n_local;
  if (pose_off) for (int i = 0; i < d->n_images; ++i) pose_off[i] = L.pose_off[i];
  if (intr_off) for (int i = 0; i < d->n_cameras; ++i) intr_off[i] = L.intr_off[i];
  if (point_off) for (int64_t i = 0; i < d->n_points; ++i) point_off[i] = L.point_off[i];
  return 0;
}

// SchurJacobiPCG on a caller's system: S [n][n] symmetric, full storage; the preconditioner blocks are
// [blk_off[k], blk_off[k] + blk_dim[k]).  x [n], iterations and stop_reason (PCGStop: 0 zeta test, 1 p.q <= 0,
// 2 iteration cap, 3 failure).  Returns 0 when the solve succeeded, 1 on failure (as the oracle's step reports it).
int orc_schur_jacobi_pcg(int n, const double* S, const double* b, int n_blocks, const int32_t* blk_off,
                         const int32_t* blk_dim, int max_iter, double eta, double* x, int* iterations, int* stop_reason) {
  std::vector<double> Sv(S, S + (size_t)n * n), bv(b, b + n), xv;
  std::vector<std::pair<int, int>> blocks;
  for (int k = 0; k < n_blocks; ++k) blocks.emplace_back(blk_off[k], blk_dim[k]);
  int it = 0, stop = kPCGFailure;
  const bool ok = SchurJacobiPCG(n, Sv, bv, blocks, max_iter, eta, &xv, &it, &stop);
  for (int i = 0; i < n; ++i) x[i] = (size_t)i < xv.size() ? xv[i] : 0.0;   // a failed block inverse leaves xv empty
  *iterations = it; *stop_reason = stop;
  return ok ? 0 : 1;
}

// Linearise at the current parameters with the full (un-shortcut) Jacobians and run ONE
// LM step computation at the given radius (jacobi scaling taken from this linearisation, as
// in iteration 0).  Outputs (any may be NULL): Hcc [nc*nc], gc [nc], Hpp [np*9], gp [np*3],
// S [nc*nc] / rhs [nc] (damped Schur complement system), delta [n_local], model_cost_change.
int orc_ba_linearize(const pxr_ba_desc* d, const pxr_interp_config* ic, const pxr_solver_options* so,
                     double radius, double* cost, double* Hcc, double* gc, double* Hpp, double* gp,
                     double* S, double* rhs, double* delta, double* model_cost_change) {
  BAEvalOptions eo = MakeEO(ic, so);
  BAEvaluator ev(*d, eo);
  std::vector<double> x(ev.NumParameters());
  ev.PackParameters(x.data());
  double c;
  if (!ev.Evaluate(x.data(), &c, true)) return 1;
  if (cost) *cost = c;
  const int nc = ev.L.n_cam_local, nl = ev.L.n_local;
  if (Hcc) std::memcpy(Hcc, ev.Hcc.data(), sizeof(double) * (size_t)nc * nc);
  if (gc) std::memcpy(gc, ev.gc.data(), sizeof(double) * nc);
  if (Hpp) std::memcpy(Hpp, ev.Hpp.data(), sizeof(double) * ev.Hpp.size());
  if (gp) std::memcpy(gp, ev.gp.data(), sizeof(double) * ev.gp.size());
  std::vector<double> diag(nl), D2(nl), dl(nl);
  ev.SquaredColumnNorm(diag.data());
  for (int i = 0; i < nl; ++i) {
    const double sc = so->jacobi_scaling ? 1.0 / (1.0 + std::sqrt(diag[i])) : 1.0;
    const double ds = diag[i] * sc * sc;
    const double cl = std::min(std::max(ds, so->min_lm_diagonal), so->max_lm_diagonal);
    D2[i] = cl / (radius * sc * sc);
  }
  int iters;
  if (!ev.SolveDamped(D2.data(), dl.data(), &iters)) return 2;
  if (S) std::memcpy(S, ev.S_last.data(), sizeof(double) * (size_t)nc * nc);
  if (rhs) std::memcpy(rhs, ev.rhs_last.data(), sizeof(double) * nc);
  if (delta) std::memcpy(delta, dl.data(), sizeof(double) * nl);
  if (model_cost_change) *model_cost_change = ev.ModelCostChange(dl.data());
  return 0;
}

static void FillSummary(const TRSummary& s, pxr_summary* out, const pxr_ba_desc* d) {
  if (!out) return;
  out->initial_cost = s.initial_cost; out->final_cost = s.final_cost;
  out->num_successful_steps = s.num_successful_steps;
  out->num_unsuccessful_steps = s.num_unsuccessful_steps;
  out->num_inner_iteration_steps = s.num_inner_iteration_steps;
  out->termination_type = s.termination_type;
  if (d) { out->num_residual_blocks = (int32_t)d->n_obs; out->num_residuals = d->n_obs * d->channels; }
  const int n = (int)s.iterations.size();
  const int m = std::min(n, out->iterations ? out->iterations_capacity : 0);
  for (int i = 0; i < m; ++i) {
    pxr_iteration_summary& o = out->iterations[i];
    const TRIteration& it = s.iterations[i];
    o.iteration = it.iteration; o.step_is_valid = it.step_is_valid; o.step_is_successful = it.step_is_successful;
    o.cost = it.cost; o.cost_change = it.cost_change; o.gradient_max_norm = it.gradient_max_norm;
    o.step_norm = it.step_norm; o.relative_decrease = it.relative_decrease;
    o.trust_region_radius = it.trust_region_radius; o.linear_solver_iterations = it.linear_solver_iterations;
    o.iteration_time_s = 0;
  }
  out->num_iterations = n;
  std::snprintf(out->message, sizeof(out->message), "%s", s.message.c_str());
}

// a11 — FeatureReferenceBundleOptimizer::Run restated: ceres::Solve on the problem IR.
int orc_ba_solve(const pxr_ba_desc* d, const pxr_interp_config* ic, const pxr_solver_options* so,
                 pxr_summary* summary, int verbose) {
  auto t0 = std::chrono::steady_clock::now();
  BAEvalOptions eo = MakeEO(ic, so);
  BAEvaluator ev(*d, eo);
  std::vector<double> x(ev.NumParameters());
  ev.PackParameters(x.data());
  TROptions to = ToTROptions(*so);
  to.verbose = verbose != 0;
  TrustRegionMinimizer tr(to);
  TRSummary s;
  tr.Minimize(&ev, x.data(), &s);
  ev.UnpackParameters(x.data());
  FillSummary(s, summary, d);
  if (summary) {
    summary->total_time_s = summary->solve_time_s =
        std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  }
  return 0;
}

// CoordinateDescentMinimizer::Minimize alone on the current parameters (updates desc->xyz)
int orc_ba_inner_iterations(const pxr_ba_desc* d, const pxr_interp_config* ic, const pxr_solver_options* so) {
  BAEvalOptions eo = MakeEO(ic, so);
  BAEvaluator ev(*d, eo);
  std::vector<double> x(ev.NumParameters());
  ev.PackParameters(x.data());
  ev.InnerIterations(x.data());
  ev.UnpackParameters(x.data());
  return 0;
}

// CPU-baseline timing: seconds for `reps` Jacobian evaluations (residuals + full Jacobians +
// normal-equation blocks, all host threads), and for one damped Schur solve.
int orc_ba_time(const pxr_ba_desc* d, const pxr_interp_config* ic, const pxr_solver_options* so,
                int reps, double* eval_s, double* cost_eval_s, double* solve_s) {
  BAEvalOptions eo = MakeEO(ic, so);
  BAEvaluator ev(*d, eo);
  std::vector<double> x(ev.NumParameters());
  ev.PackParameters(x.data());
  double c;
  ev.Evaluate(x.data(), &c, true);  // warm-up
  auto t0 = std::chrono::steady_clock::now();
  for (int i = 0; i < reps; ++i) ev.Evaluate(x.data(), &c, true);
  auto t1 = std::chrono::steady_clock::now();
  for (int i = 0; i < reps; ++i) ev.Evaluate(x.data(), &c, false);
  auto t2 = std::chrono::steady_clock::now();
  const int nl = ev.L.n_local;
  std::vector<double> diag(nl), D2(nl), dl(nl);
  ev.SquaredColumnNorm(diag.data());
  for (int i = 0; i < nl; ++i) {
    const double sc = 1.0 / (1.0 + std::sqrt(diag[i]));
    D2[i] = std::min(std::max(diag[i] * sc * sc, 1e-6), 1e32) / (1e4 * sc * sc);
  }
  int iters;
  ev.SolveDamped(D2.data(), dl.data(), &iters);
  auto t3 = std::chrono::steady_clock::now();
  if (eval_s) *eval_s = std::chrono::duration<double>(t1 - t0).count() / reps;
  if (cost_eval_s) *cost_eval_s = std::chrono::duration<double>(t2 - t1).count() / reps;
  if (solve_s) *solve_s = std::chrono::duration<double>(t3 - t2).count();
  return 0;
}

// a12
int orc_refs_compute(const pxr_ba_desc* d, const pxr_interp_config* ic, int loss_type,
                     double loss_scale, int iters, double* refs_out, int64_t* src_obs_out) {
  Loss l; l.type = loss_type; l.a = loss_scale; l.weight = 1.0;
  ComputeReferences(*d, ToInterp(ic), l, iters, refs_out, src_obs_out);
  return 0;
}
void orc_robust_mean_irls(const double* desc, int n, int C, int loss_type, double loss_scale,
                          int iters, int l2_normalize, double* mean) {
  Loss l; l.type = loss_type; l.a = loss_scale; l.weight = 1.0;
  std::vector<double> dv(desc, desc + (size_t)n * C), m;
  RobustMeanIRLS(dv, n, C, l, iters, l2_normalize != 0, &m);
  std::memcpy(mean, m.data(), sizeof(double) * C);
}

// f1 — cost maps (costmap_extractor.h:230-358); `out` in the patches' dtype, [n_patches][ph][pw][3 or 1]
int orc_costmaps_compute(const pxr_ba_desc* d, int loss_type, double loss_scale, int as_gradientfield,
                         int apply_sqrt, void* out) {
  Loss l; l.type = loss_type; l.a = loss_scale; l.weight = 1.0;
  return ComputeCostmaps(*d, l, as_gradientfield != 0, apply_sqrt != 0, out);
}

// a13/a14
void orc_graph_track_labels(int64_t n_nodes, const int32_t* node_image, int64_t n_edges,
                            const int64_t* es, const int64_t* ed, const double* sim, int64_t* labels) {
  TrackLabels(n_nodes, node_image, n_edges, es, ed, sim, labels);
}
void orc_graph_score_labels(int64_t n_nodes, int64_t n_edges, const int64_t* es, const int64_t* ed,
                            const double* sim, const int64_t* labels, double* scores) {
  ScoreLabels(n_nodes, n_edges, es, ed, sim, labels, scores);
}
void orc_graph_root_labels(int64_t n_nodes, const int64_t* labels, const double* scores, uint8_t* is_root) {
  RootLabels(n_nodes, labels, scores, is_root);
}
int orc_ka_problem_labels(int64_t n_nodes, const int64_t* labels, int max_per_problem, int32_t* out) {
  return KAProblemLabels(n_nodes, labels, max_per_problem, out);
}

// a8/a15 — featuremetric KA
int orc_ka_evaluate(const pxr_ka_desc* d, const pxr_interp_config* ic, const pxr_solver_options* so,
                    double* sq_norm, double* cost) {
  return KAEvaluateAll(*d, ToInterp(ic), *so, sq_norm, cost);
}
int orc_ka_solve(const pxr_ka_desc* d, const pxr_interp_config* ic, const pxr_solver_options* so,
                 pxr_summary* summary) {
  auto t0 = std::chrono::steady_clock::now();
  TRSummary acc;
  KASolveAll(*d, ToInterp(ic), *so, &acc);
  if (summary) {
    summary->initial_cost = acc.initial_cost; summary->final_cost = acc.final_cost;
    summary->num_successful_steps = acc.num_successful_steps;
    summary->num_unsuccessful_steps = acc.num_unsuccessful_steps;
    summary->num_residual_blocks = (int32_t)d->n_edges;
    summary->num_residuals = d->n_edges * d->channels;
    summary->num_iterations = 0;
    summary->total_time_s = summary->solve_time_s =
        std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  }
  return 0;
}

}  // extern "C"
