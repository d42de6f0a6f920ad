// oracle_geo/orc_geo.cc — TEST INFRASTRUCTURE ONLY: the CPU restatement of GEOMETRIC (reprojection-error) bundle
// adjustment (liboracle_geo.so), loaded with ctypes by tests/geo_oracle_lib.py and scripts/geometric_ba_bench.py.
// Never linked into libpxr.so.
//
// Reference: GeometricBundleOptimizer::AddResiduals (bundle_adjustment/src/geometric_bundle_optimizer.h:36-83) adds
// colmap::BundleAdjustmentCostFunction / ...ConstantPoseCostFunction (residuals/src/geometric.h:16-41):
//   r = WorldToImage(camera, R(q) X + t) - point2D.XY()       (2 residuals, image pixels)
// evaluated here with forward-mode Jets through the oracle's WorldToPixel, as ceres::AutoDiffCostFunction does.  The
// problem IR is the featuremetric one (pxr_ba_desc, patch fields unused) plus the observed keypoints obs_xy.
//
// GeoEvaluator is the featuremetric oracle's BAEvaluator (oracle/orc_ba.h, used as it is) with the residual block
// replaced: it re-states Evaluate and the per-point inner problem around a 2-row block and inherits the layout, the
// exact Schur solve / SCHUR_JACOBI PCG, the model cost change and the manifold Plus, so both paths share one solver.
#include <chrono>
#include <cstring>

#include "orc_ba.h"

using namespace orc;

namespace {

// One geometric residual block: r (2) and the ambient Jacobian columns [q(4) t(3) X(3) cam(K)] by Jets.
template <int K, bool POSE>
void EvalGeoJets(int model, const double* cam, const double* q, const double* t, const double* X, const double* kp,
                 double* r, double* J /*2 x (POSE?7:0)+3+K*/, double* xy_out) {
  constexpr int N = (POSE ? 7 : 0) + 3 + K;
  typedef Jet<N> JT;
  JT jq[4], jt[3], jX[3], jc[K > 0 ? K : 1];
  int k = 0;
  if (POSE) { for (int i = 0; i < 4; ++i) jq[i] = JT(q[i], k++); for (int i = 0; i < 3; ++i) jt[i] = JT(t[i], k++); }
  else { for (int i = 0; i < 4; ++i) jq[i] = JT(q[i]); for (int i = 0; i < 3; ++i) jt[i] = JT(t[i]); }
  for (int i = 0; i < 3; ++i) jX[i] = JT(X[i], k++);
  for (int i = 0; i < K; ++i) jc[i] = JT(cam[i], k++);
  JT xy[2];
  WorldToPixel<JT>(model, jc, jq, jt, jX, xy);
  for (int i = 0; i < 2; ++i) {
    r[i] = xy[i].a - kp[i];
    if (J) for (int n = 0; n < N; ++n) J[i * N + n] = xy[i].v[n];
  }
  if (xy_out) { xy_out[0] = xy[0].a; xy_out[1] = xy[1].a; }
}

typedef void (*EvalGeoFn)(int, const double*, const double*, const double*, const double*, const double*, double*,
                          double*, double*);
template <bool POSE>
EvalGeoFn SelectGeoEval(int model) {
  switch (CameraNumParams(model)) {
    case 3: return &EvalGeoJets<3, POSE>;
    case 4: return &EvalGeoJets<4, POSE>;
    case 5: return &EvalGeoJets<5, POSE>;
    case 8: return &EvalGeoJets<8, POSE>;
    case 12: return &EvalGeoJets<12, POSE>;
  }
  return nullptr;
}

constexpr int kMaxDc = BAEvaluator::kMaxDc;

class GeoEvaluator : public BAEvaluator {
 public:
  const double* kp;   // [n_obs][2]

  GeoEvaluator(const pxr_ba_desc& desc, const BAEvalOptions& o, const double* obs_xy) : BAEvaluator(desc, o), kp(obs_xy) {}

  // Local, loss-corrected Jacobian of one block (as BAEvaluator::LinearizeBlock): Jc (2 x kMaxDc) with column ids,
  // Jp (2 x 3), r (2).  Returns 0.5 rho(s).
  double Linearize(const double* x, int64_t o, bool with_jac, double* r, double* Jc, int* cols, int* dc_out, double* Jp,
                   double* sq_norm_out, const double* X_override = nullptr) const {
    const int img = d.obs_img[o];
    const int64_t pt = d.obs_pt[o];
    const int cam = d.img_cam[img];
    const int model = d.cam_model[cam];
    const int K = CameraNumParams(model);
    const bool pose_var = L.pose_off[img] >= 0;
    const double* q = x + L.off_q + 4 * img;
    const double* t = x + L.off_t + 3 * img;
    const double* X = X_override ? X_override : x + L.off_xyz + 3 * pt;
    const double* cp = x + L.off_cam + (int64_t)PXR_MAX_CAM_PARAMS * cam;
    const int N = (pose_var ? 7 : 0) + 3 + K;
    double Jamb[2 * (7 + 3 + PXR_MAX_CAM_PARAMS)];
    EvalGeoFn fn = pose_var ? SelectGeoEval<true>(model) : SelectGeoEval<false>(model);
    fn(model, cp, q, t, X, kp + 2 * o, r, with_jac ? Jamb : nullptr, nullptr);
    double s = 0;
    for (int i = 0; i < 2; ++i) s += r[i] * r[i];
    if (sq_norm_out) *sq_norm_out = s;
    double rho[3];
    eo.loss.Evaluate(s, rho);
    if (!with_jac) return 0.5 * rho[0];
    int dc = 0;
    const int xoff = pose_var ? 7 : 0;
    for (int k = 0; k < 2 * kMaxDc; ++k) Jc[k] = 0.0;
    if (pose_var) {
      double PJ[12];
      QuaternionPlusJacobian(q, PJ);
      for (int i = 0; i < 2; ++i)
        for (int a = 0; a < 3; ++a) {
          double v = 0;
          for (int b = 0; b < 4; ++b) v += Jamb[i * N + b] * PJ[b * 3 + a];
          Jc[i * kMaxDc + a] = v;
        }
      for (int a = 0; a < 3; ++a) cols[dc++] = L.pose_off[img] + a;
      int la = 3;
      for (int b = 0; b < 3; ++b) {
        if (d.tvec_const_mask[img] & (1u << b)) continue;
        for (int i = 0; i < 2; ++i) Jc[i * kMaxDc + dc] = Jamb[i * N + 4 + b];
        cols[dc++] = L.pose_off[img] + la++;
      }
    }
    if (L.intr_off[cam] >= 0) {
      int la = 0;
      for (int b = 0; b < K; ++b) {
        if (d.cam_const_mask[cam] & (1u << b)) continue;
        for (int i = 0; i < 2; ++i) Jc[i * kMaxDc + dc] = Jamb[i * N + xoff + 3 + b];
        cols[dc++] = L.intr_off[cam] + la++;
      }
    }
    *dc_out = dc;
    for (int i = 0; i < 2; ++i)
      for (int a = 0; a < 3; ++a) Jp[i * 3 + a] = Jamb[i * N + xoff + a];
    Corrector corr(s, rho);
    corr.CorrectJacobian(2, kMaxDc, r, Jc);
    corr.CorrectJacobian(2, 3, r, Jp);
    corr.CorrectResiduals(2, r);
    return 0.5 * rho[0];
  }

  // BAEvaluator::Evaluate with the geometric block: the same per-image block accumulation and scatter
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
    for (int i = 0; i < d.n_images; ++i) {
      int dc = 0;
      for (int a = 0; a < L.pose_dim[i]; ++a) img_cols[(size_t)i * BD + dc++] = L.pose_off[i] + a;
      const int cam = d.img_cam[i];
      for (int a = 0; a < L.intr_dim[cam]; ++a) img_cols[(size_t)i * BD + dc++] = L.intr_off[cam] + a;
      img_dc[i] = dc;
    }
#pragma omp parallel reduction(+ : total)
    {
      const int tid = omp_get_thread_num();
      double r[2], Jc[2 * kMaxDc], Jp[6];
      int cols[kMaxDc];
      if (with_jac) { tH[tid].assign((size_t)d.n_images * BD * BD, 0.0); tg[tid].assign((size_t)d.n_images * BD, 0.0); }
#pragma omp for schedule(dynamic, 16)
      for (int64_t p = 0; p < d.n_points; ++p) {
        for (int64_t o = L.pt_begin[p]; o < L.pt_begin[p + 1]; ++o) {
          int dc = 0;
          double s;
          total += Linearize(x, o, with_jac, r, Jc, cols, &dc, Jp, &s);
          obs_sq_norm[o] = s;
          if (!with_jac) continue;
          const bool pvar = L.point_off[p] >= 0;
          const int img = d.obs_img[o];
          double* Hb = &tH[tid][(size_t)img * BD * BD];
          double* gb = &tg[tid][(size_t)img * BD];
          for (int i = 0; i < 2; ++i) {
            const double* row = &Jc[i * kMaxDc];
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
            for (int i = 0; i < 2; ++i) {
              const double* jp = &Jp[i * 3];
              const double* row = &Jc[i * kMaxDc];
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

  void InnerIterations(double* x) override;
};

// One 3D point with everything else fixed (PointEvaluator of orc_ba.h with the geometric block)
class GeoPointEvaluator : public TREvaluator {
 public:
  const GeoEvaluator& ba;
  const double* xfull;
  int64_t p;
  double H[9], g[3];
  GeoPointEvaluator(const GeoEvaluator& b, const double* x, int64_t pt) : ba(b), xfull(x), p(pt) {}
  int NumParameters() const override { return 3; }
  int NumLocal() const override { return 3; }
  bool Evaluate(const double* x, double* cost, bool with_jac) override {
    double r[2], Jc[2 * kMaxDc], Jp[6];
    int cols[kMaxDc], dc;
    double total = 0;
    if (with_jac) { for (int k = 0; k < 9; ++k) H[k] = 0; g[0] = g[1] = g[2] = 0; }
    for (int64_t o = ba.L.pt_begin[p]; o < ba.L.pt_begin[p + 1]; ++o) {
      total += ba.Linearize(xfull, o, with_jac, r, Jc, cols, &dc, Jp, nullptr, x);
      if (!with_jac) continue;
      for (int a = 0; a < 3; ++a) {
        for (int i = 0; i < 2; ++i) g[a] += Jp[i * 3 + a] * r[i];
        for (int b = 0; b < 3; ++b)
          for (int i = 0; i < 2; ++i) H[a * 3 + b] += Jp[i * 3 + a] * Jp[i * 3 + b];
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

void GeoEvaluator::InnerIterations(double* x) {
  StageClock::Scope clk(&GlobalStageClock().t[5]);
  std::vector<double> xin(x, x + L.n_ambient);
#pragma omp parallel for schedule(dynamic, 8)
  for (int64_t p = 0; p < d.n_points; ++p) {
    if (L.point_off[p] < 0) continue;
    GeoPointEvaluator pe(*this, xin.data(), p);
    TrustRegionMinimizer tr(eo.inner);
    TRSummary s;
    double xp[3] = {xin[L.off_xyz + 3 * p], xin[L.off_xyz + 3 * p + 1], xin[L.off_xyz + 3 * p + 2]};
    tr.Minimize(&pe, xp, &s);
    for (int a = 0; a < 3; ++a) x[L.off_xyz + 3 * p + a] = xp[a];
  }
}

BAEvalOptions MakeEO(const pxr_solver_options* so) {
  BAEvalOptions eo;
  eo.loss.type = so->loss_type; eo.loss.a = so->loss_scale; eo.loss.weight = 1.0;
  eo.iterative_schur = so->linear_solver == PXR_SOLVER_ITERATIVE_SCHUR;
  eo.max_linear_solver_iterations = so->max_linear_solver_iterations;
  return eo;
}

}  // namespace

extern "C" {

// every residual block at the current parameters (the outputs of pxr_ba_evaluate on a geometric handle: gtr = r,
// gtg = (1, 0, 1), residuals [n_obs][2])
int orc_geo_evaluate(const pxr_ba_desc* d, const pxr_solver_options* so, const double* obs_xy, double* sq_norm,
                     double* gtr, double* gtg, double* xy, double* residuals, double* cost) {
  Loss loss; loss.type = so->loss_type; loss.a = so->loss_scale; loss.weight = 1.0;
  double total = 0;
#pragma omp parallel for reduction(+ : total) schedule(dynamic, 64)
  for (int64_t o = 0; o < d->n_obs; ++o) {
    const int img = d->obs_img[o];
    const int cam = d->img_cam[img];
    double pxy[2];
    WorldToPixel<double>(d->cam_model[cam], d->cam_params + (size_t)cam * PXR_MAX_CAM_PARAMS,
                         d->qvec + 4 * img, d->tvec + 3 * img, d->xyz + 3 * d->obs_pt[o], pxy);
    const double r0 = pxy[0] - obs_xy[2 * o], r1 = pxy[1] - obs_xy[2 * o + 1];
    double s = 0;
    s += r0 * r0; s += r1 * r1;
    if (residuals) { residuals[2 * o] = r0; residuals[2 * o + 1] = r1; }
    if (sq_norm) sq_norm[o] = s;
    if (gtr) { gtr[2 * o] = r0; gtr[2 * o + 1] = r1; }
    if (gtg) { gtg[3 * o] = 1.0; gtg[3 * o + 1] = 0.0; gtg[3 * o + 2] = 1.0; }
    if (xy) { xy[2 * o] = pxy[0]; xy[2 * o + 1] = pxy[1]; }
    double rho[3];
    loss.Evaluate(s, rho);
    total += 0.5 * rho[0];
  }
  if (cost) *cost = total;
  return 0;
}

// per block r [2] and the ambient Jacobian [2][10 + PXR_MAX_CAM_PARAMS] (q4|t3|X3|cam, unused camera columns zero)
int orc_geo_block_jacobians(const pxr_ba_desc* d, const double* obs_xy, double* residuals, double* J) {
  const int W = 10 + PXR_MAX_CAM_PARAMS;
  int bad = 0;
#pragma omp parallel for schedule(dynamic, 64)
  for (int64_t o = 0; o < d->n_obs; ++o) {
    const int img = d->obs_img[o];
    const int cam = d->img_cam[img];
    const int model = d->cam_model[cam];
    const int K = CameraNumParams(model);
    EvalGeoFn fn = SelectGeoEval<true>(model);
    if (!fn) { bad = 1; continue; }
    double r[2], Jb[2 * (10 + PXR_MAX_CAM_PARAMS)];
    fn(model, d->cam_params + (size_t)cam * PXR_MAX_CAM_PARAMS, d->qvec + 4 * img, d->tvec + 3 * img,
       d->xyz + 3 * d->obs_pt[o], obs_xy + 2 * o, r, Jb, nullptr);
    for (int i = 0; i < 2; ++i) {
      if (residuals) residuals[2 * o + i] = r[i];
      if (J) for (int n = 0; n < W; ++n) J[(2 * o + i) * W + n] = n < 10 + K ? Jb[i * (10 + K) + n] : 0.0;
    }
  }
  return bad;
}

// Linearise at the current parameters and run ONE LM step computation at `radius` (Jacobi scaling from this
// linearisation, as in iteration 0): the outputs of pxr_ba_debug_linearize.  Any output may be NULL.
int orc_geo_linearize(const pxr_ba_desc* d, const pxr_solver_options* so, const double* obs_xy, double radius,
                      double* cost, double* Hcc, double* gc, double* Hpp, double* gp, double* S, double* rhs,
                      double* delta, double* model_cost_change) {
  GeoEvaluator ev(*d, MakeEO(so), obs_xy);
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

// GeometricBundleOptimizer::Run restated: the trust-region solve on the problem IR, parameters updated in place
int orc_geo_solve(const pxr_ba_desc* d, const pxr_solver_options* so, const double* obs_xy, pxr_summary* out) {
  auto t0 = std::chrono::steady_clock::now();
  GeoEvaluator ev(*d, MakeEO(so), obs_xy);
  std::vector<double> x(ev.NumParameters());
  ev.PackParameters(x.data());
  TrustRegionMinimizer tr(ToTROptions(*so));
  TRSummary s;
  tr.Minimize(&ev, x.data(), &s);
  ev.UnpackParameters(x.data());
  if (!out) return 0;
  out->initial_cost = s.initial_cost; out->final_cost = s.final_cost;
  out->num_successful_steps = s.num_successful_steps;
  out->num_unsuccessful_steps = s.num_unsuccessful_steps;
  out->num_inner_iteration_steps = s.num_inner_iteration_steps;
  out->termination_type = s.termination_type;
  out->num_residual_blocks = (int32_t)d->n_obs; out->num_residuals = 2 * d->n_obs;
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
  out->total_time_s = out->solve_time_s = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  return 0;
}

// CoordinateDescentMinimizer::Minimize alone on the current parameters (updates desc->xyz)
int orc_geo_inner_iterations(const pxr_ba_desc* d, const pxr_solver_options* so, const double* obs_xy) {
  GeoEvaluator ev(*d, MakeEO(so), obs_xy);
  std::vector<double> x(ev.NumParameters());
  ev.PackParameters(x.data());
  ev.InnerIterations(x.data());
  ev.UnpackParameters(x.data());
  return 0;
}

}  // extern "C"
