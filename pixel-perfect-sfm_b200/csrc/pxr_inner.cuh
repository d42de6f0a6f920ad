// pxr_inner.cuh — inner iterations: one warp solves one 3D point with everything else fixed.
//
// Replaces ceres' CoordinateDescentMinimizer (enabled by the reference through
// use_inner_iterations=True, pixsfm/bundle_adjustment/main.py:41-44 and
// bundle_optimizer.h:131-134,350-355: all non-constant points form independent set 0).  Each
// point runs a Levenberg-Marquardt loop with Ceres' DEFAULT Solver::Options
// (CoordinateDescentMinimizer::Solve builds Minimizer::Options from defaults):
// max 50 iterations, function_tolerance 1e-6, gradient_tolerance 1e-10,
// parameter_tolerance 1e-8, Jacobi scaling, monotonic steps, 5 consecutive invalid steps.
// Every inner evaluation re-reads the point's feature windows.  On a large problem they are not
// L2-resident (at BASELINE configs[2] one pass over all observations touches about 2 GB of windows
// against a 50 MB L2), so the first rounds stream them from HBM like any full K1 pass; only the
// short lists of the late rounds fit in L2.
#pragma once
#include "pxr_ba_kernels.cuh"
#include "pxr_fm_eval.cuh"

namespace pxr {

struct InnerArgs {
  int64_t n_points;
  const int64_t* point_off; const int64_t* pt_begin;
  const int32_t* obs_img; const int64_t* obs_patch;
  const int32_t* img_cam; const int32_t* cam_model;
  const double* cam_params; const double* qvec; const double* tvec;
  double* xyz;                 // in/out (candidate set)
  const int32_t* corner; const double* scale; double ups;
  const uint8_t* patches; int ph, pw;
  const double* refs;
  LossParams loss;
  int l2_normalize;
};

struct PointEval { double cost, H[6], g[3]; };

// cost, J^T J (6 uniques: 00 01 02 11 12 22), J^T r of one point at X; whole warp cooperates.
template <typename T, int C, bool FS>
__device__ __forceinline__ void inner_eval(const InnerArgs& a, int64_t p, int lane, const double X[3], PointEval& e) {
  constexpr int CPL = C >= 32 ? C / 32 : 1;
  constexpr int ACTIVE = C / CPL;
  constexpr int TAP_BYTES = C * (int)sizeof(T);
  const bool active = lane < ACTIVE;
  const int64_t ob = a.pt_begin[p], oe = a.pt_begin[p + 1];
  double cost = 0, H0 = 0, H1 = 0, H2 = 0, H3 = 0, H4 = 0, H5 = 0, g0 = 0, g1 = 0, g2 = 0;
  double refv[CPL];
  if (a.refs && active) {
#pragma unroll
    for (int k = 0; k < CPL; ++k) refv[k] = __ldg(a.refs + p * C + lane * CPL + k);
  }
  for (int64_t base = ob; base < oe; base += 32) {
    const int cnt = (int)min((int64_t)32, oe - base);
    // lane i: geometry of observation base+i
    double u = 0, v = 0, Jp[2][3] = {{0, 0, 0}, {0, 0, 0}};
    const uint8_t* pbase = a.patches;
    if (lane < cnt) {
      const int64_t o = base + lane;
      const int img = a.obs_img[o];
      const int64_t pi = a.obs_patch ? a.obs_patch[o] : o;
      const int cam = a.img_cam[img];
      double q[4], t[3], cp[kMaxK], xy[2], Jpose[2][6], Jk[2][kMaxK];
#pragma unroll
      for (int i = 0; i < 4; ++i) q[i] = a.qvec[4 * (int64_t)img + i];
#pragma unroll
      for (int i = 0; i < 3; ++i) t[i] = a.tvec[3 * (int64_t)img + i];
#pragma unroll
      for (int i = 0; i < kMaxK; ++i) cp[i] = a.cam_params[(int64_t)cam * kMaxK + i];
      world_to_pixel<true>(a.cam_model[cam], cp, q, t, X, xy, Jpose, Jp, Jk);
      const double sx = a.scale[2 * pi] * a.ups, sy = a.scale[2 * pi + 1] * a.ups;
      u = (xy[0] * a.scale[2 * pi] - 0.5 - (double)a.corner[2 * pi]) * a.ups;
      v = (xy[1] * a.scale[2 * pi + 1] - 0.5 - (double)a.corner[2 * pi + 1]) * a.ups;
#pragma unroll
      for (int k = 0; k < 3; ++k) { Jp[0][k] *= sx; Jp[1][k] *= sy; }
      pbase = a.patches + pi * (int64_t)a.ph * a.pw * TAP_BYTES;
    }
    const double fu = floor(u), fv = floor(v);
    const int col = (int)fmin(fmax(fu, -4.0), (double)a.pw + 4.0);
    const int row = (int)fmin(fmax(fv, -4.0), (double)a.ph + 4.0);
    const double xc = u - fu, xr = v - fv;
    double my_red[6] = {0, 0, 0, 0, 0, 0};
    for (int j = 0; j < cnt; ++j) {
      const int jc = __shfl_sync(0xffffffffu, col, j);
      const int jr = __shfl_sync(0xffffffffu, row, j);
      const double jxc = __shfl_sync(0xffffffffu, xc, j);
      const double jxr = __shfl_sync(0xffffffffu, xr, j);
      const uint8_t* src = reinterpret_cast<const uint8_t*>((uintptr_t)__shfl_sync(0xffffffffu, (unsigned long long)(uintptr_t)pbase, j));
      GlobalWindow win;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int rr = min(max(jr - 1 + i, 0), a.ph - 1);
        win.rowp[i] = src + (int64_t)rr * a.pw * TAP_BYTES;
        win.coff[i] = min(max(jc - 1 + i, 0), a.pw - 1) * TAP_BYTES;
      }
      double f[CPL], fr[CPL], fc[CPL], r[CPL], red[6];
#pragma unroll
      for (int k = 0; k < CPL; ++k) { f[k] = 0; fr[k] = 0; fc[k] = 0; r[k] = 0; }
      if (active) bicubic_window<T, C, CPL, true, FS>(win, lane, jxc, jxr, f, fr, fc);
      normalize_and_reduce<CPL, true, true>(active, a.l2_normalize != 0, a.refs ? refv : nullptr, f, fr, fc, r, red, lane);
      if (lane == j) {
#pragma unroll
        for (int k = 0; k < 6; ++k) my_red[k] = red[k];
      }
    }
    if (lane < cnt) {
      double rho[3];
      loss_eval(a.loss, 1.0, my_red[0], rho);
      cost += 0.5 * rho[0];
      const double bu = rho[1] * my_red[1], bv = rho[1] * my_red[2];
      const double auu = rho[1] * my_red[3], auv = rho[1] * my_red[4], avv = rho[1] * my_red[5];
      double apu[3], apv[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) { apu[k] = auu * Jp[0][k] + auv * Jp[1][k]; apv[k] = auv * Jp[0][k] + avv * Jp[1][k]; }
      H0 += Jp[0][0] * apu[0] + Jp[1][0] * apv[0];
      H1 += Jp[0][0] * apu[1] + Jp[1][0] * apv[1];
      H2 += Jp[0][0] * apu[2] + Jp[1][0] * apv[2];
      H3 += Jp[0][1] * apu[1] + Jp[1][1] * apv[1];
      H4 += Jp[0][1] * apu[2] + Jp[1][1] * apv[2];
      H5 += Jp[0][2] * apu[2] + Jp[1][2] * apv[2];
      g0 += Jp[0][0] * bu + Jp[1][0] * bv;
      g1 += Jp[0][1] * bu + Jp[1][1] * bv;
      g2 += Jp[0][2] * bu + Jp[1][2] * bv;
    }
  }
  e.cost = warp_sum(cost);
  e.H[0] = warp_sum(H0); e.H[1] = warp_sum(H1); e.H[2] = warp_sum(H2);
  e.H[3] = warp_sum(H3); e.H[4] = warp_sum(H4); e.H[5] = warp_sum(H5);
  e.g[0] = warp_sum(g0); e.g[1] = warp_sum(g1); e.g[2] = warp_sum(g2);
}

template <typename T, int C, bool FS>
__global__ void __launch_bounds__(128) ba_inner_kernel(InnerArgs a) {
  const int64_t p = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (p >= a.n_points || a.point_off[p] < 0) return;
  if (a.pt_begin[p + 1] == a.pt_begin[p]) return;
  // ceres Solver::Options defaults
  const int max_iter = 50, max_invalid = 5;
  const double ftol = 1e-6, gtol = 1e-10, ptol = 1e-8, min_rel_dec = 1e-3;
  const double max_radius = 1e16, min_radius = 1e-32, min_diag = 1e-6, max_diag = 1e32;
  double x[3] = {a.xyz[3 * p], a.xyz[3 * p + 1], a.xyz[3 * p + 2]};
  PointEval cur;
  inner_eval<T, C, FS>(a, p, lane, x, cur);
  if (!isfinite(cur.cost)) return;
  double sc[3];
  sc[0] = 1.0 / (1.0 + sqrt(cur.H[0])); sc[1] = 1.0 / (1.0 + sqrt(cur.H[3])); sc[2] = 1.0 / (1.0 + sqrt(cur.H[5]));
  double radius = 1e4, decrease_factor = 2.0;
  double x_cost = cur.cost, current_cost = cur.cost;
  double x_norm = sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]);
  double gmax = fmax(fabs(cur.g[0]), fmax(fabs(cur.g[1]), fabs(cur.g[2])));
  int num_invalid = 0;
  for (int iter = 1;; ++iter) {
    // FinalizeIterationAndCheckIfMinimizerCanContinue of the previous iteration
    if (iter - 1 >= max_iter) break;
    if (gmax <= gtol) break;
    if (radius < min_radius) break;
    // LM step
    const double diag[3] = {cur.H[0], cur.H[3], cur.H[5]};
    double D2[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double s2 = sc[k] * sc[k];
      D2[k] = fmin(fmax(diag[k] * s2, min_diag), max_diag) / (radius * s2);
    }
    const double Hf[9] = {cur.H[0], cur.H[1], cur.H[2], cur.H[1], cur.H[3], cur.H[4], cur.H[2], cur.H[4], cur.H[5]};
    double inv[9];
    bool valid = inv3_sym(Hf, D2, inv);
    double d[3] = {0, 0, 0}, mcc = 0;
    if (valid) {
#pragma unroll
      for (int k = 0; k < 3; ++k) d[k] = -(inv[k * 3] * cur.g[0] + inv[k * 3 + 1] * cur.g[1] + inv[k * 3 + 2] * cur.g[2]);
      double gd = 0, dHd = 0;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        gd += cur.g[k] * d[k];
        dHd += d[k] * (Hf[k * 3] * d[0] + Hf[k * 3 + 1] * d[1] + Hf[k * 3 + 2] * d[2]);
      }
      mcc = -gd - 0.5 * dHd;
      valid = isfinite(d[0]) && isfinite(d[1]) && isfinite(d[2]) && mcc > 0.0;
    }
    if (!valid) {
      if (++num_invalid >= max_invalid) break;
      radius /= decrease_factor; decrease_factor *= 2.0;
      continue;
    }
    num_invalid = 0;
    const double xc_[3] = {x[0] + d[0], x[1] + d[1], x[2] + d[2]};
    PointEval cand;
    inner_eval<T, C, FS>(a, p, lane, xc_, cand);
    const double candidate_cost = isfinite(cand.cost) ? cand.cost : 1.7976931348623157e308;
    const double step_norm = sqrt((xc_[0] - x[0]) * (xc_[0] - x[0]) + (xc_[1] - x[1]) * (xc_[1] - x[1]) + (xc_[2] - x[2]) * (xc_[2] - x[2]));
    if (step_norm <= ptol * (x_norm + ptol)) break;               // parameter tolerance: step not applied
    const double cost_change = x_cost - candidate_cost;
    if (fabs(cost_change) <= ftol * x_cost) break;                // function tolerance: step not applied
    const double rel = (current_cost - candidate_cost) / mcc;
    if (rel > min_rel_dec) {
      x[0] = xc_[0]; x[1] = xc_[1]; x[2] = xc_[2];
      x_norm = sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]);
      cur = cand; x_cost = cand.cost; current_cost = candidate_cost;
      gmax = fmax(fabs(cur.g[0]), fmax(fabs(cur.g[1]), fabs(cur.g[2])));
      radius = radius / fmax(1.0 / 3.0, 1.0 - pow(2.0 * rel - 1.0, 3.0));
      radius = fmin(max_radius, radius);
      decrease_factor = 2.0;
    } else {
      radius /= decrease_factor; decrease_factor *= 2.0;
    }
  }
  if (lane == 0) { a.xyz[3 * p] = x[0]; a.xyz[3 * p + 1] = x[1]; a.xyz[3 * p + 2] = x[2]; }
}

// ---------------------------------------------------------------------------------------------
// Batched inner iterations: the same per-point Levenberg-Marquardt state machine, but every
// evaluation of ALL still-active points goes through the hot kernels K0 + K1 (TMA-staged; K1
// spreads even a short list over all its warps), and a thread-per-point kernel applies the LM
// logic between passes.  A round is three launches: K0 and K1 over the round's observation list,
// then inner_step_kernel over its point list, which appends the points that stay active and their
// observations to the next round's (double-buffered) lists.  The list lengths never leave the
// device except through a host-mapped slot per round that the host's stop rule reads.
struct InnerState {
  double x[3];        // last accepted point
  double cand[3];     // candidate being evaluated (also written to the parameter set)
  double cost, current_cost, H[6], g[3], sc[3];
  double radius, decf, xnorm, gmax, mcc;
  int iter, invalid, active;
};

struct InnerStepArgs {
  int64_t n_points;
  const int64_t* point_off; const int64_t* pt_begin;
  const double* obs_out; const double* jpt;   // K1's records and K0's d(uv)/dX ([n_obs][6]) of the round's observations
  double* xyz;          // candidate parameter set
  InnerState* st;
  LossParams loss;
  // a round's lists: the step kernel walks the active points plist[0..cnt[1]) of this round (their observations
  // list[0..cnt[0]) were just evaluated) and appends the points that stay active, with their observations, to
  // plist_next / list_next through cnt_next
  const int64_t* plist; const unsigned long long* cnt;
  int64_t* plist_next; int64_t* list_next; unsigned long long* cnt_next;
  unsigned long long* cnt_clear;   // the counters of the round after next: zeroed here (nobody reads them in this round)
  unsigned long long* publish;     // host-mapped [3]: cnt[0], cnt[1], then `epoch` once both are visible
  unsigned long long epoch;
};

__device__ __forceinline__ bool inner_propose(InnerState& s) {
  // ceres Solver::Options defaults (CoordinateDescentMinimizer::Solve)
  const int max_iter = 50, max_invalid = 5;
  const double gtol = 1e-10, min_radius = 1e-32, min_diag = 1e-6, max_diag = 1e32;
  for (;;) {
    s.iter += 1;
    if (s.iter - 1 >= max_iter) return false;
    if (s.gmax <= gtol) return false;
    if (s.radius < min_radius) return false;
    const double diag[3] = {s.H[0], s.H[3], s.H[5]};
    double D2[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double s2 = s.sc[k] * s.sc[k];
      D2[k] = fmin(fmax(diag[k] * s2, min_diag), max_diag) / (s.radius * s2);
    }
    const double Hf[9] = {s.H[0], s.H[1], s.H[2], s.H[1], s.H[3], s.H[4], s.H[2], s.H[4], s.H[5]};
    double inv[9];
    bool valid = inv3_sym(Hf, D2, inv);
    double d[3] = {0, 0, 0}, mcc = 0;
    if (valid) {
#pragma unroll
      for (int k = 0; k < 3; ++k) d[k] = -(inv[k * 3] * s.g[0] + inv[k * 3 + 1] * s.g[1] + inv[k * 3 + 2] * s.g[2]);
      double gd = 0, dHd = 0;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        gd += s.g[k] * d[k];
        dHd += d[k] * (Hf[k * 3] * d[0] + Hf[k * 3 + 1] * d[1] + Hf[k * 3 + 2] * d[2]);
      }
      mcc = -gd - 0.5 * dHd;
      valid = isfinite(d[0]) && isfinite(d[1]) && isfinite(d[2]) && mcc > 0.0;
    }
    if (!valid) {
      if (++s.invalid >= max_invalid) return false;
      s.radius /= s.decf; s.decf *= 2.0;
      continue;
    }
    s.invalid = 0;
    s.mcc = mcc;
#pragma unroll
    for (int k = 0; k < 3; ++k) s.cand[k] = s.x[k] + d[k];
    return true;
  }
}

constexpr int kInnerBatch = 4;   // observation records a step-kernel thread loads ahead of its serial sum

// phase 0: state from the evaluation at the start point; phase 1: judge the evaluated candidate
// returns whether point p stays active (proposes another candidate)
__device__ __forceinline__ bool inner_step_point(const InnerStepArgs& a, int64_t p, int phase) {
  InnerState s = a.st[p];
  if (phase == 0) {
    s.active = (a.point_off[p] >= 0 && a.pt_begin[p + 1] > a.pt_begin[p]) ? 1 : 0;
    s.iter = 0; s.invalid = 0;
    if (!s.active) { a.st[p] = s; return false; }
#pragma unroll
    for (int k = 0; k < 3; ++k) s.x[k] = a.xyz[3 * p + k];
  } else if (!s.active) return false;
  // cost / J^T J / J^T r of this point at the evaluated location, summed serially in observation order.  The records of
  // up to kInnerBatch observations are loaded ahead of the sum, so their loads are in flight together.
  double cost = 0, H[6] = {0, 0, 0, 0, 0, 0}, g[3] = {0, 0, 0};
  const int64_t ob = a.pt_begin[p], oe = a.pt_begin[p + 1];
  for (int64_t o0 = ob; o0 < oe; o0 += kInnerBatch) {
    const int nb = (int)min((int64_t)kInnerBatch, oe - o0);
    double2 rec[kInnerBatch][3], jac[kInnerBatch][3];
#pragma unroll
    for (int b = 0; b < kInnerBatch; ++b) {
      if (b < nb) {
        const double2* oo = reinterpret_cast<const double2*>(a.obs_out + (o0 + b) * 8);
        const double2* jj = reinterpret_cast<const double2*>(a.jpt + (o0 + b) * 6);
#pragma unroll
        for (int k = 0; k < 3; ++k) { rec[b][k] = oo[k]; jac[b][k] = jj[k]; }
      }
    }
#pragma unroll
    for (int b = 0; b < kInnerBatch; ++b) {
      if (b >= nb) break;
      const double oo[6] = {rec[b][0].x, rec[b][0].y, rec[b][1].x, rec[b][1].y, rec[b][2].x, rec[b][2].y};
      double rho[3];
      loss_eval(a.loss, 1.0, oo[0], rho);
      cost += 0.5 * rho[0];
      const double bu = rho[1] * oo[1], bv = rho[1] * oo[2];
      const double auu = rho[1] * oo[3], auv = rho[1] * oo[4], avv = rho[1] * oo[5];
      const double pu[3] = {jac[b][0].x, jac[b][0].y, jac[b][1].x}, pv[3] = {jac[b][1].y, jac[b][2].x, jac[b][2].y};
      double apu[3], apv[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) { apu[k] = auu * pu[k] + auv * pv[k]; apv[k] = auv * pu[k] + avv * pv[k]; }
      H[0] += pu[0] * apu[0] + pv[0] * apv[0];
      H[1] += pu[0] * apu[1] + pv[0] * apv[1];
      H[2] += pu[0] * apu[2] + pv[0] * apv[2];
      H[3] += pu[1] * apu[1] + pv[1] * apv[1];
      H[4] += pu[1] * apu[2] + pv[1] * apv[2];
      H[5] += pu[2] * apu[2] + pv[2] * apv[2];
#pragma unroll
      for (int k = 0; k < 3; ++k) g[k] += pu[k] * bu + pv[k] * bv;
    }
  }
  const double ftol = 1e-6, ptol = 1e-8, min_rel_dec = 1e-3, max_radius = 1e16;
  bool go = true;
  if (phase == 0) {
    if (!isfinite(cost)) go = false;
    s.cost = s.current_cost = cost;
#pragma unroll
    for (int k = 0; k < 6; ++k) s.H[k] = H[k];
#pragma unroll
    for (int k = 0; k < 3; ++k) s.g[k] = g[k];
    s.sc[0] = 1.0 / (1.0 + sqrt(H[0])); s.sc[1] = 1.0 / (1.0 + sqrt(H[3])); s.sc[2] = 1.0 / (1.0 + sqrt(H[5]));
    s.radius = 1e4; s.decf = 2.0;
    s.xnorm = sqrt(s.x[0] * s.x[0] + s.x[1] * s.x[1] + s.x[2] * s.x[2]);
    s.gmax = fmax(fabs(g[0]), fmax(fabs(g[1]), fabs(g[2])));
  } else {
    const double candidate_cost = isfinite(cost) ? cost : 1.7976931348623157e308;
    const double dx = s.cand[0] - s.x[0], dy = s.cand[1] - s.x[1], dz = s.cand[2] - s.x[2];
    const double step_norm = sqrt(dx * dx + dy * dy + dz * dz);
    if (step_norm <= ptol * (s.xnorm + ptol)) go = false;                      // parameter tolerance
    else if (fabs(s.cost - candidate_cost) <= ftol * s.cost) go = false;       // function tolerance
    else {
      const double rel = (s.current_cost - candidate_cost) / s.mcc;
      if (rel > min_rel_dec) {
#pragma unroll
        for (int k = 0; k < 3; ++k) { s.x[k] = s.cand[k]; s.g[k] = g[k]; }
#pragma unroll
        for (int k = 0; k < 6; ++k) s.H[k] = H[k];
        s.xnorm = sqrt(s.x[0] * s.x[0] + s.x[1] * s.x[1] + s.x[2] * s.x[2]);
        s.cost = cost; s.current_cost = candidate_cost;
        s.gmax = fmax(fabs(g[0]), fmax(fabs(g[1]), fabs(g[2])));
        s.radius = s.radius / fmax(1.0 / 3.0, 1.0 - pow(2.0 * rel - 1.0, 3.0));
        s.radius = fmin(max_radius, s.radius);
        s.decf = 2.0;
      } else {
        s.radius /= s.decf; s.decf *= 2.0;
      }
    }
  }
  if (go) go = inner_propose(s);
  if (go) {
#pragma unroll
    for (int k = 0; k < 3; ++k) a.xyz[3 * p + k] = s.cand[k];
  } else {
    s.active = 0;
#pragma unroll
    for (int k = 0; k < 3; ++k) a.xyz[3 * p + k] = s.x[k];
  }
  a.st[p] = s;
  return go;
}

// The next round's lists from one warp: lane i holds point p (when `stays`).  One atomic per counter per warp; the
// warp's points land in lane order, and their observations, each point's in pt_begin order, are written by the whole
// warp with consecutive stores.  Every lane of the warp must call this.
__device__ __forceinline__ void inner_append(const InnerStepArgs& a, bool stays, int64_t p) {
  const int lane = threadIdx.x & 31;
  const unsigned mask = __ballot_sync(0xffffffffu, stays);
  if (!mask) return;
  int64_t ob = 0, no = 0;
  if (stays) { ob = a.pt_begin[p]; no = a.pt_begin[p + 1] - ob; }
  int64_t inc = no;   // inclusive scan of the observation counts over the lanes
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int64_t t = __shfl_up_sync(0xffffffffu, inc, d);
    if (lane >= d) inc += t;
  }
  const int64_t total = __shfl_sync(0xffffffffu, inc, 31), exc = inc - no;
  unsigned long long obase = 0, pbase = 0;
  if (lane == 0) {
    obase = atomicAdd(&a.cnt_next[0], (unsigned long long)total);
    pbase = atomicAdd(&a.cnt_next[1], (unsigned long long)__popc(mask));
  }
  obase = __shfl_sync(0xffffffffu, obase, 0);
  pbase = __shfl_sync(0xffffffffu, pbase, 0);
  if (stays) a.plist_next[pbase + __popc(mask & ((1u << lane) - 1u))] = p;
  for (int64_t j0 = 0; j0 < total; j0 += 32) {
    const int64_t j = j0 + lane;
    int src = 0;   // the last lane whose observations start at or before entry j (lanes with no observations are skipped
#pragma unroll    // over: they share their start with the next lane that has some)
    for (int step = 16; step > 0; step >>= 1)
      if (__shfl_sync(0xffffffffu, exc, src + step) <= j) src += step;
    const int64_t sob = __shfl_sync(0xffffffffu, ob, src), sexc = __shfl_sync(0xffffffffu, exc, src);
    if (j < total) a.list_next[obase + j] = sob + (j - sexc);
  }
}

static __global__ void __launch_bounds__(128) inner_step_kernel(InnerStepArgs a, int phase) {
  const unsigned long long n = a.cnt[1];
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    a.cnt_clear[0] = 0; a.cnt_clear[1] = 0;
    a.publish[0] = a.cnt[0]; a.publish[1] = n;
    __threadfence_system();
    *(volatile unsigned long long*)(a.publish + 2) = a.epoch;
  }
  // warp-uniform trip count: the whole warp takes part in inner_append
  const uint64_t lane = threadIdx.x & 31;
  for (uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x - lane; w < n; w += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t i = w + lane;
    int64_t p = -1;
    bool stays = false;
    if (i < n) { p = a.plist[i]; stays = inner_step_point(a, p, phase); }
    inner_append(a, stays, p);
  }
}

// round 0's lists: every variable point with observations, and those observations
static __global__ void __launch_bounds__(128) inner_list_kernel(InnerStepArgs a) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const bool listed = p < a.n_points && a.point_off[p] >= 0 && a.pt_begin[p + 1] > a.pt_begin[p];
  inner_append(a, listed, p);
}

// ||a - b|| over two parameter sets (ambient), for step_norm after inner iterations
static __global__ void __launch_bounds__(256) diff_norm_kernel(const double* a, const double* b, int64_t n, double* acc, double* part = nullptr) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  double v = 0.0;
  if (i < n) { const double d = a[i] - b[i]; v = d * d; }
  __shared__ double sh[8];
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0; for (int k = 0; k < 8; ++k) s += sh[k];
    if (part) part[blockIdx.x] = s;          // deterministic mode (det_reduce_add_kernel)
    else atomicAdd(acc, s);
  }
}

// multi-GPU: S += lower(Hcc) + diag(D2c), rhs += -gc after the allreduce of the Schur parts
static __global__ void ba_add_reduced_kernel(const double* Hcc, const double* gc, const double* D2, double* S,
                                      double* rhs, int nc) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t n2 = (int64_t)nc * nc;
  if (i < n2) {
    const int r = (int)(i / nc), c = (int)(i % nc);
    double v = c <= r ? Hcc[i] : 0.0;
    if (r == c) v += D2[r];
    S[i] += v;
  }
  if (i < nc) rhs[i] -= gc[i];
}

}  // namespace pxr
