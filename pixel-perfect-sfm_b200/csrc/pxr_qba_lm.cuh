// pxr_qba_lm.cuh — the Levenberg-Marquardt loop of one query's pose solve, run by one CTA: query bundle adjustment
// (pxr_qba.cu, featuremetric residuals) and the pose refinement of absolute pose estimation (pxr_pnp.cu, reprojection
// residuals) share it.  The residual evaluation is the caller's policy: a functor
//   double evaluate(const double* prm, int model, uint32_t mask, int n, double* H, double* g)
// that the whole CTA calls at the parameters prm = [cam params (kMaxK) | qvec | tvec] and that fills H (packed lower
// triangle of J^T J) and g (J^T r) in the query's n tangent columns (3 rotation, 3 translation, the free intrinsics in
// parameter order) and returns the cost, identical on every thread.
#pragma once
#include "pxr_device.cuh"
#include "pxr_internal.h"
#include "pxr_lm.cuh"

namespace pxr {

constexpr int kQThreads = 256;
constexpr int kQWarps = kQThreads / 32;
constexpr int kQMaxN = 6 + kMaxK;                       // tangent columns of one query
constexpr int kQTri = kQMaxN * (kQMaxN + 1) / 2;
constexpr int kQPart = kQTri + kQMaxN + 1;              // one warp's partial: J^T J (lower), J^T r, cost
constexpr int kQParams = kMaxK + 7;                     // cam params | qvec | tvec
constexpr int kQEntries = (kQTri + kQMaxN + 31) / 32;   // J^T J / J^T r entries per lane

struct QBAArgs {
  int n_queries;
  const int64_t* obs_begin;            // [nq+1] wave-local
  const int32_t* cam_model; const uint32_t* cam_mask;
  double* params;                      // [nq][kQParams] in/out
  const uint64_t* patch;               // [nq] address of the query's patch block
  const int64_t* patch_first;          // [nq] the query's first row of corner / scale
  const double* xyz; const int64_t* obs_patch; const double* refs;
  const int32_t* corner; const double* scale; double ups; int ph, pw;
  LossParams loss; int l2_normalize;
  int max_iter, max_invalid, max_nonmonotonic, jacobi_scaling;
  double ftol, gtol, ptol, min_rel_dec, radius0, max_radius, min_radius, min_diag, max_diag;
  int row_stride;                      // doubles per projected-block row in shared memory
  pxr_qba_result* results;             // [nq]
  pxr_iteration_summary* iters; int iter_cap;   // [nq][iter_cap] or null
  int linearize_only;                  // pxr_qba_debug_linearize: evaluate once and report
  double* dbg_cost; double* dbg_H; double* dbg_g; double* dbg_xy; double* dbg_rec;
};

__device__ __forceinline__ int qtri(int i, int j) { return i * (i + 1) / 2 + j; }   // i >= j

// ceres' gradient_max_norm = || x - Plus(x, -g) ||_inf, as ba_gradmax_kernel forms it for one image and its camera
static __device__ double qba_gradmax(const double* g, const double* qv, int n) {
  const double ng[3] = {-g[0], -g[1], -g[2]};
  double qn[4];
  quaternion_plus(qv, ng, qn);
  double m = 0.0;
  for (int k = 0; k < 4; ++k) m = fmax(m, fabs(qv[k] - qn[k]));
  for (int k = 3; k < n; ++k) m = fmax(m, fabs(g[k]));
  return m;
}

enum { QA_STOP = 0, QA_SKIP = 1, QA_EVAL = 2 };

// BA::lm_begin / lm_iterate (pxr_ba.cu) for one free image over the residual blocks [ob, ob + ...) of query q; the
// constant points' ||X||^2 (part of ceres' ||x||) is taken from a.xyz[ob, oe).  Writes a.params[q] (the lowest-cost
// iterate) and a.results[q].
template <class Eval>
__device__ __forceinline__ void qba_lm_solve(const QBAArgs& a, const int q, const int64_t ob, const int64_t oe,
                                             const Eval& evaluate) {
  __shared__ double sH[2][kQTri], sg[2][kQMaxN], sx[3][kQParams];   // parameters: 0 current, 1 candidate, 2 best
  __shared__ int sctl[2];                                           // action, current linearisation set
  const int tid = threadIdx.x;
  pxr_qba_result* res = a.results + q;
  auto report = [&](int status, double c0, double c1, int term, int64_t evals) {
    res->status = status; res->num_residual_blocks = (int32_t)(oe - ob);
    res->initial_cost = c0; res->final_cost = c1; res->num_iterations = 0;
    res->num_successful_steps = 0; res->num_unsuccessful_steps = 0; res->termination_type = term;
    res->block_evaluations = evals;
  };
  if (oe <= ob) {      // not solved (QueryBundleOptimizer::SolveProblem returns false): parameters untouched
    if (tid == 0) report(PXR_OK, 0.0, 0.0, 1, 0);
    return;
  }
  const int model = a.cam_model[q];
  const int Kc = cam_num_params(model);
  const uint32_t mask = a.cam_mask[q];
  int n = 6;
  for (int k = 0; k < Kc; ++k) n += ((mask >> k) & 1u) ? 0 : 1;
  for (int i = tid; i < kQParams; i += kQThreads) sx[0][i] = a.params[(int64_t)q * kQParams + i];
  __syncthreads();
  double x_cost = evaluate(sx[0], model, mask, n, sH[0], sg[0]);
  int64_t evals = oe - ob;
  if (a.linearize_only) {
    const int ntri = n * (n + 1) / 2;
    if (tid == 0 && a.dbg_cost) a.dbg_cost[q] = x_cost;
    if (a.dbg_H)
      for (int k = tid; k < kQMaxN * kQMaxN; k += kQThreads) {
        const int i = k / kQMaxN, j = k % kQMaxN;
        a.dbg_H[(int64_t)q * kQMaxN * kQMaxN + k] = (i < n && j <= i) ? sH[0][qtri(i, j)] : 0.0;
      }
    if (a.dbg_g)
      for (int k = tid; k < kQMaxN; k += kQThreads) a.dbg_g[(int64_t)q * kQMaxN + k] = k < n ? sg[0][k] : 0.0;
    (void)ntri;
    return;
  }
  if (!isfinite(x_cost)) {     // BA::lm_begin: "initial cost is not finite"
    if (tid == 0) report(PXR_ERR_NUMERIC, x_cost, x_cost, 2, evals);
    return;
  }
  // ---- LM state: thread 0 takes every scalar decision, the CTA evaluates
  __shared__ double sL[kQTri], sd[kQMaxN], sscale[kQMaxN];
  const double initial_cost = x_cost;
  double min_cost = x_cost, mcc = 0.0, step_norm = 0.0, x_norm = 0.0, prev_gmax = 0.0;
  int n_succ = 0, n_unsucc = 0, term = 1, n_its = 0, cur = 0;
  bool pending = true, best_is_current = true;
  pxr_iteration_summary it = pxr_iteration_summary();
  TrustRegion tr;
  double xn_points = 0.0;     // ||X||^2 of the constant points: part of ceres' ||x|| (ba_plus_kernel)
  if (tid == 0) {
    for (int i = 0; i < n; ++i) sscale[i] = a.jacobi_scaling ? jacobi_scale(sH[0][qtri(i, i)]) : 1.0;
    for (int64_t o = ob; o < oe; ++o)
      for (int k = 0; k < 3; ++k) { const double x = a.xyz[3 * o + k]; xn_points += x * x; }
    it.cost = x_cost;
    it.gradient_max_norm = qba_gradmax(sg[0], sx[0] + kMaxK, n);
    tr.init({a.max_invalid, a.max_nonmonotonic, a.radius0, a.max_radius, a.min_radius, a.gtol, a.ptol, a.ftol, a.min_rel_dec},
            x_cost);
  }
  while (true) {
    if (tid == 0) {
      int action = QA_EVAL;
      // FinalizeIterationAndCheckIfMinimizerCanContinue (BA::lm_finalize)
      if (pending) {
        if (it.step_is_successful) { ++n_succ; if (x_cost < min_cost) min_cost = x_cost; }
        else if (it.iteration > 0) ++n_unsucc;
        it.trust_region_radius = tr.radius;
        if (a.iters && n_its < a.iter_cap) a.iters[(int64_t)q * a.iter_cap + n_its] = it;
        ++n_its;
        pending = false;
      }
      if (const int stop = tr.stop(it.iteration, a.max_iter, it.gradient_max_norm)) {
        term = stop == TR_MAX_ITERATIONS ? 1 : 0;
        action = QA_STOP;
      }
      if (action != QA_STOP) {
        prev_gmax = it.gradient_max_norm;
        const int iteration = it.iteration + 1;
        it = pxr_iteration_summary();
        it.iteration = iteration;
        pending = true;
        // ---- LM step: (H + D) delta = -g, D = lm_damping of diag(H)
        const double* H = sH[cur];
        const double* g = sg[cur];
        double* L = sL;
        double* d = sd;
        for (int i = 0; i < n * (n + 1) / 2; ++i) L[i] = H[i];
        for (int i = 0; i < n; ++i) L[qtri(i, i)] += lm_damping(H[qtri(i, i)], sscale[i], tr.radius, a.min_diag, a.max_diag);
        bool ok = true;
        for (int j = 0; j < n && ok; ++j) {
          double djj = L[qtri(j, j)];
          for (int k = 0; k < j; ++k) djj -= L[qtri(j, k)] * L[qtri(j, k)];
          if (!(djj > 0.0) || !isfinite(djj)) { ok = false; break; }
          const double ljj = sqrt(djj);
          L[qtri(j, j)] = ljj;
          for (int i = j + 1; i < n; ++i) {
            double v = L[qtri(i, j)];
            for (int k = 0; k < j; ++k) v -= L[qtri(i, k)] * L[qtri(j, k)];
            L[qtri(i, j)] = v / ljj;
          }
        }
        double acc = 0.0;
        if (ok) {
          for (int i = 0; i < n; ++i) {
            double v = -g[i];
            for (int k = 0; k < i; ++k) v -= L[qtri(i, k)] * d[k];
            d[i] = v / L[qtri(i, i)];
          }
          for (int i = n - 1; i >= 0; --i) {
            double v = d[i];
            for (int k = i + 1; k < n; ++k) v -= L[qtri(k, i)] * d[k];
            d[i] = v / L[qtri(i, i)];
          }
          // model cost change = -(g.d + d^T H d / 2): ba_model_cost_kernel's sum over the blocks, in closed form
          for (int i = 0; i < n; ++i) {
            double hd = 0.0;
            for (int j = 0; j < n; ++j) hd += (i >= j ? H[qtri(i, j)] : H[qtri(j, i)]) * d[j];
            acc += g[i] * d[i] + 0.5 * d[i] * hd;
          }
        }
        mcc = -acc;
        const bool valid = ok && isfinite(acc) && mcc > 0.0;
        it.linear_solver_iterations = 1;
        it.step_is_valid = valid;
        if (!valid) {
          if (tr.invalid_step()) { term = 2; action = QA_STOP; }
          else {
            it.cost = x_cost; it.gradient_max_norm = prev_gmax;
            action = QA_SKIP;
          }
        } else {
          tr.num_invalid = 0;
          // ---- candidate = Plus(x, delta) and the norms ba_plus_kernel forms (this image and its camera)
          const double* x = sx[0];
          double* xc = sx[1];
          const double* qv = x + kMaxK;
          const double* tv = x + kMaxK + 4;
          double qn[4], dnc = 0.0, xnc = 0.0;
          quaternion_plus(qv, d, qn);
          for (int k = 0; k < 3; ++k) { const double tp = tv[k] + d[3 + k]; xc[kMaxK + 4 + k] = tp; dnc += (tp - tv[k]) * (tp - tv[k]); }
          for (int k = 0; k < 4; ++k) { xc[kMaxK + k] = qn[k]; dnc += (qn[k] - qv[k]) * (qn[k] - qv[k]); xnc += qv[k] * qv[k]; }
          for (int k = 0; k < 3; ++k) xnc += tv[k] * tv[k];
          int la = 6;
          for (int k = 0; k < kMaxK; ++k) {
            const double c0 = x[k];
            double cpv = c0;
            if (k < Kc && !((mask >> k) & 1u)) cpv += d[la++];
            xc[k] = cpv;
            dnc += (cpv - c0) * (cpv - c0);
            if (k < Kc) xnc += c0 * c0;
          }
          step_norm = sqrt(dnc);
          x_norm = sqrt(xn_points + xnc);
        }
      }
      sctl[0] = action; sctl[1] = cur;
    }
    __syncthreads();
    const int action = sctl[0], set = sctl[1];
    __syncthreads();
    if (action == QA_STOP) break;
    if (action == QA_SKIP) continue;
    // trial point, evaluated with the Jacobian: when accepted it is the next linearisation (BA's speculative pass)
    double candidate_cost = evaluate(sx[1], model, mask, n, sH[1 - set], sg[1 - set]);
    evals += oe - ob;
    if (tid == 0) {
      int act = QA_EVAL;
      if (!isfinite(candidate_cost)) candidate_cost = 1.7976931348623157e308;
      it.step_norm = step_norm;
      it.cost_change = x_cost - candidate_cost;
      if (tr.tolerance(step_norm, x_norm, it.cost_change, x_cost)) { term = 0; act = QA_STOP; }   // step not applied
      else {
        it.relative_decrease = tr.ev.quality(candidate_cost, mcc);
        if (tr.successful(it.relative_decrease)) {
          if (a.max_nonmonotonic > 0 && !(candidate_cost < min_cost) && best_is_current) {
            for (int i = 0; i < kQParams; ++i) sx[2][i] = sx[0][i];    // leaving the best iterate: keep it
            best_is_current = false;
          } else if (a.max_nonmonotonic > 0 && candidate_cost < min_cost) {
            best_is_current = true;
          }
          for (int i = 0; i < kQParams; ++i) sx[0][i] = sx[1][i];
          cur = 1 - cur;
          x_cost = candidate_cost;
          it.cost = x_cost;
          it.gradient_max_norm = qba_gradmax(sg[cur], sx[0] + kMaxK, n);
          it.step_is_successful = 1;
          tr.accept(it.relative_decrease, candidate_cost, mcc);
        } else {
          it.step_is_successful = 0;
          it.cost = candidate_cost;
          it.gradient_max_norm = prev_gmax;
          tr.reject();
        }
      }
      sctl[0] = act;
    }
    __syncthreads();
    const int act = sctl[0];
    __syncthreads();
    if (act == QA_STOP) break;
  }
  if (tid == 0) {
    if (x_cost < min_cost) min_cost = x_cost;
    const double* out = (a.max_nonmonotonic > 0 && !best_is_current) ? sx[2] : sx[0];
    for (int i = 0; i < kQParams; ++i) a.params[(int64_t)q * kQParams + i] = out[i];
    res->status = PXR_OK;
    res->num_residual_blocks = (int32_t)(oe - ob);
    res->initial_cost = initial_cost;
    res->final_cost = min_cost;
    res->num_iterations = n_its;
    res->num_successful_steps = n_succ;
    res->num_unsuccessful_steps = n_unsucc;
    res->termination_type = term;
    res->block_evaluations = evals;
  }
}

}  // namespace pxr
