// pxr_inner.cuh — inner iterations: each 3D point solved with everything else fixed.
//
// Replaces ceres' CoordinateDescentMinimizer (enabled by the reference through
// use_inner_iterations=True, pixsfm/bundle_adjustment/main.py:41-44 and
// bundle_optimizer.h:131-134,350-355: all non-constant points form independent set 0).  Each
// point runs a Levenberg-Marquardt loop with Ceres' default Solver::Options; its rules and those
// options are pxr_lm.cuh's (inner_options, inner_start / inner_judge / inner_propose).
// Every inner evaluation re-reads the point's feature windows.  On a large problem they are not
// L2-resident (at BASELINE configs[2] one pass over all observations touches about 2 GB of windows
// against a 50 MB L2), so the first rounds stream them from HBM like any full K1 pass; only the
// short lists of the late rounds fit in L2.
#pragma once
#include "pxr_ba_kernels.cuh"
#include "pxr_fm_eval.cuh"
#include "pxr_lm.cuh"

namespace pxr {

// ---------------------------------------------------------------------------------------------
// Batched inner iterations: every evaluation of ALL still-active points goes through the hot
// kernels K0 + K1 (TMA-staged; K1 spreads even a short list over all its warps), and a
// thread-per-point kernel applies the LM logic between passes.  A round is three launches: K0 and K1 over the round's observation list,
// then inner_step_kernel over its point list, which appends the points that stay active and their
// observations to the next round's (double-buffered) lists.  The list lengths never leave the
// device except through a host-mapped slot per round that the host's stop rule reads.
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

constexpr int kInnerBatch = 4;   // observation records a step-kernel thread loads ahead of its serial sum

// The GPU side of one point's step between evaluations (the rules are pxr_lm.cuh's inner_start / inner_judge /
// inner_propose).  phase 0: state from the evaluation at the start point; phase 1: judge the evaluated candidate.
// Returns whether point p stays active (proposes another candidate).
__device__ __forceinline__ bool inner_step_point(const InnerStepArgs& a, int64_t p, int phase) {
  InnerState s = a.st[p];
  if (phase == 0) {
    s.active = (a.point_off[p] >= 0 && a.pt_begin[p + 1] > a.pt_begin[p]) ? 1 : 0;
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
  bool go = phase == 0 ? inner_start(s, cost, H, g) : inner_judge(s, cost, H, g) == TR_CONTINUE;
  if (go) go = inner_propose(s) == TR_CONTINUE;
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
