// pxr_qba.cu — batched query bundle adjustment: many localization queries refined in one launch.
//
// Replaces a loop of _localization.QueryBundleOptimizer.run (reference localization/src/single_query_bundle_optimizer.h,
// query_bundle_optimizer.h): per query one image pose (QuaternionManifold rotation + translation) and optionally some
// intrinsics, against constant 3D points and fixed reference descriptors.  pxr_ba_run solves such a query with a whole
// BA handle and a host-driven LM loop; here one CTA carries a query's whole solve:
//   evaluation  per residual block world_to_pixel<true> + ToPixelCoordinates (K0's arithmetic), the clamped 4x4 tap window
//               read from global memory, K1's bicubic pass, L2 normalisation and r = f - ref with the butterfly order of
//               K1 (so the record (||r||^2, G^T r, G^T G) is K1's), scaled by rho' and accumulated into J^T J / J^T r
//               per warp; the warps' partials are summed in warp order, so a query's bits never depend on its neighbours
//   LM          BA::lm_begin / lm_iterate (pxr_ba.cu) for one free image, no free points, no inner iterations: Jacobi
//               scaling from iteration zero, clamped LM diagonal, invalid steps, parameter / function / gradient
//               tolerances, step quality and radius update through the trust-region rules of pxr_lm.cuh, with
//               use_nonmonotonic_steps, the lowest-cost iterate written back and the termination types of lm_finalize
//   solve       exact dense Cholesky of the damped n x n system (n = 6 + free intrinsics <= 18), one thread
// The host packs consecutive queries into waves that fit a byte budget; one wave is one launch, and the next wave's
// upload is enqueued before the host waits for the current one.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "pxr_fm_eval.cuh"
#include "pxr_qba_lm.cuh"
#include "pxr_waves.h"

namespace pxr {

int fm_supported(int dtype, int C);


// Linearisation of one query at prm (whole CTA): H (packed lower) and g in the query's tangent columns; returns the cost.
// Each warp takes batches of 32 blocks: every lane projects one block into its shared row [u, v, x, y, Ju(n), Jv(n)],
// then the warp evaluates the batch one block at a time, one channel group per lane.
template <typename T, int C, bool FS>
__device__ double qba_evaluate(const QBAArgs& a, int q, const double* prm, int model, uint32_t mask, int n, double* H,
                               double* g, double* rows, double* part, int64_t ob, int64_t oe) {
  constexpr int CPL = C >= 32 ? C / 32 : 1;
  constexpr int ACTIVE = C / CPL;
  constexpr int TAP_BYTES = C * (int)sizeof(T);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool active = lane < ACTIVE;
  const int RS = a.row_stride;
  double* wrow = rows + (size_t)warp * 32 * RS;
  const int ntri = n * (n + 1) / 2, nent = ntri + n;
  int ea[kQEntries], eb[kQEntries];    // this lane's entries k = lane + 32 i: H(ea, eb), or g(ea) when eb < 0
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
  const uint8_t* pbase = reinterpret_cast<const uint8_t*>(a.patch[q]);
  const int64_t patch_bytes = (int64_t)a.ph * a.pw * TAP_BYTES;
  const int64_t pf = a.patch_first[q];
  for (int64_t b0 = ob + (int64_t)warp * 32; b0 < oe; b0 += kQWarps * 32) {
    __syncwarp();
    const int64_t o = b0 + lane;
    if (o < oe) {
      double X[3], xy[2], Jpose[2][6], Jpt[2][3], Jk[2][kMaxK];
#pragma unroll
      for (int k = 0; k < 3; ++k) X[k] = a.xyz[3 * o + k];
      world_to_pixel<true>(model, prm, prm + kMaxK, prm + kMaxK + 4, X, xy, Jpose, Jpt, Jk);
      const int64_t pi = pf + a.obs_patch[o];
      const double sx = a.scale[2 * pi], sy = a.scale[2 * pi + 1];
      const double cx = (double)a.corner[2 * pi], cy = (double)a.corner[2 * pi + 1];
      double* r = wrow + lane * RS;
      r[0] = (xy[0] * sx - 0.5 - cx) * a.ups;
      r[1] = (xy[1] * sy - 0.5 - cy) * a.ups;
      r[2] = xy[0]; r[3] = xy[1];
      const double s0 = sx * a.ups, s1 = sy * a.ups;
#pragma unroll
      for (int k = 0; k < 6; ++k) { r[4 + k] = s0 * Jpose[0][k]; r[4 + n + k] = s1 * Jpose[1][k]; }
      int c = 6;
#pragma unroll
      for (int k = 0; k < kMaxK; ++k)
        if (k < Kc && !((mask >> k) & 1u)) { r[4 + c] = s0 * Jk[0][k]; r[4 + n + c] = s1 * Jk[1][k]; ++c; }
    }
    __syncwarp();
    const int nb = (int)min((int64_t)32, oe - b0);
    for (int j = 0; j < nb; ++j) {
      const double* r = wrow + j * RS;
      const int64_t oj = b0 + j;
      const double u = r[0], v = r[1];
      const double fu = floor(u), fv = floor(v);
      const int col = (int)fmin(fmax(fu, -4.0), (double)a.pw + 4.0);   // as K1: NaN / far projections clamp to the border
      const int row = (int)fmin(fmax(fv, -4.0), (double)a.ph + 4.0);
      const uint8_t* src = pbase + a.obs_patch[oj] * patch_bytes;
      GlobalWindow w;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        w.rowp[i] = src + (int64_t)min(max(row - 1 + i, 0), a.ph - 1) * a.pw * TAP_BYTES;
        w.coff[i] = min(max(col - 1 + i, 0), a.pw - 1) * TAP_BYTES;
      }
      double f[CPL], fr[CPL], fc[CPL], res[CPL], red[6];
#pragma unroll
      for (int k = 0; k < CPL; ++k) { f[k] = 0.0; fr[k] = 0.0; fc[k] = 0.0; res[k] = 0.0; }
      if (active) bicubic_window<T, C, CPL, true, FS>(w, lane, u - fu, v - fv, f, fr, fc);
      normalize_and_reduce<CPL, true, true>(active, a.l2_normalize != 0, a.refs + oj * C + lane * CPL, f, fr, fc, res, red,
                                            lane);
      double rho[3];
      loss_eval(a.loss, 1.0, red[0], rho);
      cost += 0.5 * rho[0];
      const double bu = rho[1] * red[1], bv = rho[1] * red[2];
      const double auu = rho[1] * red[3], auv = rho[1] * red[4], avv = rho[1] * red[5];
      const double* Ju = r + 4;
      const double* Jv = r + 4 + n;
#pragma unroll
      for (int i = 0; i < kQEntries; ++i) {
        const int ia = ea[i], ib = eb[i];
        if (ia < 0) continue;
        if (ib >= 0) {      // ba_build_kernel's camera block term
          const double aju = auu * Ju[ia] + auv * Jv[ia], ajv = auv * Ju[ia] + avv * Jv[ia];
          acc[i] += Ju[ib] * aju + Jv[ib] * ajv;
        } else {
          acc[i] += Ju[ia] * bu + Jv[ia] * bv;
        }
      }
      if (a.linearize_only && lane == 0) {
        if (a.dbg_rec) {
          double* rec = a.dbg_rec + oj * 8;
          for (int k = 0; k < 6; ++k) rec[k] = red[k];
          rec[6] = 0.0; rec[7] = 0.0;
        }
        if (a.dbg_xy) { a.dbg_xy[2 * oj] = r[2]; a.dbg_xy[2 * oj + 1] = r[3]; }
      }
    }
  }
  double* mine = part + warp * kQPart;
#pragma unroll
  for (int i = 0; i < kQEntries; ++i)
    if (ea[i] >= 0) mine[lane + 32 * i] = acc[i];
  if (lane == 0) mine[nent] = cost;
  __syncthreads();
  for (int k = threadIdx.x; k <= nent; k += kQThreads) {   // fixed order over the warps
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

template <typename T, int C, bool FS>
__global__ void __launch_bounds__(kQThreads) qba_solve_kernel(QBAArgs a) {
  extern __shared__ __align__(16) double qrows[];
  __shared__ double spart[kQWarps * kQPart + 1];
  const int q = blockIdx.x;
  if (q >= a.n_queries) return;
  const int64_t ob = a.obs_begin[q], oe = a.obs_begin[q + 1];
  qba_lm_solve(a, q, ob, oe, [&](const double* prm, int model, uint32_t mask, int n, double* H, double* g) {
    return qba_evaluate<T, C, FS>(a, q, prm, model, mask, n, H, g, qrows, spart, ob, oe);
  });
}

template <typename T, int C, bool FS>
static int launch_qba_t(pxr_ctx* ctx, const QBAArgs& a, size_t smem) {
  PXR_CUDA(cudaFuncSetAttribute(qba_solve_kernel<T, C, FS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  PXR_LAUNCH(ctx, (qba_solve_kernel<T, C, FS>), a.n_queries, kQThreads, smem, a);
  PXR_CUDA(cudaGetLastError());
  return PXR_OK;
}

static int launch_qba(pxr_ctx* ctx, int dtype, int C, bool fs, const QBAArgs& a, size_t smem) {
#define PXR_QBA_CASE(T, CC) \
  if (C == CC) return fs ? launch_qba_t<T, CC, true>(ctx, a, smem) : launch_qba_t<T, CC, false>(ctx, a, smem);
  if (dtype == PXR_F16) {
    PXR_QBA_CASE(__half, 128) PXR_QBA_CASE(__half, 64) PXR_QBA_CASE(__half, 32) PXR_QBA_CASE(__half, 16)
    PXR_QBA_CASE(__half, 8) PXR_QBA_CASE(__half, 256)
  } else if (dtype == PXR_F32) {
    PXR_QBA_CASE(float, 128) PXR_QBA_CASE(float, 64) PXR_QBA_CASE(float, 16)
  } else if (dtype == PXR_F64) {
    PXR_QBA_CASE(double, 128) PXR_QBA_CASE(double, 16)
  }
#undef PXR_QBA_CASE
  return fail(PXR_ERR_UNSUPPORTED, "Unsupported dimensions (CHANNELS,N_NODES).");
}

// ---- host side --------------------------------------------------------------------------------------------------
constexpr double kQueryStateBytes = kQParams * 8 + 8 + 8 + 8 + 4 + 4;   // params, obs_begin, patch address, first row, model, mask

static int check_qba(const pxr_qba_desc* d, const pxr_interp_config* ic, const pxr_solver_options* so) {
  if (!d) return fail(PXR_ERR_INVALID_ARGUMENT, "desc is NULL");
  if (d->n_queries < 0) return fail(PXR_ERR_INVALID_ARGUMENT, "n_queries < 0");
  if (d->n_queries > 0 && (!d->cam_model || !d->cam_params || !d->cam_const_mask || !d->qvec || !d->tvec ||
                           !d->obs_begin || !d->patch_blocks || !d->patch_counts))
    return fail(PXR_ERR_INVALID_ARGUMENT, "a required array is NULL");
  if (so && so->use_inner_iterations)
    return fail(PXR_ERR_INVALID_ARGUMENT, "query bundle adjustment has no free points: use_inner_iterations must be 0");
  if (so && so->linear_solver == PXR_SOLVER_ITERATIVE_SCHUR)
    return fail(PXR_ERR_UNSUPPORTED, "ITERATIVE_SCHUR is not supported for query bundle adjustment (exact dense solve)");
  if (ic && ic->check_bounds) return fail(PXR_ERR_UNSUPPORTED, "check_bounds=true is not supported on this path");
  if (d->channels < 8 || !fm_supported(d->patch_dtype, d->channels))
    return fail(PXR_ERR_UNSUPPORTED, "Unsupported dimensions (CHANNELS,N_NODES).");
  if (d->ph < 1 || d->pw < 1) return fail(PXR_ERR_INVALID_ARGUMENT, "bad patch size");
  if (!(d->upsampling_factor > 0.0)) return fail(PXR_ERR_INVALID_ARGUMENT, "upsampling_factor must be > 0");
  if (d->n_queries == 0) return PXR_OK;
  if (d->obs_begin[0] != 0) return fail(PXR_ERR_INVALID_ARGUMENT, "obs_begin[0] must be 0");
  int64_t n_patches = 0;
  for (int q = 0; q < d->n_queries; ++q) {
    if (d->obs_begin[q + 1] < d->obs_begin[q]) return fail(PXR_ERR_INVALID_ARGUMENT, "obs_begin must be non-decreasing");
    if (cam_num_params(d->cam_model[q]) == 0) return fail(PXR_ERR_UNSUPPORTED, "unsupported camera model id %d", d->cam_model[q]);
    if (d->patch_counts[q] < 0) return fail(PXR_ERR_INVALID_ARGUMENT, "patch_counts[%d] < 0", q);
    if (d->patch_counts[q] > 0 && !d->patch_blocks[q]) return fail(PXR_ERR_INVALID_ARGUMENT, "patch block %d is NULL", q);
    n_patches += d->patch_counts[q];
  }
  const int64_t n_obs = d->obs_begin[d->n_queries];
  if (n_obs > 0 && (!d->xyz || !d->obs_patch || !d->refs)) return fail(PXR_ERR_INVALID_ARGUMENT, "a required array is NULL");
  if (n_patches > 0 && (!d->corner || !d->scale)) return fail(PXR_ERR_INVALID_ARGUMENT, "a required array is NULL");
  for (int q = 0; q < d->n_queries; ++q)
    for (int64_t o = d->obs_begin[q]; o < d->obs_begin[q + 1]; ++o)
      if (d->obs_patch[o] < 0 || d->obs_patch[o] >= d->patch_counts[q])
        return fail(PXR_ERR_INVALID_ARGUMENT, "obs_patch[%lld] is not a patch of query %d", (long long)o, q);
  return PXR_OK;
}

static int qba_args(pxr_ctx* ctx, const pxr_qba_desc* d, const pxr_interp_config* ic, const pxr_solver_options* so) {
  PXR_TRY(check_qba(d, ic, so));
  return require_ctx(ctx);
}

static double query_bytes(const pxr_qba_desc* d, int q, bool host_patch) {
  const double patch = (double)d->ph * d->pw * d->channels * dtype_bytes(d->patch_dtype);
  const double m = (double)(d->obs_begin[q + 1] - d->obs_begin[q]);
  return (host_patch ? d->patch_counts[q] * patch : 0.0) + m * (d->channels * 8.0 + 24.0 + 8.0) +
         d->patch_counts[q] * 16.0 + kQueryStateBytes;
}

static void plan_waves(const pxr_qba_desc* d, double budget, WavePlan* p) {
  plan_waves(d->n_queries, d->patch_blocks, d->patch_counts, 8.0 /* obs_begin's closing entry */, budget,
             [d](int q, bool host_patch) { return query_bytes(d, q, host_patch); }, p);
}

// Device memory of one wave: [host patch blocks | refs | xyz | obs_patch | corner | scale | per-query state]
struct WaveBufs {
  DevBuf<uint8_t> arena;
  DevBuf<pxr_qba_result> results;
  DevBuf<pxr_iteration_summary> iters;
  std::vector<uint8_t> state;       // host staging of the per-query state
};
struct WaveView {
  int q0, nq; int64_t o0, no, p0, np;
  size_t off_refs, off_xyz, off_op, off_corner, off_scale, off_params, off_ob, off_ptr, off_pf, off_model, off_mask, end;
};

static WaveView wave_view(const pxr_qba_desc* d, const WavePlan& p, int w) {
  WaveView v;
  v.q0 = p.begin[w]; v.nq = p.begin[w + 1] - v.q0;
  v.o0 = d->obs_begin[v.q0]; v.no = d->obs_begin[v.q0 + v.nq] - v.o0;
  v.p0 = 0; for (int q = 0; q < v.q0; ++q) v.p0 += d->patch_counts[q];
  v.np = 0; for (int q = v.q0; q < v.q0 + v.nq; ++q) v.np += d->patch_counts[q];
  const size_t patch = (size_t)d->ph * d->pw * d->channels * dtype_bytes(d->patch_dtype);
  size_t off = 0;
  for (int q = v.q0; q < v.q0 + v.nq; ++q) if (p.host_patch[q]) off += (size_t)d->patch_counts[q] * patch;
  v.off_refs = off; off += (size_t)v.no * d->channels * 8;
  v.off_xyz = off; off += (size_t)v.no * 24;
  v.off_op = off; off += (size_t)v.no * 8;
  v.off_corner = off; off += (size_t)v.np * 8;
  v.off_scale = off; off += (size_t)v.np * 16;
  v.off_params = off; off += (size_t)v.nq * kQParams * 8;
  v.off_ob = off; off += (size_t)(v.nq + 1) * 8;
  v.off_ptr = off; off += (size_t)v.nq * 8;
  v.off_pf = off; off += (size_t)v.nq * 8;
  v.off_model = off; off += (size_t)v.nq * 4;
  v.off_mask = off; off += (size_t)v.nq * 4;
  v.end = off;
  return v;
}

// enqueue the upload of wave v into `b` on `stream`
static int upload_wave(pxr_ctx* ctx, const pxr_qba_desc* d, const WavePlan& p, const WaveView& v, WaveBufs& b,
                       cudaStream_t stream, double* h2d) {
  uint8_t* base = b.arena.p;
  const size_t patch = (size_t)d->ph * d->pw * d->channels * dtype_bytes(d->patch_dtype);
  // per-query state, staged on the host
  b.state.assign(v.end - v.off_params, 0);
  uint8_t* st = b.state.data();
  double* params = reinterpret_cast<double*>(st);
  int64_t* obl = reinterpret_cast<int64_t*>(st + (v.off_ob - v.off_params));
  uint64_t* ptrs = reinterpret_cast<uint64_t*>(st + (v.off_ptr - v.off_params));
  int64_t* pf = reinterpret_cast<int64_t*>(st + (v.off_pf - v.off_params));
  int32_t* model = reinterpret_cast<int32_t*>(st + (v.off_model - v.off_params));
  uint32_t* mask = reinterpret_cast<uint32_t*>(st + (v.off_mask - v.off_params));
  std::vector<const void*> srcs;
  std::vector<size_t> sizes;
  size_t slab = 0;
  int64_t prow = 0;
  for (int i = 0; i < v.nq; ++i) {
    const int q = v.q0 + i;
    std::memcpy(params + (size_t)i * kQParams, d->cam_params + (size_t)q * kMaxK, kMaxK * 8);
    std::memcpy(params + (size_t)i * kQParams + kMaxK, d->qvec + (size_t)q * 4, 32);
    std::memcpy(params + (size_t)i * kQParams + kMaxK + 4, d->tvec + (size_t)q * 3, 24);
    obl[i] = d->obs_begin[q] - v.o0;
    pf[i] = prow; prow += d->patch_counts[q];
    model[i] = d->cam_model[q]; mask[i] = d->cam_const_mask[q];
    if (p.host_patch[q]) {
      ptrs[i] = (uint64_t)(base + slab);
      srcs.push_back(d->patch_blocks[q]); sizes.push_back((size_t)d->patch_counts[q] * patch);
      slab += sizes.back();
    } else {
      ptrs[i] = (uint64_t)d->patch_blocks[q];
    }
  }
  obl[v.nq] = v.no;
  auto seg = [&](const void* src, size_t bytes) { srcs.push_back(src); sizes.push_back(bytes); };
  seg(d->refs ? d->refs + v.o0 * d->channels : nullptr, (size_t)v.no * d->channels * 8);
  seg(d->xyz ? d->xyz + v.o0 * 3 : nullptr, (size_t)v.no * 24);
  seg(d->obs_patch ? d->obs_patch + v.o0 : nullptr, (size_t)v.no * 8);
  seg(d->corner ? d->corner + v.p0 * 2 : nullptr, (size_t)v.np * 8);
  seg(d->scale ? d->scale + v.p0 * 2 : nullptr, (size_t)v.np * 16);
  seg(st, b.state.size());
  // segments of zero bytes (no observations) are skipped by upload_segments
  for (size_t i = 0; i < srcs.size(); ++i) if (!sizes[i]) srcs[i] = st;
  PXR_TRY(upload_segments(ctx, base, srcs.data(), sizes.data(), (int)srcs.size(), h2d, stream));
  return PXR_OK;
}

static QBAArgs make_args(const pxr_qba_desc* d, const pxr_interp_config& ic, const pxr_solver_options& so,
                         const WaveView& v, WaveBufs& b, int iter_cap) {
  uint8_t* base = b.arena.p;
  QBAArgs a;
  std::memset(&a, 0, sizeof(a));
  a.n_queries = v.nq;
  a.obs_begin = reinterpret_cast<const int64_t*>(base + v.off_ob);
  a.cam_model = reinterpret_cast<const int32_t*>(base + v.off_model);
  a.cam_mask = reinterpret_cast<const uint32_t*>(base + v.off_mask);
  a.params = reinterpret_cast<double*>(base + v.off_params);
  a.patch = reinterpret_cast<const uint64_t*>(base + v.off_ptr);
  a.patch_first = reinterpret_cast<const int64_t*>(base + v.off_pf);
  a.xyz = reinterpret_cast<const double*>(base + v.off_xyz);
  a.obs_patch = reinterpret_cast<const int64_t*>(base + v.off_op);
  a.refs = reinterpret_cast<const double*>(base + v.off_refs);
  a.corner = reinterpret_cast<const int32_t*>(base + v.off_corner);
  a.scale = reinterpret_cast<const double*>(base + v.off_scale);
  a.ups = d->upsampling_factor; a.ph = d->ph; a.pw = d->pw;
  a.loss.type = so.loss_type; a.loss.a = so.loss_scale; a.l2_normalize = ic.l2_normalize;
  a.max_iter = so.max_num_iterations; a.max_invalid = so.max_num_consecutive_invalid_steps;
  a.max_nonmonotonic = so.use_nonmonotonic_steps ? so.max_consecutive_nonmonotonic_steps : 0;
  a.jacobi_scaling = so.jacobi_scaling;
  a.ftol = so.function_tolerance; a.gtol = so.gradient_tolerance; a.ptol = so.parameter_tolerance;
  a.min_rel_dec = so.min_relative_decrease; a.radius0 = so.initial_trust_region_radius;
  a.max_radius = so.max_trust_region_radius; a.min_radius = so.min_trust_region_radius;
  a.min_diag = so.min_lm_diagonal; a.max_diag = so.max_lm_diagonal;
  int nmax = 6;
  for (int q = v.q0; q < v.q0 + v.nq; ++q) {
    int n = 6;
    for (int k = 0; k < cam_num_params(d->cam_model[q]); ++k) n += ((d->cam_const_mask[q] >> k) & 1u) ? 0 : 1;
    nmax = std::max(nmax, n);
  }
  a.row_stride = (4 + 2 * nmax) | 1;
  a.results = b.results.p;
  a.iters = iter_cap > 0 ? b.iters.p : nullptr; a.iter_cap = iter_cap;
  return a;
}

static size_t qba_smem(const QBAArgs& a) { return (size_t)kQWarps * 32 * a.row_stride * sizeof(double); }

}  // namespace pxr

using namespace pxr;

extern "C" int pxr_qba_plan_waves(const pxr_qba_desc* d, int32_t* wave_begin, int32_t* n_waves, double* wave_bytes) {
  PXR_TRY(check_qba(d, nullptr, nullptr));
  if (!wave_begin || !n_waves) return fail(PXR_ERR_INVALID_ARGUMENT, "wave_begin / n_waves is NULL");
  double budget = 0.0;
  PXR_TRY(wave_budget(d->max_wave_bytes, &budget));
  WavePlan p;
  plan_waves(d, budget, &p);
  *n_waves = (int32_t)p.bytes.size();
  for (size_t i = 0; i < p.begin.size(); ++i) wave_begin[i] = p.begin[i];
  if (wave_bytes) for (size_t i = 0; i < p.bytes.size(); ++i) wave_bytes[i] = p.bytes[i];
  return PXR_OK;
}

extern "C" int pxr_qba_run(pxr_ctx* ctx, const pxr_qba_desc* d, const pxr_interp_config* interp_in,
                           const pxr_solver_options* opt_in, pxr_qba_result* results, pxr_iteration_summary* iterations,
                           int32_t iterations_capacity, int32_t* n_waves_out, pxr_summary* total) {
  const auto t0 = std::chrono::steady_clock::now();
  PXR_TRY(qba_args(ctx, d, interp_in, opt_in));
  if (!results && d->n_queries > 0) return fail(PXR_ERR_INVALID_ARGUMENT, "results is NULL");
  if (iterations_capacity < 0 || (iterations_capacity > 0 && !iterations))
    return fail(PXR_ERR_INVALID_ARGUMENT, "iterations is NULL or iterations_capacity < 0");
  pxr_interp_config ic; if (interp_in) ic = *interp_in; else pxr_default_interp_config(&ic);
  pxr_solver_options so; if (opt_in) so = *opt_in; else { pxr_default_ba_options(&so); so.use_inner_iterations = 0; }
  PXR_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  cudaStream_t us = nullptr;
  PXR_TRY(upload_stream(ctx, &us));
  const int64_t launches0 = ctx->launches;
  double budget = 0.0;
  PXR_TRY(wave_budget(d->max_wave_bytes, &budget));
  WavePlan plan;
  plan_waves(d, budget, &plan);
  const int nw = (int)plan.bytes.size();
  size_t max_arena = 0; int max_nq = 0;
  for (int w = 0; w < nw; ++w) {
    const WaveView v = wave_view(d, plan, w);
    max_arena = std::max(max_arena, v.end); max_nq = std::max(max_nq, v.nq);
  }
  int nsets = 1;
  PXR_TRY(wave_sets(nw, max_arena, &nsets));
  WaveBufs bufs[2];
  // per buffer set, the pinned host copy of a wave's outputs: params | results | iteration summaries
  const size_t out_params = (size_t)std::max(max_nq, 1) * kQParams * 8;
  const size_t out_res = (size_t)std::max(max_nq, 1) * sizeof(pxr_qba_result);
  const size_t out_bytes = out_params + out_res + (size_t)std::max(max_nq, 1) * iterations_capacity * sizeof(pxr_iteration_summary);
  struct Pinned { void* p = nullptr; ~Pinned() { if (p) cudaFreeHost(p); } } hout[2];
  for (int k = 0; k < nsets; ++k) {
    PXR_TRY(bufs[k].arena.alloc(std::max<size_t>(max_arena, 16)));
    PXR_TRY(bufs[k].results.alloc(std::max(max_nq, 1)));
    if (iterations_capacity > 0) PXR_TRY(bufs[k].iters.alloc((size_t)std::max(max_nq, 1) * iterations_capacity));
    PXR_CUDA(cudaMallocHost(&hout[k].p, out_bytes));
  }
  cudaEvent_t kt0 = nullptr, kt1 = nullptr;
  struct Events { cudaEvent_t* a; cudaEvent_t* b; ~Events() { if (*a) cudaEventDestroy(*a); if (*b) cudaEventDestroy(*b); } } guard{&kt0, &kt1};
  PXR_CUDA(cudaEventCreate(&kt0));
  PXR_CUDA(cudaEventCreate(&kt1));
  double h2d = 0.0, kernel_ms = 0.0;
  double ic0 = 0.0, fc = 0.0; int ns = 0, nu = 0;
  WaveSteps steps;
  steps.upload = [&](int w, int set) { return upload_wave(ctx, d, plan, wave_view(d, plan, w), bufs[set], us, &h2d); };
  steps.launch = [&](int w, int set) {
    const WaveView v = wave_view(d, plan, w);
    WaveBufs& b = bufs[set];
    const QBAArgs a = make_args(d, ic, so, v, b, iterations_capacity);
    PXR_CUDA(cudaEventRecord(kt0, s));
    PXR_TRY(launch_qba(ctx, d->patch_dtype, d->channels, ic.use_float_simd != 0, a, qba_smem(a)));
    PXR_CUDA(cudaEventRecord(kt1, s));
    // the wave's outputs leave the arena before the wave is done: a later upload into this arena waits for that
    uint8_t* ho = static_cast<uint8_t*>(hout[set].p);
    PXR_CUDA(cudaMemcpyAsync(ho, a.params, (size_t)v.nq * kQParams * 8, cudaMemcpyDeviceToHost, s));
    PXR_CUDA(cudaMemcpyAsync(ho + out_params, b.results.p, (size_t)v.nq * sizeof(pxr_qba_result), cudaMemcpyDeviceToHost, s));
    if (iterations_capacity > 0)
      PXR_CUDA(cudaMemcpyAsync(ho + out_params + out_res, b.iters.p,
                               (size_t)v.nq * iterations_capacity * sizeof(pxr_iteration_summary), cudaMemcpyDeviceToHost, s));
    return (int)PXR_OK;
  };
  steps.finish = [&](int w, int set) {
    const WaveView v = wave_view(d, plan, w);
    const uint8_t* ho = static_cast<const uint8_t*>(hout[set].p);
    const double* params = reinterpret_cast<const double*>(ho);
    const pxr_qba_result* wres = reinterpret_cast<const pxr_qba_result*>(ho + out_params);
    const pxr_iteration_summary* wits = reinterpret_cast<const pxr_iteration_summary*>(ho + out_params + out_res);
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, kt0, kt1) == cudaSuccess) kernel_ms += ms;
    for (int i = 0; i < v.nq; ++i) {
      const int q = v.q0 + i;
      const pxr_qba_result& r = wres[i];
      results[q] = r;
      if (iterations_capacity > 0) {
        std::memcpy(iterations + (size_t)q * iterations_capacity, wits + (size_t)i * iterations_capacity,
                    (size_t)iterations_capacity * sizeof(pxr_iteration_summary));
      }
      if (r.status != PXR_OK || r.num_residual_blocks == 0) continue;   // parameters untouched
      const double* p = params + (size_t)i * kQParams;
      std::memcpy(d->cam_params + (size_t)q * kMaxK, p, kMaxK * 8);
      std::memcpy(d->qvec + (size_t)q * 4, p + kMaxK, 32);
      std::memcpy(d->tvec + (size_t)q * 3, p + kMaxK + 4, 24);
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
    total->num_residual_blocks = (int32_t)(d->n_queries ? d->obs_begin[d->n_queries] : 0);
    total->num_residuals = (int64_t)total->num_residual_blocks * d->channels;
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

extern "C" int pxr_qba_debug_linearize(pxr_ctx* ctx, const pxr_qba_desc* d, const pxr_interp_config* interp_in,
                                       const pxr_solver_options* opt_in, double* cost, double* H, double* g, double* xy,
                                       double* rec) {
  PXR_TRY(qba_args(ctx, d, interp_in, opt_in));
  pxr_interp_config ic; if (interp_in) ic = *interp_in; else pxr_default_interp_config(&ic);
  pxr_solver_options so; if (opt_in) so = *opt_in; else { pxr_default_ba_options(&so); so.use_inner_iterations = 0; }
  if (d->n_queries == 0) return PXR_OK;
  PXR_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  WavePlan plan;
  plan_waves(d, 1e300, &plan);            // one wave
  const WaveView v = wave_view(d, plan, 0);
  WaveBufs b;
  PXR_TRY(b.arena.alloc(std::max<size_t>(v.end, 16)));
  PXR_TRY(b.results.alloc(v.nq));
  double h2d = 0.0;
  PXR_TRY(upload_wave(ctx, d, plan, v, b, s, &h2d));
  const int64_t n_obs = v.no;
  DevBuf<double> dc, dH, dg, dxy, drec;
  PXR_TRY(dc.alloc(v.nq)); PXR_TRY(dH.alloc((size_t)v.nq * kQMaxN * kQMaxN)); PXR_TRY(dg.alloc((size_t)v.nq * kQMaxN));
  PXR_TRY(dxy.alloc((size_t)std::max<int64_t>(n_obs, 1) * 2)); PXR_TRY(drec.alloc((size_t)std::max<int64_t>(n_obs, 1) * 8));
  PXR_TRY(dc.zero(s)); PXR_TRY(dH.zero(s)); PXR_TRY(dg.zero(s)); PXR_TRY(dxy.zero(s)); PXR_TRY(drec.zero(s));
  QBAArgs a = make_args(d, ic, so, v, b, 0);
  a.linearize_only = 1;
  a.dbg_cost = dc.p; a.dbg_H = dH.p; a.dbg_g = dg.p; a.dbg_xy = dxy.p; a.dbg_rec = drec.p;
  PXR_TRY(launch_qba(ctx, d->patch_dtype, d->channels, ic.use_float_simd != 0, a, qba_smem(a)));
  if (cost) PXR_CUDA(cudaMemcpyAsync(cost, dc.p, (size_t)v.nq * 8, cudaMemcpyDeviceToHost, s));
  if (H) PXR_CUDA(cudaMemcpyAsync(H, dH.p, (size_t)v.nq * kQMaxN * kQMaxN * 8, cudaMemcpyDeviceToHost, s));
  if (g) PXR_CUDA(cudaMemcpyAsync(g, dg.p, (size_t)v.nq * kQMaxN * 8, cudaMemcpyDeviceToHost, s));
  if (xy && n_obs) PXR_CUDA(cudaMemcpyAsync(xy, dxy.p, (size_t)n_obs * 16, cudaMemcpyDeviceToHost, s));
  if (rec && n_obs) PXR_CUDA(cudaMemcpyAsync(rec, drec.p, (size_t)n_obs * 64, cudaMemcpyDeviceToHost, s));
  PXR_CUDA(cudaStreamSynchronize(s));
  return PXR_OK;
}
