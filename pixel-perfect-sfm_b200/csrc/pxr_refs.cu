// pxr_refs.cu — reference extraction on the device.
//
// Replaces _bundle_adjustment.ReferenceExtractor.run (reference
// pixsfm/bundle_adjustment/src/reference_extractor.h:171-318): per 3D point, interpolate the
// L2-normalised descriptor of every track element at the current projection
// (FillDescriptorTrack :300-318 -> K0 + K1 in descriptor mode), run RobustMeanIRLS
// (pixsfm/base/src/irls_optim.h:23-71; weights 1/rho(||d_i - mu||^2), NB rho not rho') and keep
// the observation closest to the robust mean (closest_to_robust_mean, :249-272; first minimum).
#include <cmath>

#include "pxr_ba_host.h"
#include "pxr_waves.h"

namespace pxr {

template <int C>
__global__ void __launch_bounds__(128) irls_kernel(const double* __restrict__ desc, const int64_t* __restrict__ pt_begin,
                                                   int64_t n_points, LossParams loss, int iters, int l2,
                                                   double* __restrict__ refs_out, int64_t* __restrict__ src_out) {
  constexpr int CPL = C >= 32 ? C / 32 : 1;
  constexpr int ACTIVE = C / CPL;
  const int64_t p = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (p >= n_points) return;
  const int64_t ob = pt_begin[p], oe = pt_begin[p + 1];
  const int n = (int)(oe - ob);
  if (n == 0) { if (lane == 0) src_out[p] = -1; return; }
  const bool active = lane < ACTIVE;
  const double* D = desc + ob * C + lane * CPL;
  double mean[CPL];
  // weights live in registers, observation i -> lane (i % 32), slot (i / 32); tracks > 128 obs use the
  // tail slots of the last lane group via recomputation (kMaxSlots*32 observations supported)
  constexpr int kMaxSlots = 8;
  double w[kMaxSlots];
#pragma unroll
  for (int s = 0; s < kMaxSlots; ++s) w[s] = 1.0;
  if (n > kMaxSlots * 32) { if (lane == 0) src_out[p] = -2; return; }  // host falls back to chunking: unsupported length
  int early = -1;
  for (int k = 0; k < iters && early < 0; ++k) {
    double wsum = 0.0;
#pragma unroll
    for (int s = 0; s < kMaxSlots; ++s) if (s * 32 + lane < n) wsum += w[s];
    // sequential-order sum over observations to mirror Eigen's weights.sum() is not required
    // (documented tolerance); warp tree reduction
    wsum = warp_sum(wsum);
#pragma unroll
    for (int s = 0; s < kMaxSlots; ++s) w[s] = w[s] / wsum;
#pragma unroll
    for (int c = 0; c < CPL; ++c) mean[c] = 0.0;
    for (int i = 0; i < n; ++i) {
      const double wi = __shfl_sync(0xffffffffu, w[i >> 5], i & 31);
      if (active) {
#pragma unroll
        for (int c = 0; c < CPL; ++c) mean[c] += D[(int64_t)i * C + c] * wi;
      }
    }
    if (l2) {
      double nn = 0.0;
      if (active) {
#pragma unroll
        for (int c = 0; c < CPL; ++c) nn += mean[c] * mean[c];
      }
      nn = sqrt(warp_sum(nn));
      if (nn > 0.0) {
#pragma unroll
        for (int c = 0; c < CPL; ++c) mean[c] /= nn;
      }
    }
    for (int i = 0; i < n; ++i) {
      double s = 0.0;
      if (active) {
#pragma unroll
        for (int c = 0; c < CPL; ++c) { const double dd = D[(int64_t)i * C + c] - mean[c]; s += dd * dd; }
      }
      s = warp_sum(s);
      double rho[3];
      loss_eval(loss, 1.0, s, rho);
      if (rho[0] > 0.0) { if ((i & 31) == lane) w[i >> 5] = 1.0 / rho[0]; }
      else { early = i; break; }
    }
  }
  if (early >= 0 && active) {
#pragma unroll
    for (int c = 0; c < CPL; ++c) mean[c] = D[(int64_t)early * C + c];
  }
  // closest observation to the robust mean (first minimum)
  int best = 0;
  double best_s = 0.0;
  for (int i = 0; i < n; ++i) {
    double s = 0.0;
    if (active) {
#pragma unroll
      for (int c = 0; c < CPL; ++c) { const double dd = D[(int64_t)i * C + c] - mean[c]; s += dd * dd; }
    }
    s = warp_sum(s);
    if (i == 0 || s < best_s) { best_s = s; best = i; }
  }
  if (active) {
#pragma unroll
    for (int c = 0; c < CPL; ++c) refs_out[p * C + lane * CPL + c] = D[(int64_t)best * C + c];
  }
  if (lane == 0) src_out[p] = ob + best;
}

template <int C>
static int launch_irls(pxr_ctx* ctx, const double* desc, const int64_t* pt_begin, int64_t n_points, LossParams loss,
                       int iters, int l2, double* refs, int64_t* src) {
  PXR_LAUNCH(ctx, irls_kernel<C>, (unsigned)cdiv(n_points * 32, 128), 128, 0, desc, pt_begin, n_points, loss, iters, l2, refs, src);
  PXR_CUDA(cudaGetLastError());
  return PXR_OK;
}

// Reference extraction on an uploaded problem: descriptors at the current projections (K0 + K1 in
// descriptor mode), then one warp per point of IRLS + argmin. refs [n_points][C], src [n_points].
static int refs_on_device(pxr_ctx* ctx, BA& b, int loss_type, double loss_scale, int iters, DevBuf<double>& refs,
                          DevBuf<int64_t>& src) {
  cudaStream_t s = ctx->stream;
  DevBuf<double> dsc;
  PXR_TRY(dsc.alloc((size_t)b.n_obs * b.C));
  PXR_TRY(refs.alloc((size_t)b.n_points * b.C));
  PXR_TRY(src.alloc(b.n_points));
  PXR_TRY(refs.zero(s));
  PXR_TRY(b.project(b.cur, false, nullptr));
  FmEvalArgs a;
  a.uv = b.uv.p; a.item_patch = b.obs_patch.p; a.item_ref = nullptr;
  a.patches = b.d_patches; a.ph = b.ph; a.pw = b.pw; a.refs = nullptr;
  a.begin = 0; a.end = b.n_obs; a.item_index = nullptr; a.out = nullptr; a.residuals = nullptr; a.desc = dsc.p;
  a.loss.type = loss_type; a.loss.a = loss_scale;
  a.l2_normalize = b.interp.l2_normalize;
  int np = 0;
  b.resident_args(a);       // window residency: the 4x4 taps under the projections are all that was brought over
  if (b.n_obs > 0) PXR_TRY(launch_fm_eval(ctx, b.dtype, b.C, 0, b.interp.use_float_simd != 0, a, &np));
  for (;;) {                // (cannot trigger with windows cut from these very projections; kept as the general contract)
    int64_t n_fixed = 0;
    PXR_TRY(b.resident_fix(&n_fixed));
    if (n_fixed == 0) break;
    a.item_index = b.res_fix_list.p; a.begin = 0; a.end = n_fixed;
    PXR_TRY(launch_fm_eval(ctx, b.dtype, b.C, 0, b.interp.use_float_simd != 0, a, &np));
  }
  LossParams lp; lp.type = loss_type; lp.a = loss_scale;
  if (b.n_points > 0) {
    switch (b.C) {
      case 8: PXR_TRY(launch_irls<8>(ctx, dsc.p, b.pt_begin.p, b.n_points, lp, iters, b.interp.l2_normalize, refs.p, src.p)); break;
      case 16: PXR_TRY(launch_irls<16>(ctx, dsc.p, b.pt_begin.p, b.n_points, lp, iters, b.interp.l2_normalize, refs.p, src.p)); break;
      case 32: PXR_TRY(launch_irls<32>(ctx, dsc.p, b.pt_begin.p, b.n_points, lp, iters, b.interp.l2_normalize, refs.p, src.p)); break;
      case 64: PXR_TRY(launch_irls<64>(ctx, dsc.p, b.pt_begin.p, b.n_points, lp, iters, b.interp.l2_normalize, refs.p, src.p)); break;
      case 128: PXR_TRY(launch_irls<128>(ctx, dsc.p, b.pt_begin.p, b.n_points, lp, iters, b.interp.l2_normalize, refs.p, src.p)); break;
      case 256: PXR_TRY(launch_irls<256>(ctx, dsc.p, b.pt_begin.p, b.n_points, lp, iters, b.interp.l2_normalize, refs.p, src.p)); break;
      default: return fail(PXR_ERR_UNSUPPORTED, "Unsupported channel count %d in reference extraction", b.C);
    }
  }
  PXR_CUDA(cudaStreamSynchronize(s));   // dsc is released on return
  return PXR_OK;
}

static int read_src(pxr_ctx* ctx, const BA& b, const DevBuf<int64_t>& src, int64_t* src_obs_out) {
  std::vector<int64_t> hsrc(b.n_points);
  PXR_CUDA(cudaMemcpyAsync(hsrc.data(), src.p, (size_t)b.n_points * 8, cudaMemcpyDeviceToHost, ctx->stream));
  PXR_CUDA(cudaStreamSynchronize(ctx->stream));
  for (int64_t p = 0; p < b.n_points; ++p) {
    if (hsrc[p] == -2) return fail(PXR_ERR_UNSUPPORTED, "track of point %lld longer than 256 observations", (long long)p);
    if (src_obs_out) src_obs_out[p] = hsrc[p];
  }
  return PXR_OK;
}

// Nearest candidate (FindNearestReferences, nearest_references.h:40-47): one warp per item walks its candidate rows;
// lanes stride the channels, each lane sums its channels in order, the lanes' partials meet in a butterfly (fixed
// order), and the first row with the smallest distance wins (strict <; a NaN distance counts as smallest, as in
// numpy's argmin, which the per-query path uses).  Reads C * 8 bytes per candidate once.
constexpr int kNCMaxC = 256;
__global__ void __launch_bounds__(256) nearest_candidate_kernel(const double* __restrict__ qd,
                                                                const int64_t* __restrict__ cand_begin,
                                                                const int64_t* __restrict__ cand_end,
                                                                const double* __restrict__ cand, int64_t n_items, int C,
                                                                int64_t* __restrict__ best, double* __restrict__ d_min) {
  const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (i >= n_items) return;
  double q[kNCMaxC / 32];
#pragma unroll
  for (int k = 0; k < kNCMaxC / 32; ++k) { const int c = lane + 32 * k; q[k] = c < C ? qd[i * C + c] : 0.0; }
  const int64_t b = cand_begin[i], e = cand_end[i];
  int64_t arg = -1;
  double dm = INFINITY;
  for (int64_t r = b; r < e; ++r) {
    const double* row = cand + r * C;
    double s = 0.0;
#pragma unroll
    for (int k = 0; k < kNCMaxC / 32; ++k) {
      const int c = lane + 32 * k;
      if (c < C) { const double t = row[c] - q[k]; s += t * t; }
    }
    s = warp_sum(s);
    if (s < dm || (s != s && dm == dm)) { dm = s; arg = r; }   // numpy's argmin: the first NaN wins
  }
  if (lane == 0) { best[i] = arg; if (d_min) d_min[i] = dm; }
}

template <typename T>
static int launch_costmaps(pxr_ctx* ctx, const CostmapArgs& a) {
  const int64_t warps = a.n_items * a.ph * a.pw;
  if (warps > 0) PXR_LAUNCH(ctx, (costmap_extract_kernel<T, T>), (unsigned)cdiv(warps * 32, 256), 256, 0, a);
  PXR_CUDA(cudaGetLastError());
  return PXR_OK;
}

}  // namespace pxr

using namespace pxr;

extern "C" int pxr_refs_compute(pxr_ctx* ctx, const pxr_ba_desc* desc, const pxr_interp_config* interp, int loss_type,
                                double loss_scale, int iters, double* refs_out, int64_t* src_obs_out,
                                pxr_summary* summary) {
  if (!ctx || !desc || !refs_out) return fail(PXR_ERR_INVALID_ARGUMENT, "NULL argument");
  // reuse the BA upload path with refs = NULL (descriptor mode)
  pxr_ba_desc d = *desc;
  d.refs = nullptr;
  pxr_solver_options so;
  pxr_default_ba_options(&so);
  so.loss_type = loss_type; so.loss_scale = loss_scale;
  BA b;
  const int64_t launches0 = ctx->launches;
  // the descriptors are interpolated at the projections of the CURRENT reconstruction and nothing moves: exactly the
  // 4x4 tap window of every observation is needed (1/16 of a 16x16 patch)
  b.allow_resident = true; b.res_window = 4; b.res_window_fixed = true;
  PXR_TRY(b.create(ctx, &d, interp, &so, false));
  DevBuf<double> refs;
  DevBuf<int64_t> src;
  PXR_TRY(refs_on_device(ctx, b, loss_type, loss_scale, iters, refs, src));
  PXR_CUDA(cudaMemcpyAsync(refs_out, refs.p, (size_t)b.n_points * b.C * 8, cudaMemcpyDeviceToHost, ctx->stream));
  PXR_TRY(read_src(ctx, b, src, src_obs_out));
  if (summary) {
    summary->kernel_launches = ctx->launches - launches0;
    summary->h2d_bytes = b.h2d_bytes; summary->d2h_bytes = (double)b.n_points * (b.C + 1) * 8;
  }
  return PXR_OK;
}

extern "C" int pxr_default_costmap_config(pxr_costmap_config* c) {
  if (!c) return fail(PXR_ERR_INVALID_ARGUMENT, "NULL argument");
  c->loss_type = PXR_LOSS_TRIVIAL; c->loss_scale = 1.0;      // CostMapConfig(): TrivialLoss, costmap_extractor.h:19
  c->as_gradientfield = 1; c->compute_cross_derivative = 0; c->apply_sqrt = 0; c->upsampling_factor = 1.0;
  c->compute_refs = 1; c->ref_loss_type = PXR_LOSS_CAUCHY; c->ref_loss_scale = 0.25; c->ref_iters = 100;
  return PXR_OK;
}

extern "C" int pxr_costmaps_compute(pxr_ctx* ctx, const pxr_ba_desc* desc, const pxr_interp_config* interp,
                                    const pxr_costmap_config* cfg, double* refs_io, int64_t* src_obs_out,
                                    void* out_host, void** out_device, pxr_summary* summary) {
  if (!ctx || !desc || !cfg || (!out_host && !out_device)) return fail(PXR_ERR_INVALID_ARGUMENT, "NULL argument");
  if (cfg->upsampling_factor != 1.0 || cfg->compute_cross_derivative)
    return fail(PXR_ERR_UNSUPPORTED, "cost maps: only upsampling_factor == 1 without the cross derivative (the reference's default branch)");
  if (!cfg->compute_refs && !desc->refs && !refs_io) return fail(PXR_ERR_INVALID_ARGUMENT, "references are required when compute_refs == 0");
  pxr_ba_desc d = *desc;
  d.refs = nullptr;
  pxr_solver_options so;
  pxr_default_ba_options(&so);
  BA b;
  const int64_t launches0 = ctx->launches;
  PXR_TRY(b.create(ctx, &d, interp, &so, false));
  cudaStream_t s = ctx->stream;
  DevBuf<double> refs;
  DevBuf<int64_t> src;
  double d2h = 0;
  if (cfg->compute_refs) {
    PXR_TRY(refs_on_device(ctx, b, cfg->ref_loss_type, cfg->ref_loss_scale, cfg->ref_iters, refs, src));
    if (refs_io) { PXR_CUDA(cudaMemcpyAsync(refs_io, refs.p, (size_t)b.n_points * b.C * 8, cudaMemcpyDeviceToHost, s)); d2h += (double)b.n_points * b.C * 8; }
    PXR_TRY(read_src(ctx, b, src, src_obs_out));
  } else {
    const double* hr = desc->refs ? desc->refs : refs_io;
    PXR_TRY(refs.upload(hr, (size_t)b.n_points * b.C, s));
  }
  const int OC = cfg->as_gradientfield ? 3 : 1;
  const size_t esz = b.dtype == PXR_F16 ? 2 : (b.dtype == PXR_F32 ? 4 : 8);
  const size_t out_bytes = (size_t)b.n_patches * b.ph * b.pw * OC * esz;
  uint8_t* dout = nullptr;
  PXR_CUDA(cudaMalloc((void**)&dout, std::max<size_t>(out_bytes, 16)));
  cudaError_t e = cudaMemsetAsync(dout, 0, out_bytes, s);
  CostmapArgs a;
  a.patches = b.d_patches; a.ph = b.ph; a.pw = b.pw; a.C = b.C;
  a.refs = refs.p; a.item_patch = b.obs_patch.p; a.item_ref = b.obs_pt.p; a.n_items = b.n_obs;
  a.out = dout; a.OC = OC; a.loss.type = cfg->loss_type; a.loss.a = cfg->loss_scale;
  a.as_gradientfield = cfg->as_gradientfield; a.apply_sqrt = cfg->apply_sqrt;
  int rc = e == cudaSuccess ? PXR_OK : fail(PXR_ERR_CUDA, "cudaMemsetAsync failed: %s", cudaGetErrorString(e));
  if (rc == PXR_OK) {
    if (b.dtype == PXR_F16) rc = launch_costmaps<__half>(ctx, a);
    else if (b.dtype == PXR_F32) rc = launch_costmaps<float>(ctx, a);
    else rc = launch_costmaps<double>(ctx, a);
  }
  if (rc == PXR_OK && out_host) {
    e = cudaMemcpyAsync(out_host, dout, out_bytes, cudaMemcpyDeviceToHost, s);
    if (e != cudaSuccess) rc = fail(PXR_ERR_CUDA, "cudaMemcpyAsync failed: %s", cudaGetErrorString(e));
    d2h += (double)out_bytes;
  }
  e = cudaStreamSynchronize(s);
  if (rc == PXR_OK && e != cudaSuccess) rc = fail(PXR_ERR_CUDA, "cost-map extraction failed: %s", cudaGetErrorString(e));
  if (rc != PXR_OK || !out_device) cudaFree(dout); else *out_device = dout;
  if (rc == PXR_OK && summary) {
    summary->kernel_launches = ctx->launches - launches0;
    summary->h2d_bytes = b.h2d_bytes; summary->d2h_bytes = d2h;
  }
  return rc;
}

extern "C" int pxr_interpolate_descriptors(pxr_ctx* ctx, const void* patches, int64_t n_patches, int32_t patch_dtype, int32_t ph,
                                           int32_t pw, int32_t channels, const int32_t* corner, const double* scale,
                                           double ups, int64_t n_items, const int64_t* item_patch, const double* xy,
                                           const pxr_interp_config* interp, double* out_desc) {
  if (!ctx || !patches || !corner || !scale || !xy || !out_desc || n_items < 0 || n_patches <= 0)
    return fail(PXR_ERR_INVALID_ARGUMENT, "NULL argument");
  if (!fm_supported(patch_dtype, channels))
    return fail(PXR_ERR_UNSUPPORTED, "Unsupported dimensions (CHANNELS=%d, dtype=%d, N_NODES=1).", channels, patch_dtype);
  pxr_interp_config ic; if (interp) ic = *interp; else pxr_default_interp_config(&ic);
  if (n_items == 0) return PXR_OK;
  PXR_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  // patch pixel coordinates, FeaturePatch::ToPixelCoordinates (features/src/featurepatch.h:250-255)
  std::vector<double> uv((size_t)n_items * 2);
  for (int64_t i = 0; i < n_items; ++i) {
    const int64_t pi = item_patch ? item_patch[i] : i;
    if (pi < 0 || pi >= n_patches) return fail(PXR_ERR_INVALID_ARGUMENT, "item_patch out of range");
    uv[2 * i] = (xy[2 * i] * scale[2 * pi] - 0.5 - (double)corner[2 * pi]) * ups;
    uv[2 * i + 1] = (xy[2 * i + 1] * scale[2 * pi + 1] - 0.5 - (double)corner[2 * pi + 1]) * ups;
  }
  const size_t esz = patch_dtype == PXR_F16 ? 2 : (patch_dtype == PXR_F32 ? 4 : 8);
  DevBuf<uint8_t> dp; DevBuf<double> duv, ddesc; DevBuf<int64_t> dip;
  PXR_TRY(dp.upload((const uint8_t*)patches, (size_t)n_patches * ph * pw * channels * esz, s));
  PXR_TRY(duv.upload(uv.data(), uv.size(), s));
  if (item_patch) PXR_TRY(dip.upload(item_patch, n_items, s));
  PXR_TRY(ddesc.alloc((size_t)n_items * channels));
  FmEvalArgs a;
  a.uv = duv.p; a.item_patch = item_patch ? dip.p : nullptr; a.item_ref = nullptr;
  a.patches = dp.p; a.ph = ph; a.pw = pw; a.refs = nullptr;
  a.begin = 0; a.end = n_items; a.item_index = nullptr; a.out = nullptr; a.residuals = nullptr; a.desc = ddesc.p;
  a.loss.type = 0; a.loss.a = 1.0;
  a.l2_normalize = ic.l2_normalize;
  int np = 0;
  PXR_TRY(launch_fm_eval(ctx, patch_dtype, channels, 0, ic.use_float_simd != 0, a, &np));
  PXR_CUDA(cudaMemcpyAsync(out_desc, ddesc.p, (size_t)n_items * channels * 8, cudaMemcpyDeviceToHost, s));
  PXR_CUDA(cudaStreamSynchronize(s));
  return PXR_OK;
}

extern "C" int pxr_obs_descriptors(pxr_ctx* ctx, const pxr_ba_desc* desc, const pxr_interp_config* interp, double* out_desc) {
  if (!ctx || !desc || !out_desc) return fail(PXR_ERR_INVALID_ARGUMENT, "NULL argument");
  pxr_ba_desc d = *desc;
  d.refs = nullptr;
  pxr_solver_options so;
  pxr_default_ba_options(&so);
  BA b;
  PXR_TRY(b.create(ctx, &d, interp, &so, false));
  if (b.n_obs == 0) return PXR_OK;
  DevBuf<double> dsc;
  PXR_TRY(dsc.alloc((size_t)b.n_obs * b.C));
  PXR_TRY(b.project(b.cur, false, nullptr));
  FmEvalArgs a;
  a.uv = b.uv.p; a.item_patch = b.obs_patch.p; a.item_ref = nullptr;
  a.patches = b.d_patches; a.ph = b.ph; a.pw = b.pw; a.refs = nullptr;
  a.begin = 0; a.end = b.n_obs; a.item_index = nullptr; a.out = nullptr; a.residuals = nullptr; a.desc = dsc.p;
  a.loss.type = 0; a.loss.a = 1.0;
  a.l2_normalize = b.interp.l2_normalize;
  int np = 0;
  PXR_TRY(launch_fm_eval(ctx, b.dtype, b.C, 0, b.interp.use_float_simd != 0, a, &np));
  PXR_CUDA(cudaMemcpyAsync(out_desc, dsc.p, (size_t)b.n_obs * b.C * 8, cudaMemcpyDeviceToHost, ctx->stream));
  PXR_CUDA(cudaStreamSynchronize(ctx->stream));
  return PXR_OK;
}

extern "C" int pxr_query_match_run(pxr_ctx* ctx, int32_t n_queries, const void* const* patch_blocks,
                                   const int64_t* patch_counts, const int32_t* corner, const double* scale, double ups,
                                   int32_t ph, int32_t pw, int32_t channels, int32_t patch_dtype, int64_t n_items,
                                   const int32_t* item_query, const int64_t* item_patch, const double* xy,
                                   const int64_t* cand_begin, const int64_t* cand_end, const double* cand, int64_t n_cand,
                                   int32_t cand_on_device,
                                   const pxr_interp_config* interp, int64_t* best, double* d_min, double* out_desc) {
  // ---- arguments, before the context
  if (n_queries < 0 || n_items < 0 || n_cand < 0) return fail(PXR_ERR_INVALID_ARGUMENT, "negative count");
  if ((n_queries > 0 && (!patch_blocks || !patch_counts)) ||
      (n_items > 0 && (!item_query || !item_patch || !xy || !cand_begin || !cand_end || !best)) || (n_cand > 0 && !cand))
    return fail(PXR_ERR_INVALID_ARGUMENT, "a required array is NULL");
  if (interp && interp->check_bounds) return fail(PXR_ERR_UNSUPPORTED, "check_bounds=true is not supported on this path");
  if (!fm_supported(patch_dtype, channels) || channels > kNCMaxC)
    return fail(PXR_ERR_UNSUPPORTED, "Unsupported dimensions (CHANNELS=%d, dtype=%d, N_NODES=1).", channels, patch_dtype);
  if (ph < 1 || pw < 1) return fail(PXR_ERR_INVALID_ARGUMENT, "bad patch size");
  if (!(ups > 0.0)) return fail(PXR_ERR_INVALID_ARGUMENT, "upsampling_factor must be > 0");
  std::vector<int64_t> first((size_t)n_queries + 1, 0);
  for (int q = 0; q < n_queries; ++q) {
    if (patch_counts[q] < 0) return fail(PXR_ERR_INVALID_ARGUMENT, "patch_counts[%d] < 0", q);
    if (patch_counts[q] > 0 && !patch_blocks[q]) return fail(PXR_ERR_INVALID_ARGUMENT, "patch block %d is NULL", q);
    first[q + 1] = first[q] + patch_counts[q];
  }
  if (first[n_queries] > 0 && (!corner || !scale)) return fail(PXR_ERR_INVALID_ARGUMENT, "a required array is NULL");
  // patch pixel coordinates, FeaturePatch::ToPixelCoordinates, as pxr_interpolate_descriptors computes them
  std::vector<double> uv((size_t)n_items * 2);
  std::vector<int64_t> gpatch((size_t)n_items);
  for (int64_t i = 0; i < n_items; ++i) {
    const int q = item_query[i];
    if (q < 0 || q >= n_queries) return fail(PXR_ERR_INVALID_ARGUMENT, "item_query[%lld] out of range", (long long)i);
    if (item_patch[i] < 0 || item_patch[i] >= patch_counts[q])
      return fail(PXR_ERR_INVALID_ARGUMENT, "item_patch[%lld] is not a patch of query %d", (long long)i, q);
    if (cand_begin[i] < 0 || cand_end[i] < cand_begin[i] || cand_end[i] > n_cand)
      return fail(PXR_ERR_INVALID_ARGUMENT, "candidate range of item %lld is out of bounds", (long long)i);
    const int64_t pi = first[q] + item_patch[i];
    gpatch[i] = pi;
    uv[2 * i] = (xy[2 * i] * scale[2 * pi] - 0.5 - (double)corner[2 * pi]) * ups;
    uv[2 * i + 1] = (xy[2 * i + 1] * scale[2 * pi + 1] - 0.5 - (double)corner[2 * pi + 1]) * ups;
  }
  PXR_TRY(require_ctx(ctx));
  pxr_interp_config ic; if (interp) ic = *interp; else pxr_default_interp_config(&ic);
  if (n_items == 0) return PXR_OK;
  PXR_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  // the query blocks back to back in one slab (device blocks are copied on the device)
  const size_t per = (size_t)ph * pw * channels * dtype_bytes(patch_dtype);
  std::vector<const void*> srcs((size_t)n_queries);
  std::vector<size_t> sizes((size_t)n_queries);
  static const uint8_t kNoPatch = 0;
  for (int q = 0; q < n_queries; ++q) {
    srcs[q] = patch_counts[q] > 0 ? patch_blocks[q] : &kNoPatch;
    sizes[q] = (size_t)patch_counts[q] * per;
  }
  DevBuf<uint8_t> dp; DevBuf<double> duv, ddesc, dcand, dmin; DevBuf<int64_t> dip, dcb, dce, dbest;
  PXR_TRY(dp.alloc(std::max<size_t>((size_t)first[n_queries] * per, 16)));
  PXR_TRY(upload_segments(ctx, dp.p, srcs.data(), sizes.data(), n_queries, nullptr, s));
  PXR_TRY(duv.upload(uv.data(), uv.size(), s));
  PXR_TRY(dip.upload(gpatch.data(), gpatch.size(), s));
  PXR_TRY(dcb.upload(cand_begin, (size_t)n_items, s));
  PXR_TRY(dce.upload(cand_end, (size_t)n_items, s));
  const double* cp = cand;
  if (!cand_on_device && n_cand > 0) { PXR_TRY(dcand.upload(cand, (size_t)n_cand * channels, s)); cp = dcand.p; }
  PXR_TRY(ddesc.alloc((size_t)n_items * channels));
  PXR_TRY(dbest.alloc((size_t)n_items));
  PXR_TRY(dmin.alloc((size_t)n_items));
  // the query descriptors: K1 in descriptor mode, as pxr_interpolate_descriptors runs it
  FmEvalArgs a;
  a.uv = duv.p; a.item_patch = dip.p; a.item_ref = nullptr;
  a.patches = dp.p; a.ph = ph; a.pw = pw; a.refs = nullptr;
  a.begin = 0; a.end = n_items; a.item_index = nullptr; a.out = nullptr; a.residuals = nullptr; a.desc = ddesc.p;
  a.loss.type = 0; a.loss.a = 1.0;
  a.l2_normalize = ic.l2_normalize;
  int np = 0;
  PXR_TRY(launch_fm_eval(ctx, patch_dtype, channels, 0, ic.use_float_simd != 0, a, &np));
  PXR_LAUNCH(ctx, nearest_candidate_kernel, (unsigned)cdiv(n_items * 32, 256), 256, 0, ddesc.p, dcb.p, dce.p, cp, n_items,
             (int)channels, dbest.p, dmin.p);
  PXR_CUDA(cudaGetLastError());
  PXR_CUDA(cudaMemcpyAsync(best, dbest.p, (size_t)n_items * 8, cudaMemcpyDeviceToHost, s));
  if (d_min) PXR_CUDA(cudaMemcpyAsync(d_min, dmin.p, (size_t)n_items * 8, cudaMemcpyDeviceToHost, s));
  if (out_desc) PXR_CUDA(cudaMemcpyAsync(out_desc, ddesc.p, (size_t)n_items * channels * 8, cudaMemcpyDeviceToHost, s));
  PXR_CUDA(cudaStreamSynchronize(s));
  return PXR_OK;
}
