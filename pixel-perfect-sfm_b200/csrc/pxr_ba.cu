// pxr_ba.cu — featuremetric bundle adjustment on the device: problem upload, the fused
// residual/Jacobian evaluation (K0+K1), and the Levenberg-Marquardt driver that replaces
// ceres::Solve for FeatureReferenceBundleOptimizer (reference
// pixsfm/bundle_adjustment/src/bundle_optimizer.h:114-245,
// feature_reference_bundle_optimizer.h:90-149).  The host only orchestrates launches and reads
// back a handful of scalars per LM iteration; all arithmetic runs in the CUDA kernels of
// pxr_fm_eval.cuh / pxr_ba_kernels.cuh / pxr_inner.cuh.
#include <chrono>
#include <cmath>
#include <cstdlib>
#include <algorithm>
#include <cstring>
#include <limits>
#include <memory>

#include "pxr_ba_host.h"

#include "pxr_resident.cuh"
#include "pxr_chol2.cuh"

namespace pxr {

// -------------------------------------------------------------------------------- fm_eval dispatch
// K1 CTAs for n items: enough for one item per half-warp, up to what is resident; the kernel spreads the items evenly
// over the half-warps it gets
template <typename T, int C>
static int64_t fm_grid(const pxr_ctx* ctx, int64_t n) {
  typedef FmCfg<T, C> Cfg;
  int64_t grid = cdiv(n, 2 * Cfg::kWarps);
  const int64_t resident = (int64_t)ctx->sm_count * std::max(1, (int)(200 * 1024 / Cfg::kSmem));
  if (grid > resident) grid = resident;
  return grid < 1 ? 1 : grid;
}

template <typename T, int C, int MODE, bool FS>
static int launch_fm(pxr_ctx* ctx, const FmEvalArgs& a, int* n_partials) {
  typedef FmCfg<T, C> Cfg;
  auto kern = fm_eval_kernel<T, C, MODE, FS>;
  static bool attr_set = false;
  if (!attr_set) {
    PXR_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmem));
    attr_set = true;
  }
  const int64_t grid = fm_grid<T, C>(ctx, a.end - a.begin);
  *n_partials = (int)(grid * Cfg::kWarps);
  PXR_LAUNCH(ctx, kern, (unsigned)grid, Cfg::kWarps * 32, Cfg::kSmem, a);
  PXR_CUDA(cudaGetLastError());
  return PXR_OK;
}

template <typename T, int C>
static int launch_fm_tc(pxr_ctx* ctx, const FmEvalArgs& a, int mode, bool fs, int* np) {
  if (mode == 1) return fs ? launch_fm<T, C, 1, true>(ctx, a, np) : launch_fm<T, C, 1, false>(ctx, a, np);
  return fs ? launch_fm<T, C, 0, true>(ctx, a, np) : launch_fm<T, C, 0, false>(ctx, a, np);
}

template <typename T, int C>
static int launch_fm_small(pxr_ctx* ctx, const FmEvalArgs& a, int mode, int* np) {
  const int64_t n = a.end - a.begin;
  *np = 0;
  if (n <= 0) return PXR_OK;
  if (mode == 1) PXR_LAUNCH(ctx, (fm_eval_small_kernel<T, C, 1>), (unsigned)cdiv(n, 128), 128, 0, a);
  else PXR_LAUNCH(ctx, (fm_eval_small_kernel<T, C, 0>), (unsigned)cdiv(n, 128), 128, 0, a);
  PXR_CUDA(cudaGetLastError());
  return PXR_OK;
}

int fm_supported(int dtype, int C) {
  // C < 8: the reference's all-double bicubic branch (interpolation.h:224); 3/4 = cost maps, 1 = scalar maps
  if ((C == 1 || C == 3 || C == 4) && (dtype == PXR_F16 || dtype == PXR_F32 || dtype == PXR_F64)) return 1;
  if (dtype == PXR_F16) return C == 8 || C == 16 || C == 32 || C == 64 || C == 128 || C == 256;
  if (dtype == PXR_F32) return C == 16 || C == 64 || C == 128;
  if (dtype == PXR_F64) return C == 16 || C == 128;
  return 0;
}

int fm_max_partials(pxr_ctx* ctx) { return ctx->sm_count * 16 * 64; }

// half-warps of the K1 launch over n items (its grid x warps per CTA x 2); 0 for C < 8 (one thread per item)
static int64_t fm_half_warps(const pxr_ctx* ctx, int dtype, int C, int64_t n) {
#define PXR_HW(T, CC) \
  if (C == CC) return fm_grid<T, CC>(ctx, n) * FmCfg<T, CC>::kWarps * 2;
  if (dtype == PXR_F16) { PXR_HW(__half, 8) PXR_HW(__half, 16) PXR_HW(__half, 32) PXR_HW(__half, 64) PXR_HW(__half, 128) PXR_HW(__half, 256) }
  else if (dtype == PXR_F32) { PXR_HW(float, 16) PXR_HW(float, 64) PXR_HW(float, 128) }
  else if (dtype == PXR_F64) { PXR_HW(double, 16) PXR_HW(double, 128) }
#undef PXR_HW
  return 0;
}

int launch_fm_eval(pxr_ctx* ctx, int dtype, int C, int mode, bool float_simd, const FmEvalArgs& a, int* np) {
#define PXR_SMALL(T) \
  { if (C == 3) return launch_fm_small<T, 3>(ctx, a, mode, np); if (C == 4) return launch_fm_small<T, 4>(ctx, a, mode, np); \
    if (C == 1) return launch_fm_small<T, 1>(ctx, a, mode, np); }
  if (C < 8) {
    if (dtype == PXR_F16) PXR_SMALL(__half) else if (dtype == PXR_F32) PXR_SMALL(float) else if (dtype == PXR_F64) PXR_SMALL(double)
    return fail(PXR_ERR_UNSUPPORTED, "Unsupported dimensions (CHANNELS=%d, dtype=%d, N_NODES=1).", C, dtype);
  }
#undef PXR_SMALL
#define PXR_CASE(T, CC) \
  if (C == CC) return launch_fm_tc<T, CC>(ctx, a, mode, float_simd, np);
  if (dtype == PXR_F16) {
    PXR_CASE(__half, 128) PXR_CASE(__half, 64) PXR_CASE(__half, 32) PXR_CASE(__half, 16) PXR_CASE(__half, 8)
    PXR_CASE(__half, 256)
  } else if (dtype == PXR_F32) {
    PXR_CASE(float, 128) PXR_CASE(float, 64) PXR_CASE(float, 16)
  } else if (dtype == PXR_F64) {
    PXR_CASE(double, 128) PXR_CASE(double, 16)
  }
#undef PXR_CASE
  return fail(PXR_ERR_UNSUPPORTED, "Unsupported dimensions (CHANNELS=%d, dtype=%d, N_NODES=1).", C, dtype);
}

// -------------------------------------------------------------------------------- problem upload
static int check_desc(const pxr_ba_desc* d) {
  if (!d) return fail(PXR_ERR_INVALID_ARGUMENT, "desc is NULL");
  if (d->n_cameras <= 0 || d->n_images <= 0 || d->n_points < 0 || d->n_obs < 0)
    return fail(PXR_ERR_INVALID_ARGUMENT, "empty problem");
  if (!d->cam_model || !d->cam_params || !d->cam_const_mask || !d->qvec || !d->tvec || !d->img_cam ||
      !d->pose_const || !d->tvec_const_mask || (d->n_points && (!d->xyz || !d->point_const)) ||
      (d->n_obs && (!d->obs_img || !d->obs_pt)) || (!d->patches && d->n_patch_blocks <= 0) || !d->corner || !d->scale)
    return fail(PXR_ERR_INVALID_ARGUMENT, "a required array is NULL");
  if (!fm_supported(d->patch_dtype, d->channels))
    return fail(PXR_ERR_UNSUPPORTED, "Unsupported dimensions (CHANNELS=%d, dtype=%d, N_NODES=1).", d->channels, d->patch_dtype);
  if (d->ph < 1 || d->pw < 1) return fail(PXR_ERR_INVALID_ARGUMENT, "bad patch size");
  for (int c = 0; c < d->n_cameras; ++c)
    if (cam_num_params(d->cam_model[c]) == 0) return fail(PXR_ERR_UNSUPPORTED, "unsupported camera model id %d", d->cam_model[c]);
  for (int i = 0; i < d->n_images; ++i)
    if (d->img_cam[i] < 0 || d->img_cam[i] >= d->n_cameras) return fail(PXR_ERR_INVALID_ARGUMENT, "img_cam out of range");
  const int64_t np = d->obs_patch ? d->n_patches : d->n_obs;
  for (int64_t o = 0; o < d->n_obs; ++o) {
    if (d->obs_img[o] < 0 || d->obs_img[o] >= d->n_images) return fail(PXR_ERR_INVALID_ARGUMENT, "obs_img out of range");
    if (d->obs_pt[o] < 0 || d->obs_pt[o] >= d->n_points) return fail(PXR_ERR_INVALID_ARGUMENT, "obs_pt out of range");
    if (o && d->obs_pt[o] < d->obs_pt[o - 1]) return fail(PXR_ERR_INVALID_ARGUMENT, "observations must be sorted by point index");
    if (d->obs_patch && (d->obs_patch[o] < 0 || d->obs_patch[o] >= np)) return fail(PXR_ERR_INVALID_ARGUMENT, "obs_patch out of range");
  }
  if (!d->obs_patch && d->n_patches < d->n_obs) return fail(PXR_ERR_INVALID_ARGUMENT, "n_patches < n_obs with identity patch map");
  return PXR_OK;
}

// A geometric desc: the same geometry and observation lists, no patch slab (channels 0, patches / patch blocks / refs
// NULL; corner, scale and obs_patch are ignored) and one finite observed keypoint per observation.  Host only.
static int check_desc_geometric(const pxr_ba_desc* d, const double* obs_xy) {
  if (!d) return fail(PXR_ERR_INVALID_ARGUMENT, "desc is NULL");
  if (d->n_cameras <= 0 || d->n_images <= 0 || d->n_points < 0 || d->n_obs < 0)
    return fail(PXR_ERR_INVALID_ARGUMENT, "empty problem");
  if (!d->cam_model || !d->cam_params || !d->cam_const_mask || !d->qvec || !d->tvec || !d->img_cam ||
      !d->pose_const || !d->tvec_const_mask || (d->n_points && (!d->xyz || !d->point_const)) ||
      (d->n_obs && (!d->obs_img || !d->obs_pt)))
    return fail(PXR_ERR_INVALID_ARGUMENT, "a required array is NULL");
  if (d->channels != 0 || d->patches || d->n_patch_blocks != 0 || d->refs)
    return fail(PXR_ERR_INVALID_ARGUMENT, "a geometric problem has no feature patches (channels 0, patches, patch blocks and refs NULL)");
  if (!obs_xy) return fail(PXR_ERR_INVALID_ARGUMENT, "obs_xy is NULL");
  for (int c = 0; c < d->n_cameras; ++c)
    if (cam_num_params(d->cam_model[c]) == 0) return fail(PXR_ERR_UNSUPPORTED, "unsupported camera model id %d", d->cam_model[c]);
  for (int i = 0; i < d->n_images; ++i)
    if (d->img_cam[i] < 0 || d->img_cam[i] >= d->n_cameras) return fail(PXR_ERR_INVALID_ARGUMENT, "img_cam out of range");
  for (int64_t o = 0; o < d->n_obs; ++o) {
    if (d->obs_img[o] < 0 || d->obs_img[o] >= d->n_images) return fail(PXR_ERR_INVALID_ARGUMENT, "obs_img out of range");
    if (d->obs_pt[o] < 0 || d->obs_pt[o] >= d->n_points) return fail(PXR_ERR_INVALID_ARGUMENT, "obs_pt out of range");
    if (o && d->obs_pt[o] < d->obs_pt[o - 1]) return fail(PXR_ERR_INVALID_ARGUMENT, "observations must be sorted by point index");
    if (!std::isfinite(obs_xy[2 * o]) || !std::isfinite(obs_xy[2 * o + 1]))
      return fail(PXR_ERR_INVALID_ARGUMENT, "obs_xy[%lld] is not finite", (long long)o);
  }
  return PXR_OK;
}

int BA::create(pxr_ctx* c, const pxr_ba_desc* d, const pxr_interp_config* ic, const pxr_solver_options* so, bool for_solve,
               const double* obs_xy) {
  ctx = c;
  geometric = obs_xy != nullptr;
  PXR_TRY(geometric ? check_desc_geometric(d, obs_xy) : check_desc(d));
  if (ic) interp = *ic; else pxr_default_interp_config(&interp);
  if (so) opt = *so; else pxr_default_ba_options(&opt);
  if (interp.check_bounds) return fail(PXR_ERR_UNSUPPORTED, "check_bounds=true is not supported on this path");
  env.pcg_sparse = getenv("PXR_PCG_SPARSE") != nullptr; env.build_atomic = getenv("PXR_BUILD_ATOMIC") != nullptr;
  env.chol_multikernel = getenv("PXR_CHOL_MULTIKERNEL") != nullptr; env.chol_test_abort = getenv("PXR_CHOL_TEST_ABORT") != nullptr;
  env.build_staged = getenv("PXR_BUILD_UNSTAGED") == nullptr;
  env.project_staged = getenv("PXR_PROJECT_UNSTAGED") == nullptr;
  env.cg_multi = getenv("PXR_CG_MULTI") != nullptr; env.no_speculation = getenv("PXR_NO_SPECULATION") != nullptr;
  if (const char* t = getenv("PXR_CHOL_TRACE")) env.chol_trace = t;
  PXR_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  n_cameras = d->n_cameras; n_images = d->n_images; n_points = d->n_points; n_obs = d->n_obs;
  C = d->channels; ph = d->ph; pw = d->pw; dtype = d->patch_dtype; ups = d->upsampling_factor;
  n_patches = d->obs_patch ? d->n_patches : std::max(d->n_patches, d->n_obs);
  if (geometric) { C = 2; ups = 1.0; n_patches = n_obs; }   // two residuals per observation; K0 in the identity patch frame
  has_refs = d->refs != nullptr;
  // the big patch upload goes first, on the context's side stream: the host-side layout / co-visibility work below
  // (and the small synchronous uploads it makes on `s`) overlaps with the DMA; joined when create() returns
  cudaStream_t us = nullptr;
  PXR_TRY(upload_stream(ctx, &us));
  struct JoinUpload { BA* ba; cudaStream_t us; ~JoinUpload() { if (ba->res_thread.joinable()) ba->res_thread.join(); cudaStreamSynchronize(us); } } join_upload{this, us};
  double h2d_patch = 0;
  const size_t esz = dtype == PXR_F16 ? 2 : (dtype == PXR_F32 ? 4 : 8);
  const size_t pbytes = (size_t)n_patches * ph * pw * C * esz;
  if (geometric) {
    // no patch slab to upload
  } else if (d->n_patch_blocks > 0) {
    if (!d->patch_block_ptrs || !d->patch_block_counts) return fail(PXR_ERR_INVALID_ARGUMENT, "patch block arrays are NULL");
    int64_t tot = 0;
    for (int b = 0; b < d->n_patch_blocks; ++b) tot += d->patch_block_counts[b];
    if (tot < n_patches) return fail(PXR_ERR_INVALID_ARGUMENT, "patch blocks hold %lld patches, %lld needed", (long long)tot, (long long)n_patches);
    PXR_TRY(patches_owned.alloc(ctx, (size_t)tot * ph * pw * C * esz));
    PXR_TRY(resident_setup(d, esz));                      // window residency where it applies (copies issued further down)
    if (!resident) {
      // a block may live in host OR device memory (device-resident feature store): UVA resolves the direction
      std::vector<size_t> seg_bytes((size_t)d->n_patch_blocks);
      for (int b = 0; b < d->n_patch_blocks; ++b) seg_bytes[b] = (size_t)d->patch_block_counts[b] * ph * pw * C * esz;
      PXR_TRY(upload_segments(ctx, patches_owned.p, d->patch_block_ptrs, seg_bytes.data(), d->n_patch_blocks, &h2d_patch, us));
    }
    d_patches = patches_owned.p;
  } else if (d->patches_on_device) {
    d_patches = (const uint8_t*)d->patches;
  } else {
    PXR_TRY(patches_owned.alloc(ctx, pbytes));
    PXR_TRY(resident_setup(d, esz));
    if (!resident) {
      PXR_TRY(upload_bytes(ctx, patches_owned.p, d->patches, pbytes, nullptr, us));
      h2d_patch = (double)pbytes;
    }
    d_patches = patches_owned.p;
  }
  // ---- layout (same rules as BundleOptimizer::Parameterize*, resolved into masks by the caller)
  K = 0;
  for (int i = 0; i < n_cameras; ++i) K = std::max(K, cam_num_params(d->cam_model[i]));
  dcmax = 6 + K;
  juv_stride = 2 * (9 + K);
  h_pose_off.assign(n_images, -1); h_intr_off.assign(n_cameras, -1); h_point_off.assign(n_points, -1);
  int off = 0;
  for (int i = 0; i < n_images; ++i) {
    if (d->pose_const[i]) continue;
    h_pose_off[i] = off;
    off += 3 + (3 - __builtin_popcount(d->tvec_const_mask[i] & 7u));
  }
  std::vector<uint32_t> cmask(n_cameras);
  for (int i = 0; i < n_cameras; ++i) {
    const int k = cam_num_params(d->cam_model[i]);
    const uint32_t full = (1u << k) - 1u;
    cmask[i] = d->cam_const_mask[i] & full;
    if (cmask[i] == full) continue;
    h_intr_off[i] = off;
    off += k - __builtin_popcount(cmask[i]);
  }
  nc = off;
  int64_t po = off;
  for (int64_t p = 0; p < n_points; ++p) if (!d->point_const[p]) { h_point_off[p] = po; po += 3; }
  nl = (int64_t)po;
  h_pt_begin.assign(n_points + 1, 0);
  for (int64_t o = 0; o < n_obs; ++o) h_pt_begin[d->obs_pt[o] + 1]++;
  for (int64_t p = 0; p < n_points; ++p) h_pt_begin[p + 1] += h_pt_begin[p];

  double h2d = h2d_patch;
  auto up = [&](auto& buf, const auto* host, size_t n) -> int { h2d += n * sizeof(*host); return buf.upload(host, n, s); };
  PXR_TRY(up(obs_img, d->obs_img, n_obs));
  PXR_TRY(up(obs_pt, d->obs_pt, n_obs));
  if (d->obs_patch && !geometric) PXR_TRY(up(obs_patch, d->obs_patch, n_obs));
  PXR_TRY(up(img_cam, d->img_cam, n_images));
  PXR_TRY(up(cam_model, d->cam_model, n_cameras));
  PXR_TRY(up(cam_mask, cmask.data(), n_cameras));
  PXR_TRY(up(tmask, d->tvec_const_mask, n_images));
  PXR_TRY(up(pose_off, h_pose_off.data(), n_images));
  PXR_TRY(up(intr_off, h_intr_off.data(), n_cameras));
  PXR_TRY(up(point_off, h_point_off.data(), n_points));
  PXR_TRY(up(pt_begin, h_pt_begin.data(), n_points + 1));
  // geometric: identity frame per observation (corner 0, scale 1), so K0's Jacobian record is d(xy)/d(theta) exactly
  const std::vector<int32_t> geo_corner(geometric ? (size_t)n_obs * 2 : 0, 0);
  const std::vector<double> geo_scale(geometric ? (size_t)n_obs * 2 : 0, 1.0);
  PXR_TRY(up(corner, geometric ? geo_corner.data() : d->corner, (size_t)n_patches * 2));
  PXR_TRY(up(scale, geometric ? geo_scale.data() : d->scale, (size_t)n_patches * 2));
  if (has_refs) PXR_TRY(up(refs, d->refs, (size_t)n_points * C));
  if (geometric) { PXR_TRY(up(geo_target, obs_xy, (size_t)n_obs * 2)); PXR_TRY(geo_xy.alloc((size_t)n_obs * 2)); }
  for (int k = 0; k < 2; ++k) {
    PXR_TRY(cam[k].upload(d->cam_params, (size_t)n_cameras * kMaxK, s));
    PXR_TRY(q[k].upload(d->qvec, (size_t)n_images * 4, s));
    PXR_TRY(t[k].upload(d->tvec, (size_t)n_images * 3, s));
    PXR_TRY(X[k].upload(d->xyz, (size_t)n_points * 3, s));
  }
  h2d += ((size_t)n_cameras * kMaxK + n_images * 7 + n_points * 3) * 8.0;
  cur = 0;
  // per-observation and linearisation buffers
  PXR_TRY(uv.alloc((size_t)n_obs * 2));
  if (resident) { double wbytes = 0; PXR_TRY(resident_begin(us, &wbytes)); h2d += wbytes; }
  PXR_TRY(obs_out.alloc((size_t)n_obs * 8));
  PXR_TRY(juv.alloc((size_t)n_obs * juv_stride));
  if (for_solve) {
    PXR_TRY(uv_alt.alloc((size_t)n_obs * 2)); PXR_TRY(obs_out_alt.alloc((size_t)n_obs * 8)); PXR_TRY(juv_alt.alloc((size_t)n_obs * juv_stride));
    PXR_TRY(obs_out_alt.zero(s));
  }
  // linear solver as BundleOptimizer::SolveProblem picks it (bundle_optimizer.h:181-191): exact factorisation up to
  // 1000 images, ITERATIVE_SCHUR + SCHUR_JACOBI above (or when asked for)
  use_pcg = opt.linear_solver == PXR_SOLVER_ITERATIVE_SCHUR || (opt.linear_solver == PXR_SOLVER_AUTO && n_images > 1000);
  {
    // per-image column tables: an observation's camera columns are [pose columns | intrinsics columns] of its image
    int dc_needed = 0;
    h_img_cols.assign((size_t)n_images * 8, -1); h_img_pd.assign(n_images, 0);
    std::vector<int8_t> h_src((size_t)n_images * 8, -1);     // entry of the Jacobian row [rot3 | t3 | X3 | cam K] per column
    std::vector<int32_t> h_dc(n_images, 0);
    for (int i = 0; i < n_images; ++i) {
      std::vector<int> cols, src;
      if (h_pose_off[i] >= 0) {
        for (int k = 0; k < 3; ++k) { cols.push_back(h_pose_off[i] + k); src.push_back(k); }
        int la = 3;
        for (int k = 0; k < 3; ++k) if (!(d->tvec_const_mask[i] & (1u << k))) { cols.push_back(h_pose_off[i] + la++); src.push_back(3 + k); }
      }
      const int pd = (int)cols.size();
      const int cam_i = d->img_cam[i];
      if (h_intr_off[cam_i] >= 0) {
        const int kc = cam_num_params(d->cam_model[cam_i]);
        int la = 0;
        for (int k = 0; k < kc; ++k) if (!(cmask[cam_i] & (1u << k))) { cols.push_back(h_intr_off[cam_i] + la++); src.push_back(9 + k); }
      }
      dc_needed = std::max(dc_needed, (int)cols.size());
      h_img_pd[i] = pd;
      h_dc[i] = (int32_t)cols.size();
      for (size_t k = 0; k < cols.size() && k < 8; ++k) { h_img_cols[(size_t)i * 8 + k] = cols[k]; h_src[(size_t)i * 8 + k] = (int8_t)src[k]; }
    }
    img_dc_max = dc_needed;
    if (dc_needed <= 8) {
      PXR_TRY(img_cols8.upload(h_img_cols.data(), h_img_cols.size(), s));
      PXR_TRY(img_src8.upload(h_src.data(), h_src.size(), s));
      PXR_TRY(img_dc8.upload(h_dc.data(), h_dc.size(), s));
      PXR_CUDA(cudaStreamSynchronize(s));   // h_src / h_dc are locals
    }
    h_img_cam.assign(d->img_cam, d->img_cam + n_images);
    // implicit block-sparse reduced system: on request, or when the dense one would not fit comfortably
    sparse_schur = for_solve && use_pcg && dc_needed <= 8 && (n_obs > 0 || ctx->world > 1) &&
                   (env.pcg_sparse || (int64_t)nc * nc * 8 > (int64_t)4e9);
    // block mode: image-block assembly + ONE all-reduce per LM iteration (pxr_block.cuh).  Always on with several ranks
    // (the image tables are replicated, so every rank takes the same decision); PXR_BLOCK_ASSEMBLY=1 runs the same code on
    // one GPU (tests).  Images with more than 8 camera columns keep the dense multi-collective path.
    deterministic = for_solve && opt.deterministic != 0;
    if (deterministic && dc_needed > 8)
      return fail(PXR_ERR_UNSUPPORTED, "deterministic assembly needs <= 8 camera columns per image (pose 6 + intrinsics), got %d", dc_needed);
    block_mode = for_solve && dc_needed <= 8 && (ctx->world > 1 || deterministic || getenv("PXR_BLOCK_ASSEMBLY") != nullptr);
    if (ctx->world > 1 && sparse_schur && !block_mode) sparse_schur = false;
    if (!sparse_schur && (int64_t)nc * nc * 8 > (int64_t)40e9)
      return fail(PXR_ERR_UNSUPPORTED, "reduced camera system too large for the dense path (nc=%d) and the block-sparse path needs ITERATIVE_SCHUR with <= 8 camera columns per image", nc);
  }
  if (!sparse_schur && !block_mode) PXR_TRY(Hcc.alloc((size_t)nc * nc));
  PXR_TRY(gc.alloc(nc));
  PXR_TRY(Hpp.alloc((size_t)n_points * 9)); PXR_TRY(gp.alloc((size_t)n_points * 3));
  h_obs_img.assign(d->obs_img, d->obs_img + n_obs);
  if (for_solve) PXR_TRY(build_schur_pairs());
  if (block_mode) PXR_TRY(block_setup());
  if (for_solve && n_obs > 0 && n_obs < ((int64_t)1 << 31)) {
    // per-image observation chunks for the camera-block build (ba_build_cam_kernel): images whose pose and
    // intrinsics are both constant contribute nothing and are left out; usable when every image has <= 8 columns
    int dc_needed = 0;
    std::vector<int> img_dc(n_images, 0);
    for (int i = 0; i < n_images; ++i) {
      int dc = 0;
      if (h_pose_off[i] >= 0) dc += 3 + (3 - __builtin_popcount(d->tvec_const_mask[i] & 7u));
      const int cam_i = d->img_cam[i];
      if (h_intr_off[cam_i] >= 0) dc += cam_num_params(d->cam_model[cam_i]) - __builtin_popcount(cmask[cam_i]);
      img_dc[i] = dc;
      dc_needed = std::max(dc_needed, dc);
    }
    if (dc_needed <= 8) {
      std::vector<int64_t> cnt(n_images + 1, 0);
      for (int64_t o = 0; o < n_obs; ++o) if (img_dc[d->obs_img[o]] > 0) cnt[d->obs_img[o] + 1]++;
      for (int i = 0; i < n_images; ++i) cnt[i + 1] += cnt[i];
      std::vector<int32_t> list(cnt[n_images]);
      {
        std::vector<int64_t> cur_pos(cnt.begin(), cnt.end() - 1);
        for (int64_t o = 0; o < n_obs; ++o) if (img_dc[d->obs_img[o]] > 0) list[cur_pos[d->obs_img[o]]++] = (int32_t)o;
      }
      std::vector<int64_t> cb;
      h_img_chunk_begin.assign((size_t)n_images + 1, 0);
      for (int i = 0; i < n_images; ++i) {
        h_img_chunk_begin[i] = (int64_t)cb.size();
        for (int64_t b = cnt[i]; b < cnt[i + 1]; b += 128) cb.push_back(b);
      }
      h_img_chunk_begin[n_images] = (int64_t)cb.size();
      cb.push_back(cnt[n_images]);
      io_n_chunks = (int64_t)cb.size() - 1;
      if (io_n_chunks > 0) {
        PXR_TRY(io_obs.upload(list.data(), list.size(), s));
        PXR_TRY(io_chunk_begin.upload(cb.data(), cb.size(), s));
        PXR_CUDA(cudaStreamSynchronize(s));   // host vectors go out of scope
      }
      if (deterministic) {                    // fixed-order reduction of the camera-block chunk partials (pxr_block.cuh)
        PXR_TRY(det_cam_part.alloc((size_t)std::max<int64_t>(io_n_chunks, 1) * 48));
        PXR_TRY(det_img_chunk_begin.upload(h_img_chunk_begin.data(), h_img_chunk_begin.size(), s));
        PXR_CUDA(cudaStreamSynchronize(s));
      }
    }
  }
  PXR_TRY(W.alloc((size_t)n_obs * dcmax * 3)); PXR_TRY(Wcols.alloc((size_t)n_obs * dcmax)); PXR_TRY(Wdc.alloc(n_obs));
  if (!sparse_schur) PXR_TRY(S.alloc((size_t)(nc + 1) * nc));   // block mode: filled from the global blocks (blk_gather_kernel)
  PXR_TRY(rhs.alloc(nc));
  PXR_TRY(diag.alloc(nl)); PXR_TRY(jscale.alloc(nl)); PXR_TRY(D2.alloc(nl)); PXR_TRY(delta.alloc(nl));
  PXR_TRY(partials.alloc(fm_max_partials(ctx)));
  if (deterministic) {
    const int64_t big = std::max<int64_t>({n_obs, n_points * 3, (int64_t)n_images * 4, (int64_t)n_cameras * kMaxK});
    PXR_TRY(det_scal_part.alloc((size_t)(cdiv(big, 128) * 4 + 16)));
    if (io_n_chunks == 0 && n_obs > 0) return fail(PXR_ERR_UNSUPPORTED, "deterministic assembly needs the per-image chunk lists (problem too large for 32-bit observation ids)");
  }
  PXR_TRY(scalars.alloc(16));
  PXR_TRY(flags.alloc(4));
  PXR_TRY(rdiag.alloc(kNB));
  PXR_TRY(Hpp.zero(s)); PXR_TRY(gp.zero(s)); PXR_TRY(obs_out.zero(s));
  PXR_CUDA(cudaStreamSynchronize(s));
  if (res_thread.joinable()) {       // the window upload runs beside all of the above
    res_thread.join();
    if (res_thread_rc != PXR_OK) return fail(res_thread_rc, "%s", res_thread_err.c_str());
  }
  h2d_bytes = h2d;
  return PXR_OK;
}

// Static structure of the Schur complement: every pair of observations (i >= j) of a variable point,
// grouped by the (image_i, image_j) pair they address in the reduced camera system; long groups are
// split into chunks of at most kChunk entries (one warp each).
int BA::build_schur_pairs() {
  if (sp_built) return PXR_OK;
  PXR_TRY(Tbuf.alloc((size_t)n_obs * dcmax * 3));
  PXR_TRY(Hinv.alloc((size_t)std::max<int64_t>(n_points, 1) * 6));
  const int64_t kChunk = 128;
  const int64_t ni = n_images;
  auto key_of = [&](int ia, int ib, bool self) -> int64_t {  // ia >= ib
    return ((int64_t)ia * (ia + 1) / 2 + ib) * 2 + (self ? 1 : 0);
  };
  const int64_t n_keys = (ni * (ni + 1) / 2) * 2;
  std::vector<int64_t> count(n_keys + 1, 0);
  int64_t total = 0;
  for (int64_t p = 0; p < n_points; ++p) {
    if (h_point_off[p] < 0) continue;
    for (int64_t i = h_pt_begin[p]; i < h_pt_begin[p + 1]; ++i)
      for (int64_t j = h_pt_begin[p]; j <= i; ++j) {
        const int a = h_obs_img[i], b = h_obs_img[j];
        count[key_of(std::max(a, b), std::min(a, b), i == j) + 1]++;
        ++total;
      }
  }
  if (total >= ((int64_t)1 << 31) || n_obs >= ((int64_t)1 << 31) || n_points >= ((int64_t)1 << 31))
    return fail(PXR_ERR_UNSUPPORTED, "too many observation pairs for 32-bit pair indices");
  for (int64_t k = 0; k < n_keys; ++k) count[k + 1] += count[k];
  std::vector<int32_t> px(total), py(total), pp(total);
  {
    std::vector<int64_t> cursor(count.begin(), count.end() - 1);
    for (int64_t p = 0; p < n_points; ++p) {
      if (h_point_off[p] < 0) continue;
      for (int64_t i = h_pt_begin[p]; i < h_pt_begin[p + 1]; ++i)
        for (int64_t j = h_pt_begin[p]; j <= i; ++j) {
          const int a = h_obs_img[i], b = h_obs_img[j];
          const int64_t k = cursor[key_of(std::max(a, b), std::min(a, b), i == j)]++;
          // x = the observation in the image with the larger index
          if (a >= b) { px[k] = (int32_t)i; py[k] = (int32_t)j; } else { px[k] = (int32_t)j; py[k] = (int32_t)i; }
          pp[k] = (int32_t)p;
        }
    }
  }
  std::vector<int64_t> cb;
  std::vector<uint8_t> cself;
  std::vector<int32_t> ckey, ka, kbv;      // sparse path: compact id of every non-empty (image pair, self) key
  std::vector<uint8_t> kself;
  {
    int64_t k = 0;
    for (int64_t ia = 0; ia < ni; ++ia)
      for (int64_t ib = 0; ib <= ia; ++ib)
        for (int self = 0; self < 2; ++self, ++k) {
          if (count[k + 1] == count[k]) continue;
          if (sparse_schur || block_mode) { ka.push_back((int32_t)ia); kbv.push_back((int32_t)ib); kself.push_back((uint8_t)self); h_key_code_local.push_back(k); }
          for (int64_t s = count[k]; s < count[k + 1]; s += kChunk) {
            cb.push_back(s); cself.push_back((uint8_t)self);
            if (sparse_schur || block_mode) ckey.push_back((int32_t)ka.size() - 1);
          }
        }
  }
  cb.push_back(total);
  if (block_mode) {
    // the key list becomes the union over the ranks, the blocks live in the packed buffer (block_setup)
    h_key_a = ka; h_key_b = kbv; h_key_self = kself;
    PXR_TRY(ss_chunk_key.upload(ckey.data(), ckey.size(), ctx->stream));     // local ids for now; block_setup remaps them
    PXR_CUDA(cudaStreamSynchronize(ctx->stream));
    h_chunk_key_local = ckey;
  } else if (sparse_schur) {
    ss_n_keys = (int)ka.size();
    PXR_TRY(ss_key_a.upload(ka.data(), ka.size(), ctx->stream)); PXR_TRY(ss_key_b.upload(kbv.data(), kbv.size(), ctx->stream));
    PXR_TRY(ss_key_self.upload(kself.data(), kself.size(), ctx->stream));
    PXR_TRY(ss_chunk_key.upload(ckey.data(), ckey.size(), ctx->stream));
    PXR_TRY(ss_Bk.alloc((size_t)std::max(ss_n_keys, 1) * 64));
    PXR_TRY(ss_Himg.alloc((size_t)n_images * 64));
    PXR_TRY(ss_img_cols.upload(h_img_cols.data(), h_img_cols.size(), ctx->stream));
    PXR_TRY(ss_img_pd.upload(h_img_pd.data(), h_img_pd.size(), ctx->stream));
    PXR_CUDA(cudaStreamSynchronize(ctx->stream));
  }
  sp_n_chunks = (int64_t)cself.size();
  cudaStream_t s = ctx->stream;
  PXR_TRY(sp_px.upload(px.data(), px.size(), s));
  PXR_TRY(sp_py.upload(py.data(), py.size(), s));
  PXR_TRY(sp_pp.upload(pp.data(), pp.size(), s));
  PXR_TRY(sp_chunk_begin.upload(cb.data(), cb.size(), s));
  PXR_TRY(sp_chunk_self.upload(cself.data(), cself.size(), s));
  PXR_CUDA(cudaStreamSynchronize(s));  // host vectors go out of scope
  sp_built = true;
  return PXR_OK;
}

SchurPairs BA::schur_pairs() {
  SchurPairs sp;
  sp.px = sp_px.p; sp.py = sp_py.p; sp.pp = sp_pp.p; sp.chunk_begin = sp_chunk_begin.p; sp.chunk_self = sp_chunk_self.p;
  sp.n_chunks = sp_n_chunks;
  return sp;
}

// -------------------------------------------------------------------------------- evaluation
int BA::project(int set, bool jac, double* xy_out) {
  ProjectArgs a;
  a.obs_img = obs_img.p; a.obs_pt = obs_pt.p; a.obs_patch = obs_patch.p;
  a.img_cam = img_cam.p; a.cam_model = cam_model.p;
  a.cam_params = cam[set].p; a.qvec = q[set].p; a.tvec = t[set].p; a.xyz = X[set].p;
  a.corner = corner.p; a.scale = scale.p; a.ups = ups;
  a.obs_begin = 0; a.obs_end = n_obs; a.item_index = nullptr;
  a.uv = uv.p; a.xy = xy_out; a.juv = jac ? juv.p : nullptr; a.juv_stride = juv_stride; a.juv_k = K;
  if (geometric) a.xy = geo_xy.p;     // the geometric residual is formed from the projection itself
  if (n_obs == 0) return PXR_OK;
  StageScope st(this, 2);
  const size_t staged_smem = (size_t)128 * (juv_stride | 1) * sizeof(double);
  if (jac && env.project_staged && staged_smem <= 48 * 1024)
    PXR_LAUNCH(ctx, ba_project_staged_kernel, (unsigned)cdiv(n_obs, 128), 128, staged_smem, a);
  else if (jac) PXR_LAUNCH(ctx, ba_project_kernel<true>, (unsigned)cdiv(n_obs, 128), 128, 0, a);
  else PXR_LAUNCH(ctx, ba_project_kernel<false>, (unsigned)cdiv(n_obs, 128), 128, 0, a);
  PXR_CUDA(cudaGetLastError());
  if (geometric && xy_out) PXR_CUDA(cudaMemcpyAsync(xy_out, geo_xy.p, (size_t)n_obs * 16, cudaMemcpyDeviceToDevice, ctx->stream));
  return PXR_OK;
}

// ---- window residency -----------------------------------------------------------------------------------------
int BA::resident_setup(const pxr_ba_desc* d, size_t esz) {
  resident = false;
  if (!allow_resident || n_obs == 0) return PXR_OK;
  if (const char* v = getenv("PXR_RESIDENT_WINDOW")) { const int e = std::atoi(v); if (e == 0 || !res_window_fixed) res_window = e; }
  const int W = res_window;
  if (W < 4 || C < 8 || ph > 255 || pw > 255 || ph < W + 2 || pw < W + 2) return PXR_OK;       // nothing to gain / not representable
  if ((size_t)ph * pw * C * esz > staged_chunk_bytes()) return PXR_OK;      // a whole (shared) patch must fit a staging buffer
  // the blocks must be HOST memory (a device-resident block needs no upload at all)
  auto is_device = [](const void* ptr) -> bool {
    cudaPointerAttributes pa;
    if (cudaPointerGetAttributes(&pa, ptr) != cudaSuccess) { cudaGetLastError(); return false; }
    return pa.type == cudaMemoryTypeDevice || pa.type == cudaMemoryTypeManaged;
  };
  res_srcs.clear(); res_block_first.assign(1, 0);
  if (d->n_patch_blocks > 0) {
    for (int b = 0; b < d->n_patch_blocks; ++b) {
      if (is_device(d->patch_block_ptrs[b])) return PXR_OK;
      res_srcs.push_back(d->patch_block_ptrs[b]);
      res_block_first.push_back(res_block_first.back() + d->patch_block_counts[b]);
    }
  } else {
    if (is_device(d->patches)) return PXR_OK;
    res_srcs.push_back(d->patches);
    res_block_first.push_back(n_patches);
  }
  res_esz = esz;
  cudaStream_t s = ctx->stream;
  // patches several observations read are brought over whole
  std::vector<uint8_t> shared((size_t)n_patches, 0);
  if (d->obs_patch) {
    h_obs_patch.assign(d->obs_patch, d->obs_patch + n_obs);
    std::vector<uint8_t> seen((size_t)n_patches, 0);
    for (int64_t o = 0; o < n_obs; ++o) { const int64_t p = d->obs_patch[o]; if (seen[p]) shared[p] = 1; seen[p] = 1; }
  }
  PXR_TRY(res_shared.upload(shared.data(), shared.size(), s));
  PXR_CUDA(cudaStreamSynchronize(s));             // `shared` is a local
  PXR_TRY(res_rect.alloc((size_t)n_patches)); PXR_TRY(res_rect.zero(s));
  PXR_TRY(res_viol_count.alloc(1)); PXR_TRY(res_viol_count.zero(s));
  PXR_TRY(res_viol_list.alloc((size_t)n_obs)); PXR_TRY(res_fix_list.alloc((size_t)n_obs));
  resident = true;
  return PXR_OK;
}

// K0 at the initial parameters -> rectangle of every patch -> packed window upload on its own thread (joined when
// create() returns), so the host-side layout work of create() overlaps it as it overlaps the plain slab upload
int BA::resident_begin(cudaStream_t us, double* h2d_patch) {
  cudaStream_t s = ctx->stream;
  ProjectArgs pa;
  pa.obs_img = obs_img.p; pa.obs_pt = obs_pt.p; pa.obs_patch = obs_patch.p; pa.img_cam = img_cam.p; pa.cam_model = cam_model.p;
  pa.cam_params = cam[0].p; pa.qvec = q[0].p; pa.tvec = t[0].p; pa.xyz = X[0].p;
  pa.corner = corner.p; pa.scale = scale.p; pa.ups = ups; pa.obs_begin = 0; pa.obs_end = n_obs; pa.item_index = nullptr;
  pa.uv = uv.p; pa.xy = nullptr; pa.juv = nullptr; pa.juv_stride = juv_stride; pa.juv_k = K;
  PXR_LAUNCH(ctx, ba_project_kernel<false>, (unsigned)cdiv(n_obs, 128), 128, 0, pa);
  PXR_LAUNCH(ctx, resident_rect_kernel, (unsigned)cdiv(n_obs, 256), 256, 0, uv.p, obs_patch.p, res_shared.p, n_obs, ph, pw, res_window, res_rect.p);
  PXR_CUDA(cudaGetLastError());
  auto h_rect = std::make_shared<std::vector<uint32_t>>((size_t)n_patches);
  PXR_CUDA(cudaMemcpyAsync(h_rect->data(), res_rect.p, (size_t)n_patches * 4, cudaMemcpyDeviceToHost, s));
  PXR_CUDA(cudaStreamSynchronize(s));
  double bytes = 0;
  for (uint32_t rc : *h_rect) bytes += (double)((rc >> 16) & 255u) * (double)(rc >> 24) * C * (double)res_esz;
  *h2d_patch = bytes;
  res_thread_rc = PXR_OK;
  pxr_ctx* c = ctx;
  uint8_t* slab = patches_owned.p;
  const uint32_t* d_rect = res_rect.p;
  const int64_t np = n_patches; const int ph_ = ph, pw_ = pw, tap = C * (int)res_esz;
  res_thread = std::thread([this, c, slab, d_rect, np, ph_, pw_, tap, us, h_rect]() {
    cudaSetDevice(c->device);
    res_thread_rc = upload_windows(c, slab, res_srcs.data(), res_block_first.data(), (int)res_srcs.size(), h_rect->data(), d_rect,
                                   np, ph_, pw_, tap, nullptr, us);
    if (res_thread_rc != PXR_OK) res_thread_err = pxr_last_error();
  });
  return PXR_OK;
}

void BA::resident_args(FmEvalArgs& a) {
  if (!resident) return;
  a.res_rect = res_rect.p; a.viol_count = res_viol_count.p; a.viol_list = res_viol_list.p; a.viol_capacity = (long long)n_obs;
}

// Called after an evaluation pass: did any observation read outside its resident rectangle?  Then fetch those
// patches whole; the caller evaluates the listed observations (res_fix_list[0 .. n_fixed)) again.
int BA::resident_fix(int64_t* n_fixed) {
  *n_fixed = 0;
  if (!resident) return PXR_OK;
  cudaStream_t s = ctx->stream;
  unsigned long long n = 0;
  PXR_CUDA(cudaMemcpyAsync(&n, res_viol_count.p, sizeof(n), cudaMemcpyDeviceToHost, s));
  PXR_CUDA(cudaStreamSynchronize(s));
  if (n == 0) return PXR_OK;
  n = std::min<unsigned long long>(n, (unsigned long long)n_obs);      // entries beyond the capacity were dropped (reported again later)
  std::vector<int64_t> list((size_t)n);
  PXR_CUDA(cudaMemcpyAsync(list.data(), res_viol_list.p, (size_t)n * 8, cudaMemcpyDeviceToHost, s));
  PXR_CUDA(cudaMemcpyAsync(res_fix_list.p, res_viol_list.p, (size_t)n * 8, cudaMemcpyDeviceToDevice, s));
  PXR_CUDA(cudaMemsetAsync(res_viol_count.p, 0, sizeof(unsigned long long), s));
  PXR_CUDA(cudaStreamSynchronize(s));
  const size_t patch_bytes = (size_t)ph * pw * C * res_esz;
  // an observation is reported by every pass that evaluates it before its patch is whole (several inner-iteration rounds
  // run between two looks at the list): fetch each patch once
  if (res_whole.size() != (size_t)n_patches) res_whole.assign((size_t)n_patches, 0);
  int64_t fetched = 0;
  for (int64_t o : list) {
    const int64_t p = h_obs_patch.empty() ? o : h_obs_patch[(size_t)o];
    if (res_whole[(size_t)p]) continue;
    res_whole[(size_t)p] = 1; ++fetched;
    const size_t blk = (size_t)(std::upper_bound(res_block_first.begin(), res_block_first.end(), p) - res_block_first.begin()) - 1;
    const uint8_t* src = (const uint8_t*)res_srcs[blk] + (size_t)(p - res_block_first[blk]) * patch_bytes;
    PXR_CUDA(cudaMemcpyAsync(patches_owned.p + (size_t)p * patch_bytes, src, patch_bytes, cudaMemcpyHostToDevice, s));
  }
  PXR_LAUNCH(ctx, resident_mark_full_kernel, (unsigned)cdiv((int64_t)n, 256), 256, 0, res_fix_list.p, (int64_t)n, obs_patch.p, ph, pw, res_rect.p);
  PXR_CUDA(cudaGetLastError());
  res_refetched += fetched; res_passes_repeated++;
  h2d_bytes += (double)fetched * (double)patch_bytes;
  *n_fixed = (int64_t)n;
  return PXR_OK;
}

int BA::fm(int mode, double* residuals_out, double* cost_dev, double* grad_out) {
  PXR_TRY(fm_k1(mode, residuals_out, grad_out, nullptr, n_obs));
  for (;;) {      // window residency: observations that left their window are evaluated again once their patch is whole
    int64_t n_fixed = 0;
    PXR_TRY(resident_fix(&n_fixed));
    if (n_fixed == 0) break;
    PXR_TRY(fm_k1(mode, residuals_out, grad_out, res_fix_list.p, n_fixed));
  }
  return fm_cost(cost_dev);
}

int BA::fm_k1(int mode, double* residuals_out, double* grad_out, const int64_t* list, int64_t n) {
  if (n <= 0 || n_obs == 0) return PXR_OK;
  if (geometric) {
    StageScope st(this, mode ? 1 : 0);
    return geo_k1(mode, residuals_out, grad_out, list, n);
  }
  FmEvalArgs a;
  a.uv = uv.p; a.item_patch = obs_patch.p; a.item_ref = obs_pt.p;
  a.patches = d_patches; a.ph = ph; a.pw = pw;
  a.refs = has_refs ? refs.p : nullptr;
  a.begin = 0; a.end = n; a.item_index = list;
  a.out = obs_out.p; a.residuals = residuals_out; a.desc = nullptr; a.grad = grad_out;
  a.loss.type = opt.loss_type; a.loss.a = opt.loss_scale;
  a.l2_normalize = interp.l2_normalize;
  resident_args(a);
  int np = 0;
  StageScope st(this, mode ? 1 : 0);
  return launch_fm_eval(ctx, dtype, C, mode, interp.use_float_simd != 0, a, &np);
}

// K1 of a geometric handle (pxr_geo.cuh) over all observations or a list; with n_dev the list length is read on the
// device and n is the upper bound the grid is sized for
int BA::geo_k1(int mode, double* residuals_out, double* grad_out, const int64_t* list, int64_t n, const unsigned long long* n_dev) {
  if (n <= 0) return PXR_OK;
  GeoEvalArgs a;
  a.xy = geo_xy.p; a.target = geo_target.p;
  a.begin = 0; a.end = n; a.item_index = list; a.end_dev = n_dev;
  a.out = obs_out.p; a.residuals = residuals_out; a.grad = grad_out;
  const unsigned grid = (unsigned)std::min<int64_t>(cdiv(n, 128), (int64_t)ctx->sm_count * 16);
  if (mode == 1) PXR_LAUNCH(ctx, geo_eval_kernel<1>, grid, 128, 0, a);
  else PXR_LAUNCH(ctx, geo_eval_kernel<0>, grid, 128, 0, a);
  PXR_CUDA(cudaGetLastError());
  return PXR_OK;
}

int BA::fm_cost(double* cost_dev /* device scalar */) {
  if (n_obs > 0) {
    StageScope st2(this, 10);
    LossParams loss; loss.type = opt.loss_type; loss.a = opt.loss_scale;
    const int cb = std::min<int>(fm_max_partials(ctx), ctx->sm_count * 8);
    PXR_LAUNCH(ctx, cost_from_sq_norm_kernel, cb, 256, 0, obs_out.p, (int64_t)0, n_obs, loss, partials.p);
    PXR_LAUNCH(ctx, reduce_partials_kernel, 1, 1024, 0, partials.p, (int64_t)cb, cost_dev);
  } else {
    PXR_CUDA(cudaMemsetAsync(cost_dev, 0, 8, ctx->stream));
  }
  return PXR_OK;
}

// cost (and with jac the full linearisation) at parameter set `set`; returns the global cost
int BA::evaluate(int set, bool jac, double* cost_out) {
  PXR_TRY(project(set, jac, nullptr));
  PXR_TRY(fm(jac ? 1 : 0, nullptr, scalars.p + 0));
  if (jac) PXR_TRY(build());
  if (block_mode) return global_cost_block(cost_out);
  PXR_TRY(allreduce_f64(ctx, scalars.p + 0, 1));
  double c = 0;
  PXR_CUDA(cudaMemcpyAsync(&c, scalars.p + 0, 8, cudaMemcpyDeviceToHost, ctx->stream));
  PXR_CUDA(cudaStreamSynchronize(ctx->stream));
  *cost_out = c;
  return PXR_OK;
}

BADev BA::dev() {
  BADev d;
  d.n_cameras = n_cameras; d.n_images = n_images; d.K = K; d.n_points = n_points; d.n_obs = n_obs;
  d.nc = nc; d.nl = (int)nl; d.dcmax = dcmax; d.juv_stride = juv_stride;
  d.obs_img = obs_img.p; d.obs_pt = obs_pt.p; d.img_cam = img_cam.p; d.cam_model = cam_model.p;
  d.cam_mask = cam_mask.p; d.tmask = tmask.p; d.pose_off = pose_off.p; d.intr_off = intr_off.p;
  d.point_off = point_off.p; d.pt_begin = pt_begin.p; d.obs_out = obs_out.p; d.juv = juv.p;
  d.img_cols8 = img_cols8.p; d.img_src8 = img_src8.p; d.img_dc8 = img_dc8.p;
  d.Hcc = Hcc.p; d.Hpp = Hpp.p; d.gp = gp.p; d.W = W.p; d.Wcols = Wcols.p; d.Wdc = Wdc.p;
  d.gc = block_mode ? pack_local.p + pk_off_gc : gc.p;   // block mode: the partial gradient lives in the packed buffer
  d.loss.type = opt.loss_type; d.loss.a = opt.loss_scale;
  return d;
}

int BA::build() {
  if (block_mode) return build_block();
  StageScope st(this, 3);
  if (!sparse_schur) PXR_TRY(Hcc.zero(ctx->stream));
  PXR_TRY(gc.zero(ctx->stream));
  PXR_TRY(Hpp.zero(ctx->stream));
  PXR_TRY(gp.zero(ctx->stream));
  const bool chunked = io_n_chunks > 0 && (sparse_schur || !env.build_atomic);
  if (sparse_schur && !chunked && n_obs > 0) return fail(PXR_ERR_INTERNAL, "block-sparse path without per-image chunks");
  if (sparse_schur) PXR_TRY(ss_Himg.zero(ctx->stream));
  if (n_obs > 0) {
    const BADev dv = dev();
    const size_t staged_smem = (size_t)128 * ((std::max(dv.juv_stride, dv.dcmax * 3) | 1) + 9) * sizeof(double);
    if (img_src8.p && chunked && env.build_staged && staged_smem <= 48 * 1024)
      PXR_LAUNCH(ctx, ba_build_staged_kernel, (unsigned)cdiv(n_obs, 128), 128, staged_smem, dv);
    else if (img_src8.p) PXR_LAUNCH(ctx, ba_build_kernel<true>, (unsigned)cdiv(n_obs, 128), 128, 0, dv, chunked ? 0 : 1);
    else PXR_LAUNCH(ctx, ba_build_kernel<false>, (unsigned)cdiv(n_obs, 128), 128, 0, dv, chunked ? 0 : 1);
  }
  if (n_obs > 0 && chunked)
    PXR_LAUNCH(ctx, ba_build_cam_kernel, (unsigned)cdiv(io_n_chunks * 32, 256), 256, 0, dev(), io_obs.p, io_chunk_begin.p, io_n_chunks,
               sparse_schur ? ss_Himg.p : nullptr);
  const int64_t n = std::max<int64_t>(nc, n_points);
  if (sparse_schur && nc > 0) PXR_CUDA(cudaMemsetAsync(diag.p, 0, (size_t)nc * 8, ctx->stream));
  if (n > 0) PXR_LAUNCH(ctx, ba_diag_kernel, (unsigned)cdiv(n, 256), 256, 0, dev(), diag.p);
  if (sparse_schur && nc > 0) PXR_LAUNCH(ctx, sp_diag_kernel, (unsigned)cdiv((int64_t)n_images * 8, 256), 256, 0, sparse(), diag.p);
  if (ctx->world > 1 && nc > 0) {
    // multi-GPU: Hcc stays a per-rank partial sum (it only ever enters the reduced system, which is all-reduced
    // anyway); globally needed are its diagonal (Jacobi scaling / LM damping) and the gradient
    if (!gc_local.p) { PXR_TRY(gc_local.alloc(nc)); PXR_TRY(ar_buf.alloc((size_t)2 * nc)); }
    PXR_CUDA(cudaMemcpyAsync(gc_local.p, gc.p, (size_t)nc * 8, cudaMemcpyDeviceToDevice, ctx->stream));
    // one collective for [diag(Hcc) | gc]
    PXR_CUDA(cudaMemcpyAsync(ar_buf.p, diag.p, (size_t)nc * 8, cudaMemcpyDeviceToDevice, ctx->stream));
    PXR_CUDA(cudaMemcpyAsync(ar_buf.p + nc, gc.p, (size_t)nc * 8, cudaMemcpyDeviceToDevice, ctx->stream));
    PXR_TRY(allreduce_f64(ctx, ar_buf.p, (size_t)2 * nc));
    PXR_CUDA(cudaMemcpyAsync(diag.p, ar_buf.p, (size_t)nc * 8, cudaMemcpyDeviceToDevice, ctx->stream));
    PXR_CUDA(cudaMemcpyAsync(gc.p, ar_buf.p + nc, (size_t)nc * 8, cudaMemcpyDeviceToDevice, ctx->stream));
  }
  PXR_CUDA(cudaGetLastError());
  return PXR_OK;
}

SparseSchur BA::sparse() {
  SparseSchur q;
  q.n_images = n_images; q.n_keys = ss_n_keys; q.nc = nc;
  q.img_cols = ss_img_cols.p; q.img_pd = ss_img_pd.p; q.img_pose_blk = ss_img_pose_blk.p; q.img_cam_blk = ss_img_cam_blk.p;
  q.key_a = ss_key_a.p; q.key_b = ss_key_b.p; q.key_self = ss_key_self.p;
  q.Himg = ss_Himg.p; q.Bk = ss_Bk.p;
  return q;
}

// Dense Cholesky of [S; rhs] + both substitutions (pxr_chol.cuh) -> delta[0..nc): captured once into a CUDA graph.
int BA::chol_launch() {
  cudaStream_t s = ctx->stream;
    // The factorisation + back-substitution is a fixed sequence of ~3*nc/32 dependent launches: it is
    // captured once into a CUDA graph and replayed, which removes the per-launch gaps.
    if (!chol_graph_exec) {
      chol_multikernel = chol_force_multikernel || env.chol_multikernel;
      if (!chol_multikernel) {
        // every CTA of the persistent kernel must be resident at once: grid = occupancy x SMs
        int per_sm = 0, sms = 0, dev = 0;
        PXR_CUDA(cudaGetDevice(&dev));
        PXR_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
        chol_band = getenv("PXR_CHOL_BAND") != nullptr;     // the band design (pxr_chol2.cuh) is opt-in: see DESIGN.md section 3
        if (chol_band) {
          PXR_CUDA(cudaFuncSetAttribute(pxr_chol2::chol_band_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pxr_chol2::smem_bytes()));
          PXR_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, pxr_chol2::chol_band_kernel, pxr_chol::kThreads, pxr_chol2::smem_bytes()));
        } else {
          PXR_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, pxr_chol::chol_persistent_kernel, pxr_chol::kThreads, 0));
        }
        if (per_sm < 1) return pxr::fail(PXR_ERR_CUDA, "persistent Cholesky kernel does not fit on an SM");
        const int nbt = (int)cdiv(nc, kNB);
        const int64_t tiles = (int64_t)(nbt + 1) * nbt / 2 + nbt;
        chol_grid = (int)std::min<int64_t>((int64_t)per_sm * sms, std::max<int64_t>(2, tiles + 1));
        PXR_TRY(chol_sync.alloc(pxr_chol::sync_ints(nbt)));
        if (!env.chol_trace.empty()) { PXR_TRY(chol_trace.alloc((size_t)(nbt + 3) * 8 + nbt)); PXR_TRY(chol_trace.zero(s)); }
      }
      cudaGraph_t graph = nullptr;
      PXR_CUDA(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
      // an error between Begin and EndCapture must not leave the context's stream capturing
      struct CaptureGuard { cudaStream_t s; bool armed = true; ~CaptureGuard() { if (armed) { cudaGraph_t g = nullptr; cudaStreamEndCapture(s, &g); if (g) cudaGraphDestroy(g); } } } cap_guard{s};
      const int nb = (int)cdiv(nc, kNB);
      int64_t captured = 0;
      if (!chol_multikernel) {
        // one persistent kernel: tile DAG with flags (pxr_chol.cuh); the memset of the flags is part of the graph
        PXR_CUDA(cudaMemsetAsync(chol_sync.p, 0, chol_sync.n * sizeof(int), s));
        PXR_CUDA(cudaMemsetAsync(delta.p, 0xFF, (size_t)nc * 8, s));   // x doubles as its own ready flag (pxr_chol.cuh)
        pxr_chol::Args ca;
        ca.A = S.p; ca.x = delta.p; ca.n = nc; ca.nb = nb;
        ca.diag_ready = chol_sync.p; ca.ready = ca.diag_ready + nb; ca.upd = ca.ready + (size_t)(nb + 1) * nb;
        ca.xready = ca.upd + (size_t)(nb + 1) * nb; ca.abort = ca.xready + nb; ca.fail_flag = flags.p + 1; ca.trace = chol_trace.p;
        if (chol_band) pxr_chol2::chol_band_kernel<<<chol_grid, pxr_chol::kThreads, pxr_chol2::smem_bytes(), s>>>(ca);
        else pxr_chol::chol_persistent_kernel<<<chol_grid, pxr_chol::kThreads, 0, s>>>(ca);
        ++captured;
      } else {
      for (int k = 0; k < nb; ++k) {
        const int k0 = k * kNB, kb = std::min(kNB, nc - k0);
        const int rows_below = nc + 1 - (k0 + kb);               // includes the rhs row
        chol_diag_kernel<<<1, 32, 0, s>>>(S.p, nc, k, rdiag.p, flags.p + 1); ++captured;
        if (rows_below > 0) { chol_panel_kernel<<<(unsigned)cdiv(rows_below, kNB), kPanelThreads, 0, s>>>(S.p, nc, nc + 1, k, rdiag.p); ++captured; }
        const int nrb = (int)cdiv(nc + 1, kNB);
        const int rem = nrb - (k + 1);
        if (rem > 0 && kb == kNB) { chol_update_kernel<<<rem * (rem + 1) / 2, kNB * kNB, 0, s>>>(S.p, nc, nc + 1, k); ++captured; }
      }
      chol_backsolve_kernel<<<1, 1024, 0, s>>>(S.p, S.p + (size_t)nc * nc, delta.p, nc); ++captured;
      }
      cap_guard.armed = false;
      PXR_CUDA(cudaStreamEndCapture(s, &graph));
      PXR_CUDA(cudaGraphInstantiate(&chol_graph_exec, graph, 0));
      cudaGraphDestroy(graph);
      chol_graph_kernels = captured;
    }
    PXR_CUDA(cudaGraphLaunch(chol_graph_exec, s));
    ctx->launches += chol_graph_kernels;
    if (chol_trace.p) {   // debugging aid: dump the panel CTA's time line of this factorisation
      std::vector<long long> h(chol_trace.n);
      PXR_CUDA(cudaMemcpyAsync(h.data(), chol_trace.p, h.size() * 8, cudaMemcpyDeviceToHost, s));
      PXR_CUDA(cudaStreamSynchronize(s));
      if (FILE* f = fopen(env.chol_trace.c_str(), "w")) {
        const int nbt = (int)cdiv(nc, kNB);
        const int rows = chol_band ? nbt + 1 : nbt;      // the band kernel also walks the rhs row
        for (int k = 0; k < rows; ++k) { for (int q = 0; q < 7; ++q) fprintf(f, "%lld ", h[(size_t)k * 8 + q] - h[0]); fprintf(f, "\n"); }
        const size_t tail = (size_t)(chol_band ? nbt + 1 : nbt) * 8;
        fprintf(f, "backsolve_start %lld\n", h[tail] - h[0]);
        for (int c = nbt - 1; c >= 0; --c) fprintf(f, "x %d %lld\n", c, h[tail + 8 + c] - h[0]);
        fclose(f);
      }
    }
    return PXR_OK;
}

// S -= sum over observation pairs T_x W_y^T, rhs += sum T gp: the staged pair kernel when every image has at most 8
// columns (the usual case: pose + up to two intrinsics, or pose only), the direct kernels otherwise
int BA::launch_schur_pairs(const BADev& d) {
  if (sp_n_chunks <= 0) return PXR_OK;
  const unsigned pair_grid = (unsigned)cdiv(sp_n_chunks * 32, kPairThreads);
  const bool small = img_dc_max <= 8 && dcmax >= 9;   // dcmax = 6 + K >= 9 for every camera model: row 8 of a record exists
  if (small && schur_kernel == 0) {                   // fused tensor-core walk: no T buffer
    if (schur_ctas == 3) PXR_LAUNCH(ctx, (ba_schur_pairs_mma_kernel<3, true>), pair_grid, kPairThreads, 0, d, schur_pairs(), Hinv.p, S.p, rhs.p);
    else PXR_LAUNCH(ctx, (ba_schur_pairs_mma_kernel<4, true>), pair_grid, kPairThreads, 0, d, schur_pairs(), Hinv.p, S.p, rhs.p);
    return PXR_OK;
  }
  PXR_LAUNCH(ctx, ba_schur_prep_kernel, (unsigned)cdiv(n_obs * dcmax, 256), 256, 0, d, Hinv.p, Tbuf.p);
  if (small && schur_kernel == 3) {
    if (schur_ctas == 4) PXR_LAUNCH(ctx, (ba_schur_pairs_mma_kernel<4, false>), pair_grid, kPairThreads, 0, d, schur_pairs(), Tbuf.p, S.p, rhs.p);
    else PXR_LAUNCH(ctx, (ba_schur_pairs_mma_kernel<3, false>), pair_grid, kPairThreads, 0, d, schur_pairs(), Tbuf.p, S.p, rhs.p);
  } else if (small && schur_kernel == 1) {
    const bool vec = dcmax % 2 == 0;               // 16-byte gathers need 16-byte records
    if (schur_ctas == 3) {
      if (vec) PXR_LAUNCH(ctx, (ba_schur_pairs_staged_kernel<true, 3>), pair_grid, kPairThreads, 0, d, schur_pairs(), Tbuf.p, S.p, rhs.p);
      else PXR_LAUNCH(ctx, (ba_schur_pairs_staged_kernel<false, 3>), pair_grid, kPairThreads, 0, d, schur_pairs(), Tbuf.p, S.p, rhs.p);
    } else {
      if (vec) PXR_LAUNCH(ctx, (ba_schur_pairs_staged_kernel<true, 4>), pair_grid, kPairThreads, 0, d, schur_pairs(), Tbuf.p, S.p, rhs.p);
      else PXR_LAUNCH(ctx, (ba_schur_pairs_staged_kernel<false, 4>), pair_grid, kPairThreads, 0, d, schur_pairs(), Tbuf.p, S.p, rhs.p);
    }
  } else if (img_dc_max <= 8) PXR_LAUNCH(ctx, ba_schur_pairs_kernel<true>, pair_grid, kPairThreads, 0, d, schur_pairs(), Tbuf.p, S.p, rhs.p);
  else PXR_LAUNCH(ctx, ba_schur_pairs_kernel<false>, pair_grid, kPairThreads, 0, d, schur_pairs(), Tbuf.p, S.p, rhs.p);
  return PXR_OK;
}

// the same walk with the image-pair blocks as the sink (block-sparse ITERATIVE_SCHUR, block mode); these paths only
// exist for images of at most 8 columns
int BA::launch_sp_schur_pairs(const BADev& d, double* Bk, double* rhs_out, double* part) {
  if (sp_n_chunks <= 0) return PXR_OK;
  const unsigned pair_grid = (unsigned)cdiv(sp_n_chunks * 32, kPairThreads);
  if (dcmax >= 9 && schur_kernel == 0) {
    PXR_LAUNCH(ctx, sp_schur_pairs_kernel<4>, pair_grid, kPairThreads, 0, d, schur_pairs(), ss_chunk_key.p, Hinv.p, Bk, rhs_out, part);
    return PXR_OK;
  }
  PXR_LAUNCH(ctx, ba_schur_prep_kernel, (unsigned)cdiv(n_obs * dcmax, 256), 256, 0, d, Hinv.p, Tbuf.p);
  if (dcmax >= 9 && schur_kernel == 3) PXR_LAUNCH(ctx, sp_schur_pairs_kernel<3>, pair_grid, kPairThreads, 0, d, schur_pairs(), ss_chunk_key.p, Tbuf.p, Bk, rhs_out, part);
  else if (dcmax >= 9 && schur_kernel == 1) {
    if (dcmax % 2 == 0) PXR_LAUNCH(ctx, sp_schur_pairs_kernel<1>, pair_grid, kPairThreads, 0, d, schur_pairs(), ss_chunk_key.p, Tbuf.p, Bk, rhs_out, part);
    else PXR_LAUNCH(ctx, sp_schur_pairs_kernel<2>, pair_grid, kPairThreads, 0, d, schur_pairs(), ss_chunk_key.p, Tbuf.p, Bk, rhs_out, part);
  } else PXR_LAUNCH(ctx, sp_schur_pairs_kernel<0>, pair_grid, kPairThreads, 0, d, schur_pairs(), ss_chunk_key.p, Tbuf.p, Bk, rhs_out, part);
  return PXR_OK;
}

// Stage 5: S delta_c = rhs with the reduced system where the assembly leaves it (S / rhs, or the image blocks of the
// block-sparse path), by the handle's solver: PCG or the dense Cholesky -> delta[0..nc).  A failure sets flags[1].
int BA::solve_reduced() {
  StageScope st(this, 5);
  last_linear_iterations = 1;
  if (nc == 0) return PXR_OK;
  if (sparse_schur) return pcg_solve_sparse();
  if (use_pcg) return pcg_solve();
  return chol_launch();
}

// One LM step attempt at the current linearisation: fills delta, returns validity and model cost change
int BA::compute_step(double radius, bool* valid, double* model_cost_change) {
  cudaStream_t s = ctx->stream;
  PXR_TRY(build_schur_pairs());
  if (block_mode) return compute_step_block_sync(radius, valid, model_cost_change);
  BADev d = dev();
  std::unique_ptr<StageScope> st(new StageScope(this, 4));   // RAII: an early error return still closes the stage
  if (nl > 0) PXR_LAUNCH(ctx, ba_d2_kernel, (unsigned)cdiv(nl, 256), 256, 0, diag.p, jscale.p, D2.p, nl, radius,
                         opt.min_lm_diagonal, opt.max_lm_diagonal);
  PXR_CUDA(cudaMemsetAsync(flags.p, 0, 4 * sizeof(int), s));
  if (sparse_schur) {
    // image-block form (pxr_sparse_schur.cuh): rhs = -gc + sum T gp, B_ab = sum T_x W_y^T; nothing of size nc^2
    if (nc > 0) PXR_LAUNCH(ctx, sp_init_rhs_kernel, (unsigned)cdiv(nc, 256), 256, 0, ctx->world > 1 ? gc_local.p : gc.p, rhs.p, nc);
    PXR_TRY(ss_Bk.zero(s));
    if (n_points > 0) {
      PXR_LAUNCH(ctx, ba_point_inverse_kernel, (unsigned)cdiv(n_points, 256), 256, 0, d, D2.p, Hinv.p, flags.p);
      PXR_TRY(launch_sp_schur_pairs(d, ss_Bk.p, rhs.p, nullptr));   // T = W Hinv first, unless the walk forms it itself
    }
    if (ctx->world > 1 && nc > 0) PXR_TRY(allreduce_f64(ctx, rhs.p, nc));
  } else {
  // multi-GPU: every rank starts from ITS partial Hcc / gc (rank 0 adds the damping), subtracts its points' Schur
  // contributions, and ONE all-reduce of [S | rhs] (rhs is row nc of the same array) yields the reduced system
  if (nc > 0) PXR_LAUNCH(ctx, ba_init_reduced_kernel, (unsigned)cdiv((int64_t)nc * nc, 256), 256, 0, Hcc.p,
                         ctx->world > 1 ? gc_local.p : gc.p, D2.p, S.p, rhs.p, nc, (ctx->world <= 1 || ctx->rank == 0) ? 1 : 0);
  if (n_points > 0) {
    PXR_LAUNCH(ctx, ba_point_inverse_kernel, (unsigned)cdiv(n_points, 256), 256, 0, d, D2.p, Hinv.p, flags.p);
    PXR_TRY(launch_schur_pairs(d));
  }
  // rhs rides along as row nc of S: the factorisation performs the forward substitution
  if (nc > 0) PXR_CUDA(cudaMemcpyAsync(S.p + (size_t)nc * nc, rhs.p, (size_t)nc * 8, cudaMemcpyDeviceToDevice, s));
  if (ctx->world > 1 && nc > 0) {
    PXR_TRY(allreduce_f64(ctx, S.p, (size_t)(nc + 1) * nc));
    PXR_CUDA(cudaMemcpyAsync(rhs.p, S.p + (size_t)nc * nc, (size_t)nc * 8, cudaMemcpyDeviceToDevice, s));   // PCG / debug read rhs
  }
  }
  st.reset();
  PXR_TRY(solve_reduced());
  st.reset(new StageScope(this, 7));
  PXR_CUDA(cudaMemsetAsync(scalars.p + 4, 0, 4 * 8, s));  // acc[0..3]
  if (n_points > 0) PXR_LAUNCH(ctx, ba_backsub_kernel, (unsigned)cdiv(n_points * 32, 256), 256, 0, d, D2.p, delta.p);
  if (n_obs > 0) {
    if (img_src8.p) PXR_LAUNCH(ctx, ba_model_cost_kernel<true>, (unsigned)cdiv(n_obs, 256), 256, 0, d, delta.p, scalars.p + 4);
    else PXR_LAUNCH(ctx, ba_model_cost_kernel<false>, (unsigned)cdiv(n_obs, 256), 256, 0, d, delta.p, scalars.p + 4);
  }
  PXR_CUDA(cudaGetLastError());
  st.reset();
  double acc = 0, fld = 0;
  if (chol_graph_exec && !chol_multikernel && !use_pcg && env.chol_test_abort) {
    // test hook: pretend the persistent kernel bailed out of a wait (abort word + failure flag)
    const int one = 1;
    PXR_CUDA(cudaMemcpyAsync(chol_sync.p + (pxr_chol::sync_ints((int)cdiv(nc, kNB)) - 1), &one, sizeof(int), cudaMemcpyHostToDevice, s));
    PXR_CUDA(cudaMemcpyAsync(flags.p + 1, &one, sizeof(int), cudaMemcpyHostToDevice, s));
    PXR_CUDA(cudaStreamSynchronize(s));
  }
  PXR_LAUNCH(ctx, flags_to_double_kernel, 1, 1, 0, flags.p, scalars.p + 5);
  PXR_TRY(allreduce_f64(ctx, scalars.p + 4, 2));   // model cost change + failure flag: every rank takes the same branch
  double two[2] = {0, 0};
  PXR_CUDA(cudaMemcpyAsync(two, scalars.p + 4, 16, cudaMemcpyDeviceToHost, s));
  PXR_CUDA(cudaStreamSynchronize(s));
  acc = two[0]; fld = two[1];
  if (fld != 0.0 && chol_graph_exec && !chol_multikernel && !use_pcg && ctx->world <= 1) {
    // Did the persistent Cholesky bail out of a wait?  That only happens when its CTAs were not all resident at
    // once (GPU shared with another client, MPS/MIG partition smaller than queried): switch, for the rest of this
    // handle's life, to the launch-per-panel path, which needs no co-residency, and redo this step.
    int aborted = 0;
    const int nbt = (int)cdiv(nc, kNB);
    PXR_CUDA(cudaMemcpyAsync(&aborted, chol_sync.p + (pxr_chol::sync_ints(nbt) - 1), sizeof(int), cudaMemcpyDeviceToHost, s));
    PXR_CUDA(cudaStreamSynchronize(s));
    if (aborted) {
      cudaGraphExecDestroy(chol_graph_exec); chol_graph_exec = nullptr;
      chol_force_multikernel = true;
      return compute_step(radius, valid, model_cost_change);
    }
  }
  const bool solved = fld == 0.0 && std::isfinite(acc);
  *model_cost_change = -acc;
  *valid = solved && (*model_cost_change > 0.0);
  return PXR_OK;
}

// candidate (other set) = Plus(current, delta); ||step||^2 and ||x||^2 (ambient; point parts, camera parts) to scalars[5..8]
int BA::apply_step() {
  PlusArgs a;
  a.n_cameras = n_cameras; a.n_images = n_images; a.n_points = n_points;
  a.cam_model = cam_model.p; a.cam_mask = cam_mask.p; a.tmask = tmask.p;
  a.pose_off = pose_off.p; a.intr_off = intr_off.p; a.point_off = point_off.p;
  a.cam = cam[cur].p; a.q = q[cur].p; a.t = t[cur].p; a.X = X[cur].p;
  a.cam_o = cam[1 - cur].p; a.q_o = q[1 - cur].p; a.t_o = t[1 - cur].p; a.X_o = X[1 - cur].p;
  a.delta = delta.p; a.acc = scalars.p + 4;
  StageScope st(this, 8);
  PXR_CUDA(cudaMemsetAsync(scalars.p + 5, 0, 4 * 8, ctx->stream));
  const int64_t n = std::max<int64_t>(std::max<int64_t>(n_points, n_images), n_cameras);
  if (deterministic) a.part = det_scal_part.p;
  PXR_LAUNCH(ctx, ba_plus_kernel, (unsigned)cdiv(n, 128), 128, 0, a);
  if (deterministic)
    for (int k = 0; k < 4; ++k) PXR_LAUNCH(ctx, det_reduce_add_kernel, 1, 1024, 0, det_scal_part.p, cdiv(n, 128), 4, k, a.acc + 1 + k);
  PXR_CUDA(cudaGetLastError());
  if (!block_mode) PXR_TRY(allreduce_f64(ctx, scalars.p + 5, 2));  // point parts are sharded, camera parts replicated (block mode: scalar exchange)
  return PXR_OK;
}

// ba_project_point_kernel over list[0..n) (or [0..*n_dev), grid sized for n): uv (xy on a geometric handle) and d(uv)/dX
// to inner_jpt.
int BA::alloc_inner_jpt() {
  if (!inner_jpt.p) PXR_TRY(inner_jpt.alloc((size_t)n_obs * 6));
  return PXR_OK;
}

int BA::project_point_list(int set, const int64_t* list, int64_t n, const unsigned long long* n_dev, int64_t grid_bound) {
  if (!inner_jpt.p) return fail(PXR_ERR_INTERNAL, "the point-only projection ran before its buffer was allocated");
  if (grid_bound <= 0) return PXR_OK;
  ProjectArgs pa;
  pa.obs_img = obs_img.p; pa.obs_pt = obs_pt.p; pa.obs_patch = obs_patch.p;
  pa.img_cam = img_cam.p; pa.cam_model = cam_model.p;
  pa.cam_params = cam[set].p; pa.qvec = q[set].p; pa.tvec = t[set].p; pa.xyz = X[set].p;
  pa.corner = corner.p; pa.scale = scale.p; pa.ups = ups;
  pa.obs_begin = 0; pa.obs_end = n; pa.item_index = list; pa.n_dev = n_dev;
  pa.uv = uv.p; pa.xy = geometric ? geo_xy.p : nullptr; pa.juv = nullptr; pa.juv_stride = juv_stride; pa.juv_k = K;
  pa.jpt = inner_jpt.p;
  PXR_LAUNCH(ctx, ba_project_point_kernel, (unsigned)std::min<int64_t>(cdiv(grid_bound, 128), (int64_t)ctx->sm_count * 16), 128,
             (size_t)128 * (juv_stride | 1) * sizeof(double), pa);
  return PXR_OK;
}

// K0 (uv and the point Jacobian only, to inner_jpt) + K1 (Jacobian mode) over an explicit list of observations, what
// an inner-iteration round evaluates: its step kernel reads d(uv)/dX and nothing else of the Jacobian, and the driver
// projects afresh after the rounds, so juv is left alone.  With n_dev the number of entries is read on the device (n is
// then the upper bound K1's grid is sized for, k0_bound, when >= 0, a tighter one for K0's); settle = false leaves the
// window-residency check to the caller (inner_rounds checks once per batch of rounds).  after_k0 / after_k1, when
// given, are recorded right after the K0 and K1 launches (round timing).
int BA::eval_list(int set, const int64_t* list, int64_t n, const unsigned long long* n_dev, bool settle,
                  cudaEvent_t after_k0, cudaEvent_t after_k1, int64_t k0_bound) {
  if (n <= 0) return PXR_OK;
  PXR_TRY(project_point_list(set, list, n, n_dev, k0_bound >= 0 ? std::min(k0_bound, n) : n));
  if (after_k0) PXR_CUDA(cudaEventRecord(after_k0, ctx->stream));
  if (geometric) {   // no patches, so nothing for window residency to settle
    PXR_TRY(geo_k1(1, nullptr, nullptr, list, n, n_dev));
    if (after_k1) PXR_CUDA(cudaEventRecord(after_k1, ctx->stream));
    return PXR_OK;
  }
  FmEvalArgs a;
  a.uv = uv.p; a.item_patch = obs_patch.p; a.item_ref = obs_pt.p;
  a.patches = d_patches; a.ph = ph; a.pw = pw;
  a.refs = has_refs ? refs.p : nullptr;
  a.begin = 0; a.end = n; a.item_index = list; a.end_dev = n_dev;
  a.out = obs_out.p; a.residuals = nullptr; a.desc = nullptr;
  a.loss.type = opt.loss_type; a.loss.a = opt.loss_scale;
  a.l2_normalize = interp.l2_normalize;
  resident_args(a);
  int np = 0;
  PXR_TRY(launch_fm_eval(ctx, dtype, C, 1, interp.use_float_simd != 0, a, &np));
  if (after_k1) PXR_CUDA(cudaEventRecord(after_k1, ctx->stream));
  if (!settle) return PXR_OK;
  for (;;) {     // window residency: whoever consumes these results right away needs them settled first
    int64_t n_fixed = 0;
    PXR_TRY(resident_fix(&n_fixed));
    if (n_fixed == 0) break;
    a.item_index = res_fix_list.p; a.begin = 0; a.end = n_fixed; a.end_dev = nullptr;
    PXR_TRY(launch_fm_eval(ctx, dtype, C, 1, interp.use_float_simd != 0, a, &np));
  }
  return PXR_OK;
}

// Inner iterations: see pxr_inner.cuh; the per-point rules are pxr_lm.cuh's.
// Round 0's lists come from every variable point (round 0 itself evaluates every observation); from then on a round is
// three launches (K0, K1, inner_step_kernel) and the step kernel builds the next round's lists.  Lists alternate between two buffers, counters rotate through three sets
// (the step kernel of round r appends to set r+1 and zeroes set r+2, which no launch of round r touches).  The rounds are
// enqueued WITHOUT waiting for the host: each step kernel copies its round's list lengths to a host-mapped slot, tagged
// with the call's epoch, and the host stops enqueuing once a round two behind has reported an empty list (the two extra
// rounds find nothing to do).
constexpr int kInnerRounds = 53;
int BA::inner_rounds(int set, double* trial_cost) {
  cudaStream_t s = ctx->stream;
  volatile unsigned long long* slots = inner_cnt_host;
  const unsigned long long epoch = ++inner_epoch;
  auto published = [&](int r) { return slots[3 * r + 2] == epoch; };
  InnerStepArgs a;
  a.n_points = n_points; a.point_off = point_off.p; a.pt_begin = pt_begin.p;
  a.obs_out = obs_out.p; a.jpt = inner_jpt.p;
  a.xyz = X[set].p; a.st = inner_state.p;
  a.loss.type = opt.loss_type; a.loss.a = opt.loss_scale;
  a.epoch = epoch;
  const unsigned pgrid = (unsigned)cdiv(n_points, 128);
  // Round r's lists are a subset of round r-2's, so the lengths that round published bound K0's and the step kernel's
  // grids (both read the exact length on the device); before any round has published, n_obs / n_points do.
  int64_t bound_obs = n_obs, bound_pts = n_points;
  if (time_inner_rounds && inner_round_timed.empty()) {
    inner_round_timed.resize(kInnerRounds, {nullptr, nullptr, nullptr, nullptr});
    for (auto& ev : inner_round_timed)
      for (cudaEvent_t& e : ev) PXR_CUDA(cudaEventCreate(&e));
  }
  inner_rounds_timed = time_inner_rounds;
  inner_rounds_run = 0;
  cap_plist.clear(); cap_list.clear(); cap_active.clear();
  PXR_CUDA(cudaMemsetAsync(inner_counters.p, 0, 6 * sizeof(unsigned long long), s));
  a.plist_next = inner_plist[0].p; a.list_next = inner_list[0].p; a.cnt_next = inner_counters.p;
  PXR_LAUNCH(ctx, inner_list_kernel, pgrid, 128, 0, a);
  for (int round = 0; round < kInnerRounds; ++round) {
    if (round >= 2) {
      const int r2 = round - 2;
      if (!published(r2) && round >= 8 && (round & 3) == 0) {   // far ahead of the device: let it catch up rather than pile up empty rounds
        while (!published(r2)) {
          const cudaError_t q = cudaStreamQuery(s);
          if (q == cudaSuccess) {
            if (published(r2)) break;
            return fail(PXR_ERR_CUDA, "inner iterations: round %d did not report its list", r2);
          }
          if (q != cudaErrorNotReady) PXR_CUDA(q);
          (void)cudaGetLastError();
          std::this_thread::yield();
        }
      }
      if (published(r2)) {
        if (slots[3 * r2] == 0) break;
        bound_obs = std::min<int64_t>(bound_obs, (int64_t)slots[3 * r2]);
        bound_pts = std::min<int64_t>(bound_pts, (int64_t)slots[3 * r2 + 1]);
      }
    }
    const int cur = round & 1;
    unsigned long long* cnt = inner_counters.p + 2 * (round % 3);
    if (capture_inner_lists) PXR_TRY(capture_round_lists(inner_plist[cur].p, inner_list[cur].p, cnt));
    a.plist = inner_plist[cur].p; a.cnt = cnt;
    a.plist_next = inner_plist[1 - cur].p; a.list_next = inner_list[1 - cur].p;
    a.cnt_next = inner_counters.p + 2 * ((round + 1) % 3); a.cnt_clear = inner_counters.p + 2 * ((round + 2) % 3);
    a.publish = inner_cnt_dev + 3 * round;
    cudaEvent_t* ev = inner_rounds_timed ? inner_round_timed[round].data() : nullptr;
    if (ev) PXR_CUDA(cudaEventRecord(ev[0], s));
    if (round == 0) {
      // every observation, those of constant points included, so that the records also give the cost at the starting
      // point: reduced here, before the step kernel, with the kernels and partial order of fm_cost's full pass.  Under
      // window residency a batch with violations is run again from round 0, which overwrites the cost.
      PXR_TRY(eval_list(set, nullptr, n_obs, nullptr, false, ev ? ev[1] : nullptr, ev ? ev[2] : nullptr));
      if (trial_cost) PXR_TRY(fm_cost(trial_cost));
    } else {
      PXR_TRY(eval_list(set, inner_list[cur].p, n_obs, cnt, false, ev ? ev[1] : nullptr, ev ? ev[2] : nullptr, bound_obs));
    }
    const unsigned sgrid = (unsigned)std::min<int64_t>(cdiv(bound_pts, 128), (int64_t)ctx->sm_count * 8);
    PXR_LAUNCH(ctx, inner_step_kernel, sgrid, 128, 0, a, round == 0 ? 0 : 1);
    if (ev) PXR_CUDA(cudaEventRecord(ev[3], s));
    if (capture_inner_lists) PXR_TRY(capture_round_active());
    inner_rounds_run = round + 1;
  }
  PXR_CUDA(cudaGetLastError());
  return PXR_OK;
}

// pxr_ba_debug_inner_capture: a round's point and observation lists as the round starts (synchronous, tests only)
int BA::capture_round_lists(const int64_t* plist, const int64_t* list, const unsigned long long* cnt) {
  cudaStream_t s = ctx->stream;
  unsigned long long c[2] = {0, 0};
  PXR_CUDA(cudaMemcpyAsync(c, cnt, sizeof(c), cudaMemcpyDeviceToHost, s));
  PXR_CUDA(cudaStreamSynchronize(s));
  cap_list.emplace_back((size_t)c[0]); cap_plist.emplace_back((size_t)c[1]);
  if (c[0]) PXR_CUDA(cudaMemcpyAsync(cap_list.back().data(), list, (size_t)c[0] * 8, cudaMemcpyDeviceToHost, s));
  if (c[1]) PXR_CUDA(cudaMemcpyAsync(cap_plist.back().data(), plist, (size_t)c[1] * 8, cudaMemcpyDeviceToHost, s));
  PXR_CUDA(cudaStreamSynchronize(s));
  return PXR_OK;
}

// ... and, after the round's step kernel, whether each of its points stays active
int BA::capture_round_active() {
  cudaStream_t s = ctx->stream;
  std::vector<int32_t> act((size_t)n_points);
  PXR_CUDA(cudaMemcpy2DAsync(act.data(), sizeof(int32_t), reinterpret_cast<const char*>(inner_state.p) + offsetof(InnerState, active),
                             sizeof(InnerState), sizeof(int32_t), (size_t)n_points, cudaMemcpyDeviceToHost, s));
  PXR_CUDA(cudaStreamSynchronize(s));
  const std::vector<int64_t>& pl = cap_plist.back();
  cap_active.emplace_back(pl.size());
  for (size_t i = 0; i < pl.size(); ++i) cap_active.back()[i] = act[(size_t)pl[i]] != 0 ? 1 : 0;
  return PXR_OK;
}

int BA::inner_iterations(int set, double* trial_cost) {
  if (n_points == 0 || n_obs == 0) return trial_cost ? fm_cost(trial_cost) : PXR_OK;
  StageScope stg(this, 9);
  cudaStream_t s = ctx->stream;
  if (!inner_state.p) {
    PXR_TRY(inner_state.alloc(n_points));
    for (int k = 0; k < 2; ++k) { PXR_TRY(inner_list[k].alloc(n_obs)); PXR_TRY(inner_plist[k].alloc(n_points)); }
    PXR_TRY(alloc_inner_jpt());
    PXR_TRY(inner_counters.alloc(6));
    PXR_CUDA(cudaHostAlloc((void**)&inner_cnt_host, (size_t)kInnerRounds * 3 * sizeof(unsigned long long), cudaHostAllocMapped));
    std::memset(inner_cnt_host, 0, (size_t)kInnerRounds * 3 * sizeof(unsigned long long));
    PXR_CUDA(cudaHostGetDevicePointer((void**)&inner_cnt_dev, inner_cnt_host, 0));
  }
  if (!resident) return inner_rounds(set, trial_cost);
  // window residency: an observation may leave its window in any round and nobody looks before the rounds are over — keep
  // the starting points, and if something was reported fetch those patches and run the rounds again from the start
  if (!inner_snapshot.p) PXR_TRY(inner_snapshot.alloc((size_t)n_points * 3));
  PXR_CUDA(cudaMemcpyAsync(inner_snapshot.p, X[set].p, (size_t)n_points * 24, cudaMemcpyDeviceToDevice, s));
  for (;;) {
    PXR_TRY(inner_rounds(set, trial_cost));
    int64_t n_fixed = 0;
    PXR_TRY(resident_fix(&n_fixed));
    if (n_fixed == 0) break;
    PXR_CUDA(cudaMemcpyAsync(X[set].p, inner_snapshot.p, (size_t)n_points * 24, cudaMemcpyDeviceToDevice, s));
  }
  return PXR_OK;
}

// ||set 0 - set 1||^2 (ambient), the step after inner iterations: points to scalars[11], cameras to scalars[12].  Only
// enqueued; the drivers read it with the iteration's other scalars.
int BA::step_norm_between_sets() {
  cudaStream_t s = ctx->stream;
  PXR_CUDA(cudaMemsetAsync(scalars.p + 11, 0, 16, s));
  auto run = [&](const double* a, const double* b, int64_t n, double* acc) -> int {
    if (n <= 0) return PXR_OK;
    PXR_LAUNCH(ctx, diff_norm_kernel, (unsigned)cdiv(n, 256), 256, 0, a, b, n, acc, deterministic ? det_scal_part.p : nullptr);
    if (deterministic) PXR_LAUNCH(ctx, det_reduce_add_kernel, 1, 1024, 0, det_scal_part.p, cdiv(n, 256), 1, 0, acc);
    return PXR_OK;
  };
  PXR_TRY(run(cam[0].p, cam[1].p, (int64_t)n_cameras * kMaxK, scalars.p + 12));
  PXR_TRY(run(q[0].p, q[1].p, (int64_t)n_images * 4, scalars.p + 12));
  PXR_TRY(run(t[0].p, t[1].p, (int64_t)n_images * 3, scalars.p + 12));
  PXR_TRY(run(X[0].p, X[1].p, n_points * 3, scalars.p + 11));
  return PXR_OK;
}

// S delta_c = rhs by Schur-Jacobi preconditioned CG (pxr_pcg.cuh); result in delta[0..nc)
int BA::pcg_setup_blocks() {
  if (cg_state.p) return PXR_OK;
  cudaStream_t s = ctx->stream;
  // SCHUR_JACOBI blocks = the camera-side parameter blocks (one per variable pose, one per variable intrinsics)
  std::vector<int32_t> off;
  for (int i = 0; i < n_images; ++i) if (h_pose_off[i] >= 0) off.push_back(h_pose_off[i]);
  for (int c = 0; c < n_cameras; ++c) if (h_intr_off[c] >= 0) off.push_back(h_intr_off[c]);
  std::sort(off.begin(), off.end());
  std::vector<int32_t> sd(off.size());
  for (size_t k = 0; k < off.size(); ++k) sd[k] = (k + 1 < off.size() ? off[k + 1] : nc) - off[k];
  cg_nblk = (int)off.size();
  // every row's block (offset, dimension) depends on the layout only: the preconditioner kernels read it from here
  std::vector<int32_t> row_off(nc), row_dim(nc);
  for (size_t k = 0; k < off.size(); ++k)
    for (int i = 0; i < sd[k]; ++i) { row_off[off[k] + i] = off[k]; row_dim[off[k] + i] = sd[k]; }
  PXR_TRY(cg_blk_off.upload(off.data(), off.size(), s)); PXR_TRY(cg_blk_dim.upload(sd.data(), sd.size(), s));
  PXR_TRY(cg_row_off.upload(row_off.data(), row_off.size(), s)); PXR_TRY(cg_row_dim.upload(row_dim.data(), row_dim.size(), s));
  PXR_TRY(cg_Minv.alloc((size_t)nc * 12));
  PXR_TRY(cg_z.alloc(nc)); PXR_TRY(cg_p.alloc(nc)); PXR_TRY(cg_q.alloc(nc)); PXR_TRY(cg_r.alloc(nc)); PXR_TRY(cg_x.alloc(nc)); PXR_TRY(cg_tmp.alloc(nc));
  PXR_TRY(cg_state.alloc(1));
  if (sparse_schur) {
    auto blk_of = [&](int offset) -> int32_t { return (int32_t)(std::lower_bound(off.begin(), off.end(), offset) - off.begin()); };
    h_img_pose_blk.assign(n_images, -1); h_img_cam_blk.assign(n_images, -1);
    for (int i = 0; i < n_images; ++i) {
      if (h_pose_off[i] >= 0) h_img_pose_blk[i] = blk_of(h_pose_off[i]);
      const int io = h_intr_off[h_img_cam[i]];
      if (io >= 0) h_img_cam_blk[i] = blk_of(io);
    }
    PXR_TRY(ss_img_pose_blk.upload(h_img_pose_blk.data(), h_img_pose_blk.size(), s));
    PXR_TRY(ss_img_cam_blk.upload(h_img_cam_blk.data(), h_img_cam_blk.size(), s));
    PXR_TRY(ss_Dblk.alloc((size_t)std::max(cg_nblk, 1) * 144));
  }
  PXR_CUDA(cudaStreamSynchronize(s));
  return PXR_OK;
}

// ITERATIVE_SCHUR on the implicit block-sparse reduced system (pxr_sparse_schur.cuh).  Same CG recurrences and
// termination as pcg_solve(); the mat-vec gathers/scatters through the image blocks, and in the multi-GPU path the
// product (nc doubles) is all-reduced per iteration instead of the matrix once.
int BA::pcg_solve_sparse() {
  cudaStream_t s = ctx->stream;
  PXR_TRY(pcg_setup_blocks());
  const int n = nc;
  const SparseSchur sp = sparse();
  const int64_t nthreads = std::max<int64_t>(((int64_t)n_images + ss_n_keys) * 8, n);
  const unsigned gs = (unsigned)cdiv(nthreads, 256);
  const int add_d2 = (ctx->world <= 1 || ctx->rank == 0) ? 1 : 0;
  auto spmv = [&](const double* x, double* y) -> int {
    PXR_CUDA(cudaMemsetAsync(y, 0, (size_t)n * 8, s));
    PXR_LAUNCH(ctx, sp_spmv_kernel, gs, 256, 0, sp, D2.p, x, y, add_d2, cg_state.p);
    if (ctx->world > 1) PXR_TRY(allreduce_f64(ctx, y, n));
    return PXR_OK;
  };
  PXR_TRY(ss_Dblk.zero(s));
  PXR_LAUNCH(ctx, sp_blockdiag_kernel, (unsigned)cdiv(((int64_t)n_images + ss_n_keys) * 8, 256), 256, 0, sp, ss_Dblk.p);
  if (ctx->world > 1) PXR_TRY(allreduce_f64(ctx, ss_Dblk.p, (size_t)cg_nblk * 144));
  PXR_LAUNCH(ctx, sp_block_inverse_kernel, (unsigned)cdiv(cg_nblk, 64), 64, 0, ss_Dblk.p, D2.p, 1, cg_blk_off.p, cg_blk_dim.p, cg_nblk,
             cg_Minv.p, flags.p + 1);
  return run_cg(spmv);
}

int BA::pcg_solve() {
  cudaStream_t s = ctx->stream;
  PXR_TRY(pcg_setup_blocks());
  const int n = nc;
  const unsigned gv = (unsigned)cdiv((int64_t)n * 32, 256);
  PXR_LAUNCH(ctx, cg_mirror_kernel, (unsigned)cdiv((int64_t)n * n, 256), 256, 0, S.p, n);
  PXR_LAUNCH(ctx, cg_block_inverse_kernel, (unsigned)cdiv(cg_nblk, 64), 64, 0, S.p, n, cg_blk_off.p, cg_blk_dim.p, cg_nblk, cg_Minv.p,
             flags.p + 1);
  auto spmv = [&](const double* x, double* y) -> int {
    PXR_LAUNCH(ctx, cg_gemv_kernel, gv, 256, 0, S.p, x, y, n, cg_state.p);
    return PXR_OK;
  };
  return run_cg(spmv);
}

// Preconditioned CG on the reduced system given its product; Ceres' ConjugateGradientsSolver recurrences and
// termination (Q-decrease ratio, residual refresh every 10 iterations).  Small systems run the single-CTA vector
// kernels (deterministic sums); from 4096 unknowns the multi-CTA variants.  The block inverse that ran before reports a
// failure in flags[1]; the init kernels then finish the solve with 0 iterations.
int BA::run_cg(const std::function<int(const double*, double*)>& spmv) {
  cudaStream_t s = ctx->stream;
  const int n = nc;
  const bool multi = n >= 4096 || env.cg_multi;
  const unsigned gn = (unsigned)cdiv(n, 256);
  CGState hs;
  if (multi) {
    if (cg_part.n < (size_t)3 * gn) PXR_TRY(cg_part.alloc((size_t)3 * gn));
    PXR_LAUNCH(ctx, cgm_init_state_kernel, 1, 1, 0, cg_state.p, opt.max_linear_solver_iterations, 0.1, flags.p + 1);
    PXR_LAUNCH(ctx, cgm_init_kernel, gn, 256, 0, rhs.p, cg_x.p, cg_r.p, n, cg_state.p, cg_part.p);
    PXR_LAUNCH(ctx, cgm_init_done_kernel, 1, 32, 0, cg_state.p, cg_part.p, (int)gn);
  } else {
    PXR_LAUNCH(ctx, cg_init_kernel, 1, 1024, 0, rhs.p, cg_x.p, cg_r.p, n, cg_state.p, opt.max_linear_solver_iterations, 0.1, flags.p + 1);
  }
  for (int it = 0; it < opt.max_linear_solver_iterations; ++it) {
    const bool refresh = (it + 1) % 10 == 0;   // residual_reset_period
    if (multi) {
      PXR_LAUNCH(ctx, cgm_precond_kernel, gn, 256, 0, cg_Minv.p, cg_row_off.p, cg_row_dim.p, cg_r.p, cg_z.p, n, cg_state.p, cg_part.p);
      PXR_LAUNCH(ctx, cgm_beta_kernel, 1, 32, 0, cg_state.p, cg_part.p, (int)gn);
      PXR_LAUNCH(ctx, cgm_dir_kernel, gn, 256, 0, cg_z.p, cg_p.p, n, cg_state.p);
      PXR_TRY(spmv(cg_p.p, cg_q.p));
      PXR_LAUNCH(ctx, cgm_pq_kernel, gn, 256, 0, cg_p.p, cg_q.p, n, cg_state.p, cg_part.p);
      PXR_LAUNCH(ctx, cgm_alpha_kernel, 1, 32, 0, cg_state.p, cg_part.p, (int)gn);
      PXR_LAUNCH(ctx, cgm_update_kernel, gn, 256, 0, rhs.p, cg_p.p, cg_q.p, cg_x.p, cg_r.p, n, cg_state.p, cg_part.p);
      if (refresh) {
        PXR_TRY(spmv(cg_x.p, cg_tmp.p));
        PXR_LAUNCH(ctx, cgm_refresh_kernel, gn, 256, 0, rhs.p, cg_tmp.p, cg_x.p, cg_r.p, n, cg_state.p, cg_part.p);
      }
      PXR_LAUNCH(ctx, cgm_check_kernel, 1, 32, 0, cg_state.p, cg_part.p, (int)gn);
    } else {
      PXR_LAUNCH(ctx, cg_precond_kernel, 1, 1024, 0, cg_Minv.p, cg_row_off.p, cg_row_dim.p, cg_r.p, cg_z.p, cg_p.p, n, cg_state.p);
      PXR_TRY(spmv(cg_p.p, cg_q.p));
      PXR_LAUNCH(ctx, cg_update_kernel, 1, 1024, 0, rhs.p, cg_p.p, cg_q.p, cg_x.p, cg_r.p, n, cg_state.p);
      if (refresh) {
        PXR_TRY(spmv(cg_x.p, cg_tmp.p));
        PXR_LAUNCH(ctx, cg_refresh_kernel, 1, 1024, 0, rhs.p, cg_tmp.p, cg_r.p, n, cg_state.p);
      }
      PXR_LAUNCH(ctx, cg_check_kernel, 1, 1024, 0, rhs.p, cg_x.p, cg_r.p, n, cg_state.p);
    }
    if ((it + 1) % 8 == 0 || it + 1 == opt.max_linear_solver_iterations) {
      PXR_CUDA(cudaMemcpyAsync(&hs, cg_state.p, sizeof(hs), cudaMemcpyDeviceToHost, s));
      PXR_CUDA(cudaStreamSynchronize(s));
      if (hs.done) break;
    }
  }
  PXR_CUDA(cudaMemcpyAsync(&hs, cg_state.p, sizeof(hs), cudaMemcpyDeviceToHost, s));
  PXR_CUDA(cudaMemcpyAsync(delta.p, cg_x.p, (size_t)n * 8, cudaMemcpyDeviceToDevice, s));
  PXR_CUDA(cudaStreamSynchronize(s));
  last_linear_iterations = hs.it;
  if (hs.failed) { int one = 1; PXR_CUDA(cudaMemcpyAsync(flags.p + 1, &one, sizeof(int), cudaMemcpyHostToDevice, s)); }
  return PXR_OK;
}

int BA::gradient_max_norm(double* out) {
  PXR_CUDA(cudaMemsetAsync(scalars.p + 10, 0, 8, ctx->stream));
  const int64_t n = std::max<int64_t>(std::max<int64_t>(n_images, n_cameras), n_points);
  const BADev d = dev();
  if (n > 0) PXR_LAUNCH(ctx, ba_gradmax_kernel, (unsigned)cdiv(n, 256), 256, 0, d, d.gc, q[cur].p, 1, scalars.p + 10);
  PXR_TRY(allreduce_f64(ctx, scalars.p + 10, 1, true));
  PXR_CUDA(cudaMemcpyAsync(out, scalars.p + 10, 8, cudaMemcpyDeviceToHost, ctx->stream));
  PXR_CUDA(cudaStreamSynchronize(ctx->stream));
  return PXR_OK;
}

// -------------------------------------------------------------------------------- LM driver
// Mirrors ceres::internal::TrustRegionMinimizer::Minimize (Ceres 2.1) with LevenbergMarquardtStrategy, monotonic or
// non-monotonic steps, Jacobi scaling, inner iterations; the rules themselves are TrustRegion's (pxr_lm.cuh).  The loop
// state lives in the BA object so that a solve can be continued (pxr_ba_iterate) — bench.py times K consecutive
// iterations of one trajectory after W warm-up iterations.  One loop serves both modes; lm_linearize_start, lm_trial
// and lm_move hold what block mode (pxr_ba_block.cu) does differently: it enqueues a whole iteration and learns its
// scalars from one exchange, where the single-GPU driver reads them back as it goes.
int BA::lm_begin() {
  PXR_CUDA(cudaSetDevice(ctx->device));
  lm = LMState();
  lm.inner_enabled = opt.use_inner_iterations != 0;
  // ---- IterationZero
  PXR_TRY(lm_linearize_start());
  std::memset(&lm.it, 0, sizeof(lm.it));
  lm.it.cost = lm.x_cost;
  PXR_TRY(lm_gradient(&lm.it.gradient_max_norm));
  lm.initial_cost = lm.minimum_cost = lm.x_cost;
  TrustRegionOptions o;
  o.max_consecutive_invalid_steps = opt.max_num_consecutive_invalid_steps;
  o.max_nonmonotonic = opt.use_nonmonotonic_steps ? opt.max_consecutive_nonmonotonic_steps : 0;
  o.initial_radius = opt.initial_trust_region_radius;
  o.max_radius = opt.max_trust_region_radius;
  o.min_radius = opt.min_trust_region_radius;
  o.gradient_tolerance = opt.gradient_tolerance;
  o.parameter_tolerance = opt.parameter_tolerance;
  o.function_tolerance = opt.function_tolerance;
  o.min_relative_decrease = opt.min_relative_decrease;
  lm.tr.init(o, lm.x_cost);
  lm.best_is_current = true;
  lm.started = true;
  lm.pending_finalize = true;
  lm.term = 1;
  lm.message = "Maximum number of iterations reached.";
  return PXR_OK;
}

int BA::lm_linearize_start() {
  if (!block_mode) {
    PXR_TRY(evaluate(cur, true, &lm.x_cost));
  } else {
    PXR_TRY(project(cur, true, nullptr));
    PXR_TRY(fm(1, nullptr, scalars.p + 0));
    PXR_TRY(build_block());
    PXR_TRY(global_cost_block(&lm.x_cost));
  }
  if (!std::isfinite(lm.x_cost)) return fail(PXR_ERR_NUMERIC, "initial cost is not finite");
  if (!block_mode) {
    if (nl > 0) PXR_LAUNCH(ctx, ba_scale_kernel, (unsigned)cdiv(nl, 256), 256, 0, diag.p, jscale.p, nl, opt.jacobi_scaling);
  } else {
    // block mode: point columns now, camera columns right after the first all-reduce (they need the global diagonal)
    if (nl - nc > 0) PXR_LAUNCH(ctx, ba_scale_kernel, (unsigned)cdiv(nl - nc, 256), 256, 0, diag.p + nc, jscale.p + nc, nl - nc, opt.jacobi_scaling);
    jscale_c_pending = true;
  }
  return PXR_OK;
}

int BA::lm_gradient(double* out) {
  if (blk_lag_gmax) {   // block mode, several ranks: it arrives with the next all-reduce (finish_gmax_block at the end)
    *out = std::numeric_limits<double>::quiet_NaN();
    lm.gmax_pending = true;
    return PXR_OK;
  }
  return gradient_max_norm(out);
}

// FinalizeIterationAndCheckIfMinimizerCanContinue
bool BA::lm_finalize(int max_iteration) {
  pxr_iteration_summary& it = lm.it;
  if (lm.pending_finalize) {
    if (it.step_is_successful) {
      // ceres copies x into the user's parameters only when it is the best iterate so far; with monotonic steps every
      // accepted iterate is, with use_nonmonotonic_steps the best one is snapshotted on the device
      ++lm.n_succ;
      if (lm.x_cost < lm.minimum_cost) lm.minimum_cost = lm.x_cost;
    } else if (it.iteration > 0) ++lm.n_unsucc;
    it.trust_region_radius = lm.tr.radius;
    it.iteration_time_s = std::chrono::duration<double>(std::chrono::steady_clock::now() - lm.it_start).count();
    lm.its.push_back(it);
    lm.pending_finalize = false;
  }
  switch (lm.tr.stop(it.iteration, max_iteration, it.gradient_max_norm)) {
    case TR_MAX_ITERATIONS: lm.term = 1; lm.message = "Maximum number of iterations reached."; return false;
    case TR_GRADIENT_TOLERANCE: lm.term = 0; lm.message = "Gradient tolerance reached."; lm.finished = true; return false;
    case TR_MIN_RADIUS: lm.term = 0; lm.message = "Minimum trust region radius reached."; lm.finished = true; return false;
  }
  return true;
}

// Enqueues the step and its trial evaluation, and reads back what the host decides on.
int BA::lm_trial(bool interrupted, bool ran_inner, LMTrial* t) {
  // Trial point.  Ceres evaluates the cost here and, if the step is accepted, residuals AND Jacobians again at the
  // point it moves to.  Both passes stream the same patch windows, so with speculation (DESIGN §4) the pass at that
  // point runs in Jacobian mode right away, into the alternate buffer set; a rejected step merely discards it.
  // Without inner iterations that pass is the trial pass.  With them the trial cost comes from inner-iteration round 0,
  // which evaluates every observation at the trial point, and the pass after the rounds is the one at the final point.
  // Ceres skips inner iterations when the trial cost is not finite; here they run regardless and their result is
  // ignored (such a step is rejected, and its parameter set with it).  PXR_NO_SPECULATION: cost-only passes, and the
  // accepted point is evaluated again.
  const bool speculate = !env.no_speculation;
  const bool round0_cost = ran_inner && speculate;
  if (!block_mode) {
    // single GPU: an interrupt stops the solve before anything is enqueued
    if (interrupted) { t->interrupted = true; return PXR_OK; }
    // host synchronisation 1 of 2: the step's validity and model cost change
    PXR_TRY(compute_step(lm.tr.radius, &t->valid, &t->model_cost_change));
    if (!t->valid) return PXR_OK;     // single GPU: no trial after an invalid step
    PXR_TRY(apply_step());
    swap_sets();
    int rc = round0_cost ? inner_iterations(1 - cur, scalars.p + 0) : project(1 - cur, speculate, nullptr);
    if (rc == PXR_OK && !round0_cost) rc = fm(speculate ? 1 : 0, nullptr, scalars.p + 0);
    if (ran_inner) {
      if (rc == PXR_OK && !round0_cost) rc = inner_iterations(1 - cur);
      if (rc == PXR_OK) rc = project(1 - cur, speculate, nullptr);
      if (rc == PXR_OK) rc = fm(speculate ? 1 : 0, nullptr, scalars.p + 1);
      if (rc == PXR_OK) rc = step_norm_between_sets();
      if (rc == PXR_OK) rc = allreduce_f64(ctx, scalars.p + 11, 1);
    }
    if (rc == PXR_OK) rc = allreduce_f64(ctx, scalars.p + 0, ran_inner ? 2 : 1);
    double v[13] = {};     // [0] trial cost, [1] cost after the inner iterations, [5..8] apply_step's norms, [11..12] the step after them
    if (rc == PXR_OK) {
      // host synchronisation 2 of 2: the costs and the norms of the step in one round trip
      cudaError_t e = cudaMemcpyAsync(v, scalars.p, sizeof(v), cudaMemcpyDeviceToHost, ctx->stream);
      if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
      if (e != cudaSuccess) rc = fail(PXR_ERR_CUDA, "trial evaluation failed: %s", cudaGetErrorString(e));
    }
    swap_sets();   // back: uv/obs_out/juv = linearisation at the current point again
    PXR_TRY(rc);
    t->cost = v[0]; t->inner_cost = v[1];
    t->step_sq[0] = v[5]; t->step_sq[1] = v[7]; t->x_sq[0] = v[6]; t->x_sq[1] = v[8];
    t->inner_step_sq[0] = v[11]; t->inner_step_sq[1] = v[12];
    return PXR_OK;
  }
  // block mode: the whole iteration is enqueued before the host knows whether the step is valid, and the interrupt is
  // agreed on through the scalar exchange (a rank must not leave alone)
  cudaStream_t s = ctx->stream;
  PXR_TRY(compute_step_block(lm.tr.radius));
  pack_scalars(0, interrupted ? 1 : 0);
  PXR_TRY(apply_step());
  swap_sets();
  // ceres skips inner iterations when the trial cost is not finite — a GLOBAL fact that is only known after the
  // exchange; they are per-point and local, so they run regardless
  int rc = round0_cost ? inner_iterations(1 - cur, scalars.p + 0) : project(1 - cur, speculate, nullptr);
  if (rc == PXR_OK && !round0_cost) rc = fm(speculate ? 1 : 0, nullptr, scalars.p + 0);
  if (rc != PXR_OK) { swap_sets(); return rc; }
  pack_scalars(1);
  if (ran_inner) {
    if (!round0_cost) rc = inner_iterations(1 - cur);
    if (rc == PXR_OK) rc = project(1 - cur, speculate, nullptr);
    if (rc == PXR_OK) rc = fm(speculate ? 1 : 0, nullptr, scalars.p + 0);
    if (rc == PXR_OK) rc = step_norm_between_sets();
    if (rc != PXR_OK) { swap_sets(); return rc; }
    pack_scalars(2);
  }
  PXR_TRY(exchange_scalars(11));
  double o[12]; double gmax_here = 0; int mfail = 0;
  PXR_CUDA(cudaMemcpyAsync(o, mb_out.p, sizeof(o), cudaMemcpyDeviceToHost, s));
  PXR_CUDA(cudaMemcpyAsync(&gmax_here, scalars.p + 10, 8, cudaMemcpyDeviceToHost, s));
  PXR_CUDA(cudaMemcpyAsync(&mfail, flags.p + 3, sizeof(int), cudaMemcpyDeviceToHost, s));
  PXR_CUDA(cudaStreamSynchronize(s));                         // the ONE host synchronisation of the iteration
  swap_sets();   // back: uv/obs_out/juv = linearisation at the current point again
  if (mfail) { lm.finished = true; lm.term = 2; return fail(PXR_ERR_NCCL, "a peer rank did not deliver its scalars (mailbox time-out)"); }
  t->gmax = std::max(gmax_here, o[11]);    // camera part (global g_c) | point part (max over the ranks)
  t->interrupted = o[10] > 0.0;
  t->model_cost_change = -o[0];
  t->valid = o[1] == 0.0 && std::isfinite(o[0]) && t->model_cost_change > 0.0;
  t->cost = o[2]; t->inner_cost = o[7];
  t->step_sq[0] = o[3]; t->step_sq[1] = o[5]; t->x_sq[0] = o[4]; t->x_sq[1] = o[6];
  t->inner_step_sq[0] = o[8]; t->inner_step_sq[1] = o[9];
  return PXR_OK;
}

// Moves the linearisation to the accepted point (cur already names it) and sets lm.x_cost and its max |g|.
int BA::lm_move(double candidate_cost, double next_cost) {
  pxr_iteration_summary& it = lm.it;
  const bool reuse = !env.no_speculation && candidate_cost < std::numeric_limits<double>::max();
  if (!block_mode) {
    if (reuse) {
      swap_sets();                   // the speculative pass IS the linearisation at the new point
      PXR_TRY(build());
      lm.x_cost = next_cost;         // single GPU: the cost of that pass
    } else {
      PXR_TRY(evaluate(cur, true, &lm.x_cost));
    }
  } else {
    if (reuse) {
      swap_sets();
    } else {
      PXR_TRY(project(cur, true, nullptr));
      PXR_TRY(fm(1, nullptr, scalars.p + 0));
    }
    PXR_TRY(build_block());
    lm.x_cost = candidate_cost;      // block mode: the trial cost (after the inner iterations) is the new cost
  }
  it.cost = lm.x_cost;
  return lm_gradient(&it.gradient_max_norm);   // single GPU: a host synchronisation
}

// Runs LM iterations until iteration index `max_iteration` (absolute) or termination.
int BA::lm_iterate(int max_iteration) {
  using clk = std::chrono::steady_clock;
  const double kMax = std::numeric_limits<double>::max();
  if (!lm.started) PXR_TRY(lm_begin());
  lm.it_start = clk::now();
  while (!lm.finished && lm_finalize(max_iteration)) {
    const bool interrupted = interrupt_pending();     // Ctrl-C in the host (util/src/py_interrupt.h:29-38)
    lm.it_start = clk::now();
    pxr_iteration_summary& it = lm.it;
    const pxr_iteration_summary prev_it = it;
    const double prev_gmax = it.gradient_max_norm;
    const int iteration = it.iteration + 1;
    std::memset(&it, 0, sizeof(it));
    it.iteration = iteration;
    lm.pending_finalize = true;

    const bool ran_inner = lm.inner_enabled;
    LMTrial t;
    PXR_TRY(lm_trial(interrupted, ran_inner, &t));
    it.linear_solver_iterations = last_linear_iterations;
    if (lm.gmax_pending) {
      // block mode, several ranks: max |g| at the CURRENT point arrives with this iteration's all-reduce; ceres tests it
      // before starting the iteration: when it already meets the tolerance, this iteration never happened
      lm.gmax_pending = false;
      if (!lm.its.empty()) lm.its.back().gradient_max_norm = t.gmax;
      if (t.gmax <= opt.gradient_tolerance) {
        it = prev_it; it.gradient_max_norm = t.gmax;
        lm.pending_finalize = false;
        lm.term = 0; lm.message = "Gradient tolerance reached."; lm.finished = true;
        break;
      }
    }
    // the max |g| an invalid or rejected step reports: the one at the current point, which block mode with several
    // ranks learns only now
    const double known_gmax = blk_lag_gmax ? t.gmax : prev_gmax;
    if (t.interrupted) {     // stop between iterations: this one never happened
      it = prev_it; lm.pending_finalize = false;
      lm.finished = true; lm.term = 3; lm.message = "interrupted by the host";
      return fail(PXR_ERR_INTERRUPTED, "interrupted by the host after LM iteration %d", it.iteration);
    }
    it.step_is_valid = t.valid;
    if (!t.valid) {
      if (lm.tr.invalid_step()) {
        lm.term = 2; lm.finished = true;
        lm.message = "Number of consecutive invalid steps more than Solver::Options::max_num_consecutive_invalid_steps";
        break;
      }
      it.cost = lm.x_cost; it.gradient_max_norm = known_gmax;
      continue;
    }
    lm.tr.num_invalid = 0;

    double model_cost_change = t.model_cost_change;
    double candidate_cost = std::isfinite(t.cost) ? t.cost : kMax;
    double step_norm = std::sqrt(t.step_sq[0] + t.step_sq[1]);
    const double x_norm = std::sqrt(t.x_sq[0] + t.x_sq[1]);
    const double next_cost = ran_inner ? t.inner_cost : candidate_cost;     // the cost of the pass left in the alternate set
    bool inner_useful = false;
    if (ran_inner && candidate_cost < kMax) {
      ++lm.n_inner;
      const double inner_cost = t.inner_cost;
      if (std::isfinite(inner_cost)) {
        model_cost_change += candidate_cost - inner_cost;
        inner_useful = inner_cost < lm.x_cost;
        const double rel = 1.0 - inner_cost / candidate_cost;
        lm.inner_enabled = rel > opt.inner_iteration_tolerance;
        candidate_cost = inner_cost;
        step_norm = std::sqrt(t.inner_step_sq[0] + t.inner_step_sq[1]);
      }
    }
    it.step_norm = step_norm;
    it.cost_change = lm.x_cost - candidate_cost;
    const int tol = lm.tr.tolerance(step_norm, x_norm, it.cost_change, lm.x_cost);
    if (tol) {
      lm.term = 0; lm.finished = true;
      lm.message = tol == TR_PARAMETER_TOLERANCE ? "Parameter tolerance reached." : "Function tolerance reached.";
      break;
    }
    it.relative_decrease = lm.tr.ev.quality(candidate_cost, model_cost_change);
    if (inner_useful || lm.tr.successful(it.relative_decrease)) {
      cur = 1 - cur;
      // The accepted cost: the single-GPU driver takes the post-inner pass (next_cost), block mode the trial cost after
      // the inner iterations.  They differ only when the post-inner cost is not finite while the trial cost is.
      PXR_TRY(lm_move(candidate_cost, next_cost));
      it.step_is_successful = 1;
      lm.tr.accept(it.relative_decrease, candidate_cost, model_cost_change);
      if (opt.use_nonmonotonic_steps) {
        // ceres copies x into the user's parameter blocks only when it is the best iterate so far
        // (FinalizeIterationAndCheckIfMinimizerCanContinue); a non-monotonic acceptance moves away from it, so the
        // iterate being left (still intact in the other parameter set) is snapshotted on the device
        if (lm.x_cost < lm.minimum_cost) lm.best_is_current = true;
        else if (lm.best_is_current) { PXR_TRY(save_best(1 - cur)); lm.best_is_current = false; }
      }
    } else {
      it.step_is_successful = 0;
      it.cost = candidate_cost;
      it.gradient_max_norm = known_gmax;
      lm.tr.reject();
    }
  }
  if (lm.x_cost < lm.minimum_cost) lm.minimum_cost = lm.x_cost;
  if (lm.finished) PXR_TRY(finish_gmax_block());   // block mode, several ranks: the max |g| no iteration delivered
  PXR_CUDA(cudaStreamSynchronize(ctx->stream));
  return PXR_OK;
}

void BA::fill_summary(pxr_summary* sum, double seconds, int64_t launches) {
  if (!sum) return;
  sum->initial_cost = lm.initial_cost; sum->final_cost = lm.minimum_cost;
  sum->num_residual_blocks = (int32_t)n_obs; sum->num_residuals = n_obs * C;
  sum->num_successful_steps = lm.n_succ; sum->num_unsuccessful_steps = lm.n_unsucc;
  sum->num_inner_iteration_steps = lm.n_inner; sum->termination_type = lm.term;
  sum->solve_time_s = seconds; sum->total_time_s = seconds;
  sum->h2d_bytes = h2d_bytes; sum->d2h_bytes = 0;
  sum->num_iterations = (int32_t)lm.its.size();
  const int m = std::min<int>((int)lm.its.size(), sum->iterations ? sum->iterations_capacity : 0);
  for (int i = 0; i < m; ++i) sum->iterations[i] = lm.its[i];
  sum->kernel_launches = launches;
  std::snprintf(sum->message, sizeof(sum->message), "%s", lm.message.c_str());
  sum->resident_window = resident ? res_window : 0;
  sum->resident_passes_repeated = (int32_t)res_passes_repeated; sum->resident_refetched = res_refetched;
}

int BA::solve(pxr_summary* sum) {
  const auto t0 = std::chrono::steady_clock::now();
  const int64_t l0 = ctx->launches;
  PXR_TRY(lm_begin());
  PXR_TRY(lm_iterate(opt.max_num_iterations));
  if (block_mode) PXR_TRY(finish_gmax_block());
  fill_summary(sum, std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count(), ctx->launches - l0);
  return PXR_OK;
}

int BA::save_best(int set) {
  cudaStream_t s = ctx->stream;
  if (!best_cam.p) {
    PXR_TRY(best_cam.alloc((size_t)n_cameras * kMaxK)); PXR_TRY(best_q.alloc((size_t)n_images * 4));
    PXR_TRY(best_t.alloc((size_t)n_images * 3)); PXR_TRY(best_X.alloc((size_t)n_points * 3));
  }
  PXR_CUDA(cudaMemcpyAsync(best_cam.p, cam[set].p, best_cam.n * 8, cudaMemcpyDeviceToDevice, s));
  PXR_CUDA(cudaMemcpyAsync(best_q.p, q[set].p, best_q.n * 8, cudaMemcpyDeviceToDevice, s));
  PXR_CUDA(cudaMemcpyAsync(best_t.p, t[set].p, best_t.n * 8, cudaMemcpyDeviceToDevice, s));
  if (best_X.n) PXR_CUDA(cudaMemcpyAsync(best_X.p, X[set].p, best_X.n * 8, cudaMemcpyDeviceToDevice, s));
  return PXR_OK;
}

int BA::read_params(double* cam_o, double* q_o, double* t_o, double* X_o) {
  cudaStream_t s = ctx->stream;
  // the lowest-cost iterate, as ceres leaves it in the user's parameter blocks
  const bool best = lm.started && !lm.best_is_current && best_cam.p;
  const double* pc = best ? best_cam.p : cam[cur].p; const double* pq = best ? best_q.p : q[cur].p;
  const double* pt = best ? best_t.p : t[cur].p; const double* pX = best ? best_X.p : X[cur].p;
  if (cam_o) PXR_CUDA(cudaMemcpyAsync(cam_o, pc, (size_t)n_cameras * kMaxK * 8, cudaMemcpyDeviceToHost, s));
  if (q_o) PXR_CUDA(cudaMemcpyAsync(q_o, pq, (size_t)n_images * 4 * 8, cudaMemcpyDeviceToHost, s));
  if (t_o) PXR_CUDA(cudaMemcpyAsync(t_o, pt, (size_t)n_images * 3 * 8, cudaMemcpyDeviceToHost, s));
  if (X_o) PXR_CUDA(cudaMemcpyAsync(X_o, pX, (size_t)n_points * 3 * 8, cudaMemcpyDeviceToHost, s));
  PXR_CUDA(cudaStreamSynchronize(s));
  return PXR_OK;
}

}  // namespace pxr

using namespace pxr;

extern "C" {

int pxr_ba_create(pxr_ctx* ctx, const pxr_ba_desc* desc, const pxr_interp_config* interp,
                  const pxr_solver_options* opt, pxr_ba** out) {
  if (!ctx || !out) return fail(PXR_ERR_INVALID_ARGUMENT, "ctx/out is NULL");
  BA* b = new BA();
  const int rc = b->create(ctx, desc, interp, opt, true);
  if (rc != PXR_OK) { delete b; return rc; }
  *out = reinterpret_cast<pxr_ba*>(b);
  return PXR_OK;
}
int pxr_ba_destroy(pxr_ba* ba) {
  if (ba) { BA* b = reinterpret_cast<BA*>(ba); cudaSetDevice(b->ctx->device); delete b; }
  return PXR_OK;
}
int pxr_ba_solve(pxr_ba* ba, pxr_summary* summary) {
  if (!ba) return fail(PXR_ERR_INVALID_ARGUMENT, "ba is NULL");
  return reinterpret_cast<BA*>(ba)->solve(summary);
}
int pxr_ba_iterate(pxr_ba* ba, int n_iterations, pxr_summary* summary) {
  if (!ba || n_iterations < 0) return fail(PXR_ERR_INVALID_ARGUMENT, "bad arguments");
  BA* b = reinterpret_cast<BA*>(ba);
  const auto t0 = std::chrono::steady_clock::now();
  const int64_t l0 = b->ctx->launches;
  if (!b->lm.started) PXR_TRY(b->lm_begin());
  PXR_TRY(b->lm_iterate(b->lm.it.iteration + n_iterations));
  b->fill_summary(summary, std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count(), b->ctx->launches - l0);
  return PXR_OK;
}
int pxr_ba_kernel_timing(pxr_ba* ba, int enable, int which, double* total_ms, int* count) {
  if (!ba) return fail(PXR_ERR_INVALID_ARGUMENT, "ba is NULL");
  BA* b = reinterpret_cast<BA*>(ba);
  PXR_CUDA(cudaSetDevice(b->ctx->device));
  if (total_ms || count) {
    PXR_CUDA(cudaStreamSynchronize(b->ctx->stream));
    double tot = 0; int n = 0;
    if (which < 0 || which >= BA::kNumStages) return fail(PXR_ERR_INVALID_ARGUMENT, "bad stage id");
    for (auto& pr : b->timed[which]) {
      float ms = 0;
      if (cudaEventElapsedTime(&ms, pr.first, pr.second) == cudaSuccess) { tot += ms; ++n; }
    }
    if (total_ms) *total_ms = tot;
    if (count) *count = n;
  }
  if (enable >= 0) {
    for (int k = 0; k < BA::kNumStages; ++k) { for (auto& pr : b->timed[k]) { cudaEventDestroy(pr.first); cudaEventDestroy(pr.second); } b->timed[k].clear(); }
    b->time_kernels = enable != 0;
  }
  return PXR_OK;
}
int pxr_ba_read_params(pxr_ba* ba, double* cam_params, double* qvec, double* tvec, double* xyz) {
  if (!ba) return fail(PXR_ERR_INVALID_ARGUMENT, "ba is NULL");
  return reinterpret_cast<BA*>(ba)->read_params(cam_params, qvec, tvec, xyz);
}
int pxr_ba_reset(pxr_ba* ba, const double* cam_params, const double* qvec, const double* tvec, const double* xyz) {
  if (!ba || !cam_params || !qvec || !tvec) return fail(PXR_ERR_INVALID_ARGUMENT, "NULL argument");
  BA* b = reinterpret_cast<BA*>(ba);
  PXR_CUDA(cudaSetDevice(b->ctx->device));
  cudaStream_t s = b->ctx->stream;
  if (b->n_points > 0 && !xyz) return fail(PXR_ERR_INVALID_ARGUMENT, "xyz is NULL");
  for (int k = 0; k < 2; ++k) {
    PXR_CUDA(cudaMemcpyAsync(b->cam[k].p, cam_params, (size_t)b->n_cameras * kMaxK * 8, cudaMemcpyHostToDevice, s));
    PXR_CUDA(cudaMemcpyAsync(b->q[k].p, qvec, (size_t)b->n_images * 4 * 8, cudaMemcpyHostToDevice, s));
    PXR_CUDA(cudaMemcpyAsync(b->t[k].p, tvec, (size_t)b->n_images * 3 * 8, cudaMemcpyHostToDevice, s));
    if (b->n_points > 0) PXR_CUDA(cudaMemcpyAsync(b->X[k].p, xyz, (size_t)b->n_points * 3 * 8, cudaMemcpyHostToDevice, s));
  }
  PXR_CUDA(cudaStreamSynchronize(s));
  b->cur = 0;
  b->lm = LMState();
  return PXR_OK;
}
int pxr_ba_run(pxr_ctx* ctx, const pxr_ba_desc* desc, const pxr_interp_config* interp,
               const pxr_solver_options* opt, pxr_summary* summary) {
  const auto t0 = std::chrono::steady_clock::now();
  if (!ctx) return fail(PXR_ERR_INVALID_ARGUMENT, "ctx is NULL");
  // one-shot call: the caller's patch buffer outlives the solve, so the slab may stay partially resident
  // (pxr_resident.cuh) — only the tap windows the solve touches cross PCIe
  BA* b = new BA();
  b->allow_resident = true;
  {
    const int rc0 = b->create(ctx, desc, interp, opt, true);
    if (rc0 != PXR_OK) { delete b; return rc0; }
  }
  pxr_ba* h = reinterpret_cast<pxr_ba*>(b);
  int rc = b->solve(summary);
  if (rc == PXR_OK) rc = b->read_params(desc->cam_params, desc->qvec, desc->tvec, desc->xyz);
  pxr_ba_destroy(h);      // inside the timed call: what the caller waits for
  if (summary) {
    summary->d2h_bytes = ((double)desc->n_cameras * kMaxK + desc->n_images * 7.0 + desc->n_points * 3.0) * 8.0;
    summary->total_time_s = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  }
  return rc;
}

// Geometric BA (GeometricBundleOptimizer): the arguments are checked on the host first, so a bad problem is reported
// as such on any machine; a NULL context then means there is no device to run on.
static int geometric_args(pxr_ctx* ctx, const pxr_ba_desc* desc, const double* obs_xy) {
  PXR_TRY(check_desc_geometric(desc, obs_xy));
  if (ctx) return PXR_OK;
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0) {
    cudaGetLastError();
    return fail(PXR_ERR_NO_DEVICE, "no CUDA device available; libpxr has no CPU fallback");
  }
  return fail(PXR_ERR_INVALID_ARGUMENT, "ctx is NULL");
}

int pxr_ba_create_geometric(pxr_ctx* ctx, const pxr_ba_desc* desc, const double* obs_xy, const pxr_solver_options* opt,
                            pxr_ba** out) {
  if (!out) return fail(PXR_ERR_INVALID_ARGUMENT, "out is NULL");
  PXR_TRY(geometric_args(ctx, desc, obs_xy));
  BA* b = new BA();
  const int rc = b->create(ctx, desc, nullptr, opt, true, obs_xy);
  if (rc != PXR_OK) { delete b; return rc; }
  *out = reinterpret_cast<pxr_ba*>(b);
  return PXR_OK;
}

int pxr_ba_run_geometric(pxr_ctx* ctx, const pxr_ba_desc* desc, const double* obs_xy, const pxr_solver_options* opt,
                         pxr_summary* summary) {
  const auto t0 = std::chrono::steady_clock::now();
  PXR_TRY(geometric_args(ctx, desc, obs_xy));
  BA* b = new BA();
  {
    const int rc0 = b->create(ctx, desc, nullptr, opt, true, obs_xy);
    if (rc0 != PXR_OK) { delete b; return rc0; }
  }
  int rc = b->solve(summary);
  if (rc == PXR_OK) rc = b->read_params(desc->cam_params, desc->qvec, desc->tvec, desc->xyz);
  pxr_ba_destroy(reinterpret_cast<pxr_ba*>(b));
  if (summary) {
    summary->d2h_bytes = ((double)desc->n_cameras * kMaxK + desc->n_images * 7.0 + desc->n_points * 3.0) * 8.0;
    summary->total_time_s = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  }
  return rc;
}

int pxr_ba_evaluate(pxr_ba* ba, double* sq_norm, double* gtr, double* gtg, double* xy, double* residuals,
                    double* cost) {
  if (!ba) return fail(PXR_ERR_INVALID_ARGUMENT, "ba is NULL");
  BA* b = reinterpret_cast<BA*>(ba);
  pxr_ctx* ctx = b->ctx;
  PXR_CUDA(cudaSetDevice(ctx->device));
  DevBuf<double> dxy, dres;
  if (xy) PXR_TRY(dxy.alloc((size_t)b->n_obs * 2));
  if (residuals) PXR_TRY(dres.alloc((size_t)b->n_obs * b->C));
  PXR_TRY(b->project(b->cur, true, dxy.p));
  PXR_TRY(b->fm(1, dres.p, b->scalars.p + 0));
  std::vector<double> out((size_t)b->n_obs * 8);
  double c = 0;
  PXR_CUDA(cudaMemcpyAsync(out.data(), b->obs_out.p, out.size() * 8, cudaMemcpyDeviceToHost, ctx->stream));
  PXR_CUDA(cudaMemcpyAsync(&c, b->scalars.p, 8, cudaMemcpyDeviceToHost, ctx->stream));
  if (xy) PXR_CUDA(cudaMemcpyAsync(xy, dxy.p, (size_t)b->n_obs * 16, cudaMemcpyDeviceToHost, ctx->stream));
  if (residuals) PXR_CUDA(cudaMemcpyAsync(residuals, dres.p, (size_t)b->n_obs * b->C * 8, cudaMemcpyDeviceToHost, ctx->stream));
  PXR_CUDA(cudaStreamSynchronize(ctx->stream));
  for (int64_t o = 0; o < b->n_obs; ++o) {
    const double* r = &out[(size_t)o * 8];
    if (sq_norm) sq_norm[o] = r[0];
    if (gtr) { gtr[2 * o] = r[1]; gtr[2 * o + 1] = r[2]; }
    if (gtg) { gtg[3 * o] = r[3]; gtg[3 * o + 1] = r[4]; gtg[3 * o + 2] = r[5]; }
  }
  if (cost) *cost = c;
  return PXR_OK;
}

// The cost-functor surface (residuals/bindings.cc:14-30): residual vectors and the two factors of every block's
// Jacobian, J = G * P.
int pxr_ba_evaluate_jacobians(pxr_ba* ba, double* residuals, double* grad, double* juv, int32_t* juv_cols, double* xy) {
  if (!ba) return fail(PXR_ERR_INVALID_ARGUMENT, "ba is NULL");
  BA* b = reinterpret_cast<BA*>(ba);
  pxr_ctx* ctx = b->ctx;
  PXR_CUDA(cudaSetDevice(ctx->device));
  const size_t n = (size_t)b->n_obs, C = (size_t)b->C;
  const int W = 9 + b->K;
  if (juv_cols) *juv_cols = W;
  DevBuf<double> dxy, dres, dgrad;
  if (xy) PXR_TRY(dxy.alloc(n * 2));
  if (residuals) PXR_TRY(dres.alloc(n * C));
  if (grad) PXR_TRY(dgrad.alloc(n * 2 * C));
  PXR_TRY(b->project(b->cur, true, dxy.p));
  PXR_TRY(b->fm(1, dres.p, b->scalars.p + 0, dgrad.p));
  cudaStream_t s = ctx->stream;
  if (xy) PXR_CUDA(cudaMemcpyAsync(xy, dxy.p, n * 16, cudaMemcpyDeviceToHost, s));
  if (residuals) PXR_CUDA(cudaMemcpyAsync(residuals, dres.p, n * C * 8, cudaMemcpyDeviceToHost, s));
  if (grad) PXR_CUDA(cudaMemcpyAsync(grad, dgrad.p, n * 2 * C * 8, cudaMemcpyDeviceToHost, s));
  if (juv && n > 0)     // device rows are juv_stride doubles apart, 2 x W of them used
    PXR_CUDA(cudaMemcpy2DAsync(juv, (size_t)2 * W * 8, b->juv.p, (size_t)b->juv_stride * 8, (size_t)2 * W * 8, n, cudaMemcpyDeviceToHost, s));
  PXR_CUDA(cudaStreamSynchronize(s));
  return PXR_OK;
}


// Introspection for parity tests: linearise at the current parameters and compute one LM step at
// `radius` (Jacobi scaling from this linearisation, as in iteration 0).  Any output may be NULL.
int pxr_ba_debug_linearize(pxr_ba* ba, double radius, double* cost, double* Hcc, double* gc, double* Hpp,
                           double* gp, double* S, double* rhs, double* delta, double* model_cost_change) {
  if (!ba) return fail(PXR_ERR_INVALID_ARGUMENT, "ba is NULL");
  BA* b = reinterpret_cast<BA*>(ba);
  pxr_ctx* ctx = b->ctx;
  cudaStream_t s = ctx->stream;
  PXR_CUDA(cudaSetDevice(ctx->device));
  if ((b->sparse_schur || b->block_mode) && (Hcc || S)) return fail(PXR_ERR_UNSUPPORTED, "the block-sparse path has no dense Hcc / S to return");
  double c = 0;
  PXR_TRY(b->evaluate(b->cur, true, &c));
  if (cost) *cost = c;
  if (b->block_mode) {   // point columns now, camera columns after the all-reduce inside compute_step
    if (b->nl - b->nc > 0) PXR_LAUNCH(ctx, ba_scale_kernel, (unsigned)cdiv(b->nl - b->nc, 256), 256, 0, b->diag.p + b->nc, b->jscale.p + b->nc, b->nl - b->nc, b->opt.jacobi_scaling);
    b->jscale_c_pending = true;
  } else if (b->nl > 0) PXR_LAUNCH(ctx, ba_scale_kernel, (unsigned)cdiv(b->nl, 256), 256, 0, b->diag.p, b->jscale.p, b->nl, b->opt.jacobi_scaling);
  const size_t nc = b->nc;
  if (Hcc) PXR_CUDA(cudaMemcpyAsync(Hcc, b->Hcc.p, nc * nc * 8, cudaMemcpyDeviceToHost, s));
  if (gc) PXR_CUDA(cudaMemcpyAsync(gc, b->block_mode ? b->pack_local.p + b->pk_off_gc : b->gc.p, nc * 8, cudaMemcpyDeviceToHost, s));   // block mode: this rank's partial
  if (Hpp) PXR_CUDA(cudaMemcpyAsync(Hpp, b->Hpp.p, (size_t)b->n_points * 72, cudaMemcpyDeviceToHost, s));
  if (gp) PXR_CUDA(cudaMemcpyAsync(gp, b->gp.p, (size_t)b->n_points * 24, cudaMemcpyDeviceToHost, s));
  PXR_CUDA(cudaStreamSynchronize(s));
  if (S || rhs) {
    // the damped Schur system before factorisation: rerun the assembly part only
    PXR_TRY(b->build_schur_pairs());
    BADev d = b->dev();
    if (b->nl > 0) PXR_LAUNCH(ctx, ba_d2_kernel, (unsigned)cdiv(b->nl, 256), 256, 0, b->diag.p, b->jscale.p, b->D2.p, b->nl, radius,
                              b->opt.min_lm_diagonal, b->opt.max_lm_diagonal);
    if (nc > 0) PXR_LAUNCH(ctx, ba_init_reduced_kernel, (unsigned)cdiv((int64_t)nc * nc, 256), 256, 0, b->Hcc.p, b->gc.p, b->D2.p, b->S.p, b->rhs.p, (int)nc, 1);
    PXR_CUDA(cudaMemsetAsync(b->flags.p, 0, 4 * sizeof(int), s));
    if (b->n_points > 0) {
      PXR_LAUNCH(ctx, ba_point_inverse_kernel, (unsigned)cdiv(b->n_points, 256), 256, 0, d, b->D2.p, b->Hinv.p, b->flags.p);
      PXR_TRY(b->launch_schur_pairs(d));
    }
    if (S) PXR_CUDA(cudaMemcpyAsync(S, b->S.p, nc * nc * 8, cudaMemcpyDeviceToHost, s));
    if (rhs) PXR_CUDA(cudaMemcpyAsync(rhs, b->rhs.p, nc * 8, cudaMemcpyDeviceToHost, s));
    PXR_CUDA(cudaStreamSynchronize(s));
  }
  bool valid = false;
  double mcc = 0;
  PXR_TRY(b->compute_step(radius, &valid, &mcc));
  if (delta) PXR_CUDA(cudaMemcpyAsync(delta, b->delta.p, (size_t)b->nl * 8, cudaMemcpyDeviceToHost, s));
  PXR_CUDA(cudaStreamSynchronize(s));
  if (model_cost_change) *model_cost_change = mcc;
  return PXR_OK;
}

// The reduced solve on a caller's system (tests): S [nc][nc] (lower triangle read) and rhs go where compute_step's
// assembly puts them, then BA::solve_reduced runs the handle's solver.
int pxr_ba_debug_reduced_solve(pxr_ba* ba, const double* S, const double* rhs, double* x, double* factor, int* status,
                               int* linear_iterations) {
  if (!ba || !S || !rhs || !x) return fail(PXR_ERR_INVALID_ARGUMENT, "ba, S, rhs and x must not be NULL");
  BA* b = reinterpret_cast<BA*>(ba);
  if (b->sparse_schur || b->block_mode) return fail(PXR_ERR_UNSUPPORTED, "the block-sparse path has no dense S to solve");
  pxr_ctx* ctx = b->ctx;
  cudaStream_t s = ctx->stream;
  PXR_CUDA(cudaSetDevice(ctx->device));
  const size_t nc = (size_t)b->nc;
  if (nc > 0) {
    PXR_CUDA(cudaMemcpyAsync(b->S.p, S, nc * nc * 8, cudaMemcpyHostToDevice, s));
    PXR_CUDA(cudaMemcpyAsync(b->S.p + nc * nc, rhs, nc * 8, cudaMemcpyHostToDevice, s));   // row nc: the Cholesky's rhs
    PXR_CUDA(cudaMemcpyAsync(b->rhs.p, rhs, nc * 8, cudaMemcpyHostToDevice, s));           // the PCG's
  }
  PXR_CUDA(cudaMemsetAsync(b->flags.p, 0, 4 * sizeof(int), s));
  PXR_TRY(b->solve_reduced());
  int fl[4] = {0, 0, 0, 0};
  PXR_CUDA(cudaMemcpyAsync(fl, b->flags.p, sizeof(fl), cudaMemcpyDeviceToHost, s));
  if (nc > 0) PXR_CUDA(cudaMemcpyAsync(x, b->delta.p, nc * 8, cudaMemcpyDeviceToHost, s));
  if (factor && nc > 0 && !b->use_pcg) PXR_CUDA(cudaMemcpyAsync(factor, b->S.p, (nc + 1) * nc * 8, cudaMemcpyDeviceToHost, s));
  PXR_CUDA(cudaStreamSynchronize(s));
  int st = fl[1] != 0 ? 1 : 0;
  if (st && !b->use_pcg && b->chol_graph_exec && !b->chol_multikernel) {
    // the persistent kernel raises the same flag when it bails out of a wait; its abort word tells the two apart
    int aborted = 0;
    PXR_CUDA(cudaMemcpy(&aborted, b->chol_sync.p + (pxr_chol::sync_ints((int)cdiv((int64_t)nc, kNB)) - 1), sizeof(int), cudaMemcpyDeviceToHost));
    if (aborted) st = 2;
  }
  if (status) *status = st;
  if (linear_iterations) *linear_iterations = b->last_linear_iterations;
  return PXR_OK;
}

// Runs inner iterations on the current parameter set (parity tests).
int pxr_ba_debug_inner_iterations(pxr_ba* ba) {
  if (!ba) return fail(PXR_ERR_INVALID_ARGUMENT, "ba is NULL");
  BA* b = reinterpret_cast<BA*>(ba);
  PXR_CUDA(cudaSetDevice(b->ctx->device));
  PXR_TRY(b->inner_iterations(b->cur));
  PXR_CUDA(cudaStreamSynchronize(b->ctx->stream));
  return PXR_OK;
}

// K0 + K1 (Jacobian mode) at the current parameters over a list of observations, as one inner-iteration round evaluates
// them (tests): out [n_obs][8] is the per-observation record, NaN for observations not in the list.  count_on_device = 1
// passes the list length through device memory with the grids sized for all observations, as the rounds do.
int pxr_ba_debug_eval_list(pxr_ba* ba, const int64_t* list, int64_t n, int count_on_device, double* out) {
  if (!ba || n < 0 || (n > 0 && !list) || !out) return fail(PXR_ERR_INVALID_ARGUMENT, "bad arguments");
  BA* b = reinterpret_cast<BA*>(ba);
  pxr_ctx* ctx = b->ctx;
  cudaStream_t s = ctx->stream;
  PXR_CUDA(cudaSetDevice(ctx->device));
  if (count_on_device && n > b->n_obs) return fail(PXR_ERR_INVALID_ARGUMENT, "a list counted on the device holds at most n_obs entries");
  for (int64_t i = 0; i < n; ++i)
    if (list[i] < 0 || list[i] >= b->n_obs) return fail(PXR_ERR_INVALID_ARGUMENT, "list entry out of range");
  DevBuf<int64_t> dlist;
  DevBuf<unsigned long long> dn;
  if (n > 0) PXR_TRY(dlist.upload(list, (size_t)n, s));
  PXR_CUDA(cudaMemsetAsync(b->obs_out.p, 0xff, (size_t)b->n_obs * 64, s));
  PXR_TRY(b->alloc_inner_jpt());
  if (count_on_device) {
    const unsigned long long hn = (unsigned long long)n;
    PXR_TRY(dn.upload(&hn, 1, s));
    PXR_TRY(b->eval_list(b->cur, dlist.p, b->n_obs, dn.p));
  } else {
    PXR_TRY(b->eval_list(b->cur, dlist.p, n));
  }
  PXR_CUDA(cudaMemcpyAsync(out, b->obs_out.p, (size_t)b->n_obs * 64, cudaMemcpyDeviceToHost, s));
  PXR_CUDA(cudaStreamSynchronize(s));
  return PXR_OK;
}

// The point-only K0 of the inner-iteration rounds next to the full K0 (tests), at the current parameters: uv_full
// [n_obs][2] from the full projection over all observations, then uv [n_obs][2] and jpt [n_obs][6] (d(uv)/dX, rows u
// then v) from the point-only one over list[0..n), NaN outside the list.  count_on_device as in pxr_ba_debug_eval_list.
int pxr_ba_debug_project_point(pxr_ba* ba, const int64_t* list, int64_t n, int count_on_device, double* uv, double* jpt,
                               double* uv_full) {
  if (!ba || n < 0 || (n > 0 && !list) || !uv || !jpt || !uv_full) return fail(PXR_ERR_INVALID_ARGUMENT, "bad arguments");
  BA* b = reinterpret_cast<BA*>(ba);
  pxr_ctx* ctx = b->ctx;
  cudaStream_t s = ctx->stream;
  PXR_CUDA(cudaSetDevice(ctx->device));
  if (n > b->n_obs) return fail(PXR_ERR_INVALID_ARGUMENT, "a list holds at most n_obs entries");
  for (int64_t i = 0; i < n; ++i)
    if (list[i] < 0 || list[i] >= b->n_obs) return fail(PXR_ERR_INVALID_ARGUMENT, "list entry out of range");
  DevBuf<int64_t> dlist;
  DevBuf<unsigned long long> dn;
  if (n > 0) PXR_TRY(dlist.upload(list, (size_t)n, s));
  PXR_TRY(b->project(b->cur, true, nullptr));
  PXR_CUDA(cudaMemcpyAsync(uv_full, b->uv.p, (size_t)b->n_obs * 16, cudaMemcpyDeviceToHost, s));
  PXR_CUDA(cudaMemsetAsync(b->uv.p, 0xff, (size_t)b->n_obs * 16, s));
  PXR_TRY(b->alloc_inner_jpt());
  PXR_CUDA(cudaMemsetAsync(b->inner_jpt.p, 0xff, (size_t)b->n_obs * 48, s));
  if (count_on_device) {
    const unsigned long long hn = (unsigned long long)n;
    PXR_TRY(dn.upload(&hn, 1, s));
    PXR_TRY(b->project_point_list(b->cur, dlist.p, b->n_obs, dn.p, b->n_obs));
  } else {
    PXR_TRY(b->project_point_list(b->cur, dlist.p, n, nullptr, n));
  }
  PXR_CUDA(cudaMemcpyAsync(uv, b->uv.p, (size_t)b->n_obs * 16, cudaMemcpyDeviceToHost, s));
  PXR_CUDA(cudaMemcpyAsync(jpt, b->inner_jpt.p, (size_t)b->n_obs * 48, cudaMemcpyDeviceToHost, s));
  PXR_CUDA(cudaStreamSynchronize(s));
  return PXR_OK;
}

// K0 over all observations at the current parameters, cost-only (jac = 0) or with Jacobians (tests): uv and xy
int pxr_ba_debug_project(pxr_ba* ba, int jac, double* uv, double* xy) {
  if (!ba || (jac != 0 && jac != 1)) return fail(PXR_ERR_INVALID_ARGUMENT, "bad arguments");
  BA* b = reinterpret_cast<BA*>(ba);
  pxr_ctx* ctx = b->ctx;
  cudaStream_t s = ctx->stream;
  PXR_CUDA(cudaSetDevice(ctx->device));
  DevBuf<double> dxy;
  if (xy) PXR_TRY(dxy.alloc((size_t)b->n_obs * 2));
  PXR_TRY(b->project(b->cur, jac != 0, dxy.p));
  if (uv) PXR_CUDA(cudaMemcpyAsync(uv, b->uv.p, (size_t)b->n_obs * 16, cudaMemcpyDeviceToHost, s));
  if (xy) PXR_CUDA(cudaMemcpyAsync(xy, dxy.p, (size_t)b->n_obs * 16, cudaMemcpyDeviceToHost, s));
  PXR_CUDA(cudaStreamSynchronize(s));
  return PXR_OK;
}

int pxr_ba_debug_inner_capture(pxr_ba* ba, int enable) {
  if (!ba) return fail(PXR_ERR_INVALID_ARGUMENT, "ba is NULL");
  reinterpret_cast<BA*>(ba)->capture_inner_lists = enable != 0;
  return PXR_OK;
}

// Round `round` of the most recent batched inner iterations run with capture on (tests): *n_points / *n_obs are its list
// lengths; plist / list / active (each may be NULL) receive its point list, its observation list and, per listed point,
// whether the round's step kernel kept it active.
int pxr_ba_debug_inner_round_lists(pxr_ba* ba, int round, int64_t* plist, int64_t* list, uint8_t* active, int64_t* n_points,
                                   int64_t* n_obs) {
  if (!ba) return fail(PXR_ERR_INVALID_ARGUMENT, "ba is NULL");
  BA* b = reinterpret_cast<BA*>(ba);
  if (round < 0 || round >= (int)b->cap_active.size()) return fail(PXR_ERR_INVALID_ARGUMENT, "round %d was not captured", round);
  const std::vector<int64_t>& pl = b->cap_plist[round];
  const std::vector<int64_t>& ol = b->cap_list[round];
  if (n_points) *n_points = (int64_t)pl.size();
  if (n_obs) *n_obs = (int64_t)ol.size();
  if (plist) std::copy(pl.begin(), pl.end(), plist);
  if (list) std::copy(ol.begin(), ol.end(), list);
  if (active) std::copy(b->cap_active[round].begin(), b->cap_active[round].end(), active);
  return PXR_OK;
}

int pxr_fm_k1_half_warps(pxr_ctx* ctx, int dtype, int channels, int64_t n_items, int64_t* half_warps) {
  if (!ctx || !half_warps || n_items < 0 || !fm_supported(dtype, channels)) return fail(PXR_ERR_INVALID_ARGUMENT, "bad arguments");
  *half_warps = fm_half_warps(ctx, dtype, channels, n_items);
  return PXR_OK;
}

// K0 + K1 in `mode` (0 cost only, 1 Jacobian) over all observations at the current parameters (tests, K1 measurements):
// out [n_obs][8] is every observation's record as the pass leaves it (mode 0 writes s only; the rest stays NaN).
int pxr_ba_debug_eval_records(pxr_ba* ba, int mode, double* out) {
  if (!ba || (mode != 0 && mode != 1) || !out) return fail(PXR_ERR_INVALID_ARGUMENT, "bad arguments");
  BA* b = reinterpret_cast<BA*>(ba);
  pxr_ctx* ctx = b->ctx;
  cudaStream_t s = ctx->stream;
  PXR_CUDA(cudaSetDevice(ctx->device));
  PXR_CUDA(cudaMemsetAsync(b->obs_out.p, 0xff, (size_t)b->n_obs * 64, s));
  PXR_TRY(b->project(b->cur, true, nullptr));
  PXR_TRY(b->fm(mode, nullptr, b->scalars.p + 0));
  PXR_CUDA(cudaMemcpyAsync(out, b->obs_out.p, (size_t)b->n_obs * 64, cudaMemcpyDeviceToHost, s));
  PXR_CUDA(cudaStreamSynchronize(s));
  return PXR_OK;
}

// The rounds of the most recent batched inner iterations (profiling): for every round r < *n_rounds (at most `capacity`
// are written) counts[2r] active observations and counts[2r+1] active points, and ms[r] its stream time if round timing
// was on during that call (else -1): events around the round's launches, so any time the device waits for the host to
// enqueue the round's work counts too.  enable_timing >= 0 switches round timing on / off for the calls that follow.
int pxr_ba_debug_inner_rounds(pxr_ba* ba, int enable_timing, int capacity, unsigned long long* counts, double* ms, int* n_rounds) {
  if (!ba || capacity < 0) return fail(PXR_ERR_INVALID_ARGUMENT, "bad arguments");
  BA* b = reinterpret_cast<BA*>(ba);
  PXR_CUDA(cudaSetDevice(b->ctx->device));
  PXR_CUDA(cudaStreamSynchronize(b->ctx->stream));
  const int n = b->inner_cnt_host ? b->inner_rounds_run : 0;
  if (n_rounds) *n_rounds = n;
  for (int r = 0; r < std::min(n, capacity); ++r) {
    if (counts) { counts[2 * r] = b->inner_cnt_host[3 * r]; counts[2 * r + 1] = b->inner_cnt_host[3 * r + 1]; }
    if (ms) {
      float t = -1.f;
      if (b->inner_rounds_timed)
        PXR_CUDA(cudaEventElapsedTime(&t, b->inner_round_timed[r][0], b->inner_round_timed[r][3]));
      ms[r] = t;
    }
  }
  if (enable_timing >= 0) b->time_inner_rounds = enable_timing != 0;
  return PXR_OK;
}

// The per-launch split of those rounds (profiling): ms[3r] from the round's start to the end of K0, ms[3r+1] from
// there to the end of K1, ms[3r+2] from there to the end of the step kernel (-1 where round timing was off).  Each part
// is stream time, so it includes the launch gap in front of its kernel.
int pxr_ba_debug_inner_round_split(pxr_ba* ba, int capacity, double* ms, int* n_rounds) {
  if (!ba || capacity < 0 || (capacity > 0 && !ms)) return fail(PXR_ERR_INVALID_ARGUMENT, "bad arguments");
  BA* b = reinterpret_cast<BA*>(ba);
  PXR_CUDA(cudaSetDevice(b->ctx->device));
  PXR_CUDA(cudaStreamSynchronize(b->ctx->stream));
  const int n = b->inner_cnt_host ? b->inner_rounds_run : 0;
  if (n_rounds) *n_rounds = n;
  for (int r = 0; r < std::min(n, capacity); ++r)
    for (int k = 0; k < 3; ++k) {
      float t = -1.f;
      if (b->inner_rounds_timed)
        PXR_CUDA(cudaEventElapsedTime(&t, b->inner_round_timed[r][k], b->inner_round_timed[r][k + 1]));
      ms[3 * r + k] = t;
    }
  return PXR_OK;
}

int pxr_ba_time_stage(pxr_ba* ba, int stage, int iters, double* ms_per_launch) {
  if (!ba || iters < 1 || !ms_per_launch) return fail(PXR_ERR_INVALID_ARGUMENT, "bad arguments");
  BA* b = reinterpret_cast<BA*>(ba);
  pxr_ctx* ctx = b->ctx;
  cudaStream_t s = ctx->stream;
  PXR_CUDA(cudaSetDevice(ctx->device));
  cudaEvent_t e0, e1;
  PXR_CUDA(cudaEventCreate(&e0)); PXR_CUDA(cudaEventCreate(&e1));
  double c;
  PXR_TRY(b->project(b->cur, true, nullptr));  // uv for the current parameters
  DevBuf<int64_t> half_list;                    // stage 6: every second observation
  if (stage == 6) {
    std::vector<int64_t> h((size_t)(b->n_obs / 2));
    for (size_t i = 0; i < h.size(); ++i) h[i] = 2 * (int64_t)i;
    if (!h.empty()) PXR_TRY(half_list.upload(h.data(), h.size(), s));
  }
  PXR_CUDA(cudaStreamSynchronize(s));
  PXR_CUDA(cudaEventRecord(e0, s));
  for (int i = 0; i < iters; ++i) {
    if (stage == 0) PXR_TRY(b->fm(1, nullptr, b->scalars.p));
    else if (stage == 1) PXR_TRY(b->fm(0, nullptr, b->scalars.p));
    else if (stage == 6) PXR_TRY(b->fm_k1(1, nullptr, nullptr, half_list.p, b->n_obs / 2));
    else if (stage == 3) PXR_TRY(b->project(b->cur, true, nullptr));
    else if (stage == 4) PXR_TRY(b->build());
    else if (stage == 5) PXR_TRY(b->inner_iterations(1 - b->cur));
    else PXR_TRY(b->evaluate(b->cur, true, &c));
  }
  PXR_CUDA(cudaEventRecord(e1, s));
  PXR_CUDA(cudaEventSynchronize(e1));
  float ms = 0;
  PXR_CUDA(cudaEventElapsedTime(&ms, e0, e1));
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  *ms_per_launch = (double)ms / iters;
  return PXR_OK;
}

}  // extern "C"
