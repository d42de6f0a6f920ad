// pxr_fm_eval.cuh — the residual/Jacobian hot kernels of the featuremetric path.
//
// K0  ba_project_kernel : one thread per observation. WorldToPixel (reference
//     pixsfm/base/src/projection.h:60-75) + FeaturePatch::ToPixelCoordinates
//     (features/src/featurepatch.h:250-255) with analytic d(uv)/d(pose,point,intrinsics)
//     instead of ceres Jets (residuals/src/feature_reference.h:87-96).
// K1  fm_eval_kernel    : one half-warp per observation, lane <-> 2 groups of C/32 channels.  The 4x4xC
//     tap window of the observation's patch is staged HBM -> shared memory by the TMA bulk-copy
//     engine (cp.async.bulk + mbarrier complete_tx; SASS UBLKCP) through a per-half-warp ring of
//     kFmStages slots, so every half-warp keeps kFmStages*4 KiB of loads in flight while it computes.
//     Border semantics = per-tap clamp (base/src/grid2d.h:29-35): in-range columns are copied
//     as 4 x (4 taps) contiguous rows, clamped windows fall back to 16 per-tap copies.
//     Bicubic: horizontal pass in the input's SIMD precision (fp32 for f16/f32), vertical pass in
//     fp64, same op order as the reference (base/src/interpolation.h:177-218); L2 normalisation
//     with its chain rule (interpolation.h:648-666); residual r = f - ref
//     (feature_reference.h:132-134).  The C-channel contraction collapses to
//     ||r||^2, G^T r (2) and G^T G (3 uniques) by half-warp shuffles — the per-observation Jacobian is
//     rank 2 (J = G * d(uv)/d(theta)).
#pragma once
#include "pxr_device.cuh"

namespace pxr {

struct ProjectArgs {
  const int32_t* obs_img; const int64_t* obs_pt; const int64_t* obs_patch;
  const int32_t* img_cam; const int32_t* cam_model;
  const double* cam_params; const double* qvec; const double* tvec; const double* xyz;
  const int32_t* corner; const double* scale; double ups;
  int64_t obs_begin, obs_end;
  const int64_t* item_index;  // optional: process observations item_index[obs_begin..obs_end) (inner iterations)
  const unsigned long long* n_dev = nullptr;   // optional: the item count lives on the device (obs_end = obs_begin + *n_dev; the
                                               // grid is sized for an upper bound) — no host round trip between list and launch
  double* uv;    // [n_obs][2] (u = col, v = row), patch pixel units
  double* xy;    // optional [n_obs][2]
  double* juv;   // optional [n_obs][juv_stride]: 2 x (6 pose | 3 point | K intr), row-major
  int juv_stride;
  int juv_k;     // K columns stored per row
  double* jpt = nullptr;   // ba_project_point_kernel: [n_obs][6] d(uv)/dX, rows u then v (the point columns of juv)
};

// one observation: uv (and xy) to global memory, the 2 x (9 + K) record d(uv)/d(theta) to `out` (global or shared)
template <bool JAC>
__device__ __forceinline__ void project_observation(const ProjectArgs& a, int64_t o, double* out) {
  const int img = a.obs_img[o];
  const int64_t pt = a.obs_pt[o];
  const int64_t pi = a.obs_patch ? a.obs_patch[o] : o;
  const int cam = a.img_cam[img];
  const int model = a.cam_model[cam];
  double q[4], t[3], X[3], cp[kMaxK];
#pragma unroll
  for (int i = 0; i < 4; ++i) q[i] = a.qvec[4 * (int64_t)img + i];
#pragma unroll
  for (int i = 0; i < 3; ++i) { t[i] = a.tvec[3 * (int64_t)img + i]; X[i] = a.xyz[3 * pt + i]; }
#pragma unroll
  for (int i = 0; i < kMaxK; ++i) cp[i] = a.cam_params[(int64_t)cam * kMaxK + i];
  double xy[2], Jpose[2][6], Jpt[2][3], Jk[2][kMaxK];
  world_to_pixel<JAC>(model, cp, q, t, X, xy, Jpose, Jpt, Jk);
  const double sx = a.scale[2 * pi], sy = a.scale[2 * pi + 1];
  const double cx = (double)a.corner[2 * pi], cy = (double)a.corner[2 * pi + 1];
  a.uv[2 * o] = (xy[0] * sx - 0.5 - cx) * a.ups;
  a.uv[2 * o + 1] = (xy[1] * sy - 0.5 - cy) * a.ups;
  if (a.xy) { a.xy[2 * o] = xy[0]; a.xy[2 * o + 1] = xy[1]; }
  if (JAC && out) {
    const int W = 9 + a.juv_k;
    const double s[2] = {sx * a.ups, sy * a.ups};
#pragma unroll
    for (int r = 0; r < 2; ++r) {
#pragma unroll
      for (int k = 0; k < 6; ++k) out[r * W + k] = s[r] * Jpose[r][k];
#pragma unroll
      for (int k = 0; k < 3; ++k) out[r * W + 6 + k] = s[r] * Jpt[r][k];
      for (int k = 0; k < a.juv_k; ++k) out[r * W + 9 + k] = s[r] * Jk[r][k];
    }
  }
}

template <bool JAC>
__global__ void __launch_bounds__(128) ba_project_kernel(ProjectArgs a) {
  const int64_t end = a.n_dev ? a.obs_begin + (int64_t)*a.n_dev : a.obs_end;
  // grid-stride: a list whose length lives on the device gets a grid bounded by the SM count, not by its upper bound
  for (int64_t k = a.obs_begin + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < end; k += (int64_t)gridDim.x * blockDim.x) {
    const int64_t o = a.item_index ? a.item_index[k] : k;
    project_observation<JAC>(a, o, (JAC && a.juv) ? a.juv + o * (int64_t)a.juv_stride : nullptr);
  }
}

// Point-only variant for the inner-iteration rounds, whose step kernel reads nothing of the record but d(uv)/dX: uv (and
// xy) as above and the 2 x 3 point block to the compact `jpt` ([n_obs][6], rows u then v), 48 B per observation instead
// of 2 x (9 + K) strided doubles in `juv`.  The whole record is still formed, into the thread's row of shared memory as
// ba_project_staged_kernel does: left with nothing to store, the compiler would drop the pose and intrinsics columns
// and could then contract the shared subexpressions differently, and the point columns must be the full K0's bit for
// bit.  Dynamic shared memory: 128 * (juv_stride | 1) doubles, within the 48 KiB a launch gets without an opt-in.
static_assert(128 * ((2 * (9 + kMaxK)) | 1) * sizeof(double) <= 48 * 1024,
              "ba_project_point_kernel's shared rows need the dynamic shared memory opt-in");
static __global__ void __launch_bounds__(128) ba_project_point_kernel(ProjectArgs a) {
  extern __shared__ double sm_proj[];
  const int W = 9 + a.juv_k;
  double* row = sm_proj + threadIdx.x * (a.juv_stride | 1);
  const int64_t end = a.n_dev ? a.obs_begin + (int64_t)*a.n_dev : a.obs_end;
  for (int64_t k = a.obs_begin + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < end; k += (int64_t)gridDim.x * blockDim.x) {
    const int64_t o = a.item_index ? a.item_index[k] : k;
    project_observation<true>(a, o, row);
    double2* out = reinterpret_cast<double2*>(a.jpt + 6 * o);
    out[0] = make_double2(row[6], row[7]);
    out[1] = make_double2(row[8], row[W + 6]);
    out[2] = make_double2(row[W + 7], row[W + 8]);
  }
}

// Full-pass variant (no item list): the 128 records of a CTA are contiguous in `juv`, so they are assembled in shared
// memory (rows padded to an odd number of doubles) and written out with coalesced stores instead of 22 strided
// 8 B stores per thread.  Dynamic shared memory: 128 * (juv_stride | 1) doubles.
static __global__ void __launch_bounds__(128) ba_project_staged_kernel(ProjectArgs a) {
  extern __shared__ double sm_proj[];
  const int tid = threadIdx.x;
  const int64_t o0 = a.obs_begin + (int64_t)blockIdx.x * 128;
  const int n = (int)min((int64_t)128, a.obs_end - o0);
  const int js = a.juv_stride, SP = js | 1;
  if (tid < n) project_observation<true>(a, o0 + tid, sm_proj + tid * SP);
  __syncthreads();
  double* dst = a.juv + o0 * (int64_t)js;
  int r = tid / js, c = tid - r * js;
  const int dr = 128 / js, dcol = 128 - dr * js;
  for (int i = tid; i < n * js; i += 128) {
    dst[i] = sm_proj[r * SP + c];
    r += dr; c += dcol;
    if (c >= js) { c -= js; ++r; }
  }
}

// ---------------------------------------------------------------------------------------------
struct FmEvalArgs {
  const double* uv;            // [n][2]
  const int64_t* item_patch;   // [n] or null (identity)
  const int64_t* item_ref;     // [n] index into refs (point id) or null (identity)
  const uint8_t* patches; int ph, pw;
  const double* refs;          // [n_refs][C] or null -> residual = f
  int64_t begin, end;          // item range
  const int64_t* item_index;   // optional indirection: item k is observation item_index[k] (all per-item arrays use that id)
  double* out;                 // [n][8]: s, b_u, b_v, a_uu, a_uv, a_vv, 0, 0  (JAC) / only s (COST)
  double* residuals;           // optional [n][C]
  double* desc;                // optional [n][C]: interpolated (normalised) descriptor f (reference extraction)
  double* grad = nullptr;      // optional [n][2][C]: d r/d u, d r/d v per channel (Jacobian mode; the cost-functor surface)
  // window residency (pxr_resident.cuh): when set, only the rectangle res_rect[patch] of every patch has been brought
  // to the device; an item whose 4x4 tap window leaves it is appended to viol_list (its outputs are garbage and the
  // host re-runs the pass after fetching the patch)
  const uint32_t* res_rect = nullptr;        // [n_patches] r0 | c0 << 8 | rows << 16 | cols << 24
  unsigned long long* viol_count = nullptr;  // [1]
  int64_t* viol_list = nullptr;              // [viol_capacity]
  long long viol_capacity = 0;               // entries beyond it are dropped (they are reported again by the repeated pass)
  const unsigned long long* end_dev = nullptr;   // optional: item count on the device (end = begin + *end_dev; `end` is then the
                                                 // upper bound the grid was sized for)
  LossParams loss;
  int l2_normalize;
};

// the taps an item reads are rows clamp(row-1 .. row+2) and columns clamp(col-1 .. col+2) (per-tap clamp, grid2d.h:29-35):
// are they all inside the resident rectangle?
__device__ __forceinline__ bool window_resident(uint32_t rect, int row, int col, int ph, int pw) {
  const int r0 = (int)(rect & 255u), c0 = (int)((rect >> 8) & 255u), nr = (int)((rect >> 16) & 255u), ncol = (int)(rect >> 24);
  const int rlo = min(max(row - 1, 0), ph - 1), rhi = min(max(row + 2, 0), ph - 1);
  const int clo = min(max(col - 1, 0), pw - 1), chi = min(max(col + 2, 0), pw - 1);
  return rlo >= r0 && rhi < r0 + nr && clo >= c0 && chi < c0 + ncol;
}

#ifndef PXR_FM_WARPS
#define PXR_FM_WARPS 16        // most warps per K1 CTA
#endif
constexpr int kFmStages = 2;   // TMA ring slots per half-warp
// shared memory for the ring slots of one CTA: 128 KiB for windows of up to 4 KiB (fp16 128 channels), 192 KiB for
// larger ones, which would otherwise leave one warp per scheduler
template <int SLOT> constexpr int fm_ring_bytes() { return SLOT <= 4096 ? 128 * 1024 : 192 * 1024; }
struct FmAux {                 // per-item window geometry, one entry per item of a half-warp's batch (40 B)
  double xc, xr;
  int64_t item;
  const uint8_t* src;
  int col, row;
};
// Warps per CTA: as many as the ring fits into fm_ring_bytes (two halves x kFmStages slots per warp), at most
// PXR_FM_WARPS.  fp16 128 channels: 8 warps, 151 808 B per CTA (the ring, 32 mbarriers, 512 FmAux entries).  Larger rings were
// slower on the H100 (DESIGN.md §3, K1 in detail); why was not isolated.
template <typename T, int C> struct FmCfg {
  static constexpr int kSlot = 16 * C * (int)sizeof(T);
  static constexpr int kFit = fm_ring_bytes<kSlot>() / (2 * kFmStages * kSlot);
  static constexpr int kWarps = kFit < 1 ? 1 : (kFit > PXR_FM_WARPS ? PXR_FM_WARPS : kFit);
  static constexpr int kSmem = kWarps * (2 * kFmStages * kSlot + 2 * kFmStages * 8 + 64 * (int)sizeof(FmAux));
};

template <typename T> struct HorizT { typedef float type; };
template <> struct HorizT<double> { typedef double type; };

// load CPL consecutive channels of one tap from shared memory and widen
template <typename T, int CPL>
__device__ __forceinline__ void load_tap(const uint8_t* p, typename HorizT<T>::type v[CPL]);
template <> __device__ __forceinline__ void load_tap<__half, 4>(const uint8_t* p, float v[4]) {
  const uint2 w = *reinterpret_cast<const uint2*>(p);
  const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&w.x));
  const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&w.y));
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
}
template <> __device__ __forceinline__ void load_tap<__half, 2>(const uint8_t* p, float v[2]) {
  const float2 a = __half22float2(*reinterpret_cast<const __half2*>(p));
  v[0] = a.x; v[1] = a.y;
}
template <> __device__ __forceinline__ void load_tap<__half, 1>(const uint8_t* p, float v[1]) {
  v[0] = __half2float(*reinterpret_cast<const __half*>(p));
}
template <> __device__ __forceinline__ void load_tap<__half, 8>(const uint8_t* p, float v[8]) {
  const uint4 w = *reinterpret_cast<const uint4*>(p);
  const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) { const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&ws[i])); v[2 * i] = a.x; v[2 * i + 1] = a.y; }
}
template <> __device__ __forceinline__ void load_tap<float, 4>(const uint8_t* p, float v[4]) {
  const float4 w = *reinterpret_cast<const float4*>(p); v[0] = w.x; v[1] = w.y; v[2] = w.z; v[3] = w.w;
}
template <> __device__ __forceinline__ void load_tap<float, 2>(const uint8_t* p, float v[2]) {
  const float2 w = *reinterpret_cast<const float2*>(p); v[0] = w.x; v[1] = w.y;
}
template <> __device__ __forceinline__ void load_tap<float, 1>(const uint8_t* p, float v[1]) { v[0] = *reinterpret_cast<const float*>(p); }
template <> __device__ __forceinline__ void load_tap<float, 8>(const uint8_t* p, float v[8]) {
  load_tap<float, 4>(p, v); load_tap<float, 4>(p + 16, v + 4);
}
template <> __device__ __forceinline__ void load_tap<double, 4>(const uint8_t* p, double v[4]) {
  const double2 a = *reinterpret_cast<const double2*>(p); const double2 b = *reinterpret_cast<const double2*>(p + 16);
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
}
template <> __device__ __forceinline__ void load_tap<double, 2>(const uint8_t* p, double v[2]) {
  const double2 a = *reinterpret_cast<const double2*>(p); v[0] = a.x; v[1] = a.y;
}
template <> __device__ __forceinline__ void load_tap<double, 1>(const uint8_t* p, double v[1]) { v[0] = *reinterpret_cast<const double*>(p); }
template <> __device__ __forceinline__ void load_tap<double, 8>(const uint8_t* p, double v[8]) {
  load_tap<double, 4>(p, v); load_tap<double, 4>(p + 32, v + 4);
}

// Bicubic f / dfdr / dfdc for CPL channels from a staged 4x4 window (tap t = 4*i + j at
// win + t*TAP_BYTES), reference op order (interpolation.h:177-218).
// tap address providers: addr(i, j) -> pointer to channel 0 of tap (row i, col j) of the window
template <int TAP_BYTES>
struct SmemWindow {
  const uint8_t* win;
  __device__ __forceinline__ const uint8_t* operator()(int i, int j) const { return win + (4 * i + j) * TAP_BYTES; }
};
struct GlobalWindow {  // clamped rows/cols resolved by the caller (grid2d.h:29-35)
  const uint8_t* rowp[4];
  int coff[4];
  __device__ __forceinline__ const uint8_t* operator()(int i, int j) const { return rowp[i] + coff[j]; }
};

template <typename T, int C, int CPL, bool DERIV, bool FLOAT_SIMD, typename Addr>
__device__ __forceinline__ void bicubic_window(const Addr& addr, int lane, double xc, double xr,
                                               double f[CPL], double fr[CPL], double fc[CPL]) {
  typedef typename HorizT<T>::type H;
  const size_t loff = (size_t)lane * CPL * sizeof(T);
  if (C >= 8) {
    H hf[4][CPL], hd[4][CPL];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      H p0[CPL], p1[CPL], p2[CPL], p3[CPL];
      load_tap<T, CPL>(addr(i, 0) + loff, p0);
      load_tap<T, CPL>(addr(i, 1) + loff, p1);
      load_tap<T, CPL>(addr(i, 2) + loff, p2);
      load_tap<T, CPL>(addr(i, 3) + loff, p3);
      if (sizeof(H) == 4) {
        const SplineCoefF32 cc(xc);
        // Hopper has no packed fp32x2 FMA: one scalar FFMA chain per channel
#pragma unroll
        for (int k = 0; k < CPL; ++k) {
          float ff, dd = 0.f;
          spline_f32<DERIV>((float)p0[k], (float)p1[k], (float)p2[k], (float)p3[k], cc, ff, dd);
          hf[i][k] = (H)ff; hd[i][k] = (H)dd;
        }
      } else {
        const SplineCoefF64 cc(xc);
#pragma unroll
        for (int k = 0; k < CPL; ++k) {
          double ff, dd = 0.0;
          spline_f64<true, DERIV>((double)p0[k], (double)p1[k], (double)p2[k], (double)p3[k], cc, ff, dd);
          hf[i][k] = (H)ff; hd[i][k] = (H)dd;
        }
      }
    }
    if (FLOAT_SIMD) {
      const SplineCoefF32 cr(xr);
#pragma unroll
      for (int k = 0; k < CPL; ++k) {
        float ff, dd = 0.f;
        spline_f32<DERIV>((float)hf[0][k], (float)hf[1][k], (float)hf[2][k], (float)hf[3][k], cr, ff, dd);
        f[k] = (double)ff;
        if (DERIV) {
          fr[k] = (double)dd;
          float gg, unused = 0.f;
          spline_f32<false>((float)hd[0][k], (float)hd[1][k], (float)hd[2][k], (float)hd[3][k], cr, gg, unused);
          fc[k] = (double)gg;
        }
      }
    } else {
      const SplineCoefF64 cr(xr);
#pragma unroll
      for (int k = 0; k < CPL; ++k) {
        double dd = 0.0;
        spline_f64<true, DERIV>((double)hf[0][k], (double)hf[1][k], (double)hf[2][k], (double)hf[3][k], cr, f[k], dd);
        if (DERIV) {
          fr[k] = dd;
          double unused = 0.0;
          spline_f64<true, false>((double)hd[0][k], (double)hd[1][k], (double)hd[2][k], (double)hd[3][k], cr, fc[k], unused);
        }
      }
    }
  } else {
    // C < 8: ceres::CubicHermiteSpline in double (interpolation.h:230-262)
    double hf[4][CPL], hd[4][CPL];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      H p0[CPL], p1[CPL], p2[CPL], p3[CPL];
      load_tap<T, CPL>(addr(i, 0) + loff, p0);
      load_tap<T, CPL>(addr(i, 1) + loff, p1);
      load_tap<T, CPL>(addr(i, 2) + loff, p2);
      load_tap<T, CPL>(addr(i, 3) + loff, p3);
#pragma unroll
      for (int k = 0; k < CPL; ++k) {
        hd[i][k] = 0.0;
        spline_ceres<DERIV>((double)p0[k], (double)p1[k], (double)p2[k], (double)p3[k], xc, hf[i][k], hd[i][k]);
      }
    }
#pragma unroll
    for (int k = 0; k < CPL; ++k) {
      double dd = 0.0, unused = 0.0;
      spline_ceres<DERIV>(hf[0][k], hf[1][k], hf[2][k], hf[3][k], xr, f[k], dd);
      if (DERIV) { fr[k] = dd; spline_ceres<false>(hd[0][k], hd[1][k], hd[2][k], hd[3][k], xr, fc[k], unused); }
    }
  }
}

// PixelInterpolator L2 normalisation + residual + rank-2 reduction for one item, whole warp.
// ALLRED=true : red[0..5] valid in every lane (butterfly all-reduce).
// ALLRED=false: transposed reduction — returns in lane L the total of value ((L>>4)&1)*4+((L>>3)&1)*2+((L>>2)&1)
//               (0:s 1:b_u 2:b_v 3:a_uu 4:a_uv 5:a_vv), 9 double shuffles instead of 30.
template <int CPL, bool DERIV, bool ALLRED>
__device__ __forceinline__ double normalize_and_reduce(bool active, bool l2, const double* refp /*lane's CPL refs or null*/,
                                                       double f[CPL], double fr[CPL], double fc[CPL],
                                                       double r[CPL], double red[6], int lane) {
  if (l2) {
    double n2 = 0.0;
    if (active) {
#pragma unroll
      for (int k = 0; k < CPL; ++k) n2 += f[k] * f[k];
    }
    n2 = warp_sum(n2);
    const double ninv = 1.0 / sqrt(n2);
    double dc = 0.0, dr = 0.0;
#pragma unroll
    for (int k = 0; k < CPL; ++k) {
      f[k] *= ninv;
      if (DERIV) { fc[k] *= ninv; fr[k] *= ninv; if (active) { dc += f[k] * fc[k]; dr += f[k] * fr[k]; } }
    }
    if (DERIV) {
      dc = warp_sum(dc); dr = warp_sum(dr);
#pragma unroll
      for (int k = 0; k < CPL; ++k) { fc[k] -= dc * f[k]; fr[k] -= dr * f[k]; }
    }
  }
  double v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (active) {
#pragma unroll
    for (int k = 0; k < CPL; ++k) {
      r[k] = refp ? f[k] - refp[k] : f[k];
      v[0] += r[k] * r[k];
      if (DERIV) {
        v[1] += fc[k] * r[k]; v[2] += fr[k] * r[k];
        v[3] += fc[k] * fc[k]; v[4] += fc[k] * fr[k]; v[5] += fr[k] * fr[k];
      }
    }
  }
  if (!DERIV) { red[0] = warp_sum(v[0]); return red[0]; }
  if (ALLRED) {
#pragma unroll
    for (int k = 0; k < 6; ++k) red[k] = warp_sum(v[k]);
    return red[0];
  }
  return warp_reduce8_transposed(v, lane);
}

// ---------------------------------------------------------------------------------------------
// K1 runs one observation per half-warp.  Lane q (0-15) of a half holds the channels lanes q and q + 16 of a
// warp-per-observation layout would hold: group A at q*CPL and group B at (q+16)*CPL.  Every fp64 sum over the
// channels is the butterfly of that layout, levels 16, 8, 4, 2, 1: a lane forms each group's partial on its own, the
// xor-16 level becomes the in-lane sum A + B, and levels 8, 4, 2, 1 stay inside the half.  The records are therefore
// bit-identical to a warp per observation, and one shuffle serves two observations.

// levels 8, 4, 2, 1 of the butterfly: every lane of the half gets the half's total
__device__ __forceinline__ double half_sum(double v) {
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Transposed reduction of 8 per-lane doubles over each half-warp (levels 8, 4, 2, 1), 8 double shuffles for both halves.
// On return lane L holds the half's total of value index ((L>>3)&1)*4 + ((L>>2)&1)*2 + ((L>>1)&1).
__device__ __forceinline__ double half_reduce8_transposed(const double v[8], int lane) {
  const bool b3 = lane & 8, b2 = lane & 4, b1 = lane & 2;
  double a[4], b[2];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const double keep = b3 ? v[4 + j] : v[j];
    const double send = b3 ? v[j] : v[4 + j];
    a[j] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
  }
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const double keep = b2 ? a[2 + j] : a[j];
    const double send = b2 ? a[j] : a[2 + j];
    b[j] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
  }
  const double keep = b1 ? b[1] : b[0];
  const double send = b1 ? b[0] : b[1];
  double c = keep + __shfl_xor_sync(0xffffffffu, send, 2);
  c += __shfl_xor_sync(0xffffffffu, c, 1);
  return c;
}

// One channel group's share of the L2 norm, the residual and the rank-2 terms, with the operation order of a lane of
// the warp-per-observation layout.
template <int CPL>
__device__ __forceinline__ double group_sq_norm(bool active, const double f[CPL]) {
  double n2 = 0.0;
  if (active) {
#pragma unroll
    for (int k = 0; k < CPL; ++k) n2 += f[k] * f[k];
  }
  return n2;
}
template <int CPL, bool DERIV>
__device__ __forceinline__ void group_scale(bool active, double ninv, double f[CPL], double fr[CPL], double fc[CPL],
                                            double& dc, double& dr) {
  dc = 0.0; dr = 0.0;
#pragma unroll
  for (int k = 0; k < CPL; ++k) {
    f[k] *= ninv;
    if (DERIV) { fc[k] *= ninv; fr[k] *= ninv; if (active) { dc += f[k] * fc[k]; dr += f[k] * fr[k]; } }
  }
}
template <int CPL>
__device__ __forceinline__ void group_project(double dc, double dr, const double f[CPL], double fr[CPL], double fc[CPL]) {
#pragma unroll
  for (int k = 0; k < CPL; ++k) { fc[k] -= dc * f[k]; fr[k] -= dr * f[k]; }
}
template <int CPL, bool DERIV>
__device__ __forceinline__ void group_terms(bool active, bool has_ref, const double refv[CPL], const double f[CPL],
                                            const double fr[CPL], const double fc[CPL], double r[CPL], double v[8]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) v[i] = 0.0;
  if (active) {
#pragma unroll
    for (int k = 0; k < CPL; ++k) {
      r[k] = has_ref ? f[k] - refv[k] : f[k];
      v[0] += r[k] * r[k];
      if (DERIV) {
        v[1] += fc[k] * r[k]; v[2] += fr[k] * r[k];
        v[3] += fc[k] * fc[k]; v[4] += fc[k] * fr[k]; v[5] += fr[k] * fr[k];
      }
    }
  }
}

// PixelInterpolator L2 normalisation + residual + rank-2 reduction of the observation of a half-warp (groups A and B).
// Returns, MODE 0: ||r||^2 in every lane; MODE 1: the transposed totals of half_reduce8_transposed
// (0:s 1:b_u 2:b_v 3:a_uu 4:a_uv 5:a_vv).
template <int CPL, bool DERIV>
__device__ __forceinline__ double normalize_and_reduce_half(bool act_a, bool act_b, bool l2, bool has_ref,
                                                            const double ref_a[CPL], const double ref_b[CPL],
                                                            double fa[CPL], double fra[CPL], double fca[CPL], double ra[CPL],
                                                            double fb[CPL], double frb[CPL], double fcb[CPL], double rb[CPL],
                                                            int lane) {
  if (l2) {
    const double n2a = group_sq_norm<CPL>(act_a, fa), n2b = group_sq_norm<CPL>(act_b, fb);
    const double ninv = 1.0 / sqrt(half_sum(n2a + n2b));
    double dca, dra, dcb, drb;
    group_scale<CPL, DERIV>(act_a, ninv, fa, fra, fca, dca, dra);
    group_scale<CPL, DERIV>(act_b, ninv, fb, frb, fcb, dcb, drb);
    if (DERIV) {
      const double dc = half_sum(dca + dcb), dr = half_sum(dra + drb);
      group_project<CPL>(dc, dr, fa, fra, fca);
      group_project<CPL>(dc, dr, fb, frb, fcb);
    }
  }
  double va[8], vb[8];
  group_terms<CPL, DERIV>(act_a, has_ref, ref_a, fa, fra, fca, ra, va);
  group_terms<CPL, DERIV>(act_b, has_ref, ref_b, fb, frb, fcb, rb, vb);
  if (!DERIV) return half_sum(va[0] + vb[0]);
#pragma unroll
  for (int i = 0; i < 8; ++i) va[i] += vb[i];
  return half_reduce8_transposed(va, lane);
}

// the CPL channels of one group to out[item * C + ch0 ..]
template <int CPL>
__device__ __forceinline__ void store_group(double* out, int64_t row, int C, int ch0, const double v[CPL]) {
#pragma unroll
  for (int k = 0; k < CPL; ++k) out[row * C + ch0 + k] = v[k];
}

// MODE 0: cost only (f), MODE 1: value + derivatives
template <typename T, int C, int MODE, bool FLOAT_SIMD>
__global__ void __launch_bounds__(FmCfg<T, C>::kWarps * 32, 1) fm_eval_kernel(FmEvalArgs a) {
  constexpr int kFmWarps = FmCfg<T, C>::kWarps;
  constexpr bool DERIV = MODE == 1;
  constexpr int CPL = C >= 32 ? C / 32 : 1;
  constexpr int ACTIVE = C / CPL;             // channel lanes of the warp-per-observation layout
  constexpr int TAP_BYTES = C * (int)sizeof(T);
  constexpr int SLOT_BYTES = 16 * TAP_BYTES;
  static_assert(TAP_BYTES % 16 == 0, "bulk copies need 16-byte multiples");
  extern __shared__ __align__(128) uint8_t smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int half = lane >> 4, q = lane & 15;
  const int hw = warp * 2 + half;             // half-warp of the CTA
  uint8_t* hbase = smem + (size_t)hw * kFmStages * SLOT_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)kFmWarps * 2 * kFmStages * SLOT_BYTES) + hw * kFmStages;
  FmAux* aux = reinterpret_cast<FmAux*>(smem + (size_t)kFmWarps * 2 * kFmStages * SLOT_BYTES + kFmWarps * 2 * kFmStages * 8) + hw * 32;
  if (q == 0) {
#pragma unroll
    for (int s = 0; s < kFmStages; ++s) mbar_init(&bars[s], 1);
    mbar_fence_init();
  }
  __syncwarp();
  const bool act_a = q < ACTIVE, act_b = q + 16 < ACTIVE;
  const int64_t item_end = a.end_dev ? a.begin + (int64_t)*a.end_dev : a.end;
  const int64_t n_items = item_end - a.begin;
  const int64_t halves_total = (int64_t)gridDim.x * kFmWarps * 2;
  // balanced batches: every half-warp walks at most R = ceil(n / (32 W2)) batches of bsz = ceil(n / (W2 R)) <= 32
  // consecutive items (W2 half-warps in the launch), so a short list spreads one item over every half-warp and a long one
  // leaves no partial last wave of 32-item batches.  The halves of a warp take consecutive batches, so half 1 never has
  // more items than half 0; past its last item a half computes nothing it stores.
  const int64_t rounds = n_items > 0 ? (n_items + 32 * halves_total - 1) / (32 * halves_total) : 0;
  const int bsz = rounds > 0 ? (int)((n_items + halves_total * rounds - 1) / (halves_total * rounds)) : 32;
  const int64_t n_batches = rounds > 0 ? (n_items + bsz - 1) / bsz : 0;
  uint32_t phase_bits = 0;
  const int64_t patch_bytes = (int64_t)a.ph * a.pw * TAP_BYTES;
  const bool has_ref = a.refs != nullptr;

  for (int64_t batch0 = ((int64_t)blockIdx.x * kFmWarps + warp) * 2; batch0 < n_batches; batch0 += halves_total) {
    const int64_t batch = batch0 + half;
    const int nvalid = batch < n_batches ? (int)min((int64_t)bsz, item_end - (a.begin + batch * bsz)) : 0;
    const int nwarp = __shfl_sync(0xffffffffu, nvalid, 0);   // half 0's count, the larger one
    // ---- phase 1: window geometry of items q and q + 16 of the half's batch, published through shared memory
    __syncwarp();
    int64_t ref_idx[2] = {0, 0};
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      const int jj = q + 16 * s;
      int64_t o = a.begin + batch * bsz + jj;
      double u = 0.0, v = 0.0;
      int64_t pidx = 0;
      if (jj < nvalid) {
        if (a.item_index) o = a.item_index[o];
        u = a.uv[2 * o]; v = a.uv[2 * o + 1];
        pidx = a.item_patch ? a.item_patch[o] : o;
        ref_idx[s] = a.item_ref ? a.item_ref[o] : o;
      }
      const double fu = floor(u), fv = floor(v);
      // guard the int conversion (NaN/huge projections clamp to the border like any far-away tap)
      FmAux x;
      x.item = o;
      x.col = (int)fmin(fmax(fu, -4.0), (double)a.pw + 4.0);
      x.row = (int)fmin(fmax(fv, -4.0), (double)a.ph + 4.0);
      x.xc = u - fu; x.xr = v - fv;
      x.src = a.patches + pidx * patch_bytes;
      aux[jj] = x;
      if (a.res_rect && jj < nvalid && !window_resident(a.res_rect[pidx], x.row, x.col, a.ph, a.pw)) {
        const unsigned long long slot = atomicAdd(a.viol_count, 1ull);
        if ((long long)slot < a.viol_capacity) a.viol_list[slot] = o;
      }
    }
    __syncwarp();

    // the 4x4 tap window of item j into slot `slot` of the half's ring (lanes of one half; the other may be idle)
    auto issue = [&](int j, int slot) {
      const int jc = aux[j].col, jr = aux[j].row;
      const uint8_t* src = aux[j].src;
      uint8_t* dst = hbase + (size_t)slot * SLOT_BYTES;
      if (q == 0) mbar_expect_tx(&bars[slot], SLOT_BYTES);
      const bool contiguous = (jc - 1 >= 0) && (jc + 2 <= a.pw - 1);
      if (contiguous) {
        if (q < 4) {
          const int rr = min(max(jr - 1 + q, 0), a.ph - 1);
          bulk_g2s(dst + q * 4 * TAP_BYTES, src + ((int64_t)rr * a.pw + (jc - 1)) * TAP_BYTES, 4 * TAP_BYTES, &bars[slot]);
        }
      } else {
        const int rr = min(max(jr - 1 + (q >> 2), 0), a.ph - 1);
        const int cc = min(max(jc - 1 + (q & 3), 0), a.pw - 1);
        bulk_g2s(dst + q * TAP_BYTES, src + ((int64_t)rr * a.pw + cc) * TAP_BYTES, TAP_BYTES, &bars[slot]);
      }
    };

    // ---- phase 2: software pipeline over the batch, both halves in step
#pragma unroll
    for (int s = 0; s < kFmStages; ++s)
      if (s < nvalid) issue(s, s);
    __syncwarp();
    for (int j = 0; j < nwarp; ++j) {
      const bool valid = j < nvalid;
      const int slot = j % kFmStages;
      const double jxc = aux[j].xc, jxr = aux[j].xr;
      const int64_t jref = __shfl_sync(0xffffffffu, (long long)(j < 16 ? ref_idx[0] : ref_idx[1]), (lane & 16) | (j & 15));
      double ref_a[CPL], ref_b[CPL];
#pragma unroll
      for (int k = 0; k < CPL; ++k) { ref_a[k] = 0.0; ref_b[k] = 0.0; }
      if (has_ref && valid) {
        const double* rp = a.refs + jref * C;
#pragma unroll
        for (int k = 0; k < CPL; ++k) ref_a[k] = __ldg(rp + (act_a ? q * CPL : 0) + k);
        if (act_b) {
#pragma unroll
          for (int k = 0; k < CPL; ++k) ref_b[k] = __ldg(rp + (q + 16) * CPL + k);
        }
      }
      double fa[CPL], fra[CPL], fca[CPL], ra[CPL], fb[CPL], frb[CPL], fcb[CPL], rb[CPL];
#pragma unroll
      for (int k = 0; k < CPL; ++k) { fa[k] = 0; fra[k] = 0; fca[k] = 0; ra[k] = 0; fb[k] = 0; frb[k] = 0; fcb[k] = 0; rb[k] = 0; }
      if (valid) {
        mbar_wait(&bars[slot], (phase_bits >> slot) & 1u);
        phase_bits ^= (1u << slot);
        const SmemWindow<TAP_BYTES> win{hbase + (size_t)slot * SLOT_BYTES};
        if (act_a) bicubic_window<T, C, CPL, DERIV, FLOAT_SIMD>(win, q, jxc, jxr, fa, fra, fca);
        if (act_b) bicubic_window<T, C, CPL, DERIV, FLOAT_SIMD>(win, q + 16, jxc, jxr, fb, frb, fcb);
      }
      __syncwarp();
      if (valid && j + kFmStages < nvalid) issue(j + kFmStages, slot);  // refill the slot just consumed
      const double tot = normalize_and_reduce_half<CPL, DERIV>(act_a, act_b, a.l2_normalize != 0, has_ref, ref_a, ref_b,
                                                               fa, fra, fca, ra, fb, frb, fcb, rb, lane);
      if (!valid) continue;
      const int64_t oj = aux[j].item;
      if (a.residuals) {
        if (act_a) store_group<CPL>(a.residuals, oj, C, q * CPL, ra);
        if (act_b) store_group<CPL>(a.residuals, oj, C, (q + 16) * CPL, rb);
      }
      if (a.desc) {
        if (act_a) store_group<CPL>(a.desc, oj, C, q * CPL, fa);
        if (act_b) store_group<CPL>(a.desc, oj, C, (q + 16) * CPL, fb);
      }
      if (DERIV && a.grad) {
        if (act_a) { store_group<CPL>(a.grad, 2 * oj, C, q * CPL, fca); store_group<CPL>(a.grad, 2 * oj + 1, C, q * CPL, fra); }
        if (act_b) { store_group<CPL>(a.grad, 2 * oj, C, (q + 16) * CPL, fcb); store_group<CPL>(a.grad, 2 * oj + 1, C, (q + 16) * CPL, frb); }
      }
      if (a.out) {
        if (DERIV) {
          // lanes q = 0, 2, .., 10 of each half hold s, b_u, b_v, a_uu, a_uv, a_vv: value index = bit3*4 + bit2*2 + bit1
          const int idx = ((q >> 3) & 1) * 4 + ((q >> 2) & 1) * 2 + ((q >> 1) & 1);
          if ((q & 1) == 0 && idx < 6) a.out[oj * 8 + idx] = tot;
        } else if (q == 0) {
          a.out[oj * 8] = tot;
        }
      }
    }
  }
}

// cost = sum_i 0.5 * rho(s_i) over items (s at out[i*8]); per-block partials, fixed order
static __global__ void __launch_bounds__(256) cost_from_sq_norm_kernel(const double* __restrict__ out, int64_t begin, int64_t end,
                                                                       LossParams loss, double* __restrict__ partials) {
  double acc = 0.0;
  for (int64_t i = begin + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < end; i += (int64_t)gridDim.x * blockDim.x) {
    double rho[3];
    loss_eval(loss, 1.0, out[i * 8], rho);
    acc += 0.5 * rho[0];
  }
  __shared__ double sh[8];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) { double t = 0; for (int k = 0; k < 8; ++k) t += sh[k]; partials[blockIdx.x] = t; }
}

}  // namespace pxr
