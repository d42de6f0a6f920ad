// pxr_ba_kernels.cuh — "geometric BA with a 2x2 weight per observation".
//
// After K1 has collapsed every residual block to (||r||^2, G^T r, G^T G), the normal equations of
// the featuremetric BA are  J^T J = P^T (rho' G^T G) P,  J^T r = P^T (rho' G^T r)  with
// P = d(uv)/d(theta) from K0.  These kernels replace what Ceres does inside ceres::Solve for
// the reference (bundle_optimizer.h:224): block assembly, per-point Schur elimination
// (SchurEliminator), the reduced camera system solve (DENSE_SCHUR / SPARSE_SCHUR are exact
// factorizations -> dense Cholesky here), back-substitution, and the manifold Plus
// (QuaternionManifold, SubsetManifold — bundle_optimizer.h:384-389,436-438).
#pragma once
#include "pxr_device.cuh"
#include "pxr_lm.cuh"

namespace pxr {

constexpr int kMaxDc = 6 + kMaxK;

struct BADev {
  // per-image column tables (present when every image has <= 8 camera columns): local column of block row a, and
  // which entry of the per-observation Jacobian row feeds it; lets the kernels keep cols/Ju/Jv in registers
  const int32_t* img_cols8; const int8_t* img_src8; const int32_t* img_dc8;
  // sizes
  int n_cameras, n_images, K;  // K = max #intrinsics in the problem (juv columns)
  int64_t n_points, n_obs;
  int nc, nl;                  // reduced camera system size, total tangent size
  int dcmax;                   // 6 + K
  int juv_stride;
  // topology / masks
  const int32_t* obs_img; const int64_t* obs_pt; const int32_t* img_cam; const int32_t* cam_model;
  const uint32_t* cam_mask; const uint8_t* tmask;
  const int32_t* pose_off; const int32_t* intr_off; const int64_t* point_off; const int64_t* pt_begin;
  // per-observation data
  const double* obs_out; const double* juv;
  // linearisation
  double* Hcc; double* gc; double* Hpp; double* gp; double* W; int32_t* Wcols; int32_t* Wdc;
  LossParams loss;
};

__device__ __forceinline__ void atomic_add_f64(double* p, double v) { atomicAdd(p, v); }

// local camera-side columns of one observation: pose (3 rot + non-constant t) then intrinsics
__device__ __forceinline__ int obs_local_columns(const BADev& d, int64_t o, const double* J, int Wd, int* cols, double* Ju, double* Jv) {
  const int img = d.obs_img[o];
  const int cam = d.img_cam[img];
  int dc = 0;
  const int po = d.pose_off[img];
  if (po >= 0) {
    const uint32_t tm = d.tmask[img];
    for (int k = 0; k < 3; ++k) { cols[dc] = po + k; Ju[dc] = J[k]; Jv[dc] = J[Wd + k]; ++dc; }
    int la = 3;
    for (int k = 0; k < 3; ++k) {
      if (tm & (1u << k)) continue;
      cols[dc] = po + la++; Ju[dc] = J[3 + k]; Jv[dc] = J[Wd + 3 + k]; ++dc;
    }
  }
  const int io = d.intr_off[cam];
  if (io >= 0) {
    const uint32_t cm = d.cam_mask[cam];
    const int Kc = cam_num_params(d.cam_model[cam]);
    int la = 0;
    for (int k = 0; k < Kc; ++k) {
      if (cm & (1u << k)) continue;
      cols[dc] = io + la++; Ju[dc] = J[9 + k]; Jv[dc] = J[Wd + 9 + k]; ++dc;
    }
  }
  return dc;
}

// register-only variant of obs_local_columns for images with <= 8 camera columns (static indexing throughout)
__device__ __forceinline__ int obs_local_columns8(const BADev& d, int64_t o, const double* J, int Wd, int cols[8], double Ju[8], double Jv[8]) {
  const int img = d.obs_img[o];
  const int32_t* ic = d.img_cols8 + img * 8;
  const int8_t* is = d.img_src8 + img * 8;
#pragma unroll
  for (int a = 0; a < 8; ++a) {
    const int sidx = is[a];
    cols[a] = ic[a];
    Ju[a] = sidx >= 0 ? J[sidx] : 0.0;
    Jv[a] = sidx >= 0 ? J[Wd + sidx] : 0.0;
  }
  return d.img_dc8[img];
}

// K2: one thread per observation.  W_o = J_c^T A' J_p, camera blocks J_c^T A' J_c / J_c^T b' into
// the dense Hcc (lower triangle) / gc and the point blocks Hpp / gp, all with fp64 atomics
// (Hpp/gp/Hcc/gc are zeroed by the caller).
template <bool FAST>
static __global__ void __launch_bounds__(128) ba_build_kernel(BADev d, int cam_blocks) {
  const int64_t o = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= d.n_obs) return;
  const int64_t p = d.obs_pt[o];
  const bool pvar = d.point_off[p] >= 0;
  const int Wd = 9 + d.K;
  const double* oo = d.obs_out + o * 8;
  double rho[3];
  loss_eval(d.loss, 1.0, oo[0], rho);
  const double bu = rho[1] * oo[1], bv = rho[1] * oo[2];
  const double auu = rho[1] * oo[3], auv = rho[1] * oo[4], avv = rho[1] * oo[5];
  const double* J = d.juv + o * (int64_t)d.juv_stride;  // rows: J[0..Wd), J[Wd..2Wd)
  constexpr int NA = FAST ? 8 : kMaxDc;
  int cols[NA];
  double Ju[NA], Jv[NA];
  int dc;
  if constexpr (FAST) dc = obs_local_columns8(d, o, J, Wd, cols, Ju, Jv);
  else dc = obs_local_columns(d, o, J, Wd, cols, Ju, Jv);
  d.Wdc[o] = dc;
  const double pu[3] = {J[6], J[7], J[8]}, pv[3] = {J[Wd + 6], J[Wd + 7], J[Wd + 8]};
  double apu[3], apv[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) { apu[k] = auu * pu[k] + auv * pv[k]; apv[k] = auv * pu[k] + avv * pv[k]; }
  if (pvar) {
    double* Hp = d.Hpp + p * 9;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      atomic_add_f64(&d.gp[p * 3 + a], pu[a] * bu + pv[a] * bv);
#pragma unroll
      for (int b = 0; b < 3; ++b) atomic_add_f64(&Hp[a * 3 + b], pu[a] * apu[b] + pv[a] * apv[b]);
    }
  }
  double* Wo = d.W + o * (int64_t)d.dcmax * 3;
  int32_t* Wc = d.Wcols + o * (int64_t)d.dcmax;
#pragma unroll
  for (int a = 0; a < NA; ++a) {
    if (a >= dc) break;
    Wc[a] = cols[a];
    if (pvar) {
      Wo[a * 3 + 0] = Ju[a] * apu[0] + Jv[a] * apv[0];
      Wo[a * 3 + 1] = Ju[a] * apu[1] + Jv[a] * apv[1];
      Wo[a * 3 + 2] = Ju[a] * apu[2] + Jv[a] * apv[2];
    }
    if (!cam_blocks) continue;   // the per-image chunk kernel below accumulates Hcc / gc
    const double aju = auu * Ju[a] + auv * Jv[a], ajv = auv * Ju[a] + avv * Jv[a];
    atomic_add_f64(&d.gc[cols[a]], Ju[a] * bu + Jv[a] * bv);
    for (int b = 0; b <= a; ++b)  // cols ascending within an observation -> lower triangle
      atomic_add_f64(&d.Hcc[(int64_t)cols[a] * d.nc + cols[b]], Ju[b] * aju + Jv[b] * ajv);
  }
}

// K2s: ba_build_kernel<true> without the camera part, with the per-observation records moved through shared memory.
// The unstaged K2 is latency-bound (low issue activity, stalls on long_scoreboard + lg_throttle): every
// thread walks its own 176 B `juv` record and 192 B `W` row (32 different lines per warp instruction) and ten
// neighbouring threads hit the same Hpp/gp words with atomics.  Here a CTA of 128 observations
//   * copies the `juv` / `obs_out` records of its observations with coalesced 8 B-per-lane loads into shared memory
//     (rows padded to an odd number of doubles: conflict-free per-thread access),
//   * reduces Hpp / gp over the observations of a point with a segmented warp scan (observations are sorted by
//     point): one atomic per element per (point, warp) instead of one per observation,
//   * stages the W rows in the same shared memory and writes them back coalesced (entries beyond an observation's
//     column count, which nothing reads, are written as zeros).
// Dynamic shared memory: 128 * (max(juv_stride, 3*dcmax) | 1  +  9) doubles.
static __global__ void __launch_bounds__(128) ba_build_staged_kernel(BADev d) {
  extern __shared__ double sm_build[];
  const int tid = threadIdx.x, lane = tid & 31;
  const int64_t o0 = (int64_t)blockIdx.x * 128;
  const int n = (int)min((int64_t)128, d.n_obs - o0);
  const int js = d.juv_stride, wrow = d.dcmax * 3;
  const int SP = max(js, wrow) | 1;                  // padded row (doubles), shared by the J and the W staging
  double* sJ = sm_build;                             // [128][SP]
  double* sO = sm_build + (size_t)128 * SP;          // [128][9]
  {
    const double* src = d.juv + o0 * (int64_t)js;
    int r = tid / js, c = tid - r * js;
    const int dr = 128 / js, dcol = 128 - dr * js;
    for (int i = tid; i < n * js; i += 128) {
      sJ[r * SP + c] = __ldg(src + i);
      r += dr; c += dcol;
      if (c >= js) { c -= js; ++r; }
    }
    const double* so = d.obs_out + o0 * 8;
    for (int i = tid; i < n * 8; i += 128) sO[(i >> 3) * 9 + (i & 7)] = __ldg(so + i);
  }
  __syncthreads();
  const bool live = tid < n;
  const int64_t o = o0 + tid;
  const int64_t p = live ? d.obs_pt[o] : -1;
  const bool pvar = live && d.point_off[p] >= 0;
  const int Wd = 9 + d.K;
  int cols[8];
  double Ju[8], Jv[8];
  int dc = 0;
  double v[12];                                      // gp (3) | Hpp (9)
#pragma unroll
  for (int k = 0; k < 12; ++k) v[k] = 0.0;
  double apu[3] = {0, 0, 0}, apv[3] = {0, 0, 0};
  if (live) {
    const double* oo = sO + tid * 9;
    double rho[3];
    loss_eval(d.loss, 1.0, oo[0], rho);
    const double bu = rho[1] * oo[1], bv = rho[1] * oo[2];
    const double auu = rho[1] * oo[3], auv = rho[1] * oo[4], avv = rho[1] * oo[5];
    const double* J = sJ + tid * SP;
    dc = obs_local_columns8(d, o, J, Wd, cols, Ju, Jv);
    const double pu[3] = {J[6], J[7], J[8]}, pv[3] = {J[Wd + 6], J[Wd + 7], J[Wd + 8]};
#pragma unroll
    for (int k = 0; k < 3; ++k) { apu[k] = auu * pu[k] + auv * pv[k]; apv[k] = auv * pu[k] + avv * pv[k]; }
    if (pvar) {
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        v[a] = pu[a] * bu + pv[a] * bv;
#pragma unroll
        for (int b = 0; b < 3; ++b) v[3 + a * 3 + b] = pu[a] * apu[b] + pv[a] * apv[b];
      }
    }
    d.Wdc[o] = dc;
    int32_t* Wc = d.Wcols + o * (int64_t)d.dcmax;
#pragma unroll
    for (int a = 0; a < 8; ++a) if (a < dc) Wc[a] = cols[a];
  }
  // segmented inclusive scan over the lanes of one point (contiguous), then the last lane of a segment adds once
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const int64_t pq = __shfl_up_sync(0xffffffffu, p, off);
    const bool take = lane >= off && pq == p;
#pragma unroll
    for (int k = 0; k < 12; ++k) {
      const double w = __shfl_up_sync(0xffffffffu, v[k], off);
      if (take) v[k] += w;
    }
  }
  const int64_t pnext = __shfl_down_sync(0xffffffffu, p, 1);
  if (pvar && (lane == 31 || pnext != p)) {
#pragma unroll
    for (int a = 0; a < 3; ++a) atomic_add_f64(&d.gp[p * 3 + a], v[a]);
#pragma unroll
    for (int k = 0; k < 9; ++k) atomic_add_f64(&d.Hpp[p * 9 + k], v[3 + k]);
  }
  __syncthreads();                                   // every thread has its J values in registers: reuse sJ for W
  if (live) {
    double* Ws = sJ + tid * SP;
#pragma unroll
    for (int a = 0; a < 8; ++a) {
      if (a * 3 + 2 < wrow) {
        const bool on = pvar && a < dc;
        Ws[a * 3 + 0] = on ? Ju[a] * apu[0] + Jv[a] * apv[0] : 0.0;
        Ws[a * 3 + 1] = on ? Ju[a] * apu[1] + Jv[a] * apv[1] : 0.0;
        Ws[a * 3 + 2] = on ? Ju[a] * apu[2] + Jv[a] * apv[2] : 0.0;
      }
    }
    for (int k = 24; k < wrow; ++k) Ws[k] = 0.0;     // dcmax > 8 cannot reach this kernel with dc > 8; keep rows defined
  }
  __syncthreads();
  {
    double* dst = d.W + o0 * (int64_t)wrow;
    int r = tid / wrow, c = tid - r * wrow;
    const int dr = 128 / wrow, dcol = 128 - dr * wrow;
    for (int i = tid; i < n * wrow; i += 128) {
      dst[i] = sJ[r * SP + c];
      r += dr; c += dcol;
      if (c >= wrow) { c -= wrow; ++r; }
    }
  }
}

// K2c: camera blocks without per-observation atomics.  Observations are listed per image in chunks of
// <= 128 (all observations of an image share their parameter columns); one warp per chunk accumulates
// J_c^T A' J_c (lower triangle, 36 values for dc <= 8) and J_c^T b' (8) in registers, reduces them across
// the warp with the transposed butterfly (9 double shuffles per 8 values) and issues ONE atomic per
// element per chunk: 128x fewer L2 atomics than ba_build_kernel's camera part.  Used when dcmax <= 8.
static __global__ void __launch_bounds__(256) ba_build_cam_kernel(BADev d, const int32_t* __restrict__ io_obs,
                                                                  const int64_t* __restrict__ chunk_begin, int64_t n_chunks,
                                                                  double* __restrict__ Himg /* [n_images][64] or null: dense Hcc */,
                                                                  double* __restrict__ part = nullptr /* deterministic mode: [n_chunks][48] partial sums, no atomics */) {
  const int lane = threadIdx.x & 31;
  const int64_t chunk = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (chunk >= n_chunks) return;
  const int64_t beg = chunk_begin[chunk], end = chunk_begin[chunk + 1];
  const int Wd = 9 + d.K;
  double acc[48];
#pragma unroll
  for (int k = 0; k < 48; ++k) acc[k] = 0.0;
  int cols[8];
  int dc = 0;
  for (int64_t e = beg + lane; e < end; e += 32) {
    const int64_t o = io_obs[e];
    const double* oo = d.obs_out + o * 8;
    double rho[3];
    loss_eval(d.loss, 1.0, oo[0], rho);
    const double bu = rho[1] * oo[1], bv = rho[1] * oo[2];
    const double auu = rho[1] * oo[3], auv = rho[1] * oo[4], avv = rho[1] * oo[5];
    const double* J = d.juv + o * (int64_t)d.juv_stride;
    double Ju[8], Jv[8];
    dc = obs_local_columns8(d, o, J, Wd, cols, Ju, Jv);
#pragma unroll
    for (int a = 0; a < 8; ++a) {
      if (a < dc) {
        const double aju = auu * Ju[a] + auv * Jv[a], ajv = auv * Ju[a] + avv * Jv[a];
        acc[36 + a] += Ju[a] * bu + Jv[a] * bv;
#pragma unroll
        for (int b = 0; b <= a; ++b)
          if (b < dc) acc[a * (a + 1) / 2 + b] += Ju[b] * aju + Jv[b] * ajv;
      }
    }
  }
  // the chunk's columns: every observation of the image has the same ones; lane 0 always has an observation
  dc = __shfl_sync(0xffffffffu, dc, 0);
#pragma unroll
  for (int a = 0; a < 8; ++a) cols[a] = __shfl_sync(0xffffffffu, cols[a], 0);
  const int idx = ((lane >> 4) & 1) * 4 + ((lane >> 3) & 1) * 2 + ((lane >> 2) & 1);
#pragma unroll
  for (int gsel = 0; gsel < 6; ++gsel) {
    const double tot = warp_reduce8_transposed(acc + gsel * 8, lane);
    if ((lane & 3) != 0) continue;
    const int vi = gsel * 8 + idx;
    if (part) { part[chunk * 48 + vi] = tot; continue; }       // reduced per image in chunk order by det_cam_reduce_kernel
    if (vi < 36) {
      int a = 0;
      while ((a + 1) * (a + 2) / 2 <= vi) ++a;
      const int b = vi - a * (a + 1) / 2;
      if (a < dc) {
        if (Himg) atomic_add_f64(&Himg[(int64_t)d.obs_img[io_obs[beg]] * 64 + a * 8 + b], tot);
        else atomic_add_f64(&d.Hcc[(int64_t)cols[a] * d.nc + cols[b]], tot);
      }
    } else if (vi < 44) {
      const int a = vi - 36;
      if (a < dc) atomic_add_f64(&d.gc[cols[a]], tot);
    }
  }
}

// diag(J^T J) in local order: cameras from Hcc's diagonal, points from Hpp
static __global__ void ba_diag_kernel(BADev d, double* diag) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < d.nc && d.Hcc) diag[i] = d.Hcc[i * d.nc + i];     // sparse mode (Hcc == null): sp_diag_kernel fills the camera part
  const int64_t p = i;
  if (p < d.n_points) {
    const int64_t po = d.point_off[p];
    if (po >= 0) { diag[po] = d.Hpp[p * 9]; diag[po + 1] = d.Hpp[p * 9 + 4]; diag[po + 2] = d.Hpp[p * 9 + 8]; }
  }
}

// jacobi scaling (iteration 0)
static __global__ void ba_scale_kernel(const double* diag, double* scale, int64_t n, int enabled) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) scale[i] = enabled ? jacobi_scale(diag[i]) : 1.0;
}
// LM diagonal in unscaled variables
static __global__ void ba_d2_kernel(const double* diag, const double* scale, double* D2, int64_t n, double radius,
                             double lo, double hi) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  D2[i] = lm_damping(diag[i], scale[i], radius, lo, hi);
}

// S = Hcc + diag(D2c) (lower), rhs = -gc
// (multi-GPU: Hcc / gc are this rank's partial sums and only rank 0 adds the damping, add_d2)
static __global__ void ba_init_reduced_kernel(const double* Hcc, const double* gc, const double* D2, double* S,
                                       double* rhs, int nc, int add_d2) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t n2 = (int64_t)nc * nc;
  if (i < n2) {
    const int r = (int)(i / nc), c = (int)(i % nc);
    double v = c <= r ? Hcc[i] : 0.0;
    if (r == c && add_d2) v += D2[r];
    S[i] = v;
  }
  if (i < nc) rhs[i] = -gc[i];
}

// K3: per-point Schur elimination without per-entry atomics.
//   S[cols_i, cols_j] -= W_i (Hpp + D)^-1 W_j^T ,   rhs[cols_i] += W_i (Hpp + D)^-1 gp
// K3a (one thread per point): T_i = W_i (Hpp+D)^-1 for every observation of the point, rhs terms.
// K3b (one warp per co-visibility chunk): all observation pairs (i,j) of all points that fall on
//      the same (image_i, image_j) pair address the same block of S; the pair list is sorted by that
//      key once on the host (static sparsity), a warp accumulates the dc_i x dc_j block of a chunk in
//      registers and touches S once per element.
// K3a': (Hpp + D)^-1 once per point (6 unique entries), instead of once per (observation, row)
static __global__ void __launch_bounds__(256) ba_point_inverse_kernel(BADev d, const double* D2, double* Hinv, int* fail_flag) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= d.n_points) return;
  const int64_t po = d.point_off[p];
  if (po < 0) return;
  double inv[9];
  if (!inv3_sym(d.Hpp + p * 9, D2 + po, inv)) { *fail_flag = 1; inv[0] = inv[1] = inv[2] = inv[4] = inv[5] = inv[8] = 0.0; }
  double* h = Hinv + p * 6;
  h[0] = inv[0]; h[1] = inv[1]; h[2] = inv[2]; h[3] = inv[4]; h[4] = inv[5]; h[5] = inv[8];
}

// K3a: T = W (Hpp + D)^-1, one thread per (observation, local camera row).  The right-hand side part
// sum_obs T gp is accumulated by the pair kernel on its self pairs (per image chunk, 8 atomics per 128 observations).
static __global__ void __launch_bounds__(256) ba_schur_prep_kernel(BADev d, const double* __restrict__ Hinv, double* T) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int dcm = d.dcmax;
  const int64_t o = idx / dcm;
  const int a = (int)(idx - o * dcm);
  if (o >= d.n_obs) return;
  const int64_t p = d.obs_pt[o];
  if (d.point_off[p] < 0) return;
  if (a >= d.Wdc[o]) {
    // record row 8 is free when the image has at most 8 columns: it carries the point's gradient, so that the staged
    // pair kernel finds everything a self pair needs in ONE record (dcm = 6 + K >= 9 for every camera model)
    if (a == 8) { double* tp = T + (o * dcm + 8) * 3; const double* g = d.gp + p * 3; tp[0] = g[0]; tp[1] = g[1]; tp[2] = g[2]; }
    return;
  }
  const double* h = Hinv + p * 6;
  const double* w = d.W + (o * dcm + a) * 3;
  double* tp = T + (o * dcm + a) * 3;
  tp[0] = w[0] * h[0] + w[1] * h[1] + w[2] * h[2];
  tp[1] = w[0] * h[1] + w[1] * h[3] + w[2] * h[4];
  tp[2] = w[0] * h[2] + w[1] * h[4] + w[2] * h[5];
}

struct SchurPairs {
  const int32_t* px; const int32_t* py;   // observation pair entries, sorted by chunk
  const int32_t* pp;                      // the pairs' 3D point (fused tensor-core walk: H_pp^-1 and g_p without a detour over obs_pt)
  const int64_t* chunk_begin;             // [n_chunks + 1]
  const uint8_t* chunk_self;              // [n_chunks] 1: entries are (o,o) self pairs
  int64_t n_chunks;
};

// Fast path of the pair kernels (dc <= 8): the 4 groups of 8 lanes of a warp each walk every 4th pair of the chunk;
// lane (g, a) owns row a of the 8x8 block.  On self chunks the same pass accumulates rhs += T gp.
// (A variant that staged 16 pairs at a time through shared memory to widen the gathers needed 126 registers, left
//  16 resident warps, measured slower, and was dropped.)
constexpr int kPairThreads = 256;
__device__ __forceinline__ void schur_pairs_accumulate(const BADev& d, const SchurPairs& sp, const double* __restrict__ T,
                                                       int64_t kb, int64_t ke, int lane, int dcx, int dcy, bool self,
                                                       double acc[8], double& racc) {
  const int dcm = d.dcmax;
  const int g = lane >> 3, a = lane & 7;
#pragma unroll
  for (int b = 0; b < 8; ++b) acc[b] = 0.0;
  racc = 0.0;
  for (int64_t k = kb + g; k < ke; k += 4) {
    const int64_t ox = sp.px[k];
    const double* Tx = T + (ox * dcm + a) * 3;
    const double* Wy = d.W + (int64_t)sp.py[k] * dcm * 3;
    if (a < dcx) {
      const double t0 = Tx[0], t1 = Tx[1], t2 = Tx[2];
#pragma unroll
      for (int b = 0; b < 8; ++b)
        if (b < dcy) acc[b] += t0 * Wy[b * 3] + t1 * Wy[b * 3 + 1] + t2 * Wy[b * 3 + 2];
      if (self) { const double* gpv = d.gp + d.obs_pt[ox] * 3; racc += t0 * gpv[0] + t1 * gpv[1] + t2 * gpv[2]; }
    }
  }
#pragma unroll
  for (int b = 0; b < 8; ++b) {
    acc[b] += __shfl_xor_sync(0xffffffffu, acc[b], 8);
    acc[b] += __shfl_xor_sync(0xffffffffu, acc[b], 16);
  }
  racc += __shfl_xor_sync(0xffffffffu, racc, 8);
  racc += __shfl_xor_sync(0xffffffffu, racc, 16);
}

template <bool FAST>
static __global__ void __launch_bounds__(kPairThreads, FAST ? 5 : 2) ba_schur_pairs_kernel(BADev d, SchurPairs sp, const double* __restrict__ T,
                                                                    double* S, double* rhs) {
  const int64_t c = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (c >= sp.n_chunks) return;
  const int64_t kb = sp.chunk_begin[c], ke = sp.chunk_begin[c + 1];
  if (ke <= kb) return;
  const int dcm = d.dcmax;
  const int64_t ox0 = sp.px[kb], oy0 = sp.py[kb];
  const int dcx = d.Wdc[ox0], dcy = d.Wdc[oy0];
  const bool self = sp.chunk_self[c] != 0;
  if (FAST || (dcx <= 8 && dcy <= 8)) {
    // fast path: 4 groups of 8 lanes work on 4 entries at a time; lane (g, a) owns row a of the block
    const int g = lane >> 3, a = lane & 7;
    double acc[8], racc;
    schur_pairs_accumulate(d, sp, T, kb, ke, lane, dcx, dcy, self, acc, racc);
    if (self && g == 0 && a < dcx) atomic_add_f64(&rhs[d.Wcols[ox0 * dcm + a]], racc);
    if (g == 0 && a < dcx) {
      const int ca = d.Wcols[ox0 * dcm + a];
#pragma unroll
      for (int b = 0; b < 8; ++b) {
        if (b >= dcy) continue;
        const int cb = d.Wcols[oy0 * dcm + b];
        const double v = -acc[b];
        if (self) { if (a >= b) atomic_add_f64(&S[(int64_t)ca * d.nc + cb], v); }
        else if (ca > cb) atomic_add_f64(&S[(int64_t)ca * d.nc + cb], v);
        else if (ca < cb) atomic_add_f64(&S[(int64_t)cb * d.nc + ca], v);
        else atomic_add_f64(&S[(int64_t)ca * d.nc + ca], 2.0 * v);
      }
    }
    return;
  }
  if constexpr (!FAST) {
  if (self) {   // rhs += sum_obs T gp (generic path: lanes over rows)
    for (int r = lane; r < dcx; r += 32) {
      double rs = 0.0;
      for (int64_t k = kb; k < ke; ++k) {
        const int64_t o = sp.px[k];
        const double* Tx = T + ((int64_t)o * dcm + r) * 3;
        const double* gpv = d.gp + d.obs_pt[o] * 3;
        rs += Tx[0] * gpv[0] + Tx[1] * gpv[1] + Tx[2] * gpv[2];
      }
      atomic_add_f64(&rhs[d.Wcols[ox0 * dcm + r]], rs);
    }
  }
  const int nel = dcx * dcy;
  constexpr int kMaxT = (kMaxDc * kMaxDc + 31) / 32;
  double acc[kMaxT];
#pragma unroll
  for (int t = 0; t < kMaxT; ++t) acc[t] = 0.0;
  for (int64_t k = kb; k < ke; ++k) {
    const double* Tx = T + (int64_t)sp.px[k] * dcm * 3;
    const double* Wy = d.W + (int64_t)sp.py[k] * dcm * 3;
#pragma unroll
    for (int t = 0; t < kMaxT; ++t) {
      const int e = lane + 32 * t;
      if (e < nel) {
        const int a = e / dcy, b = e - a * dcy;
        acc[t] += Tx[a * 3] * Wy[b * 3] + Tx[a * 3 + 1] * Wy[b * 3 + 1] + Tx[a * 3 + 2] * Wy[b * 3 + 2];
      }
    }
  }
#pragma unroll
  for (int t = 0; t < kMaxT; ++t) {
    const int e = lane + 32 * t;
    if (e >= nel) continue;
    const int a = e / dcy, b = e - a * dcy;
    const int ca = d.Wcols[ox0 * dcm + a], cb = d.Wcols[oy0 * dcm + b];
    const double v = -acc[t];
    if (self) { if (a >= b) atomic_add_f64(&S[(int64_t)ca * d.nc + cb], v); }
    else if (ca > cb) atomic_add_f64(&S[(int64_t)ca * d.nc + cb], v);
    else if (ca < cb) atomic_add_f64(&S[(int64_t)cb * d.nc + ca], v);
    else atomic_add_f64(&S[(int64_t)ca * d.nc + ca], 2.0 * v);
  }
  }
}

// Staged pair kernel (dc <= 8, the default): the same chunk-per-warp walk as above, 4 pairs per round, but the two
// 192 B records of a pair (T of x, W of y) are fetched ONCE per round by the 8 lanes of the pair's group — 48 contiguous
// bytes per lane — one round AHEAD of their use, staged through a per-warp double buffer in shared memory and read back
// as a row (T, 3 x LDS.64) and a broadcast block (W, 12 x LDS.128).  Against the direct kernel: 4 instead of 27 global
// load instructions per lane and round, every gather a full 32 B sector run, the gather latency of round r+1 hidden
// behind the FMAs of round r, and the pair indices prefetched two rounds ahead.  On self chunks lane 0 of a group also
// brings row 8 of the T record (the point's gradient, written by ba_schur_prep_kernel) for rhs += T gp.
constexpr int kStageStride = 56;                      // doubles per staged pair: T rows at 0..23, gp at 24..26, W at 28..51;
                                                      // 448 B = 16 banks mod 32, so two groups' row reads never collide
constexpr int kStageDoubles = (kPairThreads / 32) * 2 * 4 * kStageStride;   // per CTA: 8 warps x 2 buffers x 4 pairs
// The walk over one chunk; `stage_all` is the CTA's staging area (kStageDoubles, 16-byte aligned).  Leaves the chunk's
// 8x8 block in acc (row a on the lanes of EVERY group after the final butterfly) and the rhs row in racc.
template <bool VEC>
__device__ __forceinline__ void schur_pairs_accumulate_staged(const BADev& d, const SchurPairs& sp, const double* __restrict__ T,
                                                              int64_t kb, int64_t ke, int lane, bool self, double* stage_all,
                                                              double acc[8], double& racc) {
  const int dcm = d.dcmax;
  const int g = lane >> 3, a = lane & 7;
  // this lane's share of a pair's fetch: lanes 0..3 of a group the T record of x, lanes 4..7 the W record of y
  const int32_t* __restrict__ my_idx = (a < 4 ? sp.px : sp.py) + kb;
  const double* __restrict__ my_src = (a < 4 ? T : d.W) + (a & 3) * 6;
  const bool take_gp = self && a == 0;
  const int n = (int)(ke - kb), last = n - 1;
  const int rounds = (n + 3) >> 2;
  double* const st0 = stage_all + (threadIdx.x >> 5) * (2 * 4 * kStageStride) + g * kStageStride;   // this group's pair, buffer 0
  double* const st1 = st0 + 4 * kStageStride;
  const int my_slot = (a < 4 ? 0 : 28) + (a & 3) * 6; // where this lane's 6 doubles go inside the staged pair

  double2 r0, r1, r2;                                 // the 48 bytes in flight
  double g0 = 0.0, g1 = 0.0, g2 = 0.0;                // row 8 (self chunks, lane 0 of the group)
  const uint32_t rec = (uint32_t)dcm * 3u;
  auto fetch = [&](int32_t o) {
    const double* src = my_src + (uint64_t)(uint32_t)o * rec;
    if (VEC) {
      const double2* s2 = reinterpret_cast<const double2*>(src);
      r0 = __ldg(s2); r1 = __ldg(s2 + 1); r2 = __ldg(s2 + 2);
    } else {
      r0 = make_double2(__ldg(src), __ldg(src + 1)); r1 = make_double2(__ldg(src + 2), __ldg(src + 3)); r2 = make_double2(__ldg(src + 4), __ldg(src + 5));
    }
    if (take_gp) { g0 = __ldg(src + 24); g1 = __ldg(src + 25); g2 = __ldg(src + 26); }   // a == 0: src is the T record's start
  };
  racc = 0.0;
#pragma unroll
  for (int b = 0; b < 8; ++b) acc[b] = 0.0;
  // Rows of T beyond the image's column count and columns beyond dcy hold whatever the buffers hold: they are multiplied
  // along (no predicates in the loop) and never written out.  Entries past the chunk's end re-read its last pair and
  // are skipped by the `live` test.
  int32_t o_next;
  auto round = [&](double* st, int r) {
    double2* dst = reinterpret_cast<double2*>(st + my_slot);
    dst[0] = r0; dst[1] = r1; dst[2] = r2;
    if (take_gp) { st[24] = g0; st[25] = g1; st[26] = g2; }
    __syncwarp();
    if (r + 1 < rounds) {                             // next round's gathers leave before this round's arithmetic
      fetch(o_next);
      o_next = __ldg(my_idx + min(4 * (r + 2) + g, last));
    }
    if (4 * r + g <= last) {                          // live: this group's pair of the round exists
      const double t0 = st[a * 3], t1 = st[a * 3 + 1], t2 = st[a * 3 + 2];
      const double2* w2 = reinterpret_cast<const double2*>(st + 28);
#pragma unroll
      for (int q = 0; q < 4; ++q) {                   // rows 2q, 2q+1 of W: 6 doubles = 3 double2
        const double2 u0 = w2[q * 3], u1 = w2[q * 3 + 1], u2 = w2[q * 3 + 2];
        acc[2 * q] = fma(t0, u0.x, fma(t1, u0.y, fma(t2, u1.x, acc[2 * q])));
        acc[2 * q + 1] = fma(t0, u1.y, fma(t1, u2.x, fma(t2, u2.y, acc[2 * q + 1])));
      }
      if (self) racc = fma(t0, st[24], fma(t1, st[25], fma(t2, st[26], racc)));
    }
  };
  // pipeline prologue: data of round 0, index of round 1
  fetch(__ldg(my_idx + min(g, last)));
  o_next = __ldg(my_idx + min(4 + g, last));
  // two buffers, one barrier per round: round r+1 stages into the other buffer, and every lane has left round r-1's
  // reads of it before it passed round r's __syncwarp
  for (int r = 0; r < rounds; r += 2) {
    round(st0, r);
    if (r + 1 < rounds) round(st1, r + 1);
  }
#pragma unroll
  for (int b = 0; b < 8; ++b) {
    acc[b] += __shfl_xor_sync(0xffffffffu, acc[b], 8);
    acc[b] += __shfl_xor_sync(0xffffffffu, acc[b], 16);
  }
  racc += __shfl_xor_sync(0xffffffffu, racc, 8);
  racc += __shfl_xor_sync(0xffffffffu, racc, 16);
}

template <bool VEC, int CTAS>
static __global__ void __launch_bounds__(kPairThreads, CTAS) ba_schur_pairs_staged_kernel(BADev d, SchurPairs sp, const double* __restrict__ T,
                                                                                          double* S, double* rhs) {
  __shared__ __align__(16) double stage_all[kStageDoubles];
  const int64_t c = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (c >= sp.n_chunks) return;
  const int64_t kb = sp.chunk_begin[c], ke = sp.chunk_begin[c + 1];
  if (ke <= kb) return;
  const int dcm = d.dcmax;
  const bool self = sp.chunk_self[c] != 0;
  const int g = lane >> 3, a = lane & 7;
  double acc[8], racc;
  schur_pairs_accumulate_staged<VEC>(d, sp, T, kb, ke, lane, self, stage_all, acc, racc);
  const int64_t ox0 = sp.px[kb], oy0 = sp.py[kb];
  const int dcx = d.Wdc[ox0], dcy = d.Wdc[oy0];
  if (g != 0 || a >= dcx) return;
  const int ca = d.Wcols[ox0 * dcm + a];
  if (self) atomic_add_f64(&rhs[ca], racc);
#pragma unroll
  for (int b = 0; b < 8; ++b) {
    if (b >= dcy) continue;
    const int cb = d.Wcols[oy0 * dcm + b];
    const double v = -acc[b];
    if (self) { if (a >= b) atomic_add_f64(&S[(int64_t)ca * d.nc + cb], v); }
    else if (ca > cb) atomic_add_f64(&S[(int64_t)ca * d.nc + cb], v);
    else if (ca < cb) atomic_add_f64(&S[(int64_t)cb * d.nc + ca], v);
    else atomic_add_f64(&S[(int64_t)ca * d.nc + ca], 2.0 * v);
  }
}

// Tensor-core pair walk (the default when every image has at most 8 columns).  One observation pair contributes the
// 8x8 block T_x W_y^T = (8x3)(3x8): exactly ONE fp64 tensor-core instruction, mma.sync m8n8k4 with k padded from 3 to 4.
// Its fragment layout wants from lane L = 4*gid + tig the elements A[gid][tig] = T_x[gid][tig] and
// B[tig][gid] = W_y[gid][tig] — the SAME offset 3*gid + tig into both records, and over the 24 lanes with tig < 3 those
// offsets are the 24 consecutive doubles of the record: one fully coalesced 192-byte gather per record, no staging, no
// shuffles, no per-lane copies of W.  A warp walks its chunk 8 pairs at a time (16 gathers in flight, then 8 MMAs into
// 4 rotating accumulators); the block ends up distributed as D[gid][2*tig + i].  On self chunks a second MMA against
// B2[k][0] = gp[k] (row 8 of the T record, see ba_schur_prep_kernel) yields rhs += T gp in the lanes with tig == 0.
// Rows / columns beyond an image's column count multiply whatever the buffers hold into rows / columns of D that are
// never written out (an MMA never mixes rows of A or columns of B).
__device__ __forceinline__ void dmma_884(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

__device__ __forceinline__ double ldg_f64_at(const char* base, uint32_t index, uint32_t stride_bytes) {
  return __ldg(reinterpret_cast<const double*>(base + (uint64_t)index * stride_bytes));   // one IMAD.WIDE.U32
}
template <bool SELF, int U>
__device__ __forceinline__ void schur_pairs_walk_mma(const int32_t* __restrict__ px, const int32_t* __restrict__ py, int n, int lane,
                                                     const char* Tl, const char* Wl, const char* Gl, uint32_t rec_bytes,
                                                     bool ld, bool ldg, double c[4][2], double r[2]) {
  for (int k0 = 0; k0 < n; k0 += 32) {
    // the next 32 pair indices, one per lane (coalesced); broadcast by shuffle as the walk reaches them
    const int kk = min(k0 + lane, n - 1);              // past the end: the last pair again, its MMA is skipped
    const int32_t oxl = __ldg(px + kk);
    const int32_t oyl = SELF ? oxl : __ldg(py + kk);
    const int m = min(32, n - k0);
    for (int u0 = 0; u0 < m; u0 += U) {
      double a[U], b[U], g[SELF ? U : 1];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const uint32_t ox = (uint32_t)__shfl_sync(0xffffffffu, oxl, u0 + u);
        const uint32_t oy = SELF ? ox : (uint32_t)__shfl_sync(0xffffffffu, oyl, u0 + u);
        a[u] = ld ? ldg_f64_at(Tl, ox, rec_bytes) : 0.0;
        b[u] = ld ? ldg_f64_at(Wl, oy, rec_bytes) : 0.0;
        if (SELF) g[u] = ldg ? ldg_f64_at(Gl, ox, rec_bytes) : 0.0;
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (u0 + u < m) {                              // warp-uniform
          dmma_884(c[u & 3][0], c[u & 3][1], a[u], b[u]);
          if (SELF) dmma_884(r[0], r[1], a[u], g[u]);
        }
      }
    }
  }
}

// leaves D[gid][2*tig], D[gid][2*tig + 1] in c0, c1 and (self chunks, lanes with tig == 0) the rhs entry of row gid in racc;
// U = pairs in flight per warp (8 wants the 80-register build: 3 CTAs of 256 threads per SM)
template <int U>
__device__ __forceinline__ void schur_pairs_accumulate_mma(const BADev& d, const SchurPairs& sp, const double* __restrict__ T,
                                                           int64_t kb, int64_t ke, int lane, bool self,
                                                           double& c0, double& c1, double& racc) {
  const int gid = lane >> 2, tig = lane & 3;
  const bool ld = tig < 3;
  const uint32_t rec_bytes = (uint32_t)d.dcmax * 24u;
  const int e = ld ? gid * 3 + tig : 0;                // lanes with tig == 3 carry the zero padding of k
  const char* Tl = reinterpret_cast<const char*>(T + e);
  const char* Wl = reinterpret_cast<const char*>(d.W + e);
  const char* Gl = reinterpret_cast<const char*>(T + 24 + (ld ? tig : 0));   // row 8 of the T record: the point's gradient
  double c[4][2] = {{0.0, 0.0}, {0.0, 0.0}, {0.0, 0.0}, {0.0, 0.0}}, r[2] = {0.0, 0.0};
  if (self) schur_pairs_walk_mma<true, 4>(sp.px + kb, sp.py + kb, (int)(ke - kb), lane, Tl, Wl, Gl, rec_bytes, ld, ld && gid == 0, c, r);
  else schur_pairs_walk_mma<false, U>(sp.px + kb, sp.py + kb, (int)(ke - kb), lane, Tl, Wl, Gl, rec_bytes, ld, false, c, r);
  c0 = (c[0][0] + c[1][0]) + (c[2][0] + c[3][0]);
  c1 = (c[0][1] + c[1][1]) + (c[2][1] + c[3][1]);
  racc = r[0];
}

// Fused variant (the default): T_x = W_x (H_pp + D)^-1 is not read from a precomputed buffer but formed per pair by one
// more MMA — A = the W_x fragment, B[k][2j] = Hinv[k][j] (the point's symmetric 3x3 inverse in the EVEN columns, 9 lanes
// load it) — whose accumulator D[gid][2*tig] = T[gid][tig] already is the A fragment of the product with W_y.
// Both record gathers now hit the SAME array (W; 120 MB at configs[2] instead of 240 MB for W and T), which is what
// the kernel is bound by (random 192-byte gathers against an L2 that cannot hold both arrays), ba_schur_prep_kernel
// and its 0.2 GB of traffic disappear, and g_p comes from its own array by the pair's point index.
template <bool SELF, int U>
__device__ __forceinline__ void schur_pairs_walk_fused(const int32_t* __restrict__ px, const int32_t* __restrict__ py,
                                                       const int32_t* __restrict__ pp, int n, int lane,
                                                       const char* Wl, const char* Hl, const char* Gl, uint32_t rec_bytes,
                                                       bool ld, bool ldh, bool ldg, double c[2][2], double r[2]) {
  // the next 32 pair indices, one per lane, fetched one block ahead (past the end: the last pair again, its MMAs are skipped)
  int kk = min(lane, n - 1);
  int32_t oxn = __ldg(px + kk), oyn = SELF ? 0 : __ldg(py + kk), ppn = __ldg(pp + kk);
  for (int k0 = 0; k0 < n; k0 += 32) {
    const int32_t oxl = oxn, oyl = oyn, ppl = ppn;
    kk = min(k0 + 32 + lane, n - 1);
    oxn = __ldg(px + kk); if (!SELF) oyn = __ldg(py + kk); ppn = __ldg(pp + kk);
    const int m = min(32, n - k0);
    for (int u0 = 0; u0 < m; u0 += U) {
      double a[U], b[U], h[U], g[SELF ? U : 1];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const uint32_t ox = (uint32_t)__shfl_sync(0xffffffffu, oxl, u0 + u);
        const uint32_t oy = SELF ? ox : (uint32_t)__shfl_sync(0xffffffffu, oyl, u0 + u);
        const uint32_t pt = (uint32_t)__shfl_sync(0xffffffffu, ppl, u0 + u);
        a[u] = ld ? ldg_f64_at(Wl, ox, rec_bytes) : 0.0;
        b[u] = SELF ? a[u] : (ld ? ldg_f64_at(Wl, oy, rec_bytes) : 0.0);
        h[u] = ldh ? ldg_f64_at(Hl, pt, 48u) : 0.0;
        if (SELF) g[u] = ldg ? ldg_f64_at(Gl, pt, 24u) : 0.0;
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (u0 + u < m) {                              // warp-uniform
          double t = 0.0, unused = 0.0;
          dmma_884(t, unused, a[u], h[u]);             // T = W_x Hinv with Hinv's column j placed in column 2j of B:
                                                       // D[gid][2*tig] = T[gid][tig] IS the A fragment of the next MMA
          dmma_884(c[u & 1][0], c[u & 1][1], t, b[u]);
          if (SELF) dmma_884(r[0], r[1], t, g[u]);
        }
      }
    }
  }
}

template <int U>
__device__ __forceinline__ void schur_pairs_accumulate_fused(const BADev& d, const SchurPairs& sp, const double* __restrict__ Hinv,
                                                             int64_t kb, int64_t ke, int lane, bool self,
                                                             double& c0, double& c1, double& racc) {
  const int gid = lane >> 2, tig = lane & 3;
  // B of the first MMA: B[k][2j] = Hinv[k][j], j < 3 (odd columns and columns 6, 7 zero): lane (gid = 2j, tig = k) loads it
  const bool ld = tig < 3, ldh = ld && gid < 6 && (gid & 1) == 0;
  const uint32_t rec_bytes = (uint32_t)d.dcmax * 24u;
  const int e = ld ? gid * 3 + tig : 0;                // lanes with tig == 3 carry the zero padding of k
  // symmetric storage of the inverse: (0,0) (0,1) (0,2) (1,1) (1,2) (2,2)
  const int lo = min(gid >> 1, tig), hi = max(gid >> 1, tig);
  const int hidx = ldh ? (lo == 0 ? hi : (lo == 1 ? 2 + hi : 5)) : 0;
  const char* Wl = reinterpret_cast<const char*>(d.W + e);
  const char* Hl = reinterpret_cast<const char*>(Hinv + hidx);
  const char* Gl = reinterpret_cast<const char*>(d.gp + (ld ? tig : 0));
  double c[2][2] = {{0.0, 0.0}, {0.0, 0.0}}, r[2] = {0.0, 0.0};
  const int n = (int)(ke - kb);
  if (self) schur_pairs_walk_fused<true, 4>(sp.px + kb, sp.py + kb, sp.pp + kb, n, lane, Wl, Hl, Gl, rec_bytes, ld, ldh, ld && gid == 0, c, r);
  else schur_pairs_walk_fused<false, U>(sp.px + kb, sp.py + kb, sp.pp + kb, n, lane, Wl, Hl, Gl, rec_bytes, ld, ldh, false, c, r);
  c0 = c[0][0] + c[1][0];
  c1 = c[0][1] + c[1][1];
  racc = r[0];
}

template <int CTAS, bool FUSED>
static __global__ void __launch_bounds__(kPairThreads, CTAS) ba_schur_pairs_mma_kernel(BADev d, SchurPairs sp, const double* __restrict__ T /* FUSED: Hinv */,
                                                                                       double* S, double* rhs) {
  const int64_t c = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (c >= sp.n_chunks) return;
  const int64_t kb = sp.chunk_begin[c], ke = sp.chunk_begin[c + 1];
  if (ke <= kb) return;
  const int dcm = d.dcmax;
  const bool self = sp.chunk_self[c] != 0;
  double acc[2], racc;
  if constexpr (FUSED) schur_pairs_accumulate_fused<(CTAS <= 3 ? 8 : 4)>(d, sp, T, kb, ke, lane, self, acc[0], acc[1], racc);
  else schur_pairs_accumulate_mma<(CTAS <= 3 ? 8 : 4)>(d, sp, T, kb, ke, lane, self, acc[0], acc[1], racc);
  const int a = lane >> 2, tig = lane & 3;
  const int64_t ox0 = sp.px[kb], oy0 = sp.py[kb];
  const int dcx = d.Wdc[ox0], dcy = d.Wdc[oy0];
  if (a >= dcx) return;
  const int ca = d.Wcols[ox0 * dcm + a];
  if (self && tig == 0) atomic_add_f64(&rhs[ca], racc);
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int b = 2 * tig + i;
    if (b >= dcy) continue;
    const int cb = d.Wcols[oy0 * dcm + b];
    const double v = -acc[i];
    if (self) { if (a >= b) atomic_add_f64(&S[(int64_t)ca * d.nc + cb], v); }
    else if (ca > cb) atomic_add_f64(&S[(int64_t)ca * d.nc + cb], v);
    else if (ca < cb) atomic_add_f64(&S[(int64_t)cb * d.nc + ca], v);
    else atomic_add_f64(&S[(int64_t)ca * d.nc + ca], 2.0 * v);
  }
}

// ---------------------------------------------------------------- dense Cholesky (lower, in place)
// The reduced system is stored as an (n+1) x n row-major array: rows 0..n-1 hold the lower
// triangle of S, row n holds the right-hand side.  Factorising with the extra row performs the
// forward substitution for free: after the last panel row n holds y = L^-1 rhs.
constexpr int kNB = 32;
// Panel step k: every CTA factors the diagonal block A_kk redundantly in shared memory (one warp,
// warp-synchronous); CTA 0 writes L_kk back, CTA b>0 solves its 32-row block L_bk = A_bk L_kk^-T
// with one warp per row.
// Panel step k, part 1: one warp factors the 32x32 diagonal block A_kk entirely in registers (lane i
// keeps row i, column values travel by shuffle) and writes L_kk back plus the reciprocal diagonal.
static __global__ void __launch_bounds__(32) chol_diag_kernel(double* A, int n, int k, double* rdiag_out, int* fail_flag) {
  const int tx = threadIdx.x;
  const int k0 = k * kNB;
  const int kb = min(kNB, n - k0);
  double r[kNB];
#pragma unroll
  for (int c = 0; c < kNB; ++c) r[c] = (tx < kb && c < kb && c <= tx) ? A[(int64_t)(k0 + tx) * n + k0 + c] : (c == tx ? 1.0 : 0.0);
  bool ok = true;
#pragma unroll
  for (int j = 0; j < kNB; ++j) {
    const double dj = __shfl_sync(0xffffffffu, r[j], j);
    if (!(dj > 0.0) || !isfinite(dj)) ok = false;
    const double rj = rsqrt(dj);
    if (tx == j) { r[j] = dj * rj; rdiag_out[j] = rj; }
    else if (tx > j) r[j] *= rj;
    const double lij = r[j];
#pragma unroll
    for (int c = j + 1; c < kNB; ++c) {
      const double lcj = __shfl_sync(0xffffffffu, lij, c);
      if (tx >= c) r[c] -= lij * lcj;
    }
  }
  if (!ok && tx == 0) *fail_flag = 1;
#pragma unroll
  for (int c = 0; c < kNB; ++c)
    if (tx < kb && c < kb && c <= tx) A[(int64_t)(k0 + tx) * n + k0 + c] = r[c];
}

// Panel step k, part 2: rows below the diagonal block (including the appended rhs row):
// L_bk = A_bk L_kk^-T, one warp per row, CTA b handles the 32 rows starting at k0 + kb + b*32.
constexpr int kPanelThreads = 1024;
static __global__ void __launch_bounds__(kPanelThreads) chol_panel_kernel(double* A, int n, int n_rows, int k, const double* rdiag_in) {
  __shared__ double Lkk[kNB][kNB + 1];
  __shared__ double rdiag[kNB];
  const int tx = threadIdx.x % kNB, ty = threadIdx.x / kNB;
  const int k0 = k * kNB;
  const int kb = min(kNB, n - k0);
  Lkk[ty][tx] = (ty < kb && tx < kb && tx <= ty) ? A[(int64_t)(k0 + ty) * n + k0 + tx] : 0.0;
  if (ty == 0) rdiag[tx] = rdiag_in[tx];
  __syncthreads();
  const int r = k0 + kb + blockIdx.x * kNB + ty;
  if (r >= n_rows) return;
  double v = tx < kb ? A[(int64_t)r * n + k0 + tx] : 0.0;
  for (int j = 0; j < kb; ++j) {
    const double xj = __shfl_sync(0xffffffffu, v, j) * rdiag[j];
    if (tx == j) v = xj;
    else if (tx > j && tx < kb) v -= xj * Lkk[tx][j];
  }
  if (tx < kb) A[(int64_t)r * n + k0 + tx] = v;
}

// Trailing update after panel k: A_ij -= L_ik L_jk^T for row tiles i >= column tiles j > k, rows
// up to n_rows (the rhs row rides along), columns < n.
static __global__ void __launch_bounds__(kNB* kNB) chol_update_kernel(double* A, int n, int n_rows, int k) {
  int t = blockIdx.x;
  int bi = (int)((sqrt(8.0 * t + 1.0) - 1.0) * 0.5);
  while ((bi + 1) * (bi + 2) / 2 <= t) ++bi;
  while (bi * (bi + 1) / 2 > t) --bi;
  const int bj = t - bi * (bi + 1) / 2;
  const int i0 = (k + 1 + bi) * kNB, j0 = (k + 1 + bj) * kNB, k0 = k * kNB;
  if (i0 >= n_rows || j0 >= n) return;
  const int kb = min(kNB, n - k0);
  __shared__ double Li[kNB][kNB + 1];
  __shared__ double Lj[kNB][kNB + 1];
  const int tx = threadIdx.x % kNB, ty = threadIdx.x / kNB;
  Li[ty][tx] = (i0 + ty < n_rows && tx < kb) ? A[(int64_t)(i0 + ty) * n + k0 + tx] : 0.0;
  Lj[ty][tx] = (j0 + ty < n && tx < kb) ? A[(int64_t)(j0 + ty) * n + k0 + tx] : 0.0;
  __syncthreads();
  const int r = i0 + ty, c = j0 + tx;
  if (r < n_rows && c < n && (c <= r)) {
    double s = 0.0;
#pragma unroll
    for (int q = 0; q < kNB; ++q) s += Li[ty][q] * Lj[tx][q];
    A[(int64_t)r * n + c] -= s;
  }
}

// Backward substitution L^T x = y (y = row n of the factorised array, see above), single CTA.
// Each 32-block: stage L_kk in shared memory, one warp solves it with shuffles, then all threads
// apply the block's contribution to the remaining entries with coalesced row reads.
static __global__ void __launch_bounds__(1024) chol_backsolve_kernel(const double* L, const double* y_in, double* x, int n) {
  __shared__ double Lkk[kNB][kNB + 1];
  __shared__ double xb[kNB];
  const int nb = (n + kNB - 1) / kNB;
  const int tx = threadIdx.x % kNB, ty = threadIdx.x / kNB;
  for (int i = threadIdx.x; i < n; i += blockDim.x) x[i] = y_in[i];
  __syncthreads();
  for (int k = nb - 1; k >= 0; --k) {
    const int k0 = k * kNB, kb = min(kNB, n - k0);
    Lkk[ty][tx] = (ty < kb && tx < kb && tx <= ty) ? L[(int64_t)(k0 + ty) * n + k0 + tx] : (ty == tx ? 1.0 : 0.0);
    __syncthreads();
    if (ty == 0) {
      double v = tx < kb ? x[k0 + tx] : 0.0;
      const double rd = 1.0 / Lkk[tx][tx];
      for (int j = kb - 1; j >= 0; --j) {
        const double xj = __shfl_sync(0xffffffffu, v, j) * __shfl_sync(0xffffffffu, rd, j);
        if (tx == j) v = xj;
        else if (tx < j) v -= Lkk[j][tx] * xj;
      }
      if (tx < kb) { x[k0 + tx] = v; xb[tx] = v; }
    }
    __syncthreads();
    for (int c = threadIdx.x; c < k0; c += blockDim.x) {
      double s = 0.0;
      for (int j = 0; j < kb; ++j) s += L[(int64_t)(k0 + j) * n + c] * xb[j];
      x[c] -= s;
    }
    __syncthreads();
  }
}

// K5a: back-substitution, one warp per point:  delta_p = (Hpp+D)^-1 (-gp - sum_i W_i^T delta_c[cols_i])
static __global__ void __launch_bounds__(256) ba_backsub_kernel(BADev d, const double* D2, double* delta) {
  const int64_t p = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (p >= d.n_points || d.point_off[p] < 0) return;
  const int64_t po = d.point_off[p];
  const int64_t ob = d.pt_begin[p];
  const int n = (int)(d.pt_begin[p + 1] - ob) * d.dcmax;
  double w0 = 0, w1 = 0, w2 = 0;
  for (int e = lane; e < n; e += 32) {
    const int64_t o = ob + e / d.dcmax;
    const int a = e % d.dcmax;
    if (a < d.Wdc[o]) {
      const double dca = delta[d.Wcols[o * d.dcmax + a]];
      const double* w = d.W + (o * d.dcmax + a) * 3;
      w0 += w[0] * dca; w1 += w[1] * dca; w2 += w[2] * dca;
    }
  }
  w0 = warp_sum(w0); w1 = warp_sum(w1); w2 = warp_sum(w2);
  if (lane == 0) {
    double inv[9];
    inv3_sym(d.Hpp + p * 9, D2 + po, inv);
    const double v[3] = {-d.gp[p * 3] - w0, -d.gp[p * 3 + 1] - w1, -d.gp[p * 3 + 2] - w2};
    for (int a = 0; a < 3; ++a) delta[po + a] = inv[a * 3] * v[0] + inv[a * 3 + 1] * v[1] + inv[a * 3 + 2] * v[2];
  }
}

// K5b: model cost change, the literal ceres formula  -(J d)^T (r + J d / 2)  per residual block in
// the reduced 2-D space:  u = d(uv)/d(theta) * delta ;  acc += u^T b' + u^T A' u / 2   (one thread per obs)
template <bool FAST>
static __global__ void __launch_bounds__(256) ba_model_cost_kernel(BADev d, const double* delta, double* acc, double* block_part = nullptr) {
  const int64_t o = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  double part = 0.0;
  if (o < d.n_obs) {
    const int Wd = 9 + d.K;
    const double* oo = d.obs_out + o * 8;
    double rho[3];
    loss_eval(d.loss, 1.0, oo[0], rho);
    const double* J = d.juv + o * (int64_t)d.juv_stride;
    constexpr int NA = FAST ? 8 : kMaxDc;
    int cols[NA];
    double Ju[NA], Jv[NA];
    int dc;
    if constexpr (FAST) dc = obs_local_columns8(d, o, J, Wd, cols, Ju, Jv);
    else dc = obs_local_columns(d, o, J, Wd, cols, Ju, Jv);
    double uu = 0.0, uv = 0.0;
#pragma unroll
    for (int a = 0; a < NA; ++a) {
      if (a >= dc) break;
      const double dl = delta[cols[a]]; uu += Ju[a] * dl; uv += Jv[a] * dl;
    }
    const int64_t po = d.point_off[d.obs_pt[o]];
    if (po >= 0) {
#pragma unroll
      for (int k = 0; k < 3; ++k) { const double dl = delta[po + k]; uu += J[6 + k] * dl; uv += J[Wd + 6 + k] * dl; }
    }
    part = rho[1] * (uu * oo[1] + uv * oo[2] + 0.5 * (uu * (oo[3] * uu + oo[4] * uv) + uv * (oo[4] * uu + oo[5] * uv)));
  }
  __shared__ double sh[8];
  part = warp_sum(part);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = part;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0; for (int k = 0; k < 8; ++k) t += sh[k];
    if (block_part) block_part[blockIdx.x] = t;   // deterministic mode: summed in block order by det_reduce_add_kernel
    else atomic_add_f64(&acc[0], t);
  }
}

// (A variant of K5b that staged its records through shared memory like ba_build_staged_kernel measured no gain when
//  the kernels were written; not re-measured on H100 — the kernel reads, it does not scatter.)
// K6: x_plus = Plus(x, delta) for every block; also accumulates ||x||^2, ||x_plus - x||^2 (ambient)
struct PlusArgs {
  int n_cameras, n_images; int64_t n_points;
  const int32_t* cam_model; const uint32_t* cam_mask; const uint8_t* tmask;
  const int32_t* pose_off; const int32_t* intr_off; const int64_t* point_off;
  const double* cam; const double* q; const double* t; const double* X;
  double* cam_o; double* q_o; double* t_o; double* X_o;
  const double* delta;
  double* acc;  // points: [1] += ||x_plus - x||^2, [2] += ||x||^2 ; cameras/poses: [3], [4] (replicated across ranks)
  double* part = nullptr;   // deterministic mode: [gridDim.x][4] per-block sums instead of the atomics
};
static __global__ void __launch_bounds__(128) ba_plus_kernel(PlusArgs a) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  double dn = 0.0, xn = 0.0, dnc = 0.0, xnc = 0.0;
  if (i < a.n_points) {
    const int64_t po = a.point_off[i];
    for (int k = 0; k < 3; ++k) {
      const double x = a.X[3 * i + k];
      const double xp = po >= 0 ? x + a.delta[po + k] : x;
      a.X_o[3 * i + k] = xp;
      dn += (xp - x) * (xp - x); xn += x * x;
    }
  }
  if (i < a.n_images) {
    const int po = a.pose_off[i];
    double qn[4];
    const double* q = a.q + 4 * i;
    const double* t = a.t + 3 * i;
    if (po >= 0) {
      quaternion_plus(q, a.delta + po, qn);
      int la = 3;
      for (int k = 0; k < 3; ++k) {
        double tp = t[k];
        if (!(a.tmask[i] & (1u << k))) tp += a.delta[po + la++];
        a.t_o[3 * i + k] = tp;
        dnc += (tp - t[k]) * (tp - t[k]);
      }
    } else {
      for (int k = 0; k < 4; ++k) qn[k] = q[k];
      for (int k = 0; k < 3; ++k) a.t_o[3 * i + k] = t[k];
    }
    for (int k = 0; k < 4; ++k) { a.q_o[4 * i + k] = qn[k]; dnc += (qn[k] - q[k]) * (qn[k] - q[k]); xnc += q[k] * q[k]; }
    for (int k = 0; k < 3; ++k) xnc += t[k] * t[k];
  }
  if (i < a.n_cameras) {
    const int io = a.intr_off[i];
    const int Kc = cam_num_params(a.cam_model[i]);
    int la = 0;
    for (int k = 0; k < kMaxK; ++k) {
      const double c = a.cam[i * kMaxK + k];
      double cpv = c;
      if (io >= 0 && k < Kc && !(a.cam_mask[i] & (1u << k))) cpv += a.delta[io + la++];
      a.cam_o[i * kMaxK + k] = cpv;
      dnc += (cpv - c) * (cpv - c);
      if (k < Kc) xnc += c * c;
    }
  }
  __shared__ double sh[4][4];
  dn = warp_sum(dn); xn = warp_sum(xn); dnc = warp_sum(dnc); xnc = warp_sum(xnc);
  if ((threadIdx.x & 31) == 0) { sh[0][threadIdx.x >> 5] = dn; sh[1][threadIdx.x >> 5] = xn; sh[2][threadIdx.x >> 5] = dnc; sh[3][threadIdx.x >> 5] = xnc; }
  __syncthreads();
  if (threadIdx.x < 4) {
    const double v = sh[threadIdx.x][0] + sh[threadIdx.x][1] + sh[threadIdx.x][2] + sh[threadIdx.x][3];
    if (a.part) a.part[(int64_t)blockIdx.x * 4 + threadIdx.x] = v;
    else if (v != 0.0) atomic_add_f64(&a.acc[1 + threadIdx.x], v);
  }
}

// deterministic mode: out[0] += sum_b part[b * stride + k] in block order (one CTA, fixed tree)
static __global__ void __launch_bounds__(1024) det_reduce_add_kernel(const double* __restrict__ part, int64_t n_blocks, int stride, int k, double* out) {
  __shared__ double sh[32];
  double s = 0.0;
  for (int64_t i = threadIdx.x; i < n_blocks; i += blockDim.x) s += part[i * stride + k];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    double v = sh[threadIdx.x];
    v = warp_sum(v);
    if (threadIdx.x == 0) out[0] += v;
  }
}

static __global__ void flags_to_double_kernel(const int* flags, double* out) { out[0] = (double)(flags[0] + flags[1]); }

// deterministic final reduction of per-warp cost partials: out[0] = sum
static __global__ void __launch_bounds__(1024) reduce_partials_kernel(const double* partials, int64_t n, double* out) {
  __shared__ double sh[32];
  double s = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) s += partials[i];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    double v = sh[threadIdx.x];
    v = warp_sum(v);
    if (threadIdx.x == 0) out[0] = v;
  }
}

// ceres' gradient_max_norm = || x - Plus(x, -g) ||_inf (trust_region_minimizer.cc: ComputeGradientNorms): for
// Euclidean blocks (translations, intrinsics, points) that is max |g_i|, for the quaternion block the gradient step goes
// through the manifold.  One thread per image / camera / point; `gc` is passed explicitly (block mode: the all-reduced
// copy), with_points = 0 leaves the point part to the caller (block mode: per-rank maximum exchanged separately).
static __global__ void __launch_bounds__(256) ba_gradmax_kernel(BADev d, const double* __restrict__ gc, const double* __restrict__ q,
                                                                int with_points, double* out /* as ordered-uint max */) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  double m = 0.0;
  if (i < d.n_images) {
    const int po = d.pose_off[i];
    if (po >= 0) {
      const double ng[3] = {-gc[po], -gc[po + 1], -gc[po + 2]};
      double qn[4];
      quaternion_plus(q + 4 * i, ng, qn);
#pragma unroll
      for (int k = 0; k < 4; ++k) m = fmax(m, fabs(q[4 * i + k] - qn[k]));
      const int nt = 3 - __popc(d.tmask[i] & 7u);
      for (int k = 0; k < nt; ++k) m = fmax(m, fabs(gc[po + 3 + k]));
    }
  }
  if (i < d.n_cameras) {
    const int io = d.intr_off[i];
    if (io >= 0) {
      const int Kc = cam_num_params(d.cam_model[i]);
      const int nk = Kc - __popc(d.cam_mask[i] & ((1u << Kc) - 1u));
      for (int k = 0; k < nk; ++k) m = fmax(m, fabs(gc[io + k]));
    }
  }
  if (with_points && i < d.n_points && d.point_off[i] >= 0)
    m = fmax(m, fmax(fabs(d.gp[i * 3]), fmax(fabs(d.gp[i * 3 + 1]), fabs(d.gp[i * 3 + 2]))));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > 0.0)
    atomicMax(reinterpret_cast<unsigned long long*>(out), (unsigned long long)__double_as_longlong(m));
}

}  // namespace pxr
