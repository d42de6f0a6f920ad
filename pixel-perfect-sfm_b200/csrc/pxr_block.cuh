// pxr_block.cuh — the reduced camera system in "image-block" form as the ONE message of a multi-GPU LM iteration.
//
// north_star: "observations (BA) shard across the GPUs of one box with a single NCCL allreduce of the reduced camera
// normal-equation blocks per LM iteration".  The reference has no counterpart (it is single-process,
// base/src/parallel_optimizer.h:77-211); what is replaced is the Schur elimination + reduced solve inside ceres::Solve
// (bundle_adjustment/src/bundle_optimizer.h:181-191,224).
//
// Every rank eliminates ITS points and accumulates, into one contiguous buffer `pack`:
//     [ H_img  n_images x 64 | B_key  n_keys x 64 | rhsS  nc | g_c  nc | slots  kPackSlots ]
//   H_img  = sum_obs J_c^T A' J_c per image (8x8, lower triangle filled)        (ba_build_cam_kernel)
//   B_key  = sum_pairs T_x W_y^T per co-visible image pair (a >= b, self flag)   (sp_schur_pairs_kernel)
//   rhsS   = sum_obs T g_p,  g_c = this rank's partial camera gradient
//   slots  = reserved (zeros)
// The key list is the UNION of the ranks' co-visible image pairs (all-gathered once at set-up), so the layout is the same
// everywhere and ONE ncclAllReduce(sum) of `pack` gives every rank the global blocks.  Everything after the all-reduce
// is a deterministic function of that buffer (no atomics: fixed-order gathers, tile-DAG Cholesky / fixed-order PCG), so
// all ranks compute bit-identical camera steps and their replicated camera state never drifts apart.  The camera
// damping D_c = clamp(diag H_cc)/radius needs the GLOBAL diagonal: it is added after the reduction.
#pragma once
#include "pxr_sparse_schur.cuh"

namespace pxr {

constexpr int kPackSlots = 16;

// out[dest] = sum_j sign_j * buf[src_j]  over the CSR row of `dest` (fixed order).  src >= 0: +buf[src]; src < 0: -buf[~src].
struct GatherMap {
  const int64_t* dest;      // [n_rows] destination index
  const int64_t* ptr;       // [n_rows + 1]
  const int32_t* src;       // [nnz]
  int64_t n_rows;
};

// dense S (lower triangle, (nc+1) x nc array zeroed by the caller) from the global blocks, + camera damping on the diagonal
static __global__ void __launch_bounds__(256) blk_gather_kernel(GatherMap m, const double* __restrict__ buf, double* __restrict__ out,
                                                                const double* __restrict__ D2, int nc) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= m.n_rows) return;
  double v = 0.0;
  for (int64_t j = m.ptr[r]; j < m.ptr[r + 1]; ++j) {
    const int32_t s = m.src[j];
    v += s >= 0 ? buf[s] : -buf[~s];
  }
  const int64_t d = m.dest[r];
  if (D2) { const int64_t row = d / nc, col = d - row * nc; if (row == col) v += D2[row]; }
  out[d] = v;
}

// after the all-reduce: diag(H_cc) of the camera columns (fixed-order gather through `dg`), Jacobi scale of the camera
// columns at LM iteration 0, LM damping of the camera columns, rhs = -g_c + rhsS, and max_i |g_c[i]| (the point part of
// max |g| is a per-rank maximum that travels with the scalar exchange)
static __global__ void __launch_bounds__(256) blk_post_kernel(GatherMap dg, const double* __restrict__ buf, const double* __restrict__ gc,
                                                              const double* __restrict__ rhsS, double* diag, double* jscale, int set_scale,
                                                              int jacobi_scaling, double* D2, double radius, double lo, double hi, double* rhs,
                                                              int nc, double* gmax_out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double m = 0.0;
  if (i < nc) {
    double v = 0.0;
    for (int64_t j = dg.ptr[i]; j < dg.ptr[i + 1]; ++j) v += buf[dg.src[j]];
    diag[i] = v;
    if (set_scale) jscale[i] = jacobi_scaling ? jacobi_scale(v) : 1.0;
    D2[i] = lm_damping(v, jscale[i], radius, lo, hi);
    rhs[i] = -gc[i] + rhsS[i];
    m = fabs(gc[i]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > 0.0)
    atomicMax(reinterpret_cast<unsigned long long*>(gmax_out), (unsigned long long)__double_as_longlong(m));   // max is order-free
}
static __global__ void __launch_bounds__(256) blk_absmax_kernel(const double* __restrict__ v, int n, double* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double m = i < n ? fabs(v[i]) : 0.0;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > 0.0)
    atomicMax(reinterpret_cast<unsigned long long*>(out), (unsigned long long)__double_as_longlong(m));
}

// ---------------------------------------------------------------- deterministic assembly (pxr_solver_options.deterministic)
// The block build sums with fp64 atomics: one per element per 128-observation chunk (camera blocks), per pair chunk (B_key,
// rhs) and per (point, warp) (H_pp, g_p) — the order of those additions changes from run to run (1e-16 relative per sum).
// In deterministic mode the chunk kernels write their partial sums instead and these kernels add them in a fixed order.

// H_img (36 lower-triangle entries) and the image's gradient (8) from its chunks, in chunk order
static __global__ void __launch_bounds__(256) det_cam_reduce_kernel(const double* __restrict__ part, const int64_t* __restrict__ img_chunk_begin,
                                                                    int n_images, double* __restrict__ Himg, double* __restrict__ gimg) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (int64_t)n_images * 48) return;
  const int img = (int)(t / 48), e = (int)(t % 48);
  if (e >= 44) return;
  double v = 0.0;
  for (int64_t c = img_chunk_begin[img]; c < img_chunk_begin[img + 1]; ++c) v += part[c * 48 + e];
  if (e < 36) {
    int a = 0;
    while ((a + 1) * (a + 2) / 2 <= e) ++a;
    Himg[(int64_t)img * 64 + a * 8 + (e - a * (a + 1) / 2)] = v;
  } else {
    gimg[(int64_t)img * 8 + (e - 36)] = v;
  }
}

// B_key (64) and, for self keys, the image's  sum T g_p  (8) from the key's pair chunks, in chunk order
static __global__ void __launch_bounds__(256) det_pair_reduce_kernel(const double* __restrict__ part, const int64_t* __restrict__ key_chunk_begin,
                                                                     int n_keys, const int32_t* __restrict__ key_a, const uint8_t* __restrict__ key_self,
                                                                     double* __restrict__ Bk, double* __restrict__ rimg) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (int64_t)n_keys * 72) return;
  const int key = (int)(t / 72), e = (int)(t % 72);
  double v = 0.0;
  for (int64_t c = key_chunk_begin[key]; c < key_chunk_begin[key + 1]; ++c) v += part[c * 72 + e];
  if (e < 64) Bk[(int64_t)key * 64 + e] = v;
  else if (key_self[key]) rimg[(int64_t)key_a[key] * 8 + (e - 64)] = v;
}

// out[col] = sum over the images that own the column of vec[img][a], in the fixed order of the diagonal gather map
// (dg.src = img*64 + a*9): the camera gradient and the Schur right-hand side
static __global__ void __launch_bounds__(256) det_gather_cols_kernel(GatherMap dg, const double* __restrict__ vec, double* __restrict__ out, int nc) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nc) return;
  double v = 0.0;
  for (int64_t j = dg.ptr[i]; j < dg.ptr[i + 1]; ++j) { const int32_t s = dg.src[j]; v += vec[(int64_t)(s >> 6) * 8 + (s & 63) / 9]; }
  out[i] = v;
}

// H_pp / g_p of every point from its observations in observation order (they are sorted by point): overwrites what
// ba_build_staged_kernel accumulated with atomics
static __global__ void __launch_bounds__(128) det_point_blocks_kernel(BADev d) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= d.n_points) return;
  double v[12];
#pragma unroll
  for (int k = 0; k < 12; ++k) v[k] = 0.0;
  if (d.point_off[p] >= 0) {
    const int Wd = 9 + d.K;
    for (int64_t o = d.pt_begin[p]; o < d.pt_begin[p + 1]; ++o) {
      const double* oo = d.obs_out + o * 8;
      double rho[3];
      loss_eval(d.loss, 1.0, oo[0], rho);
      const double bu = rho[1] * oo[1], bv = rho[1] * oo[2];
      const double auu = rho[1] * oo[3], auv = rho[1] * oo[4], avv = rho[1] * oo[5];
      const double* J = d.juv + o * (int64_t)d.juv_stride;
      const double pu[3] = {J[6], J[7], J[8]}, pv[3] = {J[Wd + 6], J[Wd + 7], J[Wd + 8]};
      double apu[3], apv[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) { apu[k] = auu * pu[k] + auv * pv[k]; apv[k] = auv * pu[k] + avv * pv[k]; }
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        v[a] += pu[a] * bu + pv[a] * bv;
#pragma unroll
        for (int b = 0; b < 3; ++b) v[3 + a * 3 + b] += pu[a] * apu[b] + pv[a] * apv[b];
      }
    }
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) d.gp[p * 3 + a] = v[a];
#pragma unroll
  for (int k = 0; k < 9; ++k) d.Hpp[p * 9 + k] = v[3 + k];
}

// max |g_p| over this rank's variable points -> slot (as ordered-uint max; the slot is zeroed by the caller)
static __global__ void __launch_bounds__(256) blk_gpmax_kernel(const double* __restrict__ gp, const int64_t* __restrict__ point_off,
                                                               int64_t n_points, double* slot) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  double m = 0.0;
  if (i < n_points && point_off[i] >= 0) m = fmax(fabs(gp[i * 3]), fmax(fabs(gp[i * 3 + 1]), fabs(gp[i * 3 + 2])));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > 0.0)
    atomicMax(reinterpret_cast<unsigned long long*>(slot), (unsigned long long)__double_as_longlong(m));
}

// ---------------------------------------------------------------- deterministic block-row product  q = S p
// Rows are images.  The entries of image `a` — (key k, transposed) for every co-visible pair it takes part in — are cut
// into row chunks of <= kRowChunk entries; one 8-lane group per chunk accumulates  -B x_b  (or -B^T x_a') in registers in
// list order and stores its 8 partial results; the first chunk of an image also adds H_img x_a.  A second kernel
// gathers, per camera column and in fixed order, the partials of the (image, row) slots that map to the column (pose
// columns: one image; shared intrinsics: all images of the camera) and adds the damping.  No atomics anywhere.
constexpr int kRowChunk = 16;
struct BlockRows {
  const int64_t* chunk_begin;   // [n_chunks + 1] into entries
  const int32_t* chunk_img;     // [n_chunks]
  const uint8_t* chunk_first;   // [n_chunks] 1: adds the H_img term
  const int32_t* ent_key;       // [n_entries] key id, bit 31 set: transposed (the row image is the key's b side)
  int64_t n_chunks;
  GatherMap cols;               // per camera column: the (chunk * 8 + a) partials that feed it
};

static __global__ void __launch_bounds__(256) blk_rows_kernel(SparseSchur s, BlockRows br, const double* __restrict__ p,
                                                              double* __restrict__ ypart, const CGState* st) {
  if (st && st->done) return;
  const int64_t c = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 3;
  const int a = threadIdx.x & 7;
  const unsigned gmask = 0xFFu << (threadIdx.x & 24);
  if (c >= br.n_chunks) return;
  const int img = br.chunk_img[c];
  double acc = 0.0;
  if (br.chunk_first[c]) {
    const int ca = s.img_cols[img * 8 + a];
    const double xa = ca >= 0 ? p[ca] : 0.0;
    const double* H = s.Himg + (int64_t)img * 64;
#pragma unroll
    for (int b = 0; b < 8; ++b) {
      const double xb = __shfl_sync(gmask, xa, b, 8);
      acc += (a >= b ? H[a * 8 + b] : H[b * 8 + a]) * xb;
    }
  }
  for (int64_t e = br.chunk_begin[c]; e < br.chunk_begin[c + 1]; ++e) {
    const int32_t ek = br.ent_key[e];
    const bool tr = ek < 0;
    const int64_t k = ek & 0x7fffffff;
    const int other = tr ? s.key_a[k] : s.key_b[k];
    const int co = s.img_cols[other * 8 + a];
    const double xo = co >= 0 ? p[co] : 0.0;
    const double* B = s.Bk + k * 64;
    double y = 0.0;
#pragma unroll
    for (int b = 0; b < 8; ++b) y += (tr ? B[b * 8 + a] : B[a * 8 + b]) * __shfl_sync(gmask, xo, b, 8);
    acc -= y;
  }
  ypart[c * 8 + a] = acc;
}

static __global__ void __launch_bounds__(256) blk_cols_kernel(GatherMap cols, const double* __restrict__ ypart, const double* __restrict__ D2,
                                                              const double* __restrict__ p, double* __restrict__ q, int nc, const CGState* st) {
  if (st && st->done) return;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nc) return;
  double v = 0.0;
  for (int64_t j = cols.ptr[i]; j < cols.ptr[i + 1]; ++j) v += ypart[cols.src[j]];
  q[i] = v + D2[i] * p[i];
}

}  // namespace pxr
