// pxr_sparse_schur.cuh — the reduced camera system WITHOUT a dense matrix, for ITERATIVE_SCHUR at camera counts
// where nc^2 does not fit (BASELINE config 5: 5 000 cameras -> nc = 40 000, dense S = 12.8 GB, block-sparse ~0.2 GB).
//
// The reference hands this case to Ceres' ITERATIVE_SCHUR + SCHUR_JACOBI (bundle_optimizer.h:188-190), which never
// forms S either (ImplicitSchurComplement).  Here S is kept in "image-block" form: every observation's camera
// columns are the columns of its image (pose block + the intrinsics block of the image's camera), so
//     S = sum_img P_img^T H_img P_img + D  -  sum_{co-visible image pairs (a >= b)} [ P_a^T B_ab P_b (+ transpose) ]
// with H_img = sum_obs J_c^T A' J_c (8x8, from ba_build_cam_kernel) and B_ab = sum_pairs T_x W_y^T (8x8, from
// the Schur pair list whose chunks are already grouped by image pair).  P_img gathers the <= 8 columns of an image.
// What PCG needs:
//   sp_spmv_kernel        q = S p           one 8-lane group per block, gathers p, scatters with fp64 atomics
//   sp_blockdiag_kernel   the parameter-block diagonal of S (SCHUR_JACOBI), pose and camera blocks
//   sp_diag_kernel        diag(H_cc) for the Jacobi scaling / LM damping
// In the multi-GPU path every rank holds the blocks of ITS points; q is all-reduced per CG iteration (nc doubles),
// the block diagonal once per LM attempt — no rank ever needs another rank's co-visibility structure.
#pragma once
#include "pxr_ba_kernels.cuh"
#include "pxr_pcg.cuh"

namespace pxr {

constexpr int kSB = 8;                    // block edge: images with more than 8 camera columns use the dense path

struct SparseSchur {
  int n_images, n_keys, nc;
  const int32_t* img_cols;                // [n_images][8] local column of each block row, -1 beyond dc
  const int32_t* img_pd;                  // [n_images] number of pose columns (the first pd entries of img_cols)
  const int32_t* img_pose_blk;            // [n_images] SCHUR_JACOBI block id of the pose, -1 if constant
  const int32_t* img_cam_blk;             // [n_images] block id of the intrinsics, -1 if constant
  const int32_t* key_a; const int32_t* key_b; const uint8_t* key_self;   // [n_keys] image pair (a >= b)
  double* Himg;                           // [n_images][64] (lower triangle filled)
  double* Bk;                             // [n_keys][64]   sum T_x W_y^T  (x in image a)
};

// Schur pair chunks -> image-pair blocks (the fast path of ba_schur_pairs_kernel with a different sink)
// STAGED: 0 the direct walk, 1 the staged one with 16-byte gathers, 2 with 8-byte gathers (odd record length),
//         3 the tensor-core walk on the precomputed T, 4 the fused tensor-core walk (the default; `T` is Hinv then)
template <int STAGED>
static __global__ void __launch_bounds__(kPairThreads, STAGED == 3 ? 3 : (STAGED ? 4 : 1)) sp_schur_pairs_kernel(BADev d, SchurPairs sp, const int32_t* __restrict__ chunk_key,
                                                                    const double* __restrict__ T, double* __restrict__ Bk, double* rhs,
                                                                    double* __restrict__ part = nullptr /* deterministic mode: [n_chunks][72] */) {
  __shared__ __align__(16) double stage_all[(STAGED == 1 || STAGED == 2) ? kStageDoubles : 2];
  const int64_t c = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (c >= sp.n_chunks) return;
  const int64_t kb = sp.chunk_begin[c], ke = sp.chunk_begin[c + 1];
  if (ke <= kb) return;
  const int dcm = d.dcmax;
  const int64_t ox0 = sp.px[kb], oy0 = sp.py[kb];
  const int dcx = d.Wdc[ox0], dcy = d.Wdc[oy0];
  const bool self = sp.chunk_self[c] != 0;
  if constexpr (STAGED >= 3) {
    // block distributed as D[row][2*tig + i] over the warp (schur_pairs_accumulate_mma / _fused)
    double cc[2], rr;
    if constexpr (STAGED == 4) schur_pairs_accumulate_fused<4>(d, sp, T, kb, ke, lane, self, cc[0], cc[1], rr);
    else schur_pairs_accumulate_mma<8>(d, sp, T, kb, ke, lane, self, cc[0], cc[1], rr);
    const int row = lane >> 2, tig = lane & 3;
    if (part) {
      double* dst = part + c * 72;
#pragma unroll
      for (int i = 0; i < 2; ++i) dst[row * 8 + 2 * tig + i] = (row < dcx && 2 * tig + i < dcy) ? cc[i] : 0.0;
      if (tig == 0) dst[64 + row] = (self && row < dcx) ? rr : 0.0;
      return;
    }
    if (row >= dcx) return;
    if (self && tig == 0) atomic_add_f64(&rhs[d.Wcols[ox0 * d.dcmax + row]], rr);
    double* dst = Bk + ((int64_t)chunk_key[c] * 8 + row) * 8;
#pragma unroll
    for (int i = 0; i < 2; ++i)
      if (2 * tig + i < dcy) atomic_add_f64(dst + 2 * tig + i, cc[i]);
    return;
  }
  const int g = lane >> 3, a = lane & 7;
  double acc[8], racc;
  if constexpr (STAGED == 1) schur_pairs_accumulate_staged<true>(d, sp, T, kb, ke, lane, self, stage_all, acc, racc);
  else if constexpr (STAGED == 2) schur_pairs_accumulate_staged<false>(d, sp, T, kb, ke, lane, self, stage_all, acc, racc);
  else schur_pairs_accumulate(d, sp, T, kb, ke, lane, dcx, dcy, self, acc, racc);
  if (part) {        // fixed-order reduction per key afterwards (det_pair_reduce_kernel): no atomics
    if (g == 0) {
      double* dst = part + c * 72;
#pragma unroll
      for (int b = 0; b < 8; ++b) dst[a * 8 + b] = (a < dcx && b < dcy) ? acc[b] : 0.0;
      dst[64 + a] = (self && a < dcx) ? racc : 0.0;
    }
    return;
  }
  if (self && g == 0 && a < dcx) atomic_add_f64(&rhs[d.Wcols[ox0 * d.dcmax + a]], racc);
  if (g == 0 && a < dcx) {
    double* dst = Bk + ((int64_t)chunk_key[c] * 8 + a) * 8;
#pragma unroll
    for (int b = 0; b < 8; ++b)
      if (b < dcy) atomic_add_f64(dst + b, acc[b]);
  }
}

// diag(J_c^T J_c) of the camera part from the image blocks (shared intrinsics accumulate)
static __global__ void sp_diag_kernel(SparseSchur s, double* diag) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)s.n_images * 8) return;
  const int img = (int)(i >> 3), a = (int)(i & 7);
  const int col = s.img_cols[img * 8 + a];
  if (col >= 0) atomic_add_f64(&diag[col], s.Himg[(int64_t)img * 64 + a * 8 + a]);
}

// q += S_local p  (q zeroed by the caller; D2 is added when add_d2)
static __global__ void __launch_bounds__(256) sp_spmv_kernel(SparseSchur s, const double* __restrict__ D2, const double* __restrict__ p,
                                                             double* __restrict__ q, int add_d2, const CGState* st) {
  if (st && st->done) return;
  const int64_t gid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 3;   // one 8-lane group per block
  const int a = threadIdx.x & 7;
  const unsigned gmask = 0xFFu << (threadIdx.x & 24);
  const int64_t n_blocks = (int64_t)s.n_images + s.n_keys;
  if (gid < n_blocks) {
    if (gid < s.n_images) {
      const int img = (int)gid;
      const int ca = s.img_cols[img * 8 + a];
      const double xa = ca >= 0 ? p[ca] : 0.0;
      const double* H = s.Himg + (int64_t)img * 64;
      double acc = 0.0;
#pragma unroll
      for (int b = 0; b < 8; ++b) {
        const double xb = __shfl_sync(gmask, xa, b, 8);
        acc += (a >= b ? H[a * 8 + b] : H[b * 8 + a]) * xb;        // symmetric, lower stored
      }
      if (ca >= 0) atomic_add_f64(&q[ca], acc);
    } else {
      const int64_t k = gid - s.n_images;
      const int ia = s.key_a[k], ib = s.key_b[k];
      const int ca = s.img_cols[ia * 8 + a], cb = s.img_cols[ib * 8 + a];
      const double xa = ca >= 0 ? p[ca] : 0.0, xb = cb >= 0 ? p[cb] : 0.0;
      const double* B = s.Bk + k * 64;
      double ya = 0.0, yb = 0.0;
#pragma unroll
      for (int b = 0; b < 8; ++b) {
        ya += B[a * 8 + b] * __shfl_sync(gmask, xb, b, 8);           // (B x_b)[a]
        yb += B[b * 8 + a] * __shfl_sync(gmask, xa, b, 8);           // (B^T x_a)[a]
      }
      if (ca >= 0) atomic_add_f64(&q[ca], -ya);
      if (!s.key_self[k] && cb >= 0) atomic_add_f64(&q[cb], -yb);
    }
  }
  if (add_d2) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < s.nc) atomic_add_f64(&q[i], D2[i] * p[i]);
  }
}

// Parameter-block diagonal of S_local into Dblk [nblk][12*12] (zeroed by the caller): pose blocks and camera blocks.
static __global__ void __launch_bounds__(256) sp_blockdiag_kernel(SparseSchur s, double* __restrict__ Dblk) {
  const int64_t gid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 3;
  const int a = threadIdx.x & 7;
  const int64_t n_blocks = (int64_t)s.n_images + s.n_keys;
  if (gid >= n_blocks) return;
  if (gid < s.n_images) {
    const int img = (int)gid;
    const int pd = s.img_pd[img];
    const double* H = s.Himg + (int64_t)img * 64;
    const int pb = s.img_pose_blk[img], cb = s.img_cam_blk[img];
    for (int b = 0; b < 8; ++b) {
      const double v = a >= b ? H[a * 8 + b] : H[b * 8 + a];
      if (s.img_cols[img * 8 + a] < 0 || s.img_cols[img * 8 + b] < 0) continue;
      if (a < pd && b < pd) { if (pb >= 0) atomic_add_f64(&Dblk[(int64_t)pb * 144 + a * 12 + b], v); }
      else if (a >= pd && b >= pd) { if (cb >= 0) atomic_add_f64(&Dblk[(int64_t)cb * 144 + (a - pd) * 12 + (b - pd)], v); }
    }
  } else {
    const int64_t k = gid - s.n_images;
    const int ia = s.key_a[k], ib = s.key_b[k];
    const bool self = s.key_self[k] != 0;
    const int pda = s.img_pd[ia], pdb = s.img_pd[ib];
    const double* B = s.Bk + k * 64;
    const bool same_img = ia == ib;
    const bool same_cam = s.img_cam_blk[ia] >= 0 && s.img_cam_blk[ia] == s.img_cam_blk[ib];
    for (int b = 0; b < 8; ++b) {
      if (s.img_cols[ia * 8 + a] < 0 || s.img_cols[ib * 8 + b] < 0) continue;
      const double v = B[a * 8 + b];
      // pose x pose lands on a diagonal block only for pairs inside one image
      if (a < pda && b < pdb && same_img && s.img_pose_blk[ia] >= 0) {
        double* D = &Dblk[(int64_t)s.img_pose_blk[ia] * 144];
        atomic_add_f64(&D[a * 12 + b], -v);
        if (!self) atomic_add_f64(&D[b * 12 + a], -v);
      }
      if (a >= pda && b >= pdb && same_cam) {
        double* D = &Dblk[(int64_t)s.img_cam_blk[ia] * 144];
        atomic_add_f64(&D[(a - pda) * 12 + (b - pdb)], -v);
        if (!self) atomic_add_f64(&D[(b - pdb) * 12 + (a - pda)], -v);
      }
    }
  }
}

// invert the (damped) diagonal blocks: Dblk + diag(D2) -> Minv rows; same output layout as cg_block_inverse_kernel
static __global__ void sp_block_inverse_kernel(const double* Dblk, const double* D2, int add_d2, const int32_t* blk_off,
                                               const int32_t* blk_dim, int nblk, double* Minv, int* fail) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= nblk) return;
  const int o = blk_off[b], d = blk_dim[b];
  double A[12][24];
  for (int i = 0; i < d; ++i)
    for (int j = 0; j < d; ++j) {
      A[i][j] = Dblk[(int64_t)b * 144 + i * 12 + j] + ((i == j && add_d2) ? D2[o + i] : 0.0);
      A[i][d + j] = i == j ? 1.0 : 0.0;
    }
  for (int k = 0; k < d; ++k) {
    const double pv = A[k][k];
    if (!(pv > 0.0)) { *fail = 1; return; }
    for (int j = 0; j < 2 * d; ++j) A[k][j] /= pv;
    for (int i = 0; i < d; ++i) {
      if (i == k) continue;
      const double f = A[i][k];
      for (int j = 0; j < 2 * d; ++j) A[i][j] -= f * A[k][j];
    }
  }
  for (int i = 0; i < d; ++i)
    for (int j = 0; j < d; ++j) Minv[(int64_t)(o + i) * 12 + j] = A[i][d + j];
}

// rhs = -gc (the Schur part is added by ba_schur_prep_kernel)
static __global__ void sp_init_rhs_kernel(const double* gc, double* rhs, int nc) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nc) rhs[i] = -gc[i];
}

}  // namespace pxr
