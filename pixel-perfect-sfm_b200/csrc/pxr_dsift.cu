// pxr_dsift.cu — dense SIFT descriptors of one grayscale image, straight into the patch-slab layout.
//
// Reference: the `dsift` model (features/models/dsift.py, kornia's DenseSIFTDescriptor with stride 1 and padding 1) and
// FeatureExtractor.tensor_to_fmap (features/extractor.py:176-201).  The reference builds the whole [1, A*S*S, H', W']
// float32 map with nine convolutions, normalises and casts it, copies it to the host and cuts one window per keypoint.
// Here one fused kernel computes only the pixels it is asked for — the keypoints' windows, or every pixel of the map —
// and writes each pixel's C = A*S*S channels as one row of the HWC slab the optimizers read.
//
// The descriptor (I = G / 255, cross-correlations, hb = b / 2):
//   gx = (I(y,x+1) - I(y,x-1)) / 2, gy likewise, replicate borders
//   mag = sqrt(gx^2 + gy^2 + 1e-10), o = A (atan2(gy, gx + 1e-10) + 2 pi) / (2 pi), k = floor(o), w = o - k
//   E_a = [k mod A = a] (1 - w) mag + [(k + 1) mod A = a] w mag                         (zero outside the image)
//   P_a(py,px) = sum_{u,v} t(u) t(v) / hb'^2 E_a(py - hb + u, px - hb + v), t(u) = b/2 - |u + 0.5 - b/2|, hb' = b/2
//                                                                         (py in [0, Hp), Hp = H + 2 hb - b + 1)
//   D[a S^2 + i S + j](y,x) = P_a(y - 1 + i, x - 1 + j), zero outside P; the map is H' = Hp + 3 - S rows
//   v = clamp(D / ||D||, 0, clipval); v /= ||v||; rootsift: v = sqrt(v / |v|_1 + 1e-10); l2_normalize: v /= ||v||
// with every norm taken as max(norm, 1e-12), as torch.nn.functional.normalize does.
//
// One CTA owns a 16 x 16 tile of output pixels.  It stages the tile's image halo (S + b extra rows and columns), builds
// E on it, pools E separably (rows, then columns) into P — all in shared memory, fp32 — and finishes each output pixel
// with one warp: lane l holds channels [l * C/32, (l+1) * C/32), the norms are warp reductions, and the C channels go
// out as one contiguous row.  Dense and sparse mode run the same kernel and differ only in where a tile starts and
// where its rows go, so a window of the slab is bit for bit the same window of the dense map.
#include <cuda_fp16.h>

#include "pxr_internal.h"

namespace pxr {

namespace {

constexpr int kTile = 16;
constexpr int kThreads = 256;

template <typename T> __device__ __forceinline__ T ds_cast(float v);
template <> __device__ __forceinline__ __half ds_cast<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ float ds_cast<float>(float v) { return v; }
template <> __device__ __forceinline__ double ds_cast<double>(float v) { return (double)v; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

struct DsiftArgs {
  const uint8_t* image; int H, W;       // image, row-major
  int b; float clipval; int rootsift, l2_normalize;
  int Hp, Wp;                           // size of the pooled maps P
  int Hm, Wm;                           // size of the descriptor map
  const int32_t* corners;               // sparse: [n][2] (x0, y0) in map coordinates; nullptr: dense
  int ps, tiles_per_side;               // sparse: window size, tiles along one side of a window
  void* out;                            // sparse: [n][ps][ps][C]; dense: [Hm][Wm][C]
};

// shared memory of one CTA, in floats: image halo NI^2, E (later P) A*NE^2, row-pooled A*NE*NP
__host__ __device__ inline int ds_ni(int S, int b) { return kTile + S + b; }
__host__ __device__ inline int ds_ne(int S, int b) { return kTile + S + b - 2; }
__host__ __device__ inline int ds_np(int S) { return kTile + S - 1; }
inline size_t ds_smem_bytes(int A, int S, int b) {
  const size_t ni = ds_ni(S, b), ne = ds_ne(S, b), np = ds_np(S);
  return (ni * ni + (size_t)A * ne * ne + (size_t)A * ne * np) * sizeof(float);
}

template <int A, int S, typename TO>
__global__ void __launch_bounds__(kThreads) dsift_kernel(DsiftArgs a) {
  constexpr int C = A * S * S;
  constexpr int CPL = C >= 32 ? C / 32 : 1;           // channels per lane
  extern __shared__ float smem[];
  const int b = a.b, hb = b / 2;
  const int NI = ds_ni(S, b), NE = ds_ne(S, b), NP = ds_np(S);
  float* sI = smem;                                   // [NI][NI]
  float* sE = sI + NI * NI;                           // [A][NE][NE], reused as P [A][NP][NP]
  float* sR = sE + A * NE * NE;                       // [A][NE][NP]

  // the tile's first output pixel (map coordinates) and, in sparse mode, its window
  int64_t win = 0;
  int y0, x0;
  if (a.corners) {
    const int t = blockIdx.x % (a.tiles_per_side * a.tiles_per_side);
    win = blockIdx.x / (a.tiles_per_side * a.tiles_per_side);
    y0 = a.corners[2 * win + 1] + (t / a.tiles_per_side) * kTile;
    x0 = a.corners[2 * win] + (t % a.tiles_per_side) * kTile;
  } else {
    y0 = blockIdx.y * kTile;
    x0 = blockIdx.x * kTile;
  }
  const int py0 = y0 - 1, px0 = x0 - 1;               // first P row / column the tile reads
  const int ey0 = py0 - hb, ex0 = px0 - hb;           // first E row / column
  const int iy0 = ey0 - 1, ix0 = ex0 - 1;             // first image row / column (gradient stencil)

  for (int k = threadIdx.x; k < NI * NI; k += kThreads) {
    const int r = k / NI, c = k % NI;
    const int y = min(max(iy0 + r, 0), a.H - 1), x = min(max(ix0 + c, 0), a.W - 1);   // replicate border
    sI[k] = (float)__ldg(a.image + (int64_t)y * a.W + x) / 255.f;
  }
  __syncthreads();

  const float two_pi = 6.283185307179586f;
  for (int k = threadIdx.x; k < NE * NE; k += kThreads) {
    const int r = k / NE, c = k % NE;
    const int ey = ey0 + r, ex = ex0 + c;
    float e[A];
#pragma unroll
    for (int q = 0; q < A; ++q) e[q] = 0.f;
    if (ey >= 0 && ey < a.H && ex >= 0 && ex < a.W) {
      const float* row = sI + (r + 1) * NI + (c + 1);
      const float gx = 0.5f * (row[1] - row[-1]);
      const float gy = 0.5f * (row[NI] - row[-NI]);
      const float mag = sqrtf(gx * gx + gy * gy + 1e-10f);
      const float o = (float)A * (atan2f(gy, gx + 1e-10f) + two_pi) / two_pi;
      const float fk = floorf(o), w = o - fk;
      const int b0 = ((int)fk) % A, b1 = (b0 + 1) % A;
#pragma unroll
      for (int q = 0; q < A; ++q) e[q] = (q == b0 ? (1.f - w) * mag : 0.f) + (q == b1 ? w * mag : 0.f);
    }
#pragma unroll
    for (int q = 0; q < A; ++q) sE[q * NE * NE + k] = e[q];
  }
  __syncthreads();

  // triangular weights t(u) and the 1 / (b/2)^2 of the kernel
  const float half_b = 0.5f * (float)b, knorm = 1.f / (half_b * half_b);
  for (int k = threadIdx.x; k < A * NE * NP; k += kThreads) {
    const int q = k / (NE * NP), rc = k % (NE * NP), r = rc / NP, c = rc % NP;
    const float* src = sE + q * NE * NE + r * NE + c;
    float s = 0.f;
    for (int v = 0; v < b; ++v) s += (half_b - fabsf((float)v + 0.5f - half_b)) * src[v];
    sR[k] = s;
  }
  __syncthreads();
  for (int k = threadIdx.x; k < A * NP * NP; k += kThreads) {
    const int q = k / (NP * NP), rc = k % (NP * NP), r = rc / NP, c = rc % NP;
    const int py = py0 + r, px = px0 + c;
    float s = 0.f;
    if (py >= 0 && py < a.Hp && px >= 0 && px < a.Wp) {
      const float* src = sR + q * NE * NP + r * NP + c;
      for (int u = 0; u < b; ++u) s += (half_b - fabsf((float)u + 0.5f - half_b)) * src[u * NP];
      s *= knorm;
    }
    sE[k] = s;                                        // P [A][NP][NP]
  }
  __syncthreads();

  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int limit_y = a.corners ? a.ps : a.Hm, limit_x = a.corners ? a.ps : a.Wm;
  const int oy = a.corners ? y0 - a.corners[2 * win + 1] : y0;   // tile origin inside the window / map
  const int ox = a.corners ? x0 - a.corners[2 * win] : x0;
  for (int p = warp; p < kTile * kTile; p += kThreads / 32) {
    const int ty = p / kTile, tx = p % kTile;
    if (oy + ty >= limit_y || ox + tx >= limit_x) continue;       // warp-uniform
    float v[CPL];
    float sq = 0.f;
#pragma unroll
    for (int j = 0; j < CPL; ++j) {
      const int ch = lane * CPL + j;
      float d = 0.f;
      if (ch < C) {
        const int q = ch / (S * S), i = (ch / S) % S, jj = ch % S;
        d = sE[q * NP * NP + (ty + i) * NP + (tx + jj)];
      }
      v[j] = d;
      sq += d * d;
    }
    float n = fmaxf(sqrtf(warp_sum(sq)), 1e-12f);
    sq = 0.f;
#pragma unroll
    for (int j = 0; j < CPL; ++j) { v[j] = fminf(fmaxf(v[j] / n, 0.f), a.clipval); sq += v[j] * v[j]; }
    n = fmaxf(sqrtf(warp_sum(sq)), 1e-12f);
    float s1 = 0.f;
#pragma unroll
    for (int j = 0; j < CPL; ++j) { v[j] = v[j] / n; s1 += v[j]; }
    if (a.rootsift) {
      n = fmaxf(warp_sum(s1), 1e-12f);
#pragma unroll
      for (int j = 0; j < CPL; ++j) v[j] = sqrtf(v[j] / n + 1e-10f);
    }
    if (a.l2_normalize) {
      sq = 0.f;
#pragma unroll
      for (int j = 0; j < CPL; ++j) sq += (lane * CPL + j < C) ? v[j] * v[j] : 0.f;
      n = fmaxf(sqrtf(warp_sum(sq)), 1e-12f);
#pragma unroll
      for (int j = 0; j < CPL; ++j) v[j] = v[j] / n;
    }
    const int64_t pix = a.corners ? (win * a.ps + oy + ty) * a.ps + (ox + tx) : (int64_t)(oy + ty) * a.Wm + (ox + tx);
    TO* dst = reinterpret_cast<TO*>(a.out) + pix * C;
#pragma unroll
    for (int j = 0; j < CPL; ++j)
      if (lane * CPL + j < C) dst[lane * CPL + j] = ds_cast<TO>(v[j]);
  }
}

template <int A, int S>
int launch_dsift(pxr_ctx* ctx, const DsiftArgs& a, int64_t n, int out_dtype) {
  dim3 grid;
  if (a.corners) grid = dim3((unsigned)(n * a.tiles_per_side * a.tiles_per_side));
  else grid = dim3((unsigned)cdiv(a.Wm, kTile), (unsigned)cdiv(a.Hm, kTile));
  const size_t smem = ds_smem_bytes(A, S, a.b);
  if (out_dtype == PXR_F16) PXR_LAUNCH(ctx, (dsift_kernel<A, S, __half>), grid, kThreads, smem, a);
  else if (out_dtype == PXR_F32) PXR_LAUNCH(ctx, (dsift_kernel<A, S, float>), grid, kThreads, smem, a);
  else PXR_LAUNCH(ctx, (dsift_kernel<A, S, double>), grid, kThreads, smem, a);
  PXR_CUDA(cudaGetLastError());
  return PXR_OK;
}

}  // namespace

}  // namespace pxr

using namespace pxr;

extern "C" int pxr_dsift(pxr_ctx* ctx, const uint8_t* image, int32_t image_on_device, int32_t height, int32_t width,
                         int32_t num_ang_bins, int32_t num_spatial_bins, int32_t spatial_bin_size, float clipval,
                         int32_t rootsift, int32_t l2_normalize, const int32_t* corners, int64_t n_patches,
                         int32_t patch_size, int32_t out_dtype, void* out_host, void** out_device) {
  const int A = num_ang_bins, S = num_spatial_bins, b = spatial_bin_size;
  if (!ctx || !image || (!out_host && !out_device)) return fail(PXR_ERR_INVALID_ARGUMENT, "NULL argument");
  if (out_device) *out_device = nullptr;
  if ((A != 4 && A != 8) || (S != 2 && S != 4) || b < 1 || b > 8)
    return fail(PXR_ERR_UNSUPPORTED, "dense SIFT supports num_ang_bins 4 or 8, num_spatial_bins 2 or 4 and "
                "spatial_bin_size 1..8 (got %d, %d, %d)", A, S, b);
  if (out_dtype < PXR_F16 || out_dtype > PXR_F64) return fail(PXR_ERR_INVALID_ARGUMENT, "bad dtype");
  if (!(clipval > 0.f)) return fail(PXR_ERR_INVALID_ARGUMENT, "clipval must be positive (got %g)", (double)clipval);
  const int Hm = height + 2 * (b / 2) - b + 1 + 3 - S, Wm = width + 2 * (b / 2) - b + 1 + 3 - S;
  if (height < 1 || width < 1 || Hm < 1 || Wm < 1)
    return fail(PXR_ERR_INVALID_ARGUMENT, "image %d x %d gives an empty descriptor map", width, height);
  if (corners) {
    if (n_patches < 0 || patch_size < 1 || patch_size > Hm || patch_size > Wm)
      return fail(PXR_ERR_INVALID_ARGUMENT, "bad window size %d for a %d x %d map", patch_size, Wm, Hm);
    for (int64_t k = 0; k < n_patches; ++k)
      if (corners[2 * k] < 0 || corners[2 * k + 1] < 0 || corners[2 * k] + patch_size > Wm ||
          corners[2 * k + 1] + patch_size > Hm)
        return fail(PXR_ERR_INVALID_ARGUMENT, "window %lld leaves the %d x %d map (corner %d,%d)", (long long)k, Wm, Hm,
                    corners[2 * k], corners[2 * k + 1]);
    const int64_t tiles = (int64_t)cdiv(patch_size, kTile) * cdiv(patch_size, kTile);
    if (n_patches * tiles > 0x7fffffffLL) return fail(PXR_ERR_INVALID_ARGUMENT, "too many windows in one call");
  }
  const int C = A * S * S;
  const size_t osz = out_dtype == PXR_F16 ? 2 : (out_dtype == PXR_F32 ? 4 : 8);
  const int64_t rows = corners ? n_patches * patch_size * patch_size : (int64_t)Hm * Wm;
  const size_t out_bytes = (size_t)rows * C * osz;
  if (rows == 0) return PXR_OK;

  PXR_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  DevBuf<uint8_t> d_image;
  DevBuf<int32_t> d_corners;
  DsiftArgs a;
  a.image = image;
  if (!image_on_device) {
    PXR_TRY(d_image.upload(image, (size_t)height * width, s));
    a.image = d_image.p;
  }
  if (corners) PXR_TRY(d_corners.upload(corners, (size_t)n_patches * 2, s));
  uint8_t* d_out = nullptr;
  PXR_CUDA(cudaMalloc((void**)&d_out, out_bytes));
  a.H = height; a.W = width; a.b = b; a.clipval = clipval; a.rootsift = rootsift != 0; a.l2_normalize = l2_normalize != 0;
  a.Hp = height + 2 * (b / 2) - b + 1; a.Wp = width + 2 * (b / 2) - b + 1; a.Hm = Hm; a.Wm = Wm;
  a.corners = d_corners.p; a.ps = patch_size; a.tiles_per_side = corners ? (int)cdiv(patch_size, kTile) : 0;
  a.out = d_out;
  int rc;
  if (A == 4 && S == 2) rc = launch_dsift<4, 2>(ctx, a, n_patches, out_dtype);
  else if (A == 4) rc = launch_dsift<4, 4>(ctx, a, n_patches, out_dtype);
  else if (S == 2) rc = launch_dsift<8, 2>(ctx, a, n_patches, out_dtype);
  else rc = launch_dsift<8, 4>(ctx, a, n_patches, out_dtype);
  if (rc == PXR_OK && out_host) {
    const cudaError_t e = cudaMemcpyAsync(out_host, d_out, out_bytes, cudaMemcpyDeviceToHost, s);
    if (e != cudaSuccess) rc = fail(PXR_ERR_CUDA, "cudaMemcpyAsync failed: %s", cudaGetErrorString(e));
  }
  if (rc == PXR_OK) {
    const cudaError_t e = cudaStreamSynchronize(s);      // the staged image and corners are locals of this call
    if (e != cudaSuccess) rc = fail(PXR_ERR_CUDA, "dsift failed: %s", cudaGetErrorString(e));
  }
  if (rc == PXR_OK && out_device) *out_device = d_out;
  else cudaFree(d_out);
  return rc;
}
