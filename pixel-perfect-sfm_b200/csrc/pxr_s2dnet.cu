// pxr_s2dnet.cu — S2DNet features (num_layers 1) of one RGB image, straight into the patch-slab layout.
//
// Reference: the `s2dnet` model (features/models/s2dnet.py with num_layers 1: VGG16's conv1_1 / ReLU / conv1_2 / ReLU,
// then the adaptation layer 1x1 conv / ReLU / 5x5 conv / BatchNorm) and FeatureExtractor.tensor_to_fmap.  The reference
// runs the four convolutions through cuDNN over the whole image, keeps three 64-channel and one 128-channel fp32 map at
// full resolution, then normalises, casts and cuts one window per keypoint.  Here one fused kernel computes only the
// pixels it is asked for — the keypoints' windows, or every pixel of the map — and writes each pixel's 128 channels as
// one row of the HWC slab the optimizers read.  No intermediate map goes to global memory.
//
// The network (every convolution pads its own input with zeros, so every intermediate outside the image is 0):
//   x  = (u8 / 255 - mean) / std                                     (fp32, ImageNet mean / std, not folded)
//   a1 = relu(conv3x3(x; 3 -> 64))                                   CUDA cores, fp32, stored fp16
//   a2 = relu(conv3x3(a1; 64 -> 64))                                 tensor cores (fp16 x fp16 -> fp32), stored fp16
//   a3 = relu(conv1x1(a2; 64 -> 64))                                 tensor cores, stored fp16
//   f  = conv5x5(a3; 64 -> 128) with the eval-mode BatchNorm folded in (host, fp64); no ReLU
//   out = f / max(||f||, 1e-12) when l2_normalize, then cast
//
// One CTA owns a 16 x 16 tile of output pixels.  It stages the 24 x 24 image halo, computes a1 on the 22 x 22 halo, a2
// and a3 on the 20 x 20 halo and f on the tile, all in shared memory ([pixel][64] fp16 rows padded to 72 halves, so the
// ldmatrix row gathers are free of bank conflicts).  The three tensor-core layers are implicit GEMMs with mma.sync
// m16n8k16: A rows are gathered by ldmatrix from the shifted activation tile, B is the layer's weights for one tap,
// pre-arranged on the host in the mma fragment order (one 16-byte load per lane per pair of n-fragments).  The taps
// stream through a two-slot shared-memory ring by bulk copy (cp.async.bulk) on an mbarrier each; the weights (0.47 MB)
// stay in L2 across CTAs.  Every intermediate pixel is computed from the same operands in the same K order whatever the
// tile's origin, so a window of the slab is bit for bit the same window of the dense map.
//
// A stored fp16 intermediate that is not finite (fp16 tops out at 65504) raises a device flag; the call then fails with
// PXR_ERR_NUMERIC instead of returning features.
#include <cuda_fp16.h>

#include <cmath>
#include <vector>

#include "pxr_device.cuh"
#include "pxr_internal.h"

struct pxr_s2dnet_weights {
  int device = 0;
  void* d = nullptr;       // kFloats fp32 (w1 in [co][ky][kx][ci] order, b1, b2, b3, b4), then the packed taps
};

namespace pxr {

namespace {

constexpr int kTile = 16;
constexpr int kThreads = 256;
constexpr int kLd = 72;                         // halves per pixel row of an activation tile (64 + 8 against conflicts)
constexpr int kRI = kTile + 8, kR1 = kTile + 6, kR2 = kTile + 4;   // image, a1 and a2 / a3 regions
constexpr int kTaps2 = 9, kTaps3 = 1, kTaps4 = 25, kTaps = kTaps2 + kTaps3 + kTaps4;
constexpr int kTapSmall = 4 * 4 * 32 * 16;      // one tap of a 64 -> 64 layer in fragment order: 8 KB
constexpr int kTapLarge = 4 * 8 * 32 * 16;      // one tap of the 64 -> 128 layer: 16 KB
constexpr int kW1 = 64 * 27;
constexpr int kFloats = kW1 + 64 + 64 + 64 + 128;                  // 2048: w1 and the four biases
constexpr int64_t kPackedBytes = (int64_t)(kTaps2 + kTaps3) * kTapSmall + (int64_t)kTaps4 * kTapLarge;
constexpr int64_t kInputFloats = 64 * 27 + 64 + 64 * 64 * 9 + 64 + 64 * 64 + 64 + 128 * 64 * 25 + 128;

// shared memory, bytes
constexpr int kOffBar = 0;
constexpr int kOffWB = 128;                                        // two tap slots
constexpr int kOffA1 = kOffWB + 2 * kTapLarge;                     // a1 [484][kLd], later a3 [400][kLd]
constexpr int kOffA2 = kOffA1 + kR1 * kR1 * kLd * 2;               // a2 [400][kLd]
constexpr int kOffX = kOffA2 + kR2 * kR2 * kLd * 2;                // x [24][24][3] fp32
constexpr int kOffW1 = kOffX + kRI * kRI * 3 * 4;                  // w1 and biases, kFloats fp32
constexpr int kOffNrm = kOffW1 + kFloats * 4;                      // per-pixel sum of squares of each half of f
constexpr int kSmem = kOffNrm + 2 * kTile * kTile * 4;

template <typename T> __device__ __forceinline__ void s2_store2(T* dst, float a, float b);
template <> __device__ __forceinline__ void s2_store2<__half>(__half* dst, float a, float b) {
  *reinterpret_cast<__half2*>(dst) = __floats2half2_rn(a, b);
}
template <> __device__ __forceinline__ void s2_store2<float>(float* dst, float a, float b) {
  *reinterpret_cast<float2*>(dst) = make_float2(a, b);
}
template <> __device__ __forceinline__ void s2_store2<double>(double* dst, float a, float b) {
  *reinterpret_cast<double2*>(dst) = make_double2((double)a, (double)b);
}

struct S2dArgs {
  const uint8_t* image; int H, W;      // [H][W][3]
  const float* params;                 // kFloats fp32
  const uint8_t* taps;                 // kTaps taps in fragment order
  const int32_t* corners;              // sparse: [n][2] (x0, y0); nullptr: dense
  int ps, tiles_per_side;
  int l2_normalize;
  void* out;                           // sparse: [n][ps][ps][128]; dense: [H][W][128]
  int* bad;                            // set to 1 when a stored intermediate is not finite
};

__device__ __forceinline__ uint32_t tap_bytes(int g) { return g < kTaps2 + kTaps3 ? kTapSmall : kTapLarge; }
__device__ __forceinline__ const uint8_t* tap_src(const uint8_t* taps, int g) {
  return g < kTaps2 + kTaps3 ? taps + (int64_t)g * kTapSmall
                             : taps + (int64_t)(kTaps2 + kTaps3) * kTapSmall + (int64_t)(g - kTaps2 - kTaps3) * kTapLarge;
}

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// One implicit-GEMM layer over `KW` x `KW` taps for one warp: up to four m-tiles (mt0, mt0 + mt_step, ...; those at or
// past n_mt are skipped) of a `wout`-wide output region, eight n-fragments starting at pair np0 of an NP-pair tap.  The
// input tile `in` is `win` = wout + KW - 1 pixels wide.  Tap g0 + t of the weight stream sits in slot (g0 + t) & 1; tap
// g0 is already in flight, and each tap issues the next one of the stream (up to kTaps) once every warp is done with
// the slot it overwrites.
template <int KW, int NP>
__device__ __forceinline__ void conv_layer(float (&acc)[4][8][4], const __half* in, int win, int wout, int mt0, int mt_step,
                                           int n_mt, int np0, int g0, uint8_t* slots, uint64_t* bars, const uint8_t* taps) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int f = 0; f < 8; ++f)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[i][f][e] = 0.f;
  uint32_t a_addr[4];
  bool valid[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int mt = mt0 + i * mt_step;
    valid[i] = mt < n_mt;
    const int m = (valid[i] ? mt : 0) * 16 + (lane & 15);
    a_addr[i] = smem_u32(in + ((m / wout) * win + (m % wout)) * kLd + (lane >> 4) * 8);
  }
  for (int t = 0; t < KW * KW; ++t) {
    const int g = g0 + t;
    if (threadIdx.x == 0 && g + 1 < kTaps) {
      uint64_t* bar = bars + ((g + 1) & 1);
      mbar_expect_tx(bar, tap_bytes(g + 1));
      bulk_g2s(slots + ((g + 1) & 1) * kTapLarge, tap_src(taps, g + 1), tap_bytes(g + 1), bar);
    }
    mbar_wait(bars + (g & 1), (g >> 1) & 1);
    const uint4* wb = reinterpret_cast<const uint4*>(slots + (g & 1) * kTapLarge);
    const uint32_t shift = (uint32_t)(((t / KW) * win + (t % KW)) * kLd * 2);
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      uint4 b[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = wb[(ks * NP + np0 + j) * 32 + lane];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (!valid[i]) continue;                                   // warp-uniform
        uint32_t a[4];
        ldsm_x4(a_addr[i] + shift + ks * 32, a[0], a[1], a[2], a[3]);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          mma16816(acc[i][2 * j], a, b[j].x, b[j].y);
          mma16816(acc[i][2 * j + 1], a, b[j].z, b[j].w);
        }
      }
    }
    __syncthreads();                                               // the slot is free for tap g + 2
  }
}

// bias, ReLU and the zero padding of a 64-channel layer on the 20 x 20 region whose pixel (0, 0) is image pixel (gy0, gx0)
__device__ __forceinline__ bool store_hidden(const float (&acc)[4][8][4], __half* out, const float* bias, int mt0, int mt_step,
                                             int n_mt, int gy0, int gx0, int H, int W) {
  const int lane = threadIdx.x & 31;
  bool bad = false;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int mt = mt0 + i * mt_step;
    if (mt >= n_mt) continue;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = mt * 16 + (lane >> 2) + 8 * h;
      const int gy = gy0 + m / kR2, gx = gx0 + m % kR2;
      const bool inside = gy >= 0 && gy < H && gx >= 0 && gx < W;
#pragma unroll
      for (int f = 0; f < 8; ++f) {
        const int n = f * 8 + 2 * (lane & 3);
        const float v0 = inside ? fmaxf(acc[i][f][2 * h] + bias[n], 0.f) : 0.f;
        const float v1 = inside ? fmaxf(acc[i][f][2 * h + 1] + bias[n + 1], 0.f) : 0.f;
        const __half2 hv = __floats2half2_rn(v0, v1);
        bad |= !(isfinite(__low2float(hv)) && isfinite(__high2float(hv)));
        *reinterpret_cast<__half2*>(out + m * kLd + n) = hv;
      }
    }
  }
  return bad;
}

template <typename TO>
__global__ void __launch_bounds__(kThreads, 1) s2dnet_kernel(S2dArgs a) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kOffBar);
  uint8_t* slots = smem + kOffWB;
  __half* sA1 = reinterpret_cast<__half*>(smem + kOffA1);
  __half* sA2 = reinterpret_cast<__half*>(smem + kOffA2);
  float* sX = reinterpret_cast<float*>(smem + kOffX);
  float* sP = reinterpret_cast<float*>(smem + kOffW1);
  float* sNrm = reinterpret_cast<float*>(smem + kOffNrm);
  const float* b1 = sP + kW1;
  const float* b2 = b1 + 64;
  const float* b3 = b2 + 64;
  const float* b4 = b3 + 64;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  if (tid == 0) {
    mbar_init(bars, 1);
    mbar_init(bars + 1, 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (tid == 0) {                                                  // tap 0 loads while a1 is computed
    mbar_expect_tx(bars, tap_bytes(0));
    bulk_g2s(slots, tap_src(a.taps, 0), tap_bytes(0), bars);
  }

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

  for (int k = tid; k < kRI * kRI * 3; k += kThreads) {
    const int q = k / 3, ci = k % 3;
    const float mean = ci == 0 ? 0.485f : (ci == 1 ? 0.456f : 0.406f);
    const float stdv = ci == 0 ? 0.229f : (ci == 1 ? 0.224f : 0.225f);
    const int gy = y0 - 4 + q / kRI, gx = x0 - 4 + q % kRI;
    float v = 0.f;                                                 // conv1_1 pads the NORMALISED image with zeros
    if (gy >= 0 && gy < a.H && gx >= 0 && gx < a.W)
      v = ((float)__ldg(a.image + ((int64_t)gy * a.W + gx) * 3 + ci) / 255.f - mean) / stdv;
    sX[k] = v;
  }
  for (int k = tid; k < kFloats; k += kThreads) sP[k] = __ldg(a.params + k);
  __syncthreads();

  bool bad = false;
  // a1 on the 22 x 22 region at (y0 - 3, x0 - 3): one item is one pixel and 8 channels, fp32 in a fixed K order
  for (int it = tid; it < 8 * kR1 * kR1; it += kThreads) {
    const int cg = it / (kR1 * kR1), p = it % (kR1 * kR1);
    const int r = p / kR1, c = p % kR1;
    const int gy = y0 - 3 + r, gx = x0 - 3 + c;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = 0.f;
    if (gy >= 0 && gy < a.H && gx >= 0 && gx < a.W) {
      const float* w = sP + cg * 8 * 27;
#pragma unroll
      for (int ky = 0; ky < 3; ++ky)
#pragma unroll
        for (int kx = 0; kx < 3; ++kx)
#pragma unroll
          for (int ci = 0; ci < 3; ++ci) {
            const float x = sX[((r + ky) * kRI + c + kx) * 3 + ci];
            const int k = (ky * 3 + kx) * 3 + ci;
#pragma unroll
            for (int j = 0; j < 8; ++j) v[j] = fmaf(x, w[j * 27 + k], v[j]);
          }
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = fmaxf(v[j] + b1[cg * 8 + j], 0.f);
    }
    uint32_t h[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const __half2 hv = __floats2half2_rn(v[2 * j], v[2 * j + 1]);
      bad |= !(isfinite(__low2float(hv)) && isfinite(__high2float(hv)));
      h[j] = *reinterpret_cast<const uint32_t*>(&hv);
    }
    *reinterpret_cast<uint4*>(sA1 + p * kLd + cg * 8) = make_uint4(h[0], h[1], h[2], h[3]);
  }
  __syncthreads();

  float acc[4][8][4];
  constexpr int kMt2 = kR2 * kR2 / 16;                             // 25 m-tiles of the 20 x 20 region
  // a2 = relu(conv1_2(a1)) on the 20 x 20 region at (y0 - 2, x0 - 2); warp w takes m-tiles w, w + 8, w + 16, w + 24
  conv_layer<3, 4>(acc, sA1, kR1, kR2, warp, 8, kMt2, 0, 0, slots, bars, a.taps);
  bad |= store_hidden(acc, sA2, b2, warp, 8, kMt2, y0 - 2, x0 - 2, a.H, a.W);
  __syncthreads();
  // a3 = relu(conv1x1(a2)), into a1's place
  conv_layer<1, 4>(acc, sA2, kR2, kR2, warp, 8, kMt2, 0, kTaps2, slots, bars, a.taps);
  bad |= store_hidden(acc, sA1, b3, warp, 8, kMt2, y0 - 2, x0 - 2, a.H, a.W);
  __syncthreads();
  // f = conv5x5(a3) + folded BatchNorm on the tile: warp w takes rows (w & 3) + 4i and channels 64 (w >> 2) ..
  const int mg = warp & 3, nh = warp >> 2;
  conv_layer<5, 8>(acc, sA1, kR2, kTile, mg, 4, kTile, nh * 4, kTaps2 + kTaps3, slots, bars, a.taps);

  // epilogue: bias, the 128-channel norm (each half's sum of squares over a lane quad, the halves added in a fixed
  // order), cast, one contiguous row per pixel
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float s = 0.f;
#pragma unroll
      for (int f = 0; f < 8; ++f) {
        const int n = nh * 64 + f * 8 + 2 * (lane & 3);
        acc[i][f][2 * h] += b4[n];
        acc[i][f][2 * h + 1] += b4[n + 1];
        s += acc[i][f][2 * h] * acc[i][f][2 * h] + acc[i][f][2 * h + 1] * acc[i][f][2 * h + 1];
      }
      s += __shfl_xor_sync(0xffffffffu, s, 1);
      s += __shfl_xor_sync(0xffffffffu, s, 2);
      if ((lane & 3) == 0) sNrm[nh * kTile * kTile + (mg + 4 * i) * 16 + (lane >> 2) + 8 * h] = s;
    }
  __syncthreads();

  const int limit_y = a.corners ? a.ps : a.H, limit_x = a.corners ? a.ps : a.W;
  const int oy = a.corners ? y0 - a.corners[2 * win + 1] : y0;    // tile origin inside the window / map
  const int ox = a.corners ? x0 - a.corners[2 * win] : x0;
  TO* out = reinterpret_cast<TO*>(a.out);
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int ty = mg + 4 * i, tx = (lane >> 2) + 8 * h, m = ty * 16 + tx;
      const float sq = sNrm[m] + sNrm[kTile * kTile + m];
      bad |= !isfinite(sq);
      if (oy + ty >= limit_y || ox + tx >= limit_x) continue;
      const float nrm = a.l2_normalize ? fmaxf(sqrtf(sq), 1e-12f) : 1.f;
      const int64_t pix = a.corners ? (win * a.ps + oy + ty) * a.ps + (ox + tx) : (int64_t)(oy + ty) * a.W + (ox + tx);
      TO* dst = out + pix * 128 + nh * 64 + 2 * (lane & 3);
#pragma unroll
      for (int f = 0; f < 8; ++f) {
        float v0 = acc[i][f][2 * h], v1 = acc[i][f][2 * h + 1];
        if (a.l2_normalize) { v0 = v0 / nrm; v1 = v1 / nrm; }
        s2_store2<TO>(dst + f * 8, v0, v1);
      }
    }
  if (bad) *a.bad = 1;                                             // a status flag, every writer stores the same value
}

// the packed fragment order of one layer: tap t, k-step ks (16 input channels), n-pair np (16 output channels), lane;
// lane l holds, for n-fragments 2 np and 2 np + 1, the B values at k = 2 (l % 4) + {0, 1} and k + 8, column l / 4
void pack_taps(const float* w, int cout, int kw, std::vector<__half>& dst) {
  const int np_count = cout / 16;
  for (int t = 0; t < kw * kw; ++t)
    for (int ks = 0; ks < 4; ++ks)
      for (int np = 0; np < np_count; ++np)
        for (int lane = 0; lane < 32; ++lane)
          for (int fr = 0; fr < 2; ++fr)
            for (int reg = 0; reg < 2; ++reg)
              for (int e = 0; e < 2; ++e) {
                const int n = (2 * np + fr) * 8 + lane / 4;
                const int ci = ks * 16 + 2 * (lane % 4) + e + 8 * reg;
                dst.push_back(__float2half_rn(w[((size_t)n * 64 + ci) * kw * kw + t]));
              }
}

template <typename TO>
int launch_s2dnet(pxr_ctx* ctx, dim3 grid, const S2dArgs& a) {
  PXR_CUDA(cudaFuncSetAttribute(s2dnet_kernel<TO>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));
  PXR_LAUNCH(ctx, s2dnet_kernel<TO>, grid, kThreads, kSmem, a);
  PXR_CUDA(cudaGetLastError());
  return PXR_OK;
}

}  // namespace

}  // namespace pxr

using namespace pxr;

extern "C" int pxr_s2dnet_weights_create(pxr_ctx* ctx, const float* packed, int64_t n_floats, pxr_s2dnet_weights** out) {
  if (!packed || !out) return fail(PXR_ERR_INVALID_ARGUMENT, "NULL argument");
  *out = nullptr;
  if (n_floats != kInputFloats)
    return fail(PXR_ERR_INVALID_ARGUMENT, "S2DNet weights are %lld floats (got %lld)", (long long)kInputFloats,
                (long long)n_floats);
  for (int64_t k = 0; k < n_floats; ++k)
    if (!std::isfinite(packed[k])) return fail(PXR_ERR_INVALID_ARGUMENT, "S2DNet weight %lld is not finite", (long long)k);
  const float* w1 = packed;
  const float* b1 = w1 + 64 * 27;
  const float* w2 = b1 + 64;
  const float* b2 = w2 + 64 * 64 * 9;
  const float* w3 = b2 + 64;
  const float* b3 = w3 + 64 * 64;
  const float* w4 = b3 + 64;
  const float* b4 = w4 + 128 * 64 * 25;
  const float* fp16_parts[3][2] = {{w2, b2}, {w3, b3}, {w4, b4}};   // the tensor-core layers' weights become fp16
  for (const auto& part : fp16_parts)
    for (const float* p = part[0]; p < part[1]; ++p)
      if (std::fabs(*p) > 65504.f)
        return fail(PXR_ERR_INVALID_ARGUMENT, "S2DNet weight %g is outside the fp16 range", (double)*p);
  if (!ctx) return fail(PXR_ERR_INVALID_ARGUMENT, "NULL context");
  std::vector<float> params;
  params.reserve(kFloats);
  for (int co = 0; co < 64; ++co)                                  // [co][ci][ky][kx] -> [co][ky][kx][ci]
    for (int k = 0; k < 9; ++k)
      for (int ci = 0; ci < 3; ++ci) params.push_back(w1[(co * 3 + ci) * 9 + k]);
  params.insert(params.end(), b1, b1 + 64);
  params.insert(params.end(), b2, b2 + 64);
  params.insert(params.end(), b3, b3 + 64);
  params.insert(params.end(), b4, b4 + 128);
  std::vector<__half> taps;
  taps.reserve(kPackedBytes / 2);
  pack_taps(w2, 64, 3, taps);
  pack_taps(w3, 64, 1, taps);
  pack_taps(w4, 128, 5, taps);
  if ((int64_t)taps.size() * 2 != kPackedBytes) return fail(PXR_ERR_INTERNAL, "S2DNet tap packing");

  PXR_CUDA(cudaSetDevice(ctx->device));
  pxr_s2dnet_weights* wts = new pxr_s2dnet_weights;
  wts->device = ctx->device;
  cudaError_t e = cudaMalloc(&wts->d, kFloats * 4 + kPackedBytes);
  if (e == cudaSuccess) e = cudaMemcpy(wts->d, params.data(), kFloats * 4, cudaMemcpyHostToDevice);
  if (e == cudaSuccess)
    e = cudaMemcpy((uint8_t*)wts->d + kFloats * 4, taps.data(), kPackedBytes, cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    if (wts->d) cudaFree(wts->d);
    delete wts;
    return fail(PXR_ERR_CUDA, "S2DNet weight upload failed: %s", cudaGetErrorString(e));
  }
  *out = wts;
  return PXR_OK;
}

extern "C" void pxr_s2dnet_weights_destroy(pxr_s2dnet_weights* weights) {
  if (!weights) return;
  if (weights->d) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaSetDevice(weights->device);
    cudaFree(weights->d);
    cudaSetDevice(dev);
  }
  delete weights;
}

extern "C" int pxr_s2dnet(pxr_ctx* ctx, const pxr_s2dnet_weights* weights, const uint8_t* image, int32_t image_on_device,
                          int32_t height, int32_t width, const int32_t* corners, int64_t n_patches, int32_t patch_size,
                          int32_t l2_normalize, int32_t out_dtype, void* out_host, void** out_device) {
  if (!image || (!out_host && !out_device)) return fail(PXR_ERR_INVALID_ARGUMENT, "NULL argument");
  if (out_device) *out_device = nullptr;
  if (out_dtype < PXR_F16 || out_dtype > PXR_F64) return fail(PXR_ERR_INVALID_ARGUMENT, "bad dtype");
  if (height < 1 || width < 1) return fail(PXR_ERR_INVALID_ARGUMENT, "empty image %d x %d", width, height);
  if (!corners && (cdiv(width, kTile) > 0x7fffffffLL || cdiv(height, kTile) > 65535))
    return fail(PXR_ERR_INVALID_ARGUMENT, "image %d x %d exceeds the grid", width, height);
  if (corners) {
    if (n_patches < 0 || patch_size < 1 || patch_size > height || patch_size > width)
      return fail(PXR_ERR_INVALID_ARGUMENT, "bad window size %d for a %d x %d map", patch_size, width, height);
    for (int64_t k = 0; k < n_patches; ++k)
      if (corners[2 * k] < 0 || corners[2 * k + 1] < 0 || corners[2 * k] + patch_size > width ||
          corners[2 * k + 1] + patch_size > height)
        return fail(PXR_ERR_INVALID_ARGUMENT, "window %lld leaves the %d x %d map (corner %d,%d)", (long long)k, width,
                    height, corners[2 * k], corners[2 * k + 1]);
    const int64_t tiles = (int64_t)cdiv(patch_size, kTile) * cdiv(patch_size, kTile);
    if (n_patches * tiles > 0x7fffffffLL) return fail(PXR_ERR_INVALID_ARGUMENT, "too many windows in one call");
  }
  if (!ctx || !weights) return fail(PXR_ERR_INVALID_ARGUMENT, "NULL context or weights");
  if (weights->device != ctx->device)
    return fail(PXR_ERR_INVALID_ARGUMENT, "the weights live on device %d, the context on %d", weights->device, ctx->device);
  const size_t osz = out_dtype == PXR_F16 ? 2 : (out_dtype == PXR_F32 ? 4 : 8);
  const int64_t rows = corners ? n_patches * patch_size * patch_size : (int64_t)height * width;
  const size_t out_bytes = (size_t)rows * 128 * osz;
  if (rows == 0) return PXR_OK;

  PXR_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  DevBuf<uint8_t> d_image;
  DevBuf<int32_t> d_corners;
  DevBuf<int> d_bad;
  S2dArgs a;
  a.image = image;
  if (!image_on_device) {
    PXR_TRY(d_image.upload(image, (size_t)height * width * 3, s));
    a.image = d_image.p;
  }
  if (corners) PXR_TRY(d_corners.upload(corners, (size_t)n_patches * 2, s));
  PXR_TRY(d_bad.alloc(1));
  PXR_TRY(d_bad.zero(s));
  uint8_t* d_out = nullptr;
  PXR_CUDA(cudaMalloc((void**)&d_out, out_bytes));
  a.H = height; a.W = width;
  a.params = reinterpret_cast<const float*>(weights->d);
  a.taps = reinterpret_cast<const uint8_t*>(weights->d) + kFloats * 4;
  a.corners = d_corners.p; a.ps = patch_size; a.tiles_per_side = corners ? (int)cdiv(patch_size, kTile) : 0;
  a.l2_normalize = l2_normalize != 0;
  a.out = d_out;
  a.bad = d_bad.p;
  dim3 grid = corners ? dim3((unsigned)(n_patches * a.tiles_per_side * a.tiles_per_side))
                      : dim3((unsigned)cdiv(width, kTile), (unsigned)cdiv(height, kTile));
  int rc = out_dtype == PXR_F16 ? launch_s2dnet<__half>(ctx, grid, a)
         : out_dtype == PXR_F32 ? launch_s2dnet<float>(ctx, grid, a) : launch_s2dnet<double>(ctx, grid, a);
  cudaError_t e;
  int bad = 0;
  if (rc == PXR_OK) {
    e = cudaMemcpyAsync(&bad, d_bad.p, sizeof(int), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) rc = fail(PXR_ERR_CUDA, "s2dnet failed: %s", cudaGetErrorString(e));
    else if (bad) rc = fail(PXR_ERR_NUMERIC, "S2DNet: an intermediate activation is not finite in fp16 (|x| > 65504)");
  }
  if (rc == PXR_OK && out_host) {
    e = cudaMemcpyAsync(out_host, d_out, out_bytes, cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) rc = fail(PXR_ERR_CUDA, "cudaMemcpyAsync failed: %s", cudaGetErrorString(e));
  }
  if (rc == PXR_OK && out_device) *out_device = d_out;
  else cudaFree(d_out);
  return rc;
}
