// pxr_waves.h — the wave machinery of the batched query solvers (pxr_qba.cu, pxr_ka.cu): consecutive queries packed
// into waves that fit a byte budget, and the loop that uploads the next wave while the current one solves.
#pragma once
#include <cuda_runtime.h>

#include <cstdlib>
#include <functional>
#include <vector>

#include "pxr_internal.h"

namespace pxr {

inline size_t dtype_bytes(int dt) { return dt == PXR_F16 ? 2 : (dt == PXR_F32 ? 4 : 8); }

inline bool on_device(const void* p) {
  cudaPointerAttributes pa;
  if (!p || cudaPointerGetAttributes(&pa, p) != cudaSuccess) { cudaGetLastError(); return false; }
  return pa.type == cudaMemoryTypeDevice || pa.type == cudaMemoryTypeManaged;
}

struct WavePlan {
  std::vector<int32_t> begin;       // [n_waves + 1]
  std::vector<double> bytes;        // [n_waves]
  std::vector<uint8_t> host_patch;  // [n_queries] 1: the block is in host memory
};

// Consecutive queries while the wave fits the budget; a query larger than the budget gets a wave of its own.  Every
// wave starts at `fixed` bytes; query q adds query_bytes(q, its block is in host memory), and starts a new wave where
// splits(q) (a query that cannot share a launch with the one before it).
template <class Bytes>
void plan_waves(int n, const void* const* blocks, const int64_t* counts, double fixed, double budget, Bytes query_bytes,
                WavePlan* p, const std::function<bool(int)>& splits = nullptr) {
  p->begin.assign(1, 0); p->bytes.clear();
  p->host_patch.assign((size_t)n, 0);
  double cur = fixed;
  for (int q = 0; q < n; ++q) {
    p->host_patch[q] = (counts[q] > 0 && !on_device(blocks[q])) ? 1 : 0;
    const double b = query_bytes(q, p->host_patch[q] != 0);
    if (q > p->begin.back() && (cur + b > budget || (splits && splits(q)))) {
      p->bytes.push_back(cur); p->begin.push_back(q); cur = fixed;
    }
    cur += b;
  }
  if (n > 0) { p->bytes.push_back(cur); p->begin.push_back(n); }
}

// the batched entry points check their arguments first; then a NULL context is reported as no device when there is none
inline int require_ctx(pxr_ctx* ctx) {
  if (ctx) return PXR_OK;
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0) {
    cudaGetLastError();
    return fail(PXR_ERR_NO_DEVICE, "no CUDA device available; libpxr has no CPU fallback");
  }
  return fail(PXR_ERR_INVALID_ARGUMENT, "ctx is NULL");
}

// max_wave_bytes > 0: itself; 0: half of the free device memory
inline int wave_budget(double max_wave_bytes, double* budget) {
  if (max_wave_bytes > 0.0) { *budget = max_wave_bytes; return PXR_OK; }
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0) {
    cudaGetLastError();
    return fail(PXR_ERR_NO_DEVICE, "max_wave_bytes 0 means half of the free device memory, and there is no CUDA device");
  }
  size_t fr = 0, tot = 0;
  PXR_CUDA(cudaMemGetInfo(&fr, &tot));
  *budget = 0.5 * (double)fr;
  return PXR_OK;
}

// Wave buffer sets: two (the next upload runs while the current wave solves) when both fit in free device memory,
// else one.  PXR_QBA_WAVE_BUFFERS=1 keeps one (tests: the one-buffer ordering is otherwise reached only by waves near
// half the free memory).
inline int wave_sets(int n_waves, size_t max_wave_device_bytes, int* nsets) {
  size_t fr = 0, tot = 0;
  PXR_CUDA(cudaMemGetInfo(&fr, &tot));
  const char* one_buf = std::getenv("PXR_QBA_WAVE_BUFFERS");
  const bool force_one = one_buf && std::atoi(one_buf) == 1;
  *nsets = (!force_one && n_waves > 1 && 2.0 * (double)max_wave_device_bytes < 0.9 * (double)fr) ? 2 : 1;
  return PXR_OK;
}

// The wave loop.  upload(w, set) enqueues wave w's inputs into buffer set `set` on the upload stream us; launch(w,
// set) enqueues its solve and the copies of its outputs to the host on ctx->stream; finish(w, set) runs on the host
// once those are complete.  With one set the next upload waits for the current wave's outputs to leave the buffer.
// *n_done receives the waves finished (also when the interrupt callback stops the loop between waves).
struct WaveSteps {
  std::function<int(int, int)> upload, launch, finish;
};

inline int run_waves(pxr_ctx* ctx, int nw, int nsets, cudaStream_t us, const WaveSteps& st, int* n_done) {
  cudaStream_t s = ctx->stream;
  cudaEvent_t up_done[2] = {nullptr, nullptr}, k_done[2] = {nullptr, nullptr};
  struct Events {
    cudaEvent_t* e[2];
    ~Events() { for (int k = 0; k < 2; ++k) for (int i = 0; i < 2; ++i) if (e[k][i]) cudaEventDestroy(e[k][i]); }
  } guard{{up_done, k_done}};
  for (cudaEvent_t* e : {&up_done[0], &up_done[1], &k_done[0], &k_done[1]})
    PXR_CUDA(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
  *n_done = 0;
  if (nw > 0) PXR_TRY(st.upload(0, 0));
  for (int w = 0; w < nw; ++w) {
    const int set = nsets == 2 ? (w & 1) : 0;
    PXR_CUDA(cudaEventRecord(up_done[set], us));
    PXR_CUDA(cudaStreamWaitEvent(s, up_done[set], 0));
    PXR_TRY(st.launch(w, set));
    PXR_CUDA(cudaEventRecord(k_done[set], s));
    if (w + 1 < nw) {        // the next upload goes out before the host waits for this wave
      const int nset = nsets == 2 ? 1 - set : 0;
      if (nsets == 1) PXR_CUDA(cudaStreamWaitEvent(us, k_done[set], 0));
      PXR_TRY(st.upload(w + 1, nset));
    }
    PXR_CUDA(cudaEventSynchronize(k_done[set]));
    PXR_TRY(st.finish(w, set));
    *n_done = w + 1;
    if (w + 1 < nw && interrupt_pending()) {
      cudaStreamSynchronize(us);
      return fail(PXR_ERR_INTERRUPTED, "interrupted by the host after wave %d of %d", w + 1, nw);
    }
  }
  PXR_CUDA(cudaStreamSynchronize(us));
  return PXR_OK;
}

}  // namespace pxr
