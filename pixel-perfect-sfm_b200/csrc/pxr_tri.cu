// pxr_tri.cu — point triangulation from known poses: COLMAP's point_triangulator as hloc's triangulation drives it.
//
//   verify kernel   one thread per match: both keypoints to the normalised plane (cam_image_to_world), the two
//                   point-to-epipolar-line distances of E = [t]x R (cam1_from_cam0), kept when each is within its
//                   camera's threshold (hloc's geometric_verification).
//   ray kernel      one thread per observation: the world-frame unit ray d and the camera centre c, so no camera model
//                   runs per hypothesis.
//   track kernel    one warp per track, grid-stride over tracks: lanes take hypotheses (observation pairs), score each
//                   against every observation of the track (MSAC over the angular error), a butterfly argmin picks the
//                   winner (ties to the lowest index), then the warp refits the N-view midpoint point on the inliers with
//                   butterfly sums.  No atomics: a track's result does not depend on the launch it shares.
//   error kernel    one thread per observation: the pixel reprojection error of its track's point (world_to_pixel).
//   angle kernel    one warp per track: the largest triangulation angle among all observations (evaluate mode).
// The rules are include/pxr.h's; tests/triangulation_reference.py restates them in numpy.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <vector>

#include "pxr_device.cuh"
#include "pxr_waves.h"

namespace pxr {

constexpr int kTThreads = 256;
constexpr int kTWarps = kTThreads / 32;
constexpr double kRadPerDeg = 0.017453292519943295;

struct TriArgs {
  const int32_t* cam_model; const double* cam_params;   // [n_cameras], [n_cameras][kMaxK]
  const int32_t* img_cam; const double* qvec; const double* tvec;
  int64_t n_tracks, n_obs;
  const int64_t* track_begin; const int64_t* track_key;
  const int32_t* obs_img; const double* obs_xy;
  double* ray;                     // [n_obs][6] d | c
};

// the angle between a and b in [0, pi]
__device__ __forceinline__ double angle_between(const double* a, const double* b) {
  const double cx = a[1] * b[2] - a[2] * b[1], cy = a[2] * b[0] - a[0] * b[2], cz = a[0] * b[1] - a[1] * b[0];
  return atan2(sqrt(cx * cx + cy * cy + cz * cz), a[0] * b[0] + a[1] * b[1] + a[2] * b[2]);
}

// COLMAP's CalculateTriangulationAngle: the angle at X between the directions to two camera centres, folded to [0, pi/2]
__device__ __forceinline__ double tri_angle(const double* ci, const double* cj, const double* X) {
  const double a[3] = {X[0] - ci[0], X[1] - ci[1], X[2] - ci[2]}, b[3] = {X[0] - cj[0], X[1] - cj[1], X[2] - cj[2]};
  const double t = angle_between(a, b);
  return fmin(t, M_PI - t);
}

// the midpoint least-squares point of the normal equations A X = b (A symmetric: a00 a01 a02 a11 a12 a22); false when
// A is numerically singular (parallel rays)
__device__ __forceinline__ bool solve_sym3(const double* A, const double* b, double* X) {
  const double c00 = A[3] * A[5] - A[4] * A[4], c01 = A[2] * A[4] - A[1] * A[5], c02 = A[1] * A[4] - A[2] * A[3];
  const double c11 = A[0] * A[5] - A[2] * A[2], c12 = A[1] * A[2] - A[0] * A[4], c22 = A[0] * A[3] - A[1] * A[1];
  const double det = A[0] * c00 + A[1] * c01 + A[2] * c02;
  const double tr = (A[0] + A[3] + A[5]) / 3.0;
  if (!(det > 1e-14 * tr * tr * tr)) return false;
  const double inv = 1.0 / det;
  X[0] = (c00 * b[0] + c01 * b[1] + c02 * b[2]) * inv;
  X[1] = (c01 * b[0] + c11 * b[1] + c12 * b[2]) * inv;
  X[2] = (c02 * b[0] + c12 * b[1] + c22 * b[2]) * inv;
  return true;
}

// adds (I - d d^T) and (I - d d^T) c of one ray to A (6) and b (3)
__device__ __forceinline__ void add_ray(const double* r, double* A, double* b) {
  const double* d = r;
  const double* c = r + 3;
  const double dc = d[0] * c[0] + d[1] * c[1] + d[2] * c[2];
  A[0] += 1.0 - d[0] * d[0]; A[1] -= d[0] * d[1]; A[2] -= d[0] * d[2];
  A[3] += 1.0 - d[1] * d[1]; A[4] -= d[1] * d[2]; A[5] += 1.0 - d[2] * d[2];
  b[0] += c[0] - d[0] * dc; b[1] += c[1] - d[1] * dc; b[2] += c[2] - d[2] * dc;
}

// angular error of one ray to X; false when X is not in front of it
__device__ __forceinline__ bool ray_error(const double* r, const double* X, double& e) {
  const double v[3] = {X[0] - r[3], X[1] - r[4], X[2] - r[5]};
  e = angle_between(r, v);
  return r[0] * v[0] + r[1] * v[1] + r[2] * v[2] > 0.0;
}

__global__ void tri_verify_kernel(TriArgs a, int64_t n, const int32_t* __restrict__ mimg, const double* __restrict__ mxy,
                                  const double* __restrict__ noise, double max_error, uint8_t* keep, double* err) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int im[2] = {mimg[2 * i], mimg[2 * i + 1]};
  double x[2][3], R[2][9], thr[2];
  for (int s = 0; s < 2; ++s) {
    const int cam = a.img_cam[im[s]];
    const int model = a.cam_model[cam];
    const double* p = a.cam_params + (size_t)cam * kMaxK;
    cam_image_to_world(model, p, mxy[4 * i + 2 * s], mxy[4 * i + 2 * s + 1], x[s][0], x[s][1]);
    x[s][2] = 1.0;
    quat_to_rot(a.qvec + 4 * (size_t)im[s], R[s]);
    thr[s] = noise[2 * i + s] * max_error / mean_focal(model, p);
  }
  // cam1_from_cam0: Rr = R1 R0^T, tr = t1 - Rr t0
  double Rr[9], tr[3];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) Rr[3 * r + c] = R[1][3 * r] * R[0][3 * c] + R[1][3 * r + 1] * R[0][3 * c + 1] + R[1][3 * r + 2] * R[0][3 * c + 2];
  const double* t0 = a.tvec + 3 * (size_t)im[0];
  const double* t1 = a.tvec + 3 * (size_t)im[1];
  for (int r = 0; r < 3; ++r) tr[r] = t1[r] - (Rr[3 * r] * t0[0] + Rr[3 * r + 1] * t0[1] + Rr[3 * r + 2] * t0[2]);
  // E = [tr]x Rr
  double E[9];
  for (int c = 0; c < 3; ++c) {
    E[c] = -tr[2] * Rr[3 + c] + tr[1] * Rr[6 + c];
    E[3 + c] = tr[2] * Rr[c] - tr[0] * Rr[6 + c];
    E[6 + c] = -tr[1] * Rr[c] + tr[0] * Rr[3 + c];
  }
  double Ex0[3], Etx1[3];
  for (int r = 0; r < 3; ++r) {
    Ex0[r] = E[3 * r] * x[0][0] + E[3 * r + 1] * x[0][1] + E[3 * r + 2];
    Etx1[r] = E[r] * x[1][0] + E[3 + r] * x[1][1] + E[6 + r];
  }
  const double dist = fabs(x[1][0] * Ex0[0] + x[1][1] * Ex0[1] + Ex0[2]);
  const double e0 = dist / sqrt(Etx1[0] * Etx1[0] + Etx1[1] * Etx1[1]);
  const double e1 = dist / sqrt(Ex0[0] * Ex0[0] + Ex0[1] * Ex0[1]);
  err[2 * i] = e0; err[2 * i + 1] = e1;
  keep[i] = (e0 <= thr[0] && e1 <= thr[1]) ? 1 : 0;
}

__global__ void tri_ray_kernel(TriArgs a) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n_obs) return;
  const int im = a.obs_img[i];
  const int cam = a.img_cam[im];
  double u, v, R[9];
  cam_image_to_world(a.cam_model[cam], a.cam_params + (size_t)cam * kMaxK, a.obs_xy[2 * i], a.obs_xy[2 * i + 1], u, v);
  quat_to_rot(a.qvec + 4 * (size_t)im, R);
  const double* t = a.tvec + 3 * (size_t)im;
  double d[3];
  for (int k = 0; k < 3; ++k) d[k] = R[k] * u + R[3 + k] * v + R[6 + k];    // R^T (u, v, 1)
  const double nd = 1.0 / sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
  double* out = a.ray + 6 * i;
  for (int k = 0; k < 3; ++k) {
    out[k] = d[k] * nd;
    out[3 + k] = -(R[k] * t[0] + R[3 + k] * t[1] + R[6 + k] * t[2]);          // -R^T t
  }
}

struct TriRunArgs {
  double min_angle, tau;           // radians
  int max_pairs;
  uint64_t seed;
  double* xyz; int32_t* status; int32_t* n_inl; double* angle; uint8_t* inlier;
};

// observation pair of hypothesis h: lexicographic (exhaustive) or drawn from the stream; false when none
__device__ __forceinline__ bool hypothesis_pair(bool exhaustive, int64_t h, int n, uint64_t s0, int& i, int& j) {
  if (exhaustive) {
    int64_t rem = h;
    i = 0;
    while (rem >= n - 1 - i) { rem -= n - 1 - i; ++i; }
    j = i + 1 + (int)rem;
    return true;
  }
  int k = 0, idx[2];
  for (int dd = 0; dd < 64 && k < 2; ++dd) {
    const uint64_t w = splitmix64(s0 ^ ((uint64_t)h << 8) ^ (uint64_t)dd);
    const int x = (int)(((w >> 32) * (uint64_t)n) >> 32);
    if (k == 1 && idx[0] == x) continue;
    idx[k++] = x;
  }
  i = idx[0]; j = idx[1];
  return k == 2;
}

// the point of one observation pair; false when its rays are closer than min_angle or parallel
__device__ __forceinline__ bool two_view_point(const double* ri, const double* rj, double min_angle, double* X) {
  const double t = angle_between(ri, rj);
  if (!(fmin(t, M_PI - t) >= min_angle)) return false;
  double A[6] = {0, 0, 0, 0, 0, 0}, b[3] = {0, 0, 0};
  add_ray(ri, A, b);
  add_ray(rj, A, b);
  return solve_sym3(A, b, X);
}

// marks the inliers of X in flags (lanes over the observations); returns the count and whether any flag changed
__device__ __forceinline__ int mark_inliers(const double* __restrict__ ray, int n, const double* X, double tau,
                                            uint8_t* flags, int lane, bool& changed) {
  int cnt = 0;
  bool ch = false;
  for (int k = lane; k < n; k += 32) {
    double e;
    const bool in = ray_error(ray + 6 * k, X, e) && e <= tau;
    ch |= (flags[k] != 0) != in;
    flags[k] = in ? 1 : 0;
    cnt += in;
  }
  for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  changed = __any_sync(0xffffffffu, ch);
  __syncwarp();
  return cnt;
}

// the N-view midpoint point of the flagged observations (butterfly sums: the same bits in every launch)
__device__ __forceinline__ bool fit_flagged(const double* __restrict__ ray, int n, const uint8_t* flags, int lane,
                                            double* X) {
  double A[6] = {0, 0, 0, 0, 0, 0}, b[3] = {0, 0, 0};
  for (int k = lane; k < n; k += 32)
    if (flags[k]) add_ray(ray + 6 * k, A, b);
  for (int m = 0; m < 6; ++m) A[m] = warp_sum(A[m]);
  for (int m = 0; m < 3; ++m) b[m] = warp_sum(b[m]);
  return solve_sym3(A, b, X);
}

// the largest triangulation angle over pairs of flagged observations (flags NULL: all); max is order-free
__device__ __forceinline__ double max_tri_angle(const double* __restrict__ ray, int n, const uint8_t* flags,
                                                const double* X, int lane) {
  double best = 0.0;
  for (int i = lane; i < n; i += 32) {
    if (flags && !flags[i]) continue;
    for (int j = i + 1; j < n; ++j)
      if (!flags || flags[j]) best = fmax(best, tri_angle(ray + 6 * i + 3, ray + 6 * j + 3, X));
  }
  for (int o = 16; o > 0; o >>= 1) best = fmax(best, __shfl_xor_sync(0xffffffffu, best, o));
  return best;
}

__global__ void __launch_bounds__(kTThreads) tri_track_kernel(TriArgs a, TriRunArgs r) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * kTWarps;
  for (int64_t t = (int64_t)blockIdx.x * kTWarps + (threadIdx.x >> 5); t < a.n_tracks; t += warps) {
    const int64_t b0 = a.track_begin[t];
    const int n = (int)(a.track_begin[t + 1] - b0);
    const double* ray = a.ray + 6 * b0;
    uint8_t* flags = r.inlier + b0;
    const int64_t all = (int64_t)n * (n - 1) / 2;
    const bool exhaustive = all <= r.max_pairs;
    const int64_t H = exhaustive ? all : r.max_pairs;
    const uint64_t key = a.track_key ? (uint64_t)a.track_key[t] : (uint64_t)t;
    const uint64_t s0 = splitmix64(r.seed ^ splitmix64(key));
    const double tau2 = r.tau * r.tau;
    double best = INFINITY;
    int64_t best_h = -1;
    for (int64_t h = lane; h < H; h += 32) {
      int i, j;
      double X[3];
      if (!hypothesis_pair(exhaustive, h, n, s0, i, j) || !two_view_point(ray + 6 * i, ray + 6 * j, r.min_angle, X))
        continue;
      double score = 0.0;
      for (int k = 0; k < n; ++k) {
        double e;
        score += (ray_error(ray + 6 * k, X, e) && e < r.tau) ? e * e : tau2;
      }
      if (score < best) { best = score; best_h = h; }       // h rises per lane: ties stay with the lower index
    }
    for (int o = 16; o > 0; o >>= 1) {
      const double os = __shfl_xor_sync(0xffffffffu, best, o);
      const int64_t oh = __shfl_xor_sync(0xffffffffu, best_h, o);
      if (oh >= 0 && (best_h < 0 || os < best || (os == best && oh < best_h))) { best = os; best_h = oh; }
    }
    int status = PXR_TRI_OK, cnt = 0;
    double X[3] = {0.0, 0.0, 0.0};
    if (best_h < 0) {
      status = PXR_TRI_ANGLE_TOO_SMALL;
      for (int k = lane; k < n; k += 32) flags[k] = 0;
      __syncwarp();
    } else {
      int i, j;
      hypothesis_pair(exhaustive, best_h, n, s0, i, j);
      two_view_point(ray + 6 * i, ray + 6 * j, r.min_angle, X);
      bool changed;
      for (int k = lane; k < n; k += 32) flags[k] = 0;
      __syncwarp();
      cnt = mark_inliers(ray, n, X, r.tau, flags, lane, changed);             // S0
      double X1[3];
      if (cnt < 2) {
        status = PXR_TRI_TOO_FEW_INLIERS;
      } else if (!fit_flagged(ray, n, flags, lane, X1)) {
        status = PXR_TRI_ANGLE_TOO_SMALL;
      } else {
        X[0] = X1[0]; X[1] = X1[1]; X[2] = X1[2];
        cnt = mark_inliers(ray, n, X, r.tau, flags, lane, changed);           // S1
        if (changed) {
          if (cnt < 2) status = PXR_TRI_TOO_FEW_INLIERS;
          else if (fit_flagged(ray, n, flags, lane, X1)) { X[0] = X1[0]; X[1] = X1[1]; X[2] = X1[2]; }
          else status = PXR_TRI_ANGLE_TOO_SMALL;
        }
      }
    }
    const double ang = cnt >= 2 ? max_tri_angle(ray, n, flags, X, lane) : 0.0;
    if (status == PXR_TRI_OK && !(ang >= r.min_angle)) status = PXR_TRI_ANGLE_TOO_SMALL;
    if (lane == 0) {
      for (int k = 0; k < 3; ++k) r.xyz[3 * t + k] = X[k];
      r.status[t] = status; r.n_inl[t] = cnt; r.angle[t] = ang / kRadPerDeg;
    }
  }
}

// pixel reprojection error of every observation against its track's point; +inf when not in front of the camera
__global__ void tri_error_kernel(TriArgs a, const int64_t* __restrict__ obs_track, const double* __restrict__ xyz,
                                 double* err) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n_obs) return;
  const int im = a.obs_img[i];
  const int cam = a.img_cam[im];
  const double* X = xyz + 3 * obs_track[i];
  const double* q = a.qvec + 4 * (size_t)im;
  const double* t = a.tvec + 3 * (size_t)im;
  double R[9];
  quat_to_rot(q, R);
  const double z = R[6] * X[0] + R[7] * X[1] + R[8] * X[2] + t[2];
  if (!(z > 2.220446049250313e-16)) { err[i] = INFINITY; return; }
  double xy[2], Jp[2][6], Jx[2][3], Jk[2][kMaxK];
  world_to_pixel<false>(a.cam_model[cam], a.cam_params + (size_t)cam * kMaxK, q, t, X, xy, Jp, Jx, Jk);
  const double dx = xy[0] - a.obs_xy[2 * i], dy = xy[1] - a.obs_xy[2 * i + 1];
  err[i] = sqrt(dx * dx + dy * dy);
}

__global__ void __launch_bounds__(kTThreads) tri_angle_kernel(TriArgs a, const double* __restrict__ xyz, double* angle) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * kTWarps;
  for (int64_t t = (int64_t)blockIdx.x * kTWarps + (threadIdx.x >> 5); t < a.n_tracks; t += warps) {
    const int64_t b0 = a.track_begin[t];
    const double ang = max_tri_angle(a.ray + 6 * b0, (int)(a.track_begin[t + 1] - b0), nullptr, xyz + 3 * t, lane);
    if (lane == 0) angle[t] = ang / kRadPerDeg;
  }
}

// ---- host side --------------------------------------------------------------------------------------------------
static int check_cameras(const pxr_tri_desc* d) {
  if (!d) return fail(PXR_ERR_INVALID_ARGUMENT, "desc is NULL");
  if (d->n_cameras < 0 || d->n_images < 0 || d->n_tracks < 0) return fail(PXR_ERR_INVALID_ARGUMENT, "negative count");
  if ((d->n_cameras && (!d->cam_model || !d->cam_params)) || (d->n_images && (!d->img_cam || !d->qvec || !d->tvec)))
    return fail(PXR_ERR_INVALID_ARGUMENT, "a required array is NULL");
  for (int c = 0; c < d->n_cameras; ++c)
    if (cam_num_params(d->cam_model[c]) == 0) return fail(PXR_ERR_UNSUPPORTED, "unsupported camera model id %d", d->cam_model[c]);
  for (int i = 0; i < d->n_images; ++i)
    if (d->img_cam[i] < 0 || d->img_cam[i] >= d->n_cameras)
      return fail(PXR_ERR_INVALID_ARGUMENT, "image %d has camera index %d out of range", i, d->img_cam[i]);
  return PXR_OK;
}

static int check_tracks(const pxr_tri_desc* d) {
  PXR_TRY(check_cameras(d));
  if (!d->track_begin) return fail(PXR_ERR_INVALID_ARGUMENT, "track_begin is NULL");
  if (d->track_begin[0] != 0) return fail(PXR_ERR_INVALID_ARGUMENT, "track_begin[0] must be 0");
  for (int64_t t = 0; t < d->n_tracks; ++t) {
    const int64_t n = d->track_begin[t + 1] - d->track_begin[t];
    if (n < 2) return fail(PXR_ERR_INVALID_ARGUMENT, "track %lld has %lld observations (track_begin must rise by >= 2)",
                           (long long)t, (long long)n);
    if (n > INT32_MAX) return fail(PXR_ERR_INVALID_ARGUMENT, "track %lld has more than 2^31 - 1 observations", (long long)t);
  }
  const int64_t n_obs = d->track_begin[d->n_tracks];
  if (n_obs && (!d->obs_img || !d->obs_xy)) return fail(PXR_ERR_INVALID_ARGUMENT, "a required array is NULL");
  for (int64_t i = 0; i < n_obs; ++i)
    if (d->obs_img[i] < 0 || d->obs_img[i] >= d->n_images)
      return fail(PXR_ERR_INVALID_ARGUMENT, "observation %lld has image index %d out of range", (long long)i, d->obs_img[i]);
  return PXR_OK;
}

// device copies of the cameras and poses, and of the tracks when asked
struct TriUpload {
  DevBuf<int32_t> model, img_cam, obs_img;
  DevBuf<double> params, qvec, tvec, obs_xy, ray;
  DevBuf<int64_t> begin, key, obs_track;
  double h2d = 0.0;
  int upload(const pxr_tri_desc* d, bool tracks, cudaStream_t s, TriArgs& a) {
    PXR_TRY(model.upload(d->cam_model, d->n_cameras, s));
    PXR_TRY(params.upload(d->cam_params, (size_t)d->n_cameras * kMaxK, s));
    PXR_TRY(img_cam.upload(d->img_cam, d->n_images, s));
    PXR_TRY(qvec.upload(d->qvec, (size_t)d->n_images * 4, s));
    PXR_TRY(tvec.upload(d->tvec, (size_t)d->n_images * 3, s));
    h2d = (double)d->n_cameras * (4 + kMaxK * 8) + (double)d->n_images * (4 + 56);
    std::memset(&a, 0, sizeof(a));
    a.cam_model = model.p; a.cam_params = params.p; a.img_cam = img_cam.p; a.qvec = qvec.p; a.tvec = tvec.p;
    if (!tracks) return PXR_OK;
    const int64_t nt = d->n_tracks, no = d->track_begin[nt];
    std::vector<int64_t> ot((size_t)no);
    for (int64_t t = 0; t < nt; ++t)
      for (int64_t i = d->track_begin[t]; i < d->track_begin[t + 1]; ++i) ot[i] = t;
    PXR_TRY(begin.upload(d->track_begin, (size_t)nt + 1, s));
    if (d->track_key) PXR_TRY(key.upload(d->track_key, nt, s));
    PXR_TRY(obs_img.upload(d->obs_img, no, s));
    PXR_TRY(obs_xy.upload(d->obs_xy, (size_t)no * 2, s));
    PXR_TRY(obs_track.upload(ot.data(), no, s));
    PXR_TRY(ray.alloc((size_t)no * 6));
    h2d += (double)(nt + 1) * 8 + (d->track_key ? nt * 8.0 : 0.0) + (double)no * (4 + 16 + 8);
    a.n_tracks = nt; a.n_obs = no; a.track_begin = begin.p; a.track_key = d->track_key ? key.p : nullptr;
    a.obs_img = obs_img.p; a.obs_xy = obs_xy.p; a.ray = ray.p;
    return PXR_OK;
  }
};

struct Events {
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  ~Events() { if (e0) cudaEventDestroy(e0); if (e1) cudaEventDestroy(e1); }
  int create() { PXR_CUDA(cudaEventCreate(&e0)); PXR_CUDA(cudaEventCreate(&e1)); return PXR_OK; }
  double ms() const { float m = 0.f; return cudaEventElapsedTime(&m, e0, e1) == cudaSuccess ? m : 0.0; }
};

static void fill_summary(pxr_summary* total, const pxr_ctx* ctx, int64_t launches0, double h2d, double kernel_ms,
                         std::chrono::steady_clock::time_point t0, const char* what, int64_t n) {
  if (!total) return;
  const int cap_it = total->iterations_capacity;
  pxr_iteration_summary* keep = total->iterations;
  std::memset(total, 0, sizeof(*total));
  total->iterations_capacity = cap_it; total->iterations = keep;
  total->h2d_bytes = h2d;
  total->kernel_launches = ctx ? ctx->launches - launches0 : 0;
  total->total_time_s = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  total->solve_time_s = kernel_ms * 1e-3;
  std::snprintf(total->message, sizeof(total->message), "%lld %s, kernels %.3f ms", (long long)n, what, kernel_ms);
}

static unsigned warp_grid(const pxr_ctx* ctx, int64_t n_tracks) {
  return (unsigned)std::max<int64_t>(1, std::min<int64_t>(cdiv(n_tracks, kTWarps), (int64_t)ctx->sm_count * 16));
}

}  // namespace pxr

using namespace pxr;

extern "C" void pxr_default_tri_options(pxr_tri_options* o) {
  if (!o) return;
  std::memset(o, 0, sizeof(*o));
  o->min_angle = 1.5; o->create_max_angle_error = 2.0; o->tri_max_pairs = 1024; o->seed = 0;
}

extern "C" int pxr_tri_verify(pxr_ctx* ctx, const pxr_tri_desc* d, int64_t n, const int32_t* mimg, const double* mxy,
                              const double* noise, double max_error, uint8_t* keep, double* err, pxr_summary* total) {
  const auto t0 = std::chrono::steady_clock::now();
  PXR_TRY(check_cameras(d));
  if (n < 0) return fail(PXR_ERR_INVALID_ARGUMENT, "n_matches < 0");
  if (!(max_error > 0.0)) return fail(PXR_ERR_INVALID_ARGUMENT, "max_error must be > 0");
  if (n && (!mimg || !mxy || !noise || !keep || !err)) return fail(PXR_ERR_INVALID_ARGUMENT, "a required array is NULL");
  for (int64_t i = 0; i < 2 * n; ++i)
    if (mimg[i] < 0 || mimg[i] >= d->n_images)
      return fail(PXR_ERR_INVALID_ARGUMENT, "match %lld has image index %d out of range", (long long)(i / 2), mimg[i]);
  PXR_TRY(require_ctx(ctx));
  const int64_t launches0 = ctx->launches;
  double kernel_ms = 0.0, h2d = 0.0;
  if (n > 0) {
    PXR_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    TriUpload up;
    TriArgs a;
    PXR_TRY(up.upload(d, false, s, a));
    DevBuf<int32_t> dimg;
    DevBuf<double> dxy, dnoise, derr;
    DevBuf<uint8_t> dkeep;
    PXR_TRY(dimg.upload(mimg, (size_t)n * 2, s));
    PXR_TRY(dxy.upload(mxy, (size_t)n * 4, s));
    PXR_TRY(dnoise.upload(noise, (size_t)n * 2, s));
    PXR_TRY(dkeep.alloc(n));
    PXR_TRY(derr.alloc((size_t)n * 2));
    h2d = up.h2d + (double)n * (8 + 32 + 16);
    Events ev;
    PXR_TRY(ev.create());
    PXR_CUDA(cudaEventRecord(ev.e0, s));
    PXR_LAUNCH(ctx, tri_verify_kernel, (unsigned)cdiv(n, 128), 128, 0, a, n, dimg.p, dxy.p, dnoise.p, max_error, dkeep.p, derr.p);
    PXR_CUDA(cudaGetLastError());
    PXR_CUDA(cudaEventRecord(ev.e1, s));
    PXR_CUDA(cudaMemcpyAsync(keep, dkeep.p, (size_t)n, cudaMemcpyDeviceToHost, s));
    PXR_CUDA(cudaMemcpyAsync(err, derr.p, (size_t)n * 16, cudaMemcpyDeviceToHost, s));
    PXR_CUDA(cudaStreamSynchronize(s));
    kernel_ms = ev.ms();
  }
  fill_summary(total, ctx, launches0, h2d, kernel_ms, t0, "matches", n);
  return PXR_OK;
}

extern "C" int pxr_tri_run(pxr_ctx* ctx, const pxr_tri_desc* d, const pxr_tri_options* o, double* xyz, int32_t* status,
                           int32_t* n_inliers, double* tri_angle_out, uint8_t* obs_inlier, double* obs_error,
                           pxr_summary* total) {
  const auto t0 = std::chrono::steady_clock::now();
  if (!o) return fail(PXR_ERR_INVALID_ARGUMENT, "options is NULL");
  if (!(o->min_angle >= 0.0 && o->min_angle < 90.0)) return fail(PXR_ERR_INVALID_ARGUMENT, "min_angle must be in [0, 90)");
  if (!(o->create_max_angle_error > 0.0 && o->create_max_angle_error < 90.0))
    return fail(PXR_ERR_INVALID_ARGUMENT, "create_max_angle_error must be in (0, 90)");
  if (o->tri_max_pairs < 1) return fail(PXR_ERR_INVALID_ARGUMENT, "tri_max_pairs must be >= 1");
  PXR_TRY(check_tracks(d));
  const int64_t nt = d->n_tracks, no = d->track_begin[nt];
  if (nt && (!xyz || !status || !n_inliers || !tri_angle_out || !obs_inlier || !obs_error))
    return fail(PXR_ERR_INVALID_ARGUMENT, "an output array is NULL");
  PXR_TRY(require_ctx(ctx));
  const int64_t launches0 = ctx->launches;
  double kernel_ms = 0.0, h2d = 0.0;
  if (nt > 0) {
    PXR_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    TriUpload up;
    TriArgs a;
    PXR_TRY(up.upload(d, true, s, a));
    h2d = up.h2d;
    DevBuf<double> dxyz, dang, derr;
    DevBuf<int32_t> dstat, dcnt;
    DevBuf<uint8_t> dinl;
    PXR_TRY(dxyz.alloc((size_t)nt * 3)); PXR_TRY(dang.alloc(nt)); PXR_TRY(derr.alloc(no));
    PXR_TRY(dstat.alloc(nt)); PXR_TRY(dcnt.alloc(nt)); PXR_TRY(dinl.alloc(no));
    TriRunArgs r;
    r.min_angle = o->min_angle * kRadPerDeg; r.tau = o->create_max_angle_error * kRadPerDeg;
    r.max_pairs = o->tri_max_pairs; r.seed = o->seed;
    r.xyz = dxyz.p; r.status = dstat.p; r.n_inl = dcnt.p; r.angle = dang.p; r.inlier = dinl.p;
    Events ev;
    PXR_TRY(ev.create());
    PXR_CUDA(cudaEventRecord(ev.e0, s));
    PXR_LAUNCH(ctx, tri_ray_kernel, (unsigned)cdiv(no, 128), 128, 0, a);
    PXR_LAUNCH(ctx, tri_track_kernel, warp_grid(ctx, nt), kTThreads, 0, a, r);
    PXR_LAUNCH(ctx, tri_error_kernel, (unsigned)cdiv(no, 128), 128, 0, a, up.obs_track.p, dxyz.p, derr.p);
    PXR_CUDA(cudaGetLastError());
    PXR_CUDA(cudaEventRecord(ev.e1, s));
    PXR_CUDA(cudaMemcpyAsync(xyz, dxyz.p, (size_t)nt * 24, cudaMemcpyDeviceToHost, s));
    PXR_CUDA(cudaMemcpyAsync(status, dstat.p, (size_t)nt * 4, cudaMemcpyDeviceToHost, s));
    PXR_CUDA(cudaMemcpyAsync(n_inliers, dcnt.p, (size_t)nt * 4, cudaMemcpyDeviceToHost, s));
    PXR_CUDA(cudaMemcpyAsync(tri_angle_out, dang.p, (size_t)nt * 8, cudaMemcpyDeviceToHost, s));
    PXR_CUDA(cudaMemcpyAsync(obs_inlier, dinl.p, (size_t)no, cudaMemcpyDeviceToHost, s));
    PXR_CUDA(cudaMemcpyAsync(obs_error, derr.p, (size_t)no * 8, cudaMemcpyDeviceToHost, s));
    PXR_CUDA(cudaStreamSynchronize(s));
    kernel_ms = ev.ms();
  }
  fill_summary(total, ctx, launches0, h2d, kernel_ms, t0, "tracks", nt);
  return PXR_OK;
}

extern "C" int pxr_tri_evaluate(pxr_ctx* ctx, const pxr_tri_desc* d, const double* xyz, double* obs_error,
                                double* tri_angle_out, pxr_summary* total) {
  const auto t0 = std::chrono::steady_clock::now();
  PXR_TRY(check_tracks(d));
  const int64_t nt = d->n_tracks, no = d->track_begin[nt];
  if (nt && (!xyz || !obs_error || !tri_angle_out)) return fail(PXR_ERR_INVALID_ARGUMENT, "a required array is NULL");
  PXR_TRY(require_ctx(ctx));
  const int64_t launches0 = ctx->launches;
  double kernel_ms = 0.0, h2d = 0.0;
  if (nt > 0) {
    PXR_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    TriUpload up;
    TriArgs a;
    PXR_TRY(up.upload(d, true, s, a));
    DevBuf<double> dxyz, dang, derr;
    PXR_TRY(dxyz.upload(xyz, (size_t)nt * 3, s));
    PXR_TRY(dang.alloc(nt)); PXR_TRY(derr.alloc(no));
    h2d = up.h2d + (double)nt * 24;
    Events ev;
    PXR_TRY(ev.create());
    PXR_CUDA(cudaEventRecord(ev.e0, s));
    PXR_LAUNCH(ctx, tri_ray_kernel, (unsigned)cdiv(no, 128), 128, 0, a);
    PXR_LAUNCH(ctx, tri_error_kernel, (unsigned)cdiv(no, 128), 128, 0, a, up.obs_track.p, dxyz.p, derr.p);
    PXR_LAUNCH(ctx, tri_angle_kernel, warp_grid(ctx, nt), kTThreads, 0, a, dxyz.p, dang.p);
    PXR_CUDA(cudaGetLastError());
    PXR_CUDA(cudaEventRecord(ev.e1, s));
    PXR_CUDA(cudaMemcpyAsync(obs_error, derr.p, (size_t)no * 8, cudaMemcpyDeviceToHost, s));
    PXR_CUDA(cudaMemcpyAsync(tri_angle_out, dang.p, (size_t)nt * 8, cudaMemcpyDeviceToHost, s));
    PXR_CUDA(cudaStreamSynchronize(s));
    kernel_ms = ev.ms();
  }
  fill_summary(total, ctx, launches0, h2d, kernel_ms, t0, "tracks", nt);
  return PXR_OK;
}
