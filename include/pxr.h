/*
 * pxr.h — C-ABI of the H100-native featuremetric refinement engine (libpxr.so).
 *
 * Drop-in boundary for the featuremetric keypoint-adjustment (KA) and
 * bundle-adjustment (BA) hot path of cvg/pixel-perfect-sfm.  The reference has
 * no C-ABI: its boundary is the pybind11 module `pixsfm._pixsfm`
 * (reference pixsfm/_pixsfm/bindings.cc:34-63).  Every entry point below names
 * the reference interface it replaces; the pybind/ctypes stub a maintainer
 * would add on the reference side is shown in INTEGRATION.md.
 *
 * Conventions
 *  - plain C, `extern "C"`, no C++/torch types; all sizes explicit.
 *  - every function returns a pxr_status; pxr_last_error() gives the message
 *    for the calling thread.  No exception crosses the boundary, nothing
 *    aborts the process (the reference's glog CHECKs abort:
 *    bundle_optimizer.h:222).
 *  - the caller owns all host memory; the library owns all device memory.
 *  - there is NO CPU fallback: every compute entry point fails with
 *    PXR_ERR_NO_DEVICE when no CUDA device is usable.
 *  - one handle is used by one host thread at a time (thread-compatible).
 *
 * Problem IR (SoA, independent of COLMAP objects).  The host adapter resolves
 * the reference's BundleAdjustmentSetup + BundleOptimizerOptions into plain
 * constancy masks exactly as BundleOptimizer::Parameterize{Points,Images,
 * Cameras} does (reference bundle_adjustment/src/bundle_optimizer.h:335-442).
 */
#ifndef PXR_H_
#define PXR_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PXR_VERSION_MAJOR 0
#define PXR_VERSION_MINOR 1
#define PXR_MAX_CAM_PARAMS 12

typedef enum {
  PXR_OK = 0,
  PXR_ERR_INVALID_ARGUMENT = 1, /* -> Python ValueError / std::invalid_argument */
  PXR_ERR_UNSUPPORTED = 2,      /* unsupported (channels, nodes, model) combination */
  PXR_ERR_NO_DEVICE = 3,        /* no CUDA device: the product never falls back to CPU */
  PXR_ERR_CUDA = 4,             /* CUDA runtime error (message has the cudaError string) */
  PXR_ERR_NCCL = 5,
  PXR_ERR_NUMERIC = 6,          /* solver failure (non-PD reduced system that damping could not fix) */
  PXR_ERR_INTERRUPTED = 7,      /* interrupt callback asked to stop (PyInterrupt, util/src/py_interrupt.h) */
  PXR_ERR_INTERNAL = 8
} pxr_status;

/* COLMAP 3.8 camera model ids (colmap/base/camera_models.h; used through
 * CAMERA_MODEL_SWITCH_CASES in reference residuals/src/feature_reference.h:224-252). */
typedef enum {
  PXR_CAM_SIMPLE_PINHOLE = 0, /* f, cx, cy */
  PXR_CAM_PINHOLE = 1,        /* fx, fy, cx, cy */
  PXR_CAM_SIMPLE_RADIAL = 2,  /* f, cx, cy, k */
  PXR_CAM_RADIAL = 3,         /* f, cx, cy, k1, k2 */
  PXR_CAM_OPENCV = 4,         /* fx, fy, cx, cy, k1, k2, p1, p2 */
  PXR_CAM_OPENCV_FISHEYE = 5, /* fx, fy, cx, cy, k1, k2, k3, k4 */
  PXR_CAM_FULL_OPENCV = 6     /* fx, fy, cx, cy, k1, k2, p1, p2, k3, k4, k5, k6 */
} pxr_camera_model;

typedef enum { PXR_F16 = 0, PXR_F32 = 1, PXR_F64 = 2 } pxr_dtype;

/* ceres loss functions reachable from the reference's {"name","params"} dicts
 * (bundle_adjustment/main.py:37-40). */
typedef enum {
  PXR_LOSS_TRIVIAL = 0,
  PXR_LOSS_CAUCHY = 1, /* default, scale 0.25 (bundle_adjustment_options.h:49) */
  PXR_LOSS_HUBER = 2,
  PXR_LOSS_SOFT_L1 = 3,
  PXR_LOSS_ARCTAN = 4
} pxr_loss_type;

typedef enum {
  PXR_SOLVER_AUTO = 0,        /* by #images as bundle_optimizer.h:181-191 */
  PXR_SOLVER_DENSE_SCHUR = 1, /* explicit reduced camera system + dense Cholesky */
  PXR_SOLVER_SPARSE_SCHUR = 2,/* exact too: runs the dense-Cholesky path */
  PXR_SOLVER_ITERATIVE_SCHUR = 3 /* block-Jacobi PCG on the reduced system */
} pxr_linear_solver;

/* InterpolationConfig subset on the named path (base/src/interpolation.h:39-51):
 * mode BICUBIC, one node {0,0}. */
typedef struct {
  int32_t l2_normalize;   /* default 1 */
  int32_t use_float_simd; /* 0: fp32 horizontal + fp64 vertical (reference default), 1: all fp32 */
  int32_t check_bounds;   /* must be 0 on this path (reference default) */
  int32_t reserved;
} pxr_interp_config;

/* Solver options = ceres::Solver::Options fields the reference sets
 * (bundle_adjustment_options.h:48-64, base/main.py:9-22). */
typedef struct {
  int32_t loss_type;                /* pxr_loss_type */
  double loss_scale;                /* "params"[0] */
  int32_t linear_solver;            /* pxr_linear_solver */
  int32_t max_num_iterations;       /* 100 */
  int32_t max_linear_solver_iterations; /* 200 */
  int32_t max_num_consecutive_invalid_steps; /* 10 */
  double function_tolerance;        /* 0 */
  double gradient_tolerance;        /* 0 */
  double parameter_tolerance;       /* 0 (KA: 1e-5) */
  int32_t use_inner_iterations;     /* BA python default: 1 (bundle_adjustment/main.py:41-44) */
  double inner_iteration_tolerance; /* 1e-3 (ceres default) */
  double initial_trust_region_radius; /* 1e4 */
  double max_trust_region_radius;   /* 1e16 */
  double min_trust_region_radius;   /* 1e-32 */
  double min_relative_decrease;     /* 1e-3 */
  double min_lm_diagonal;           /* 1e-6 */
  double max_lm_diagonal;           /* 1e32 */
  int32_t jacobi_scaling;           /* 1 */
  int32_t deterministic;            /* 1: bit-reproducible solve.  The normal equations are assembled by fixed-order reductions
                                     * instead of fp64 atomics (image / pair chunk partials summed in chunk order, point blocks
                                     * observation by observation, scalar sums block by block: csrc/pxr_block.cuh) on the
                                     * block-mode driver; needs <= 8 camera columns per image.  0: atomics (run-to-run
                                     * differences ~1e-16 relative per sum).  tests/test_gpu_deterministic.py */
  int32_t use_nonmonotonic_steps;   /* ceres::Solver::Options::use_nonmonotonic_steps (the reference's configs/default.yaml
                                     * sets it for KA, BA and QKA); 0 */
  int32_t max_consecutive_nonmonotonic_steps; /* 5 */
} pxr_solver_options;

/* One featuremetric BA problem (reference: what BundleOptimizer::SetUp turns a
 * colmap::Reconstruction + FeatureView + references into,
 * bundle_optimizer.h:139-165, feature_reference_bundle_optimizer.h:90-149).
 * Parameter arrays are IN/OUT: pxr_ba_solve updates them in place, as the
 * reference updates the Reconstruction through raw double*
 * (feature_reference_bundle_optimizer.h:111-114). */
typedef struct {
  /* cameras (intrinsics) */
  int32_t n_cameras;
  const int32_t* cam_model;       /* [n_cameras] pxr_camera_model */
  double* cam_params;             /* [n_cameras][PXR_MAX_CAM_PARAMS], unused tail ignored */
  const uint32_t* cam_const_mask; /* [n_cameras] bit i: param i constant; 0xFFFFFFFF: block constant */
  /* images (poses); qvec is (w,x,y,z), world->camera, as COLMAP */
  int32_t n_images;
  double* qvec;                   /* [n_images][4] */
  double* tvec;                   /* [n_images][3] */
  const int32_t* img_cam;         /* [n_images] index into cameras */
  const uint8_t* pose_const;      /* [n_images] 1: qvec and tvec constant */
  const uint8_t* tvec_const_mask; /* [n_images] bit i: tvec[i] constant (SubsetManifold) */
  /* points */
  int64_t n_points;
  double* xyz;                    /* [n_points][3] */
  const uint8_t* point_const;     /* [n_points] 1: constant */
  /* observations = residual blocks, sorted by point index (ties: any fixed order) */
  int64_t n_obs;
  const int32_t* obs_img;         /* [n_obs] */
  const int64_t* obs_pt;          /* [n_obs] non-decreasing */
  const int64_t* obs_patch;       /* [n_obs] index into the patch slab, or NULL: patch i = obs i */
  /* feature patches: slab [n_patches][ph][pw][channels], HWC interleaved like
   * FeaturePatch (features/src/featurepatch.h:244-262, grid2d.h:29-73) */
  int64_t n_patches;
  const void* patches;            /* host pointer (or device pointer if patches_on_device) */
  int32_t patches_on_device;
  int32_t patch_dtype;            /* pxr_dtype */
  int32_t ph, pw, channels;
  const int32_t* corner;          /* [n_patches][2] (x0,y0) */
  const double* scale;            /* [n_patches][2] (sx,sy) */
  double upsampling_factor;       /* FeaturePatch::upsampling_factor_, 1.0 */
  /* per-point reference descriptors, fp64 (Reference::descriptor, references.h:32-65);
   * NULL => residual = interpolated feature (costmap use, feature_reference.h:128-130) */
  const double* refs;             /* [n_points][channels] */
  /* Optional: the patch slab given as several host blocks (one per FeatureMap numpy array, no host-side
   * concatenation: featuremap.cc:38-44 keeps references to the arrays).  When n_patch_blocks > 0,
   * `patches` is ignored and patch index i lives in the block b with offsets[b] <= i < offsets[b+1]. */
  int32_t n_patch_blocks;
  const void* const* patch_block_ptrs;   /* [n_patch_blocks]; each block may be host OR device memory */
  const int64_t* patch_block_counts;     /* [n_patch_blocks] patches per block */
} pxr_ba_desc;

typedef struct {
  int32_t iteration;
  int32_t step_is_valid;
  int32_t step_is_successful;
  double cost;
  double cost_change;
  double gradient_max_norm;
  double step_norm;
  double relative_decrease;
  double trust_region_radius;
  int32_t linear_solver_iterations;
  double iteration_time_s;
} pxr_iteration_summary;

/* Mirrors the fields of ceres::Solver::Summary that the reference reads
 * (bundle_optimizer.h:236-241, util/src/statistics.h:54-129). */
typedef struct {
  double initial_cost;
  double final_cost;
  int32_t num_residual_blocks;
  int64_t num_residuals;          /* num_residual_blocks * channels */
  int32_t num_successful_steps;
  int32_t num_unsuccessful_steps;
  int32_t num_inner_iteration_steps;
  int32_t termination_type;       /* 0 CONVERGENCE, 1 NO_CONVERGENCE, 2 FAILURE, 3 USER_FAILURE */
  double total_time_s;            /* wall, includes uploads */
  double solve_time_s;            /* wall, LM loop only (inputs resident) */
  double h2d_bytes, d2h_bytes;
  int32_t num_iterations;         /* entries valid in `iterations` */
  int32_t iterations_capacity;    /* in: capacity of `iterations` (may be 0) */
  pxr_iteration_summary* iterations; /* caller-allocated */
  int64_t kernel_launches;        /* CUDA kernels of this library launched by the call */
  char message[256];
  /* window residency of the patch slab (pxr_ba_run on a pinned host buffer, csrc/pxr_resident.cuh): side of the window
   * brought over per observation (0: the whole slab was uploaded), observations whose whole patch was fetched later
   * because the point left its window, and evaluation passes repeated for that; h2d_bytes counts what really crossed */
  int32_t resident_window;
  int32_t resident_passes_repeated;
  int64_t resident_refetched;
} pxr_summary;

typedef struct pxr_ctx pxr_ctx;
typedef struct pxr_ba pxr_ba;

/* ---- context ----------------------------------------------------------- */
const char* pxr_last_error(void);
int pxr_version(void);
/* device < 0 → current device. Fails with PXR_ERR_NO_DEVICE when no GPU. */
int pxr_ctx_create(int device, pxr_ctx** out);
int pxr_ctx_destroy(pxr_ctx* ctx);
/* Multi-GPU: point-sharded BA, one process per GPU.  nccl_unique_id is the 128-byte
 * ncclUniqueId made on rank 0 (pxr_nccl_unique_id) and distributed by the host's own
 * plumbing (torch.distributed broadcast in bench.py).  No reference counterpart
 * (the reference is single-process: base/src/parallel_optimizer.h:77-211). */
int pxr_nccl_unique_id(void* id128);
int pxr_ctx_init_comm(pxr_ctx* ctx, int rank, int world, const void* id128);
int pxr_ctx_sync(pxr_ctx* ctx);
/* NCCL collectives issued through this context so far (bench.py divides by the LM iterations it timed: the contract is
 * ONE all-reduce of the reduced camera blocks per LM iteration), and whether the per-iteration SCALAR exchange runs over
 * peer memory (cudaIpc-mapped mailboxes over NVLink, 1) or had to fall back to NCCL (0). */
int64_t pxr_ctx_nccl_collectives(pxr_ctx* ctx);
int pxr_ctx_mailbox_ready(pxr_ctx* ctx);
/* CUDA-event stopwatch on the library stream (bench.py times K LM iterations with it) */
int pxr_ctx_timer_start(pxr_ctx* ctx);
int pxr_ctx_timer_stop(pxr_ctx* ctx, double* elapsed_ms);
int64_t pxr_ctx_kernel_launches(pxr_ctx* ctx);

/* Interruptibility.  The reference polls PyErr_CheckSignals from a ceres::IterationCallback and from its thread-pool
 * wait loop (util/src/py_interrupt.h:29-38, base/src/callbacks.h:10-20, parallel_optimizer.h:186).  Here the host
 * registers ONE process-wide callback; the LM drivers call it between iterations (at most every 200 ms; the reference polls every 2 s) and stop with
 * PXR_ERR_INTERRUPTED when it returns non-zero.  fn == NULL removes it.  pxr_poll_interrupt() calls it right away
 * (no device needed) and returns its answer, 0 without a callback. */
typedef int (*pxr_interrupt_fn)(void* user);
int pxr_set_interrupt_callback(pxr_interrupt_fn fn, void* user);
int pxr_poll_interrupt(void);

/* ---- default option blocks --------------------------------------------- */
void pxr_default_interp_config(pxr_interp_config* c);  /* base/main.py:1-7 */
void pxr_default_ba_options(pxr_solver_options* o);    /* bundle_adjustment/main.py:30-62 */
void pxr_default_ka_options(pxr_solver_options* o);    /* keypoint_adjustment/main.py:60-83 */

/* ---- featuremetric BA ---------------------------------------------------
 * replaces _bundle_adjustment.FeatureReferenceBundleOptimizer.run / set_up /
 * solve_problem / summary (bundle_adjustment/bindings.cc:36-51,137-141). */
int pxr_ba_create(pxr_ctx* ctx, const pxr_ba_desc* desc, const pxr_interp_config* interp,
                  const pxr_solver_options* opt, pxr_ba** out);   /* uploads (set_up) */
int pxr_ba_solve(pxr_ba* ba, pxr_summary* summary);               /* solve_problem */
/* Continues (or starts) the LM trajectory of `ba` for n more iterations (bench.py: W warm-up, then K timed). */
int pxr_ba_iterate(pxr_ba* ba, int n_iterations, pxr_summary* summary);
/* CUDA-event timing of the residual/Jacobian kernel launches inside solve/iterate.
 * enable: 1/0 switches recording and clears the log, -1 leaves it; which: 1 Jacobian-mode K1, 0 cost-only K1.
 * total_ms/count (optional) receive the summed device time and number of recorded launches. */
int pxr_ba_kernel_timing(pxr_ba* ba, int enable, int which, double* total_ms, int* count);
int pxr_ba_read_params(pxr_ba* ba, double* cam_params, double* qvec, double* tvec, double* xyz);
/* Puts the resident problem back to the given parameters (same array shapes as in the desc) and forgets the LM
 * trajectory; patches, topology, work space and captured graphs stay.  bench.py: W warm-up iterations, reset, then K
 * timed iterations FROM ITERATION ZERO, like the CPU arm.  (The reference's optimizers are one-shot objects,
 * bundle_optimizer.h:121-122; this is what constructing a second one on the same FeatureView amounts to.) */
int pxr_ba_reset(pxr_ba* ba, const double* cam_params, const double* qvec, const double* tvec, const double* xyz);
int pxr_ba_destroy(pxr_ba* ba);
/* one-shot convenience = FeatureReferenceBundleOptimizer.run: upload, solve, write back into desc arrays */
int pxr_ba_run(pxr_ctx* ctx, const pxr_ba_desc* desc, const pxr_interp_config* interp,
               const pxr_solver_options* opt, pxr_summary* summary);

/* ---- geometric (reprojection-error) BA -------------------------------------
 * replaces _bundle_adjustment.GeometricBundleOptimizer (bundle_adjustment/bindings.cc:155-162,
 * geometric_bundle_optimizer.h:36-83): residual r = WorldToImage(X) - point2D.XY() in image pixels
 * (colmap::BundleAdjustmentCostFunction through residuals/src/geometric.h:16-41).  The desc carries the geometry, the
 * constancy masks and the observation lists; its patch fields are unused and must be empty: channels 0, patches,
 * patch_block_ptrs (n_patch_blocks 0) and refs NULL; corner, scale and obs_patch may be NULL and are ignored.
 * obs_xy [n_obs][2] is every observation's keypoint (point2D.XY()); a NULL or non-finite entry is
 * PXR_ERR_INVALID_ARGUMENT.  The handle works with every pxr_ba_* call that takes a pxr_ba; on it pxr_ba_evaluate returns gtr = r,
 * gtg = (1, 0, 1) and residuals [n_obs][2], pxr_ba_evaluate_jacobians returns grad = the 2x2 identity, and a summary's
 * num_residuals is 2 n_obs.  The arguments are checked before the context: with ctx == NULL the calls report
 * PXR_ERR_NO_DEVICE when there is no CUDA device. */
int pxr_ba_create_geometric(pxr_ctx* ctx, const pxr_ba_desc* desc, const double* obs_xy,
                            const pxr_solver_options* opt, pxr_ba** out);
/* one-shot = GeometricBundleOptimizer.run: upload, solve, write back into the desc arrays */
int pxr_ba_run_geometric(pxr_ctx* ctx, const pxr_ba_desc* desc, const double* obs_xy,
                         const pxr_solver_options* opt, pxr_summary* summary);

/* Device memory pxr_ba_create / pxr_ba_run will take for this problem, in bytes (host computation, no device needed) —
 * the counterpart of the RAM estimate the reference logs before it solves (bundle_optimizer.h:200-208,
 * util/src/memory.h:45-69).  patch_bytes: the patch slab (0 when it is already resident); state_bytes: per-observation
 * buffers, Schur pair lists and point blocks; reduced_bytes: the reduced camera system (dense, or its block-sparse form
 * when the solver is ITERATIVE_SCHUR and dense would exceed 4 GB).  Any output may be NULL. */
int pxr_ba_estimate_device_bytes(const pxr_ba_desc* desc, const pxr_solver_options* opt, double* patch_bytes,
                                 double* state_bytes, double* reduced_bytes);

/* Parity / introspection: evaluates every residual block at the current parameters.
 * Replaces calling FeatureReferenceCostFunctor::operator() per block
 * (residuals/src/feature_reference.h:98-137).  Any output may be NULL.
 *  sq_norm [n_obs]      ||r||^2 (uncorrected)
 *  gtr     [n_obs][2]   G^T r,  G = [d r/d u, d r/d v] in patch pixel units (u=col, v=row)
 *  gtg     [n_obs][3]   G^T G (uu, uv, vv)
 *  xy      [n_obs][2]   projected image point
 *  residuals [n_obs][C] r as double (large! optional)
 *  cost    scalar       sum 0.5*rho(||r||^2) */
int pxr_ba_evaluate(pxr_ba* ba, double* sq_norm, double* gtr, double* gtg, double* xy,
                    double* residuals, double* cost);
/* The cost-functor surface: what a ceres::CostFunction built by the reference's `_residuals` factories returns from
 * Evaluate() (residuals/bindings.cc:14-30; CreateFeatureReferenceCostFunctor / ...ConstantPoseCostFunctor,
 * residuals/src/feature_reference.h:256-321; parameter order of operator(), :98-137), for every residual block of the
 * problem at once and in factored form: the Jacobian of block o is  J_o = G_o^T-less product  G_o (C x 2) * P_o (2 x p).
 *  residuals [n_obs][C]       r (f - reference, or f when the problem has no references)
 *  grad      [n_obs][2][C]    d r/d u, d r/d v in patch pixel units (after the L2-normalisation chain rule)
 *  juv       [n_obs][2][W]    d(u,v)/d(3 rotation tangent (QuaternionManifold, left-multiplicative) | 3 t | 3 X | K
 *                             camera parameters), W = 9 + K returned through juv_cols, K = largest kNumParams in use
 *  xy        [n_obs][2]       projected image point.   Any output may be NULL. */
int pxr_ba_evaluate_jacobians(pxr_ba* ba, double* residuals, double* grad, double* juv, int32_t* juv_cols, double* xy);
/* Introspection for parity tests: linearise at the current parameters (camera blocks Hcc [nc*nc,
 * lower triangle], gc, point blocks Hpp [n_points*9], gp), assemble the damped Schur system S/rhs at
 * `radius` (Jacobi scaling taken from this linearisation, as in LM iteration 0), solve it and
 * return the full step `delta` [n_local] and the model cost change.  Any output may be NULL. */
int pxr_ba_debug_linearize(pxr_ba* ba, double radius, double* cost, double* Hcc, double* gc, double* Hpp,
                           double* gp, double* S, double* rhs, double* delta, double* model_cost_change);
/* The reduced camera solve S x = rhs alone (tests), on a caller's system: S [nc][nc] row-major (only the lower triangle
 * is read) and rhs [nc] are written where the LM step assembles them, then the handle's configured solver runs (dense
 * Cholesky, its path chosen by PXR_CHOL_BAND / PXR_CHOL_MULTIKERNEL, or the dense PCG for ITERATIVE_SCHUR, PXR_CG_MULTI).
 *  x       [nc]        the solution
 *  factor  [nc+1][nc]  optional, Cholesky paths only: L in the lower triangle, row nc = L^-1 rhs (the upper triangle
 *                      holds whatever S held there)
 *  status              0 solved, 1 numerical failure (non-positive pivot, failed preconditioner), 2 the persistent
 *                      Cholesky bailed out of a wait
 *  linear_iterations   CG iterations (1 for the Cholesky), 0 when the preconditioner failed.
 * The block-sparse and block-mode paths have no dense S: PXR_ERR_UNSUPPORTED.  factor, status and linear_iterations
 * may be NULL. */
int pxr_ba_debug_reduced_solve(pxr_ba* ba, const double* S, const double* rhs, double* x, double* factor, int* status,
                               int* linear_iterations);
/* Runs the per-point inner iterations (ceres CoordinateDescentMinimizer equivalent) once on the
 * current parameters (parity tests). */
int pxr_ba_debug_inner_iterations(pxr_ba* ba);
/* K0 + K1 (Jacobian mode) at the current parameters over the observations list[0..n), the evaluation one batched
 * inner-iteration round runs (tests).  out [n_obs][8]: s, g^T r (2), g^T g (3 uniques), 0, 0 of every listed
 * observation, NaN elsewhere.  count_on_device = 1 passes n (at most n_obs) through device memory, grids sized for
 * all observations. */
int pxr_ba_debug_eval_list(pxr_ba* ba, const int64_t* list, int64_t n, int count_on_device, double* out);
/* The point-only projection of the inner-iteration rounds next to the full one (tests), at the current parameters:
 * uv_full [n_obs][2] from the full projection (K0 with Jacobians) over all observations, then uv [n_obs][2] and
 * jpt [n_obs][6] (d(uv)/dX: row u, then row v) from the point-only projection over list[0..n), NaN elsewhere.
 * count_on_device as in pxr_ba_debug_eval_list. */
int pxr_ba_debug_project_point(pxr_ba* ba, const int64_t* list, int64_t n, int count_on_device, double* uv, double* jpt,
                               double* uv_full);
/* K0 over all observations at the current parameters (tests): jac = 0 the cost-only projection, 1 the one with
 * Jacobians.  uv [n_obs][2] (patch pixels), xy [n_obs][2] (image pixels).  Any output may be NULL. */
int pxr_ba_debug_project(pxr_ba* ba, int jac, double* uv, double* xy);
/* Batched inner iterations run with capture on (enable = 1) keep each round's lists (tests; the host waits for every
 * round).  pxr_ba_debug_inner_round_lists then reads round `round` of the most recent call: *n_points / *n_obs its list
 * lengths, plist [*n_points] its points, list [*n_obs] its observations, active [*n_points] 1 where the round's step
 * kernel kept the point active.  Any output may be NULL. */
int pxr_ba_debug_inner_capture(pxr_ba* ba, int enable);
int pxr_ba_debug_inner_round_lists(pxr_ba* ba, int round, int64_t* plist, int64_t* list, uint8_t* active, int64_t* n_points,
                                   int64_t* n_obs);
/* Half-warps of the K1 launch (fm_eval_kernel) over n_items items of a (dtype, channels) patch slab, as the library
 * sizes it on this context's device (tests); 0 for channels < 8, which run one thread per item. */
int pxr_fm_k1_half_warps(pxr_ctx* ctx, int dtype, int channels, int64_t n_items, int64_t* half_warps);
/* K0 + K1 in `mode` (0 cost only, 1 Jacobian) over all observations at the current parameters (tests, K1
 * measurements).  out [n_obs][8]: every observation's record; mode 0 writes s only and leaves the rest NaN. */
int pxr_ba_debug_eval_records(pxr_ba* ba, int mode, double* out);
/* The rounds of the most recent batched inner iterations (profiling).  *n_rounds = rounds run; for the first
 * min(*n_rounds, capacity) of them counts[2r] = active observations, counts[2r+1] = active points, and ms[r] = the
 * round's stream time (events around its launches, device idle time waiting for the host included) when round timing
 * was on during that call (else -1).  enable_timing >= 0 switches round timing
 * on / off for the calls that follow.  Any output may be NULL. */
int pxr_ba_debug_inner_rounds(pxr_ba* ba, int enable_timing, int capacity, unsigned long long* counts, double* ms,
                              int* n_rounds);
/* The same rounds split by launch (profiling), when round timing was on during that call (else -1): ms[3r] from the
 * round's start to the end of K0 (the projection), ms[3r+1] from there to the end of K1 (fm_eval_kernel), ms[3r+2]
 * from there to the end of the step kernel.  Stream time, so each part includes the launch gap before its kernel. */
int pxr_ba_debug_inner_round_split(pxr_ba* ba, int capacity, double* ms, int* n_rounds);
/* Timing hooks for bench.py: run `iters` LM iterations' worth of the named stage on the
 * resident problem and return the average device time per launch in ms (CUDA events on the
 * library stream).  stage: 0 residual/Jacobian kernel (K1), 1 cost-only kernel, 2 projection+K1+block build,
 * 3 projection kernel (K0), 4 block build, 5 inner-iteration kernel, 6 K1 (Jacobian) over a list of every second
 * observation */
int pxr_ba_time_stage(pxr_ba* ba, int stage, int iters, double* ms_per_launch);
/* Device-side synthetic scene generator used by bench.py (data: synthetic). Fills a patch slab
 * on the device from per-patch smooth fields; see DESIGN.md §bench. */
int pxr_synth_patches_device(pxr_ctx* ctx, void** d_patches_out, int64_t n_patches, int ps, int channels,
                             const double* uv0 /*[n][2] true location in patch px*/,
                             const int64_t* field_id /*[n] which smooth field (point id)*/,
                             uint64_t seed, double noise_sigma);
int pxr_device_free(pxr_ctx* ctx, void* dptr);
/* pinned host staging buffers for callers that want full PCIe bandwidth on the patch upload */
int pxr_host_alloc_pinned(void** out, size_t bytes);
int pxr_host_free_pinned(void* p);
int pxr_memcpy_d2h(pxr_ctx* ctx, void* host, const void* dev, size_t bytes);

/* ---- reference extraction ----------------------------------------------
 * replaces _bundle_adjustment.ReferenceExtractor.run (bindings.cc:28-34,172-177;
 * reference_extractor.h:171-318, irls_optim.h:23-71).
 *  refs_out    [n_points][C] fp64  reference descriptor (closest_to_robust_mean)
 *  src_obs_out [n_points]    index (into obs) of the observation picked as reference, -1 if none */
int pxr_refs_compute(pxr_ctx* ctx, const pxr_ba_desc* desc, const pxr_interp_config* interp,
                     int loss_type, double loss_scale, int iters,
                     double* refs_out, int64_t* src_obs_out, pxr_summary* summary);

/* descriptors of every observation at its current projection = ReferenceExtractor::FillDescriptorTrack
 * (reference_extractor.h:207-237), what Reference.observations holds with keep_observations=True (needed by
 * FindNearestReferences).  out_desc [n_obs][channels] fp64, in observation order. */
int pxr_obs_descriptors(pxr_ctx* ctx, const pxr_ba_desc* desc, const pxr_interp_config* interp, double* out_desc);

/* ---- cost maps (SURVEY 8(f) rank 1) ---------------------------------------
 * replaces _bundle_adjustment.CostMapExtractor.run (bundle_adjustment/bindings.cc:20-26,179-184;
 * costmap_extractor.h:93-228 Run/RunSubset, :230-358 FillPointCostmap) followed, on the caller's side,
 * by CostMapBundleOptimizer (costmap_bundle_optimizer.h:76-132) = pxr_ba_* on the returned
 * 3-channel patches with refs == NULL and l2_normalize == 0 (bundle_adjustment/main.py:262-281).
 * Config mirrors CostMapConfig (costmap_extractor.h:18-40) + the ReferenceConfig used by the
 * extractor's embedded ReferenceExtractor (reference_extractor.h:30-50). */
typedef struct pxr_costmap_config {
  int32_t loss_type;                /* pxr_loss_type, default TRIVIAL */
  double loss_scale;
  int32_t as_gradientfield;         /* 1: (cost, dcost/dr, dcost/dc), 0: cost only */
  int32_t compute_cross_derivative; /* must be 0 (4-channel variant not built) */
  int32_t apply_sqrt;
  double upsampling_factor;         /* must be 1.0 */
  int32_t compute_refs;             /* 1: run the reference extraction first, on the same upload */
  int32_t ref_loss_type;            /* CAUCHY 0.25, 100 IRLS iterations (bundle_adjustment/main.py:46-57) */
  double ref_loss_scale;
  int32_t ref_iters;
} pxr_costmap_config;
int pxr_default_costmap_config(pxr_costmap_config* cfg);
/*  desc        the feature problem (C-channel patches, geometry); desc->refs used when !compute_refs
 *  refs_io     [n_points][C] fp64: written when compute_refs, else read if desc->refs is NULL; may be NULL
 *  src_obs_out [n_points] or NULL (see pxr_refs_compute)
 *  out_host    [n_patches][ph][pw][OC] in desc->patch_dtype (the reference instantiates Run<dtype,dtype>), or NULL
 *  out_device  if not NULL receives a device pointer to the same array (release with pxr_device_free):
 *              feed it to pxr_ba_create with patches_on_device = 1 to skip the host round trip */
int pxr_costmaps_compute(pxr_ctx* ctx, const pxr_ba_desc* desc, const pxr_interp_config* interp,
                         const pxr_costmap_config* cfg, double* refs_io, int64_t* src_obs_out,
                         void* out_host, void** out_device, pxr_summary* summary);

/* ---- problem construction -------------------------------------------------------
 * replaces BundleOptimizer::SetUp / AddImageToProblem / AddPointToProblem / Parameterize{Points,Images,Cameras}
 * (bundle_adjustment/src/bundle_optimizer.h:139-165,247-331,335-442) and ReferenceExtractor::GetVisibleObservations
 * (bundle_adjustment/src/reference_extractor.h:171-205).  The reference walks a colmap::Reconstruction; the caller hands
 * the same data as a structure-of-arrays view (host memory, caller-owned).  Host code only, no device needed. */
typedef struct pxr_recon_view {
  int64_t n_images;
  const int64_t* image_id;          /* [n_images] */
  const int64_t* image_camera_id;   /* [n_images] */
  const int64_t* p2d_begin;         /* [n_images+1] offsets of the image's 2D points in p2d_point3D_id */
  const int64_t* p2d_point3D_id;    /* [p2d_begin[n_images]] 3D point of every 2D point, -1 = none */
  int64_t n_cameras;
  const int64_t* camera_id;         /* [n_cameras] */
  const int32_t* camera_model;      /* [n_cameras] COLMAP model id 0..6 */
  int64_t n_points;
  const int64_t* point3D_id;        /* [n_points] */
  const int64_t* track_begin;       /* [n_points+1] */
  const int64_t* track_image_id;    /* [track_begin[n_points]] */
  const int64_t* track_point2D_idx; /* [track_begin[n_points]] */
} pxr_recon_view;
/* colmap::BundleAdjustmentConfig as pixsfm::BundleAdjustmentSetup exposes it (bundle_adjustment/bindings.cc:81-111) */
typedef struct pxr_ba_setup_view {
  int64_t n_images; const int64_t* image_ids;
  int64_t n_const_poses; const int64_t* const_pose_ids;
  int64_t n_const_tvecs; const int64_t* const_tvec_ids; const uint8_t* const_tvec_masks;   /* bit k: tvec[k] constant */
  int64_t n_const_cameras; const int64_t* const_camera_ids;
  int64_t n_var_points; const int64_t* var_point_ids;
  int64_t n_const_points; const int64_t* const_point_ids;
} pxr_ba_setup_view;
typedef struct pxr_ba_build_options {
  int32_t refine_focal_length, refine_principal_point, refine_extra_params, refine_extrinsics;   /* BundleOptimizerOptions */
  int32_t min_track_length;          /* -1: off */
  int32_t mode;                      /* 0: bundle adjustment (setup required), 1: reference extraction */
  int64_t n_ref_points;              /* mode 1: the points to extract references for ...                        */
  const int64_t* ref_point_ids;
  const uint8_t* track_has_patch;    /* ... and, per track element, whether a feature patch exists (NULL: all do) */
} pxr_ba_build_options;
typedef struct pxr_problem_ir pxr_problem_ir;
int pxr_problem_build(const pxr_recon_view* rec, const pxr_ba_setup_view* setup, const pxr_ba_build_options* opt,
                      pxr_problem_ir** out);
int pxr_problem_sizes(const pxr_problem_ir* ir, int64_t* n_obs, int64_t* n_images, int64_t* n_cameras, int64_t* n_points);
/* observations sorted by point (stable), ids of the blocks in index order, index maps and constancy masks as
 * pxr_ba_desc takes them; any output may be NULL */
int pxr_problem_copy(const pxr_problem_ir* ir, int64_t* obs_point3D_id, int64_t* obs_image_id, int64_t* obs_point2D_idx,
                     int32_t* obs_img, int64_t* obs_pt, int64_t* image_ids, int64_t* camera_ids, int64_t* point_ids,
                     int32_t* img_cam, uint8_t* pose_const, uint8_t* tvec_const_mask, uint8_t* point_const,
                     uint32_t* cam_const_mask);
void pxr_problem_destroy(pxr_problem_ir* ir);

/* ---- descriptor interpolation ------------------------------------------------
 * replaces _features.PatchInterpolator(cfg).interpolate / interpolate_nodes for one node
 * (features/bindings.cc, features/src/patch_interpolator.h:125-135, dynamic_patch_interpolator.h): the bicubic
 * (+ L2-normalised) descriptor of patch item_patch[i] at image coordinates xy[i], the quantity
 * FindNearestReferences (localization/src/nearest_references.h:20-53) and find_feature_inliers compare.
 *  patches [n_patches][ph][pw][channels] host memory; corner/scale per patch; out_desc [n_items][channels] fp64 */
int pxr_interpolate_descriptors(pxr_ctx* ctx, const void* patches, int64_t n_patches, int32_t patch_dtype,
                                int32_t ph, int32_t pw, int32_t channels, const int32_t* corner, const double* scale,
                                double upsampling_factor, int64_t n_items, const int64_t* item_patch, const double* xy,
                                const pxr_interp_config* interp, double* out_desc);

/* ---- dense map -> patch slab -----------------------------------------------
 * replaces the sparse branch of FeatureExtractor.tensor_to_fmap + extract_patches_numpy
 * (features/extractor.py:176-201, features/extract_patches.py:36-44: the GPU -> CPU copy the authors flag as their
 * bottleneck): L2-normalise every pixel's C-vector (fp32, x / max(||x||, 1e-12)), cast, and gather one ps x ps window
 * per keypoint into the slab layout [n][ps][ps][C] the optimizers take.
 *  dense     one image's map, [C][H][W] (channels_first = 1, the CNN's NCHW) or [H][W][C]; host or device memory
 *  corners   host [n][2] (x0, y0), every window must lie inside the map (features/extractor.py:192-193 clamps them)
 *  out_host  optional host copy; out_device optional: receives a device pointer (release with pxr_device_free) that
 *            pxr_ba_create / pxr_ka_run accept as device patches or as a device patch block */
int pxr_extract_patches(pxr_ctx* ctx, const void* dense, int32_t dense_on_device, int32_t in_dtype, int32_t channels,
                        int32_t height, int32_t width, int32_t channels_first, const int32_t* corners, int64_t n_patches,
                        int32_t patch_size, int32_t l2_normalize, int32_t out_dtype, void* out_host, void** out_device);

/* ---- dense SIFT -> patch slab ----------------------------------------------
 * replaces the reference's `dsift` model (features/models/dsift.py: kornia's DenseSIFTDescriptor, stride 1, padding 1)
 * followed by the sparse branch of FeatureExtractor.tensor_to_fmap: the descriptor map of a grayscale image, each
 * pixel's C = num_ang_bins * num_spatial_bins^2 channels clipped, rootsift-mapped, optionally L2-normalised and cast,
 * computed by one fused kernel only where it is asked for.  The map is H' x W' with
 * H' = height + 2 (b / 2) - b + 1 + 3 - num_spatial_bins (b = spatial_bin_size), likewise W'.  Kornia parity is unverified.
 *  image      [height][width] uint8, host or device memory
 *  corners    host [n][2] (x0, y0) in map coordinates, every window inside the map: the slab [n][ps][ps][C];
 *             NULL: the whole map [H'][W'][C] (n_patches and patch_size are ignored).  A window of the slab is bit for bit
 *             the same window of the map.
 *  supported  num_ang_bins 4 or 8, num_spatial_bins 2 or 4, spatial_bin_size 1..8 (otherwise PXR_ERR_UNSUPPORTED)
 *  out_host / out_device as for pxr_extract_patches */
int pxr_dsift(pxr_ctx* ctx, const uint8_t* image, int32_t image_on_device, int32_t height, int32_t width,
              int32_t num_ang_bins, int32_t num_spatial_bins, int32_t spatial_bin_size, float clipval, int32_t rootsift,
              int32_t l2_normalize, const int32_t* corners, int64_t n_patches, int32_t patch_size, int32_t out_dtype,
              void* out_host, void** out_device);

/* ---- S2DNet -> patch slab -------------------------------------------------
 * replaces the reference's `s2dnet` model with num_layers 1 (features/models/s2dnet.py: VGG16's conv1_1, ReLU, conv1_2,
 * ReLU, then the adaptation layer 1x1 conv, ReLU, 5x5 conv, eval-mode BatchNorm) followed by the sparse branch of
 * FeatureExtractor.tensor_to_fmap: the 128-channel map of an RGB image, the size of the image, optionally L2-normalised
 * and cast, computed by one fused kernel only where it is asked for.  Convolutions 2-4 run on tensor cores with fp16
 * operands and fp32 accumulation; conv1_1 and the normalisation are fp32.
 *
 * pxr_s2dnet_weights_create uploads the weights once, in the kernel's layout.  `packed` holds n_floats = 247808 floats,
 * each tensor in PyTorch's layout, in this order:
 *   conv1_1 weight [64][3][3][3], bias [64]; conv1_2 weight [64][64][3][3], bias [64];
 *   1x1 weight [64][64][1][1], bias [64]; 5x5 weight [128][64][5][5], bias [128], both with the BatchNorm folded in.
 * A weight that is not finite, or one of layers 2-4 outside the fp16 range, is PXR_ERR_INVALID_ARGUMENT.  The weights
 * belong to the context's device; pxr_s2dnet_weights_destroy frees them (NULL is a no-op). */
typedef struct pxr_s2dnet_weights pxr_s2dnet_weights;
int pxr_s2dnet_weights_create(pxr_ctx* ctx, const float* packed, int64_t n_floats, pxr_s2dnet_weights** out);
void pxr_s2dnet_weights_destroy(pxr_s2dnet_weights* weights);

/*  image      [height][width][3] uint8 RGB, host or device memory
 *  corners    host [n][2] (x0, y0), every window inside the image: the slab [n][ps][ps][128]; NULL: the whole map
 *             [height][width][128] (n_patches and patch_size are ignored).  A window of the slab is bit for bit the same
 *             window of the map, and does not depend on the other windows of the call.
 *  out_host / out_device as for pxr_extract_patches.  Every argument is checked before anything is launched.
 *  PXR_ERR_NUMERIC: an intermediate activation is not finite in fp16 (|x| > 65504); no features are returned. */
int pxr_s2dnet(pxr_ctx* ctx, const pxr_s2dnet_weights* weights, const uint8_t* image, int32_t image_on_device,
               int32_t height, int32_t width, const int32_t* corners, int64_t n_patches, int32_t patch_size,
               int32_t l2_normalize, int32_t out_dtype, void* out_host, void** out_device);

/* ---- featuremetric KA ---------------------------------------------------
 * replaces _keypoint_adjustment.FeatureMetricKeypointOptimizer.run
 * (keypoint_adjustment/bindings.cc:17-34; featuremetric_keypoint_optimizer.h:50-202;
 * keypoint_optimizer.h:110-157). Keypoints are IN/OUT.
 * A problem may hold any number of keypoints; the normal equations are factored per connected component of its edges,
 * and a component may hold at most 80 variable keypoints (else PXR_ERR_UNSUPPORTED, keypoints untouched).  A problem
 * whose workspace does not fit in one block's shared memory is solved with its workspace in global memory; the
 * summary message reports how many did. */
typedef struct {
  int64_t n_keypoints;
  double* keypoints;            /* [n_keypoints][2] COLMAP image coords, in/out */
  const uint8_t* kp_const;      /* [n_keypoints] 1: constant (root nodes) */
  const int64_t* kp_patch;      /* [n_keypoints] patch index, or NULL: identity */
  int64_t n_edges;
  const int64_t* edge_src;      /* [n_edges] keypoint index */
  const int64_t* edge_dst;      /* [n_edges] */
  const double* edge_weight;    /* [n_edges] ScaledLoss weight (similarity) */
  const int32_t* edge_problem;  /* [n_edges] non-decreasing problem label (RunParallel groups) */
  int32_t n_problems;
  int64_t n_patches;
  const void* patches;
  int32_t patches_on_device;
  int32_t patch_dtype;
  int32_t ph, pw, channels;
  const int32_t* corner;        /* [n_patches][2] */
  const double* scale;          /* [n_patches][2] */
  double upsampling_factor;
  double bound;                 /* KeypointOptimizerOptions::bound, 4.0 from python */
  int32_t patches_are_sparse;   /* FeatureMap::IsSparse() */
  /* optional: patches given as blocks (one per FeatureMap numpy array, featuremap.cc:38-44) that are laid out
   * back to back on the device, as in pxr_ba_desc; each block may be host OR device memory */
  int32_t n_patch_blocks;
  const void* const* patch_block_ptrs;
  const int64_t* patch_block_counts;
  /* optional "query" mode (localization/src/single_query_keypoint_optimizer.h:84-203, residual
   * FeatureReference2DCostFunctor, residuals/src/feature_reference.h:14-62): when ref_desc != NULL EVERY edge is
   * (keypoint edge_src[e]) against the FIXED descriptor ref_desc[edge_dst[e]]; edge_dst then indexes ref_desc, not
   * keypoints.  The normal equations are block diagonal (2x2 per keypoint), so a problem may hold any number of
   * keypoints; all keypoints of one problem still share one trust region, as in the reference's single ceres::Problem. */
  const double* ref_desc;       /* [n_ref_desc][channels] fp64 or NULL */
  int64_t n_ref_desc;
} pxr_ka_desc;

int pxr_ka_run(pxr_ctx* ctx, const pxr_ka_desc* desc, const pxr_interp_config* interp,
               const pxr_solver_options* opt, pxr_summary* summary);

/* ---- batched query bundle adjustment ------------------------------------------
 * replaces a loop of _localization.QueryBundleOptimizer.run (localization/bindings.cc;
 * single_query_bundle_optimizer.h, query_bundle_optimizer.h SolveProblem): N independent queries, each one image's
 * pose (QuaternionManifold rotation + translation) and optionally some of its camera's intrinsics, refined against
 * fixed 3D points and fixed fp64 reference descriptors.  One CTA solves one query end to end (csrc/pxr_qba.cu); every
 * per-query decision is the one pxr_ba_run takes on that query alone (one free image, constant points, no inner
 * iterations).  A query's results do not depend on which other queries share its launch. */
typedef struct {
  int32_t n_queries;
  /* per query */
  const int32_t* cam_model;       /* [n_queries] pxr_camera_model */
  double* cam_params;             /* [n_queries][PXR_MAX_CAM_PARAMS] in/out */
  const uint32_t* cam_const_mask; /* [n_queries] bit i: param i constant; 0xFFFFFFFF: camera constant */
  double* qvec;                   /* [n_queries][4] in/out (w,x,y,z), world->camera */
  double* tvec;                   /* [n_queries][3] in/out */
  const int64_t* obs_begin;       /* [n_queries+1] non-decreasing: query q owns residual blocks [obs_begin[q], obs_begin[q+1]) */
  /* per residual block (a correspondence compared with several descriptors gives several blocks) */
  const double* xyz;              /* [n_obs][3] constant 3D point */
  const int64_t* obs_patch;       /* [n_obs] patch index within its query's patch block */
  const double* refs;             /* [n_obs][channels] fixed reference descriptor */
  /* patches: one block per query, [patch_counts[q]][ph][pw][channels], each in host OR device memory (a device block is
   * read in place, never copied) */
  const void* const* patch_blocks;   /* [n_queries] */
  const int64_t* patch_counts;       /* [n_queries] */
  const int32_t* corner;          /* [sum patch_counts][2] (x0,y0), query blocks back to back */
  const double* scale;            /* [sum patch_counts][2] */
  double upsampling_factor;
  int32_t ph, pw, channels, patch_dtype;
  /* bytes a wave may upload (host patch blocks, descriptors, points, per-query state); 0: half of the free device
   * memory at the call */
  double max_wave_bytes;
} pxr_qba_desc;

typedef struct {
  int32_t status;                 /* PXR_OK, or PXR_ERR_NUMERIC: initial cost not finite (parameters untouched) */
  int32_t num_residual_blocks;    /* 0: not solved, parameters untouched */
  double initial_cost;
  double final_cost;              /* cost of the parameters written back (the lowest-cost iterate) */
  int32_t num_iterations;         /* iteration summaries recorded, as pxr_summary::num_iterations */
  int32_t num_successful_steps;
  int32_t num_unsuccessful_steps;
  int32_t termination_type;       /* as pxr_summary */
  int64_t block_evaluations;      /* residual-block evaluations the kernel ran (blocks x passes) */
} pxr_qba_result;

/* Solves every query and writes the refined qvec / tvec / cam_params back into the desc arrays.
 *  results     [n_queries]
 *  iterations  [n_queries][iterations_capacity] or NULL: per-query iteration summaries (iteration_time_s is 0)
 *  n_waves     or NULL: launches made (one per wave)
 *  total       or NULL: h2d_bytes, kernel_launches, solve and total time, summed costs / steps, message
 * Options: use_inner_iterations must be 0 (PXR_ERR_INVALID_ARGUMENT: no free points), ITERATIVE_SCHUR is
 * PXR_ERR_UNSUPPORTED, `deterministic` is accepted and changes nothing (the path always sums in a fixed order).
 * Queries are packed in order into waves of at most max_wave_bytes uploaded bytes (a larger query gets a wave of its
 * own); the next wave's upload runs while the current one solves (two wave buffers when both fit in free device
 * memory, else one, reused once the previous wave's outputs are back), and the interrupt callback is polled between
 * waves.
 * Arguments are checked before the context: a NULL or malformed desc is reported without a device. */
int pxr_qba_run(pxr_ctx* ctx, const pxr_qba_desc* desc, const pxr_interp_config* interp, const pxr_solver_options* opt,
                pxr_qba_result* results, pxr_iteration_summary* iterations, int32_t iterations_capacity, int32_t* n_waves,
                pxr_summary* total);
/* The wave plan pxr_qba_run uses: wave_begin [n_queries+1] receives the first query of every wave (entries past
 * *n_waves are left alone), wave_bytes [n_queries] (or NULL) each wave's upload.  Host computation with two device
 * queries: with max_wave_bytes 0 the budget is half of the free device memory (PXR_ERR_NO_DEVICE without a device),
 * and each patch block's placement is asked from the CUDA runtime (a block it cannot place counts as host memory). */
int pxr_qba_plan_waves(const pxr_qba_desc* desc, int32_t* wave_begin, int32_t* n_waves, double* wave_bytes);
/* Evaluates every query at the given parameters with the solver's device code and moves nothing (tests).
 *  cost [n_queries]; H [n_queries][18][18] the lower triangle of J^T J in the query's tangent columns (3 rotation,
 *  3 translation, then the free intrinsics in parameter order; the rest 0); g [n_queries][18] J^T r;
 *  xy [n_obs][2] projected image point; rec [n_obs][8] s, G^T r (2), G^T G (3), 0, 0 as pxr_ba_evaluate.  Any output
 *  may be NULL.  All queries run in one launch. */
int pxr_qba_debug_linearize(pxr_ctx* ctx, const pxr_qba_desc* desc, const pxr_interp_config* interp,
                            const pxr_solver_options* opt, double* cost, double* H, double* g, double* xy, double* rec);

/* ---- batched absolute pose estimation ------------------------------------------
 * pycolmap 0.4's absolute_pose_estimation (COLMAP 3.8 EstimateAbsolutePose + RefineAbsolutePose) for N independent
 * queries: LO-RANSAC over P3P minimal samples (Lambda Twist), then a Cauchy-robust LM refinement of the pose (and,
 * when asked, of the focal length / extra parameters) over the RANSAC inliers.  One CTA estimates one query
 * (csrc/pxr_pnp.cu); a query's results depend only on its own inputs and seed, never on the other queries of the call.
 *
 * RANSAC, precisely (tests restate it on the host and draw the same samples):
 *  - every 2D point goes once to the normalised image plane (ImageToWorld); thr = max_error / mean focal length; the
 *    residual of a correspondence under (R, t) is, with (x, y, z) = R X + t (sums left to right, no fused
 *    multiply-add) and iz = 1 / z, (x iz - u)^2 + (y iz - v)^2; it is an inlier when z > DBL_EPSILON and the residual
 *    <= thr^2.  Support = (number of inliers, sum of their residuals): more inliers wins, then the smaller sum, then
 *    the lower (trial, solution) index.
 *  - trials run in rounds of PXR_PNP_ROUND_TRIALS; trial t of a query with n correspondences draws words
 *    w_d = splitmix64(splitmix64(seed) ^ (t << 8) ^ d), d = 0, 1, ... 63, takes index ((w_d >> 32) * n) >> 32 from
 *    each and keeps the first three distinct ones (fewer than three after 64 draws: the trial has no hypothesis);
 *    splitmix64(x): z = x + 0x9E3779B97F4A7C15, z = (z ^ z >> 30) * 0xBF58476D1CE4E5B9,
 *    z = (z ^ z >> 27) * 0x94D049BB133111EB, z ^ z >> 31 (mod 2^64).  Trials t >= max_num_trials are not run.
 *  - P3P gives up to four hypotheses per trial, solution s of trial t has index 4 t + s; after a round the best
 *    hypothesis of the round replaces the best so far when its support is better, and then, when it has more than 3
 *    inliers, local optimisation runs: 3 Gauss-Newton steps on the 6-dof pose over that hypothesis' inliers in the
 *    normalised plane, kept when its support is better still.  (COLMAP's LO-RANSAC re-estimates with EPnP there.)
 *  - after every round the required trial count is COLMAP's ceil(log(1 - confidence) / log(1 - ratio^3) *
 *    dyn_num_trials_multiplier), ratio = inliers / n, clamped to [min_num_trials, max_num_trials]; the query stops when
 *    the trials run reach it, so up to PXR_PNP_ROUND_TRIALS - 1 trials more than COLMAP's can run.
 *  - success: n >= 3 and the best support has >= 3 inliers and inliers / n >= min_inlier_ratio. */
#define PXR_PNP_ROUND_TRIALS 128

typedef struct {
  int32_t n_queries;
  const int64_t* corr_begin;      /* [n_queries+1] non-decreasing from 0: query q owns correspondences
                                     [corr_begin[q], corr_begin[q+1]) */
  const double* points2D;         /* [n_corr][2] pixels, COLMAP convention (pixel centres at +0.5) */
  const double* points3D;         /* [n_corr][3] */
  const int32_t* cam_model;       /* [n_queries] pxr_camera_model */
  double* cam_params;             /* [n_queries][PXR_MAX_CAM_PARAMS] in/out: written only when refinement refines
                                     intrinsics and the query succeeds */
  const uint64_t* seed;           /* [n_queries] */
  double* qvec;                   /* [n_queries][4] out (w,x,y,z) world->camera, written when the query succeeds */
  double* tvec;                   /* [n_queries][3] out */
  uint8_t* inlier_mask;           /* [n_corr] out: inliers of the returned pose (recomputed after refinement) */
} pxr_pnp_desc;

typedef struct {
  /* AbsolutePoseEstimationOptions / RANSACOptions */
  double max_error;               /* pixels */
  double min_inlier_ratio;
  int32_t min_num_trials, max_num_trials;
  double confidence;
  double dyn_num_trials_multiplier;
  int32_t estimate_focal_length;  /* must be 0 (PXR_ERR_UNSUPPORTED) */
  /* AbsolutePoseRefinementOptions */
  int32_t refine;                 /* 0: return the RANSAC pose */
  double gradient_tolerance;
  int32_t max_num_iterations;
  double loss_function_scale;     /* Cauchy */
  int32_t refine_focal_length, refine_extra_params;
  /* ceres' function / parameter tolerances, which COLMAP leaves at 1e-6 / 1e-8 (pycolmap has no name for them) */
  double function_tolerance, parameter_tolerance;
} pxr_pnp_options;

typedef struct {
  int32_t status;                 /* PXR_OK, or PXR_ERR_NUMERIC: refinement's initial cost not finite (pose and camera
                                     untouched, success 0) */
  int32_t success;
  int32_t num_inliers;            /* of the returned pose */
  int32_t num_trials;             /* RANSAC trials run */
  int32_t best_trial, best_solution;   /* the winning hypothesis (-1 when none) */
  int32_t local_optimized;        /* the winner is its local optimisation */
  int32_t num_iterations;         /* refinement: as pxr_qba_result */
  int32_t termination_type;
  double initial_cost, final_cost;
} pxr_pnp_result;

/* Fills opt with pycolmap 0.4's defaults (max_error 12 px). */
void pxr_default_pnp_options(pxr_pnp_options* opt);
/* Estimates every query in one launch of the RANSAC kernel and one of the refinement kernel.  results [n_queries];
 * total (or NULL): kernel time, h2d_bytes, kernel launches, message.  Arguments are checked before the context: a
 * NULL or malformed desc, a non-monotone corr_begin and an unknown camera model are PXR_ERR_INVALID_ARGUMENT /
 * PXR_ERR_UNSUPPORTED without a device; so is estimate_focal_length != 0 (PXR_ERR_UNSUPPORTED). */
int pxr_pnp_run(pxr_ctx* ctx, const pxr_pnp_desc* desc, const pxr_pnp_options* opt, pxr_pnp_result* results,
                pxr_summary* total);
/* Device code on its own (tests): ImageToWorld of n pixels xy [n][2] -> out [n][2]; P3P of n triplets of normalised
 * image points x [n][3][2] and world points X [n][3][3] -> poses [n][4][7] (qvec with w >= 0, tvec) and n_sol [n]. */
int pxr_pnp_debug_image_to_world(pxr_ctx* ctx, int32_t model, const double* params, int64_t n, const double* xy,
                                 double* out);
int pxr_pnp_debug_p3p(pxr_ctx* ctx, int64_t n, const double* x, const double* X, double* poses, int32_t* n_sol);

/* ---- point triangulation from known poses ------------------------------------------
 * COLMAP's point_triangulator as hloc's triangulation drives it, with poses and intrinsics fixed (csrc/pxr_tri.cu).
 *  pxr_tri_verify  geometric verification of matches (hloc's geometric_verification): both keypoints go to the
 *                  normalised plane (ImageToWorld), E = [t]x R of cam1_from_cam0, and the two point-to-epipolar-line
 *                  distances d0 = |x1^T E x0| / |(E^T x1)_{0,1}|, d1 = |x1^T E x0| / |(E x0)_{0,1}|; a match is kept when
 *                  d_k <= noise_k * max_error / mean focal length of camera k (COLMAP's CamFromImgThreshold).
 *  pxr_tri_run     robust triangulation of every track, one warp per track.  Each observation becomes a world ray
 *                  (unit direction d, camera centre c).  Hypotheses are observation pairs: all n(n-1)/2 of them in
 *                  lexicographic order when that is <= tri_max_pairs, else tri_max_pairs sampled ones, hypothesis h
 *                  drawing words w_k = splitmix64(s0 ^ (h << 8) ^ k), k = 0, 1, ... 63, s0 = splitmix64(seed ^
 *                  splitmix64(key)), key = track_key[t] (or t when NULL), taking index ((w_k >> 32) * n) >> 32 from each
 *                  and keeping the first two distinct ones (none after 64 draws: no hypothesis).  A pair whose rays are
 *                  less than min_angle apart makes no hypothesis.  Its point is the midpoint least-squares point
 *                  X = (sum (I - d d^T))^-1 sum (I - d d^T) c.  The error of an observation is the angle between d and
 *                  X - c, in [0, 180]; an inlier has (X - c).d > 0 (in front of the camera along its ray) and error <=
 *                  create_max_angle_error; an observation that is not in front scores as one at the threshold.  Score: MSAC sum min(e^2, tau^2); the lowest score wins, ties to the lowest
 *                  hypothesis index.  The winner's inliers S0 give X1 = midpoint(S0); when the inliers S1 of X1 differ
 *                  from S0, X2 = midpoint(S1).  The result is the last point and the set it was fitted to.
 *  pxr_tri_evaluate  the per-observation pixel errors and per-track angles of given points, no RANSAC.
 * Angles are in degrees.  The triangulation angle of a point is COLMAP's CalculateTriangulationAngle: the angle at X
 * between X - c_i and X - c_j, folded to min(a, 180 - a), largest over the pairs of the set (inliers in run mode, every
 * observation in evaluate mode). */
typedef struct {
  int32_t n_cameras;
  const int32_t* cam_model;       /* [n_cameras] pxr_camera_model */
  const double* cam_params;       /* [n_cameras][PXR_MAX_CAM_PARAMS] */
  int32_t n_images;
  const int32_t* img_cam;         /* [n_images] camera index */
  const double* qvec;             /* [n_images][4] (w,x,y,z) world->camera */
  const double* tvec;             /* [n_images][3] */
  int64_t n_tracks;
  const int64_t* track_begin;     /* [n_tracks+1] from 0, >= 2 observations per track */
  const int64_t* track_key;       /* [n_tracks] sample-stream key, or NULL (the track index) */
  const int32_t* obs_img;         /* [n_obs] image index */
  const double* obs_xy;           /* [n_obs][2] pixels, COLMAP convention */
} pxr_tri_desc;

typedef struct {
  double min_angle;               /* degrees: hypothesis pairs and points below it are rejected */
  double create_max_angle_error;  /* degrees: inlier threshold of the angular error */
  int32_t tri_max_pairs;          /* hypotheses of a track at most (exhaustive up to this many pairs) */
  uint64_t seed;
} pxr_tri_options;

enum { PXR_TRI_OK = 0, PXR_TRI_TOO_FEW_INLIERS = 1, PXR_TRI_ANGLE_TOO_SMALL = 2 };

/* min_angle 1.5, create_max_angle_error 2 (COLMAP's IncrementalTriangulator), tri_max_pairs 1024, seed 0 */
void pxr_default_tri_options(pxr_tri_options* opt);
/* Verifies n_matches matches in one launch (tracks in desc are not read).  match_img [n][2] image indices,
 * match_xy [n][4] (x0, y0, x1, y1) pixels, match_noise [n][2] keypoint noise (pixels) of each side; keep [n] and
 * err [n][2] (normalised-plane distances d0, d1) out. */
int pxr_tri_verify(pxr_ctx* ctx, const pxr_tri_desc* desc, int64_t n_matches, const int32_t* match_img,
                   const double* match_xy, const double* match_noise, double max_error, uint8_t* keep, double* err,
                   pxr_summary* total);
/* Triangulates every track.  Out: xyz [n_tracks][3], status [n_tracks] (PXR_TRI_*), n_inliers [n_tracks],
 * tri_angle [n_tracks] (of the inliers), obs_inlier [n_obs], obs_error [n_obs] pixel reprojection error of the
 * returned point (+inf behind the camera).  A track's results depend only on its own observations, key and seed. */
int pxr_tri_run(pxr_ctx* ctx, const pxr_tri_desc* desc, const pxr_tri_options* opt, double* xyz, int32_t* status,
                int32_t* n_inliers, double* tri_angle, uint8_t* obs_inlier, double* obs_error, pxr_summary* total);
/* obs_error [n_obs] and tri_angle [n_tracks] (every observation) of the points xyz [n_tracks][3]. */
int pxr_tri_evaluate(pxr_ctx* ctx, const pxr_tri_desc* desc, const double* xyz, double* obs_error, double* tri_angle,
                     pxr_summary* total);
/* total (or NULL): solve_time_s = device time of the kernels (CUDA events), total_time_s, kernel launches, h2d_bytes.
 * All three check their arguments before the context: NULL arrays, negative counts, an unknown camera model, an index
 * out of range, a track_begin that does not start at 0 or is not increasing by >= 2, bad options:
 * PXR_ERR_INVALID_ARGUMENT / PXR_ERR_UNSUPPORTED without a device. */

/* ---- batched query keypoint adjustment ------------------------------------------
 * replaces a loop of _localization.QueryKeypointOptimizer.run: N independent queries, each one problem of pxr_ka_run's
 * query mode (every residual block = one keypoint against one fixed descriptor).  One CTA solves one query; the
 * keypoints written back are those pxr_ka_run writes for that query alone. */
typedef struct {
  int32_t n_queries;
  /* per query */
  const int64_t* kp_begin;        /* [n_queries+1] non-decreasing: query q owns keypoints [kp_begin[q], kp_begin[q+1]) */
  const void* const* patch_blocks;   /* [n_queries] [patch_counts[q]][ph][pw][channels], host OR device memory */
  const int64_t* patch_counts;       /* [n_queries] */
  const uint8_t* patches_are_sparse; /* [n_queries] FeatureMap::IsSparse() */
  /* per keypoint */
  double* keypoints;              /* [n_kp][2] in/out */
  const int64_t* kp_patch;        /* [n_kp] patch index within its query's block */
  const int64_t* desc_begin;      /* [n_kp+1] non-decreasing: keypoint k has one residual block per descriptor in
                                     [desc_begin[k], desc_begin[k+1]) */
  const double* descs;            /* [desc_begin[n_kp]][channels] fixed fp64 descriptors */
  const int32_t* corner;          /* [sum patch_counts][2], query blocks back to back */
  const double* scale;            /* [sum patch_counts][2] */
  double upsampling_factor;
  double bound;                   /* KeypointOptimizerOptions::bound */
  int32_t ph, pw, channels, patch_dtype;
  /* bytes a wave may upload (patch blocks, host or device, descriptors and per-query state); 0: half of the free device
   * memory at the call */
  double max_wave_bytes;
} pxr_qka_desc;

typedef struct {
  int32_t status;                 /* PXR_OK, or PXR_ERR_NUMERIC: initial cost not finite (the keypoints are still written
                                     back as pxr_ka_run writes them: projected onto their bounds, not moved) */
  int32_t num_residual_blocks;    /* 0: not solved, keypoints untouched */
  double initial_cost;
  double final_cost;
  int32_t num_successful_steps;
  int32_t num_unsuccessful_steps;
  int32_t num_iterations;
  int32_t termination_type;       /* as pxr_summary */
} pxr_qka_result;

/* Solves every query and writes the refined keypoints back into desc->keypoints.  results [n_queries]; n_waves and
 * total (summed costs / steps, h2d_bytes, kernel launches, times, message) may be NULL.  Supported (dtype, channels):
 * those of pxr_ka_run's query mode (fp16 8/16/32/64/128, fp32 and fp64 16/128); use_float_simd is
 * PXR_ERR_UNSUPPORTED before anything is touched.  Queries are packed in order into waves of at most max_wave_bytes
 * uploaded bytes (a larger query gets a wave of its own; a wave also ends where the queries' box constraint changes,
 * i.e. between a sparse and a dense map when bound <= 0); device patch blocks are copied into the wave's slab and
 * count toward its bytes.  The next wave's upload runs while the current one solves (two wave buffers when both fit
 * in free device memory, else one), and the interrupt callback is polled between waves.
 * Arguments are checked before the context: a NULL or malformed desc is reported without a device. */
int pxr_qka_run(pxr_ctx* ctx, const pxr_qka_desc* desc, const pxr_interp_config* interp, const pxr_solver_options* opt,
                pxr_qka_result* results, int32_t* n_waves, pxr_summary* total);

/* ---- nearest candidate descriptor ------------------------------------------------
 * replaces FindNearestReferences (localization/src/nearest_references.h:20-53) and the descriptor test of
 * find_feature_inliers for many queries at once: item i is the descriptor of patch item_patch[i] of query
 * item_query[i]'s block at image point xy[i] (the K1 interpolation of pxr_interpolate_descriptors, bit for bit),
 * compared with the candidate rows [cand_begin[i], cand_end[i]) of cand [n_cand][channels] (fp64); items may share
 * rows (a table of every 3D point's stored observations, uploaded once, serves every query).
 *  best [n_items]     the first candidate row with the smallest squared L2 distance (fp64, fixed order; a NaN
 *                     distance counts as smallest, as numpy's argmin), -1 when the range is empty
 *  d_min [n_items]    that distance (+inf for an empty range); may be NULL
 *  out_desc [n_items][channels] the interpolated descriptors; may be NULL
 * patch blocks, corner and scale as in pxr_qba_desc; cand_on_device = 1 reads cand in place in device memory. */
int pxr_query_match_run(pxr_ctx* ctx, int32_t n_queries, const void* const* patch_blocks, const int64_t* patch_counts,
                        const int32_t* corner, const double* scale, double upsampling_factor, int32_t ph, int32_t pw,
                        int32_t channels, int32_t patch_dtype, int64_t n_items, const int32_t* item_query,
                        const int64_t* item_patch, const double* xy, const int64_t* cand_begin,
                        const int64_t* cand_end, const double* cand,
                        int64_t n_cand, int32_t cand_on_device, const pxr_interp_config* interp, int64_t* best,
                        double* d_min, double* out_desc);

/* ---- host-side integer algorithms (bit-exact targets) -------------------
 * replace _base.compute_track_labels / compute_score_labels / compute_root_labels
 * (base/src/graph.cc:126-256) and keypoint_adjustment/main.py:13-57 find_problem_labels. */
int pxr_graph_track_labels(int64_t n_nodes, const int32_t* node_image, int64_t n_edges,
                           const int64_t* e_src, const int64_t* e_dst, const double* e_sim,
                           int64_t* track_labels_out);
int pxr_graph_score_labels(int64_t n_nodes, int64_t n_edges, const int64_t* e_src,
                           const int64_t* e_dst, const double* e_sim,
                           const int64_t* track_labels, double* scores_out);
int pxr_graph_root_labels(int64_t n_nodes, const int64_t* track_labels, const double* scores,
                          uint8_t* is_root_out);
int pxr_ka_problem_labels(int64_t n_nodes, const int64_t* track_labels, int32_t max_per_problem,
                          int32_t* problem_labels_out, int32_t* n_problems_out);
/* BA: reference bundle_adjustment/main.py:21-27 (label = p3D_id // max_tracks_per_problem) lives in Python. */

/* Multi-GPU sharding plan: contiguous point ranges balanced by observation count (SURVEY §8e). */
int pxr_shard_points(int64_t n_points, int64_t n_obs, const int64_t* obs_pt, int world,
                     int64_t* point_begin_out /*[world+1]*/, int64_t* obs_begin_out /*[world+1]*/);
/* KA: the packed problems are independent (ParallelOptimizer::RunParallel, base/src/parallel_optimizer.h:77-211,
 * runs one task per label), so ranks take whole problems and need no collective.  `weight` = cost of a problem
 * (patch bytes or edge count); heaviest-first onto the least loaded rank, deterministic. */
int pxr_shard_ka_problems(int32_t n_problems, const int64_t* weight, int world, int32_t* rank_of_problem_out);

#ifdef __cplusplus
}
#endif
#endif /* PXR_H_ */
