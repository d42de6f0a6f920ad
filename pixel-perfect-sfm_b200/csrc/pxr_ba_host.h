// pxr_ba_host.h — host-side state of one featuremetric BA problem resident on the device.
#pragma once
#include <array>
#include <cstdlib>
#include <chrono>
#include <string>
#include <functional>
#include <thread>
#include <limits>
#include <algorithm>
#include <utility>
#include <vector>

#include "pxr_ba_kernels.cuh"
#include "pxr_chol.cuh"
#include "pxr_fm_eval.cuh"
#include "pxr_fm_small.cuh"
#include "pxr_geo.cuh"
#include "pxr_inner.cuh"
#include "pxr_internal.h"
#include "pxr_lm.cuh"
#include "pxr_pcg.cuh"
#include "pxr_sparse_schur.cuh"
#include "pxr_block.cuh"

namespace pxr {

int fm_supported(int dtype, int C);
int fm_max_partials(pxr_ctx* ctx);
int launch_fm_eval(pxr_ctx* ctx, int dtype, int C, int mode, bool float_simd, const FmEvalArgs& a, int* n_partials);

struct LMState {
  bool started = false, finished = false, pending_finalize = false, inner_enabled = false;
  TrustRegion tr;
  bool gmax_pending = false;       // block mode, several ranks: max |g| of the current point arrives with the next all-reduce
  bool best_is_current = true;     // non-monotonic steps: the lowest-cost iterate lives in BA::best_* when false
  double x_cost = 0, initial_cost = 0, minimum_cost = 0;
  int n_succ = 0, n_unsucc = 0, n_inner = 0, term = 1;
  pxr_iteration_summary it;
  std::vector<pxr_iteration_summary> its;
  std::string message;
  std::chrono::steady_clock::time_point it_start;
};

// What the host learns about one LM step: BA::lm_trial's read-back
struct LMTrial {
  bool interrupted = false, valid = false;
  double model_cost_change = 0;
  double cost = 0, inner_cost = 0;                 // the trial cost, and the cost after the inner iterations
  double step_sq[2] = {}, x_sq[2] = {};            // squared camera / point parts of |step| and |x|
  double inner_step_sq[2] = {};                    // the same parts of the step after the inner iterations
  double gmax = 0;                                 // block mode: max |g| at the current point, from the exchange
};

struct BA {
  pxr_ctx* ctx = nullptr;
  LMState lm;
  // optional CUDA-event timing of the LM stages (pxr_ba_kernel_timing): 0 K1 cost-only, 1 K1 Jacobian,
  // 2 projection K0, 3 block build, 4 damping+Schur assembly, 5 Cholesky factor, 6 Cholesky solve,
  // 7 back-substitution+model cost, 8 manifold plus, 9 inner iterations, 10 cost reduction, 11 misc
  static constexpr int kNumStages = 12;
  bool time_kernels = false;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> timed[kNumStages];
  struct StageScope {
    BA* b; int id; cudaEvent_t e0 = nullptr, e1 = nullptr;
    StageScope(BA* b_, int id_) : b(b_), id(id_) {
      if (b->time_kernels && cudaEventCreate(&e0) == cudaSuccess && cudaEventCreate(&e1) == cudaSuccess) cudaEventRecord(e0, b->ctx->stream);
    }
    ~StageScope() { if (e0 && e1) { cudaEventRecord(e1, b->ctx->stream); b->timed[id].push_back({e0, e1}); } }
  };
  pxr_interp_config interp;
  pxr_solver_options opt;
  // sizes
  int n_cameras = 0, n_images = 0, K = 0, C = 0, ph = 0, pw = 0, dtype = 0;
  int64_t n_points = 0, n_obs = 0, n_patches = 0, nl = 0;
  int nc = 0, dcmax = 0, juv_stride = 0, img_dc_max = 0;
  double ups = 1.0;
  bool has_refs = false;
  // geometric (reprojection-error) handle (pxr_ba_create_geometric): no patch slab, K0 in the identity patch frame
  // writes the projection to geo_xy, K1 is geo_eval_kernel against the observed keypoints geo_target; C = 2
  bool geometric = false;
  DevBuf<double> geo_target, geo_xy;
  double h2d_bytes = 0;
  // host layout
  std::vector<int32_t> h_pose_off, h_intr_off;
  std::vector<int64_t> h_point_off, h_pt_begin;
  // device: topology
  DevBuf<int32_t> obs_img, img_cam, cam_model, pose_off, intr_off, corner, Wcols, Wdc;
  DevBuf<int64_t> obs_pt, obs_patch, point_off, pt_begin;
  DevBuf<uint32_t> cam_mask;
  DevBuf<uint8_t> tmask;
  PatchSlab patches_owned;
  DevBuf<double> scale, refs;
  const uint8_t* d_patches = nullptr;
  // device: parameters (two sets: current / candidate)
  DevBuf<double> cam[2], q[2], t[2], X[2];
  DevBuf<double> best_cam, best_q, best_t, best_X;   // use_nonmonotonic_steps: snapshot of the lowest-cost iterate
  int save_best(int set);
  int cur = 0;
  // device: per-observation and linearisation
  // uv/obs_out/juv hold the linearisation at the CURRENT point; every trial-point evaluation (cost-only,
  // speculative Jacobian, inner iterations) runs on the *_alt set (swap_sets()) so a rejected step never
  // clobbers what the next compute_step reads.
  DevBuf<double> uv_alt, obs_out_alt, juv_alt;
  void swap_sets() { std::swap(uv.p, uv_alt.p); std::swap(uv.n, uv_alt.n); std::swap(obs_out.p, obs_out_alt.p); std::swap(obs_out.n, obs_out_alt.n); std::swap(juv.p, juv_alt.p); std::swap(juv.n, juv_alt.n); }
  DevBuf<double> ar_buf;             // staging for the fused [diag | gc] all-reduce
  DevBuf<double> gc_local;           // multi-GPU: this rank's partial gradient (gc holds the global one)
  DevBuf<double> uv, obs_out, juv, Hcc, gc, Hpp, gp, W, S, rhs, diag, jscale, D2, delta, partials, scalars;
  DevBuf<int> flags;
  DevBuf<double> rdiag;
  // ITERATIVE_SCHUR (PCG) workspace
  bool use_pcg = false;
  DevBuf<double> cg_Minv, cg_z, cg_p, cg_q, cg_r, cg_x, cg_tmp, cg_part;   // cg_part: per-CTA dot-product partials (fixed-order sums)
  DevBuf<int32_t> cg_blk_off, cg_blk_dim, cg_row_off, cg_row_dim;
  DevBuf<CGState> cg_state;
  int cg_nblk = 0, last_linear_iterations = 1;
  int pcg_solve();
  int solve_reduced();               // stage 5 of compute_step: S delta_c = rhs by PCG or the dense Cholesky
  int run_cg(const std::function<int(const double*, double*)>& spmv);
  // implicit block-sparse reduced system (pxr_sparse_schur.cuh): no nc x nc array is ever allocated
  // debugging / A-B switches, read from the environment once in create()
  struct EnvFlags { bool pcg_sparse = false, build_atomic = false, chol_multikernel = false, chol_test_abort = false,
                         cg_multi = false, no_speculation = false, build_staged = true, project_staged = true; std::string chol_trace; } env;
  bool sparse_schur = false;
  int ss_n_keys = 0;
  std::vector<int32_t> h_img_cols, h_img_pd, h_img_pose_blk, h_img_cam_blk, h_img_cam;
  DevBuf<int32_t> ss_img_cols, ss_img_pd, ss_img_pose_blk, ss_img_cam_blk, ss_key_a, ss_key_b, ss_chunk_key;
  DevBuf<uint8_t> ss_key_self;
  DevBuf<double> ss_Himg, ss_Bk, ss_Dblk;
  SparseSchur sparse();
  int pcg_solve_sparse();
  // ---- block mode (pxr_block.cuh, pxr_ba_block.cu): image-block assembly into ONE packed buffer, ONE all-reduce per
  // LM iteration, everything after it deterministic; scalar decisions travel through the peer mailboxes
  bool block_mode = false;
  DevBuf<double> pack_local, pack_global;          // world == 1: pack_global stays empty and aliases pack_local
  size_t pk_off_B = 0, pk_off_rhs = 0, pk_off_gc = 0, pk_off_slots = 0, pk_n = 0;
  double* pk(bool global) { return (global && pack_global.p) ? pack_global.p : pack_local.p; }
  SparseSchur sparse_blk(bool global);
  std::vector<int32_t> h_key_a, h_key_b; std::vector<uint8_t> h_key_self;     // global key list (host copy)
  DevBuf<int64_t> gmS_dest, gmS_ptr, dg_ptr, gmD_dest, gmD_ptr, br_chunk_begin, br_cols_ptr;
  DevBuf<int32_t> gmS_src, dg_src, gmD_src, br_chunk_img, br_ent_key, br_cols_src;
  DevBuf<uint8_t> br_chunk_first;
  DevBuf<double> br_ypart, mb_in, mb_out;
  int64_t gmS_rows = 0, gmD_rows = 0, br_n_chunks = 0;
  // deterministic assembly (pxr_solver_options.deterministic): block mode + fixed-order reductions of the chunk partials
  bool deterministic = false;
  std::vector<int64_t> h_img_chunk_begin;           // [n_images+1] chunks of every image in io order (create())
  DevBuf<int64_t> det_img_chunk_begin, det_key_chunk_begin;
  DevBuf<double> det_cam_part, det_pair_part, det_gimg, det_rimg, det_scal_part;
  bool jscale_c_pending = false;
  bool blk_lag_gmax = false;                       // world > 1: max |g| of the current point is known after the next all-reduce
  int block_setup();                               // global keys, gather maps, block rows
  int build_block();
  int compute_step_block(double radius);
  int compute_step_block_sync(double radius, bool* valid, double* model_cost_change);   // + exchange + read-back (debug entry points)
  int global_cost_block(double* cost_out);         // scalars[0] summed over the ranks
  int pcg_solve_block();
  int finish_gmax_block();
  void pack_scalars(int stage, int interrupted = 0);   // blk_pack_scalars_kernel: this rank's scalars -> mb_in
  int exchange_scalars(int n_sum);                 // mb_in -> mb_out (peer mailboxes, or NCCL when they are unavailable)
  std::vector<int32_t> h_chunk_key_local;
  std::vector<int64_t> h_key_code_local;           // local key codes in build order (set by build_schur_pairs)
  int pcg_setup_blocks();
  int launch_schur_pairs(const BADev& d);
  int launch_sp_schur_pairs(const BADev& d, double* Bk, double* rhs_out, double* part);
  cudaGraphExec_t chol_graph_exec = nullptr;
  int64_t chol_graph_kernels = 0;
  bool chol_multikernel = false, chol_force_multikernel = false, chol_band = false; int chol_grid = 0;
  // pair-walk kernel of the Schur assembly (images of <= 8 columns): 0 fused tensor-core walk (default), 3 tensor-core walk
  // on a precomputed T, 1 staged, 2 direct.  PXR_SCHUR_KERNEL=fused|mma|staged|direct and PXR_SCHUR_CTAS=3|4 (register
  // budget) are A/B switches for measurements.
  int schur_kernel = [] { const char* e = getenv("PXR_SCHUR_KERNEL"); return !e ? 0 : (e[0] == 'm' ? 3 : (e[0] == 's' ? 1 : (e[0] == 'd' ? 2 : 0))); }();
  int schur_ctas = getenv("PXR_SCHUR_CTAS") ? atoi(getenv("PXR_SCHUR_CTAS")) : 0;   // 0: the kernel's default (fused 4, mma 3, staged 4)
  DevBuf<int32_t> img_cols8, img_dc8; DevBuf<int8_t> img_src8;   // per-image column tables (<= 8 columns per image)
  DevBuf<int32_t> io_obs;           // observations grouped by image, chunks of <= 128 (camera-block build)
  DevBuf<int64_t> io_chunk_begin; int64_t io_n_chunks = 0;
  DevBuf<long long> chol_trace;     // PXR_CHOL_TRACE=<file>: panel-CTA time stamps
  DevBuf<int> chol_sync;            // flags of the persistent tile-DAG Cholesky (pxr_chol.cuh)
  void clear_inner_round_timing() { for (auto& ev : inner_round_timed) for (cudaEvent_t e : ev) cudaEventDestroy(e); inner_round_timed.clear(); }
  ~BA() { if (inner_cnt_host) cudaFreeHost(inner_cnt_host); clear_inner_round_timing(); if (res_thread.joinable()) res_thread.join(); if (chol_graph_exec) cudaGraphExecDestroy(chol_graph_exec); for (int k = 0; k < kNumStages; ++k) for (auto& pr : timed[k]) { cudaEventDestroy(pr.first); cudaEventDestroy(pr.second); } }
  // static co-visibility structure for the Schur complement (see ba_schur_pairs_kernel)
  DevBuf<int32_t> sp_px, sp_py, sp_pp;
  DevBuf<int64_t> sp_chunk_begin;
  DevBuf<uint8_t> sp_chunk_self;
  DevBuf<double> Tbuf, Hinv;
  int64_t sp_n_chunks = 0;
  bool sp_built = false;
  std::vector<int32_t> h_obs_img;
  int build_schur_pairs();
  SchurPairs schur_pairs();

  // obs_xy != nullptr: a geometric handle (the desc carries no patches)
  int create(pxr_ctx* c, const pxr_ba_desc* d, const pxr_interp_config* ic, const pxr_solver_options* so, bool for_solve,
             const double* obs_xy = nullptr);
  int geo_k1(int mode, double* residuals_out, double* grad_out, const int64_t* list, int64_t n,
             const unsigned long long* n_dev = nullptr);
  // ---- window residency of the patch slab (pxr_resident.cuh): only in the one-shot pxr_ba_run (the host source must
  // outlive the solve), mapped pinned host source, C >= 8.  A repeated pass is local to the rank, so it composes with the
  // multi-GPU block mode (it only adds a host look at the violation counter after each evaluation).
  bool allow_resident = false, resident = false;
  int res_window = 8;
  bool res_window_fixed = false;                   // the caller knows the exact window (reference extraction: the points do not move)
  DevBuf<uint32_t> res_rect;
  DevBuf<unsigned long long> res_viol_count;
  DevBuf<int64_t> res_viol_list, res_fix_list;
  DevBuf<uint8_t> res_shared;
  std::vector<const void*> res_srcs;               // host blocks of whole patches (one entry for a contiguous source)
  std::vector<int64_t> res_block_first;            // [n_blocks+1]
  std::vector<int64_t> h_obs_patch;                // host copy (which patch an observation reads), empty = identity
  std::vector<uint8_t> res_whole;                  // patches already fetched whole
  int64_t res_refetched = 0, res_passes_repeated = 0;
  size_t res_esz = 2;
  std::thread res_thread;                          // packs and uploads the windows while create() goes on
  int res_thread_rc = 0; std::string res_thread_err;
  int resident_setup(const pxr_ba_desc* d, size_t esz);                    // decides and allocates
  int resident_begin(cudaStream_t us, double* h2d_patch);                  // K0 + rectangles + the window upload (own thread)
  int resident_fix(int64_t* n_fixed);               // after an evaluation: fetch the patches of reported observations
  void resident_args(FmEvalArgs& a);                // hooks the guard into an evaluation launch
  BADev dev();
  int project(int set, bool jac, double* xy_out);
  int fm(int mode, double* residuals_out, double* cost_dev, double* grad_out = nullptr);
  int fm_k1(int mode, double* residuals_out, double* grad_out, const int64_t* list, int64_t n);   // K1 over all observations or a list
  int fm_cost(double* cost_dev);                                                                   // robustified cost from obs_out
  int build();
  int evaluate(int set, bool jac, double* cost_out);
  int compute_step(double radius, bool* valid, double* model_cost_change);
  int chol_launch();
  int apply_step();
  int gradient_max_norm(double* out);
  // trial_cost (device scalar, optional): receives the cost at the starting point, reduced from round 0's records
  int inner_iterations(int set, double* trial_cost = nullptr);
  int eval_list(int set, const int64_t* list, int64_t n, const unsigned long long* n_dev = nullptr, bool settle = true,
                cudaEvent_t after_k0 = nullptr, cudaEvent_t after_k1 = nullptr, int64_t k0_bound = -1);
  int alloc_inner_jpt();                            // inner_jpt's one allocation: before the rounds, or a debug entry
  bool capture_inner_lists = false;                // pxr_ba_debug_inner_capture: keep every round's lists (synchronous)
  std::vector<std::vector<int64_t>> cap_plist, cap_list;
  std::vector<std::vector<uint8_t>> cap_active;
  int capture_round_lists(const int64_t* plist, const int64_t* list, const unsigned long long* cnt);
  int capture_round_active();
  int project_point_list(int set, const int64_t* list, int64_t n, const unsigned long long* n_dev, int64_t grid_bound);
  int inner_rounds(int set, double* trial_cost);   // the <= 52 rounds of inner_iterations, without a host wait per round
  unsigned long long* inner_cnt_host = nullptr;    // pinned, mapped [kInnerRounds][3]: each round's list lengths + the epoch of the call
  unsigned long long* inner_cnt_dev = nullptr;     // the same slots, device view (written by inner_step_kernel)
  unsigned long long inner_epoch = 0;              // incremented per inner_rounds call: tells this call's slots from stale ones
  int inner_rounds_run = 0;                        // rounds enqueued by the most recent inner_rounds (profiling)
  bool time_inner_rounds = false;                  // pxr_ba_debug_inner_rounds: stream time of every round of the next calls
  bool inner_rounds_timed = false;                 // the most recent inner_rounds call recorded them
  std::vector<std::array<cudaEvent_t, 4>> inner_round_timed;   // per round: before K0, after K0, after K1, after the step kernel
  DevBuf<double> inner_snapshot;                   // window residency: the points before a batch of rounds (redo after a refetch)
  DevBuf<InnerState> inner_state;
  DevBuf<int64_t> inner_list[2], inner_plist[2];   // a round's observation / point lists, alternating between rounds
  DevBuf<unsigned long long> inner_counters;       // 3 x [observations, points], rotating
  DevBuf<double> inner_jpt;                        // [n_obs][6]: d(uv)/dX of the observations a round evaluated
  int step_norm_between_sets();                    // enqueues the squared point / camera parts to scalars[11] / [12]
  // LM driver (pxr_ba.cu), one loop for both modes; the three lm_* steps below are what differs with block_mode
  int lm_begin();
  bool lm_finalize(int max_iteration);
  int lm_iterate(int max_iteration);
  int lm_linearize_start();                         // IterationZero's evaluation, cost and Jacobi scaling
  int lm_trial(bool interrupted, bool ran_inner, LMTrial* t);   // enqueue the step and its trial, read back t
  int lm_move(double candidate_cost, double next_cost);          // linearise at the accepted point: x_cost, |g|
  int lm_gradient(double* out);                     // max |g| now, or NaN with lm.gmax_pending
  void fill_summary(pxr_summary* sum, double seconds, int64_t launches);
  int solve(pxr_summary* sum);
  int read_params(double* cam_o, double* q_o, double* t_o, double* X_o);
};

}  // namespace pxr
