"""ctypes mirror of include/pxr.h (the C-ABI of libpxr.so).

This module is plumbing only: struct layouts, library loading, and helpers that turn numpy
arrays into the SoA problem IR.  It contains NO arithmetic of the hot path and NO CPU
fallback: if libpxr.so is missing or no CUDA device is usable every compute entry point
raises (PxrError / RuntimeError).
"""
import ctypes as C
import os
import numpy as np

PXR_MAX_CAM_PARAMS = 12

# status codes -> exception types (reference: THROW_CHECK* -> py::value_error,
# util/src/log_exceptions.h:52-84; unsupported (C,N) -> std::invalid_argument)
PXR_OK, PXR_ERR_INVALID_ARGUMENT, PXR_ERR_UNSUPPORTED, PXR_ERR_NO_DEVICE, PXR_ERR_CUDA, \
    PXR_ERR_NCCL, PXR_ERR_NUMERIC, PXR_ERR_INTERRUPTED, PXR_ERR_INTERNAL = range(9)
# status of pxr_ba_debug_reduced_solve
REDUCED_SOLVE_OK, REDUCED_SOLVE_FAILED, REDUCED_SOLVE_BAILED_OUT = range(3)

CAMERA_MODEL_IDS = {"SIMPLE_PINHOLE": 0, "PINHOLE": 1, "SIMPLE_RADIAL": 2, "RADIAL": 3,
                    "OPENCV": 4, "OPENCV_FISHEYE": 5, "FULL_OPENCV": 6}
CAMERA_NUM_PARAMS = {0: 3, 1: 4, 2: 4, 3: 5, 4: 8, 5: 8, 6: 12}
# (focal, principal point, extra) parameter-index bit masks per model
CAMERA_PARAM_GROUPS = {0: (0x1, 0x6, 0x0), 1: (0x3, 0xC, 0x0), 2: (0x1, 0x6, 0x8),
                       3: (0x1, 0x6, 0x18), 4: (0x3, 0xC, 0xF0), 5: (0x3, 0xC, 0xF0),
                       6: (0x3, 0xC, 0xFF0)}
LOSS_IDS = {"trivial": 0, "cauchy": 1, "huber": 2, "soft_l1": 3, "softlone": 3, "arctan": 4}
DTYPE_IDS = {np.dtype(np.float16): 0, np.dtype(np.float32): 1, np.dtype(np.float64): 2}


def ptr(a):
    """ctypes pointer to a numpy array's data (None stays NULL)"""
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class ReconView(C.Structure):          # pxr_recon_view
    _fields_ = [("n_images", C.c_int64), ("image_id", C.c_void_p), ("image_camera_id", C.c_void_p), ("p2d_begin", C.c_void_p),
                ("p2d_point3D_id", C.c_void_p), ("n_cameras", C.c_int64), ("camera_id", C.c_void_p), ("camera_model", C.c_void_p),
                ("n_points", C.c_int64), ("point3D_id", C.c_void_p), ("track_begin", C.c_void_p), ("track_image_id", C.c_void_p),
                ("track_point2D_idx", C.c_void_p)]


class SetupView(C.Structure):          # pxr_ba_setup_view
    _fields_ = [("n_images", C.c_int64), ("image_ids", C.c_void_p), ("n_const_poses", C.c_int64), ("const_pose_ids", C.c_void_p),
                ("n_const_tvecs", C.c_int64), ("const_tvec_ids", C.c_void_p), ("const_tvec_masks", C.c_void_p),
                ("n_const_cameras", C.c_int64), ("const_camera_ids", C.c_void_p), ("n_var_points", C.c_int64),
                ("var_point_ids", C.c_void_p), ("n_const_points", C.c_int64), ("const_point_ids", C.c_void_p)]


class BuildOptions(C.Structure):       # pxr_ba_build_options
    _fields_ = [("refine_focal_length", C.c_int32), ("refine_principal_point", C.c_int32), ("refine_extra_params", C.c_int32),
                ("refine_extrinsics", C.c_int32), ("min_track_length", C.c_int32), ("mode", C.c_int32),
                ("n_ref_points", C.c_int64), ("ref_point_ids", C.c_void_p), ("track_has_patch", C.c_void_p)]


class PxrError(RuntimeError):
    pass


class InterpConfig(C.Structure):
    _fields_ = [("l2_normalize", C.c_int32), ("use_float_simd", C.c_int32),
                ("check_bounds", C.c_int32), ("reserved", C.c_int32)]


class SolverOptions(C.Structure):
    _fields_ = [("loss_type", C.c_int32), ("loss_scale", C.c_double),
                ("linear_solver", C.c_int32), ("max_num_iterations", C.c_int32),
                ("max_linear_solver_iterations", C.c_int32),
                ("max_num_consecutive_invalid_steps", C.c_int32),
                ("function_tolerance", C.c_double), ("gradient_tolerance", C.c_double),
                ("parameter_tolerance", C.c_double), ("use_inner_iterations", C.c_int32),
                ("inner_iteration_tolerance", C.c_double),
                ("initial_trust_region_radius", C.c_double),
                ("max_trust_region_radius", C.c_double), ("min_trust_region_radius", C.c_double),
                ("min_relative_decrease", C.c_double), ("min_lm_diagonal", C.c_double),
                ("max_lm_diagonal", C.c_double), ("jacobi_scaling", C.c_int32),
                ("deterministic", C.c_int32), ("use_nonmonotonic_steps", C.c_int32),
                ("max_consecutive_nonmonotonic_steps", C.c_int32)]


class CostmapConfig(C.Structure):
    """pxr_costmap_config == CostMapConfig (costmap_extractor.h:18-40) + the embedded ReferenceConfig."""
    _fields_ = [("loss_type", C.c_int32), ("loss_scale", C.c_double), ("as_gradientfield", C.c_int32),
                ("compute_cross_derivative", C.c_int32), ("apply_sqrt", C.c_int32),
                ("upsampling_factor", C.c_double), ("compute_refs", C.c_int32),
                ("ref_loss_type", C.c_int32), ("ref_loss_scale", C.c_double), ("ref_iters", C.c_int32)]


class BADesc(C.Structure):
    _fields_ = [("n_cameras", C.c_int32), ("cam_model", C.c_void_p), ("cam_params", C.c_void_p),
                ("cam_const_mask", C.c_void_p),
                ("n_images", C.c_int32), ("qvec", C.c_void_p), ("tvec", C.c_void_p),
                ("img_cam", C.c_void_p), ("pose_const", C.c_void_p), ("tvec_const_mask", C.c_void_p),
                ("n_points", C.c_int64), ("xyz", C.c_void_p), ("point_const", C.c_void_p),
                ("n_obs", C.c_int64), ("obs_img", C.c_void_p), ("obs_pt", C.c_void_p),
                ("obs_patch", C.c_void_p),
                ("n_patches", C.c_int64), ("patches", C.c_void_p), ("patches_on_device", C.c_int32),
                ("patch_dtype", C.c_int32), ("ph", C.c_int32), ("pw", C.c_int32),
                ("channels", C.c_int32), ("corner", C.c_void_p), ("scale", C.c_void_p),
                ("upsampling_factor", C.c_double), ("refs", C.c_void_p),
                ("n_patch_blocks", C.c_int32), ("patch_block_ptrs", C.c_void_p), ("patch_block_counts", C.c_void_p)]


class IterationSummary(C.Structure):
    _fields_ = [("iteration", C.c_int32), ("step_is_valid", C.c_int32),
                ("step_is_successful", C.c_int32), ("cost", C.c_double),
                ("cost_change", C.c_double), ("gradient_max_norm", C.c_double),
                ("step_norm", C.c_double), ("relative_decrease", C.c_double),
                ("trust_region_radius", C.c_double), ("linear_solver_iterations", C.c_int32),
                ("iteration_time_s", C.c_double)]


class Summary(C.Structure):
    _fields_ = [("initial_cost", C.c_double), ("final_cost", C.c_double),
                ("num_residual_blocks", C.c_int32), ("num_residuals", C.c_int64),
                ("num_successful_steps", C.c_int32), ("num_unsuccessful_steps", C.c_int32),
                ("num_inner_iteration_steps", C.c_int32), ("termination_type", C.c_int32),
                ("total_time_s", C.c_double), ("solve_time_s", C.c_double),
                ("h2d_bytes", C.c_double), ("d2h_bytes", C.c_double),
                ("num_iterations", C.c_int32), ("iterations_capacity", C.c_int32),
                ("iterations", C.POINTER(IterationSummary)), ("kernel_launches", C.c_int64),
                ("message", C.c_char * 256), ("resident_window", C.c_int32), ("resident_passes_repeated", C.c_int32),
                ("resident_refetched", C.c_int64)]


class KADesc(C.Structure):
    _fields_ = [("n_keypoints", C.c_int64), ("keypoints", C.c_void_p), ("kp_const", C.c_void_p),
                ("kp_patch", C.c_void_p), ("n_edges", C.c_int64), ("edge_src", C.c_void_p),
                ("edge_dst", C.c_void_p), ("edge_weight", C.c_void_p), ("edge_problem", C.c_void_p),
                ("n_problems", C.c_int32), ("n_patches", C.c_int64), ("patches", C.c_void_p),
                ("patches_on_device", C.c_int32), ("patch_dtype", C.c_int32), ("ph", C.c_int32),
                ("pw", C.c_int32), ("channels", C.c_int32), ("corner", C.c_void_p),
                ("scale", C.c_void_p), ("upsampling_factor", C.c_double), ("bound", C.c_double),
                ("patches_are_sparse", C.c_int32), ("n_patch_blocks", C.c_int32),
                ("patch_block_ptrs", C.c_void_p), ("patch_block_counts", C.c_void_p),
                ("ref_desc", C.c_void_p), ("n_ref_desc", C.c_int64)]


class QBADesc(C.Structure):            # pxr_qba_desc
    _fields_ = [("n_queries", C.c_int32), ("cam_model", C.c_void_p), ("cam_params", C.c_void_p),
                ("cam_const_mask", C.c_void_p), ("qvec", C.c_void_p), ("tvec", C.c_void_p), ("obs_begin", C.c_void_p),
                ("xyz", C.c_void_p), ("obs_patch", C.c_void_p), ("refs", C.c_void_p), ("patch_blocks", C.c_void_p),
                ("patch_counts", C.c_void_p), ("corner", C.c_void_p), ("scale", C.c_void_p),
                ("upsampling_factor", C.c_double), ("ph", C.c_int32), ("pw", C.c_int32), ("channels", C.c_int32),
                ("patch_dtype", C.c_int32), ("max_wave_bytes", C.c_double)]


class QBAResult(C.Structure):          # pxr_qba_result
    _fields_ = [("status", C.c_int32), ("num_residual_blocks", C.c_int32), ("initial_cost", C.c_double),
                ("final_cost", C.c_double), ("num_iterations", C.c_int32), ("num_successful_steps", C.c_int32),
                ("num_unsuccessful_steps", C.c_int32), ("termination_type", C.c_int32),
                ("block_evaluations", C.c_int64)]


def _patch_blocks(blocks):
    """one patch block per query, host numpy or device memory (anything with `.ptr` or __cuda_array_interface__) ->
    (ctypes pointer array, patch counts, (ph, pw, channels), dtype id)"""
    ptrs, counts, shape, dtype = [], [], None, None
    for b in blocks:
        cai = getattr(b, "__cuda_array_interface__", None)
        if getattr(b, "ptr", None) is not None:
            p, shp, dt = int(b.ptr), tuple(b.shape), np.dtype(b.dtype)
        elif cai is not None:
            p, shp, dt = int(cai["data"][0]), tuple(cai["shape"]), np.dtype(cai["typestr"])
        else:
            if b.dtype not in DTYPE_IDS or not b.flags["C_CONTIGUOUS"] or b.ndim != 4:
                raise ValueError("patch blocks must be C-contiguous [N,H,W,C] f16/f32/f64 arrays")
            p, shp, dt = b.ctypes.data, tuple(b.shape), np.dtype(b.dtype)
        if shape is not None and (shp[1:] != shape or dt != dtype):
            raise ValueError("patch blocks must share one dtype and patch shape")
        shape, dtype = shp[1:], dt
        ptrs.append(p); counts.append(shp[0])
    return ((C.c_void_p * max(len(ptrs), 1))(*ptrs), np.array(counts, np.int64), shape if shape is not None else (1, 1, 8),
            DTYPE_IDS[dtype] if dtype is not None else 0)


class QKADesc(C.Structure):            # pxr_qka_desc
    _fields_ = [("n_queries", C.c_int32), ("kp_begin", C.c_void_p), ("patch_blocks", C.c_void_p),
                ("patch_counts", C.c_void_p), ("patches_are_sparse", C.c_void_p), ("keypoints", C.c_void_p),
                ("kp_patch", C.c_void_p), ("desc_begin", C.c_void_p), ("descs", C.c_void_p), ("corner", C.c_void_p),
                ("scale", C.c_void_p), ("upsampling_factor", C.c_double), ("bound", C.c_double), ("ph", C.c_int32),
                ("pw", C.c_int32), ("channels", C.c_int32), ("patch_dtype", C.c_int32), ("max_wave_bytes", C.c_double)]


class QKAResult(C.Structure):          # pxr_qka_result
    _fields_ = [("status", C.c_int32), ("num_residual_blocks", C.c_int32), ("initial_cost", C.c_double),
                ("final_cost", C.c_double), ("num_successful_steps", C.c_int32), ("num_unsuccessful_steps", C.c_int32),
                ("num_iterations", C.c_int32), ("termination_type", C.c_int32)]

class PnPDesc(C.Structure):            # pxr_pnp_desc
    _fields_ = [("n_queries", C.c_int32), ("corr_begin", C.c_void_p), ("points2D", C.c_void_p), ("points3D", C.c_void_p),
                ("cam_model", C.c_void_p), ("cam_params", C.c_void_p), ("seed", C.c_void_p), ("qvec", C.c_void_p),
                ("tvec", C.c_void_p), ("inlier_mask", C.c_void_p)]


class PnPOptions(C.Structure):         # pxr_pnp_options
    _fields_ = [("max_error", C.c_double), ("min_inlier_ratio", C.c_double), ("min_num_trials", C.c_int32),
                ("max_num_trials", C.c_int32), ("confidence", C.c_double), ("dyn_num_trials_multiplier", C.c_double),
                ("estimate_focal_length", C.c_int32), ("refine", C.c_int32), ("gradient_tolerance", C.c_double),
                ("max_num_iterations", C.c_int32), ("loss_function_scale", C.c_double), ("refine_focal_length", C.c_int32),
                ("refine_extra_params", C.c_int32), ("function_tolerance", C.c_double), ("parameter_tolerance", C.c_double)]


class PnPResult(C.Structure):          # pxr_pnp_result
    _fields_ = [("status", C.c_int32), ("success", C.c_int32), ("num_inliers", C.c_int32), ("num_trials", C.c_int32),
                ("best_trial", C.c_int32), ("best_solution", C.c_int32), ("local_optimized", C.c_int32),
                ("num_iterations", C.c_int32), ("termination_type", C.c_int32), ("initial_cost", C.c_double),
                ("final_cost", C.c_double)]


def default_pnp_options(**kw):
    o = PnPOptions()
    load_lib().pxr_default_pnp_options(C.byref(o))
    for k, v in kw.items():
        if not hasattr(o, k):
            raise ValueError("unknown pxr_pnp_options field '%s'" % k)
        setattr(o, k, v)
    return o


class PnPBatch:
    """numpy arrays of a batch of absolute pose estimations + the ctypes view (pxr_pnp_desc): per query camera model,
    params [12] (in/out), seed, qvec / tvec (out); per correspondence a 2D point (pixels), a 3D point and the inlier flag
    (out)."""

    def __init__(self, corr_begin, points2D, points3D, cam_model, cam_params, seed):
        self.corr_begin = _as(corr_begin, np.int64)
        self.cam_model = _as(cam_model, np.int32)
        nq = len(self.cam_model)
        self.n_queries = nq
        self.points2D = _as(points2D, np.float64, (-1, 2))
        self.points3D = _as(points3D, np.float64, (-1, 3))
        self.cam_params = _as(cam_params, np.float64, (nq, PXR_MAX_CAM_PARAMS))
        self.seed = _as(seed, np.uint64)
        self.qvec = np.zeros((nq, 4)); self.qvec[:, 0] = 1.0
        self.tvec = np.zeros((nq, 3))
        self.inlier_mask = np.zeros(len(self.points2D), np.uint8)

    def desc(self):
        return PnPDesc(self.n_queries, _ptr(self.corr_begin), _ptr(self.points2D), _ptr(self.points3D), _ptr(self.cam_model),
                       _ptr(self.cam_params), _ptr(self.seed), _ptr(self.qvec), _ptr(self.tvec), _ptr(self.inlier_mask))


class TriDesc(C.Structure):            # pxr_tri_desc
    _fields_ = [("n_cameras", C.c_int32), ("cam_model", C.c_void_p), ("cam_params", C.c_void_p), ("n_images", C.c_int32),
                ("img_cam", C.c_void_p), ("qvec", C.c_void_p), ("tvec", C.c_void_p), ("n_tracks", C.c_int64),
                ("track_begin", C.c_void_p), ("track_key", C.c_void_p), ("obs_img", C.c_void_p), ("obs_xy", C.c_void_p)]


class TriOptions(C.Structure):         # pxr_tri_options
    _fields_ = [("min_angle", C.c_double), ("create_max_angle_error", C.c_double), ("tri_max_pairs", C.c_int32),
                ("seed", C.c_uint64)]


# pxr_tri_run's per-track status
TRI_OK, TRI_TOO_FEW_INLIERS, TRI_ANGLE_TOO_SMALL = range(3)


def default_tri_options(**kw):
    o = TriOptions()
    load_lib().pxr_default_tri_options(C.byref(o))
    for k, v in kw.items():
        if not hasattr(o, k):
            raise ValueError("unknown pxr_tri_options field '%s'" % k)
        setattr(o, k, v)
    return o


class TriScene:
    """numpy arrays of a triangulation problem + the ctypes view (pxr_tri_desc): cameras (model, params [12]), images
    (camera index, qvec, tvec) and, for pxr_tri_run / pxr_tri_evaluate, tracks in CSR form (track_begin, per observation
    the image index and the pixel)."""

    def __init__(self, cam_model, cam_params, img_cam, qvec, tvec, track_begin=None, obs_img=None, obs_xy=None,
                 track_key=None):
        self.cam_model = _as(cam_model, np.int32)
        self.cam_params = _as(cam_params, np.float64, (len(self.cam_model), PXR_MAX_CAM_PARAMS))
        self.img_cam = _as(img_cam, np.int32)
        self.qvec = _as(qvec, np.float64, (-1, 4))
        self.tvec = _as(tvec, np.float64, (-1, 3))
        self.track_begin = _as(track_begin if track_begin is not None else [0], np.int64)
        self.obs_img = _as(obs_img if obs_img is not None else [], np.int32)
        self.obs_xy = _as(obs_xy if obs_xy is not None else np.zeros((0, 2)), np.float64, (-1, 2))
        self.track_key = None if track_key is None else _as(track_key, np.int64)

    @property
    def n_tracks(self):
        return len(self.track_begin) - 1

    def desc(self):
        return TriDesc(len(self.cam_model), _ptr(self.cam_model), _ptr(self.cam_params), len(self.img_cam), _ptr(self.img_cam),
                       _ptr(self.qvec), _ptr(self.tvec), self.n_tracks, _ptr(self.track_begin), _ptr(self.track_key),
                       _ptr(self.obs_img), _ptr(self.obs_xy))


class QBABatch:
    """numpy arrays of a batch of query bundle adjustments + the ctypes view (pxr_qba_desc).  Per query: camera model,
    params [12] (in/out), constancy mask, qvec / tvec (in/out), a patch block [n_q, H, W, C] (host numpy array or
    anything with `.ptr` / __cuda_array_interface__ in device memory) with its corners and scales; per residual block:
    xyz, patch index within its query's block and one fp64 reference descriptor."""

    def __init__(self, cam_model, cam_params, cam_const_mask, qvec, tvec, obs_begin, xyz, obs_patch, refs,
                 patch_blocks, corner, scale, upsampling_factor=1.0, max_wave_bytes=0.0):
        self.cam_model = _as(cam_model, np.int32)
        nq = len(self.cam_model)
        cp = np.zeros((nq, PXR_MAX_CAM_PARAMS), np.float64)
        for i in range(nq):
            p = np.asarray(cam_params[i], np.float64).reshape(-1)
            cp[i, :len(p)] = p
        self.cam_params = cp
        self.cam_const_mask = _as(cam_const_mask, np.uint32)
        self.qvec = _as(qvec, np.float64, (-1, 4)).copy()
        self.tvec = _as(tvec, np.float64, (-1, 3)).copy()
        self.obs_begin = _as(obs_begin, np.int64)
        m = int(self.obs_begin[-1]) if len(self.obs_begin) else 0
        self.xyz = _as(xyz, np.float64, (-1, 3)) if m else np.zeros((0, 3))
        self.obs_patch = _as(obs_patch, np.int64) if m else np.zeros(0, np.int64)
        self.refs = np.ascontiguousarray(refs, np.float64) if m else None
        if len(patch_blocks) != nq:
            raise ValueError("one patch block per query")
        self.patch_blocks = list(patch_blocks)
        self._ptrs, self.patch_counts, (self.ph, self.pw, self.channels), self.patch_dtype = _patch_blocks(self.patch_blocks)
        self.corner = _as(corner, np.int32, (-1, 2))
        self.scale = _as(scale, np.float64, (-1, 2))
        self.upsampling_factor = float(upsampling_factor)
        self.max_wave_bytes = float(max_wave_bytes)

    @property
    def n_queries(self):
        return len(self.cam_model)

    def desc(self):
        d = QBADesc()
        d.n_queries = self.n_queries
        d.cam_model = _ptr(self.cam_model); d.cam_params = _ptr(self.cam_params)
        d.cam_const_mask = _ptr(self.cam_const_mask); d.qvec = _ptr(self.qvec); d.tvec = _ptr(self.tvec)
        d.obs_begin = _ptr(self.obs_begin); d.xyz = _ptr(self.xyz); d.obs_patch = _ptr(self.obs_patch)
        d.refs = _ptr(self.refs)
        d.patch_blocks = C.cast(self._ptrs, C.c_void_p); d.patch_counts = _ptr(self.patch_counts)
        d.corner = _ptr(self.corner); d.scale = _ptr(self.scale)
        d.upsampling_factor = self.upsampling_factor
        d.ph, d.pw, d.channels, d.patch_dtype = self.ph, self.pw, self.channels, self.patch_dtype
        d.max_wave_bytes = self.max_wave_bytes
        return d


def make_summary(capacity=256):
    s = Summary()
    buf = (IterationSummary * max(capacity, 1))()
    s.iterations = C.cast(buf, C.POINTER(IterationSummary))
    s.iterations_capacity = capacity
    s._buf = buf
    return s


def summary_to_dict(s):
    n = min(s.num_iterations, s.iterations_capacity)
    its = [{f[0]: getattr(s.iterations[i], f[0]) for f in IterationSummary._fields_} for i in range(n)]
    d = {f[0]: getattr(s, f[0]) for f in Summary._fields_ if f[0] not in ("iterations", "message")}
    d["message"] = s.message.decode(errors="replace")
    d["iterations"] = its
    return d


def default_interp(l2_normalize=True, use_float_simd=False):
    return InterpConfig(int(l2_normalize), int(use_float_simd), 0, 0)


def default_costmap_config(**kw):
    c = CostmapConfig(loss_type=0, loss_scale=1.0, as_gradientfield=1, compute_cross_derivative=0, apply_sqrt=0,
                      upsampling_factor=1.0, compute_refs=1, ref_loss_type=1, ref_loss_scale=0.25, ref_iters=100)
    for k, v in kw.items():
        if not hasattr(c, k):
            raise ValueError("unknown cost-map option %r" % k)
        setattr(c, k, v)
    return c


def default_ba_options(**kw):
    """bundle_adjustment/main.py:30-62 + bundle_adjustment_options.h:48-64 defaults."""
    o = SolverOptions(loss_type=1, loss_scale=0.25, linear_solver=0, max_num_iterations=100,
                      max_linear_solver_iterations=200, max_num_consecutive_invalid_steps=10,
                      function_tolerance=0.0, gradient_tolerance=0.0, parameter_tolerance=0.0,
                      use_inner_iterations=1, inner_iteration_tolerance=1e-3,
                      initial_trust_region_radius=1e4, max_trust_region_radius=1e16,
                      min_trust_region_radius=1e-32, min_relative_decrease=1e-3,
                      min_lm_diagonal=1e-6, max_lm_diagonal=1e32, jacobi_scaling=1, deterministic=0,
                      use_nonmonotonic_steps=0, max_consecutive_nonmonotonic_steps=5)
    for k, v in kw.items():
        setattr(o, k, v)
    return o


def default_ka_options(**kw):
    """keypoint_adjustment/main.py:60-83 + keypoint_adjustment_options.h:47-86 defaults."""
    o = default_ba_options(use_inner_iterations=0, parameter_tolerance=1e-5)
    for k, v in kw.items():
        setattr(o, k, v)
    return o


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _as(a, dtype, shape=None):
    if a is None:
        return None
    a = np.ascontiguousarray(a, dtype=dtype)
    if shape is not None:
        a = a.reshape(shape)
    return a


class BAProblem:
    """Holds the numpy arrays of one BA problem IR and the ctypes view of them."""

    def __init__(self, cam_model, cam_params, cam_const_mask, qvec, tvec, img_cam, pose_const,
                 tvec_const_mask, xyz, point_const, obs_img, obs_pt, patches, corner, scale,
                 refs=None, obs_patch=None, upsampling_factor=1.0, patches_on_device=False,
                 patch_shape=None, patch_dtype=None, patch_blocks=None, obs_xy=None):
        """obs_xy [n_obs, 2]: the observed keypoints of a geometric (reprojection-error) problem; it then has no
        patches (patches, corner, scale, refs and obs_patch are not used) and two residuals per observation"""
        self.cam_model = _as(cam_model, np.int32)
        nc = len(self.cam_model)
        cp = np.zeros((nc, PXR_MAX_CAM_PARAMS), np.float64)
        cam_params = np.asarray(cam_params, np.float64)
        if cam_params.ndim == 2 and cam_params.shape[1] == PXR_MAX_CAM_PARAMS:
            cp[:] = cam_params
        else:
            for i in range(nc):
                k = CAMERA_NUM_PARAMS[int(self.cam_model[i])]
                cp[i, :k] = np.asarray(cam_params[i], np.float64)[:k]
        self.cam_params = cp
        self.cam_const_mask = _as(cam_const_mask, np.uint32)
        self.qvec = _as(qvec, np.float64, (-1, 4)).copy()
        self.tvec = _as(tvec, np.float64, (-1, 3)).copy()
        self.img_cam = _as(img_cam, np.int32)
        self.pose_const = _as(pose_const, np.uint8)
        self.tvec_const_mask = _as(tvec_const_mask, np.uint8)
        self.xyz = _as(xyz, np.float64, (-1, 3)).copy()
        self.point_const = _as(point_const, np.uint8)
        self.obs_img = _as(obs_img, np.int32)
        self.obs_pt = _as(obs_pt, np.int64)
        if len(self.obs_pt) > 1 and np.any(np.diff(self.obs_pt) < 0):
            raise ValueError("observations must be sorted by point index")
        self.obs_patch = _as(obs_patch, np.int64)
        self.patches_on_device = bool(patches_on_device)
        self.patch_blocks = None
        self.obs_xy = None
        if obs_xy is not None:
            self.obs_xy = _as(obs_xy, np.float64, (-1, 2))
            if len(self.obs_xy) != len(self.obs_pt):
                raise ValueError("obs_xy must hold one keypoint per observation")
            self.obs_patch = None
            self.patches = None
            self._patches_ptr = None
            self.n_patches, self.ph, self.pw, self.channels, self.patch_dtype = 0, 0, 0, 0, 0
        elif patch_blocks is not None:
            # list of C-contiguous [n_i, H, W, C] arrays (one per FeatureMap), uploaded without concatenation
            blocks = [b for b in patch_blocks]
            for b in blocks:
                if b.dtype not in DTYPE_IDS or not b.flags["C_CONTIGUOUS"] or b.ndim != 4 or b.shape[1:] != blocks[0].shape[1:]:
                    raise ValueError("patch blocks must be C-contiguous [N,H,W,C] arrays of one dtype/shape")
            self.patch_blocks = blocks
            # host numpy blocks and device-resident blocks (anything with .ptr, e.g. _features.DevicePatches) can be
            # mixed: the library copies with cudaMemcpyDefault
            self._block_ptrs = (C.c_void_p * len(blocks))(*[getattr(b, "ptr", None) or b.ctypes.data for b in blocks])
            self._block_counts = np.array([b.shape[0] for b in blocks], np.int64)
            self.patches = None
            self._patches_ptr = getattr(blocks[0], "ptr", None) or blocks[0].ctypes.data
            self.n_patches = int(self._block_counts.sum())
            _, self.ph, self.pw, self.channels = blocks[0].shape
            self.patch_dtype = DTYPE_IDS[blocks[0].dtype]
        elif self.patches_on_device:
            self.patches = None
            self._patches_ptr = int(patches)
            self.n_patches, self.ph, self.pw, self.channels = patch_shape
            self.patch_dtype = patch_dtype
        else:
            if patches.dtype not in DTYPE_IDS or not patches.flags["C_CONTIGUOUS"] or patches.ndim != 4:
                raise ValueError("patches must be a C-contiguous [N,H,W,C] f16/f32/f64 array")
            self.patches = patches
            self._patches_ptr = patches.ctypes.data
            self.n_patches, self.ph, self.pw, self.channels = patches.shape
            self.patch_dtype = DTYPE_IDS[patches.dtype]
        self.corner = _as(corner, np.int32, (-1, 2))
        self.scale = _as(scale, np.float64, (-1, 2))
        self.refs = _as(refs, np.float64)
        self.upsampling_factor = float(upsampling_factor)

    @property
    def n_obs(self):
        return len(self.obs_pt)

    @property
    def residuals_per_obs(self):
        """2 for a geometric problem, the channel count otherwise"""
        return 2 if self.obs_xy is not None else self.channels

    @property
    def patch_np_dtype(self):
        return {v: k for k, v in DTYPE_IDS.items()}[self.patch_dtype]

    def with_patches(self, patches, refs=None, on_device=False, patch_shape=None, patch_dtype=None):
        """Same geometry / observation lists, other patches (e.g. the 3-channel cost maps of these features)."""
        return BAProblem(self.cam_model, self.cam_params, self.cam_const_mask, self.qvec, self.tvec, self.img_cam,
                         self.pose_const, self.tvec_const_mask, self.xyz, self.point_const, self.obs_img, self.obs_pt,
                         patches, self.corner, self.scale, refs=refs, obs_patch=self.obs_patch,
                         upsampling_factor=self.upsampling_factor, patches_on_device=on_device,
                         patch_shape=patch_shape, patch_dtype=patch_dtype)

    def desc(self):
        d = BADesc()
        d.n_cameras = len(self.cam_model)
        d.cam_model = _ptr(self.cam_model); d.cam_params = _ptr(self.cam_params)
        d.cam_const_mask = _ptr(self.cam_const_mask)
        d.n_images = len(self.img_cam)
        d.qvec = _ptr(self.qvec); d.tvec = _ptr(self.tvec); d.img_cam = _ptr(self.img_cam)
        d.pose_const = _ptr(self.pose_const); d.tvec_const_mask = _ptr(self.tvec_const_mask)
        d.n_points = len(self.xyz)
        d.xyz = _ptr(self.xyz); d.point_const = _ptr(self.point_const)
        d.n_obs = len(self.obs_pt)
        d.obs_img = _ptr(self.obs_img); d.obs_pt = _ptr(self.obs_pt); d.obs_patch = _ptr(self.obs_patch)
        d.n_patches = self.n_patches
        d.patches = C.c_void_p(self._patches_ptr)
        d.patches_on_device = int(self.patches_on_device)
        d.patch_dtype = self.patch_dtype
        d.ph, d.pw, d.channels = self.ph, self.pw, self.channels
        d.corner = _ptr(self.corner); d.scale = _ptr(self.scale)
        d.upsampling_factor = self.upsampling_factor
        d.refs = _ptr(self.refs)
        if self.patch_blocks is not None:
            d.n_patch_blocks = len(self.patch_blocks)
            d.patch_block_ptrs = C.cast(self._block_ptrs, C.c_void_p)
            d.patch_block_counts = _ptr(self._block_counts)
        return d

    def copy(self):
        import copy as _copy
        o = _copy.copy(self)
        for k in ("cam_params", "qvec", "tvec", "xyz"):
            setattr(o, k, getattr(self, k).copy())
        if self.refs is not None:
            o.refs = self.refs.copy()
        return o


_LIB = None


def lib_path():
    here = os.path.dirname(os.path.abspath(__file__))
    return os.path.normpath(os.path.join(here, "..", "..", "csrc", "libpxr.so"))


def load_lib():
    """Load libpxr.so (built in-tree by __graft_entry__.build()). Fails loudly if absent."""
    global _LIB
    if _LIB is not None:
        return _LIB
    p = lib_path()
    if not os.path.exists(p):
        raise PxrError("libpxr.so not built (%s): run `python __graft_entry__.py build`; "
                       "there is no CPU fallback" % p)
    lib = C.CDLL(p, mode=C.RTLD_GLOBAL)
    lib.pxr_last_error.restype = C.c_char_p
    lib.pxr_ctx_kernel_launches.restype = C.c_int64
    lib.pxr_ctx_nccl_collectives.restype = C.c_int64
    lib.pxr_set_interrupt_callback(_SIGNAL_POLL, None)      # Ctrl-C stops a solve between LM iterations
    _LIB = lib
    return lib


def _signals_pending(_user):
    """the library's interrupt callback: has a Python signal handler (SIGINT -> KeyboardInterrupt) fired?  Same probe
    as the reference's PyInterrupt (util/src/py_interrupt.h:29-38); ctypes re-acquires the GIL around this call."""
    try:
        return 1 if _check_signals() != 0 else 0
    except KeyboardInterrupt:
        return 1


def _check_signals():
    return C.pythonapi.PyErr_CheckSignals()


_SIGNAL_POLL = C.CFUNCTYPE(C.c_int, C.c_void_p)(_signals_pending)      # kept alive for the life of the process


def check(status):
    if status == PXR_OK:
        return
    msg = load_lib().pxr_last_error().decode(errors="replace")
    if status in (PXR_ERR_INVALID_ARGUMENT, PXR_ERR_UNSUPPORTED):
        raise ValueError(msg)
    if status == PXR_ERR_INTERRUPTED:
        raise KeyboardInterrupt(msg)
    raise PxrError("pxr status %d: %s" % (status, msg))


class Context:
    def __init__(self, device=-1):
        self.lib = load_lib()
        self.handle = C.c_void_p()
        check(self.lib.pxr_ctx_create(C.c_int(device), C.byref(self.handle)))

    def close(self):
        if self.handle:
            self.lib.pxr_ctx_destroy(self.handle)
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def kernel_launches(self):
        return int(self.lib.pxr_ctx_kernel_launches(self.handle))

    def nccl_collectives(self):
        """NCCL calls issued through this context so far (the contract: ONE all-reduce per LM iteration)"""
        return int(self.lib.pxr_ctx_nccl_collectives(self.handle))

    def mailbox_ready(self):
        """True when the per-iteration scalar exchange runs over peer memory (NVLink mailboxes), not NCCL"""
        return bool(self.lib.pxr_ctx_mailbox_ready(self.handle))

    def timer_start(self):
        check(self.lib.pxr_ctx_timer_start(self.handle))

    def timer_stop(self):
        ms = C.c_double()
        check(self.lib.pxr_ctx_timer_stop(self.handle, C.byref(ms)))
        return ms.value

    def init_comm(self, rank, world, uid_bytes):
        buf = (C.c_char * 128).from_buffer_copy(uid_bytes)
        check(self.lib.pxr_ctx_init_comm(self.handle, int(rank), int(world), buf))

    @staticmethod
    def nccl_unique_id():
        lib = load_lib()
        buf = (C.c_char * 128)()
        check(lib.pxr_nccl_unique_id(buf))
        return bytes(buf)

    def sync(self):
        check(self.lib.pxr_ctx_sync(self.handle))


_DEFAULT_CTX = None


def default_context():
    global _DEFAULT_CTX
    if _DEFAULT_CTX is None:
        _DEFAULT_CTX = Context(-1)
    return _DEFAULT_CTX


class KAProblem:
    """numpy arrays of one keypoint-adjustment problem set + the ctypes view (pxr_ka_desc)."""

    def __init__(self, keypoints, kp_const, edge_src, edge_dst, edge_weight, edge_problem, n_problems, patches,
                 corner, scale, kp_patch=None, bound=4.0, patches_are_sparse=True, upsampling_factor=1.0,
                 patch_blocks=None, ref_desc=None):
        self.keypoints = _as(keypoints, np.float64, (-1, 2)).copy()
        self.kp_const = _as(kp_const, np.uint8)
        self.edge_src = _as(edge_src, np.int64)
        self.edge_dst = _as(edge_dst, np.int64)
        self.edge_weight = _as(edge_weight, np.float64)
        self.edge_problem = _as(edge_problem, np.int32)
        if len(self.edge_problem) > 1 and np.any(np.diff(self.edge_problem) < 0):
            raise ValueError("edges must be sorted by problem label")
        self.n_problems = int(n_problems)
        # query mode: edge_dst indexes ref_desc [n_ref, C] (fixed descriptors) instead of keypoints
        self.ref_desc = None if ref_desc is None else np.ascontiguousarray(ref_desc, np.float64)
        self.patch_blocks = None
        if patch_blocks is not None:
            # one block per FeatureMap (host numpy or device-resident), uploaded without host concatenation
            blocks = list(patch_blocks)
            for b in blocks:
                if b.dtype not in DTYPE_IDS or not b.flags["C_CONTIGUOUS"] or b.ndim != 4 or b.shape[1:] != blocks[0].shape[1:]:
                    raise ValueError("patch blocks must be C-contiguous [N,H,W,C] arrays of one dtype/shape")
            self.patch_blocks = blocks
            self._block_ptrs = (C.c_void_p * len(blocks))(*[getattr(b, "ptr", None) or b.ctypes.data for b in blocks])
            self._block_counts = np.array([b.shape[0] for b in blocks], np.int64)
            patches = blocks[0]
            self._shape = (int(self._block_counts.sum()),) + tuple(blocks[0].shape[1:])
            self._dtype = np.dtype(blocks[0].dtype)
        else:
            if patches.dtype not in DTYPE_IDS or not patches.flags["C_CONTIGUOUS"] or patches.ndim != 4:
                raise ValueError("patches must be a C-contiguous [N,H,W,C] f16/f32/f64 array")
            self._shape, self._dtype = tuple(patches.shape), np.dtype(patches.dtype)
        self.patches = patches
        self.corner = _as(corner, np.int32, (-1, 2))
        self.scale = _as(scale, np.float64, (-1, 2))
        self.kp_patch = _as(kp_patch, np.int64)
        self.bound = float(bound)
        self.patches_are_sparse = bool(patches_are_sparse)
        self.upsampling_factor = float(upsampling_factor)

    @property
    def channels(self):
        return self._shape[3]

    def desc(self):
        d = KADesc()
        d.n_keypoints = len(self.keypoints)
        d.keypoints = _ptr(self.keypoints); d.kp_const = _ptr(self.kp_const); d.kp_patch = _ptr(self.kp_patch)
        d.n_edges = len(self.edge_src)
        d.edge_src = _ptr(self.edge_src); d.edge_dst = _ptr(self.edge_dst)
        d.edge_weight = _ptr(self.edge_weight); d.edge_problem = _ptr(self.edge_problem)
        d.n_problems = self.n_problems
        d.n_patches = self._shape[0]
        d.patches_on_device = 0
        if self.patch_blocks is not None:
            d.patches = None
            d.n_patch_blocks = len(self.patch_blocks)
            d.patch_block_ptrs = C.cast(self._block_ptrs, C.c_void_p)
            d.patch_block_counts = _ptr(self._block_counts)
        else:
            d.patches = _ptr(self.patches)
        d.patch_dtype = DTYPE_IDS[self._dtype]
        d.ph, d.pw, d.channels = self._shape[1:]
        d.corner = _ptr(self.corner); d.scale = _ptr(self.scale)
        d.upsampling_factor = self.upsampling_factor
        d.bound = self.bound
        d.patches_are_sparse = int(self.patches_are_sparse)
        if self.ref_desc is not None:
            if self.ref_desc.ndim != 2 or self.ref_desc.shape[1] != self._shape[3]:
                raise ValueError("ref_desc must be [n_ref, channels]")
            d.ref_desc = _ptr(self.ref_desc); d.n_ref_desc = len(self.ref_desc)
        return d

    def copy(self):
        import copy as _copy
        o = _copy.copy(self)
        o.keypoints = self.keypoints.copy()
        return o

    # ---- multi-GPU: whole problems per rank (SURVEY §8e "KA: no collective")
    def problem_weights(self):
        """patch bytes a problem pulls in = distinct keypoints of its edges x bytes of one patch"""
        per_patch = int(np.prod(self._shape[1:])) * self._dtype.itemsize
        w = np.zeros(self.n_problems, np.int64)
        stride = len(self.keypoints) + 1
        ends = (self.edge_src,) if self.ref_desc is not None else (self.edge_src, self.edge_dst)
        key = np.unique(np.concatenate([self.edge_problem.astype(np.int64) * stride + e for e in ends]))
        np.add.at(w, key // stride, 1)
        return w * per_patch

    def shard(self, rank_of_problem, rank):
        """-> (KAProblem of the problems `rank` owns, global index of each of its keypoints).  Keypoints, patches and
        metadata are compacted to what the shard touches; solve it like any problem and hand both to merge_shard."""
        rank_of_problem = np.asarray(rank_of_problem)
        if len(rank_of_problem) != self.n_problems:
            raise ValueError("rank_of_problem must have one entry per problem")
        mine = rank_of_problem[self.edge_problem] == rank
        es, ed = self.edge_src[mine], self.edge_dst[mine]
        used = np.unique(es if self.ref_desc is not None else np.concatenate([es, ed]))
        local = np.full(len(self.keypoints), -1, np.int64); local[used] = np.arange(len(used))
        plocal = np.cumsum(rank_of_problem == rank) - 1                      # relabel the owned problems 0..m-1
        kp_patch = self.kp_patch[used] if self.kp_patch is not None and len(self.kp_patch) else used
        if self.patch_blocks is not None:
            starts = np.concatenate([[0], np.cumsum(self._block_counts)])
            blk = np.searchsorted(starts, kp_patch, side="right") - 1
            patches = np.empty((len(used),) + self._shape[1:], self._dtype)
            for k, (b, g) in enumerate(zip(blk, kp_patch)):
                patches[k] = np.asarray(self.patch_blocks[b][g - starts[b]])
        else:
            patches = np.ascontiguousarray(self.patches[kp_patch])
        if len(used) == 0:
            patches = np.zeros((0,) + self._shape[1:], self._dtype)
        sub = KAProblem(keypoints=self.keypoints[used], kp_const=self.kp_const[used], edge_src=local[es],
                        edge_dst=ed if self.ref_desc is not None else local[ed], edge_weight=None if self.edge_weight is None else self.edge_weight[mine],
                        edge_problem=plocal[self.edge_problem[mine]], n_problems=int(np.sum(rank_of_problem == rank)),
                        patches=patches, corner=self.corner[kp_patch], scale=self.scale[kp_patch], kp_patch=None,
                        bound=self.bound, patches_are_sparse=self.patches_are_sparse,
                        upsampling_factor=self.upsampling_factor, ref_desc=self.ref_desc)
        return sub, used

    def merge_shard(self, sub, kp_global):
        """write a solved shard's keypoints back"""
        self.keypoints[kp_global] = sub.keypoints


class QKABatch(KAProblem):
    """numpy arrays of a batch of query keypoint adjustments + the ctypes view (pxr_qka_desc).  Per query: a keypoint
    range kp_begin, a patch block [n_q, H, W, C] (host numpy array or device memory) with its corners and scales, and
    whether its map is sparse; per keypoint: its patch within the query's block and a range of fixed fp64 descriptors,
    one residual block each.  It is also the KAProblem of the same problems (query mode, one problem per query, the
    blocks back to back) when the blocks are host arrays: desc() gives that pxr_ka_desc, qka_desc() the batched one.
    `results` holds one dict per query (the pxr_qka_result fields) once solved."""

    def __init__(self, keypoints, kp_begin, kp_patch, desc_begin, descs, patch_blocks, corner, scale, patches_are_sparse,
                 bound=4.0, upsampling_factor=1.0, max_wave_bytes=0.0):
        self.keypoints = _as(keypoints, np.float64, (-1, 2)).copy()
        self.kp_begin = _as(kp_begin, np.int64)
        self.kp_patch_local = _as(kp_patch, np.int64)
        self.desc_begin = _as(desc_begin, np.int64)
        nq, nk = len(self.kp_begin) - 1, len(self.keypoints)
        self.patch_blocks = list(patch_blocks)
        if len(self.patch_blocks) != nq:
            raise ValueError("one patch block per query")
        self._qptrs, self.patch_counts, shape, self.patch_dtype = _patch_blocks(self.patch_blocks)
        self.ph, self.pw, ch = shape
        self.ref_desc = np.ascontiguousarray(descs, np.float64).reshape(-1, ch) if len(descs) else np.zeros((0, ch))
        self.corner = _as(corner, np.int32, (-1, 2))
        self.scale = _as(scale, np.float64, (-1, 2))
        self.sparse = _as(patches_are_sparse, np.uint8)
        self.bound = float(bound)
        self.upsampling_factor = float(upsampling_factor)
        self.max_wave_bytes = float(max_wave_bytes)
        self._shape = (int(self.patch_counts.sum()), self.ph, self.pw, ch)
        self._dtype = {v: k for k, v in DTYPE_IDS.items()}[self.patch_dtype]
        # the same problems as one pxr_ka_desc: edge = (keypoint, descriptor), problem = query
        counts = np.diff(self.desc_begin) if nk else np.zeros(0, np.int64)
        self.edge_src = np.repeat(np.arange(nk, dtype=np.int64), counts)
        self.edge_dst = np.arange(len(self.edge_src), dtype=np.int64)
        self.edge_problem = np.repeat(np.arange(nq, dtype=np.int32), np.diff(self.desc_begin[self.kp_begin])) if nk else \
            np.zeros(0, np.int32)
        self.edge_weight = None
        self.kp_const = np.zeros(nk, np.uint8)
        self.n_problems = nq
        first = np.concatenate([[0], np.cumsum(self.patch_counts)])[:-1] if nq else np.zeros(0, np.int64)
        self.kp_patch = self.kp_patch_local + np.repeat(first, np.diff(self.kp_begin)).astype(np.int64)
        self.patches = None
        self.results = [dict(status=PXR_OK, num_residual_blocks=int(self.desc_begin[self.kp_begin[q + 1]] -
                                                                    self.desc_begin[self.kp_begin[q]]) if nk else 0,
                             initial_cost=0.0, final_cost=0.0, num_successful_steps=0, num_unsuccessful_steps=0,
                             num_iterations=0, termination_type=1) for q in range(nq)]

    @property
    def n_queries(self):
        return len(self.kp_begin) - 1

    @property
    def patches_are_sparse(self):
        """the one flag of the pxr_ka_desc view: it exists when the queries agree or when bound > 0 decides alone"""
        if self.bound <= 0 and len(set(self.sparse.tolist())) > 1:
            raise ValueError("the queries mix sparse and dense maps with bound <= 0: no single pxr_ka_desc holds them")
        return bool(self.sparse[0]) if len(self.sparse) else True

    def desc(self):
        if any(not isinstance(b, np.ndarray) for b in self.patch_blocks):
            raise ValueError("the pxr_ka_desc view of a query batch takes host patch blocks")
        d = KADesc()
        d.n_keypoints = len(self.keypoints)
        d.keypoints = _ptr(self.keypoints); d.kp_const = _ptr(self.kp_const); d.kp_patch = _ptr(self.kp_patch)
        d.n_edges = len(self.edge_src)
        d.edge_src = _ptr(self.edge_src); d.edge_dst = _ptr(self.edge_dst); d.edge_problem = _ptr(self.edge_problem)
        d.n_problems = self.n_problems
        d.n_patches = self._shape[0]
        d.n_patch_blocks = self.n_queries
        d.patch_block_ptrs = C.cast(self._qptrs, C.c_void_p); d.patch_block_counts = _ptr(self.patch_counts)
        d.patch_dtype = self.patch_dtype
        d.ph, d.pw, d.channels = self._shape[1:]
        d.corner = _ptr(self.corner); d.scale = _ptr(self.scale)
        d.upsampling_factor = self.upsampling_factor
        d.bound = self.bound
        d.patches_are_sparse = int(self.patches_are_sparse)
        d.ref_desc = _ptr(self.ref_desc); d.n_ref_desc = len(self.ref_desc)
        return d

    def qka_desc(self):
        d = QKADesc()
        d.n_queries = self.n_queries
        d.kp_begin = _ptr(self.kp_begin); d.patch_blocks = C.cast(self._qptrs, C.c_void_p)
        d.patch_counts = _ptr(self.patch_counts); d.patches_are_sparse = _ptr(self.sparse)
        d.keypoints = _ptr(self.keypoints); d.kp_patch = _ptr(self.kp_patch_local); d.desc_begin = _ptr(self.desc_begin)
        d.descs = _ptr(self.ref_desc); d.corner = _ptr(self.corner); d.scale = _ptr(self.scale)
        d.upsampling_factor = self.upsampling_factor; d.bound = self.bound
        d.ph, d.pw, d.channels, d.patch_dtype = self.ph, self.pw, self._shape[3], self.patch_dtype
        d.max_wave_bytes = self.max_wave_bytes
        return d
