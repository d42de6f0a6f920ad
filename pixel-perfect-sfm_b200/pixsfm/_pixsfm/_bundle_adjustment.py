"""Mirror of `pixsfm._pixsfm._bundle_adjustment` (pixsfm/bundle_adjustment/bindings.cc:28-177) backed by the
C-ABI: BundleAdjustmentSetup, BundleOptimizerOptions, ReferenceConfig, ReferenceExtractor and
FeatureReferenceBundleOptimizer.  This layer restates the reference's problem construction
(bundle_optimizer.h:139-165,247-331) and parameterisation rules (:335-442) as integer logic that
resolves to the SoA problem IR of include/pxr.h; all arithmetic runs in libpxr.so on the GPU."""
import numpy as np

from . import _capi, _engine
from ._base import InterpolationConfig
from ._features import FeatureView, PatchSlab, Reference
from .. import logger


class BundleAdjustmentSetup:
    """colmap::BundleAdjustmentConfig with pixsfm's throwing overrides (bundle_adjustment_options.cc:7-31)."""

    def __init__(self):
        self._images, self._const_poses, self._const_tvecs = set(), set(), {}
        self._const_cameras, self._var_points, self._const_points = set(), set(), set()

    # images
    def add_image(self, image_id): self._images.add(int(image_id))
    def add_images(self, image_ids):
        for i in image_ids: self.add_image(i)
    def has_image(self, image_id): return int(image_id) in self._images
    def remove_image(self, image_id): self._images.discard(int(image_id))
    @property
    def image_ids(self): return set(self._images)
    def num_images(self): return len(self._images)
    # cameras
    def set_constant_camera(self, camera_id): self._const_cameras.add(int(camera_id))
    def set_variable_camera(self, camera_id): self._const_cameras.discard(int(camera_id))
    def is_constant_camera(self, camera_id): return int(camera_id) in self._const_cameras
    # poses
    def set_constant_pose(self, image_id):
        if not self.has_image(image_id) or self.has_constant_tvec(image_id):
            raise ValueError("set_constant_pose: image must be in the setup and must not have a constant tvec")
        self._const_poses.add(int(image_id))
    def set_variable_pose(self, image_id): self._const_poses.discard(int(image_id))
    def has_constant_pose(self, image_id): return int(image_id) in self._const_poses
    def set_constant_tvec(self, image_id, idxs):
        idxs = [int(i) for i in idxs]
        if not (0 < len(idxs) <= 3) or not self.has_image(image_id) or self.has_constant_pose(image_id) or len(set(idxs)) != len(idxs):
            raise ValueError("set_constant_tvec: invalid arguments")
        self._const_tvecs[int(image_id)] = idxs
    def remove_constant_tvec(self, image_id): self._const_tvecs.pop(int(image_id), None)
    def has_constant_tvec(self, image_id): return int(image_id) in self._const_tvecs
    def constant_tvec(self, image_id): return self._const_tvecs[int(image_id)]
    # points
    def add_variable_point(self, point3D_id):
        if self.has_constant_point(point3D_id): raise ValueError("point is already constant")
        self._var_points.add(int(point3D_id))
    def add_constant_point(self, point3D_id):
        if self.has_variable_point(point3D_id): raise ValueError("point is already variable")
        self._const_points.add(int(point3D_id))
    def has_point(self, p): return self.has_variable_point(p) or self.has_constant_point(p)
    def has_variable_point(self, p): return int(p) in self._var_points
    def has_constant_point(self, p): return int(p) in self._const_points
    def remove_variable_point(self, p): self._var_points.discard(int(p))
    def remove_constant_point(self, p): self._const_points.discard(int(p))
    @property
    def variable_point3D_ids(self): return set(self._var_points)
    @property
    def constant_point3D_ids(self): return set(self._const_points)


class _DictOptions:
    """make_dataclass semantics (_pixsfm/src/helpers.h:149-303): dict/kwargs construction, strict keys."""
    _defaults = {}

    def __init__(self, conf=None, **kw):
        for k, v in self._defaults.items():
            setattr(self, k, v() if callable(v) else v)
        self.mergedict(dict(conf or {}, **kw))

    def mergedict(self, d):
        for k, v in d.items():
            if k not in self._defaults:
                raise ValueError("%s: unknown option '%s'" % (type(self).__name__, k))
            cur = getattr(self, k)
            if isinstance(cur, dict) and isinstance(v, dict):
                merged = dict(cur); merged.update(v); v = merged
            setattr(self, k, v)

    def todict(self):
        return {k: getattr(self, k) for k in self._defaults}


_SOLVER_KEYS = {"function_tolerance", "gradient_tolerance", "parameter_tolerance", "minimizer_progress_to_stdout",
                "max_num_iterations", "max_linear_solver_iterations", "max_num_consecutive_invalid_steps",
                "max_consecutive_nonmonotonic_steps", "use_inner_iterations", "use_nonmonotonic_steps",
                "update_state_every_iteration", "num_threads", "callbacks", "inner_iteration_tolerance",
                "initial_trust_region_radius", "max_trust_region_radius", "min_trust_region_radius",
                "min_relative_decrease", "min_lm_diagonal", "max_lm_diagonal", "jacobi_scaling", "logging_type",
                "deterministic"}       # the last one is this library's own: fixed-order (bit-reproducible) assembly


def solver_options_from(loss, solver, base):
    """{"name","params"} + pyceres-SolverOptions-like dict -> pxr_solver_options"""
    o = base
    name = str(loss.get("name", "cauchy")).lower()
    if name not in _capi.LOSS_IDS:
        raise ValueError("unsupported loss '%s'" % name)
    o.loss_type = _capi.LOSS_IDS[name]
    params = loss.get("params", [])
    o.loss_scale = float(params[0]) if len(params) else 1.0
    for k, v in solver.items():
        if k not in _SOLVER_KEYS:
            raise ValueError("solver: unknown option '%s'" % k)
        if hasattr(o, k) and k != "callbacks":
            setattr(o, k, type(getattr(o, k))(v))
    return o


class BundleOptimizerOptions(_DictOptions):
    """bundle_adjustment_options.h:44-98 (C++ defaults; the Python BundleAdjuster overrides `solver`)"""
    _defaults = dict(refine_focal_length=True, refine_principal_point=False, refine_extra_params=True,
                     refine_extrinsics=True, print_summary=True, min_track_length=-1,
                     loss=lambda: {"name": "cauchy", "params": [0.25]},
                     solver=lambda: {"function_tolerance": 0.0, "gradient_tolerance": 0.0, "parameter_tolerance": 0.0,
                                     "max_num_iterations": 100, "max_linear_solver_iterations": 200,
                                     "max_num_consecutive_invalid_steps": 10, "use_inner_iterations": False})


class ReferenceConfig(_DictOptions):
    """reference_extractor.h:57-67 (C++ default iters=10; the Python layer passes 100)"""
    _defaults = dict(keep_observations=False, iters=10, compute_offsets3D=False, num_threads=-1,
                     loss=lambda: {"name": "cauchy", "params": [0.25]})


class CostMapConfig(_DictOptions):
    """costmap_extractor.h:18-40 (bindings.cc:55-65); loss defaults to TrivialLoss."""
    _defaults = dict(upsampling_factor=1.0, as_gradientfield=True, compute_cross_derivative=False, apply_sqrt=False,
                     num_threads=-1, dense_cut_size=12, loss=lambda: {"name": "trivial", "params": []})

    def get_effective_channels(self):
        if self.as_gradientfield:
            return 4 if self.compute_cross_derivative else 3
        return 1


def _cam_const_mask(camera, options, setup, camera_id):
    constant_camera = not (options.refine_focal_length or options.refine_principal_point or options.refine_extra_params)
    if constant_camera or setup.is_constant_camera(camera_id):
        return 0xFFFFFFFF
    focal, pp, extra = _capi.CAMERA_PARAM_GROUPS[int(camera.model_id)]
    mask = 0
    if not options.refine_focal_length: mask |= focal
    if not options.refine_principal_point: mask |= pp
    if not options.refine_extra_params: mask |= extra
    return mask


class ProblemIR:
    """Index maps between the reconstruction and the flat problem IR."""

    def __init__(self):
        self.image_ids, self.camera_ids, self.point_ids = [], [], []
        self.obs = []  # (image_id, point2D_idx, point3D_id)


def _ids(values):
    return np.ascontiguousarray(sorted(int(v) for v in values), np.int64)


def _patch_plan(ir, feature_view):
    """obs -> global patch index, blocks in first-use order (what PatchSlab builds one observation at a time),
    vectorised per image"""
    obs_image = np.fromiter((o[0] for o in ir.obs), np.int64, len(ir.obs)) if not hasattr(ir, "obs_image_id") else ir.obs_image_id
    obs_p2d = np.fromiter((o[1] for o in ir.obs), np.int64, len(ir.obs)) if not hasattr(ir, "obs_point2D_idx") else ir.obs_point2D_idx
    uniq, first = np.unique(obs_image, return_index=True)
    order = uniq[np.argsort(first, kind="stable")]
    blocks, corners, scales, offsets = [], [], [], {}
    obs_patch = np.zeros(len(obs_image), np.int64)
    n = 0
    for image_id in order:
        image_id = int(image_id)
        name = feature_view.image_name(image_id)
        fmap = feature_view.get_feature_map(image_id)
        sel = np.flatnonzero(obs_image == image_id) if len(order) < 64 else None
        if sel is None:
            sel = ir._by_image[image_id]
        if name not in offsets:
            offsets[name] = n
            blocks.append(fmap.patches); corners.append(fmap.corners); scales.append(np.tile(fmap.scale, (fmap.size(), 1)))
            n += fmap.size()
        if not fmap.is_sparse:
            local = np.full(len(sel), fmap.local_index(0), np.int64)
        else:
            ids = np.asarray(fmap.point2D_ids, np.int64)
            srt = np.argsort(ids, kind="stable")
            pos = np.searchsorted(ids[srt], obs_p2d[sel])
            pos = np.minimum(pos, len(ids) - 1)
            if np.any(ids[srt][pos] != obs_p2d[sel]):
                missing = obs_p2d[sel][ids[srt][pos] != obs_p2d[sel]][0]
                raise KeyError(int(missing))
            local = srt[pos]
        obs_patch[sel] = offsets[name] + local
    return blocks, np.concatenate(corners), np.concatenate(scales), obs_patch, offsets


def build_problem(reconstruction, feature_view, setup, options, references=None, for_references=None):
    """BundleOptimizer::SetUp + Parameterize (bundle_optimizer.h:139-165,247-442) through the C++ builder in libpxr
    (pxr_problem_build, csrc/pxr_problem.cu) -> (_capi.BAProblem, ProblemIR).  With `for_references` (a set of
    point3D ids) the observation list is ReferenceExtractor::GetVisibleObservations' (reference_extractor.h:171-205).
    The reconstruction is handed over as arrays (`as_arrays()`); `build_problem_py` is the per-object restatement the
    tests compare it with."""
    import ctypes as C
    rec = reconstruction
    A = rec.as_arrays() if hasattr(rec, "as_arrays") else __import__("pixsfm.util.colmap_types", fromlist=["x"]).reconstruction_arrays(rec)
    lib = _capi.load_lib()
    p = _capi.ptr
    view = _capi.ReconView(n_images=len(A["image_id"]), image_id=p(A["image_id"]), image_camera_id=p(A["image_camera_id"]),
                           p2d_begin=p(A["p2d_begin"]), p2d_point3D_id=p(A["p2d_point3D_id"]),
                           n_cameras=len(A["camera_id"]), camera_id=p(A["camera_id"]), camera_model=p(A["camera_model"]),
                           n_points=len(A["point3D_id"]), point3D_id=p(A["point3D_id"]), track_begin=p(A["track_begin"]),
                           track_image_id=p(A["track_image_id"]), track_point2D_idx=p(A["track_point2D_idx"]))
    keep = [A]
    if for_references is None:
        img_ids = _ids(setup.image_ids)
        if hasattr(rec, "qvec") and isinstance(getattr(rec, "qvec"), np.ndarray):      # image.NormalizeQvec() (:251)
            rows = np.searchsorted(A["image_id"], img_ids)
            rec.qvec[rows] /= np.linalg.norm(rec.qvec[rows], axis=1, keepdims=True)
        else:
            for image_id in img_ids:
                image = rec.images[int(image_id)]
                image.qvec /= np.linalg.norm(image.qvec)
        cp, cam, vp, cpt = _ids(setup._const_poses), _ids(setup._const_cameras), _ids(setup._var_points), _ids(setup._const_points)
        tv = _ids(setup._const_tvecs.keys())
        tvm = np.array([sum(1 << int(k) for k in setup._const_tvecs[int(i)]) for i in tv], np.uint8)
        sv = _capi.SetupView(n_images=len(img_ids), image_ids=p(img_ids), n_const_poses=len(cp), const_pose_ids=p(cp),
                             n_const_tvecs=len(tv), const_tvec_ids=p(tv), const_tvec_masks=p(tvm),
                             n_const_cameras=len(cam), const_camera_ids=p(cam), n_var_points=len(vp), var_point_ids=p(vp),
                             n_const_points=len(cpt), const_point_ids=p(cpt))
        bo = _capi.BuildOptions(refine_focal_length=int(bool(options.refine_focal_length)),
                                refine_principal_point=int(bool(options.refine_principal_point)),
                                refine_extra_params=int(bool(options.refine_extra_params)),
                                refine_extrinsics=int(bool(options.refine_extrinsics)),
                                min_track_length=int(options.min_track_length), mode=0)
        keep += [img_ids, cp, cam, vp, cpt, tv, tvm]
        sv_ref = C.byref(sv)
    else:
        ref_ids = _ids(for_references)
        # which track elements have a feature patch: resolved per image
        timg, tp2d = A["track_image_id"], A["track_point2D_idx"]
        has = np.zeros(len(timg), np.uint8)
        order_t = np.argsort(timg, kind="stable")              # track elements grouped by image: one sort instead of a scan per image
        uniq_t, first_t = np.unique(timg[order_t], return_index=True)
        bounds_t = np.append(first_t, len(order_t))
        for k_img, image_id in enumerate(uniq_t):
            sel = order_t[bounds_t[k_img]:bounds_t[k_img + 1]]
            name = feature_view._id_to_name.get(int(image_id))
            if name is None or not feature_view.fset.has_fmap(name):
                continue
            fmap = feature_view.fset.fmap(name)
            if not fmap.is_sparse:
                has[sel] = 1 if fmap.has_point2D(0) else 0
            else:
                has[sel] = np.isin(tp2d[sel], np.asarray(fmap.point2D_ids, np.int64))
        bo = _capi.BuildOptions(mode=1, min_track_length=-1, n_ref_points=len(ref_ids), ref_point_ids=p(ref_ids), track_has_patch=p(has))
        keep += [ref_ids, has]
        sv_ref = None
    handle = C.c_void_p()
    _capi.check(lib.pxr_problem_build(C.byref(view), sv_ref, C.byref(bo), C.byref(handle)))
    try:
        n_obs, n_img, n_cam, n_pts = (C.c_int64() for _ in range(4))
        _capi.check(lib.pxr_problem_sizes(handle, C.byref(n_obs), C.byref(n_img), C.byref(n_cam), C.byref(n_pts)))
        n_obs, n_img, n_cam, n_pts = n_obs.value, n_img.value, n_cam.value, n_pts.value
        o_pid, o_img, o_p2d = (np.zeros(n_obs, np.int64) for _ in range(3))
        obs_img, obs_pt = np.zeros(n_obs, np.int32), np.zeros(n_obs, np.int64)
        image_ids, camera_ids, point_ids = np.zeros(n_img, np.int64), np.zeros(n_cam, np.int64), np.zeros(n_pts, np.int64)
        img_cam = np.zeros(n_img, np.int32)
        pose_const, tmask, point_const = np.zeros(n_img, np.uint8), np.zeros(n_img, np.uint8), np.zeros(n_pts, np.uint8)
        cam_mask = np.zeros(n_cam, np.uint32)
        _capi.check(lib.pxr_problem_copy(handle, p(o_pid), p(o_img), p(o_p2d), p(obs_img), p(obs_pt), p(image_ids), p(camera_ids),
                                         p(point_ids), p(img_cam), p(pose_const), p(tmask), p(point_const), p(cam_mask)))
    finally:
        lib.pxr_problem_destroy(handle)
    del keep
    if for_references is not None:
        # the reference warns about every track element without a patch (reference_extractor.h:187-191)
        missing = int((A["track_begin"][np.searchsorted(A["point3D_id"], ref_ids) + 1]
                       - A["track_begin"][np.searchsorted(A["point3D_id"], ref_ids)]).sum()) - n_obs if len(ref_ids) else 0
        if missing > 0:
            logger.warning("Warning: %d track elements have no feature patch.", missing)
    ir = ProblemIR()
    ir.image_ids, ir.camera_ids, ir.point_ids = image_ids.tolist(), camera_ids.tolist(), point_ids.tolist()
    ir.obs_image_id, ir.obs_point2D_idx, ir.obs_point3D_id = o_img, o_p2d, o_pid
    ir.obs = _LazyObs(o_img, o_p2d, o_pid)
    if n_obs == 0:
        import types
        return types.SimpleNamespace(n_obs=0), ir
    if len(image_ids) >= 64:      # one pass instead of one mask per image
        srt = np.argsort(o_img, kind="stable")
        bounds = np.searchsorted(o_img[srt], image_ids)
        bounds = np.append(bounds, len(srt))
        ir._by_image = {int(i): srt[bounds[k]:bounds[k + 1]] for k, i in enumerate(image_ids)}
    if feature_view is None:       # geometric BA: the observed keypoints instead of feature patches
        obs_xy = _observed_keypoints(rec, A, o_img, o_p2d)
    else:
        blocks, corners, scales, obs_patch, offsets = _patch_plan(ir, feature_view)
        ir.slab_offsets = offsets
    # parameters of the blocks, in index order
    if isinstance(getattr(rec, "xyz", None), np.ndarray) and hasattr(rec, "point3D_id"):
        rows_i = np.searchsorted(rec.image_id, image_ids); rows_p = np.searchsorted(rec.point3D_id, point_ids)
        rows_c = np.searchsorted(rec.camera_id, camera_ids)
        qvec, tvec, xyz = rec.qvec[rows_i], rec.tvec[rows_i], rec.xyz[rows_p]
        cam_params = [rec.cam_params[r] for r in rows_c]
        cam_model = rec.camera_model[rows_c]
        ir._rows = (rows_i, rows_c, rows_p)
    else:
        qvec = np.array([rec.images[i].qvec for i in ir.image_ids], np.float64).reshape(-1, 4)
        tvec = np.array([rec.images[i].tvec for i in ir.image_ids], np.float64).reshape(-1, 3)
        xyz = np.array([rec.points3D[q].xyz for q in ir.point_ids], np.float64).reshape(-1, 3)
        cam_params = [np.asarray(rec.cameras[c].params, np.float64) for c in ir.camera_ids]
        cam_model = np.array([int(rec.cameras[c].model_id) for c in ir.camera_ids], np.int32)
    if feature_view is None:
        prob = _capi.BAProblem(cam_model=cam_model, cam_params=cam_params, cam_const_mask=cam_mask, qvec=qvec, tvec=tvec,
                               img_cam=img_cam, pose_const=pose_const, tvec_const_mask=tmask, xyz=xyz,
                               point_const=point_const, obs_img=obs_img, obs_pt=obs_pt, patches=None, corner=None,
                               scale=None, obs_xy=obs_xy)
        return prob, ir
    refs = None
    if references is not None:
        C_ = feature_view.channels
        dense = getattr(references, "dense", None)
        if dense is not None and dense[1].shape[1] == C_ and bool(dense[2].all()) and np.array_equal(dense[0], point_ids):
            refs = np.ascontiguousarray(dense[1], np.float64)
        elif dense is not None and dense[1].shape[1] == C_ and bool(dense[2].all()) and np.all(np.isin(point_ids, dense[0])):
            refs = np.ascontiguousarray(dense[1][np.searchsorted(dense[0], point_ids)], np.float64)
        else:
            refs = np.zeros((n_pts, C_))
            for k, pid in enumerate(ir.point_ids):
                refs[k] = np.asarray(references[pid].descriptor, np.float64).reshape(-1)[:C_]
    prob = _capi.BAProblem(cam_model=cam_model, cam_params=cam_params, cam_const_mask=cam_mask, qvec=qvec, tvec=tvec,
                           img_cam=img_cam, pose_const=pose_const, tvec_const_mask=tmask, xyz=xyz, point_const=point_const,
                           obs_img=obs_img, obs_pt=obs_pt, patches=None, corner=corners, scale=scales, refs=refs,
                           obs_patch=obs_patch, patch_blocks=blocks)
    return prob, ir


def _observed_keypoints(rec, A, obs_image_id, obs_point2D_idx):
    """[n_obs, 2] point2D.XY() of every observation: what GeometricBundleOptimizer::AddResiduals hands the cost functor
    (geometric_bundle_optimizer.h:56-73).  An array-backed reconstruction provides them as `p2d_xy` [n_points2D, 2] in
    the order of its `p2d_begin`."""
    p2d_xy = getattr(rec, "p2d_xy", None)
    if p2d_xy is not None:
        rows = np.searchsorted(A["image_id"], obs_image_id)
        return np.ascontiguousarray(np.asarray(p2d_xy, np.float64)[A["p2d_begin"][rows] + obs_point2D_idx])
    if not hasattr(rec, "images") or not hasattr(rec, "points3D"):
        raise ValueError("geometric bundle adjustment needs the keypoints: an array-backed reconstruction must carry p2d_xy")
    out = np.empty((len(obs_image_id), 2))
    for k, (i, j) in enumerate(zip(obs_image_id.tolist(), obs_point2D_idx.tolist())):
        out[k] = rec.images[i].points2D[j].xy
    return out


class _LazyObs:
    """`ir.obs[k] -> (image_id, point2D_idx, point3D_id)` without materialising a list of tuples"""

    def __init__(self, image_id, point2D_idx, point3D_id):
        self._a = (image_id, point2D_idx, point3D_id)

    def __len__(self):
        return len(self._a[0])

    def __getitem__(self, k):
        if isinstance(k, slice):
            return [self[i] for i in range(*k.indices(len(self)))]
        return (int(self._a[0][k]), int(self._a[1][k]), int(self._a[2][k]))

    def __iter__(self):
        return (self[k] for k in range(len(self)))

    def __eq__(self, other):
        return list(self) == list(other)


def build_problem_py(reconstruction, feature_view, setup, options, references=None, for_references=None):
    """The per-object Python restatement of BundleOptimizer::SetUp + Parameterize (what build_problem was before the
    C++ builder): kept as the independent statement the tests compare pxr_problem_build with."""
    rec = reconstruction
    ir = ProblemIR()
    obs = []                      # (point3D_id, image_id, point2D_idx)
    reg_track = {}                # point3D_id -> set(track idx)   (point3D_reg_track_idx_)
    image_num_residuals, camera_num_residuals = {}, {}
    setup_images = sorted(setup.image_ids) if setup is not None else []
    extra_const_cameras = set()

    def add_residual(image_id, point2D_idx):
        image = rec.images[image_id]
        p2D = image.points2D[point2D_idx]
        if not p2D.has_point3D():
            return
        pid = p2D.point3D_id
        obs.append((pid, image_id, point2D_idx))
        constant_pose = (not options.refine_extrinsics) or setup.has_constant_pose(image_id)
        if not constant_pose:
            image_num_residuals[image_id] = image_num_residuals.get(image_id, 0) + 1
        track = rec.points3D[pid].track.elements
        for k, el in enumerate(track):   # RegisterPoint3DObservation (linear search, :321-327)
            if el.image_id == image_id and el.point2D_idx == point2D_idx:
                reg_track.setdefault(pid, set()).add(k)
                break
        else:
            raise RuntimeError("Failed to register track element.")
        camera_num_residuals[image.camera_id] = camera_num_residuals.get(image.camera_id, 0) + 1

    if for_references is None:
        for image_id in setup_images:                      # AddImageToProblem (:247-275)
            image = rec.images[image_id]
            image.qvec /= np.linalg.norm(image.qvec)       # image.NormalizeQvec()
            for p2D_idx in range(len(image.points2D)):
                p2D = image.points2D[p2D_idx]
                if not p2D.has_point3D():
                    continue
                if rec.points3D[p2D.point3D_id].track.length() < options.min_track_length:
                    continue
                add_residual(image_id, p2D_idx)
        for pid in list(sorted(setup.variable_point3D_ids)) + list(sorted(setup.constant_point3D_ids)):   # AddPointToProblem (:277-313)
            track = rec.points3D[pid].track.elements
            if len(reg_track.get(pid, ())) == len(track):
                continue
            for el in track:
                if setup.has_image(el.image_id):
                    continue
                cam_id = rec.images[el.image_id].camera_id
                if camera_num_residuals.get(cam_id, 0) == 0:
                    extra_const_cameras.add(cam_id)
                add_residual(el.image_id, el.point2D_idx)
    else:
        for pid in sorted(for_references):
            for el in rec.points3D[pid].track.elements:
                if not feature_view.has_feature_patch(el.image_id, el.point2D_idx):
                    logger.warning("Warning: Patch at (%d, %d) does not exist.", el.image_id, el.point2D_idx)
                    continue
                obs.append((pid, el.image_id, el.point2D_idx))

    # canonical order of the IR: observations sorted by point id (stable: image enumeration order kept)
    order = sorted(range(len(obs)), key=lambda k: obs[k][0])
    obs = [obs[k] for k in order]
    ir.point_ids = sorted({o[0] for o in obs})
    ir.image_ids = sorted({o[1] for o in obs})
    ir.camera_ids = sorted({rec.images[i].camera_id for i in ir.image_ids})
    pidx = {p: k for k, p in enumerate(ir.point_ids)}
    iidx = {i: k for k, i in enumerate(ir.image_ids)}
    cidx = {c: k for k, c in enumerate(ir.camera_ids)}
    ir.obs = [(o[1], o[2], o[0]) for o in obs]

    n_img, n_cam, n_pts = len(ir.image_ids), len(ir.camera_ids), len(ir.point_ids)
    cam_model = np.array([int(rec.cameras[c].model_id) for c in ir.camera_ids], np.int32)
    cam_params = [np.asarray(rec.cameras[c].params, np.float64) for c in ir.camera_ids]
    qvec = np.array([rec.images[i].qvec for i in ir.image_ids], np.float64).reshape(-1, 4)
    tvec = np.array([rec.images[i].tvec for i in ir.image_ids], np.float64).reshape(-1, 3)
    img_cam = np.array([cidx[rec.images[i].camera_id] for i in ir.image_ids], np.int32)
    xyz = np.array([rec.points3D[p].xyz for p in ir.point_ids], np.float64).reshape(-1, 3)
    pose_const = np.ones(n_img, np.uint8)
    tmask = np.zeros(n_img, np.uint8)
    point_const = np.zeros(n_pts, np.uint8)
    cam_mask = np.full(n_cam, 0xFFFFFFFF, np.uint32)
    if for_references is None:
        # ParameterizeImages (:360-398)
        for image_id, nres in image_num_residuals.items():
            if nres <= 0:
                continue
            constant_pose = (not options.refine_extrinsics) or setup.has_constant_pose(image_id) or not setup.has_image(image_id)
            if not constant_pose:
                pose_const[iidx[image_id]] = 0
                if setup.has_constant_tvec(image_id):
                    for k in setup.constant_tvec(image_id):
                        tmask[iidx[image_id]] |= (1 << k)
        # ParameterizeCameras (:400-442)
        for cam_id, nres in camera_num_residuals.items():
            if nres <= 0:
                continue
            if cam_id in extra_const_cameras:
                cam_mask[cidx[cam_id]] = 0xFFFFFFFF
            else:
                cam_mask[cidx[cam_id]] = _cam_const_mask(rec.cameras[cam_id], options, setup, cam_id)
        # ParameterizePoints (:335-358)
        for pid, reg in reg_track.items():
            tl = rec.points3D[pid].track.length()
            mtl = min(options.min_track_length, tl) if options.min_track_length > 0 else tl
            if mtl > len(reg):
                point_const[pidx[pid]] = 1
        for pid in setup.constant_point3D_ids:
            if pid in pidx:
                point_const[pidx[pid]] = 1

    if not obs:
        import types
        return types.SimpleNamespace(n_obs=0), ir
    slab = PatchSlab()
    obs_patch = np.zeros(len(obs), np.int64)
    for k, (pid, image_id, p2D_idx) in enumerate(obs):
        name = feature_view.image_name(image_id)
        obs_patch[k] = slab.index(name, feature_view.get_feature_map(image_id), p2D_idx)
    blocks, corners, scales = slab.arrays()
    ir.slab_offsets = dict(slab._offset)     # image name -> first global patch index, in block order
    refs = None
    if references is not None:
        C_ = feature_view.channels
        refs = np.zeros((n_pts, C_))
        for pid in ir.point_ids:
            refs[pidx[pid]] = np.asarray(references[pid].descriptor, np.float64).reshape(-1)[:C_]
    prob = _capi.BAProblem(cam_model=cam_model, cam_params=cam_params, cam_const_mask=cam_mask, qvec=qvec, tvec=tvec,
                           img_cam=img_cam, pose_const=pose_const, tvec_const_mask=tmask, xyz=xyz,
                           point_const=point_const, obs_img=np.array([iidx[o[1]] for o in obs], np.int32),
                           obs_pt=np.array([pidx[o[0]] for o in obs], np.int64), patches=None, corner=corners,
                           scale=scales, refs=refs, obs_patch=obs_patch, patch_blocks=blocks)
    return prob, ir


def write_back(reconstruction, prob, ir):
    """the reference updates the Reconstruction in place through raw double* (feature_reference_bundle_optimizer.h:111-114)"""
    rows = getattr(ir, "_rows", None)
    if rows is not None:                      # array-backed reconstruction: three scatters
        rows_i, rows_c, rows_p = rows
        reconstruction.qvec[rows_i] = prob.qvec; reconstruction.tvec[rows_i] = prob.tvec; reconstruction.xyz[rows_p] = prob.xyz
        for k, r in enumerate(rows_c):
            n = len(reconstruction.cam_params[r])
            reconstruction.cam_params[r][:] = prob.cam_params[k, :n]
        return
    for k, i in enumerate(ir.image_ids):
        reconstruction.images[i].qvec[:] = prob.qvec[k]
        reconstruction.images[i].tvec[:] = prob.tvec[k]
    for k, c in enumerate(ir.camera_ids):
        n = len(reconstruction.cameras[c].params)
        reconstruction.cameras[c].params[:] = prob.cam_params[k, :n]
    for k, p in enumerate(ir.point_ids):
        reconstruction.points3D[p].xyz[:] = prob.xyz[k]


class ReferenceMap(dict):
    """Map_IdReference (features/bindings.cc): point3D id -> Reference.  `dense` remembers that the descriptors are rows of one
    [n_points, C] array (as the extractor produces them), so an optimizer that is handed the unmodified map copies one block
    instead of walking 50 000 Python objects."""
    dense = None

    def __setitem__(self, key, value):
        if self.dense is not None and key in self and value is not self[key]:
            self.dense = None              # edited by the caller: fall back to the per-entry walk
        super().__setitem__(key, value)


class ReferenceExtractor:
    """_bundle_adjustment.ReferenceExtractor(ReferenceConfig|dict, InterpolationConfig|dict).run(problem_labels,
    reconstruction, feature_set) -> {point3D_id: Reference}"""

    def __init__(self, config, interpolation_config):
        self.config = config if isinstance(config, ReferenceConfig) else ReferenceConfig(config)
        self.interp = interpolation_config if isinstance(interpolation_config, InterpolationConfig) else InterpolationConfig(interpolation_config)
        self.interp.validate_for_device()

    def run(self, problem_labels, reconstruction, feature_set):
        if hasattr(reconstruction, "point3D_id") and not hasattr(reconstruction, "points3D"):     # array-backed
            pids = np.asarray(reconstruction.point3D_id)
            labels = np.asarray(problem_labels)
            inside = pids < len(labels)
            ids = set(pids[inside][labels[pids[inside]] >= 0].tolist())
        else:
            ids = {p for p in reconstruction.points3D.keys() if p < len(problem_labels) and problem_labels[p] >= 0}
        fview = FeatureView(feature_set, reconstruction)
        prob, ir = build_problem(reconstruction, fview, None, None, None, for_references=ids)
        refs = ReferenceMap((p, Reference()) for p in ids)   # InitReferences
        if prob.n_obs == 0:
            return refs
        loss = self.config.loss
        if str(loss.get("name", "cauchy")).lower() not in _capi.LOSS_IDS:
            raise ValueError("unsupported loss")
        ic = _capi.default_interp(self.interp.l2_normalize, self.interp.use_float_simd)
        desc, src = _engine.refs_compute(prob, ic, _capi.LOSS_IDS[str(loss.get("name", "cauchy")).lower()],
                                         float(loss.get("params", [1.0])[0]), int(self.config.iters))
        src_img = ir.obs_image_id[np.maximum(src, 0)].tolist(); src_p2d = ir.obs_point2D_idx[np.maximum(src, 0)].tolist()
        valid = (src >= 0).tolist()
        for k, pid in enumerate(ir.point_ids):
            if valid[k]:
                refs[pid] = Reference((src_img[k], src_p2d[k]), desc[k:k + 1])      # [1, C] view of the extractor's output
        refs.dense = (np.asarray(ir.point_ids, np.int64), desc, np.asarray(valid))  # the optimizer takes the block as a whole
        if self.config.keep_observations:
            # refdata.observations / costs (reference_extractor.h:258-264): every observation's descriptor, in the
            # order of the problem IR (track order), and its squared distance to the chosen reference's robust mean
            # is not kept by the device path -> costs hold the distance to the chosen reference descriptor
            obs_desc = _engine.obs_descriptors(prob, ic)
            pidx = {pid: k for k, pid in enumerate(ir.point_ids)}
            for o, (image_id, p2D_idx, pid) in enumerate(ir.obs):
                r = refs[pid]
                r.observations.append(obs_desc[o].reshape(1, -1).copy())
                r.costs.append(float(((obs_desc[o] - desc[pidx[pid]]) ** 2).sum()))
        return refs


class _Summary(dict):
    __getattr__ = dict.get


class FeatureReferenceBundleOptimizer:
    """_bundle_adjustment.FeatureReferenceBundleOptimizer(options, setup, interpolation): `run(reconstruction,
    feature_view, references) -> bool` (mutates `reconstruction` in place) = `set_up(...)` + `solve_problem()`;
    `summary()`, `problem`, `reset()` as bound in bundle_adjustment/bindings.cc:36-51 (bundle_optimizer.h:114-245).
    `problem` is the flat problem IR handed to libpxr (the reference exposes its ceres::Problem there)."""
    _channels = (8, 16, 32, 64, 128, 256)
    _banner = "Start feature-reference bundle adjustment."

    def __init__(self, options, setup, interpolation_config):
        self.options = options if isinstance(options, BundleOptimizerOptions) else BundleOptimizerOptions(options)
        self.setup = setup
        self.interp = interpolation_config if isinstance(interpolation_config, InterpolationConfig) else InterpolationConfig(interpolation_config)
        self._summary, self._used = None, False
        self._prob = self._ir = self._reconstruction = None
        logger.info(self._banner)

    # ---- BundleOptimizer::SetUp (bundle_optimizer.h:139-165): residual blocks + parameterisation -> problem IR
    def set_up(self, reconstruction, feature_view, references=None):
        if reconstruction is None:
            raise ValueError("reconstruction cannot be NULL.")
        if self._used:
            raise ValueError("Cannot use the same BundleOptimizer multiple times")
        self._used = True
        self.interp.validate_for_device()
        if len(self.interp.nodes) != 1 or feature_view.channels not in self._channels:
            raise ValueError("Unsupported dimensions (CHANNELS,N_NODES).")
        self._prob, self._ir = build_problem(reconstruction, feature_view, self.setup, self.options, references)
        self._reconstruction = reconstruction
        return True

    @property
    def problem(self):
        return self._prob

    # ---- BundleOptimizer::SolveProblem (bundle_optimizer.h:172-245)
    def solve_problem(self):
        if self._prob is None:
            raise ValueError("set_up() has to run before solve_problem()")
        prob = self._prob
        if prob.n_obs == 0:
            return False   # problem_->NumResiduals() == 0 (:175-177)
        so = solver_options_from(self.options.loss, self.options.solver, _capi.default_ba_options(use_inner_iterations=0))
        ic = _capi.default_interp(self.interp.l2_normalize, self.interp.use_float_simd)
        need = _engine.ba_estimate_device_bytes(prob, so)     # the reference logs its RAM estimate here (:200-208)
        logger.info("Estimated device memory: %.3f GB (patches %.3f, problem state %.3f, reduced system %.3f).",
                    need["total"] / 1e9, need["patches"] / 1e9, need["state"] / 1e9, need["reduced_system"] / 1e9)
        callbacks = list(self.options.solver.get("callbacks") or [])
        if not callbacks:
            s = _engine.ba_run(prob, ic, so)
        else:
            s = self._solve_with_callbacks(prob, ic, so, callbacks)
        write_back(self._reconstruction, prob, self._ir)
        self._summary = _Summary(s, num_residuals_reduced=s["num_residuals"], total_time_in_seconds=s["total_time_s"])
        nres = max(1, s["num_residuals"])
        logger.info("BA Time: %.4gs, cost change: %.6g --> %.6g", s["total_time_s"],
                    np.sqrt(s["initial_cost"] / nres), np.sqrt(s["final_cost"] / nres))
        return True

    @staticmethod
    def _solve_with_callbacks(prob, ic, so, callbacks):
        """ceres::IterationCallback semantics (the reference injects its callbacks through `solver.callbacks`,
        util/misc.py:30-36): every callback sees each iteration record right after the iteration, starting with
        iteration 0, and may stop the solve by returning 1 / "SOLVER_ABORT" (-> USER_FAILURE) or 2 /
        "SOLVER_TERMINATE_SUCCESSFULLY" (-> USER_SUCCESS); None / 0 / "SOLVER_CONTINUE" go on.  The problem stays
        resident on the device between the iterations (pxr_ba_create + pxr_ba_iterate, one LM iteration per call)."""
        import time
        t0 = time.time()
        limit = int(so.max_num_iterations)
        h = _engine.BAHandle(prob, ic, so)
        try:
            seen, verdict = 0, 0
            s = h.iterate(0)                              # iteration 0: the evaluation at the start point
            while True:
                for it in s["iterations"][seen:]:
                    for cb in callbacks:
                        r = cb(it)
                        r = {"SOLVER_CONTINUE": 0, "SOLVER_ABORT": 1, "SOLVER_TERMINATE_SUCCESSFULLY": 2}.get(getattr(r, "name", r), r)
                        verdict = max(verdict, int(r or 0))
                grew = len(s["iterations"]) > seen
                seen = len(s["iterations"])
                if verdict or not grew or seen - 1 >= limit or s["termination_type"] != 1:
                    break
                s = h.iterate(1)
            h.read_params()
        finally:
            h.close()
        if verdict:
            s["termination_type"] = 3
            s["message"] = "User callback returned %s." % ("SOLVER_ABORT" if verdict == 1 else "SOLVER_TERMINATE_SUCCESSFULLY")
        s["total_time_s"] = time.time() - t0
        return s

    def run(self, reconstruction, feature_view, references=None):
        self.set_up(reconstruction, feature_view, references)
        return self.solve_problem()

    def reset(self):
        """BundleOptimizer::Reset: forget the problem, the optimizer can be set up again"""
        self._prob = self._ir = self._reconstruction = self._summary = None
        self._used = False

    def summary(self):
        return self._summary


class GeometricBundleOptimizer(FeatureReferenceBundleOptimizer):
    """_bundle_adjustment.GeometricBundleOptimizer(options, setup) (bindings.cc:155-162; geometric_bundle_optimizer.h:
    11-83): classic bundle adjustment of the reprojection error r = WorldToImage(X) - point2D.XY() in image pixels
    (colmap::BundleAdjustmentCostFunction).  `run(reconstruction)` = `set_up(reconstruction)` + `solve_problem()`;
    `summary()`, `problem`, `reset()` as for the featuremetric optimizer.  The problem is built by the same rules; images
    outside the setup keep their pose constant (ParameterizeImages), which is the geometric functor's constant-pose
    case (geometric_bundle_optimizer.h:43-45)."""
    _banner = "Start geometric bundle adjustment."

    def __init__(self, options, setup):
        super().__init__(options, setup, InterpolationConfig())

    def set_up(self, reconstruction, loss_function=None):
        """`loss_function`: an optional {"name", "params"} dict used instead of options.loss"""
        if reconstruction is None:
            raise ValueError("reconstruction cannot be NULL.")
        if self._used:
            raise ValueError("Cannot use the same BundleOptimizer multiple times")
        self._used = True
        if loss_function is not None:
            self.options.loss = dict(loss_function)
        self._prob, self._ir = build_problem(reconstruction, None, self.setup, self.options)
        self._reconstruction = reconstruction
        return True

    def run(self, reconstruction):   # noqa: D102
        self.set_up(reconstruction)
        return self.solve_problem()


def _loss_id_scale(loss):
    name = str(loss.get("name", "trivial")).lower()
    if name not in _capi.LOSS_IDS:
        raise ValueError("unsupported loss %r" % name)
    params = list(loss.get("params", []) or [])
    return _capi.LOSS_IDS[name], float(params[0]) if params else 1.0


def slice_dense_maps(feature_set, reconstruction, point3D_ids, cut_size):
    """Dense feature maps -> one `cut_size` x `cut_size` window per observation of `point3D_ids`, cut around the CURRENT
    reprojection: what the reference's cost-map extractor does with dense maps (costmap_extractor.h:207-222 `Slice(xy,
    dense_cut_size)`, :398-428; the corner rule is FeaturePatch::ToCorner, featurepatch.cc:324-336: truncate
    `uv - cut/2` towards zero, clamp to [0, size - cut]).  Sparse maps pass through.  The windows hold the same taps as the
    map they are cut from around the projection, edge clamping included, so references extracted from them equal the ones
    extracted from the dense map."""
    from ._features import DevicePatches, FeatureMap, FeatureSet
    from ..util.cameras import world_to_image
    cut = int(cut_size)
    out = FeatureSet(feature_set.channels, feature_set.dtype)
    ids = set(point3D_ids)
    for image in reconstruction.images.values():
        if not feature_set.has_fmap(image.name):
            continue
        fmap = feature_set.fmap(image.name)
        if fmap.is_sparse:
            out.emplace(image.name, fmap)
            continue
        sel = [k for k, p in enumerate(image.points2D) if p.has_point3D() and p.point3D_id in ids]
        if not sel:
            continue
        if isinstance(fmap.patches, DevicePatches):
            raise ValueError("cost maps from device-resident dense maps are not built (the windows are cut on the host)")
        k0 = fmap.local_index(0)
        dense = fmap.patches[k0]                                   # [H, W, C]
        height, width = dense.shape[:2]
        if height < cut or width < cut:
            raise ValueError("dense_cut_size %d exceeds the %dx%d feature map of %s" % (cut, width, height, image.name))
        cam = reconstruction.cameras[image.camera_id]
        xyz = np.array([reconstruction.points3D[image.points2D[k].point3D_id].xyz for k in sel])
        xy = world_to_image(cam.model_id, cam.params, image.qvec, image.tvec, xyz)
        uv = xy * fmap.scale - 0.5 - fmap.corners[k0]
        corners = np.trunc(uv - cut / 2.0).astype(np.int64)
        corners = np.minimum(np.maximum(corners, 0), np.array([width - cut, height - cut]))
        windows = np.stack([dense[c[1]:c[1] + cut, c[0]:c[0] + cut] for c in corners])
        out.emplace(image.name, FeatureMap(np.ascontiguousarray(windows), sel, (corners + fmap.corners[k0]).astype(np.int32),
                                           {"scale": fmap.scale, "is_sparse": True}))
    return out


class CostMapExtractor:
    """_bundle_adjustment.CostMapExtractor(CostMapConfig|dict, InterpolationConfig|dict)
    .run(problem_labels, reconstruction, feature_set, ref_extractor) -> (costmap FeatureSet, {point3D_id: Reference})
    (bindings.cc:20-26,179-184; costmap_extractor.h:93-228).  References and cost maps come out of ONE upload of the
    feature patches (pxr_costmaps_compute); the cost patches keep the source patches' corner / scale."""

    def __init__(self, config, interpolation_config):
        self.config = config if isinstance(config, CostMapConfig) else CostMapConfig(config)
        self.interp = interpolation_config if isinstance(interpolation_config, InterpolationConfig) else InterpolationConfig(interpolation_config)
        self.interp.validate_for_device()

    def run(self, problem_labels, reconstruction, feature_set, ref_extractor):
        if len(self.interp.nodes) != 1:
            raise ValueError("CostMap extract: n_nodes must be 1")       # THROW_CHECK_EQ(n_nodes, 1), :107
        if ref_extractor is None:
            raise ValueError("a ReferenceExtractor is required (the references are computed in the same pass)")
        from ._features import FeatureMap, FeatureSet
        ids = {p for p in reconstruction.points3D.keys() if p < len(problem_labels) and problem_labels[p] >= 0}
        if hasattr(feature_set, "fmap") and any(not feature_set.fmap(name).is_sparse for name in feature_set.keys()):
            # dense maps: a dense_cut_size window per observation around its reprojection (costmap_extractor.h:186-224)
            feature_set = slice_dense_maps(feature_set, reconstruction, ids, self.config.dense_cut_size)
        fview = FeatureView(feature_set, reconstruction)
        prob, ir = build_problem(reconstruction, fview, None, None, None, for_references=ids)
        refs = {p: Reference() for p in ids}
        out_channels = self.config.get_effective_channels()
        cost_fset = FeatureSet(out_channels, feature_set.dtype if hasattr(feature_set, "dtype") else None)
        if prob.n_obs == 0:
            return cost_fset, refs
        lt, ls = _loss_id_scale(self.config.loss)
        rlt, rls = _loss_id_scale(ref_extractor.config.loss)
        cfg = _capi.default_costmap_config(loss_type=lt, loss_scale=ls, as_gradientfield=int(bool(self.config.as_gradientfield)),
                                           compute_cross_derivative=int(bool(self.config.compute_cross_derivative)),
                                           apply_sqrt=int(bool(self.config.apply_sqrt)),
                                           upsampling_factor=float(self.config.upsampling_factor), compute_refs=1,
                                           ref_loss_type=rlt, ref_loss_scale=rls, ref_iters=int(ref_extractor.config.iters))
        ic = _capi.default_interp(self.interp.l2_normalize, self.interp.use_float_simd)
        if any(not (feature_set.fmap(name) if hasattr(feature_set, "fmap") else feature_set[name]).is_sparse
               for name in ir.slab_offsets):
            raise ValueError("cost maps need sparse feature maps or a FeatureSet of dense ones (dense_cut_size slicing)")
        out = _engine.costmaps_compute(prob, ic, cfg)
        for k, pid in enumerate(ir.point_ids):
            if out["src_obs"][k] < 0:
                continue
            image_id, p2D_idx, _ = ir.obs[int(out["src_obs"][k])]
            refs[pid] = Reference((image_id, p2D_idx), out["refs"][k].reshape(1, -1).copy())
        cm = out["costmaps"]
        for name, off in ir.slab_offsets.items():
            fmap = feature_set.fmap(name) if hasattr(feature_set, "fmap") else feature_set[name]
            cost_fset.emplace(name, FeatureMap(cm[off:off + fmap.size()], fmap.point2D_ids, fmap.corners,
                                               {"scale": fmap.scale, "is_sparse": True}))
        return cost_fset, refs


class CostMapBundleOptimizer(FeatureReferenceBundleOptimizer):
    """_bundle_adjustment.CostMapBundleOptimizer(options, setup, interpolation).run(reconstruction, costmap_view)
    (bindings.cc:143-160; costmap_bundle_optimizer.h:60-132): the residual of an observation is the interpolated
    cost-map vector itself (no reference descriptor, no L2 normalisation)."""
    _channels = (1, 3, 4)
    _banner = "Start cost-map bundle adjustment."

    def set_up(self, reconstruction, feature_view):   # noqa: D102
        return super().set_up(reconstruction, feature_view, None)

    def run(self, reconstruction, feature_view):   # noqa: D102
        self.set_up(reconstruction, feature_view)
        return self.solve_problem()
