"""Mirror of `pixsfm._pixsfm._localization` (pixsfm/localization/bindings.cc; src/single_query_keypoint_optimizer.h,
single_query_bundle_optimizer.h, query_refinement_options.h, nearest_references.h): query keypoint adjustment and
query bundle adjustment against fixed reference descriptors.  Same kernels as KA / BA:
  * QKA  = pxr_ka_run in query mode (every edge = keypoint vs fixed descriptor; block-diagonal normal equations,
           all keypoints of the query in one trust region like the reference's single ceres::Problem)
  * QBA  = pxr_ba_run with one free image, every 3D point constant (one IR "point" per (correspondence, reference))
"""
import ctypes as C

import numpy as np

from .. import logger
from . import _capi, _engine
from ._base import InterpolationConfig
from ._bundle_adjustment import _DictOptions, _Summary, solver_options_from
from ._features import DevicePatches, Reference


class QueryKeypointOptimizerOptions(_DictOptions):
    """query_refinement_options.h:54-98 (C++ defaults; the Python layer passes parameter_tolerance 1e-5, bound 4)"""
    _defaults = dict(print_summary=True, bound=-1.0, loss=lambda: {"name": "trivial", "params": []},
                     solver=lambda: {"function_tolerance": 0.0, "gradient_tolerance": 0.0, "parameter_tolerance": 1.0e-4,
                                     "max_num_iterations": 100, "max_num_consecutive_invalid_steps": 10})


class QueryBundleOptimizerOptions(_DictOptions):
    """query_refinement_options.h:7-52"""
    _defaults = dict(print_summary=True, refine_focal_length=False, refine_principal_point=False, refine_extra_params=False,
                     loss=lambda: {"name": "cauchy", "params": [0.25]},
                     solver=lambda: {"function_tolerance": 0.0, "gradient_tolerance": 0.0, "parameter_tolerance": 1.0e-5,
                                     "max_num_iterations": 100, "max_linear_solver_iterations": 200,
                                     "max_num_consecutive_invalid_steps": 10, "max_consecutive_nonmonotonic_steps": 10})


def _host_patches(fmap):
    if isinstance(fmap.patches, DevicePatches):
        raise ValueError("query refinement takes host (numpy) feature maps")
    return fmap.patches


def _descriptors_of(ref, channels):
    """the reference descriptors one correspondence is compared with (single_query_*_optimizer.h RunQuery overloads):
    ndarray -> itself; list of ndarrays -> all of them; Reference -> its observations if kept, else its descriptor"""
    if isinstance(ref, Reference):
        obs = getattr(ref, "observations", None)
        if obs:
            return [np.asarray(o, np.float64).reshape(-1)[:channels] for o in obs]
        return [np.asarray(ref.descriptor, np.float64).reshape(-1)[:channels]]
    if isinstance(ref, np.ndarray):
        return [np.asarray(ref, np.float64).reshape(-1)[:channels]]
    return [np.asarray(r, np.float64).reshape(-1)[:channels] for r in ref]


def interpolate_descriptors(fmap, patch_idxs, xys, interpolation_config=None):
    """PatchInterpolator.interpolate_nodes for one node, batched: descriptor of fmap's patch patch_idxs[i] at xys[i]"""
    interp = interpolation_config if isinstance(interpolation_config, InterpolationConfig) else InterpolationConfig(interpolation_config or {})
    interp.validate_for_device()
    patches = _host_patches(fmap)
    ctx = _capi.default_context()
    xys = np.ascontiguousarray(xys, np.float64).reshape(-1, 2)
    item_patch = np.array([fmap.local_index(i) for i in patch_idxs], np.int64)
    scales = np.ascontiguousarray(np.tile(fmap.scale, (fmap.size(), 1)), np.float64)
    out = np.zeros((len(xys), fmap.channels))
    ic = _capi.default_interp(interp.l2_normalize, interp.use_float_simd)
    _capi.check(ctx.lib.pxr_interpolate_descriptors(
        ctx.handle, patches.ctypes.data_as(C.c_void_p), C.c_int64(fmap.size()), _capi.DTYPE_IDS[patches.dtype],
        int(patches.shape[1]), int(patches.shape[2]), int(patches.shape[3]), fmap.corners.ctypes.data_as(C.c_void_p),
        scales.ctypes.data_as(C.c_void_p), C.c_double(1.0), C.c_int64(len(xys)), item_patch.ctypes.data_as(C.c_void_p),
        xys.ctypes.data_as(C.c_void_p), C.byref(ic), out.ctypes.data_as(C.c_void_p)))
    return out


def find_nearest_references(query_fmap, references, keypoints, point3D_ids, interpolation_config, patch_idxs=None):
    """localization/src/nearest_references.h:20-53: per correspondence the stored observation descriptor of the 3D
    point that is closest (squared L2) to the query descriptor interpolated at the keypoint; first minimum wins."""
    keypoints = np.asarray(keypoints, np.float64).reshape(-1, 2)
    idxs = list(range(len(keypoints))) if patch_idxs is None else list(patch_idxs)
    q = interpolate_descriptors(query_fmap, idxs, keypoints, interpolation_config)
    out = []
    for i, pid in enumerate(point3D_ids):
        ref = references[pid]
        obs = getattr(ref, "observations", None)
        if not obs:
            raise ValueError("Missing observations in references. Extract references with option keep_observations=True.")
        obs = [np.asarray(o, np.float64).reshape(-1) for o in obs]
        d = [float(((o - q[i]) ** 2).sum()) for o in obs]
        out.append(obs[int(np.argmin(d))].reshape(1, -1).copy())
    return out


_MISSING_OBS = "Missing observations in references. Extract references with option keep_observations=True."


def observation_table(references, point_ids):
    """the stored observation descriptors of the given 3D points back to back: (rows [n, C] float64, {point id: (first
    row, number of rows)}).  Raises find_nearest_references' error for a point without observations."""
    rows, where, n = [], {}, 0
    for pid in point_ids:
        if pid in where:
            continue
        obs = getattr(references[pid], "observations", None)
        if not obs:
            raise ValueError(_MISSING_OBS)
        where[pid] = (n, len(obs))
        n += len(obs)
        rows.extend(np.asarray(o, np.float64).reshape(-1) for o in obs)
    return (np.array(rows) if rows else np.zeros((0, 0))), where


def find_nearest_references_batch(items, interpolation_config, _table=None):
    """find_nearest_references for many queries in one pxr_query_match_run.  items: (query_fmap, references, keypoints,
    point3D_ids[, patch_idxs]) -> per query the list find_nearest_references returns.  The candidates of a
    correspondence are its 3D point's stored observations; `_table` = (rows, {point id: (first row, count)}) passes a
    table already packed (rows may be device memory) instead of packing the references again."""
    interp = interpolation_config if isinstance(interpolation_config, InterpolationConfig) else InterpolationConfig(interpolation_config or {})
    interp.validate_for_device()
    items = list(items)
    blocks, corners, scales, iq, ip, xys, pids = [], [], [], [], [], [], []
    for k, it in enumerate(items):
        fmap, references, keypoints, point3D_ids = it[:4]
        patch_idxs = it[4] if len(it) > 4 else None
        keypoints = np.asarray(keypoints, np.float64).reshape(-1, 2)
        idxs = list(range(len(keypoints))) if patch_idxs is None else list(patch_idxs)
        for pid in point3D_ids:
            if (pid not in _table[1]) if _table is not None else not getattr(references[pid], "observations", None):
                raise ValueError("query %d: %s" % (k, _MISSING_OBS))
        blocks.append(fmap.patches)
        corners.append(np.asarray(fmap.corners, np.int32).reshape(-1, 2))
        scales.append(np.tile(fmap.scale, (fmap.size(), 1)))
        for i, pid in enumerate(point3D_ids):
            iq.append(k); ip.append(fmap.local_index(idxs[i])); xys.append(keypoints[i]); pids.append(pid)
    if _table is None:
        refs_of = {}
        for k, it in enumerate(items):
            for pid in it[3]:
                refs_of.setdefault(pid, it[1][pid])
        rows, where = observation_table(refs_of, list(refs_of)) if refs_of else (np.zeros((0, 0)), {})
        rows = np.asarray(rows, np.float64)
    else:
        rows, where = _table
    cb = np.array([where[p][0] for p in pids], np.int64)
    ce = np.array([where[p][0] + where[p][1] for p in pids], np.int64)
    out = [[] for _ in items]
    if not pids:
        return out
    ic = _capi.default_interp(interp.l2_normalize, interp.use_float_simd)
    best, _, _ = _engine.query_match_run(blocks, np.concatenate(corners), np.concatenate(scales), iq, ip, xys, cb, ce, rows, ic)
    for k, pid, b, first in zip(iq, pids, best, cb):
        if b < 0:          # an empty candidate range: the point has no stored observations
            raise ValueError("query %d: %s" % (k, _MISSING_OBS))
        obs = items[k][1][pid].observations
        out[k].append(np.asarray(obs[int(b - first)], np.float64).reshape(1, -1).copy())
    return out


def feature_inliers_batch(items, interpolation_config, thresh):
    """find_feature_inliers (localization/main.py) for many queries in one pxr_query_match_run.  items: (points2D, fmap,
    references, point2D_idxs or None) -> per query one bool per correspondence: a correspondence whose reference is one
    ndarray is an inlier when the interpolated descriptor lies within `thresh` (L2) of it; others always are"""
    items = list(items)
    if thresh < 0.0:
        return [[True] * len(it[0]) for it in items]
    interp = interpolation_config if isinstance(interpolation_config, InterpolationConfig) else InterpolationConfig(interpolation_config or {})
    interp.validate_for_device()
    blocks, corners, scales, iq, ip, xys, cand, cb, ce, tested = [], [], [], [], [], [], [], [], [], []
    for k, (p2Ds, fmap, references, idxs) in enumerate(items):
        idxs = list(range(len(p2Ds)) if idxs is None else idxs)
        blocks.append(fmap.patches)
        corners.append(np.asarray(fmap.corners, np.int32).reshape(-1, 2))
        scales.append(np.tile(fmap.scale, (fmap.size(), 1)))
        for i, (xy, ref) in enumerate(zip(np.asarray(p2Ds, np.float64).reshape(-1, 2), references)):
            if not isinstance(ref, np.ndarray):
                continue
            iq.append(k); ip.append(fmap.local_index(idxs[i]))
            xys.append(xy); cb.append(len(cand)); ce.append(len(cand) + 1); cand.append(np.asarray(ref, np.float64).reshape(-1))
            tested.append((k, i))
    out = [[True] * len(it[0]) for it in items]
    if not tested:
        return out
    ic = _capi.default_interp(interp.l2_normalize, interp.use_float_simd)
    _, dmin, _ = _engine.query_match_run(blocks, np.concatenate(corners), np.concatenate(scales), iq, ip, xys, cb, ce,
                                         np.array(cand), ic)
    for (k, i), d in zip(tested, dmin):
        out[k][i] = bool(np.sqrt(d) <= thresh)
    return out


class QueryKeypointOptimizer:
    """_localization.QueryKeypointOptimizer(options, interpolation).run(keypoints, fmap, references, patch_idxs=None,
    inliers=None) -> bool; `keypoints` ([N,2] float64) is refined IN PLACE."""

    def __init__(self, options, interpolation_config):
        self.options = options if isinstance(options, QueryKeypointOptimizerOptions) else QueryKeypointOptimizerOptions(options)
        self.interp = interpolation_config if isinstance(interpolation_config, InterpolationConfig) else InterpolationConfig(interpolation_config)
        self._summary = None

    def build_problem(self, keypoints, fmap, references, patch_idxs=None, inliers=None):
        """-> (KAProblem in query mode | None, indices of the keypoints it holds)"""
        if keypoints.dtype != np.float64 or keypoints.ndim != 2 or keypoints.shape[1] != 2:
            raise ValueError("keypoints must be a [N,2] float64 array")
        n = len(keypoints)
        if len(references) != n:
            raise ValueError("references.size() != keypoints.rows()")       # THROW_CHECK_EQ
        if patch_idxs is not None and len(patch_idxs) != n:
            raise ValueError("patch_idxs.size() != keypoints.rows()")
        self.interp.validate_for_device()
        if len(self.interp.nodes) != 1 or fmap.channels not in (8, 16, 32, 64, 128):
            raise ValueError("Unsupported dimensions (CHANNELS,N_NODES).")
        patches = _host_patches(fmap)
        es, ed, refs, used = [], [], [], []
        for i in range(n):
            if inliers is not None and not inliers[i]:
                continue
            descs = _descriptors_of(references[i], fmap.channels)
            for dsc in descs:
                es.append(len(used)); ed.append(len(refs)); refs.append(dsc)
            if descs:
                used.append(i)
        if not es:
            return None, used                                               # problem->NumResiduals() == 0
        kp_patch = np.array([fmap.local_index(i if patch_idxs is None else patch_idxs[i]) for i in used], np.int64)
        kps = np.ascontiguousarray(keypoints[used])
        prob = _capi.KAProblem(keypoints=kps, kp_const=np.zeros(len(used), np.uint8), edge_src=es, edge_dst=ed,
                               edge_weight=None, edge_problem=np.zeros(len(es), np.int32), n_problems=1, patches=patches,
                               corner=fmap.corners, scale=np.tile(fmap.scale, (fmap.size(), 1)), kp_patch=kp_patch,
                               bound=float(self.options.bound), patches_are_sparse=fmap.is_sparse, ref_desc=np.array(refs))
        return prob, used

    def solver_options(self):
        return solver_options_from(self.options.loss, self.options.solver, _capi.default_ka_options())

    def run(self, keypoints, fmap, references, patch_idxs=None, inliers=None):
        prob, used = self.build_problem(keypoints, fmap, references, patch_idxs, inliers)
        if prob is None:
            return False
        so = self.solver_options()
        ic = _capi.default_interp(self.interp.l2_normalize, self.interp.use_float_simd)
        s = _engine.ka_run(prob, ic, so)
        keypoints[used] = prob.keypoints
        nres = max(1, len(prob.edge_src) * fmap.channels)
        self._summary = _Summary(s, num_residuals_reduced=nres)
        logger.info("QKA Time: %.4gs, cost change: %.6g --> %.6g", s["total_time_s"], np.sqrt(s["initial_cost"] / nres),
                    np.sqrt(s["final_cost"] / nres))
        return True

    def summary(self):
        return self._summary

    # ---- batched: many queries in one pxr_qka_run
    def pack_batch(self, queries, max_wave_bytes=0.0):
        """the problems build_problem makes for every query of `queries` (argument tuples as run takes them:
        (keypoints, fmap, references[, patch_idxs[, inliers]])) as one _capi.QKABatch, and per query the indices of
        the keypoints it holds.  Feature maps may hold host (numpy) or device patches (DevicePatches)."""
        self.interp.validate_for_device()
        kps, kp_begin, kp_patch, desc_begin, descs, blocks, corners, scales, sparse, used_of = ([] for _ in range(10))
        kp_begin.append(0); desc_begin.append(0)
        channels = dtype = None
        for k, args in enumerate(queries):
            keypoints, fmap, references = args[:3]
            patch_idxs = args[3] if len(args) > 3 else None
            inliers = args[4] if len(args) > 4 else None
            try:
                if not isinstance(keypoints, np.ndarray) or keypoints.dtype != np.float64 or keypoints.ndim != 2 or \
                        keypoints.shape[1] != 2:
                    raise ValueError("keypoints must be a [N,2] float64 array")
                n = len(keypoints)
                if len(references) != n:
                    raise ValueError("references.size() != keypoints.rows()")
                if patch_idxs is not None and len(patch_idxs) != n:
                    raise ValueError("patch_idxs.size() != keypoints.rows()")
                if len(self.interp.nodes) != 1 or fmap.channels not in (8, 16, 32, 64, 128):
                    raise ValueError("Unsupported dimensions (CHANNELS,N_NODES).")
                if channels is not None and fmap.channels != channels:
                    raise ValueError("every query of a batch must have the same channel count")
                dt = np.dtype(getattr(fmap.patches, "dtype"))
                if dtype is not None and dt != dtype:
                    raise ValueError("every query of a batch must have the same patch dtype")
            except ValueError as e:
                raise ValueError("query %d: %s" % (k, e)) from None
            channels, dtype = fmap.channels, dt
            used = []
            for i in range(n):
                if inliers is not None and not inliers[i]:
                    continue
                ds = _descriptors_of(references[i], fmap.channels)
                if not ds:
                    continue
                used.append(i)
                kps.append(keypoints[i]); kp_patch.append(fmap.local_index(i if patch_idxs is None else patch_idxs[i]))
                descs.extend(ds); desc_begin.append(len(descs))
            used_of.append(used)
            kp_begin.append(len(kps))
            blocks.append(fmap.patches)
            corners.append(np.asarray(fmap.corners, np.int32).reshape(-1, 2))
            scales.append(np.tile(fmap.scale, (fmap.size(), 1)))
            sparse.append(bool(fmap.is_sparse))
        batch = _capi.QKABatch(np.array(kps).reshape(-1, 2), kp_begin, kp_patch, desc_begin,
                               np.array(descs) if descs else np.zeros((0, channels or 8)), blocks,
                               np.concatenate(corners) if corners else np.zeros((0, 2), np.int32),
                               np.concatenate(scales) if scales else np.zeros((0, 2)), sparse,
                               bound=float(self.options.bound), max_wave_bytes=max_wave_bytes)
        return batch, used_of

    def run_batch(self, queries, max_wave_bytes=0.0):
        """run() for every query of `queries` (argument tuples (keypoints, fmap, references[, patch_idxs[, inliers]]))
        in one pxr_qka_run: each query's keypoints are refined IN PLACE.  -> one bool per query, what run() returns
        (False: no residual block).  summaries() gives each query's summary; its total_time_s is that of the whole
        batch.  A query whose initial cost is not finite gets what run() gives it: its keypoints as the solver leaves
        them, True, and a summary with that cost (a warning names the query)."""
        queries = list(queries)
        batch, used_of = self.pack_batch(queries, max_wave_bytes)
        so = self.solver_options()
        ic = _capi.default_interp(self.interp.l2_normalize, self.interp.use_float_simd)
        tot = _engine.ka_run(batch, ic, so)
        ch = batch.channels
        self._summaries, ok = [], []
        for k, (args, r, used) in enumerate(zip(queries, batch.results, used_of)):
            if r["num_residual_blocks"] == 0:
                self._summaries.append(None); ok.append(False)
                continue
            if r["status"] != _capi.PXR_OK:
                logger.warning("QKA query %d: initial cost is not finite", k)
            kb, ke = int(batch.kp_begin[k]), int(batch.kp_begin[k + 1])
            args[0][used] = batch.keypoints[kb:ke]
            nres = max(1, r["num_residual_blocks"] * ch)
            s = dict(r, num_residuals=r["num_residual_blocks"] * ch, num_inner_iteration_steps=0,
                     total_time_s=tot["total_time_s"], solve_time_s=tot["solve_time_s"], iterations=[])
            self._summaries.append(_Summary(s, num_residuals_reduced=nres))
            ok.append(True)
        logger.info("QKA Time: %.4gs for %d queries", tot["total_time_s"], len(queries))
        return ok

    def summaries(self):
        """per-query summaries of the last run_batch (None for a query that was not solved)"""
        return getattr(self, "_summaries", [])


class QueryBundleOptimizer:
    """_localization.QueryBundleOptimizer(options, interpolation).run(qvec, tvec, camera, points3D, fmap, references,
    inliers=None, patch_idxs=None) -> bool; qvec / tvec / camera.params are refined IN PLACE."""

    def __init__(self, options, interpolation_config):
        self.options = options if isinstance(options, QueryBundleOptimizerOptions) else QueryBundleOptimizerOptions(options)
        self.interp = interpolation_config if isinstance(interpolation_config, InterpolationConfig) else InterpolationConfig(interpolation_config)
        self._summary = None

    def build_problem(self, qvec, tvec, camera, points3D, fmap, references, inliers=None, patch_idxs=None):
        n = len(points3D)
        if len(references) != n:
            raise ValueError("references.size() != points3D.size()")
        if patch_idxs is not None and len(patch_idxs) != n:
            raise ValueError("patch_idxs.size() != points3D.size()")
        self.interp.validate_for_device()
        if len(self.interp.nodes) != 1 or fmap.channels not in (8, 16, 32, 64, 128, 256):
            raise ValueError("Unsupported dimensions (CHANNELS,N_NODES).")
        patches = _host_patches(fmap)
        xyz, refs, obs_patch = [], [], []
        for i in range(n):
            if inliers is not None and not inliers[i]:
                continue
            pi = fmap.local_index(i if patch_idxs is None else patch_idxs[i])
            for dsc in _descriptors_of(references[i], fmap.channels):   # one residual block per reference descriptor
                xyz.append(np.asarray(points3D[i], np.float64).reshape(3)); refs.append(dsc); obs_patch.append(pi)
        if not xyz:
            return None
        m = len(xyz)
        model = int(camera.model_id)
        focal, pp, extra = _capi.CAMERA_PARAM_GROUPS[model]
        o = self.options
        if not (o.refine_focal_length or o.refine_principal_point or o.refine_extra_params):
            mask = 0xFFFFFFFF                                            # ParameterizeQuery: constant camera
        else:
            mask = (0 if o.refine_focal_length else focal) | (0 if o.refine_principal_point else pp) | (0 if o.refine_extra_params else extra)
        prob = _capi.BAProblem(cam_model=[model], cam_params=[np.asarray(camera.params, np.float64)], cam_const_mask=[mask],
                               qvec=np.asarray(qvec, np.float64).reshape(1, 4), tvec=np.asarray(tvec, np.float64).reshape(1, 3),
                               img_cam=[0], pose_const=[0], tvec_const_mask=[0], xyz=np.array(xyz), point_const=np.ones(m, np.uint8),
                               obs_img=np.zeros(m, np.int32), obs_pt=np.arange(m, dtype=np.int64), patches=patches,
                               corner=fmap.corners, scale=np.tile(fmap.scale, (fmap.size(), 1)), refs=np.array(refs),
                               obs_patch=np.array(obs_patch, np.int64))
        return prob

    def solver_options(self):
        return solver_options_from(self.options.loss, self.options.solver,
                                   _capi.default_ba_options(use_inner_iterations=0, parameter_tolerance=1e-5))

    def run(self, qvec, tvec, camera, points3D, fmap, references, inliers=None, patch_idxs=None):
        prob = self.build_problem(qvec, tvec, camera, points3D, fmap, references, inliers, patch_idxs)
        if prob is None:
            return False
        so = self.solver_options()
        ic = _capi.default_interp(self.interp.l2_normalize, self.interp.use_float_simd)
        s = _engine.ba_run(prob, ic, so)
        np.asarray(qvec).reshape(-1)[:] = prob.qvec[0]
        np.asarray(tvec).reshape(-1)[:] = prob.tvec[0]
        camera.params[:] = prob.cam_params[0, :len(camera.params)]
        nres = max(1, s["num_residuals"])
        self._summary = _Summary(s, num_residuals_reduced=nres)
        logger.info("QBA Time: %.4gs, cost change: %.6g --> %.6g", s["total_time_s"], np.sqrt(s["initial_cost"] / nres),
                    np.sqrt(s["final_cost"] / nres))
        return True

    def summary(self):
        return self._summary

    # ---- batched: many queries in one pxr_qba_run
    def pack_batch(self, queries, max_wave_bytes=0.0):
        """the per-query arrays build_problem makes, concatenated into one _capi.QBABatch.  `queries` is a list of the
        argument tuples run takes, (qvec, tvec, camera, points3D, fmap, references[, inliers[, patch_idxs]]); feature
        maps may hold host (numpy) or device patches (DevicePatches, read in place)."""
        self.interp.validate_for_device()
        model, params, masks, qv, tv, begin, xyz, refs, obs_patch, blocks, corners, scales = ([] for _ in range(12))
        begin.append(0)
        channels = None
        o = self.options
        for args in queries:
            qvec, tvec, camera, points3D, fmap, references = args[:6]
            inliers = args[6] if len(args) > 6 else None
            patch_idxs = args[7] if len(args) > 7 else None
            n = len(points3D)
            if len(references) != n:
                raise ValueError("references.size() != points3D.size()")
            if patch_idxs is not None and len(patch_idxs) != n:
                raise ValueError("patch_idxs.size() != points3D.size()")
            if len(self.interp.nodes) != 1 or fmap.channels not in (8, 16, 32, 64, 128, 256):
                raise ValueError("Unsupported dimensions (CHANNELS,N_NODES).")
            if channels is not None and fmap.channels != channels:
                raise ValueError("every query of a batch must have the same channel count")
            channels = fmap.channels
            for i in range(n):
                if inliers is not None and not inliers[i]:
                    continue
                pi = fmap.local_index(i if patch_idxs is None else patch_idxs[i])
                for dsc in _descriptors_of(references[i], fmap.channels):   # one residual block per reference descriptor
                    xyz.append(np.asarray(points3D[i], np.float64).reshape(3)); refs.append(dsc); obs_patch.append(pi)
            begin.append(len(xyz))
            m = int(camera.model_id)
            focal, pp, extra = _capi.CAMERA_PARAM_GROUPS[m]
            if not (o.refine_focal_length or o.refine_principal_point or o.refine_extra_params):
                masks.append(0xFFFFFFFF)
            else:
                masks.append((0 if o.refine_focal_length else focal) | (0 if o.refine_principal_point else pp) |
                             (0 if o.refine_extra_params else extra))
            model.append(m); params.append(np.asarray(camera.params, np.float64))
            qv.append(np.asarray(qvec, np.float64).reshape(4)); tv.append(np.asarray(tvec, np.float64).reshape(3))
            blocks.append(fmap.patches)
            corners.append(np.asarray(fmap.corners, np.int32).reshape(-1, 2))
            scales.append(np.tile(fmap.scale, (fmap.size(), 1)))
        return _capi.QBABatch(model, params, masks, np.array(qv).reshape(-1, 4), np.array(tv).reshape(-1, 3), begin,
                              np.array(xyz).reshape(-1, 3), obs_patch, np.array(refs) if refs else None, blocks,
                              np.concatenate(corners) if corners else np.zeros((0, 2), np.int32),
                              np.concatenate(scales) if scales else np.zeros((0, 2)), max_wave_bytes=max_wave_bytes)

    def run_batch(self, queries, max_wave_bytes=0.0):
        """run() for every query of `queries` (argument tuples as pack_batch takes them) in one pxr_qba_run: each
        query's qvec / tvec / camera.params are refined IN PLACE.  -> one bool per query (False: no residual block).
        summaries() gives each query's summary; its total_time_s and solve_time_s are those of the whole batch (the
        queries are solved together), which is also what the one "QBA Time" log line per batch reports.  A query whose
        initial cost is not finite raises the error run() would raise, naming the query, after every other query has
        been written back."""
        queries = list(queries)
        batch = self.pack_batch(queries, max_wave_bytes)
        so = self.solver_options()
        ic = _capi.default_interp(self.interp.l2_normalize, self.interp.use_float_simd)
        res, tot = _engine.qba_run(batch, ic, so, capacity=max(1, int(so.max_num_iterations) + 1))
        self._summaries, ok, failed = [], [], []
        for k, (args, r) in enumerate(zip(queries, res)):
            if r["num_residual_blocks"] == 0 or r["status"] != _capi.PXR_OK:
                self._summaries.append(None); ok.append(False)
                if r["num_residual_blocks"]:
                    failed.append(k)
                continue
            qvec, tvec, camera = args[:3]
            np.asarray(qvec).reshape(-1)[:] = batch.qvec[k]
            np.asarray(tvec).reshape(-1)[:] = batch.tvec[k]
            camera.params[:] = batch.cam_params[k, :len(camera.params)]
            nres = max(1, r["num_residual_blocks"] * batch.channels)
            s = dict(initial_cost=r["initial_cost"], final_cost=r["final_cost"],
                     num_residual_blocks=r["num_residual_blocks"], num_residuals=r["num_residual_blocks"] * batch.channels,
                     num_successful_steps=r["num_successful_steps"], num_unsuccessful_steps=r["num_unsuccessful_steps"],
                     num_inner_iteration_steps=0, termination_type=r["termination_type"],
                     total_time_s=tot["total_time_s"], solve_time_s=tot["solve_time_s"], num_iterations=r["num_iterations"],
                     block_evaluations=r["block_evaluations"], iterations=r.get("iterations", []))
            self._summaries.append(_Summary(s, num_residuals_reduced=nres))
            logger.info("QBA query %d: cost change: %.6g --> %.6g", k, np.sqrt(r["initial_cost"] / nres),
                        np.sqrt(r["final_cost"] / nres))
            ok.append(True)
        logger.info("QBA Time: %.4gs for %d queries in %d waves", tot["total_time_s"], len(queries), tot["n_waves"])
        if failed:
            raise _capi.PxrError("pxr status %d: query %d: initial cost is not finite" % (_capi.PXR_ERR_NUMERIC, failed[0]))
        return ok

    def summaries(self):
        """per-query summaries of the last run_batch (None for a query that was not solved)"""
        return getattr(self, "_summaries", [])


# ---- absolute pose estimation (pycolmap 0.4 absolute_pose_estimation on pxr_pnp_run)
# pycolmap 0.4's option names and defaults (AbsolutePoseEstimationOptions / RANSACOptions, AbsolutePoseRefinementOptions).
# pycolmap is not a dependency of this package, so the defaults are restated from its 0.4 sources as best known and are
# not checked against an installed copy.
ABSOLUTE_POSE_ESTIMATION_DEFAULTS = dict(
    estimate_focal_length=False, num_focal_length_samples=30, min_focal_length_ratio=0.2, max_focal_length_ratio=5.0,
    ransac=dict(max_error=12.0, min_inlier_ratio=0.01, min_num_trials=1000, max_num_trials=100000, confidence=0.9999,
                dyn_num_trials_multiplier=3.0))
ABSOLUTE_POSE_REFINEMENT_DEFAULTS = dict(gradient_tolerance=1.0, max_num_iterations=100, loss_function_scale=1.0,
                                         refine_focal_length=False, refine_extra_params=False, print_summary=False)


def _merge_options(defaults, given, where):
    out = {k: (dict(v) if isinstance(v, dict) else v) for k, v in defaults.items()}
    for k, v in (given or {}).items():
        if k not in defaults:
            raise ValueError("%s: unknown option '%s'" % (where, k))
        if isinstance(defaults[k], dict):
            out[k] = _merge_options(defaults[k], v, where + "." + k)
        else:
            out[k] = v
    return out


def pnp_options(estimation_options=None, refinement_options=None):
    """pycolmap-style nested option dicts (unknown keys rejected) merged over the defaults -> _capi.PnPOptions"""
    est = _merge_options(ABSOLUTE_POSE_ESTIMATION_DEFAULTS, estimation_options, "estimation_options")
    ref = _merge_options(ABSOLUTE_POSE_REFINEMENT_DEFAULTS, refinement_options, "refinement_options")
    if est["estimate_focal_length"]:
        raise ValueError("estimate_focal_length=True is not supported: the built-in absolute pose estimator estimates the "
                         "pose only (refinement_options refine_focal_length refines the focal length after RANSAC)")
    r = est["ransac"]
    return _capi.default_pnp_options(
        max_error=float(r["max_error"]), min_inlier_ratio=float(r["min_inlier_ratio"]),
        min_num_trials=int(r["min_num_trials"]), max_num_trials=int(r["max_num_trials"]), confidence=float(r["confidence"]),
        dyn_num_trials_multiplier=float(r["dyn_num_trials_multiplier"]), estimate_focal_length=0, refine=1,
        gradient_tolerance=float(ref["gradient_tolerance"]), max_num_iterations=int(ref["max_num_iterations"]),
        loss_function_scale=float(ref["loss_function_scale"]), refine_focal_length=int(bool(ref["refine_focal_length"])),
        refine_extra_params=int(bool(ref["refine_extra_params"])))


def absolute_pose_estimation_batch(queries, estimation_options=None, refinement_options=None, ctx=None):
    """absolute_pose_estimation for every entry of `queries`, tuples (points2D [N,2], points3D [N,3], camera[, seed]), in
    one pxr_pnp_run.  A query's result depends only on its own inputs and seed (default 0), never on the batch.  Returns
    one pycolmap 0.4 dict per query: success, qvec, tvec, num_inliers, inliers (list of bool), or {"success": False}."""
    opt = pnp_options(estimation_options, refinement_options)
    queries = [tuple(q) for q in queries]
    if not queries:
        return []
    p2, p3, begin, models, params, seeds = [], [], [0], [], [], []
    for q in queries:
        a2 = np.asarray(q[0], np.float64).reshape(-1, 2)
        a3 = np.asarray([np.asarray(getattr(p, "xyz", p), np.float64) for p in q[1]], np.float64).reshape(-1, 3)
        if len(a2) != len(a3):
            raise ValueError("points2D and points3D must have the same length")
        cam = q[2]
        cp = np.zeros(_capi.PXR_MAX_CAM_PARAMS)
        cp[:len(cam.params)] = np.asarray(cam.params, np.float64)
        p2.append(a2); p3.append(a3); begin.append(begin[-1] + len(a2))
        models.append(int(cam.model_id)); params.append(cp); seeds.append(int(q[3]) if len(q) > 3 else 0)
    batch = _capi.PnPBatch(begin, np.concatenate(p2), np.concatenate(p3), models, params, np.array(seeds, np.uint64))
    res, _ = _engine.pnp_run(batch, opt, ctx)
    out = []
    intrinsics = bool(opt.refine_focal_length or opt.refine_extra_params)
    for k, (q, r) in enumerate(zip(queries, res)):
        if not r["success"]:
            out.append({"success": False})
            continue
        if intrinsics:
            cam = q[2]
            cam.params[:] = batch.cam_params[k, :len(cam.params)]
        mask = batch.inlier_mask[begin[k]:begin[k + 1]]
        out.append({"success": True, "qvec": batch.qvec[k].copy(), "tvec": batch.tvec[k].copy(),
                    "num_inliers": int(r["num_inliers"]), "inliers": [bool(m) for m in mask]})
    return out


def absolute_pose_estimation(points2D, points3D, camera, estimation_options=None, refinement_options=None):
    """pycolmap 0.4's absolute_pose_estimation on the device: LO-RANSAC over P3P (Lambda Twist) with the pixel threshold
    estimation_options["ransac"]["max_error"], then a Cauchy-robust refinement of the pose over the inliers (and of the
    focal length / extra parameters when refinement_options ask: camera.params is then updated in place).  Options use
    pycolmap's nested names; unknown keys raise.  Defaults (pycolmap 0.4 as best known, unverified against an installed
    pycolmap): ransac max_error 12, min_inlier_ratio 0.01, min_num_trials 1000, max_num_trials 100000, confidence
    0.9999, dyn_num_trials_multiplier 3; refinement gradient_tolerance 1, max_num_iterations 100, loss_function_scale 1,
    refine_focal_length / refine_extra_params False.  Returns dict(success, qvec, tvec, num_inliers, inliers) or
    {"success": False}; estimate_focal_length=True is not supported."""
    return absolute_pose_estimation_batch([(points2D, points3D, camera)], estimation_options, refinement_options)[0]
