"""pixsfm.localization.main — the reference's query refinement surface (pixsfm/localization/main.py:20-330): helper
functions, QueryKeypointAdjuster, QueryBundleAdjuster and a QueryLocalizer whose PnP step is pluggable: a given
callable, else pycolmap.absolute_pose_estimation (the reference's call) when pycolmap imports, else the built-in
absolute_pose_estimation (LO-RANSAC over P3P and a robust pose refinement on the GPU, batched over the queries of
localize_batch)."""
import numpy as np

from .. import defaults
from .._pixsfm import _engine, _localization as loc
from ..util.conf import merge, to_ctr
from ..util.refine import level_order, optimizer_options

resolve_level_indices = level_order          # the reference's name (util/misc.py:19-23)
to_optim_ctr = optimizer_options             # the reference's name (util/misc.py:30-36)


def st_needs_features(states):
    """the queries' states need reference descriptors (QKA or QBA runs)"""
    return bool(states) and states[0]["require_feats"]


def find_feature_inliers(p2Ds, fmap, references, interpolation_config, thresh=-1, point2D_idxs=None):
    """a correspondence whose reference is ONE descriptor (ndarray) is an outlier when the descriptor interpolated at
    its keypoint is farther than `thresh` (L2) from it; other reference kinds are not tested; thresh < 0 switches the
    test off (reference main.py:20-36)"""
    n = len(p2Ds)
    if thresh < 0.0:
        return [True] * n
    idxs = range(n) if point2D_idxs is None else point2D_idxs
    desc = loc.interpolate_descriptors(fmap, list(idxs), np.asarray(p2Ds, np.float64), interpolation_config)
    return [not isinstance(ref, np.ndarray) or bool(np.linalg.norm(d - ref.reshape(-1)) <= thresh)
            for d, ref in zip(desc, references)]


def find_unique_inliers(idxs, pre_inliers=None):
    """keep the first admissible correspondence of every keypoint index (reference main.py:53-63)"""
    keep, taken = [], set()
    for k, idx in enumerate(idxs):
        ok = (pre_inliers is None or bool(pre_inliers[k])) and idx not in taken
        if ok:
            taken.add(idx)
        keep.append(ok)
    return keep


def find_unique_min_by_group(errors, idxs, pre_inliers=None):
    """per keypoint index keep the admissible correspondence with the smallest error (first on ties; main.py:66-78)"""
    if len(idxs) != len(errors):
        raise ValueError("errors and idxs must have the same length")
    best = {}
    for k, (group, err) in enumerate(zip(idxs, errors)):
        if pre_inliers is not None and not pre_inliers[k]:
            continue
        if group not in best or err < best[group][1]:
            best[group] = (k, err)
    keep = [False] * len(idxs)
    for k, _ in best.values():
        keep[k] = True
    return keep


class QueryKeypointAdjuster:
    """keypoints of one query image against fixed reference descriptors (reference main.py:81-167)"""
    default_conf = defaults.query_keypoint_adjustment()

    def __init__(self, conf=None, callbacks=()):
        self.conf = merge(self.default_conf, conf or {})
        self.solver = loc.QueryKeypointOptimizer(optimizer_options(self.conf.optimizer, list(callbacks)),
                                                 to_ctr(self.conf.interpolation))

    def refine(self, pnp_points2D, fmap, references, point2D_idxs=None):
        inliers = find_feature_inliers(pnp_points2D, fmap, references, to_ctr(self.conf.interpolation),
                                       thresh=self.conf.feature_inlier_thresh, point2D_idxs=point2D_idxs)
        if self.conf.stack_correspondences:
            return self.refine_stacked(pnp_points2D, fmap, references, point2D_idxs, inliers=inliers)
        self.solver = loc.QueryKeypointOptimizer(self.solver.options, self.solver.interp)      # optimizers are one-shot
        self.solver.run(pnp_points2D, fmap, references, patch_idxs=point2D_idxs, inliers=inliers)

    def refine_multilevel(self, pnp_points2D, query_fmaps, references, point2D_idxs=None):
        for level in level_order(self.conf.level_indices, len(query_fmaps)):
            self.refine(pnp_points2D, query_fmaps[level], references[level], point2D_idxs=point2D_idxs)

    def refine_batch(self, queries, max_wave_bytes=0.0):
        """refine() for every query of `queries`, tuples (pnp_points2D, fmap, references[, point2D_idxs]): the feature
        inlier test of all queries in one pxr_query_match_run, then one batched solve (QueryKeypointOptimizer.run_batch)"""
        queries = [tuple(q) + (None,) * (4 - len(q)) for q in queries]
        inl = loc.feature_inliers_batch(queries, to_ctr(self.conf.interpolation), self.conf.feature_inlier_thresh)
        items, stacked = [], []
        for (p2D, fmap, refs, idxs), inliers in zip(queries, inl):
            if self.conf.stack_correspondences:
                kps, targets, slots, admitted, where = self._stack(p2D, refs, idxs, inliers)
                items.append((kps, fmap, targets, slots, admitted)); stacked.append((p2D, kps, where))
            else:
                items.append((p2D, fmap, refs, idxs, inliers))
        self.solver = loc.QueryKeypointOptimizer(self.solver.options, self.solver.interp)
        self.solver.run_batch(items, max_wave_bytes)
        for p2D, kps, where in stacked:
            for k, slot in enumerate(where):
                p2D[k] = kps[slot]

    def refine_multilevel_batch(self, queries, max_wave_bytes=0.0):
        """refine_multilevel() for every query of `queries`, tuples (pnp_points2D, query_fmaps, references[,
        point2D_idxs]) with one fmap and one reference list per level: one batched refine per level"""
        queries = list(queries)
        if not queries:
            return
        n_levels = len(queries[0][1])
        if any(len(q[1]) != n_levels for q in queries):
            raise ValueError("every query of a batch must have the same number of feature levels")
        for level in level_order(self.conf.level_indices, n_levels):
            self.refine_batch([(q[0], q[1][level], q[2][level]) + tuple(q[3:]) for q in queries], max_wave_bytes)

    @staticmethod
    def _stack(pnp_points2D, references, point2D_idxs, inliers):
        """correspondences that share a keypoint as ONE keypoint with several targets: (keypoints, targets, keypoint
        indices, admitted, slot of every correspondence)"""
        if point2D_idxs is None:
            raise ValueError("point2D_idxs must not be None in stacked QKA.")
        slot_of, slots = {}, []                       # keypoint index -> position among the distinct keypoints
        for p2D_idx in point2D_idxs:
            if p2D_idx not in slot_of:
                slot_of[p2D_idx] = len(slots)
                slots.append(p2D_idx)
        where = [slot_of[p] for p in point2D_idxs]
        stacked_kps = np.zeros((len(slots), 2))
        targets = [[] for _ in slots]
        admitted = [False] * len(slots)
        for k, ref in enumerate(references):
            if not isinstance(ref, np.ndarray):
                raise ValueError("Stacked QKA requires a np.ndarray reference for each 2D-3D correspondence. "
                                 "Consider setting target_references='nearest'.")
            stacked_kps[where[k]] = pnp_points2D[k]
            targets[where[k]].append(ref)
            admitted[where[k]] = admitted[where[k]] or inliers is None or bool(inliers[k])
        return stacked_kps, targets, slots, (None if inliers is None else admitted), where

    def refine_stacked(self, pnp_points2D, fmap, references, point2D_idxs, inliers=None):
        """correspondences that share a keypoint are stacked into ONE keypoint with several targets"""
        stacked_kps, targets, slots, admitted, where = self._stack(pnp_points2D, references, point2D_idxs, inliers)
        self.solver.run(stacked_kps, fmap, targets, patch_idxs=slots, inliers=admitted)
        for k, slot in enumerate(where):
            pnp_points2D[k] = stacked_kps[slot]


class QueryBundleAdjuster:
    """pose (and optionally intrinsics) of one query image against fixed 3D points (reference main.py:170-259)"""
    default_conf = defaults.query_bundle_adjustment()

    def __init__(self, conf=None, callbacks=()):
        self.conf = merge(self.default_conf, conf or {})
        self.solver = loc.QueryBundleOptimizer(optimizer_options(self.conf.optimizer, list(callbacks)),
                                               to_ctr(self.conf.interpolation))

    def refine(self, qvec, tvec, camera, points3D, fmap, references, inliers=None, point2D_idxs=None):
        return self.solver.run(qvec, tvec, camera, points3D, fmap, references, inliers=inliers, patch_idxs=point2D_idxs)

    def refine_multilevel(self, qvec, tvec, camera, points3D, fmaps, references, inliers=None, point2D_idxs=None):
        if len(fmaps) != len(references):
            raise ValueError("one reference list per feature level is required")
        for level in level_order(self.conf.level_indices, len(fmaps)):
            self.refine(qvec, tvec, camera, points3D, fmaps[level], references[level], inliers=inliers,
                        point2D_idxs=point2D_idxs)

    def refine_batch(self, queries, max_wave_bytes=0.0):
        """refine() for every query of `queries`, tuples (qvec, tvec, camera, points3D, fmap, references[, inliers[,
        point2D_idxs]]), in one batched solve (QueryBundleOptimizer.run_batch) -> one bool per query"""
        return self.solver.run_batch(queries, max_wave_bytes)

    def refine_multilevel_batch(self, queries, max_wave_bytes=0.0):
        """refine_multilevel() for every query of `queries`, tuples (qvec, tvec, camera, points3D, fmaps, references[,
        inliers[, point2D_idxs]]) with one fmap and one reference list per level: each level is one batched solve that
        starts from the previous level's result"""
        queries = list(queries)
        if not queries:
            return
        n_levels = len(queries[0][4])
        for q in queries:
            if len(q[4]) != len(q[5]):
                raise ValueError("one reference list per feature level is required")
            if len(q[4]) != n_levels:
                raise ValueError("every query of a batch must have the same number of feature levels")
        for level in level_order(self.conf.level_indices, n_levels):
            self.refine_batch([tuple(q[:4]) + (q[4][level], q[5][level]) + tuple(q[6:]) for q in queries], max_wave_bytes)


def compute_reprojection_errors(pnp_points2D, pnp_points3D, qvec, tvec, camera):
    """pixel distance between every 2D point and the projection of its 3D point (reference main.py:96-102)"""
    from ..util.cameras import world_to_image
    xyz = np.array([np.asarray(getattr(p, "xyz", p), np.float64) for p in pnp_points3D]).reshape(-1, 3)
    proj = world_to_image(camera.model_id, np.asarray(camera.params, np.float64), np.asarray(qvec, np.float64),
                          np.asarray(tvec, np.float64), xyz)
    return [float(np.linalg.norm(proj[i] - np.asarray(p2D, np.float64))) for i, p2D in enumerate(pnp_points2D)]


def find_unique_min_reproj_inliers(pnp_points3D_id, qvec, tvec, camera, pnp_points2D, rec, pre_inliers=None, point2D_idxs=None):
    """of the correspondences that share a 3D point, then of those that share a keypoint, keep the one with the smallest
    reprojection error under the PnP pose (reference main.py:81-93)"""
    p3Ds = [rec.points3D[p3D_id] for p3D_id in pnp_points3D_id]
    errors = compute_reprojection_errors(pnp_points2D, p3Ds, qvec, tvec, camera)
    inliers = pre_inliers
    for idxs in (pnp_points3D_id, point2D_idxs):
        if idxs is None:
            continue
        inliers = find_unique_min_by_group(errors, idxs, pre_inliers=inliers)
    return inliers


class QueryLocalizer:
    """QKA -> PnP -> QBA for one query image (reference localization/main.py:262-537), with the reference's constructor
    and `localize` signatures.  Holds the reconstruction and one {point3D_id: Reference} map per feature level: given
    (`references=`), or extracted at construction from `dense_features` (a FeatureManager, or the path of a feature cache)
    or from features the `extractor` computes for `image_dir`.  The absolute-pose step is `pose_estimator(points2D [N,2],
    points3D [N,3], camera) -> dict(success, qvec, tvec, inliers)` when one is given, else
    pycolmap.absolute_pose_estimation when pycolmap imports, else this package's absolute_pose_estimation (the conf's
    PnP.estimation / PnP.refinement merged over its pycolmap defaults)."""
    default_conf = defaults.query_localizer()

    def __init__(self, reconstruction, conf=None, dense_features=None, image_dir=None, references=None, extractor=None,
                 pose_estimator=None):
        from pathlib import Path
        from .. import bundle_adjustment as ba_pkg
        from .._pixsfm import _bundle_adjustment as ba
        if isinstance(conf, (str, Path)):
            from ..refine_colmap import _load_conf
            conf = _load_conf(conf)
        if isinstance(conf, dict) and isinstance(conf.get("localization"), dict):
            from ..refine_colmap import _resolve_references
            conf = _resolve_references(conf["localization"], conf)
        self.conf = merge(self.default_conf, conf or {})
        if self.conf.QKA.stack_correspondences and self.conf.target_reference not in ("nearest", "robust_mean"):
            raise ValueError("Stacked QKA requires a np.ndarray reference for each 2D-3D correspondence. Consider setting "
                             "target_references to 'nearest' or 'robust_mean'.")
        self.query_keypoint_adjuster = QueryKeypointAdjuster(to_ctr(self.conf.QKA))
        self.query_bundle_adjuster = QueryBundleAdjuster(to_ctr(self.conf.QBA))
        if extractor is None:
            from ..refine_colmap import _builtin_extractor
            extractor = _builtin_extractor(self.conf.dense_features)
        self.extractor = extractor
        self.pose_estimator = pose_estimator
        self.reference_extractor = ba.ReferenceExtractor(to_ctr(self.conf.references), to_ctr(self.conf.interpolation))
        self.target_reference_funcs = {"nearest": self.get_nearest_references, "robust_mean": self.get_robust_mean_references,
                                       "all_observations": self.get_all_references, "full": self.get_full_references}
        if self.conf.target_reference not in self.target_reference_funcs:
            raise ValueError("unknown target_reference %r" % (self.conf.target_reference,))
        self.get_query_references = self.target_reference_funcs[self.conf.target_reference]
        self.references = references
        if self.references is None and (self.conf.QKA.apply or self.conf.QBA.apply):
            cache_path = None
            if isinstance(dense_features, (str, Path)):
                cache_path = Path(dense_features)
                if cache_path.exists():
                    from ..features.store_features import load_features_from_cache
                    dense_features = load_features_from_cache(cache_path)
                else:
                    dense_features = None
            if dense_features is None:
                if image_dir is None or self.extractor is None:
                    raise ValueError("references (one {point3D_id: Reference} map per level), dense_features, or an extractor "
                                     "together with image_dir are required")
                dense_features = self.extractor.features_from_reconstruction(reconstruction, image_dir, cache_path=cache_path)
            labels = ba_pkg.find_problem_labels(reconstruction, self.conf.max_tracks_per_problem)
            self.references = [self.reference_extractor.run(labels, reconstruction, dense_features.fset(i))
                               for i in range(dense_features.num_levels)]
        self.reconstruction = reconstruction

    # ---- the reference descriptors a query's correspondences are compared with, one list per level (main.py:499-537)
    def get_nearest_references(self, pnp_points3D_id, query_fmaps, pnp_points2D, patch_idxs):
        return [loc.find_nearest_references(query_fmaps[level], refs, pnp_points2D, pnp_points3D_id,
                                            to_ctr(self.conf.interpolation), patch_idxs)
                for level, refs in enumerate(self.references)]

    def get_robust_mean_references(self, pnp_points3D_id, *args):
        return [[np.asarray(refs[p3D_id].descriptor, np.float64) for p3D_id in pnp_points3D_id] for refs in self.references]

    def get_all_references(self, pnp_points3D_id, *args):
        out = []
        for refs in self.references:
            level = []
            for p3D_id in pnp_points3D_id:
                if not len(refs[p3D_id].observations):
                    raise RuntimeError("Missing descriptors for observations.\nAssure that references.keep_observations==True.")
                level.append([np.asarray(o) for o in refs[p3D_id].observations])
            out.append(level)
        return out

    def get_full_references(self, pnp_points3D_id, *args):
        return [[refs[p3D_id] for p3D_id in pnp_points3D_id] for refs in self.references]

    def _query_features(self, image_path, keypoints, required_kp_ids):
        """the patches of the query image around the keypoints that take part in a correspondence (main.py:432-439)"""
        if self.extractor is None:
            raise ValueError("query_fmaps or an extractor (with image_path) are required")
        name = str(image_path)
        manager = self.extractor.features_from_image_list(None, [name], {name: keypoints}, {name: required_kp_ids})
        return [manager.fset(level).fmap(name) for level in range(manager.num_levels)]

    def _pose_estimator(self, pose_estimator=None):
        """the per-query PnP callable: `pose_estimator`, else the localizer's, else pycolmap.absolute_pose_estimation when
        pycolmap imports; None: the built-in estimator (absolute_pose_estimation on the device), batched over queries"""
        estimator = pose_estimator or self.pose_estimator
        if estimator is not None:
            return lambda p2D, p3D, camera: estimator(p2D, np.array(p3D), camera)
        try:
            import pycolmap
        except ImportError:
            return None
        return lambda p2D, p3D, camera: pycolmap.absolute_pose_estimation(
            p2D, p3D, camera, estimation_options=to_ctr(self.conf.PnP.estimation),
            refinement_options=to_ctr(self.conf.PnP.refinement))

    def _absolute_pose(self, pnp_points2D, pnp_points3D, query_camera, pose_estimator):
        estimator = self._pose_estimator(pose_estimator)
        if estimator is not None:
            return estimator(pnp_points2D, pnp_points3D, query_camera)
        return loc.absolute_pose_estimation(pnp_points2D, pnp_points3D, query_camera,
                                            estimation_options=to_ctr(self.conf.PnP.estimation),
                                            refinement_options=to_ctr(self.conf.PnP.refinement))

    def localize(self, keypoints, pnp_point2D_idxs, pnp_points3D_id, query_camera, image_path=None, query_fmaps=None,
                 pose_estimator=None):
        """reference main.py:414-497.  `keypoints` [K,2] are the query image's keypoints, correspondence k pairs keypoint
        `pnp_point2D_idxs[k]` with 3D point `pnp_points3D_id[k]`.  Returns the pose dict of the PnP step with the refined
        pose, `inliers` / `num_inliers` recomputed from it, and (an addition) `keypoints`: the refined 2D points of the
        correspondences."""
        st = self._localize_begin(keypoints, pnp_point2D_idxs, pnp_points3D_id, query_camera, image_path, query_fmaps,
                                  pose_estimator)
        if "result" in st:
            return st["result"]
        if self.conf.QBA.apply:
            self.query_bundle_adjuster.refine_multilevel(*self._qba_args(st))
        return self._localize_end(st)

    def localize_batch(self, queries, max_wave_bytes=0.0):
        """localize() for every entry of `queries` (dicts of localize's keyword arguments): per feature level the
        reference selection of every query at once (one pxr_query_match_run for target_reference 'nearest', against the
        level's stored observations packed once and kept in device memory), per level one batched QKA solve, PnP (one
        pxr_pnp_run for every query on the built-in estimator, else per query), one batched QBA solve per level over every query that has a pose, then the per-query inlier
        recomputation.  Returns the list of pose dicts localize would return."""
        states = [self._localize_prepare(**q) for q in queries]
        live = [st for st in states if "result" not in st]
        if live and st_needs_features(live):
            if self.conf.target_reference == "nearest":
                per_level = [loc.find_nearest_references_batch(
                    [(st["fmaps"][level], refs, st["points2D"], st["points3D_id"], st["point2D_idxs"]) for st in live],
                    to_ctr(self.conf.interpolation), _table=self._observation_table(level))
                    for level, refs in enumerate(self.references)]
                for k, st in enumerate(live):
                    st["references"] = [lvl[k] for lvl in per_level]
            else:
                for st in live:
                    st["references"] = self.get_query_references(st["points3D_id"], st["fmaps"], st["points2D"],
                                                                 st["point2D_idxs"])
            for st in live:
                if len(st["fmaps"]) != len(st["references"]):
                    raise ValueError("one reference map per feature level is required")
            if self.conf.QKA.apply:
                self.query_keypoint_adjuster.refine_multilevel_batch(
                    [(st["points2D"], st["fmaps"], st["references"], st["point2D_idxs"]) for st in live], max_wave_bytes)
        builtin = [st for st in states if "result" not in st and self._pose_estimator(st["pose_estimator"]) is None]
        poses = {}
        if builtin:                                           # the built-in estimator: every such query in one launch
            found = loc.absolute_pose_estimation_batch([(st["points2D"], st["points3D"], st["camera"]) for st in builtin],
                                                       estimation_options=to_ctr(self.conf.PnP.estimation),
                                                       refinement_options=to_ctr(self.conf.PnP.refinement))
            poses = {id(st): pose for st, pose in zip(builtin, found)}
        states = [st if "result" in st else self._localize_pose(st, poses.get(id(st))) for st in states]
        live = [st for st in states if "result" not in st]
        if self.conf.QBA.apply and live:
            self.query_bundle_adjuster.refine_multilevel_batch([self._qba_args(st) for st in live], max_wave_bytes)
        return [st["result"] if "result" in st else self._localize_end(st) for st in states]

    def _observation_table(self, level):
        """every stored observation descriptor of the level's 3D points, packed once and kept in device memory:
        (rows, {point id: (first row, count)})"""
        cache = self.__dict__.setdefault("_obs_tables", {})
        if level not in cache:
            refs = self.references[level]
            pids = [p for p in refs if getattr(refs[p], "observations", None)]
            rows, where = loc.observation_table(refs, pids)
            cache[level] = (_engine.device_array(rows) if len(rows) else rows, where)
        return cache[level]

    @staticmethod
    def _qba_args(st):
        pose = st["pose"]
        return (pose["qvec"], pose["tvec"], st["camera"], st["points3D"], st["fmaps"], st["references"], list(st["inliers"]),
                st["point2D_idxs"])

    def _localize_begin(self, keypoints, pnp_point2D_idxs, pnp_points3D_id, query_camera, image_path=None, query_fmaps=None,
                        pose_estimator=None):
        """localize up to the QBA step: {"result": pose dict} when it ends early, else the state _localize_end takes"""
        st = self._localize_prepare(keypoints, pnp_point2D_idxs, pnp_points3D_id, query_camera, image_path, query_fmaps,
                                    pose_estimator)
        if "result" in st:
            return st
        if st_needs_features([st]):
            st["references"] = self.get_query_references(st["points3D_id"], st["fmaps"], st["points2D"], st["point2D_idxs"])
            if len(st["fmaps"]) != len(st["references"]):
                raise ValueError("one reference map per feature level is required")
        if self.conf.QKA.apply:
            self.query_keypoint_adjuster.refine_multilevel(st["points2D"], st["fmaps"], st["references"],
                                                           point2D_idxs=st["point2D_idxs"])
        return self._localize_pose(st)

    def _localize_prepare(self, keypoints, pnp_point2D_idxs, pnp_points3D_id, query_camera, image_path=None,
                          query_fmaps=None, pose_estimator=None):
        """the checks and inputs of one query: {"result": pose dict} when it ends early, else its state"""
        if len(pnp_point2D_idxs) != len(pnp_points3D_id):
            raise ValueError("one 3D point id per 2D index is required")
        if image_path is None and query_fmaps is None:
            raise ValueError("image_path or query_fmaps are required")
        if len(pnp_point2D_idxs) == 0:
            return {"result": {"success": False}}
        pnp_point2D_idxs = [int(i) for i in pnp_point2D_idxs]
        pnp_points3D = [np.asarray(self.reconstruction.points3D[p3D_id].xyz, np.float64) for p3D_id in pnp_points3D_id]
        keypoints = np.array(keypoints, dtype=np.float64)
        require_feats = bool(self.conf.QKA.apply or self.conf.QBA.apply)
        if query_fmaps is None and require_feats:
            query_fmaps = self._query_features(image_path, keypoints, sorted(set(pnp_point2D_idxs)))
        pnp_points2D = keypoints[pnp_point2D_idxs]           # a copy: QKA refines the correspondences' points
        return {"camera": query_camera, "points2D": pnp_points2D, "points3D": pnp_points3D, "points3D_id": pnp_points3D_id,
                "fmaps": query_fmaps, "references": None, "point2D_idxs": pnp_point2D_idxs, "require_feats": require_feats,
                "pose_estimator": pose_estimator}

    def _localize_pose(self, st, pose_dict=None):
        """PnP on the (refined) correspondences (unless its pose dict is given) and the inlier selection: {"result": pose
        dict} when PnP fails"""
        pnp_points2D, pnp_points3D, query_camera = st["points2D"], st["points3D"], st["camera"]
        if pose_dict is None:
            pose_dict = self._absolute_pose(pnp_points2D, pnp_points3D, query_camera, st["pose_estimator"])
        if not pose_dict.get("success", False):
            return {"result": pose_dict}
        inliers = pose_dict.get("inliers", [True] * len(pnp_points3D))
        if self.conf.unique_inliers:                          # None / False: keep what PnP says
            if self.conf.unique_inliers == "random":
                inliers = find_unique_inliers(st["points3D_id"], pre_inliers=inliers)
            elif self.conf.unique_inliers == "min_error":
                inliers = find_unique_min_reproj_inliers(st["points3D_id"], pose_dict["qvec"], pose_dict["tvec"], query_camera,
                                                         pnp_points2D, self.reconstruction, pre_inliers=inliers,
                                                         point2D_idxs=st["point2D_idxs"])
            else:
                from .. import logger
                logger.warning("Unknown unique_inlier method %s.", self.conf.unique_inliers)
        return {"pose": pose_dict, "camera": query_camera, "points2D": pnp_points2D, "points3D": pnp_points3D,
                "fmaps": st["fmaps"], "references": st["references"], "inliers": inliers,
                "point2D_idxs": st["point2D_idxs"]}

    def _localize_end(self, st):
        pose_dict = st["pose"]
        errors = compute_reprojection_errors(st["points2D"], st["points3D"], pose_dict["qvec"], pose_dict["tvec"], st["camera"])
        max_error = self.conf.PnP.estimation.ransac.max_error
        pose_dict["inliers"] = [err < max_error for err in errors]
        pose_dict["num_inliers"] = sum(pose_dict["inliers"])
        pose_dict["keypoints"] = st["points2D"]
        return pose_dict
