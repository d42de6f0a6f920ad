"""Mirror of `pixsfm._pixsfm._keypoint_adjustment` (pixsfm/keypoint_adjustment/bindings.cc:17-100): the
setup container, the options and FeatureMetricKeypointOptimizer.  Edge enumeration restates
TopologicalKeypointOptimizer::SetUp (topological_keypoint_optimizer.h:95-175) and
AddIntraResiduals (featuremetric_keypoint_optimizer.h:158-202); the solve runs in libpxr.so."""
import numpy as np

from . import _capi, _engine
from ._base import InterpolationConfig
from ._bundle_adjustment import _DictOptions, _Summary, solver_options_from
from ._features import PatchSlab
from .. import logger


class KeypointAdjustmentSetup:
    def __init__(self):
        self.constant_images, self.constant_keypoints = set(), {}

    def set_image_constant(self, image_id): self.constant_images.add(int(image_id))
    def set_node_constant(self, node): self.set_keypoint_constant(node.image_id, node.feature_idx)
    def set_keypoint_constant(self, image_id, feature_idx):
        self.constant_keypoints.setdefault(int(image_id), set()).add(int(feature_idx))
    def set_keypoints_constant(self, image_id, feature_idxs):
        for f in feature_idxs: self.set_keypoint_constant(image_id, f)
    def is_keypoint_constant(self, image_id, feature_idx):
        return int(image_id) in self.constant_images or int(feature_idx) in self.constant_keypoints.get(int(image_id), ())
    def is_node_constant(self, node): return self.is_keypoint_constant(node.image_id, node.feature_idx)
    def set_masked_nodes_constant(self, graph, mask):
        for node, m in zip(graph.nodes, mask):
            if m: self.set_node_constant(node)


class KeypointOptimizerOptions(_DictOptions):
    """keypoint_adjustment_options.h:47-86 + TopologicalKeypointOptimizer::Options (:33-39)"""
    _defaults = dict(print_summary=True, bound=-1.0, num_threads=-1, weight_by_sim=True, root_regularize_weight=-1.0,
                     root_edges_only=False, loss=lambda: {"name": "cauchy", "params": [0.25]},
                     solver=lambda: {"function_tolerance": 0.0, "gradient_tolerance": 0.0, "parameter_tolerance": 1.0e-4,
                                     "max_num_iterations": 100, "max_num_consecutive_invalid_steps": 10})


class TopologicalReferenceKeypointOptimizerOptions(KeypointOptimizerOptions):
    """topological_reference_keypoint_optimizer.h:9-16: every keypoint of a track is pulled towards the track's root
    only (linear instead of quadratic number of residuals)."""
    _defaults = dict(KeypointOptimizerOptions._defaults, weight_by_sim=False, root_regularize_weight=1.0,
                     root_edges_only=True)


class FeatureMetricKeypointOptimizer:
    _options_cls = KeypointOptimizerOptions
    _banner = "Start feature-metric keypoint adjustment."

    def __init__(self, options, setup, interpolation_config):
        self.options = options if isinstance(options, KeypointOptimizerOptions) else self._options_cls(options)
        self.setup = setup
        self.interp = interpolation_config if isinstance(interpolation_config, InterpolationConfig) else InterpolationConfig(interpolation_config)
        self._summary = None
        logger.info(self._banner)

    def run(self, *args):
        """run(keypoints, graph, track_labels, root_labels, feature_set) — one problem over all nodes, or
        run(problem_labels, keypoints, graph, track_labels, root_labels, feature_set) — one problem per label"""
        if len(args) == 5:
            keypoints, graph, track_labels, root_labels, feature_set = args
            problem_labels = [0] * len(graph.nodes)
        elif len(args) == 6:
            problem_labels, keypoints, graph, track_labels, root_labels, feature_set = args
        else:
            raise TypeError("run() takes 5 or 6 positional arguments")
        return self._run(None, problem_labels, keypoints, graph, track_labels, root_labels, feature_set)

    def run_subset(self, nodes_in_problem, keypoints, graph, track_labels, root_labels, feature_set):
        """one problem over the intra-track edges that START at the given nodes (RunSubset,
        featuremetric_keypoint_optimizer.h:118-137 — what the reference's thread pool calls per label); -> summary"""
        subset = sorted({int(n) for n in nodes_in_problem})
        if subset and (subset[0] < 0 or subset[-1] >= len(graph.nodes)):
            raise ValueError("nodes_in_problem holds an index outside the graph")
        self._run(subset, [0] * len(graph.nodes), keypoints, graph, track_labels, root_labels, feature_set)
        return self._summary

    def _run(self, subset, problem_labels, keypoints, graph, track_labels, root_labels, feature_set):
        n_nodes = len(graph.nodes)
        if not (len(track_labels) == len(root_labels) == len(problem_labels) == n_nodes):
            raise ValueError("label arrays must have one entry per graph node")
        self.interp.validate_for_device()
        if keypoints is None:
            raise ValueError("keypoints cannot be NULL.")
        opt = self.options
        # ---- TopologicalKeypointOptimizer::SetUp: intra-track edges of every node, in node order
        regularize = opt.root_regularize_weight > 0.0
        connected, track_root = [False] * n_nodes, {}
        edges = []
        for node in (graph.nodes if subset is None else [graph.nodes[n] for n in subset]):
            for m in node.out_matches:
                if track_labels[node.node_idx] != track_labels[m.node_idx]:
                    continue
                edges.append((node.node_idx, m.node_idx, m.sim))
                if regularize:
                    for a in (node.node_idx, m.node_idx):
                        if root_labels[a]:
                            track_root[track_labels[a]] = a
                            connected[node.node_idx] = connected[m.node_idx] = True
        kp_of = lambda n: (graph.image_id_to_name[graph.nodes[n].image_id], graph.nodes[n].feature_idx)
        flat = []   # (src, dst, weight)
        for (a, b, sim) in edges:
            if kp_of(a) == kp_of(b):
                continue     # same keypoint storage: "Avoid optimizing a keypoint to itself"
            if not (opt.root_edges_only and not root_labels[a] and not root_labels[b]):
                flat.append((a, b, sim if opt.weight_by_sim else 1.0))
            if regularize:
                for n in (a, b):
                    if not connected[n]:
                        # std::unordered_map::operator[] default-inserts node 0 for a track without a root
                        # (topological_keypoint_optimizer.h:161)
                        flat.append((n, track_root.get(track_labels[n], 0), opt.root_regularize_weight))
                        connected[n] = True
        if not flat:
            self._summary = _Summary(initial_cost=0.0, final_cost=0.0, num_residuals_reduced=0, total_time_in_seconds=0.0)
            return True
        flat.sort(key=lambda e: problem_labels[e[0]])   # stable: RunParallel groups by label (std::map order)
        used = sorted({n for e in flat for n in e[:2]})
        # ---- keypoint / patch tables (one entry per graph node that carries a residual)
        slab = PatchSlab()
        kidx = {n: k for k, n in enumerate(used)}
        kps = np.zeros((len(used), 2)); kconst = np.zeros(len(used), np.uint8); kpatch = np.zeros(len(used), np.int64)
        sparse = True
        held = {}    # lazily filled maps (fill=False caches): resident from here to the end of the solve, like the
                     # FeatureView every problem of the reference's RunParallel builds and drops (featureview.cc:70-126)
        for n in used:
            name, fidx = kp_of(n)
            if not feature_set.has_fmap(name) or not feature_set.fmap(name).has_point2D(fidx):
                raise ValueError("no feature patch for keypoint (%s, %d)" % (name, fidx))
            fmap = feature_set.fmap(name)
            if name not in held and hasattr(fmap, "unload"):
                held[name] = fmap.load()
            sparse = sparse and fmap.is_sparse
            kps[kidx[n]] = keypoints[name][fidx]
            kconst[kidx[n]] = 1 if self.setup.is_node_constant(graph.nodes[n]) else 0
            kpatch[kidx[n]] = slab.index(name, fmap, fidx)
        blocks, corners, scales = slab.arrays()
        labels = sorted({problem_labels[e[0]] for e in flat})
        lmap = {l: k for k, l in enumerate(labels)}
        prob = _capi.KAProblem(keypoints=kps, kp_const=kconst, edge_src=[kidx[e[0]] for e in flat],
                               edge_dst=[kidx[e[1]] for e in flat], edge_weight=[e[2] for e in flat],
                               edge_problem=[lmap[problem_labels[e[0]]] for e in flat], n_problems=len(labels),
                               patches=None, corner=corners, scale=scales, kp_patch=kpatch, bound=opt.bound,
                               patches_are_sparse=sparse, patch_blocks=blocks)
        if feature_set.channels not in (8, 16, 32, 64, 128):
            raise ValueError("Unsupported dimensions (CHANNELS,N_NODES).")
        so = solver_options_from(opt.loss, opt.solver, _capi.default_ka_options(parameter_tolerance=1e-4))
        ic = _capi.default_interp(self.interp.l2_normalize, self.interp.use_float_simd)
        try:
            s = _engine.ka_run(prob, ic, so)
        finally:
            for fmap in held.values():
                fmap.unload()
        for n in used:   # keypoints are refined in place
            name, fidx = kp_of(n)
            keypoints[name][fidx] = prob.keypoints[kidx[n]]
        self._summary = _Summary(s, num_residuals_reduced=s["num_residuals"], total_time_in_seconds=s["total_time_s"])
        nres = max(1, s["num_residuals"])
        logger.info("KA Time: %.4gs, cost change: %.6g --> %.6g", s["total_time_s"], np.sqrt(s["initial_cost"] / nres),
                    np.sqrt(s["final_cost"] / nres))
        logger.info("KA solve: %s", s["message"])   # problems, LM iterations, kernel time, problems solved off chip
        return True

    def summary(self):
        return self._summary


class TopologicalReferenceKeypointOptimizer(FeatureMetricKeypointOptimizer):
    """_keypoint_adjustment.TopologicalReferenceKeypointOptimizer (keypoint_adjustment/bindings.cc:86-100;
    topological_reference_keypoint_optimizer.h:5-28): the same optimizer with root edges only, unit edge weights
    and root regularisation on by default — same kernels, different edge set."""
    _options_cls = TopologicalReferenceKeypointOptimizerOptions
    _banner = "Start topological-reference keypoint adjustment."
