"""pixsfm.refine_colmap — the `PixSfM` driver around the two adjusters (reference pixsfm/refine_colmap.py:23-145):
COLMAP database -> keypoint adjustment -> database, COLMAP model -> bundle adjustment -> model.

What differs from the reference, and why:
  * dense features: with `dense_features.model.name == "dsift"` (the `dsift` preset) the driver builds the package's
    own `features.extractor.FeatureExtractor`, which computes dense SIFT on the GPU, and runs from an image directory.
    With the default model, S2DNet at num_layers 1, it does the same when the weights file is there: the model's
    `checkpoint_path` is set, or the file sits at `features/models/checkpoints/s2dnet_weights.pth`.  It is never
    downloaded.  For VGG, or S2DNet without its weights, pass an `extractor` object with the reference's interface
    (`extract.features_from_graph` / `features_from_reconstruction` are called on it) or hand the adjusters a ready
    `feature_manager`.  Without either the call raises — nothing is faked.
  * models are read and written by `util.colmap_model_io` (pycolmap is not installable offline); pycolmap
    reconstructions passed in by the caller work as well (duck typing, `util/colmap_types.py`).
  * configuration: dicts (or a YAML path) merged over the reference's defaults; `${..interpolation}` of the reference's
    YAML files is resolved here by handing the top-level `interpolation` block to KA and BA unless they set their own.
  * `triangulation` / `reconstruction` live in `pixsfm.refine_hloc.PixSfM`, as in the reference."""
import re
import shutil
from copy import deepcopy
from pathlib import Path

from . import logger
from .base import interpolation_default_conf
from .bundle_adjustment import BundleAdjuster
from .keypoint_adjustment import KeypointAdjuster, build_matching_graph
from .util.colmap import read_keypoints_from_db, read_matches_from_db, write_keypoints_to_db
from .util.colmap_types import Reconstruction
from .util.conf import merge, to_conf, to_ctr


def _load_conf(conf):
    """dict | preset name | YAML path -> dict"""
    if conf is None:
        return {}
    if isinstance(conf, (str, Path)):
        from .configs import parse_config_path
        conf = parse_config_path(str(conf))
        if isinstance(conf, Path):
            import yaml
            with open(conf) as f:
                conf = yaml.safe_load(f) or {}
    if not isinstance(conf, dict):
        raise TypeError("conf must be a dict, the name of a preset or the path of a YAML file")
    return conf


_REFERENCE = re.compile(r"^\$\{\.*([A-Za-z_]\w*)\}$")


def _resolve_references(node, top):
    """OmegaConf-style "${..name}" / "${name}" strings -> a copy of the top-level block of that name (the only kind of
    interpolation the reference's configuration files use); a reference to a block the file does not have is dropped"""
    if not isinstance(node, dict):
        return node
    out = {}
    for key, value in node.items():
        m = _REFERENCE.match(value) if isinstance(value, str) else None
        if m is None:
            out[key] = _resolve_references(value, top)
        elif isinstance(top.get(m.group(1)), dict):
            out[key] = deepcopy(top[m.group(1)])
    return out


def _model_name(dense_features):
    """dense_features.model.name, or None"""
    model = dense_features.get("model") if isinstance(dense_features, dict) else None
    return model.get("name") if isinstance(model, dict) else None


def _builtin_extractor(dense_features):
    """the package's own FeatureExtractor for a `dense_features` block: for dsift, and for s2dnet (the default model)
    when its weights file is given or at the default place; None otherwise"""
    name = _model_name(dense_features) or "s2dnet"
    if name == "s2dnet":
        from .features.models.s2dnet import DEFAULT_CHECKPOINT
        model = dense_features.get("model") if isinstance(dense_features, dict) else None
        if (model or {}).get("checkpoint_path") is None and not DEFAULT_CHECKPOINT.is_file():
            return None
    elif name != "dsift":
        return None
    from .features.extractor import FeatureExtractor
    return FeatureExtractor(to_ctr(dense_features))


def _no_extractor_hint():
    from .features.models.s2dnet import DEFAULT_CHECKPOINT
    return (" (S2DNet is computed here from its weights file: set dense_features.model.checkpoint_path, or put it at %s)"
            % DEFAULT_CHECKPOINT)


class PixSfM:
    default_conf = {
        "interpolation": interpolation_default_conf,
        "KA": {**KeypointAdjuster.default_conf},
        "BA": {**BundleAdjuster.default_conf},
    }

    def __init__(self, conf=None, extractor=None):
        top = _load_conf(conf)
        conf = dict(top.get("mapping", top))
        for shared in ("interpolation", "dense_features"):       # blocks a file keeps at its top level
            if shared not in conf and isinstance(top.get(shared), dict):
                conf[shared] = top[shared]
        conf = _resolve_references(conf, top)
        unknown = set(conf) - {"interpolation", "KA", "BA", "dense_features"}
        if unknown:
            raise ValueError("unknown configuration keys: %s" % sorted(unknown))
        interpolation = merge(self.default_conf["interpolation"], conf.get("interpolation"))
        self.conf = merge(self.default_conf, {k: v for k, v in conf.items() if k != "dense_features"})
        self.conf["dense_features"] = to_conf(conf.get("dense_features", {}))
        for part in ("KA", "BA"):       # "${..interpolation}": the shared block unless the adjuster has its own
            if "interpolation" not in conf.get(part, {}):
                self.conf[part]["interpolation"] = to_conf(deepcopy(interpolation))
        if extractor is None:
            extractor = _builtin_extractor(self.conf["dense_features"])
        self.extractor = extractor
        # the reference builds its extractor FROM conf.dense_features (refine_colmap.py:52-56); here the extractor comes in
        # from outside (the CNN is not part of this package), so the block is applied to it where it knows the option
        known = getattr(extractor, "default_conf", None)
        if isinstance(known, dict) and isinstance(getattr(extractor, "conf", None), dict):
            extractor.conf.update({k: v for k, v in dict(self.conf["dense_features"]).items() if k in known})
        self.keypoint_adjuster = KeypointAdjuster.create(self.conf.KA)
        self.bundle_adjuster = BundleAdjuster.create(self.conf.BA)

    # ---------------------------------------------------------------------------------------- features
    def _features(self, how, *args, cache_path=None):
        if self.extractor is None:
            raise ValueError("no feature_manager given and no extractor configured: dense feature extraction (the CNN) "
                             "is outside this package — pass feature_manager= or PixSfM(conf, extractor=...)"
                             + _no_extractor_hint())
        return getattr(self.extractor, how)(*args, cache_path=cache_path)

    # ---------------------------------------------------------------------------------------- KA
    def run_ka(self, keypoints, image_dir, pairs, matches_scores, cache_path=None, feature_manager=None):
        cache_path = self.resolve_cache_path(cache_path)
        graph = build_matching_graph(pairs, *matches_scores)
        if feature_manager is None:
            feature_manager = self._features("features_from_graph", image_dir, graph, keypoints, cache_path=cache_path)
        ka_data = self.keypoint_adjuster.refine_multilevel(keypoints, feature_manager, graph)
        return keypoints, ka_data, feature_manager

    def refine_keypoints_from_db(self, output_path, database_path, image_dir=None, cache_path=None, feature_manager=None):
        output_path, database_path = Path(output_path), Path(database_path)
        cache_path = self.resolve_cache_path(cache_path, output_path.parent)
        keypoints = read_keypoints_from_db(database_path)
        pairs, matches, scores = read_matches_from_db(database_path)
        keypoints, ka_data, feature_manager = self.run_ka(keypoints, image_dir, pairs, (matches, scores), cache_path,
                                                          feature_manager)
        if database_path != output_path:
            shutil.copy(database_path, output_path)
        write_keypoints_to_db(output_path, keypoints)
        return keypoints, ka_data, feature_manager

    # ---------------------------------------------------------------------------------------- BA
    def run_ba(self, reconstruction, image_dir=None, cache_path=None, feature_manager=None):
        cache_path = self.resolve_cache_path(cache_path)
        if feature_manager is None:
            feature_manager = self._features("features_from_reconstruction", reconstruction, image_dir, cache_path=cache_path)
        ba_data = self.bundle_adjuster.refine_multilevel(reconstruction, feature_manager)
        return reconstruction, ba_data, feature_manager

    def refine_reconstruction(self, output_path, input_path, image_dir=None, cache_path=None, feature_manager=None):
        reconstruction = Reconstruction.read(input_path)
        logger.info("Loaded a model with %d images, %d points, %d observations.", len(reconstruction.images),
                    len(reconstruction.points3D), reconstruction.num_observations())
        cache_path = self.resolve_cache_path(cache_path, Path(output_path))
        reconstruction, ba_data, feature_manager = self.run_ba(reconstruction, image_dir, cache_path=cache_path,
                                                               feature_manager=feature_manager)
        Path(output_path).mkdir(exist_ok=True, parents=True)
        reconstruction.write(str(output_path))
        return reconstruction, ba_data, feature_manager

    def resolve_cache_path(self, cache_path=None, output_dir=None):
        """refine_colmap.py:131-145: where the dense-feature cache of this run lives (None without an extractor)"""
        if self.extractor is None or getattr(self.extractor, "conf", None) is None:
            return None if cache_path is None else Path(cache_path)
        feature_conf = self.extractor.conf
        if cache_path is None:
            if output_dir is None:
                return None
            cache_path = output_dir
        cache_path = Path(cache_path)
        if cache_path.suffix != ".h5":
            model = feature_conf.get("model") if isinstance(feature_conf, dict) else getattr(feature_conf, "model", None)
            name = (model["name"] if isinstance(model, dict) else getattr(model, "name", None)) if model is not None else None
            name = name or getattr(self.extractor, "name", None) or "features"     # DenseFeatureExtractor wraps a callable
            sparse = feature_conf["sparse"] if isinstance(feature_conf, dict) else feature_conf.sparse
            cache_path = cache_path / "{}_featuremaps_{}.h5".format(name, "sparse" if sparse else "dense")
        return cache_path

    def triangulation(self, *args, **kwargs):
        raise NotImplementedError("triangulation / reconstruction from hloc files are methods of pixsfm.refine_hloc.PixSfM "
                                  "(refine_hloc.py:117-146)")

    reconstruction = triangulation
