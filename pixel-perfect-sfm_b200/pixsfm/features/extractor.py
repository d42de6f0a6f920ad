"""Dense feature maps -> the FeatureMaps the adjusters consume.

The reference's FeatureExtractor (pixsfm/features/extractor.py) owns the CNN (S2DNet, torch) AND the step after it,
`tensor_to_fmap` (:152-236): L2-normalise the C-channel map, cast it, and either keep it dense or cut one
`patch_size` x `patch_size` patch per keypoint with `corner = clip(int(kp * scale - ps / 2), 0, [w, h] - ps - 1)`.  The CNN
is not part of this package; the step after it is, so that any model — a callable image name -> list of [C,H,W] maps,
finest level first — plugs into `PixSfM(conf, extractor=DenseFeatureExtractor(model, ...))`.  The models the package
computes itself, dense SIFT and S2DNet at num_layers 1, have the reference's `FeatureExtractor(conf)`: images in,
FeatureManager out."""
import os
from pathlib import Path

import numpy as np

from .. import logger
from .._pixsfm import _features as features

_DTYPES = {"half": np.float16, "float": np.float32, "double": np.float64}


def _as_numpy(x):
    if hasattr(x, "detach"):                       # a torch tensor straight out of the network
        x = x.detach().cpu().numpy()
    return np.asarray(x)


def patch_corners(keypoints, scale, patch_size, map_wh):
    """top-left map pixel of every keypoint's patch (extractor.py:192-193): truncation towards zero, then clamped so
    that the patch and one more pixel stay inside the map"""
    corners = (np.asarray(keypoints, np.float64) * scale - patch_size / 2.0).astype(np.int32)
    return np.clip(corners, [0, 0], np.asarray(map_wh, np.int64) - patch_size - 1).astype(np.int32)


def sparse_pays_off(map_h, map_w, n_keypoints, patch_size):
    """the reference's rule (tensor_to_fmap, features/extractor.py:182-187): patches are kept only while they are smaller
    than the map they are cut from"""
    return map_h * map_w > n_keypoints * patch_size * patch_size


def cut_patches(dense_hwc, corners, patch_size):
    """[N, ps, ps, C] windows of an [H, W, C] map, rows = y (the layout of FeaturePatch, featurepatch.h:244-262)"""
    rows = corners[:, 1, None] + np.arange(patch_size)[None, :]            # [N, ps]
    cols = corners[:, 0, None] + np.arange(patch_size)[None, :]
    return np.ascontiguousarray(dense_hwc[rows[:, :, None], cols[:, None, :]])


def dense_to_fmap_on_device(featuremap, image_size, keypoints, keypoint_ids=None, patch_size=16, l2_normalize=True,
                            dtype=np.float16, channels_first=True):
    """the sparse branch of dense_to_fmap with the gather done by libpxr on the GPU: `featuremap` may be the CNN's output
    still in device memory (anything with __cuda_array_interface__) or a host array; the patches stay on the device and
    the optimizers take them from there (no GPU -> numpy -> GPU round trip)"""
    from .._pixsfm import _engine
    cai = getattr(featuremap, "__cuda_array_interface__", None)
    shape = tuple(cai["shape"]) if cai is not None else np.shape(featuremap)
    if len(shape) == 4 and shape[0] == 1:
        shape = shape[1:]
    if len(shape) != 3:
        raise ValueError("a feature map is [C,H,W] (or [H,W,C] with channels_first=False)")
    h, w = (shape[1], shape[2]) if channels_first else (shape[0], shape[1])
    keypoints = np.asarray(keypoints, np.float64).reshape(-1, 2)
    if keypoint_ids is None:
        keypoint_ids = list(range(len(keypoints)))
    elif len(keypoint_ids) != len(keypoints):
        raise ValueError("Number of provided keypoint_ids and keypoints do not match.")
    scale = np.array((w / image_size[0], h / image_size[1]))
    source = featuremap if cai is not None else _as_numpy(featuremap)
    if cai is None and source.ndim == 4:
        source = source[0]
    if not sparse_pays_off(h, w, len(keypoints), patch_size):
        # sparse does not pay off (reference tensor_to_fmap, features/extractor.py:182-187, same rule as dense_to_fmap):
        # ONE dense patch, normalised / cast / transposed to HWC by the same gather kernel with a single h x w window.
        # pxr_extract_patches takes square windows, so a non-square map goes through the host path.
        if h != w:
            return dense_to_fmap(_as_numpy(featuremap), image_size, keypoints, keypoint_ids, patch_size, True, l2_normalize,
                                 dtype, channels_first)
        slab = _engine.extract_patches(source, np.zeros((1, 2), np.int32), h, l2_normalize, dtype, channels_first)
        return features.FeatureMap(slab, [features.kDenseId], np.zeros((1, 2), np.int32),
                                   {"scale": scale, "is_sparse": False, "patch_size": patch_size})
    corners = patch_corners(keypoints, scale, patch_size, (w, h))
    slab = _engine.extract_patches(source, corners, patch_size, l2_normalize, dtype, channels_first)
    return features.FeatureMap(slab, keypoint_ids, corners, {"scale": scale, "is_sparse": True, "patch_size": patch_size})


def dense_to_fmap(featuremap, image_size, keypoints=None, keypoint_ids=None, patch_size=16, sparse=True,
                  l2_normalize=True, dtype=np.float16, channels_first=True):
    """one dense map of one image -> FeatureMap (sparse patches or one dense patch), reference tensor_to_fmap semantics"""
    fm = _as_numpy(featuremap)
    if fm.ndim == 4 and fm.shape[0] == 1:
        fm = fm[0]
    if fm.ndim != 3:
        raise ValueError("a feature map is [C,H,W] (or [H,W,C] with channels_first=False)")
    hwc = np.moveaxis(fm, 0, -1) if channels_first else fm
    if sparse and keypoints is None:
        raise RuntimeError("Cannot run sparse feature extraction without any keypoints.")
    if keypoints is not None:
        keypoints = np.asarray(keypoints, np.float64).reshape(-1, 2)
        if keypoint_ids is None:
            keypoint_ids = list(range(len(keypoints)))
        elif len(keypoint_ids) != len(keypoints):
            raise ValueError("Number of provided keypoint_ids and keypoints do not match.")
    if l2_normalize:
        hwc = hwc / np.maximum(np.linalg.norm(hwc.astype(np.float32), axis=-1, keepdims=True), 1e-12)   # F.normalize eps
    hwc = np.ascontiguousarray(hwc, dtype=dtype)
    h, w = hwc.shape[:2]
    scale = np.array((w / image_size[0], h / image_size[1]))
    # sparse only pays off while the patches are smaller than the map they are cut from
    if sparse and sparse_pays_off(h, w, len(keypoints), patch_size):
        corners = patch_corners(keypoints, scale, patch_size, (w, h))
        return features.FeatureMap(cut_patches(hwc, corners, patch_size), keypoint_ids, corners,
                                   {"scale": scale, "is_sparse": True, "patch_size": patch_size})
    return features.FeatureMap(hwc[None], [features.kDenseId], np.zeros((1, 2), np.int32),
                               {"scale": scale, "is_sparse": False, "patch_size": patch_size})


class DenseFeatureExtractor:
    """model(image_name) -> list of [C,H,W] maps (one per level) ; image_size(image_name) -> (width, height).
    Produces the FeatureManager the adjusters take: one FeatureSet per level, one FeatureMap per image."""
    default_conf = dict(patch_size=16, sparse=True, l2_normalize=True, dtype="half", on_device=False,
                        # the dense-feature cache (reference features/extractor.py:46-49, extract.py:72-147)
                        use_cache=False, overwrite_cache=False, load_cache_on_init=False, cache_format="chunked")

    def __init__(self, model, image_size, conf=None):
        self.model, self.image_size = model, image_size
        self.conf = dict(self.default_conf, **(conf or {}))
        unknown = set(self.conf) - set(self.default_conf)
        if unknown:
            raise ValueError("unknown extractor options: %s" % sorted(unknown))
        if self.conf["dtype"] not in _DTYPES:
            raise ValueError("dtype must be one of %s" % sorted(_DTYPES))

    def features_from_image_list(self, image_dir, image_names, keypoints=None, req_keypoint_ids=None, cache_path=None,
                                 level_prefix=""):
        """extract.py:57-150.  With `use_cache` an existing cache file is taken as it is (unless `overwrite_cache`), and a
        fresh extraction is written to `cache_path` and handed back THROUGH the file — filled, or with `load_cache_on_init`
        off as metadata whose patches a FeatureView brings in per image (store_features.load_features_from_cache).  The
        file is written once all images are done (h5lite writes at close), not image by image as the reference does."""
        from . import store_features
        use_cache = bool(self.conf["use_cache"])
        if use_cache and cache_path is None:
            raise RuntimeError("Trying to write features to H5 but no path given.")
        if use_cache and self.conf["on_device"]:
            raise ValueError("use_cache stores host arrays: it cannot be combined with on_device")
        if use_cache and os.path.exists(str(cache_path)):
            if self.conf["overwrite_cache"]:
                os.unlink(str(cache_path))
            else:
                return store_features.load_features_from_cache(cache_path, bool(self.conf["load_cache_on_init"]), level_prefix)
        manager = None
        for name in image_names:
            kps, ids = None, None
            if keypoints is not None:
                kps = np.asarray(keypoints[name], np.float64)
                if req_keypoint_ids is not None:
                    ids = [int(i) for i in req_keypoint_ids[name]]
                    kps = kps[ids]
            made = self._image_fmaps(image_dir, name, kps, ids)
            if manager is None:
                manager = features.FeatureManager([m.channels for m in made], _DTYPES[self.conf["dtype"]])
            for level, fmap in enumerate(made):
                manager.fset(level).emplace(name, fmap)
        if manager is None:
            raise ValueError("no image to extract features for")
        if use_cache:
            os.makedirs(os.path.dirname(os.path.abspath(str(cache_path))), exist_ok=True)
            store_features.write_feature_manager_cache(cache_path, manager, self.conf["cache_format"], level_prefix)
            return store_features.load_features_from_cache(cache_path, bool(self.conf["load_cache_on_init"]), level_prefix)
        return manager

    def _image_fmaps(self, image_dir, name, kps, ids):
        """one FeatureMap per level of image `name`: the patches around `kps` (ids `ids`) or the dense map"""
        out = []
        for fmap in self.model(name):
            if self._on_device(kps):
                out.append(dense_to_fmap_on_device(fmap, self.image_size(name), kps, ids, self.conf["patch_size"],
                                                   self.conf["l2_normalize"], _DTYPES[self.conf["dtype"]]))
            else:
                out.append(dense_to_fmap(fmap, self.image_size(name), kps, ids, self.conf["patch_size"], self.conf["sparse"],
                                         self.conf["l2_normalize"], _DTYPES[self.conf["dtype"]]))
        return out

    def _on_device(self, kps):
        """the patches stay in device memory: asked for, and sparse patches are what is made"""
        return bool(self.conf["on_device"] and self.conf["sparse"] and kps is not None)

    def features_from_graph(self, image_dir, graph, keypoints, cache_path=None):
        """patches for the keypoints that take part in a match (reference extract.py:197-215)"""
        from ..keypoint_adjustment import extract_patchdata_from_graph
        needed = extract_patchdata_from_graph(graph)
        return self.features_from_image_list(image_dir, list(needed), keypoints, needed, cache_path)

    def features_from_reconstruction(self, reconstruction, image_dir, cache_path=None):
        """patches around the PROJECTIONS of the 3D points each image observes (reference extract.py:153-194)"""
        from ..util.cameras import world_to_image
        names, keypoints, ids = [], {}, {}
        for image in reconstruction.images.values():
            seen = [(k, p.point3D_id) for k, p in enumerate(image.points2D) if p.has_point3D()]
            if not seen:
                continue
            cam = reconstruction.cameras[image.camera_id]
            xyz = np.array([reconstruction.points3D[pid].xyz for _, pid in seen])
            kps = np.zeros((len(image.points2D), 2))
            kps[[k for k, _ in seen]] = world_to_image(cam.model_id, cam.params, image.qvec, image.tvec, xyz)
            names.append(image.name); keypoints[image.name] = kps; ids[image.name] = [k for k, _ in seen]
        return self.features_from_image_list(image_dir, names, keypoints, ids, cache_path)


class FeatureExtractor(DenseFeatureExtractor):
    """The reference's FeatureExtractor (features/extractor.py:28-236) for the models this package computes itself: dense
    SIFT (`model: {name: dsift}`, features/models/dsift.py) and S2DNet at num_layers 1 (`model: {name: s2dnet}`, the
    default; features/models/s2dnet.py, from a local weights file).  Each image is opened with PIL, resized per pyramid
    scale to `round(min(max_edge / max(w, h), 1) * size * scale)` with the `resize` filter and converted to the mode the
    model takes: grayscale ("L", what torchvision's Grayscale does) for dsift, "RGB" for s2dnet, so grayscale and RGBA
    files work too.  Each scale gives one feature level.  Sparse features come from the model's fused kernel at the
    keypoints' windows only, dense ones from the same kernel over the whole map.  Cache, `on_device` and the
    sparse-or-dense rule are DenseFeatureExtractor's.  VGG is not part of this package."""
    default_conf = dict(DenseFeatureExtractor.default_conf, device="auto", fast_image_load=False, max_edge=1600,
                        model={"name": "s2dnet"}, pyr_scales=[1.0], resize="LANCZOS")
    filters = ("BILINEAR", "BICUBIC", "LANCZOS")

    def __init__(self, conf=None):
        conf = dict(conf or {})
        model_conf = dict(self.default_conf["model"], **(conf.get("model") or {}))
        super().__init__(None, None, conf)
        self.conf["model"] = model_conf
        if model_conf.get("name") not in ("dsift", "s2dnet"):
            raise ValueError("dense feature model %r is not part of this package: only 'dsift' and 's2dnet' are computed "
                             "here — pass the FeatureManager of another model or a DenseFeatureExtractor around it"
                             % (model_conf.get("name"),))
        if self.conf["device"] not in ("auto", "cuda"):
            raise ValueError("dense features run on the GPU only (device %r)" % (self.conf["device"],))
        if self.conf["resize"] not in self.filters:
            raise ValueError("resize must be one of %s" % (self.filters,))
        if not self.conf["pyr_scales"] or any(float(s) <= 0 for s in self.conf["pyr_scales"]):
            raise ValueError("pyr_scales must be a non-empty list of positive scales")
        from .models import DSIFT, S2DNet
        self.model = (DSIFT if model_conf["name"] == "dsift" else S2DNet)(model_conf)
        self.channels_per_level = list(self.model.output_dims) * len(self.conf["pyr_scales"])

    def get_scaled_image_size(self, image, pyr_scale=1.0):
        w, h = image.size
        return [int(round(min(self.conf["max_edge"] / max(w, h), 1) * x * pyr_scale)) for x in (w, h)]

    def load_image(self, path):
        """-> ([one uint8 image per pyramid scale, [h, w] grayscale or [h, w, 3] RGB as the model takes it],
        (width, height) of the file)"""
        import PIL.Image
        image = PIL.Image.open(path)
        size = image.size
        if self.conf["fast_image_load"]:
            image.draft("RGB", self.get_scaled_image_size(image, self.conf["pyr_scales"][0]))
        levels = []
        for pyr_scale in self.conf["pyr_scales"]:
            resized = image.resize(tuple(self.get_scaled_image_size(image, pyr_scale)),
                                   getattr(PIL.Image, self.conf["resize"]))
            levels.append(np.ascontiguousarray(np.asarray(resized.convert(self.model.image_mode), np.uint8)))
        return levels, size

    def _image_fmaps(self, image_dir, name, kps, ids):
        path = name if image_dir is None else Path(image_dir) / name
        images, size = self.load_image(path)
        ps, sparse = self.conf["patch_size"], self.conf["sparse"]
        if sparse and kps is None:
            raise RuntimeError("Cannot run sparse feature extraction without any keypoints.")
        if kps is not None:
            kps = np.asarray(kps, np.float64).reshape(-1, 2)
            ids = list(range(len(kps))) if ids is None else ids
        out = []
        for image in images:
            h, w = self.model.map_size(*image.shape[:2])
            scale = np.array((w / size[0], h / size[1]))
            run = dict(patch_size=ps, l2_normalize=self.conf["l2_normalize"], dtype=self.conf["dtype"],
                       to_host=not self._on_device(kps))
            if sparse and sparse_pays_off(h, w, len(kps), ps):
                corners = patch_corners(kps, scale, ps, (w, h))
                out.append(features.FeatureMap(self.model(image, corners, **run), ids, corners,
                                               {"scale": scale, "is_sparse": True, "patch_size": ps}))
            else:
                out.append(features.FeatureMap(self.model(image, None, **run), [features.kDenseId],
                                               np.zeros((1, 2), np.int32),
                                               {"scale": scale, "is_sparse": False, "patch_size": ps}))
        return out
