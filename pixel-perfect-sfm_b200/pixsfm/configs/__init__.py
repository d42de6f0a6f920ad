"""Named configuration presets (the reference ships them as YAML files in pixsfm/configs/ and resolves names with
`parse_config_path`, configs/__init__.py:8-26).  Here a preset is a function returning the nested dict; a path to a YAML
file — the reference's own files included — is accepted wherever a preset name is."""
from copy import deepcopy
from pathlib import Path

from .. import defaults


def _default():
    return {"interpolation": defaults.interpolation(),
            "mapping": {"KA": defaults.keypoint_adjustment(), "BA": defaults.bundle_adjustment()},
            "localization": {"QKA": defaults.query_keypoint_adjustment(), "QBA": defaults.query_bundle_adjustment()}}


def _low_memory():
    """8 x 8 patches, reference keypoints per track (linear number of residuals), cost-map BA with the cameras fixed"""
    ka = dict(strategy="topological_reference", apply=True, split_in_subproblems=True, max_kps_per_problem=1000,
              optimizer=dict(num_threads=-1, print_summary=False, bound=2.0, solver=dict(parameter_tolerance=1.0e-5)))
    ba = dict(strategy="costmaps", apply=True, level_indices=None, max_tracks_per_problem=100,
              references=dict(keep_observations=False), costmaps=dict(num_threads=-1),
              optimizer=dict(loss=dict(name="cauchy", params=[0.25]), print_summary=False, refine_focal_length=False,
                             refine_principal_point=False, refine_extra_params=False, refine_extrinsics=False))
    return {"dense_features": dict(sparse=True, dtype="half", use_cache=True, overwrite_cache=True, load_cache_on_init=False,
                                   patch_size=8, cache_format="chunked"),
            "interpolation": dict(nodes=[[0.0, 0.0]], mode="BICUBIC"),
            "mapping": {"KA": ka, "BA": ba}}


def _norefine():
    return {"mapping": {"KA": dict(apply=False), "BA": dict(apply=False)}}


def _dsift():
    """dense SIFT features computed here (features/models/dsift.py): PixSfM and QueryLocalizer run from images"""
    dense = dict(model=dict(name="dsift", rootsift=True, spatial_bin_size=4), sparse=True, use_cache=False, max_edge=2000,
                 patch_size=16, device="cuda", dtype="half")
    ka = dict(apply=True, strategy="featuremetric", level_indices=None, max_kps_per_problem=50,
              optimizer=dict(print_summary=False, bound=4.0))
    ba = dict(apply=True, strategy="feature_reference", repeats=1, level_indices=None,
              optimizer=dict(solver=dict(max_num_iterations=10), print_summary=False, refine_focal_length=False,
                             refine_extra_params=False, refine_extrinsics=False))
    qka = dict(apply=True, level_indices=None, feature_inlier_thresh=-1, optimizer=dict(print_summary=False))
    qba = dict(apply=True, level_indices=None,
               optimizer=dict(print_summary=False, refine_focal_length=False, refine_extra_params=False))
    return {"dense_features": dense,
            "mapping": {"dense_features": deepcopy(dense), "KA": ka, "BA": ba},
            "localization": {"dense_features": deepcopy(dense), "target_reference": "nearest", "unique_inliers": "min_error",
                             "overwrite_features_sparse": False, "QKA": qka, "QBA": qba}}


default_configs = {"default": _default, "low_memory": _low_memory, "norefine": _norefine, "dsift": _dsift}


def parse_config_path(name_or_path):
    """-> a preset dict for a known name, a Path for an existing file, None for None"""
    if name_or_path is None:
        return None
    if name_or_path in default_configs:
        return default_configs[name_or_path]()
    path = Path(name_or_path)
    if not path.exists():
        raise FileNotFoundError("Cannot find the config file: %s. Not in the default configs %s and not an existing path."
                                % (name_or_path, sorted(default_configs)))
    return path
