"""pixsfm.refine_hloc — `PixSfM` on hloc inputs (reference pixsfm/refine_hloc.py:25-146): keypoints / matches from hloc's
HDF5 files -> keypoint adjustment -> refined keypoint file -> COLMAP reconstruction or triangulation (through hloc) ->
bundle adjustment -> model on disk.

The two refinement stages are this package's (libpxr on the GPU).  The step between them — COLMAP's incremental mapper
or triangulator, which the reference reaches through `hloc.reconstruction.main` / `hloc.triangulation.main`
(refine_hloc.py:100-115) — is not part of the featuremetric path: it is called through `sfm_backend`, an object with
those two `main`-style callables (`reconstruction(model_path, image_dir, pairs_path, keypoints_path, matches_path, **args)`,
`triangulation(model_path, reference_model_path, image_dir, pairs_path, keypoints_path, matches_path, **args)`), which
defaults to hloc when it can be imported.  Without hloc, triangulation against a reference model runs on this package's
own triangulator (pixsfm.triangulation.main, same arguments); incremental mapping still raises, like the reference does
("Could not import hloc.")."""
from pathlib import Path

from . import logger
from .refine_colmap import PixSfM as PixSfM_colmap
from .util.colmap_types import Reconstruction
from .util.hloc import read_image_pairs, read_keypoints_hloc, read_matches_hloc, write_keypoints_hloc


def to_colmap_coordinates(keypoints):
    """hloc stores pixel centres at integers, COLMAP at .5 (reference util/misc.py:39-41); in place"""
    for name in keypoints.keys():
        keypoints[name] += 0.5


def to_hloc_coordinates(keypoints):
    """reference util/misc.py:44-46; in place"""
    for name in keypoints.keys():
        keypoints[name] -= 0.5


class _HlocBackend:
    """hloc.reconstruction.main / hloc.triangulation.main"""

    def __init__(self):
        import hloc.reconstruction
        import hloc.triangulation
        self.reconstruction = hloc.reconstruction.main
        self.triangulation = hloc.triangulation.main


class PixSfM(PixSfM_colmap):
    def __init__(self, conf=None, extractor=None, sfm_backend=None):
        super().__init__(conf, extractor)
        if sfm_backend is None:
            try:
                sfm_backend = _HlocBackend()
            except ImportError:
                logger.warning("Could not import hloc.")
        self.sfm_backend = sfm_backend

    def run(self, output_dir, image_dir, pairs_path, features_path, matches_path, reference_model_path=None,
            cache_path=None, feature_manager=None, **hloc_args):
        output_dir = Path(output_dir)
        output_dir.mkdir(exist_ok=True, parents=True)
        cache_path = self.resolve_cache_path(cache_path, output_dir)
        if self.conf.KA.apply:
            keypoints_path = output_dir / "refined_keypoints.h5"
            _, ka_data, feature_manager = self.refine_keypoints(keypoints_path, features_path, image_dir, pairs_path,
                                                                matches_path, cache_path=cache_path,
                                                                feature_manager=feature_manager)
        else:
            keypoints_path, ka_data = features_path, None
        model_path = self.run_reconstruction(output_dir, image_dir, pairs_path, keypoints_path, matches_path,
                                             reference_model_path, **hloc_args)
        reconstruction = Reconstruction.read(str(model_path))
        if self.conf.BA.apply:
            reconstruction, ba_data, feature_manager = self.run_ba(reconstruction, image_dir, cache_path=cache_path,
                                                                   feature_manager=feature_manager)
        else:
            ba_data = None
        reconstruction.write(str(output_dir))
        return reconstruction, {"feature_manager": feature_manager, "KA": ka_data, "BA": ba_data}

    def refine_keypoints(self, output_path, features_path, image_dir, pairs_path, matches_path, cache_path=None,
                         feature_manager=None):
        output_path = Path(output_path)
        keypoints = read_keypoints_hloc(features_path, as_cpp_map=True)
        to_colmap_coordinates(keypoints)
        pairs = read_image_pairs(pairs_path)
        matches_scores = read_matches_hloc(matches_path, pairs)
        cache_path = self.resolve_cache_path(cache_path, output_path.parent)
        keypoints, ka_data, feature_manager = self.run_ka(keypoints, image_dir, pairs, matches_scores, cache_path=cache_path,
                                                          feature_manager=feature_manager)
        to_hloc_coordinates(keypoints)
        write_keypoints_hloc(output_path, keypoints)
        return keypoints, ka_data, feature_manager

    def run_reconstruction(self, output_dir, image_dir, pairs_path, keypoints_path, matches_path, reference_model_path=None,
                           **hloc_args):
        if self.sfm_backend is None and reference_model_path is None:
            raise ValueError("Could not import hloc.")
        model_path = Path(output_dir) / "hloc"
        model_path.mkdir(exist_ok=True, parents=False)
        if self.sfm_backend is None:
            # without hloc, triangulation against the reference model runs on this package's own triangulator
            from .triangulation import main as triangulate
            triangulate(model_path, reference_model_path, image_dir, pairs_path, keypoints_path, matches_path, **hloc_args)
        elif reference_model_path is None:
            self.sfm_backend.reconstruction(model_path, image_dir, pairs_path, keypoints_path, matches_path, **hloc_args)
        else:
            self.sfm_backend.triangulation(model_path, reference_model_path, image_dir, pairs_path, keypoints_path,
                                           matches_path, **hloc_args)
        return model_path

    def triangulation(self, output_dir, reference_model_path, image_dir, pairs_path, features_path, matches_path,
                      cache_path=None, feature_manager=None, **hloc_args):
        return self.run(output_dir, image_dir, pairs_path, features_path, matches_path,
                        reference_model_path=reference_model_path, cache_path=cache_path, feature_manager=feature_manager,
                        **hloc_args)

    def reconstruction(self, output_dir, image_dir, pairs_path, features_path, matches_path, cache_path=None,
                       feature_manager=None, **hloc_args):
        return self.run(output_dir, image_dir, pairs_path, features_path, matches_path, reference_model_path=None,
                        cache_path=cache_path, feature_manager=feature_manager, **hloc_args)
