"""pixsfm.bundle_adjustment.main — the reference's BundleAdjuster surface (pixsfm/bundle_adjustment/main.py:12-286:
`create`, `refine_multilevel`, `refine`, `default_problem_setup`, `find_problem_labels`, same option names and values)
over the CUDA-backed extractors and optimizers."""
from .. import defaults, features
from .._pixsfm import _bundle_adjustment as ba
from ..util.conf import to_ctr
from ..util.refine import StrategyRefiner, optimizer_options

to_optim_ctr = optimizer_options      # the reference's name for it (util/misc.py:30-36)


def default_problem_setup(reconstruction):
    """all registered images; gauge: first pose constant, x translation of the second constant (main.py:12-18)"""
    registered = reconstruction.reg_image_ids()
    setup = ba.BundleAdjustmentSetup()
    setup.add_images(set(registered))
    setup.set_constant_pose(registered[0])
    setup.set_constant_tvec(registered[1], [0])
    return setup


def find_problem_labels(reconstruction, max_tracks_per_problem):
    """reference extraction fans out over labels p3D_id // max_tracks_per_problem (main.py:21-27); -1 = no such point"""
    ids = reconstruction.point3D_ids()
    labels = [-1] * (max(ids) + 1)
    for pid in ids:
        labels[pid] = int(pid // max_tracks_per_problem)
    return labels


class BundleAdjuster(StrategyRefiner):
    default_conf = defaults.bundle_adjustment()

    def refine_multilevel(self, reconstruction, feature_manager, problem_setup=None):
        """one adjustment per feature level; `reconstruction` is refined in place"""
        return self.per_level(feature_manager, lambda fset: self.refine(reconstruction, fset, problem_setup))

    def refine(self, reconstruction, feature_set, problem_setup=None):
        raise NotImplementedError()

    # pieces the strategies share
    def _reference_extractor(self, interpolation):
        return ba.ReferenceExtractor(to_ctr(self.conf.references), interpolation)

    def _optimizer_options(self):
        return optimizer_options(self.conf.optimizer, self.callbacks)


class FeatureReferenceBundleAdjuster(BundleAdjuster, strategy="feature_reference"):
    """featuremetric BA towards a fixed reference descriptor per 3D point — the default method (main.py:105-154)"""

    def refine(self, reconstruction, feature_set, problem_setup=None):
        setup = problem_setup if problem_setup is not None else default_problem_setup(reconstruction)
        interpolation = to_ctr(self.conf.interpolation)
        labels = find_problem_labels(reconstruction, self.conf.max_tracks_per_problem)
        references = self._reference_extractor(interpolation).run(labels, reconstruction, feature_set)
        optimizer = ba.FeatureReferenceBundleOptimizer(self._optimizer_options(), setup, interpolation)
        optimizer.run(reconstruction, features.FeatureView(feature_set, reconstruction), references)
        return {"references": references, "summary": optimizer.summary()}


class CostMapBundleAdjuster(BundleAdjuster, strategy="costmaps"):
    """cost-map BA (main.py:218-286): per observation the robustified featuremetric cost towards the point's reference
    and its gradient are cached as a 3-channel patch, then the interpolated cost maps are minimised — 43x less patch
    memory than 128-channel features"""
    default_conf = dict(defaults.bundle_adjustment(), costmaps=defaults.costmaps())

    def refine(self, reconstruction, feature_set, problem_setup=None):
        setup = problem_setup if problem_setup is not None else default_problem_setup(reconstruction)
        interpolation = to_ctr(self.conf.interpolation)
        labels = find_problem_labels(reconstruction, self.conf.max_tracks_per_problem)
        extractor = ba.CostMapExtractor(to_ctr(self.conf.costmaps), interpolation)
        costmap_fset, references = extractor.run(labels, reconstruction, feature_set, self._reference_extractor(interpolation))
        # cost maps are minimised as they are: no L2 normalisation of the 3 channels (main.py:262-263)
        optimizer = ba.CostMapBundleOptimizer(self._optimizer_options(), setup, dict(interpolation, l2_normalize=False))
        optimizer.run(reconstruction, features.FeatureView(costmap_fset, reconstruction))
        return {"costmaps": costmap_fset, "references": references, "summary": optimizer.summary()}


class GeometricBundleAdjuster(BundleAdjuster, strategy="geometric"):
    """classic bundle adjustment of the reprojection error between a 3D point's projection and its keypoint
    (main.py:289-313), e.g. as the baseline next to featuremetric BA or before / after it.  Needs no features."""

    def refine(self, reconstruction, *args, problem_setup=None):
        """`*args` takes the feature set `refine_multilevel` passes (unused) and, after it, a positional problem
        setup.  The reference drops that positional setup and falls back to the default one; here it is honoured, so
        `refine_multilevel(rec, fm, setup)` adjusts the same images as `refine(rec, problem_setup=setup)`.  One solve
        per call, so `refine_multilevel` runs one per feature level, as the reference does."""
        if problem_setup is None and len(args) > 1:
            problem_setup = args[1]
        setup = problem_setup if problem_setup is not None else default_problem_setup(reconstruction)
        optimizer = ba.GeometricBundleOptimizer(self._optimizer_options(), setup)
        optimizer.run(reconstruction)
        return {"summary": optimizer.summary()}
