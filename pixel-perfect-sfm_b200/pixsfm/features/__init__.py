"""pixsfm.features — the feature containers consumed by the hot path (reference pixsfm/features/bindings.cc:38-300) and
the step that fills them from dense feature maps (features/extractor.py), and FeatureExtractor for the models computed
here: dense SIFT (models/dsift.py) and S2DNet at num_layers 1 (models/s2dnet.py); VGG is not included."""
from .._pixsfm._features import (FeaturePatch, FeatureMap, FeatureSet, FeatureView, FeatureManager,  # noqa: F401
                                 Reference, PatchInterpolator, kDenseId)
from .extractor import (DenseFeatureExtractor, FeatureExtractor, dense_to_fmap, dense_to_fmap_on_device, patch_corners,  # noqa: F401
                        cut_patches)

from . import extract_patches, store_features, store_references  # noqa: F401,E402  (features/__init__.py:2 of the reference)

Map_IdReference = dict
