from .main import (QueryKeypointAdjuster, QueryBundleAdjuster, QueryLocalizer, find_feature_inliers,  # noqa: F401
                   find_unique_inliers, find_unique_min_by_group, find_unique_min_reproj_inliers,
                   compute_reprojection_errors)
from .._pixsfm._localization import (QueryKeypointOptimizer, QueryBundleOptimizer, QueryKeypointOptimizerOptions,  # noqa: F401
                                     QueryBundleOptimizerOptions, find_nearest_references, interpolate_descriptors,
                                     absolute_pose_estimation, absolute_pose_estimation_batch)
