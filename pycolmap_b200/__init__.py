"""pycolmap_b200 -- B200-native exhaustive feature matcher + two-view geometric verifier.

Drop-in for the hot path of pycolmap.match_exhaustive / match_sequential / verify_matches /
estimate_two_view_geometry (R:pipeline/match_features.h:219-260, R:estimators/two_view_geometry.h:95-175):
the C++ / pybind11 host (`pycolmap_b200._core`, sources in pycolmap_b200/host/) over the C ABI of
libb200match.so (include/b200match.h, hand-written sm_100a CUDA).  Same function, keyword and option names as
the reference:

    import pycolmap_b200 as pycolmap
    pycolmap.match_exhaustive(database_path, sift_options={"max_ratio": 0.8})

No CPU fallback: the import fails loudly when the extension or the CUDA library is missing, and every entry
point fails with B2M_ENODEV without an sm_90 device.
"""
try:
    from ._core import *  # noqa: F401,F403
    from ._core import (AbsolutePoseEstimationOptions, AbsolutePoseRefinementOptions,  # noqa: F401
                        absolute_pose_estimation, estimate_absolute_poses, pose_refinement)
    from ._core import (EstimateTriangulationOptions, PointData, estimate_triangulation,  # noqa: F401
                        estimate_triangulations)
    from ._core import Normalization, Sift, SiftExtractionOptions  # noqa: F401
    from ._core import PatchMatchOptions  # noqa: F401
    from ._core import StereoFusionOptions  # noqa: F401
    from ._core import CopyType, UndistortCameraOptions  # noqa: F401
    from .mvs import patch_match_stereo, stereo_fusion, undistort_images  # noqa: F401
    from ._core import (Context, Database, DatabaseTransaction, Device, ExhaustiveMatchingOptions,  # noqa: F401
                        RANSACOptions, Results, Rigid3d, Rotation3d, SequentialMatchingOptions,
                        SiftMatchingOptions, SpatialMatchingOptions, TwoViewGeometry,
                        TwoViewGeometryConfiguration, TwoViewGeometryOptions, abi_version,
                        essential_matrix_estimation, estimate_calibrated_two_view_geometry,
                        estimate_two_view_geometries, estimate_two_view_geometry,
                        estimate_two_view_geometry_pose, exhaustive_pair_blocks,
                        fundamental_matrix_estimation, has_cuda, homography_matrix_estimation,
                        image_pair_to_pair_id, match_exhaustive, match_sequential, match_spatial,
                        match_vocabtree, pair_id_to_image_pair, sequential_pairs, sqlite_version,
                        squared_sampson_error, verify_matches)
except ImportError as e:  # never fall back silently: the C++ host is a build product
    raise ImportError(
        "pycolmap_b200._core is missing or does not load: build it with "
        "`python -c 'import __graft_entry__ as g; g.build()'` (needs libb200match.so next to it)") from e

__version__ = "0.2.0"
