"""CPU: the absolute pose surface of the C++ host (pycolmap_b200._core) -- option classes with pycolmap's Python-side
defaults (R:pycolmap/estimators/absolute_pose.h:97-131), dict / keyword construction, the argument checks that come
before any GPU work, and no CPU fallback."""
import numpy as np
import pytest

from helpers.native_import import load_native

nat = load_native()

CAM = dict(model=0, width=1600, height=1200, params=[1200.0, 800.0, 600.0])


def test_option_defaults_match_pycolmap():
    e = nat.AbsolutePoseEstimationOptions().todict()
    assert {k: v for k, v in e.items() if k != "ransac"} == dict(
        estimate_focal_length=False, num_focal_length_samples=30, min_focal_length_ratio=0.2, max_focal_length_ratio=5.0)
    assert e["ransac"] == dict(max_error=12.0, min_inlier_ratio=0.01, confidence=0.9999, dyn_num_trials_multiplier=3.0,
                               min_num_trials=1000, max_num_trials=100000)
    assert nat.AbsolutePoseRefinementOptions().todict() == dict(
        gradient_tolerance=1.0, max_num_iterations=100, loss_function_scale=1.0, refine_focal_length=False,
        refine_extra_params=False, print_summary=False)


def test_dict_and_kwargs_construction():
    e = nat.AbsolutePoseEstimationOptions({"estimate_focal_length": True, "ransac": {"max_error": 4.0}})
    assert e.estimate_focal_length and e.ransac.max_error == 4.0 and e.ransac.max_num_trials == 100000
    r = nat.AbsolutePoseRefinementOptions(refine_focal_length=True, max_num_iterations=7)
    assert r.refine_focal_length and r.max_num_iterations == 7 and not r.refine_extra_params
    with pytest.raises(AttributeError):
        nat.AbsolutePoseRefinementOptions({"no_such_field": 1})


def test_length_mismatch_raises_value_error():
    p2 = np.zeros((5, 2))
    p3 = np.zeros((4, 3))
    with pytest.raises(ValueError, match="Check Failed"):
        nat.absolute_pose_estimation(p2, p3, CAM)
    with pytest.raises(ValueError, match="Check Failed"):
        nat.pose_refinement(nat.Rigid3d(), p2, p3, np.ones(5, bool), CAM)
    with pytest.raises(ValueError, match="Check Failed"):
        nat.pose_refinement(nat.Rigid3d(), p2[:4], p3, np.ones(5, bool), CAM)
    with pytest.raises(ValueError, match="Check Failed"):
        nat.estimate_absolute_poses([(CAM, p2, p3)])


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is visible")
    rng = np.random.default_rng(0)
    p2, p3 = rng.uniform(0, 1000, (20, 2)), rng.uniform(-1, 1, (20, 3)) + [0, 0, 5]
    with pytest.raises(Exception, match="device|CUDA|sm_90"):
        nat.absolute_pose_estimation(p2, p3, CAM)
    with pytest.raises(Exception, match="device|CUDA|sm_90"):
        nat.estimate_absolute_poses([(CAM, p2, p3)])
