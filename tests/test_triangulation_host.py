"""CPU: the triangulation surface of the C++ host (pycolmap_b200._core) -- EstimateTriangulationOptions with pycolmap's
Python-side defaults (R:pycolmap/estimators/triangulation.h:46-77), dict / keyword construction, the `opions`
keyword, PointData, the argument checks that come before any GPU work, and no CPU fallback."""
import math
import pickle

import numpy as np
import pytest

from helpers.native_import import load_native

nat = load_native()

CAM = dict(model=0, width=1600, height=1200, params=[1200.0, 800.0, 600.0])


def _views(n):
    pd = [nat.PointData([800.0 + i, 600.0], [i * 1e-3, 0.0]) for i in range(n)]
    rot = nat.Rotation3d([0.0, 0.0, 0.0, 1.0])
    imgs = [nat.Rigid3d(rot, [-float(i), 0.0, 0.0]) for i in range(n)]
    return pd, imgs, [CAM] * n


def test_option_defaults_match_pycolmap():
    o = nat.EstimateTriangulationOptions().todict()
    assert o == dict(min_tri_angle=0.0, ransac=dict(max_error=4.0, min_inlier_ratio=0.01, confidence=0.9999,
                                                    dyn_num_trials_multiplier=3.0, min_num_trials=1000,
                                                    max_num_trials=100000))


def test_dict_kwargs_construction_and_pickle():
    o = nat.EstimateTriangulationOptions({"min_tri_angle": 0.02, "ransac": {"max_error": 0.01}})
    assert o.min_tri_angle == 0.02 and o.ransac.max_error == 0.01 and o.ransac.min_num_trials == 1000
    k = nat.EstimateTriangulationOptions(min_tri_angle=0.5)
    assert k.min_tri_angle == 0.5 and k.ransac.max_num_trials == 100000
    assert pickle.loads(pickle.dumps(o)).todict() == o.todict()
    assert "min_tri_angle" in o.summary()
    with pytest.raises(AttributeError):
        nat.EstimateTriangulationOptions({"no_such_field": 1})


def test_point_data():
    d = nat.PointData([1.0, 2.0], [0.1, 0.2])
    assert np.array_equal(d.point, [1.0, 2.0]) and np.array_equal(d.point_normalized, [0.1, 0.2])
    with pytest.raises(AttributeError):
        d.point = [0.0, 0.0]


def test_opions_keyword():
    """The reference spells the options keyword `opions`; it is accepted (and reaches the checks) by that name."""
    pd, imgs, cams = _views(3)
    with pytest.raises(ValueError, match="Check Failed"):
        nat.estimate_triangulation(pd, imgs, cams, opions=nat.EstimateTriangulationOptions(min_tri_angle=-1.0))
    with pytest.raises(TypeError):
        nat.estimate_triangulation(pd, imgs, cams, options=nat.EstimateTriangulationOptions())


def test_single_track_checks():
    pd, imgs, cams = _views(3)
    with pytest.raises(ValueError, match="Check Failed"):          # images vs cameras
        nat.estimate_triangulation(pd, imgs, cams[:2])
    with pytest.raises(ValueError, match="Check Failed"):          # images vs point data
        nat.estimate_triangulation(pd[:2], imgs, cams)
    with pytest.raises(ValueError, match="Check Failed"):          # n < 2
        nat.estimate_triangulation(pd[:1], imgs[:1], cams[:1])
    bad = [dict(min_tri_angle=-0.1), dict(ransac=dict(max_error=0.0)), dict(ransac=dict(min_inlier_ratio=1.5)),
           dict(ransac=dict(confidence=-0.5)), dict(ransac=dict(min_num_trials=10, max_num_trials=5))]
    for b in bad:
        with pytest.raises(ValueError, match="Check Failed"):
            nat.estimate_triangulation(pd, imgs, cams, opions=nat.EstimateTriangulationOptions(b))
    with pytest.raises(ValueError, match="Check Failed"):          # neither a Rigid3d nor an image
        nat.estimate_triangulation(pd, [object()] * 3, cams)
    with pytest.raises(ValueError):                                # cameras must parse
        nat.estimate_triangulation(pd, imgs, [dict(model=99, params=[1.0])] * 3)


def test_batch_checks():
    rng = np.random.default_rng(0)
    pts = rng.normal(0, 0.1, (7, 2))
    cams = np.tile(np.c_[np.eye(3), np.zeros(3)], (4, 1, 1))
    idx = np.array([0, 1, 2, 0, 1, 2, 3])
    calls = [
        (pts, [3, 3, 1], idx, cams),           # a track shorter than 2
        (pts, [3, 3], idx, cams),              # sum(lengths) != M
        (pts, [3, 4], idx[:6], cams),          # len(image_idxs) != M
        (pts, [3, 4], idx + 1, cams),          # image index out of range
        (pts, [3, 4], idx - 1, cams),
        (pts, [3, 4], idx, cams[:, :, :3]),    # cams_from_world not I x 3 x 4
        (pts[:, :1], [3, 4], idx, cams),       # points not M x 2
    ]
    for args in calls:
        with pytest.raises(ValueError, match="Check Failed"):
            nat.estimate_triangulations(*args)
    with pytest.raises(ValueError, match="Check Failed"):
        nat.estimate_triangulations(pts, [3, 4], idx, cams, options=dict(min_tri_angle=-1.0))


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is visible")
    pd, imgs, cams = _views(3)
    with pytest.raises(Exception, match="device|CUDA|sm_90"):
        nat.estimate_triangulation(pd, imgs, cams, opions=nat.EstimateTriangulationOptions(min_tri_angle=0.0))
    pts = np.array([[0.0, 0.0], [0.1, 0.0], [0.2, 0.0]])
    cams_a = np.stack([np.c_[np.eye(3), [-float(i), 0, 0]] for i in range(3)])
    with pytest.raises(Exception, match="device|CUDA|sm_90"):
        nat.estimate_triangulations(pts, [3], [0, 1, 2], cams_a, options=dict(ransac=dict(max_error=math.radians(2))))
