"""GPU: a stand-alone two-view estimate is a batch of one.  `estimate_two_view_geometry` stages its problem as images
(0, 1), like problem 0 of `estimate_two_view_geometries`; RANSAC is keyed by (seed, image ids, kind, trial), so the
single call and problem 0 of any batch draw the same samples and must return the same bits."""
import numpy as np
import pytest

from helpers import scenes
from helpers.native_import import load_native
from oracle import ransac as R

nat = load_native()

pytestmark = pytest.mark.gpu

OPENCV = dict(model=4, width=1600, height=1200, has_prior_focal_length=1,
              params=[1200.0, 1200.0, 800.0, 600.0, -0.12, 0.03, 1e-3, -2e-3])


def _problems():
    rng = np.random.default_rng(17)
    out = {}
    for name, kind, n, cam in (("general", "general", 400, scenes.CAM), ("planar", "planar", 300, scenes.CAM),
                               ("rotation", "rotation", 300, scenes.CAM),
                               ("uncalibrated", "general", 250, scenes.CAM_NOPRIOR),
                               ("ten_matches", "general", 10, scenes.CAM)):
        p1, p2, _ = scenes.two_view_scene(rng, n, 0.3, kind)
        out[name] = (cam, p1, cam, p2)
    # the pixels OPENCV sees along the rays of the ideal pinhole camera (f = 1200, c = (800, 600))
    p1, p2, _ = scenes.two_view_scene(rng, 400, 0.3, "general")
    d1, d2 = (R.img_from_cam(OPENCV, (p - [800.0, 600.0]) / 1200.0) for p in (p1, p2))
    out["opencv"] = (OPENCV, d1, OPENCV, d2)
    p1, p2, _ = scenes.two_view_scene(rng, 350, 0.2, "general")
    perm = rng.permutation(350)[:300]
    out["match_list"] = (scenes.CAM, p1, scenes.CAM, p2, np.stack([perm, perm], 1).astype(np.uint32))
    out["empty"] = (scenes.CAM, np.zeros((0, 2)), scenes.CAM, np.zeros((0, 2)))
    return out


PROBLEMS = _problems()
CFG = nat.TwoViewGeometryConfiguration
WANT = {"general": CFG.CALIBRATED, "opencv": CFG.CALIBRATED, "match_list": CFG.CALIBRATED,
        "uncalibrated": CFG.UNCALIBRATED, "ten_matches": CFG.DEGENERATE, "empty": CFG.DEGENERATE}


def _assert_same(a, b):
    assert a.config == b.config
    for field in ("E", "F", "H", "inlier_matches", "num_inliers_EFH"):
        assert np.array_equal(np.asarray(getattr(a, field)), np.asarray(getattr(b, field))), field
    assert np.array_equal(a.cam2_from_cam1.matrix(), b.cam2_from_cam1.matrix())
    assert a.tri_angle == b.tri_angle


@pytest.mark.parametrize("relative_pose", [False, True], ids=["default", "relative_pose"])
@pytest.mark.parametrize("name", sorted(PROBLEMS))
def test_single_call_equals_problem_0_of_a_batch(name, relative_pose):
    opts = {"compute_relative_pose": relative_pose}
    p = PROBLEMS[name]
    other = PROBLEMS["planar" if name == "general" else "general"]
    single = nat.estimate_two_view_geometry(*p, options=opts)
    assert single.config == WANT.get(name, single.config)
    if relative_pose and name == "general":
        assert single.tri_angle > 0.0
    _assert_same(single, nat.estimate_two_view_geometries([p], opts)[0])
    _assert_same(single, nat.estimate_two_view_geometries([p, other], opts)[0])
