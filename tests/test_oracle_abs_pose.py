"""CPU: the numpy restatement of absolute pose estimation and refinement (oracle/abs_pose.py, SURVEY.md rows A1-A5)
on planted scenes, and OpenCV's solvePnPRansac as an independent plausibility check."""
import numpy as np
import pytest

from oracle import abs_pose as A
from oracle import ransac as R

CAM = dict(model=0, width=1600, height=1200, params=[1200.0, 800.0, 600.0])


def _rot_err(Ra, Rb):
    return float(np.arccos(np.clip((np.trace(Ra.T @ Rb) - 1) / 2, -1, 1)))


def test_p3p_contains_the_planted_pose():
    rng = np.random.default_rng(1)
    q, t, p2, p3, _ = A.planted_scene(rng, 60, CAM)
    x = R.cam_from_img(CAM, p2)
    Pt = np.c_[A.quat_to_rotation(q), t]
    err = []
    for _ in range(100):
        s = rng.choice(60, 3, replace=False)
        models = A.P3PEstimator.estimate(x[s], p3[s])
        assert 1 <= len(models) <= 4
        err.append(min(np.abs(m - Pt).max() for m in models))
    # a triple whose quartic has a near-double root is ill-conditioned (about 1 in 100 random triples here): the
    # planted pose is then only found to ~1e-5
    err = np.array(err)
    assert (err < 1e-9).mean() >= 0.97 and err.max() < 1e-4, np.sort(err)[-5:]


def test_epnp_noise_free():
    rng = np.random.default_rng(2)
    q, t, p2, p3, _ = A.planted_scene(rng, 40, CAM)
    x = R.cam_from_img(CAM, p2)
    Pt = np.c_[A.quat_to_rotation(q), t]
    for n in (6, 12, 40):
        (m,) = A.EPNPEstimator.estimate(x[:n], p3[:n])
        assert np.abs(m - Pt).max() < 1e-9


def test_loransac_recovers_the_planted_mask():
    rng = np.random.default_rng(3)
    q, t, p2, p3, inl = A.planted_scene(rng, 400, CAM, outlier_ratio=0.3, noise_px=0.5)
    est = A.estimate_absolute_pose(p2, p3, CAM)
    assert est.success
    jac = (est.inlier_mask & inl).sum() / (est.inlier_mask | inl).sum()
    assert jac >= 0.99, jac
    assert _rot_err(est.P[:, :3], A.quat_to_rotation(q)) < 2e-3


def test_refinement_lowers_the_robust_cost_and_lands_on_the_planted_pose():
    rng = np.random.default_rng(4)
    q, t, p2, p3, inl = A.planted_scene(rng, 400, CAM, outlier_ratio=0.2, noise_px=0.5)
    q0 = A._qplus(q, np.array([0.01, -0.008, 0.012]))
    t0 = t + np.array([0.05, -0.03, 0.08])
    ref = A.refine_absolute_pose(q0, t0, p2, p3, inl, CAM, covariance=True)
    assert ref.success
    assert A.robust_cost(ref.qvec, ref.tvec, p2, p3, inl, CAM) < A.robust_cost(q0, t0, p2, p3, inl, CAM)
    # sigma = 0.5 px over 320 points at 4-10 m: the planted pose is within ~1e-3 rad / 1 cm of the optimum
    assert _rot_err(A.quat_to_rotation(ref.qvec), A.quat_to_rotation(q)) < 1e-3
    assert np.linalg.norm(ref.tvec - t) < 1e-2
    C = ref.covariance
    assert np.allclose(C, C.T, rtol=1e-8, atol=1e-18) and np.linalg.eigvalsh(C).min() > 0


def test_refinement_of_camera_parameters():
    rng = np.random.default_rng(5)
    cam = dict(model=2, width=1600, height=1200, params=[1200.0, 800.0, 600.0, 0.03])
    q, t, p2, p3, inl = A.planted_scene(rng, 500, cam, noise_px=0.3)
    start = dict(cam, params=[1150.0, 800.0, 600.0, 0.0])
    ref = A.refine_absolute_pose(q, t, p2, p3, inl, start,
                                 A.RefinementOptions(refine_focal_length=True, refine_extra_params=True,
                                                     gradient_tolerance=1e-8))
    assert ref.success
    assert abs(ref.params[0] - 1200.0) < 5.0 and abs(ref.params[3] - 0.03) < 3e-3
    assert ref.params[1] == 800.0 and ref.params[2] == 600.0      # the principal point stays constant


def test_focal_length_estimation_with_focal_off_by_1_7():
    rng = np.random.default_rng(6)
    q, t, p2, p3, inl = A.planted_scene(rng, 150, CAM, outlier_ratio=0.2, noise_px=0.3)
    wrong = dict(CAM, params=[1200.0 / 1.7, 800.0, 600.0])
    opt = A.EstimationOptions(estimate_focal_length=True)
    opt.ransac.min_num_trials = 200
    res = A.absolute_pose_estimation(p2, p3, wrong, opt, A.RefinementOptions(refine_focal_length=True))
    assert res is not None
    assert abs(res["camera"]["params"][0] / 1200.0 - 1.0) < 0.02


def test_too_few_correspondences_fail():
    rng = np.random.default_rng(7)
    _, _, p2, p3, _ = A.planted_scene(rng, 10, CAM)
    for n in (0, 2):
        assert A.absolute_pose_estimation(p2[:n], p3[:n], CAM) is None


def test_agrees_with_opencv_solvepnpransac():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(8)
    K = np.array([[1200.0, 0, 800.0], [0, 1200.0, 600.0], [0, 0, 1]])
    for _ in range(3):
        q, t, p2, p3, inl = A.planted_scene(rng, 300, CAM, outlier_ratio=0.3, noise_px=0.5)
        ok, rvec, tvec, cv_inl = cv2.solvePnPRansac(p3, p2, K, None, reprojectionError=12.0, iterationsCount=2000,
                                                     confidence=0.9999, flags=cv2.SOLVEPNP_EPNP)
        assert ok
        res = A.absolute_pose_estimation(p2, p3, CAM)
        assert res is not None
        Rcv, _ = cv2.Rodrigues(rvec)
        assert _rot_err(Rcv, A.quat_to_rotation(res["qvec"])) < 5e-3
        assert np.linalg.norm(tvec.ravel() - res["tvec"]) < 0.05 * (1 + np.linalg.norm(t))
        mask_cv = np.zeros(len(p2), bool)
        mask_cv[cv_inl.ravel()] = True
        assert (mask_cv & res["inliers"]).sum() / (mask_cv | res["inliers"]).sum() > 0.97
