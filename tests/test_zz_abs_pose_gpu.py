"""GPU: batched absolute pose estimation and refinement (csrc/abs_pose.cu) against the CPU oracle (oracle/abs_pose.py)
on planted scenes: all eleven camera models, refinement of camera parameters and the caller's camera, covariance,
focal-length estimation, failures, batching and determinism, pose_refinement."""
import copy

import numpy as np
import pytest

from helpers.native_import import load_native
from oracle import abs_pose as A

pytestmark = pytest.mark.gpu
nat = load_native()

F, W, H = 1200.0, 1600, 1200
PARAMS = {
    0: [F, 800.0, 600.0],
    1: [F, F * 1.01, 800.0, 600.0],
    2: [F, 800.0, 600.0, 0.02],
    3: [F, 800.0, 600.0, 0.02, -0.01],
    4: [F, F, 800.0, 600.0, 0.02, -0.01, 0.001, -0.001],
    5: [F, F, 800.0, 600.0, 0.02, -0.01, 0.005, -0.002],
    6: [F, F, 800.0, 600.0, 0.02, -0.01, 0.001, -0.001, 0.002, 0.001, 0.0005, 0.0002],
    7: [F, F, 800.0, 600.0, 0.3],
    8: [F, 800.0, 600.0, 0.02],
    9: [F, 800.0, 600.0, 0.02, -0.01],
    10: [F, F, 800.0, 600.0, 0.02, -0.01, 0.001, -0.001, 0.002, 0.001, 0.0005, 0.0002],
}
# pose agreement between the GPU and the oracle: both refine from their own LO-RANSAC estimate and stop at
# gradient_tolerance = 1, so the two refined poses differ by the spread of that stopping point
ROT_TOL, T_TOL = 2e-3, 2e-2


def cam(model, params=None):
    return dict(model=model, width=W, height=H, params=list(PARAMS[model] if params is None else params))


def rot_err(qa, qb):
    Ra, Rb = A.quat_to_rotation(np.asarray(qa)), A.quat_to_rotation(np.asarray(qb))
    return float(np.arccos(np.clip((np.trace(Ra.T @ Rb) - 1) / 2, -1, 1)))


def gpu_pose(res):
    g = res["cam_from_world"]
    x, y, z, w = g.rotation.quat
    return np.array([w, x, y, z]), np.asarray(g.translation)


def jaccard(a, b):
    return (a & b).sum() / max(1, (a | b).sum())


@pytest.mark.parametrize("model", list(range(11)))
def test_planted_scene_every_camera_model(model):
    rng = np.random.default_rng(100 + model)
    c = cam(model)
    q, t, p2, p3, inl = A.planted_scene(rng, 300, c, outlier_ratio=0.3, noise_px=0.5)
    got = nat.absolute_pose_estimation(p2, p3, copy.deepcopy(c))
    want = A.absolute_pose_estimation(p2, p3, c)
    assert (got is None) == (want is None)
    assert got is not None
    assert abs(got["num_inliers"] - want["num_inliers"]) <= max(2, 0.01 * want["num_inliers"])
    assert got["num_inliers"] == int(got["inliers"].sum())
    assert jaccard(got["inliers"], inl) >= 0.99
    gq, gt = gpu_pose(got)
    assert rot_err(gq, want["qvec"]) < ROT_TOL
    assert np.linalg.norm(gt - want["tvec"]) < T_TOL * (1 + np.linalg.norm(want["tvec"]))


@pytest.mark.parametrize("model", [2, 4])
def test_refinement_of_camera_parameters_and_the_callers_camera(model):
    rng = np.random.default_rng(200 + model)
    c = cam(model)
    q, t, p2, p3, inl = A.planted_scene(rng, 600, c, outlier_ratio=0.2, noise_px=0.3)
    start = cam(model)
    start["params"][0] *= 0.97
    opts = dict(refine_focal_length=True, refine_extra_params=True)
    mine = copy.deepcopy(start)
    got = nat.absolute_pose_estimation(p2, p3, mine, refinement_options=opts)
    want = A.absolute_pose_estimation(p2, p3, start, refinement_options=A.RefinementOptions(**opts))
    assert got is not None and want is not None
    assert mine["params"] != start["params"]                      # mutated, as the reference's Camera& is
    gp, wp = np.array(mine["params"]), np.array(want["camera"]["params"])
    assert abs(gp[0] / wp[0] - 1) < 2e-3
    assert np.abs(gp[4 if model == 4 else 3:] - wp[4 if model == 4 else 3:]).max() < 5e-3
    pp = [1, 2] if model == 2 else [2, 3]
    assert all(gp[i] == start["params"][i] for i in pp)          # principal point constant
    # default options: neither the estimator nor the solver changes the camera
    untouched = copy.deepcopy(start)
    nat.absolute_pose_estimation(p2, p3, untouched)
    assert untouched["params"] == start["params"]


def test_covariance_spd_and_close_to_the_oracle():
    rng = np.random.default_rng(300)
    c = cam(0)
    q, t, p2, p3, inl = A.planted_scene(rng, 500, c, outlier_ratio=0.2, noise_px=0.5)
    got = nat.absolute_pose_estimation(p2, p3, c, return_covariance=True)
    want = A.absolute_pose_estimation(p2, p3, c, return_covariance=True)
    C, Cw = np.asarray(got["covariance"]), want["covariance"]
    assert np.allclose(C, C.T, rtol=1e-9, atol=1e-20)
    assert np.linalg.eigvalsh(C).min() > 0
    assert np.linalg.norm(C - Cw) / np.linalg.norm(Cw) < 0.05


def test_estimate_focal_length_off_by_1_7():
    rng = np.random.default_rng(400)
    c = cam(0)
    q, t, p2, p3, inl = A.planted_scene(rng, 400, c, outlier_ratio=0.2, noise_px=0.3)
    wrong = cam(0, [F / 1.7, 800.0, 600.0])
    got = nat.absolute_pose_estimation(p2, p3, wrong, estimation_options=dict(estimate_focal_length=True),
                                       refinement_options=dict(refine_focal_length=True))
    assert got is not None
    assert abs(wrong["params"][0] / F - 1) < 0.02


def test_failures_agree_with_the_oracle():
    rng = np.random.default_rng(500)
    c = cam(0)
    q, t, p2, p3, inl = A.planted_scene(rng, 50, c)
    for n in (0, 2):
        assert nat.absolute_pose_estimation(p2[:n], p3[:n], c) is None
        assert A.absolute_pose_estimation(p2[:n], p3[:n], c) is None
    # all outliers: bounded trials so that the oracle finishes
    p2o = np.c_[rng.uniform(0, W, 200), rng.uniform(0, H, 200)]
    p3o = rng.uniform(-2, 2, (200, 3)) + [0, 0, 8]
    eo = dict(ransac=dict(max_num_trials=2000))
    got = nat.absolute_pose_estimation(p2o, p3o, c, estimation_options=eo)
    o = A.EstimationOptions()
    o.ransac.max_num_trials = 2000
    want = A.absolute_pose_estimation(p2o, p3o, c, o)
    assert (got is None) == (want is None)
    if got is not None:
        assert got["num_inliers"] <= 12 and want["num_inliers"] <= 12


def test_batch_of_4097_ragged_problems():
    rng = np.random.default_rng(600)
    sizes = [0, 3, 4, 5] + [int(6 + (k * 37) % 3995) for k in range(4093)]
    c = cam(2)
    scenes = [A.planted_scene(rng, n, c, outlier_ratio=0.3, noise_px=0.5) if n else None for n in sizes]
    problems = [(c, s[2], s[3]) if s else (c, np.zeros((0, 2)), np.zeros((0, 3))) for s in scenes]
    res = nat.estimate_absolute_poses(problems)
    assert len(res) == len(sizes)
    assert res[0] is None
    for k, (n, s, r) in enumerate(zip(sizes, scenes, res)):
        if n >= 20:
            assert r is not None, k
            assert jaccard(r["inliers"], s[4]) >= 0.97, k
            assert rot_err(gpu_pose(r)[0], s[0]) < 5e-3, k
    for k in [1, 2, 3, 4, 5, 6, 100, 2000, 4096]:   # per-problem agreement with the oracle on a sample
        want = A.absolute_pose_estimation(problems[k][1], problems[k][2], c)
        assert (res[k] is None) == (want is None), k
        if want is not None:
            assert abs(res[k]["num_inliers"] - want["num_inliers"]) <= max(2, 0.01 * want["num_inliers"]), k
    # problem 0 of a batch equals the single call bit for bit; two identical calls are bit-identical
    one = nat.absolute_pose_estimation(problems[4][1], problems[4][2], c)
    again = nat.estimate_absolute_poses(problems[4:9])
    for a, b in [(one, again[0]), (res[5], nat.estimate_absolute_poses(problems)[5])]:
        assert a["num_inliers"] == b["num_inliers"] and np.array_equal(a["inliers"], b["inliers"])
        assert np.array_equal(a["cam_from_world"].matrix(), b["cam_from_world"].matrix())


def test_pose_refinement_converges_to_the_estimate():
    rng = np.random.default_rng(700)
    c = cam(4)
    q, t, p2, p3, inl = A.planted_scene(rng, 500, c, outlier_ratio=0.2, noise_px=0.5)
    est = nat.absolute_pose_estimation(p2, p3, c, refinement_options=dict(gradient_tolerance=1e-10))
    eq, et = gpu_pose(est)
    q0 = A._qplus(eq, np.array([0.01, -0.01, 0.005]))
    start = nat.Rigid3d(nat.Rotation3d([q0[1], q0[2], q0[3], q0[0]]), et + [0.05, -0.02, 0.04])
    out = nat.pose_refinement(start, p2, p3, est["inliers"], c, dict(gradient_tolerance=1e-10))
    assert out is not None
    rq, rt = gpu_pose(out)
    assert rot_err(rq, eq) < 1e-6 and np.linalg.norm(rt - et) < 1e-5
