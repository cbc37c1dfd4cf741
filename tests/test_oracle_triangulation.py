"""CPU: the triangulation oracle (oracle/triangulation.py) -- planted recovery, the CombinationSampler order and the
C(n, 2) clip, min_tri_angle and cheirality, two-view agreement with OpenCV, and the fast walk against
oracle.ransac.loransac itself."""
import math

import numpy as np
import pytest

from oracle import ransac as R
from oracle import triangulation as T

DEG = math.pi / 180


def _track(sc, k):
    off = np.concatenate([[0], np.cumsum(sc["track_lengths"])])
    s = slice(off[k], off[k + 1])
    return sc["points_normalized"][s], T.pose_rows(sc["cams_from_world"], sc["image_idx"][s])


def _same_report(a, b):
    return (a.success == b.success and a.num_inliers == b.num_inliers and a.num_models_scored == b.num_models_scored
            and np.array_equal(a.inlier_mask, b.inlier_mask)
            and ((a.model is None and b.model is None) or np.array_equal(a.model, b.model)))


def test_recovers_planted_points_and_flags_outliers():
    rng = np.random.default_rng(1)
    L = rng.integers(6, 30, 80)
    sc = T.planted_tracks(rng, L, n_images=300, max_error=2 * DEG, near_threshold_ratio=0.0, near_angle_ratio=0.0,
                          behind_ratio=0.0, outlier_ratio=0.2)
    out = T.estimate_triangulations(sc["points_normalized"], L, sc["image_idx"], sc["cams_from_world"], 1.5 * DEG,
                                    T.ransac_defaults(max_error=2 * DEG))
    assert out["success"].all()
    # 0.5 px at f = 1200 from about 10 units: millimetres
    assert np.abs(out["xyz"] - sc["xyz"]).max() < 0.05
    assert not (out["inliers"] & sc["outlier"]).any()
    assert (out["inliers"] | sc["outlier"]).all()


def test_fast_walk_equals_loransac_bit_for_bit():
    """estimate_triangulation (blocked hypotheses) and loransac driven by CombinationRng give identical reports."""
    rng = np.random.default_rng(2)
    L = np.r_[rng.integers(2, 40, 50), 2, 3, 31, 32, 33, 64]
    sc = T.planted_tracks(rng, L, n_images=200)
    for min_tri_angle in (0.0, 1.5 * DEG):
        for max_error in (0.5 * DEG, 2 * DEG):
            opt = T.ransac_defaults(max_error=max_error, min_num_trials=40)
            for k in range(len(L)):
                X, Y = _track(sc, k)
                a = T.estimate_triangulation(X, Y, min_tri_angle, opt, block=7)
                b = T.loransac_reference(X, Y, min_tri_angle, opt)
                assert _same_report(a, b), (k, L[k], min_tri_angle, max_error)


def test_enumeration_order_and_pair_clip():
    n = 7
    rng = T.CombinationRng(n)
    idx = np.arange(n)
    seen = []
    for _ in range(n * (n - 1) // 2):    # loransac's partial Fisher-Yates with this generator
        for i in range(2):
            j = rng.integers(i, n)
            idx[i], idx[j] = idx[j], idx[i]
        seen.append(tuple(int(v) for v in idx[:2]))
    assert seen == [(i, j) for i in range(n) for j in range(i + 1, n)]
    opt = T.ransac_defaults()
    assert T.max_trials(n, opt) == 21
    assert T.max_trials(1000, opt) == 100000
    assert T.max_trials(1000, opt.copy(min_inlier_ratio=0.5)) == R.compute_num_trials(50000, 100000, 0.9999, 3.0, 2)


@pytest.mark.parametrize("n", [2, 3, 9, 20])
def test_trial_count_without_abort(n):
    """With an abort that cannot fire (min_num_trials = max_num_trials), every one of min(C(n, 2), bound) pairs is a
    trial and, on clean data, every one of them is scored."""
    rng = np.random.default_rng(n)
    sc = T.planted_tracks(rng, [n], n_images=50, outlier_ratio=0.0, near_threshold_ratio=0.0, near_angle_ratio=0.0,
                          behind_ratio=0.0)
    X, Y = _track(sc, 0)
    for cap in (5, 100000):
        opt = T.ransac_defaults(max_error=2 * DEG, min_num_trials=cap, max_num_trials=cap)
        rep = T.estimate_triangulation(X, Y, 0.0, opt)
        trials = min(n * (n - 1) // 2, cap)
        assert rep.num_trials == trials
        assert rep.num_models_scored >= trials     # + LO refits
        assert rep.success and rep.num_inliers == n


def test_min_tri_angle_and_cheirality_reject():
    rng = np.random.default_rng(3)
    sc = T.planted_tracks(rng, [2, 5, 12] * 20, n_images=300, outlier_ratio=0.0, near_threshold_ratio=0.0,
                          near_angle_ratio=0.5, behind_ratio=0.3)
    out = T.estimate_triangulations(sc["points_normalized"], sc["track_lengths"], sc["image_idx"], sc["cams_from_world"],
                                    1.5 * DEG, T.ransac_defaults(max_error=2 * DEG))
    kind = sc["kind"]
    assert (kind == 2).sum() >= 5 and (kind == 1).sum() >= 5
    assert not out["success"][kind == 2].any()             # behind every camera: cheirality rejects every model
    # the widest angle decides for clean near-threshold tracks
    Pc = T.projection_centers(sc["cams_from_world"])
    off = np.concatenate([[0], np.cumsum(sc["track_lengths"])])
    for k in np.flatnonzero(kind == 1):
        c = Pc[sc["image_idx"][off[k]:off[k + 1]]]
        i, j = np.triu_indices(len(c), 1)
        widest = T.pair_angles(c[i], c[j], sc["xyz"][k][None]).max()
        if widest < 1.3 * DEG:
            assert not out["success"][k]
        if widest > 1.7 * DEG:
            assert out["success"][k]
    # with min_tri_angle = 0 the near-threshold tracks all triangulate
    out0 = T.estimate_triangulations(sc["points_normalized"], sc["track_lengths"], sc["image_idx"],
                                     sc["cams_from_world"], 0.0, T.ransac_defaults(max_error=2 * DEG))
    assert out0["success"][kind == 1].all()


def test_planted_errors_straddle_the_threshold():
    rng = np.random.default_rng(4)
    me = 2 * DEG
    sc = T.planted_tracks(rng, rng.integers(2, 20, 500), n_images=100, max_error=me)
    Y = T.pose_rows(sc["cams_from_world"], sc["image_idx"])
    xyz = sc["xyz"][np.repeat(np.arange(len(sc["track_lengths"])), sc["track_lengths"])]
    P = Y[:, :12].reshape(-1, 3, 4)
    pc = np.einsum("mij,mj->mi", P[:, :, :3], xyz) + P[:, :, 3]
    ray = T.normalized_rays(sc["points_normalized"])
    err = np.arccos(np.clip((ray * pc).sum(1) / np.linalg.norm(pc, axis=1), -1, 1))
    assert ((err > 0.8 * me) & (err < 1.2 * me)).mean() >= 0.10


def test_two_view_agrees_with_opencv():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(5)
    sc = T.planted_tracks(rng, [2] * 50, n_images=200, outlier_ratio=0.0, near_threshold_ratio=0.0,
                          near_angle_ratio=0.0, behind_ratio=0.0)
    for k in range(50):
        X, Y = _track(sc, k)
        P1, P2 = Y[0, :12].reshape(3, 4), Y[1, :12].reshape(3, 4)
        h = cv2.triangulatePoints(P1, P2, X[0].reshape(2, 1), X[1].reshape(2, 1)).ravel()
        want = h[:3] / h[3]
        got = T.TriangulationEstimator(0.0).estimate(X, Y)[0]
        assert np.allclose(got, want, rtol=1e-9, atol=1e-9)


def test_check_options():
    rng = np.random.default_rng(6)
    sc = T.planted_tracks(rng, [4], n_images=10)
    X, Y = _track(sc, 0)
    with pytest.raises(ValueError, match="Check Failed"):
        T.estimate_triangulation(X, Y, -0.1)
    with pytest.raises(ValueError, match="Check Failed"):
        T.estimate_triangulation(X, Y, 0.0, T.ransac_defaults(max_error=0.0))
    with pytest.raises(ValueError, match="Check Failed"):
        T.estimate_triangulation(X, Y, 0.0, T.ransac_defaults(min_num_trials=10, max_num_trials=5))
    with pytest.raises(ValueError, match="Check Failed"):
        T.estimate_triangulation(X[:1], Y[:1])
