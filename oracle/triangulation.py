"""CPU restatement (numpy, fp64) of robust multi-view triangulation -- TEST INFRASTRUCTURE ONLY.

PARITY UNPINNED, like oracle/ransac.py: the reference binds COLMAP 3.9.1 (R:pycolmap/estimators/triangulation.h:17-77),
which is not on disk.  This file restates the published algorithms; where it and csrc/triangulation.cu disagree, this
file is the specification (SURVEY.md section 8(a) rows T1-T5):

  estimate_triangulation   <- R:pycolmap/estimators/triangulation.h:17-44 -> U:estimators/triangulation.cc
                              EstimateTriangulation: LORANSAC<TriangulationEstimator x 2, InlierSupportMeasurer,
                              CombinationSampler>, residual_type = ANGULAR_ERROR                          (T1, T2)
  CombinationRng           <- U:optim/combination_sampler.h CombinationSampler: the sample pairs (i, j), i < j, in
                              lexicographic order; at most C(n, 2) trials                                  (T3)
  TriangulationEstimator   <- U:estimators/triangulation.cc TriangulationEstimator::Estimate: two-view DLT for two
                              observations, TriangulateMultiViewPoint for more (the LO refit)              (T4)
  angular_residuals        <- U:geometry/triangulation.cc CalculateNormalizedAngularError, squared          (T5)

The LO-RANSAC control flow is oracle.ransac.loransac itself: `CombinationRng` stands in for the random generator and
steers its partial Fisher-Yates draw onto the lexicographic pair sequence, and the C(n, 2) clip of the trial bound
enters through max_num_trials (the bound is a min over both).  `estimate_triangulation` is the same walk with the
hypotheses of a block of trials computed at once (numpy is slow per call); tests/test_oracle_triangulation.py
checks that both give identical reports, bit for bit.
"""
import math

import numpy as np

from . import ransac as R

DBL_EPS = np.finfo(float).eps


def ransac_defaults(**kw):
    """pycolmap's RANSACOptions() (R:optim/bindings.h:10-18): what EstimateTriangulationOptions().ransac holds."""
    o = R.RansacOptions(max_error=4.0, min_inlier_ratio=0.01, confidence=0.9999, dyn_num_trials_multiplier=3.0,
                        min_num_trials=1000, max_num_trials=100000)
    return o.copy(**kw)


def check_options(min_tri_angle, opt):
    """EstimateTriangulationOptions::Check / RANSACOptions::Check (U:estimators/triangulation.h, U:optim/ransac.h)."""
    if not min_tri_angle >= 0:
        raise ValueError("Check Failed: min_tri_angle >= 0")
    if not opt.max_error > 0:
        raise ValueError("Check Failed: max_error > 0")
    if not 0 <= opt.min_inlier_ratio <= 1:
        raise ValueError("Check Failed: min_inlier_ratio in [0, 1]")
    if not 0 <= opt.confidence <= 1:
        raise ValueError("Check Failed: confidence in [0, 1]")
    if not opt.min_num_trials <= opt.max_num_trials:
        raise ValueError("Check Failed: min_num_trials <= max_num_trials")


def projection_centers(cams_from_world):
    """-R^T t of each [3 x 4] cam_from_world matrix (what the library computes from the given matrices)."""
    P = np.asarray(cams_from_world, np.float64).reshape(-1, 3, 4)
    return -np.einsum("kji,kj->ki", P[:, :, :3], P[:, :, 3])


def pose_rows(cams_from_world, image_idx=None):
    """Y rows of the estimator: the 12 entries of P (row-major) followed by the projection centre."""
    P = np.asarray(cams_from_world, np.float64).reshape(-1, 3, 4)
    Y = np.concatenate([P.reshape(-1, 12), projection_centers(P)], 1)
    return Y if image_idx is None else Y[np.asarray(image_idx)]


def normalized_rays(X):
    """normalize((u, v, 1)) per observation, Eigen's normalized(): v / sqrt(squaredNorm)."""
    X = np.asarray(X, np.float64)
    nrm = np.sqrt(X[:, 0] * X[:, 0] + X[:, 1] * X[:, 1] + 1.0)
    return np.stack([X[:, 0] / nrm, X[:, 1] / nrm, 1.0 / nrm], 1)


def angular_residuals(X, Y, xyz, rays=None):
    """acos(normalize((u, v, 1)) . normalize(P X~))^2 per observation; NaN (an outlier) when the cosine rounds above 1.
    xyz: (3,) -> (n,) residuals, or (K, 3) -> (K, n).  Element-wise arithmetic only, so both shapes give the same bits."""
    r = normalized_rays(X) if rays is None else rays
    xyz = np.asarray(xyz, np.float64)
    x, y, z = xyz[..., 0, None], xyz[..., 1, None], xyz[..., 2, None]
    px = Y[:, 0] * x + Y[:, 1] * y + Y[:, 2] * z + Y[:, 3]
    py = Y[:, 4] * x + Y[:, 5] * y + Y[:, 6] * z + Y[:, 7]
    pz = Y[:, 8] * x + Y[:, 9] * y + Y[:, 10] * z + Y[:, 11]
    nrm = np.sqrt(px * px + py * py + pz * pz)
    with np.errstate(invalid="ignore", divide="ignore"):
        c = r[:, 0] * (px / nrm) + r[:, 1] * (py / nrm) + r[:, 2] * (pz / nrm)
        a = np.arccos(c)
    return a * a


def depths(Y, xyz):
    """HasPointPositiveDepth's P.row(2) . X~ per view."""
    xyz = np.asarray(xyz, np.float64)
    x, y, z = xyz[..., 0, None], xyz[..., 1, None], xyz[..., 2, None]
    return Y[:, 8] * x + Y[:, 9] * y + Y[:, 10] * z + Y[:, 11]


def pair_angles(c1, c2, X):
    """oracle.ransac.triangulation_angles element-wise over rows of c1, c2, X (the clipped min(theta, pi - theta))."""
    b2 = ((c1 - c2) ** 2).sum(-1)
    r1, r2 = ((X - c1) ** 2).sum(-1), ((X - c2) ** 2).sum(-1)
    den = 2.0 * np.sqrt(r1 * r2)
    ok = den > 0
    with np.errstate(invalid="ignore", divide="ignore"):
        ang = np.abs(np.arccos(np.clip(np.where(ok, (r1 + r2 - b2) / np.where(ok, den, 1.0), 1.0), -1.0, 1.0)))
    ang = np.where(ok, ang, 0.0)
    return np.minimum(ang, np.pi - ang)


def dlt_matrices(X, Y, i, j):
    """The 4 x 4 DLT of TriangulatePoint (U:geometry/triangulation.cc) for the pairs (i[k], j[k]): [K x 4 x 4]."""
    P1, P2 = Y[i, :12].reshape(-1, 3, 4), Y[j, :12].reshape(-1, 3, 4)
    x1, x2 = X[i], X[j]
    return np.stack([x1[:, 0, None] * P1[:, 2] - P1[:, 0], x1[:, 1, None] * P1[:, 2] - P1[:, 1],
                     x2[:, 0, None] * P2[:, 2] - P2[:, 0], x2[:, 1, None] * P2[:, 2] - P2[:, 1]], 1)


def triangulate_multiview(X, Y):
    """TriangulateMultiViewPoint: the eigenvector of the smallest eigenvalue of sum term^T term, term = P - x x^T P."""
    r = normalized_rays(X)
    P = Y[:, :12].reshape(-1, 3, 4)
    term = P - r[:, :, None] * np.einsum("ki,kij->kj", r, P)[:, None, :]
    A = np.einsum("kij,kil->jl", term, term)
    v = np.linalg.eigh(A)[1][:, 0]
    return v[:3] / v[3]


class TriangulationEstimator:
    """TriangulationEstimator (U:estimators/triangulation.cc) with the ANGULAR_ERROR residual.
    X: [n x 2] normalised points; Y: [n x 15] pose rows (pose_rows)."""
    kMinNumSamples = 2

    def __init__(self, min_tri_angle=0.0):
        self.min_tri_angle = float(min_tri_angle)

    def estimate(self, X, Y):
        X, Y = np.asarray(X, np.float64), np.asarray(Y, np.float64)
        n = len(X)
        if n == 2:
            xyz = R.triangulate_point(Y[0, :12].reshape(3, 4), Y[1, :12].reshape(3, 4), X[0], X[1])
            if (depths(Y, xyz) >= DBL_EPS).all() and \
                    R.triangulation_angles(Y[0, 12:], Y[1, 12:], xyz)[0] >= self.min_tri_angle:
                return [xyz]
            return []
        xyz = triangulate_multiview(X, Y)
        if not (depths(Y, xyz) >= DBL_EPS).all():
            return []
        # some pair (i, j < i) with angle >= min_tri_angle; the loop order does not change the outcome
        i, j = np.tril_indices(n, -1)
        if (pair_angles(Y[i, 12:], Y[j, 12:], xyz[None, :]) >= self.min_tri_angle).any():
            return [xyz]
        return []

    @staticmethod
    def residuals(X, Y, xyz):
        return angular_residuals(X, Y, xyz)


class CombinationRng:
    """Drives oracle.ransac.loransac's partial Fisher-Yates draw (`rng.integers(i, n)` on a persistent index vector)
    so that trial k samples the k-th pair of the lexicographic sequence (0, 1), (0, 2), ..., (1, 2), ...: the
    CombinationSampler (U:optim/combination_sampler.h) without touching loransac."""

    def __init__(self, n):
        self.n = n
        self.idx = np.arange(n)        # mirrors loransac's index vector
        self.pairs = zip(*np.triu_indices(n, 1))
        self.pending = []

    def integers(self, lo, hi):
        if lo == 0:
            self.pending = list(next(self.pairs))
        target = self.pending[lo]
        pos = int(np.flatnonzero(self.idx == target)[0])
        assert lo <= pos < hi
        self.idx[lo], self.idx[pos] = self.idx[pos], self.idx[lo]
        return pos


def max_trials(n, opt):
    """min(max_num_trials, trials needed at min_inlier_ratio, C(n, 2)) (T3)."""
    return min(opt.max_num_trials,
               R.compute_num_trials(int(opt.min_inlier_ratio * 100000), 100000, opt.confidence,
                                    opt.dyn_num_trials_multiplier, 2),
               n * (n - 1) // 2)


def loransac_reference(X, Y, min_tri_angle=0.0, ransac=None):
    """EstimateTriangulation through oracle.ransac.loransac verbatim (slow; the yardstick of the fast walk)."""
    opt = ransac or ransac_defaults()
    n = len(X)
    est = TriangulationEstimator(min_tri_angle)
    o = opt.copy(max_num_trials=min(opt.max_num_trials, n * (n - 1) // 2))
    return R.loransac(est, est, np.asarray(X, np.float64), np.asarray(Y, np.float64), o, CombinationRng(n))


def estimate_triangulation(X, Y, min_tri_angle=0.0, ransac=None, block=256):
    """EstimateTriangulation over one track: X [n x 2] normalised points, Y [n x 15] pose rows.  Returns a
    ransac.Report (success, num_inliers, model = xyz, inlier_mask, num_models_scored, num_trials).

    The walk of oracle.ransac.loransac, trial by trial in the same order, with the two-view hypotheses of `block`
    consecutive trials and their residuals computed at once."""
    opt = ransac or ransac_defaults()
    check_options(min_tri_angle, opt)
    X, Y = np.asarray(X, np.float64), np.asarray(Y, np.float64)
    n = len(X)
    if n < 2:
        raise ValueError("Check Failed: point_data.size() >= 2")
    est = TriangulationEstimator(min_tri_angle)
    rays = normalized_rays(X)
    rep = R.Report()
    rep.inlier_mask = np.zeros(n, bool)
    K = int(max_trials(n, opt))
    max_residual = opt.max_error * opt.max_error
    dyn_max = K
    best = (0, float("inf"))
    best_model = None
    ii, jj = np.triu_indices(n, 1)
    trial, abort = 0, False
    while trial < K and not abort:
        k1 = min(K, trial + block)
        i, j = ii[trial:k1], jj[trial:k1]
        A = dlt_matrices(X, Y, i, j)
        V = np.linalg.svd(A)[2][:, 3]
        xyz = V[:, :3] / V[:, 3:]
        d_i = (Y[i, 8] * xyz[:, 0] + Y[i, 9] * xyz[:, 1] + Y[i, 10] * xyz[:, 2] + Y[i, 11])
        d_j = (Y[j, 8] * xyz[:, 0] + Y[j, 9] * xyz[:, 1] + Y[j, 10] * xyz[:, 2] + Y[j, 11])
        ok = (d_i >= DBL_EPS) & (d_j >= DBL_EPS) & (pair_angles(Y[i, 12:], Y[j, 12:], xyz) >= est.min_tri_angle)
        res = angular_residuals(X, Y, xyz, rays)
        with np.errstate(invalid="ignore"):
            inl = res <= max_residual
        cnt = inl.sum(1)
        for b in range(k1 - trial):
            t = trial + b
            if ok[b]:
                rep.num_models_scored += 1
                if cnt[b] >= best[0]:
                    sup = (int(cnt[b]), float(res[b][inl[b]].sum()))
                    if R._better(sup, best):
                        best, best_model = sup, xyz[b]
                        if sup[0] > 2:
                            best, best_model = _local_optimization(est, X, Y, res[b], best, best_model, max_residual,
                                                                   rep)
                        dyn_max = R.compute_num_trials(best[0], n, opt.confidence, opt.dyn_num_trials_multiplier, 2)
                if t >= dyn_max and t >= opt.min_num_trials:
                    abort = True
                    trial = t + 1
                    break
        if not abort:
            trial = k1
    rep.num_trials = trial
    rep.num_inliers, rep.residual_sum, rep.model = best[0], best[1], best_model
    if best[0] < 2 or best_model is None:
        return rep
    rep.success = True
    with np.errstate(invalid="ignore"):
        rep.inlier_mask = est.residuals(X, Y, best_model) <= max_residual
    return rep


def _local_optimization(est, X, Y, res, best, best_model, max_residual, rep):
    """The up-to-10 LO rounds of LORANSAC::Estimate (oracle.ransac.loransac), multi-view refits on the inliers."""
    for _ in range(10):
        with np.errstate(invalid="ignore"):
            inl = res <= max_residual
        prev = best[0]
        best_local_res = None
        for lm in est.estimate(X[inl], Y[inl]):
            lres = est.residuals(X, Y, lm)
            rep.num_models_scored += 1
            lsup = R._support(lres, max_residual)
            if R._better(lsup, best):
                best, best_model, best_local_res = lsup, lm, lres
        if best[0] <= prev:
            break
        res = best_local_res
    return best, best_model


def estimate_triangulations(points_normalized, track_lengths, image_idx, cams_from_world, min_tri_angle=0.0,
                            ransac=None):
    """The batched form (pycolmap_b200.estimate_triangulations): dict of xyz (NaN rows on failure), success,
    num_inliers, inliers, and the total num_models_scored."""
    X = np.asarray(points_normalized, np.float64).reshape(-1, 2)
    L = np.asarray(track_lengths, np.int64)
    Y = pose_rows(cams_from_world, image_idx)
    T = len(L)
    off = np.concatenate([[0], np.cumsum(L)])
    out = dict(xyz=np.full((T, 3), np.nan), success=np.zeros(T, bool), num_inliers=np.zeros(T, np.int64),
               inliers=np.zeros(len(X), bool), num_models_scored=0, reports=[])
    for k in range(T):
        s = slice(off[k], off[k + 1])
        rep = estimate_triangulation(X[s], Y[s], min_tri_angle, ransac)
        out["reports"].append(rep)
        out["num_models_scored"] += rep.num_models_scored
        out["num_inliers"][k] = rep.num_inliers
        if rep.success:
            out["success"][k] = True
            out["xyz"][k] = rep.model
            out["inliers"][s] = rep.inlier_mask
    return out


# ---------------------------------------------------------------------------------------------
# planted scenes (tests and tools/bench_triangulation.py)
# ---------------------------------------------------------------------------------------------
def look_at(center, target=(0.0, 0.0, 0.0)):
    """cam_from_world [3 x 4] of a camera at `center` looking at `target` (+z forward)."""
    c = np.asarray(center, np.float64)
    z = np.asarray(target, np.float64) - c
    z /= np.linalg.norm(z)
    x = np.cross([0.0, 0.0, 1.0], z)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    Rm = np.stack([x, y, z])
    return np.concatenate([Rm, (-Rm @ c)[:, None]], 1)


def _perturb_rays(rng, d, theta):
    """Rotate unit rays d [m x 3] by angles theta [m] towards random perpendicular directions."""
    e = rng.normal(size=d.shape)
    e -= (e * d).sum(1, keepdims=True) * d
    e /= np.linalg.norm(e, axis=1, keepdims=True)
    return np.cos(theta)[:, None] * d + np.sin(theta)[:, None] * e


def planted_tracks(rng, lengths, n_images=1000, max_error=math.radians(2.0), min_tri_angle=math.radians(1.5),
                   noise_px=0.5, focal=1200.0, outlier_ratio=0.1, near_threshold_ratio=0.12, near_angle_ratio=0.1,
                   behind_ratio=0.03):
    """Planted tracks seen by a ring of `n_images` cameras (radius 10, heights in [-2, 2]) that look at the origin.

    - Every track observes distinct images, (s + j * step) mod n_images, so lengths must not exceed n_images.
    - Points lie within 2 units of the origin; observations carry `noise_px` of pixel noise at `focal`.
    - `outlier_ratio` of the observations are gross outliers (5 to 50 x max_error off the true ray) and
      `near_threshold_ratio` sit 0.8 to 1.2 x max_error off it, so that the <= test and LO decide real cases.
    - `near_angle_ratio` of the tracks use neighbouring cameras and a point placed so that the widest pair angle is
      0.5 to 2 x min_tri_angle (1.5 degrees when min_tri_angle is 0).
    - `behind_ratio` of the tracks have their point behind all their cameras (observations are consistent
      projections of it, so only the cheirality test rejects them).

    Returns dict(points_normalized [M x 2], track_lengths [T], image_idx [M], cams_from_world [I x 3 x 4],
    xyz [T x 3] (truth), outlier [M] (gross outliers), kind [T] (0 normal, 1 near min_tri_angle, 2 behind))."""
    L = np.asarray(lengths, np.int64)
    T, I = len(L), int(n_images)
    if (L > I).any() or (L < 2).any():
        raise ValueError("track lengths must lie in [2, n_images]")
    phi = 2 * np.pi * np.arange(I) / I
    centers = np.stack([10 * np.cos(phi), 10 * np.sin(phi), rng.uniform(-2, 2, I)], 1)
    cams = np.stack([look_at(c, rng.uniform(-0.5, 0.5, 3)) for c in centers])
    off = np.concatenate([[0], np.cumsum(L)])
    M = int(off[-1])
    kind = np.zeros(T, np.int64)
    u = rng.random(T)
    kind[u < near_angle_ratio + behind_ratio] = 1
    kind[u < behind_ratio] = 2
    # images: start + j * step (mod I); normal tracks spread over the ring, the others use neighbouring cameras
    start = rng.integers(0, I, T)
    step = np.where(kind == 0, np.maximum(1, (rng.random(T) * (I // np.maximum(L, 1))).astype(np.int64)), 1)
    track_of = np.repeat(np.arange(T), L)
    j = np.arange(M) - off[track_of]
    image_idx = ((start[track_of] + j * step[track_of]) % I).astype(np.int32)
    # points
    xyz = rng.uniform(-2, 2, (T, 3))
    first, last = image_idx[off[:-1]], image_idx[off[1:] - 1]
    mid = 0.5 * (centers[first] + centers[last])
    chord = np.linalg.norm(centers[first] - centers[last], axis=1)
    inward = -mid / np.linalg.norm(mid, axis=1, keepdims=True)
    target = (min_tri_angle if min_tri_angle > 0 else math.radians(1.5)) * np.exp(rng.uniform(np.log(0.5), np.log(2.0), T))
    dist = chord / (2 * np.tan(target / 2))
    xyz = np.where((kind == 1)[:, None], mid + inward * dist[:, None], xyz)
    xyz = np.where((kind == 2)[:, None], mid - inward * rng.uniform(1, 5, T)[:, None], xyz)
    # observations: exact rays, pixel noise, planted angular errors
    P = cams[image_idx]
    Xw = xyz[track_of]
    pc = np.einsum("mij,mj->mi", P[:, :, :3], Xw) + P[:, :, 3]
    d = pc / np.linalg.norm(pc, axis=1, keepdims=True)
    v = rng.random(M)
    outlier = v < outlier_ratio
    near = (v >= outlier_ratio) & (v < outlier_ratio + near_threshold_ratio)
    theta = np.zeros(M)
    theta[outlier] = max_error * rng.uniform(5, 50, outlier.sum())
    theta[near] = max_error * rng.uniform(0.8, 1.2, near.sum())
    d = np.where((outlier | near)[:, None], _perturb_rays(rng, d, theta), d)
    pts = d[:, :2] / d[:, 2:]
    pts = pts + rng.normal(0, noise_px / focal, (M, 2))
    return dict(points_normalized=pts, track_lengths=L, image_idx=image_idx, cams_from_world=cams, xyz=xyz,
                outlier=outlier, kind=kind)
