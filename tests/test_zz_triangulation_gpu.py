"""GPU: batched triangulation (csrc/triangulation.cu) against the CPU oracle (oracle/triangulation.py).  The sampler
enumerates pairs in a fixed order, so the decisions must be the oracle's exactly: success, the number of inliers and
the inlier mask on every track, and the number of models scored over the batch."""
import math

import numpy as np
import pytest

from helpers.native_import import load_native
from oracle import ransac as R
from oracle import triangulation as T

pytestmark = pytest.mark.gpu
nat = load_native()

DEG = math.pi / 180
N_IMAGES = 1200
# xyz agreement, relative to the distance from the point to its nearest camera: 1e-9 for ordinary tracks; the tracks
# placed near min_tri_angle (points up to a few hundred units away, seen under 0.75-3 degrees) get 1e-7.  Largest
# differences seen on an H100 over these tests: 2.1e-12 (ordinary) and 3.4e-13 (near min_tri_angle).
REL_TOL, REL_TOL_FAR = 1e-9, 1e-7


def _opts(min_tri_angle, max_error, **ransac):
    return dict(min_tri_angle=min_tri_angle, ransac=dict(max_error=max_error, **ransac))


def _run(ctx, sc, opts):
    ctx.reset_stats()
    got = ctx.estimate_triangulations(sc["points_normalized"], sc["track_lengths"], sc["image_idx"],
                                      sc["cams_from_world"], nat.EstimateTriangulationOptions(opts))
    scored = ctx.stats()["tri_models_scored"]
    want = T.estimate_triangulations(sc["points_normalized"], sc["track_lengths"], sc["image_idx"],
                                     sc["cams_from_world"], opts["min_tri_angle"], T.ransac_defaults(**opts["ransac"]))
    return got, want, scored


def _rel_xyz_err(sc, got, want):
    ok = want["success"]
    Pc = T.projection_centers(sc["cams_from_world"])
    off = np.concatenate([[0], np.cumsum(sc["track_lengths"])])
    rel = np.zeros(len(ok))
    for k in np.flatnonzero(ok):
        c = Pc[sc["image_idx"][off[k]:off[k + 1]]]
        d = np.linalg.norm(c - want["xyz"][k], axis=1).min()
        rel[k] = np.abs(got["xyz"][k] - want["xyz"][k]).max() / d
    return rel


def _assert_parity(sc, got, want, scored):
    bad = np.flatnonzero((got["success"] != want["success"]) | (got["num_inliers"] != want["num_inliers"]))
    assert len(bad) == 0, (bad[:10], got["num_inliers"][bad[:10]], want["num_inliers"][bad[:10]])
    assert np.array_equal(got["inliers"], want["inliers"])
    assert np.isnan(got["xyz"][~got["success"]]).all()
    rel = _rel_xyz_err(sc, got, want)
    far = sc["kind"] == 1
    print(f"tracks {len(rel)}, success {int(want['success'].sum())}; largest relative xyz difference: "
          f"{rel[~far].max():.2e} (ordinary), {rel[far].max() if far.any() else 0.0:.2e} (near min_tri_angle)")
    assert rel[~far].max() <= REL_TOL
    assert rel[far].max(initial=0.0) <= REL_TOL_FAR
    assert scored == want["num_models_scored"]


@pytest.mark.parametrize("min_tri_angle", [0.0, 1.5 * DEG])
@pytest.mark.parametrize("max_error", [0.5 * DEG, 2.0 * DEG])
def test_parity_with_oracle(ctx, min_tri_angle, max_error):
    rng = np.random.default_rng(int(1000 * max_error + 10 * min_tri_angle) + 7)
    L = np.r_[rng.integers(2, 65, 480), 2, 3, 31, 32, 33, 64, rng.integers(200, 1001, 3)]
    rng.shuffle(L)
    sc = T.planted_tracks(rng, L, n_images=N_IMAGES, max_error=max_error,
                          min_tri_angle=min_tri_angle if min_tri_angle > 0 else 1.5 * DEG)
    got, want, scored = _run(ctx, sc, _opts(min_tri_angle, max_error))
    _assert_parity(sc, got, want, scored)
    assert want["success"].mean() > 0.5


@pytest.mark.parametrize("min_num_trials", [45, 77, 200])
def test_abort_inside_a_round(ctx, min_num_trials):
    """C(n, 2) well above min_num_trials: the abort lands inside a round of 32 trials, after the tracks' clean
    hypotheses drove the dynamic bound below it.  The total of models scored is the oracle's."""
    rng = np.random.default_rng(min_num_trials)
    L = rng.integers(14, 90, 300)
    sc = T.planted_tracks(rng, L, n_images=N_IMAGES)
    assert (L * (L - 1) // 2 > min_num_trials).mean() > 0.8
    got, want, scored = _run(ctx, sc, _opts(1.5 * DEG, 2.0 * DEG, min_num_trials=min_num_trials))
    _assert_parity(sc, got, want, scored)
    trials = [r.num_trials for r in want["reports"]]
    assert any(t % 32 not in (0, 1) and t < min(n * (n - 1) // 2, 100000) for t, n in zip(trials, L))


def test_failures_match_the_oracle(ctx):
    """All-outlier tracks, points behind the cameras and baselines below min_tri_angle fail exactly when the oracle
    fails, in the batch and as single calls (None)."""
    rng = np.random.default_rng(11)
    L = rng.integers(2, 12, 240)
    sc = T.planted_tracks(rng, L, n_images=N_IMAGES, outlier_ratio=0.0, near_threshold_ratio=0.0,
                          near_angle_ratio=0.35, behind_ratio=0.35)
    off = np.concatenate([[0], np.cumsum(L)])
    junk = rng.random(len(L)) < 0.2     # all-outlier tracks: random rays
    for k in np.flatnonzero(junk):
        sc["points_normalized"][off[k]:off[k + 1]] = rng.uniform(-0.6, 0.6, (L[k], 2))
    opts = _opts(1.5 * DEG, 0.5 * DEG)
    got, want, scored = _run(ctx, sc, opts)
    _assert_parity(sc, got, want, scored)
    kind = sc["kind"]
    assert not want["success"][(kind == 2) & ~junk].any()
    assert (~want["success"][kind == 1]).sum() >= 5 and (~want["success"][junk]).sum() >= 5
    o = nat.EstimateTriangulationOptions(opts)
    rigid, cams = _rigids(sc["cams_from_world"])
    for k in list(np.flatnonzero(~want["success"])[:15]) + list(np.flatnonzero(want["success"])[:5]):
        s = slice(off[k], off[k + 1])
        pd = [nat.PointData(p * 1200.0, p) for p in sc["points_normalized"][s]]
        r = nat.estimate_triangulation(pd, [rigid[i] for i in sc["image_idx"][s]], [dict(model=0, params=[1200.0, 0, 0])] * L[k],
                                       opions=o)
        assert (r is None) == (not want["success"][k])


def _rigids(cams_from_world):
    """Rigid3d objects for the given matrices, and the matrices those objects give back (Rigid3d.matrix())."""
    out = []
    for P in cams_from_world:
        w, x, y, z = R.rotation_to_quat(P[:, :3])
        out.append(nat.Rigid3d(nat.Rotation3d([x, y, z, w]), P[:, 3]))
    return out, np.stack([g.matrix() for g in out])


class _Image:
    def __init__(self, g):
        self.cam_from_world = g


def test_determinism(ctx):
    rng = np.random.default_rng(12)
    L = np.r_[rng.integers(2, 70, 400), 150, 300]
    sc = T.planted_tracks(rng, L, n_images=N_IMAGES)
    rigid, cams = _rigids(sc["cams_from_world"])
    sc["cams_from_world"] = cams
    opts = nat.EstimateTriangulationOptions(_opts(1.5 * DEG, 2.0 * DEG))
    args = (sc["points_normalized"], L, sc["image_idx"], cams)
    a = ctx.estimate_triangulations(*args, opts)
    b = ctx.estimate_triangulations(*args, opts)
    for key in a:
        assert np.array_equal(a[key], b[key], equal_nan=True), key
    # permuted batch: per-track results identical
    off = np.concatenate([[0], np.cumsum(L)])
    perm = rng.permutation(len(L))
    obs = np.concatenate([np.arange(off[k], off[k + 1]) for k in perm])
    c = ctx.estimate_triangulations(sc["points_normalized"][obs], L[perm], sc["image_idx"][obs], cams, opts)
    assert np.array_equal(c["xyz"], a["xyz"][perm], equal_nan=True)
    assert np.array_equal(c["success"], a["success"][perm]) and np.array_equal(c["num_inliers"], a["num_inliers"][perm])
    assert np.array_equal(c["inliers"], a["inliers"][obs])
    # single calls equal row k of the batch, images as Rigid3d or as objects with cam_from_world
    for n, k in enumerate(list(range(6)) + [len(L) - 2, len(L) - 1]):
        s = slice(off[k], off[k + 1])
        pd = [nat.PointData(p * 1200.0, p) for p in sc["points_normalized"][s]]
        imgs = [rigid[i] if n % 2 else _Image(rigid[i]) for i in sc["image_idx"][s]]
        r = nat.estimate_triangulation(pd, imgs, [dict(model=0, params=[1200.0, 0, 0])] * L[k], opions=opts)
        assert (r is None) == (not a["success"][k])
        if r is not None:
            assert np.array_equal(r["xyz"], a["xyz"][k]) and np.array_equal(r["inliers"], a["inliers"][s])


def test_split_batch_larger_than_a_chunk(ctx):
    """A batch of more tracks than one internal chunk (32768) equals the same tracks in two separate calls."""
    rng = np.random.default_rng(13)
    L = rng.integers(2, 7, 40000)
    sc = T.planted_tracks(rng, L, n_images=N_IMAGES)
    opts = nat.EstimateTriangulationOptions(_opts(1.5 * DEG, 2.0 * DEG))
    a = ctx.estimate_triangulations(sc["points_normalized"], L, sc["image_idx"], sc["cams_from_world"], opts)
    h = 17000
    m = int(L[:h].sum())
    b1 = ctx.estimate_triangulations(sc["points_normalized"][:m], L[:h], sc["image_idx"][:m], sc["cams_from_world"], opts)
    b2 = ctx.estimate_triangulations(sc["points_normalized"][m:], L[h:], sc["image_idx"][m:], sc["cams_from_world"], opts)
    for key in ("xyz", "success", "num_inliers"):
        assert np.array_equal(a[key], np.concatenate([b1[key], b2[key]]), equal_nan=True), key
    assert np.array_equal(a["inliers"], np.concatenate([b1["inliers"], b2["inliers"]]))
    assert a["success"].mean() > 0.5
