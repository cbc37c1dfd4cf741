"""GPU: SIFT extraction (csrc/sift.cu) against the oracle (oracle/sift.py) on rendered images -- keypoints,
orientations and descriptors --, transpose equivariance, determinism, extract against extract_batch, and an end-to-end
run from pixels through match_exhaustive to the planted homography."""
import numpy as np
import pytest

from helpers.native_import import load_native
from helpers.sift_check import TRANSPOSE_PERM, groups, wrap
from oracle import sift as X
from pycolmap_b200 import synthetic as syn

nat = load_native()
pytestmark = pytest.mark.gpu

MARGIN = 1e-4   # an oracle decision this close (relative) to its threshold may go either way under rounding
# Tolerances as the H100 shows them: keypoint positions equal bit for bit (the pyramid, DoG and refinement restate
# VLFeat's arithmetic without FMA), angles differ by at most an fp32 ulp of pi, descriptors by at most 1 (the lane-order
# histogram sums round differently from VLFeat's running sum).
ANGLE_TOL = 1e-5
DESC_TOL = 1

CASES = [
    ((16, 16), dict()),
    ((97, 61), dict()),
    ((130, 257), dict(first_octave=-1)),
    ((320, 240), dict(num_octaves=9)),
    ((320, 240), dict(first_octave=-1, upright=True)),
    ((320, 240), dict(normalization="L2", max_num_orientations=4)),
    ((320, 240), dict(max_num_orientations=3)),
    ((320, 240), dict(max_num_orientations=1, max_num_features=60)),
    ((640, 480), dict()),
    ((640, 480), dict(first_octave=-1)),
    ((1600, 1200), dict()),
]


def _render(w, h, seed=0):
    rng = np.random.default_rng(seed + w * 7 + h)
    a, _, _ = syn.homography_pair(rng, w, h, 512)
    return a


def compare(gk, gd, want):
    """Pairs GPU and oracle keypoints both ways; asserts orientation counts, angles and descriptors of every pair;
    returns statistics.  Anything unpaired or different must be explained by an oracle margin < MARGIN."""
    wk, wd, wm = want["keypoints"], want["descriptors"].astype(np.int64), want["margin"]
    gd = np.round(gd * 512).astype(np.int64)
    gg, wg = groups(gk), groups(wk)
    gpos = np.array([gk[a, :3] for a, _ in gg]).reshape(-1, 3)
    used = np.zeros(len(gg), bool)
    st = dict(paired=0, unpaired=0, accepted_margin=0.0, desc=0, desc_le1=0, desc_maxdiff=0, max_dxy=0.0, max_dang=0.0)

    def accept(m):
        assert m < MARGIN, m
        st["accepted_margin"] = max(st["accepted_margin"], m)

    for a, b in wg:
        p = wk[a]
        c = np.where(~used & (np.abs(gpos[:, 0] - p[0]) < 1e-3) & (np.abs(gpos[:, 1] - p[1]) < 1e-3)
                     & (np.abs(gpos[:, 2] - p[2]) < 1e-4 * p[2]))[0] if len(gpos) else []
        if not len(c):
            st["unpaired"] += 1
            accept(wm[a])
            continue
        used[c[0]] = True
        st["paired"] += 1
        ga, gb = gg[c[0]]
        st["max_dxy"] = max(st["max_dxy"], float(np.abs(gk[ga, :2] - p[:2]).max()))
        if gb - ga != b - a:   # orientation count differs: only the 0.8-peak margin may explain it
            accept(wm[a])
            continue
        dang = np.abs(wrap(gk[ga:gb, 3].astype(np.float64) - wk[a:b, 3]))
        st["max_dang"] = max(st["max_dang"], float(dang.max()))
        assert dang.max() < ANGLE_TOL, dang
        diff = np.abs(gd[ga:gb] - wd[a:b]).max(axis=1)
        st["desc"] += len(diff)
        st["desc_le1"] += int((diff <= 1).sum())
        st["desc_maxdiff"] = max(st["desc_maxdiff"], int(diff.max()))
        assert diff.max() <= DESC_TOL, diff
    assert (~used).sum() <= max(2, 0.01 * len(wg)), "GPU keypoints without an oracle partner"
    return st


@pytest.mark.parametrize("case", range(len(CASES)))
def test_parity(case):
    (w, h), kw = CASES[case]
    img = _render(w, h, case)
    opts = X.pycolmap_defaults(**kw)
    want = X.extract(img, opts)
    gk, gd = nat.Sift(nat.SiftExtractionOptions(dict(opts))).extract(img)
    st = compare(gk, gd, want)
    n = len(groups(want["keypoints"]))
    print(f"\n{w}x{h} {kw}: oracle {len(want['keypoints'])} features / {n} keypoints, gpu {len(gk)}; {st}")
    assert st["paired"] >= 0.99 * n
    assert st["max_dxy"] == 0.0          # x, y of every paired keypoint equal the oracle's bit for bit
    assert st["desc_le1"] >= 0.99 * st["desc"]


def test_transpose_equivariance():
    img = _render(320, 240, 11)
    # all four orientations: COLMAP keeps the first ones in bin order, and the transpose reverses that order
    s = nat.Sift({"peak_threshold": 0.01, "first_octave": 0, "max_num_orientations": 4})
    k1, d1 = s.extract(img)
    k2, d2 = s.extract(img.T.copy())
    d1 = np.round(d1 * 512).astype(np.int64)
    d2 = np.round(d2 * 512).astype(np.int64)
    margin = X.extract(img, X.pycolmap_defaults(max_num_orientations=4))["margin"]
    assert len(margin) == len(k1)
    ok = tot = 0
    for i in range(len(k1)):
        if margin[i] < 1e-3:
            continue
        tot += 1
        c = np.where((np.abs(k2[:, 0] - k1[i, 1]) < 1e-2) & (np.abs(k2[:, 1] - k1[i, 0]) < 1e-2)
                     & (np.abs(k2[:, 2] - k1[i, 2]) < 1e-3 * k1[i, 2]))[0]
        c = [j for j in c if abs(wrap(np.pi / 2 - k1[i, 3] - k2[j, 3])) < 1e-3]
        ok += any(np.abs(d1[i] - d2[j][TRANSPOSE_PERM]).max() <= 2 for j in c)
    print(f"\ntranspose: {ok} / {tot} features map to their transposed partner")
    assert tot > 100 and ok >= 0.99 * tot


def test_determinism_and_batch():
    imgs = [_render(320, 240, 1), _render(97, 61, 2), _render(640, 480, 3)]
    s = nat.Sift()
    a = s.extract_batch(imgs)
    b = s.extract_batch(imgs[::-1])[::-1]
    for (k1, d1), (k2, d2), img in zip(a, b, imgs):
        assert np.array_equal(k1, k2) and np.array_equal(d1, d2)
        k3, d3 = s.extract(img)
        assert np.array_equal(k1, k3) and np.array_equal(d1, d3)
    # float32 input goes through the truncating (x * 255) cast: an exact image / 255 round-trips except where
    # x * 255 rounds below the integer, so compare against the oracle's own float path
    f = imgs[0].astype(np.float32) / np.float32(255)
    k, d = s.extract(f)
    want = X.extract(f, X.pycolmap_defaults())
    assert len(k) == len(want["keypoints"]) and len(k) > 0


def test_end_to_end_homography(tmp_path):
    """Pixels -> GPU SIFT -> database -> match_exhaustive -> PLANAR_OR_PANORAMIC; the stored inliers give back the
    planted homography within 1 px at the image corners."""
    w, h = 1024, 768
    a, b, H = syn.homography_pair(np.random.default_rng(21), w, h, 1024)
    feats = nat.Sift().extract_batch([a, b])
    path = tmp_path / "pair.db"
    with nat.Database(path) as db:
        cid = db.add_camera(0, w, h, [1.2 * max(w, h), w / 2, h / 2], True)
        ids = []
        for i, (kp, desc) in enumerate(feats):
            iid = db.add_image(f"view{i}.png", cid)
            db.write_keypoints(iid, kp.astype(np.float32))
            db.write_descriptors(iid, np.round(desc * 512).astype(np.uint8))
            ids.append(iid)
    nat.match_exhaustive(path)
    with nat.Database(path) as db:
        g = db.read_two_view_geometry(ids[0], ids[1])
    inl = np.asarray(g.inlier_matches)
    print(f"\nend to end: {len(feats[0][0])} / {len(feats[1][0])} features, config {g.config}, {len(inl)} inliers")
    assert int(g.config) == 6 and len(inl) >= 300          # PLANAR_OR_PANORAMIC
    p1 = feats[0][0][inl[:, 0], :2].astype(np.float64)
    p2 = feats[1][0][inl[:, 1], :2].astype(np.float64)
    r = nat.homography_matrix_estimation(p1, p2, nat.RANSACOptions(max_error=2.0))
    c = np.array([[0, 0, 1], [w, 0, 1], [w, h, 1], [0, h, 1]], np.float64)
    pa, pb = c @ r["H"].T, c @ H.T
    err = np.linalg.norm(pa[:, :2] / pa[:, 2:] - pb[:, :2] / pb[:, 2:], axis=1).max()
    print(f"corner error {err:.3f} px")
    assert err < 1.0
