"""CPU: known answers of the SIFT oracle (oracle/sift.py) -- blob localisation, descriptor norms, VLFeat's fast math against the exact functions, and (with OpenCV) homography recovery on a rendered pair."""
import math

import numpy as np
import pytest

from helpers.sift_check import TRANSPOSE_PERM, wrap
from oracle import sift as X
from pycolmap_b200 import synthetic as syn


@pytest.mark.parametrize("sigma", [2.0, 4.0, 8.0])
def test_blob(sigma):
    n = int(16 * sigma) + 32
    cx, cy = n / 2 + 0.3, n / 2 - 0.2   # in pixel-centre coordinates (+0.5 convention)
    ys, xs = np.mgrid[0:n, 0:n] + 0.5
    img = 40 + 180 * np.exp(-((xs - cx) ** 2 + (ys - cy) ** 2) / (2 * sigma ** 2))
    # first_octave -1 (the C++ default): at first_octave 0 the smallest detectable scale is 2
    r = X.extract(np.round(img).astype(np.uint8), X.defaults())
    kp = r["keypoints"]
    d = np.hypot(kp[:, 0] - cx, kp[:, 1] - cy)
    k = np.argmin(d)
    assert d[k] < 0.05 * sigma
    assert abs(kp[k, 2] / sigma - 1) < 0.2


def test_transpose_equivariance():
    """Transposing the image swaps x and y, maps the orientation to pi / 2 - theta and permutes the descriptor
    (TRANSPOSE_PERM), for all features whose decisions are not within rounding of a threshold.  All four
    orientations are kept: COLMAP keeps the first ones in bin order, and the transpose reverses that order."""
    rng = np.random.default_rng(3)
    a, _, _ = syn.homography_pair(rng, 160, 128, 256)
    o = X.pycolmap_defaults(max_num_orientations=4)
    r1, r2 = X.extract(a, o), X.extract(a.T.copy(), o)
    k1, k2 = r1["keypoints"], r2["keypoints"]
    d1, d2 = r1["descriptors"].astype(np.int64), r2["descriptors"].astype(np.int64)
    ok = tot = 0
    for i in range(len(k1)):
        if r1["margin"][i] < 1e-3:
            continue
        tot += 1
        c = np.where((np.abs(k2[:, 0] - k1[i, 1]) < 1e-2) & (np.abs(k2[:, 1] - k1[i, 0]) < 1e-2)
                     & (np.abs(k2[:, 2] - k1[i, 2]) < 1e-3 * k1[i, 2]))[0]
        c = [j for j in c if abs(wrap(math.pi / 2 - k1[i, 3] - k2[j, 3])) < 1e-3]
        ok += any(np.abs(d1[i] - d2[j][TRANSPOSE_PERM]).max() <= 2 for j in c)
    assert tot > 50 and ok >= 0.99 * tot, (ok, tot)


def test_descriptor_norms():
    rng = np.random.default_rng(1)
    a, _, _ = syn.homography_pair(rng, 160, 120, 256)
    for norm in ("L1_ROOT", "L2"):
        d = X.extract(a, X.pycolmap_defaults(normalization=norm))["descriptors"].astype(np.float64)
        assert len(d) > 20
        n = np.linalg.norm(d, axis=1)
        assert np.all(np.abs(n / 512 - 1) < 0.03), (norm, n.min(), n.max())


def test_fast_math():
    rng = np.random.default_rng(0)
    x = rng.uniform(0, 25, 100000)
    assert np.max(np.abs(X.fast_expn(x) - np.exp(-x))) < 1.5e-3  # linear interpolation, step 25 / 256
    assert X.fast_expn(np.array([30.0]))[0] == 0.0
    y, z = rng.normal(size=(2, 100000)).astype(np.float32)
    assert np.max(np.abs(X.fast_atan2_f(y, z) - np.arctan2(y, z))) < 6.5e-3  # the cubic peaks at about 6.1e-3 rad
    v = rng.uniform(1e-6, 10, 100000).astype(np.float32)
    assert np.max(np.abs(X.fast_sqrt_f(v) / np.sqrt(v) - 1)) < 1e-5
    assert X.fast_sqrt_f(np.float32(1e-9)) == 0


def test_opencv_plausibility():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(7)
    a, b, H = syn.homography_pair(rng, 320, 240, 512)
    corners = np.array([[0, 0], [320, 0], [320, 240], [0, 240]], np.float64)

    def corner_err(p1, d1, p2, d2):
        m = cv2.BFMatcher(cv2.NORM_L2, crossCheck=True).match(d1.astype(np.float32), d2.astype(np.float32))
        s = np.float32([p1[x.queryIdx] for x in m])
        t = np.float32([p2[x.trainIdx] for x in m])
        Hh, _ = cv2.findHomography(s, t, cv2.RANSAC, 2.0)
        c = np.c_[corners, np.ones(4)]
        pa, pb = c @ Hh.T, c @ H.T
        return np.max(np.linalg.norm(pa[:, :2] / pa[:, 2:] - pb[:, :2] / pb[:, 2:], axis=1))

    o = X.pycolmap_defaults()
    r1, r2 = X.extract(a, o), X.extract(b, o)
    assert corner_err(r1["keypoints"][:, :2], r1["descriptors"], r2["keypoints"][:, :2], r2["descriptors"]) < 1.0
    s = cv2.SIFT_create()
    k1, d1 = s.detectAndCompute(a, None)
    k2, d2 = s.detectAndCompute(b, None)
    p1 = np.float32([k.pt for k in k1]) + 0.5
    p2 = np.float32([k.pt for k in k2]) + 0.5
    assert corner_err(p1, d1, p2, d2) < 1.0
