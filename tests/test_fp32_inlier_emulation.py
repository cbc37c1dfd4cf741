"""CPU emulation of the division-free fp32 inlier test of the two-view verifier (verify.cu inlier_f32 and
ransac_common.cuh classify_f32) against the fp64 residual, at the image sizes and thresholds where DESIGN.md states
that its confident decisions equal fp64.

The emulation uses fp32 operands, fmaf as the fp64 product-sum of the fp32 operands rounded to fp32, and the 0.99 /
1.01 band.  Points are placed 0.5-5 % off the threshold of a planted model (H: transfer error; F: perpendicular to the
epipolar line).  A decision counts as wrong when it is confident (in or out, not borderline) and differs from fp64.
Outside the tested range the H arm does go wrong (20 000 px at 0.25 px, 40 000 px at <= 0.5 px): it scores raw pixel
coordinates, so ex = x2 w - u cancels."""
import numpy as np
import pytest

F32 = np.float32
OFFSETS = np.array([0.95, 0.97, 0.985, 0.995, 1.005, 1.015, 1.03, 1.05])


def fma(a, b, c):
    return F32(np.float64(a) * np.float64(b) + np.float64(c))


def classify(lhs, rhs):
    """1 clearly in, 0 clearly out, 2 borderline (classify_f32)."""
    return np.where(lhs < F32(0.99) * rhs, 1, np.where(lhs > F32(1.01) * rhs, 0, 2))


def h_f32(M, x1, y1, x2, y2, thr):
    M, x1, y1, x2, y2, thr = M.astype(F32), x1.astype(F32), y1.astype(F32), x2.astype(F32), y2.astype(F32), F32(thr)
    u = fma(M[0], x1, fma(M[1], y1, M[2]))
    v = fma(M[3], x1, fma(M[4], y1, M[5]))
    w = fma(M[6], x1, fma(M[7], y1, M[8]))
    ex, ey = fma(x2, w, -u), fma(y2, w, -v)
    return classify(fma(ex, ex, ey * ey), thr * w * w)


def f_f32(M, x1, y1, x2, y2, thr):
    M, x1, y1, x2, y2, thr = M.astype(F32), x1.astype(F32), y1.astype(F32), x2.astype(F32), y2.astype(F32), F32(thr)
    a0 = fma(M[0], x1, fma(M[1], y1, M[2]))
    a1 = fma(M[3], x1, fma(M[4], y1, M[5]))
    a2 = fma(M[6], x1, fma(M[7], y1, M[8]))
    b0 = fma(M[0], x2, fma(M[3], y2, M[6]))
    b1 = fma(M[1], x2, fma(M[4], y2, M[7]))
    num = fma(x2, a0, fma(y2, a1, a2))
    return classify(num * num, thr * fma(a0, a0, fma(a1, a1, fma(b0, b0, b1 * b1))))


def rotation(rng, angle):
    a = rng.normal(size=3)
    k = a / np.linalg.norm(a)
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(angle) * K + (1 - np.cos(angle)) * K @ K


def intrinsics(width):
    return np.array([[width, 0, width / 2], [0, width, 0.375 * width], [0, 0, 1.0]])


def points(rng, width, n):
    return np.c_[rng.uniform(0, width, n), rng.uniform(0, 0.75 * width, n), np.ones(n)]


def wrong_h(rng, width, max_error, n=4000):
    K = intrinsics(width)
    Hm = K @ (rotation(rng, 0.2) + np.outer([0.3, 0.1, 0.05], [0.1, 0.2, 1.0]) / 5.0) @ np.linalg.inv(K)
    Hm /= Hm[2, 2]
    x1 = points(rng, width, n)
    q = x1 @ Hm.T
    p = q[:, :2] / q[:, 2:]
    ang = rng.uniform(0, 2 * np.pi, n)
    x2 = p + (max_error * rng.choice(OFFSETS, n))[:, None] * np.c_[np.cos(ang), np.sin(ang)]
    thr = max_error ** 2
    r64 = ((x2 - p) ** 2).sum(1)
    c = h_f32(Hm.ravel(), x1[:, 0], x1[:, 1], x2[:, 0], x2[:, 1], thr)
    return int((((c == 1) & (r64 > thr)) | ((c == 0) & (r64 <= thr))).sum())


def wrong_f(rng, width, max_error, n=4000):
    K = intrinsics(width)
    Ki = np.linalg.inv(K)
    R, t = rotation(rng, 0.2), np.array([1.0, 0.2, 0.1])
    tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
    Fm = Ki.T @ tx @ R @ Ki
    Fm /= np.linalg.norm(Fm)
    x1 = points(rng, width, n)
    Xc = (x1 @ Ki.T) * rng.uniform(3, 20, n)[:, None] @ R.T + t
    p = Xc @ K.T
    p = p[:, :2] / p[:, 2:]
    line = x1 @ Fm.T
    normal = line[:, :2] / np.linalg.norm(line[:, :2], axis=1)[:, None]
    x2 = p + (max_error * rng.choice(OFFSETS, n))[:, None] * normal
    thr = max_error ** 2
    X2 = np.c_[x2, np.ones(n)]
    Fx1, Ftx2 = x1 @ Fm.T, X2 @ Fm
    r64 = (X2 * Fx1).sum(1) ** 2 / (Fx1[:, 0] ** 2 + Fx1[:, 1] ** 2 + Ftx2[:, 0] ** 2 + Ftx2[:, 1] ** 2)
    c = f_f32(Fm.ravel(), x1[:, 0], x1[:, 1], x2[:, 0], x2[:, 1], thr)
    return int((((c == 1) & (r64 > thr)) | ((c == 0) & (r64 <= thr))).sum())


def test_emulation_places_points_on_both_sides_and_in_the_band():
    """The scenes are adversarial: all three outcomes occur, so a zero below is not for want of borderline points."""
    rng = np.random.default_rng(0)
    width, max_error = 8000, 0.5
    K = intrinsics(width)
    Hm = K @ (rotation(rng, 0.2) + np.outer([0.3, 0.1, 0.05], [0.1, 0.2, 1.0]) / 5.0) @ np.linalg.inv(K)
    x1 = points(rng, width, 2000)
    q = x1 @ Hm.T
    x2 = q[:, :2] / q[:, 2:] + max_error * np.c_[rng.choice(np.r_[OFFSETS, 1.001], 2000), np.zeros(2000)]
    c = h_f32(Hm.ravel(), x1[:, 0], x1[:, 1], x2[:, 0], x2[:, 1], max_error ** 2)
    assert {0, 1, 2} <= set(np.unique(c).tolist())


@pytest.mark.parametrize("width,max_error", [(1600, 4), (1600, 0.25), (8000, 1), (8000, 0.25), (20000, 4), (20000, 0.5),
                                             (40000, 4), (40000, 1)])
def test_h_arm_agrees_with_fp64_within_the_stated_range(width, max_error):
    rng = np.random.default_rng(width + int(100 * max_error))
    assert sum(wrong_h(rng, width, max_error) for _ in range(5)) == 0


@pytest.mark.parametrize("width", [1600, 8000, 20000, 40000])
@pytest.mark.parametrize("max_error", [4, 1, 0.5, 0.25])
def test_f_arm_agrees_with_fp64(width, max_error):
    rng = np.random.default_rng(width + int(100 * max_error))
    assert sum(wrong_f(rng, width, max_error) for _ in range(5)) == 0
