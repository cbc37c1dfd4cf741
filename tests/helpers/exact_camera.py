"""Exact reference for the pose-refinement Jacobians of csrc/abs_pose.cu.

ImgFromCam of the eleven COLMAP camera models is written here as sympy expressions in the normalised camera
coordinates (u, v) and the camera parameters, one expression per branch of the model (the branches of
camera_models.h: fisheye r <= eps, FOV |omega| < 1e-8 and |2 r tan(omega / 2)| < 1e-6, thin-prism r <= eps).
Derivatives come from sympy.diff and are lambdified to float64 (or to mpmath for a high-precision check).  Nothing
here is derived from the CUDA sources or from the oracle's finite differences.

On top of the projection sit the pose chain rule on Ceres' quaternion manifold (q <- (cos|d|, sin|d| d / |d|) * q,
a rotation by 2|d| on the camera side, so dXc/dd = -2 [R X]_x), the Cauchy loss with Ceres' corrector (residual and
Jacobian scaled by sqrt(rho')) and a restatement of the Levenberg-Marquardt iteration of RefineAbsolutePose (Jacobi
scaling, diagonal clamp [1e-6, 1e32], initial radius 1e4, step accepted when the gain ratio exceeds 1e-3).
"""
import functools
import math

import numpy as np
import sympy as sp

EPS = float(np.finfo(float).eps)
NUM_PARAMS = {0: 3, 1: 4, 2: 4, 3: 5, 4: 8, 5: 8, 6: 12, 7: 5, 8: 4, 9: 5, 10: 12}
SINGLE_FOCAL = (0, 2, 3, 8, 9)
MODEL_NAMES = {0: "SIMPLE_PINHOLE", 1: "PINHOLE", 2: "SIMPLE_RADIAL", 3: "RADIAL", 4: "OPENCV", 5: "OPENCV_FISHEYE",
               6: "FULL_OPENCV", 7: "FOV", 8: "SIMPLE_RADIAL_FISHEYE", 9: "RADIAL_FISHEYE", 10: "THIN_PRISM_FISHEYE"}

_U, _V = sp.symbols("u v", real=True)
_P = sp.symbols("p0:12", real=True)


def focal_idxs(model):
    return [0] if model in SINGLE_FOCAL else [0, 1]


def extra_idxs(model):
    return list(range(3 if model in SINGLE_FOCAL else 4, NUM_PARAMS[model]))


def refined_idxs(model, refine_focal, refine_extra):
    return (focal_idxs(model) if refine_focal else []) + (extra_idxs(model) if refine_extra else [])


# ---- ImgFromCam, one expression pair per branch ---------------------------------------------------------------
def _branch_exprs(model):
    u, v, p = _U, _V, _P
    if model in SINGLE_FOCAL:
        fx = fy = p[0]
        cx, cy, k = p[1], p[2], p[3:]
    else:
        fx, fy, cx, cy, k = p[0], p[1], p[2], p[3], p[4:]
    r2 = u * u + v * v
    r = sp.sqrt(r2)

    def pix(ud, vd):
        return fx * ud + cx, fy * vd + cy

    def opencv_tangential(a, b, radial, p1, p2):
        ab, rr = a * b, a * a + b * b
        return (a * radial + 2 * p1 * ab + p2 * (rr + 2 * a * a), b * radial + 2 * p2 * ab + p1 * (rr + 2 * b * b))

    if model in (0, 1):
        return [pix(u, v)]
    if model in (2, 3):
        radial = k[0] * r2 + (k[1] * r2 ** 2 if model == 3 else 0)
        return [pix(u * (1 + radial), v * (1 + radial))]
    if model == 4:
        du, dv = opencv_tangential(u, v, k[0] * r2 + k[1] * r2 ** 2, k[2], k[3])
        return [pix(u + du, v + dv)]
    if model == 6:   # k1, k2, p1, p2, k3, k4, k5, k6: rational radial factor
        ratio = (1 + k[0] * r2 + k[1] * r2 ** 2 + k[4] * r2 ** 3) / (1 + k[5] * r2 + k[6] * r2 ** 2 + k[7] * r2 ** 3)
        du, dv = opencv_tangential(u, v, ratio - 1, k[2], k[3])
        return [pix(u + du, v + dv)]
    if model in (5, 8, 9):   # equidistant fisheye: theta_d = theta (1 + k1 theta^2 + ...), scaled by theta_d / r
        th = sp.atan(r)
        kk = list(k[:{5: 4, 8: 1, 9: 2}[model]])
        thd = th * (1 + sum(c * th ** (2 * (j + 1)) for j, c in enumerate(kk)))
        return [pix(u * thd / r, v * thd / r),          # r > eps
                pix(u, v)]                              # r <= eps
    if model == 7:   # FOV: factor = atan(2 r tan(w / 2)) / (r w)
        w = k[0]
        t = sp.tan(w / 2)
        taylor = (2 * t / w) * (1 - (4 * r2 * t * t) / 3)
        full = sp.atan(2 * r * t) / (r * w)
        return [pix(u * full, v * full),                # |w| >= 1e-8, |2 r tan(w / 2)| >= 1e-6
                pix(u * taylor, v * taylor),            # |w| >= 1e-8, |2 r tan(w / 2)| < 1e-6
                pix(u, v)]                              # |w| < 1e-8
    if model == 10:  # thin prism on the equidistant fisheye coordinates theta (u, v) / r
        out = []
        for a, b in ((sp.atan(r) * u / r, sp.atan(r) * v / r), (u, v)):    # r > eps, r <= eps
            aa = a * a + b * b
            radial = k[0] * aa + k[1] * aa ** 2 + k[4] * aa ** 3 + k[5] * aa ** 4
            da, db = opencv_tangential(a, b, radial, k[2], k[3])
            out.append(pix(a + da + k[6] * aa, b + db + k[7] * aa))
        return out
    raise ValueError(model)


def branch_of(model, params, u, v):
    """Index into _branch_exprs(model) for each point, by the tests of camera_models.h."""
    u, v = np.asarray(u, np.float64), np.asarray(v, np.float64)
    r = np.sqrt(u * u + v * v)
    if model in (5, 8, 9, 10):
        return np.where(r > EPS, 0, 1)
    if model == 7:
        w = float(params[4])
        if abs(w) < 1e-8:
            return np.full(r.shape, 2)
        return np.where(np.abs(2.0 * r * math.tan(0.5 * w)) < 1e-6, 1, 0)
    return np.zeros(r.shape, int)


@functools.lru_cache(maxsize=None)
def _compiled(model, module):
    """Per branch: f(u, v, *params) -> [x, y, dx/du, dx/dv, dy/du, dy/dv, dx/dp_0.., dy/dp_0..]."""
    n = NUM_PARAMS[model]
    args = (_U, _V) + tuple(_P[:n])
    fns = []
    for x, y in _branch_exprs(model):
        exprs = [x, y, sp.diff(x, _U), sp.diff(x, _V), sp.diff(y, _U), sp.diff(y, _V)]
        exprs += [sp.diff(x, p) for p in _P[:n]] + [sp.diff(y, p) for p in _P[:n]]
        fns.append(sp.lambdify(args, exprs, modules=module, cse=(module == "numpy")))
    return fns


def project(model, params, uv):
    """ImgFromCam and its exact derivatives for [m x 2] normalised points.
    Returns pix [m x 2], d pix / d(u, v) [m x 2 x 2], d pix / d params [m x 2 x n]."""
    uv = np.asarray(uv, np.float64).reshape(-1, 2)
    m, n = len(uv), NUM_PARAMS[model]
    params = [float(p) for p in params]
    assert len(params) == n
    pix, duv, dp = np.zeros((m, 2)), np.zeros((m, 2, 2)), np.zeros((m, 2, n))
    br = branch_of(model, params, uv[:, 0], uv[:, 1])
    for b, fn in enumerate(_compiled(model, "numpy")):
        sel = br == b
        if not sel.any():
            continue
        with np.errstate(all="ignore"):
            vals = [np.broadcast_to(np.asarray(e, np.float64), (int(sel.sum()),))
                    for e in fn(uv[sel, 0], uv[sel, 1], *params)]
        pix[sel] = np.stack(vals[0:2], 1)
        duv[sel] = np.stack(vals[2:6], 1).reshape(-1, 2, 2)
        dp[sel] = np.stack(vals[6:], 1).reshape(-1, 2, n)
    return pix, duv, dp


def project_mp(model, params, u, v, dps=40):
    """One point at `dps` digits with mpmath: [x, y, dx/du, dx/dv, dy/du, dy/dv, dx/dp.., dy/dp..] as mpf."""
    import mpmath
    b = int(branch_of(model, params, np.array([u]), np.array([v]))[0])
    with mpmath.workdps(dps):
        return _compiled(model, "mpmath")[b](mpmath.mpf(u), mpmath.mpf(v), *[mpmath.mpf(float(p)) for p in params])


# ---- pose, loss, residual Jacobian ----------------------------------------------------------------------------
def quat_to_rotation(q):
    w, x, y, z = np.asarray(q, np.float64) / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def qmul(a, b):
    w1, x1, y1, z1 = a
    w2, x2, y2, z2 = b
    return np.array([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                     w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2])


def qplus(q, d):
    """Ceres' quaternion manifold: (cos|d|, sin|d| d / |d|) * q."""
    d = np.asarray(d, np.float64)
    nd = float(np.linalg.norm(d))
    if nd == 0.0:
        return np.asarray(q, np.float64).copy()
    return qmul(np.r_[math.cos(nd), math.sin(nd) / nd * d], q)


def qminus(qn, q):
    """The d with qplus(q, d) == qn (both unit quaternions)."""
    dq = qmul(qn, np.r_[q[0], -np.asarray(q[1:])])
    if dq[0] < 0:
        dq = -dq
    s = float(np.linalg.norm(dq[1:]))
    return np.zeros(3) if s == 0.0 else math.atan2(s, dq[0]) / s * dq[1:]


def residuals_and_jacobian(model, params, q, t, X, x2, ridx):
    """Raw residuals r = ImgFromCam(R X + t) - x2 [m x 2] and d r / d(d_rot, t, params[ridx]) [m x 2 x (6 + k)]."""
    Rm = quat_to_rotation(q)
    RX = np.asarray(X, np.float64) @ Rm.T
    Xc = RX + np.asarray(t, np.float64)
    z = Xc[:, 2]
    uv = Xc[:, :2] / z[:, None]
    pix, duv, dp = project(model, params, uv)
    duv_dXc = np.zeros((len(z), 2, 3))
    duv_dXc[:, 0, 0] = duv_dXc[:, 1, 1] = 1 / z
    duv_dXc[:, 0, 2] = -uv[:, 0] / z
    duv_dXc[:, 1, 2] = -uv[:, 1] / z
    dpix_dXc = duv @ duv_dXc
    skew = np.zeros((len(z), 3, 3))      # [R X]_x
    skew[:, 0, 1], skew[:, 0, 2], skew[:, 1, 2] = -RX[:, 2], RX[:, 1], -RX[:, 0]
    skew[:, 1, 0], skew[:, 2, 0], skew[:, 2, 1] = RX[:, 2], -RX[:, 1], RX[:, 0]
    J = np.concatenate([dpix_dXc @ (-2.0 * skew), dpix_dXc, dp[:, :, list(ridx)]], 2)
    return pix - np.asarray(x2, np.float64), J


def robust(r, J, loss_scale=1.0):
    """Cauchy loss: cost 1/2 sum a^2 log(1 + s / a^2), and the residuals / Jacobian scaled by sqrt(rho')."""
    a2 = loss_scale * loss_scale
    s = (r * r).sum(1)
    w = np.sqrt(1.0 / (1.0 + s / a2))
    return 0.5 * float((a2 * np.log1p(s / a2)).sum()), (r * w[:, None]).reshape(-1), (J * w[:, None, None]).reshape(
        -1, J.shape[2])


class Problem:
    """Refinement problem over the inliers: the state is (q, t, params), the unknowns (d_rot, t, params[ridx])."""

    def __init__(self, model, X, x2, ridx, loss_scale=1.0):
        self.model, self.X, self.x2, self.ridx, self.loss_scale = model, np.asarray(X), np.asarray(x2), list(ridx), loss_scale

    def evaluate(self, q, t, params):
        r, J = residuals_and_jacobian(self.model, params, q, t, self.X, self.x2, self.ridx)
        return robust(r, J, self.loss_scale)

    def cost(self, q, t, params):
        return self.evaluate(q, t, params)[0]

    def gradient(self, q, t, params):
        _, rr, JJ = self.evaluate(q, t, params)
        return JJ.T @ rr

    def covariance(self, q, t, params):
        _, _, JJ = self.evaluate(q, t, params)
        return np.linalg.inv(JJ.T @ JJ)[:6, :6], JJ.T @ JJ

    def apply(self, q, t, params, step):
        pn = np.array(params, np.float64)
        for j, i in enumerate(self.ridx):
            pn[i] += step[6 + j]
        return qplus(q, step[:3]), np.asarray(t) + step[3:6], pn


def lm_step(rr, JJ, radius):
    """One trust-region solve of the LM restatement: returns (step, model cost change, Jacobi-scaled A)."""
    g = JJ.T @ rr
    A = JJ.T @ JJ
    scale = 1.0 / (1.0 + np.sqrt(np.diag(A)))
    As = A * np.outer(scale, scale)
    gs = g * scale
    D = np.clip(np.diag(As), 1e-6, 1e32)
    xs = np.linalg.solve(As + np.diag(D / radius), -gs)
    return xs * scale, -(gs @ xs + 0.5 * xs @ As @ xs), As


def minimise(prob, q, t, params, max_iterations=100, gradient_tolerance=0.0, function_tolerance=1e-6):
    """The LM iteration of RefineAbsolutePose.  Returns (q, t, params, cost, accepted steps)."""
    q = np.asarray(q, np.float64) / np.linalg.norm(q)
    t, params = np.asarray(t, np.float64), np.asarray(params, np.float64)
    cost, rr, JJ = prob.evaluate(q, t, params)
    radius, decrease, it, accepted = 1e4, 2.0, 0, 0
    while True:
        if np.abs(JJ.T @ rr).max() <= gradient_tolerance or it >= max_iterations:
            break
        it += 1
        step, mc, _ = lm_step(rr, JJ, radius)
        xn = math.sqrt(float(q @ q + t @ t + sum(params[i] ** 2 for i in prob.ridx)))
        if np.linalg.norm(step) <= 1e-8 * (xn + 1e-8):
            break
        qn, tn, pn = prob.apply(q, t, params, step)
        cn, rn, Jn = prob.evaluate(qn, tn, pn)
        ratio = (cost - cn) / mc if mc > 0 else -1.0
        if np.isfinite(cn) and ratio > 1e-3:
            done = abs(cost - cn) <= function_tolerance * cost
            q, t, params, cost, rr, JJ = qn, tn, pn, cn, rn, Jn
            radius = min(1e16, radius / max(1.0 / 3.0, 1.0 - (2.0 * ratio - 1.0) ** 3))
            decrease = 2.0
            accepted += 1
            if done:
                break
        else:
            radius /= decrease
            decrease *= 2.0
            if radius < 1e-32:
                break
    return q, t, params, cost, accepted


# ---- planted scenes with edge geometry --------------------------------------------------------------------------
F, W, H = 1200.0, 1600, 1200
# strong distortion: at the image corners the distortion moves points by tens of pixels
CASES = {
    "SIMPLE_PINHOLE": (0, [F, 800.0, 600.0]),
    "PINHOLE": (1, [F, 1.02 * F, 800.0, 600.0]),
    "SIMPLE_RADIAL": (2, [F, 800.0, 600.0, -0.08]),
    "RADIAL": (3, [F, 800.0, 600.0, -0.08, 0.02]),
    "OPENCV": (4, [F, 1.02 * F, 800.0, 600.0, -0.08, 0.02, 0.004, -0.003]),
    "OPENCV_FISHEYE": (5, [F, 1.02 * F, 800.0, 600.0, 0.05, -0.02, 0.01, -0.005]),
    "FULL_OPENCV": (6, [F, 1.02 * F, 800.0, 600.0, -0.1, 0.03, 0.004, -0.003, 0.01, 0.05, 0.02, 0.01]),
    "FOV": (7, [F, 1.02 * F, 800.0, 600.0, 0.3]),
    "FOV_OMEGA_1E-9": (7, [F, 1.02 * F, 800.0, 600.0, 1e-9]),
    "SIMPLE_RADIAL_FISHEYE": (8, [F, 800.0, 600.0, 0.05]),
    "RADIAL_FISHEYE": (9, [F, 800.0, 600.0, 0.05, -0.02]),
    "THIN_PRISM_FISHEYE": (10, [F, 1.02 * F, 800.0, 600.0, -0.05, 0.02, 0.004, -0.003, 0.01, 0.005, 0.003, -0.002]),
}
# refinement configurations: (refine_focal_length, refine_extra_params)
CONFIGS = {"pose": (False, False), "focal": (True, False), "focal_extra": (True, True)}


def edge_uv(model, params):
    """Normalised points on and next to the optical axis (the fisheye / thin-prism r <= eps branch and r just above
    eps) and, for FOV, on both sides of the |2 r tan(w / 2)| = 1e-6 switch to the Taylor branch."""
    pts = [(0.0, 0.0), (1e-9, 0.0), (0.0, -1e-9), (7e-10, -7e-10), (2.3e-16, 0.0), (1.6e-16, -1.6e-16),
           (0.0, 1e-15), (3e-16, 3e-16)]
    if model == 7 and abs(params[4]) >= 1e-8:
        rs = 1e-6 / (2.0 * math.tan(0.5 * params[4]))
        for j, f in enumerate((1 - 1e-3, 1 + 1e-3, 0.9, 1.1, 1 - 1e-9, 1 + 1e-9)):
            a = 0.7 * j
            pts.append((rs * f * math.cos(a), rs * f * math.sin(a)))
    return np.array(pts)


def border_pixels(inset=4.0):
    xs, ys = (inset, W / 2, W - inset), (inset, H / 2, H - inset)
    return np.array([(x, y) for x in xs for y in ys if (x, y) != (W / 2, H / 2)])


def planted(case, rng, n=240, noise_px=0.5):
    """A scene whose world frame is the camera frame of the identity pose, which is the start of the refinement tests:
    at that start the edge points sit exactly at their normalised coordinates (depth 4, so u = X / Z is exact).
    The observations are the exact projections under a true pose about 0.008 rad / 0.05 away, plus pixel noise.
    Returns (camera dict, X [m x 3], points2D [m x 2], q_true, t_true, number of edge points)."""
    from oracle import ransac as R
    model, params = CASES[case]
    cam = dict(model=model, width=W, height=H, params=list(params))
    pix = np.r_[np.c_[rng.uniform(0.05 * W, 0.95 * W, n), rng.uniform(0.05 * H, 0.95 * H, n)], border_pixels()]
    uv = R.cam_from_img(cam, pix)
    z = rng.uniform(4.0, 10.0, len(uv))
    e = edge_uv(model, params)
    X = np.r_[np.c_[uv * z[:, None], z], np.c_[4.0 * e, np.full(len(e), 4.0)]]
    d = rng.normal(size=3)
    q_true = qplus(np.array([1.0, 0.0, 0.0, 0.0]), 0.004 * d / np.linalg.norm(d))
    t_true = rng.uniform(-0.05, 0.05, 3)
    Xc = X @ quat_to_rotation(q_true).T + t_true
    x2 = project(model, params, Xc[:, :2] / Xc[:, 2:])[0] + rng.normal(scale=noise_px, size=(len(X), 2))
    return cam, X, x2, q_true, t_true, len(e)


def perturbed_params(case, ridx):
    """Start values for the refined camera parameters: focal lengths 1 % short, distortion 10 % off."""
    model, params = CASES[case]
    p = np.array(params, np.float64)
    for i in ridx:
        p[i] *= 0.99 if i in focal_idxs(model) else 1.1
    return p
