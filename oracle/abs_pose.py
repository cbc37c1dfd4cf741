"""CPU restatement (numpy, fp64) of absolute pose estimation and refinement -- TEST INFRASTRUCTURE ONLY.

PARITY UNPINNED, like oracle/ransac.py: the reference binds COLMAP 3.9.1 (R:pycolmap/estimators/absolute_pose.h:18-166),
which is not on disk.  This file restates the published algorithms; where it and the CUDA kernels disagree, this
file is the specification (SURVEY.md section 8(a) rows A1-A5):

  estimate_absolute_pose  <- U:estimators/pose.cc EstimateAbsolutePose / EstimateAbsolutePoseKernel        (A1)
  P3PEstimator            <- U:estimators/absolute_pose.cc P3PEstimator (3 samples, <= 4 models)           (A2)
  EPNPEstimator           <- U:estimators/absolute_pose.cc EPNPEstimator (Lepetit et al., EPnP)            (A3)
  refine_absolute_pose    <- U:estimators/pose.cc RefineAbsolutePose, Ceres LM with CauchyLoss             (A4)

P3P solves Grunert's quartic (Haralick et al., "Review and analysis of solutions of the three point perspective
pose estimation problem", 1994); every P3P formulation has the same real solution set.  The LO-RANSAC control
flow is the generic oracle.ransac.loransac.

Refinement restates Ceres' Levenberg-Marquardt as configured by RefineAbsolutePose: cost 1/2 sum_i rho(|r_i|^2),
rho = CauchyLoss(a): a^2 log(1 + s / a^2), one 2-D residual block per inlier; Ceres' corrector for a loss with
rho'' < 0 scales residual and Jacobian by sqrt(rho'); Jacobi column scaling; initial trust radius 1e4; step accepted
when the gain ratio exceeds 1e-3; stop on |g|_inf <= gradient_tolerance, |dcost| / cost <= 1e-6,
|dx| <= 1e-8 (|x| + 1e-8) or max_num_iterations.  The rotation moves on Ceres' quaternion manifold:
q <- (cos|d|, sin|d| d / |d|) * q, i.e. a rotation by 2|d| applied on the camera side.  The covariance is the 6 x 6
(rotation tangent, translation) block of the inverse of J^T J (loss-corrected J, refined camera parameters
included and marginalised out).
"""
import math

import numpy as np

from . import ransac as R

DBL_EPS = np.finfo(float).eps
_FOCAL_IDX = {0: [0], 1: [0, 1], 2: [0], 3: [0], 4: [0, 1], 5: [0, 1], 6: [0, 1], 7: [0, 1], 8: [0], 9: [0], 10: [0, 1]}
_PP_IDX = {m: ([1, 2] if m in R._SINGLE_FOCAL else [2, 3]) for m in R.CAMERA_NUM_PARAMS}


def focal_idxs(model):
    return list(_FOCAL_IDX[model])


def extra_idxs(model):
    n = R.CAMERA_NUM_PARAMS[model]
    return list(range(3 if model in R._SINGLE_FOCAL else 4, n))


# ---------------------------------------------------------------------------------------------
# residual (A2): squared reprojection error on the normalised image plane, DBL_MAX behind the camera
# ---------------------------------------------------------------------------------------------
def squared_reprojection_error(points2D, points3D, P):
    Xc = points3D @ P[:, :3].T + P[:, 3]
    z = Xc[:, 2]
    ok = z > DBL_EPS
    zs = np.where(ok, z, 1.0)
    d = Xc[:, :2] / zs[:, None] - points2D
    return np.where(ok, (d * d).sum(1), np.finfo(float).max)


def _frame(a, b, c):
    e1 = b - a
    e1 = e1 / np.linalg.norm(e1)
    e3 = np.cross(b - a, c - a)
    e3 = e3 / np.linalg.norm(e3)
    return np.stack([e1, np.cross(e3, e1), e3], 1)


class P3PEstimator:
    kMinNumSamples = 3

    @staticmethod
    def estimate(points2D, points3D):
        f = np.c_[points2D, np.ones(3)]
        f = f / np.linalg.norm(f, axis=1)[:, None]
        P = points3D
        a2 = float(((P[1] - P[2]) ** 2).sum())
        b2 = float(((P[0] - P[2]) ** 2).sum())
        c2 = float(((P[0] - P[1]) ** 2).sum())
        if not (b2 > 0 and a2 > 0 and c2 > 0):
            return []
        ca, cb, cg = float(f[1] @ f[2]), float(f[0] @ f[2]), float(f[0] @ f[1])
        p, q = (a2 - c2) / b2, (a2 + c2) / b2
        A4 = (p - 1) ** 2 - 4 * c2 / b2 * ca * ca
        A3 = 4 * (p * (1 - p) * cb - (1 - q) * ca * cg + 2 * c2 / b2 * ca * ca * cb)
        A2 = 2 * (p * p - 1 + 2 * p * p * cb * cb + 2 * (b2 - c2) / b2 * ca * ca - 4 * q * ca * cb * cg
                  + 2 * (b2 - a2) / b2 * cg * cg)
        A1 = 4 * (-p * (1 + p) * cb + 2 * a2 / b2 * cg * cg * cb - (1 - q) * ca * cg)
        A0 = (1 + p) ** 2 - 4 * a2 / b2 * cg * cg
        coef = np.array([A4, A3, A2, A1, A0])
        if not np.all(np.isfinite(coef)) or np.abs(coef).max() == 0:
            return []
        models = []
        for v in np.roots(coef):
            if abs(v.imag) > 1e-4 * max(1.0, abs(v.real)):   # near-double roots come out as complex pairs
                continue
            v = v.real
            for _ in range(3):   # polish the companion-matrix root (Newton on the quartic)
                fv, dfv = np.polyval(coef, v), np.polyval(np.polyder(coef), v)
                if dfv == 0 or not np.isfinite(fv / dfv):
                    break
                v -= fv / dfv
            den = 2 * (cg - v * ca)
            if den == 0:
                continue
            u = ((p - 1) * v * v - 2 * p * cb * v + 1 + p) / den
            s1sq = c2 / (1 + u * u - 2 * u * cg)
            if not (s1sq > 0 and u > 0 and v > 0):
                continue
            s1 = math.sqrt(s1sq)
            Q = np.stack([s1 * f[0], u * s1 * f[1], v * s1 * f[2]])
            Rm = _frame(*Q) @ _frame(*P).T
            t = Q[0] - Rm @ P[0]
            models.append(np.c_[Rm, t])
        return models[:4]

    @staticmethod
    def residuals(points2D, points3D, P):
        return squared_reprojection_error(points2D, points3D, P)


class EPNPEstimator:
    kMinNumSamples = 4

    @staticmethod
    def estimate(points2D, points3D):
        P = compute_epnp(points2D, points3D)
        return [] if P is None else [P]

    @staticmethod
    def residuals(points2D, points3D, P):
        return squared_reprojection_error(points2D, points3D, P)


_PAIRS = [(0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3)]


def _lstsq(A, b):
    return np.linalg.lstsq(A, b, rcond=None)[0]


def _epnp_rt(Ut, betas, alphas, pws):
    ccs = np.zeros((4, 3))
    for j in range(4):
        ccs += betas[j] * Ut[11 - j].reshape(4, 3)
    pcs = alphas @ ccs
    if pcs[0, 2] < 0:
        ccs, pcs = -ccs, -pcs
    pc0, pw0 = pcs.mean(0), pws.mean(0)
    abt = (pcs - pc0).T @ (pws - pw0)
    U, _, Vt = np.linalg.svd(abt)
    Rm = U @ Vt
    if np.linalg.det(Rm) < 0:
        Vt2 = Vt.copy()
        Vt2[2] = -Vt2[2]
        Rm = U @ Vt2
    return np.c_[Rm, pc0 - Rm @ pw0]


def compute_epnp(points2D, points3D):
    """EPNPEstimator::ComputePose; None where upstream returns no model."""
    n = len(points3D)
    pws = np.asarray(points3D, np.float64)
    c0 = pws.mean(0)
    PW0 = pws - c0
    U, D, _ = np.linalg.svd(PW0.T @ PW0)
    cws = np.stack([c0] + [c0 + math.sqrt(D[i] / n) * U[:, i] for i in range(3)])
    CC = (cws[1:] - cws[0]).T
    if np.linalg.matrix_rank(CC) < 3:
        return None
    a = np.linalg.solve(CC, (pws - cws[0]).T).T
    alphas = np.c_[1 - a.sum(1), a]
    M = np.zeros((2 * n, 12))
    for j in range(4):
        M[0::2, 3 * j] = alphas[:, j]
        M[0::2, 3 * j + 2] = -alphas[:, j] * points2D[:, 0]
        M[1::2, 3 * j + 1] = alphas[:, j]
        M[1::2, 3 * j + 2] = -alphas[:, j] * points2D[:, 1]
    w, V = np.linalg.eigh(M.T @ M)
    Ut = V[:, ::-1].T            # rows by decreasing eigenvalue: Ut[11 - i] is the i-th smallest
    dv = np.zeros((4, 6, 3))
    for i in range(4):
        v = Ut[11 - i].reshape(4, 3)
        for k, (p, q) in enumerate(_PAIRS):
            dv[i, k] = v[p] - v[q]
    L = np.zeros((6, 10))
    for k in range(6):
        d = dv[:, k]
        L[k] = [d[0] @ d[0], 2 * d[0] @ d[1], d[1] @ d[1], 2 * d[0] @ d[2], 2 * d[1] @ d[2], d[2] @ d[2],
                2 * d[0] @ d[3], 2 * d[1] @ d[3], 2 * d[2] @ d[3], d[3] @ d[3]]
    rho = np.array([((cws[p] - cws[q]) ** 2).sum() for p, q in _PAIRS])

    def approx1():
        b4 = _lstsq(L[:, [0, 1, 3, 6]], rho)
        s = math.sqrt(abs(b4[0]))
        sg = -1.0 if b4[0] < 0 else 1.0
        return np.array([s, sg * b4[1] / s, sg * b4[2] / s, sg * b4[3] / s]) if s > 0 else np.zeros(4)

    def approx2():
        b3 = _lstsq(L[:, [0, 1, 2]], rho)
        if b3[0] < 0:
            be = [math.sqrt(-b3[0]), math.sqrt(-b3[2]) if b3[2] < 0 else 0.0]
        else:
            be = [math.sqrt(b3[0]), math.sqrt(b3[2]) if b3[2] > 0 else 0.0]
        if b3[1] < 0:
            be[0] = -be[0]
        return np.array(be + [0.0, 0.0])

    def approx3():
        b5 = _lstsq(L[:, [0, 1, 2, 3, 4]], rho)
        if b5[0] < 0:
            be = [math.sqrt(-b5[0]), math.sqrt(-b5[2]) if b5[2] < 0 else 0.0]
        else:
            be = [math.sqrt(b5[0]), math.sqrt(b5[2]) if b5[2] > 0 else 0.0]
        if b5[1] < 0:
            be[0] = -be[0]
        b2 = b5[3] / be[0] if be[0] != 0 else 0.0
        return np.array(be + [b2, 0.0])

    def gauss_newton(b):
        b = b.copy()
        for _ in range(5):
            A = np.zeros((6, 4))
            r = np.zeros(6)
            for i in range(6):
                l = L[i]
                A[i] = [2 * l[0] * b[0] + l[1] * b[1] + l[3] * b[2] + l[6] * b[3],
                        l[1] * b[0] + 2 * l[2] * b[1] + l[4] * b[2] + l[7] * b[3],
                        l[3] * b[0] + l[4] * b[1] + 2 * l[5] * b[2] + l[8] * b[3],
                        l[6] * b[0] + l[7] * b[1] + l[8] * b[2] + 2 * l[9] * b[3]]
                bb = [b[0] * b[0], b[0] * b[1], b[1] * b[1], b[0] * b[2], b[1] * b[2], b[2] * b[2],
                      b[0] * b[3], b[1] * b[3], b[2] * b[3], b[3] * b[3]]
                r[i] = rho[i] - l @ bb
            b += _lstsq(A, r)
        return b

    best, best_err = None, float("inf")
    for approx in (approx1, approx2, approx3):
        with np.errstate(all="ignore"):
            Pm = _epnp_rt(Ut, gauss_newton(approx()), alphas, pws)
            err = float(np.sqrt(squared_reprojection_error(points2D, pws, Pm)).sum())
        if np.all(np.isfinite(Pm)) and err < best_err:
            best, best_err = Pm, err
    return best


# ---------------------------------------------------------------------------------------------
# A1: EstimateAbsolutePose
# ---------------------------------------------------------------------------------------------
class EstimationOptions:
    """pycolmap's AbsolutePoseEstimationOptions() (R:absolute_pose.h:101-108): RANSACOptions() with max_error 12."""

    def __init__(self, **kw):
        self.estimate_focal_length = False
        self.num_focal_length_samples = 30
        self.min_focal_length_ratio = 0.2
        self.max_focal_length_ratio = 5.0
        self.ransac = R.RansacOptions(max_error=12.0, min_inlier_ratio=0.01, confidence=0.9999, min_num_trials=1000,
                                      max_num_trials=100000)
        self.__dict__.update(kw)


class RefinementOptions:
    """pycolmap's AbsolutePoseRefinementOptions() (R:absolute_pose.h:125-131)."""

    def __init__(self, **kw):
        self.gradient_tolerance = 1.0
        self.max_num_iterations = 100
        self.loss_function_scale = 1.0
        self.refine_focal_length = False
        self.refine_extra_params = False
        self.__dict__.update(kw)


def focal_length_factors(opt):
    if not opt.estimate_focal_length:
        return [1.0]
    n = opt.num_focal_length_samples
    return [opt.min_focal_length_ratio + (opt.max_focal_length_ratio - opt.min_focal_length_ratio) * (i / n) ** 2
            for i in range(n + 1)]


def scaled_camera(cam, factor):
    c = dict(cam)
    p = [float(x) for x in cam["params"]]
    for i in focal_idxs(cam["model"]):
        p[i] *= factor
    c["params"] = p
    return c


class PoseResult:
    def __init__(self):
        self.success, self.num_inliers, self.inlier_mask = False, 0, None
        self.P, self.camera, self.factor_index = None, None, -1


def estimate_absolute_pose(points2D, points3D, camera, options=None, seed=0):
    """Returns a PoseResult; .camera holds the parameters the caller's camera ends up with."""
    opt = options or EstimationOptions()
    points2D = np.asarray(points2D, np.float64).reshape(-1, 2)
    points3D = np.asarray(points3D, np.float64).reshape(-1, 3)
    out = PoseResult()
    out.camera = dict(camera)
    best = 0
    for i, fac in enumerate(focal_length_factors(opt)):
        cam = scaled_camera(camera, fac)
        x = R.cam_from_img(cam, points2D) if len(points2D) else np.zeros((0, 2))
        ro = opt.ransac.copy(max_error=R.cam_from_img_threshold(cam, opt.ransac.max_error))
        rep = R.loransac(P3PEstimator, EPNPEstimator, x, points3D, ro, np.random.default_rng(seed + i))
        if rep.success and rep.num_inliers > best:
            best = rep.num_inliers
            out.num_inliers, out.inlier_mask, out.P, out.factor_index = rep.num_inliers, rep.inlier_mask, rep.model, i
            out.camera = cam if opt.estimate_focal_length else dict(camera)
    if best == 0:
        out.camera = dict(camera)
        out.inlier_mask = np.zeros(len(points2D), bool)
        return out
    out.success = bool(np.all(np.isfinite(out.P[:, 3])))
    return out


# ---------------------------------------------------------------------------------------------
# A4: RefineAbsolutePose
# ---------------------------------------------------------------------------------------------
def quat_to_rotation(q):
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def rotation_to_quat(Rm):
    return np.asarray(R.rotation_to_quat(Rm), np.float64)


def _qmul(a, b):
    w1, x1, y1, z1 = a
    w2, x2, y2, z2 = b
    return np.array([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                     w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2])


def _qplus(q, d):
    n = np.linalg.norm(d)
    if n == 0:
        return q.copy()
    dq = np.r_[math.cos(n), math.sin(n) / n * d]
    return _qmul(dq, q)


class RefineResult:
    def __init__(self):
        self.success, self.qvec, self.tvec, self.params, self.covariance, self.num_iterations = False, None, None, None, None, 0


def refine_absolute_pose(qvec, tvec, points2D, points3D, inlier_mask, camera, options=None, covariance=False):
    """LM restatement of RefineAbsolutePose (header docstring).  qvec = (w, x, y, z), cam_from_world."""
    opt = options or RefinementOptions()
    model = camera["model"]
    params = np.array(camera["params"], np.float64)
    sel = np.asarray(inlier_mask, bool)
    x2 = np.asarray(points2D, np.float64).reshape(-1, 2)[sel]
    X3 = np.asarray(points3D, np.float64).reshape(-1, 3)[sel]
    ridx = []
    if opt.refine_focal_length or opt.refine_extra_params:
        if opt.refine_focal_length:
            ridx += focal_idxs(model)
        if opt.refine_extra_params:
            ridx += extra_idxs(model)
    a2 = opt.loss_function_scale ** 2
    npar = 6 + len(ridx)
    q, t = np.asarray(qvec, np.float64) / np.linalg.norm(qvec), np.asarray(tvec, np.float64).copy()
    out = RefineResult()

    def residuals(q, t, p):
        Xc = X3 @ quat_to_rotation(q).T + t
        uv = Xc[:, :2] / Xc[:, 2:]
        cam = dict(camera)
        cam["params"] = p
        return R.img_from_cam(cam, uv) - x2

    def cost_of(r):
        return 0.5 * float((a2 * np.log1p((r * r).sum(1) / a2)).sum())

    def jacobian(q, t, p):
        # pose: exact chain rule; camera: central differences of img_from_cam on (u, v, params)
        Rm = quat_to_rotation(q)
        RX = X3 @ Rm.T
        Xc = RX + t
        u, v, z = Xc[:, 0] / Xc[:, 2], Xc[:, 1] / Xc[:, 2], Xc[:, 2]
        cam = dict(camera)
        cam["params"] = p

        def proj(uu, vv, pp):
            c = dict(camera)
            c["params"] = pp
            return R.img_from_cam(c, np.c_[uu, vv])
        hu = 1e-7 * np.maximum(1.0, np.abs(u))
        hv = 1e-7 * np.maximum(1.0, np.abs(v))
        dpu = (proj(u + hu, v, p) - proj(u - hu, v, p)) / (2 * hu)[:, None]
        dpv = (proj(u, v + hv, p) - proj(u, v - hv, p)) / (2 * hv)[:, None]
        duv_dX = np.zeros((len(u), 2, 3))
        duv_dX[:, 0, 0] = 1 / z
        duv_dX[:, 0, 2] = -u / z
        duv_dX[:, 1, 1] = 1 / z
        duv_dX[:, 1, 2] = -v / z
        dpix_dX = np.stack([dpu, dpv], 2) @ duv_dX          # n x 2 x 3
        J = np.zeros((len(u), 2, npar))
        skew = np.zeros((len(u), 3, 3))
        skew[:, 0, 1], skew[:, 0, 2], skew[:, 1, 2] = -RX[:, 2], RX[:, 1], -RX[:, 0]
        skew[:, 1, 0], skew[:, 2, 0], skew[:, 2, 1] = RX[:, 2], -RX[:, 1], RX[:, 0]
        J[:, :, 0:3] = dpix_dX @ (-2.0 * skew)
        J[:, :, 3:6] = dpix_dX
        for k, i in enumerate(ridx):
            h = 1e-7 * max(1.0, abs(p[i]))
            pp, pm = p.copy(), p.copy()
            pp[i] += h
            pm[i] -= h
            J[:, :, 6 + k] = (proj(u, v, pp) - proj(u, v, pm)) / (2 * h)
        return J

    def corrected(r, J):
        s = (r * r).sum(1)
        w = np.sqrt(1.0 / (1.0 + s / a2))                   # sqrt(rho') of the Cauchy loss
        return (r * w[:, None]).reshape(-1), (J * w[:, None, None]).reshape(-1, npar)

    r = residuals(q, t, params)
    cost = cost_of(r)
    if not np.isfinite(cost):
        return out
    if len(x2) == 0:
        out.success, out.qvec, out.tvec, out.params = True, q, t, params
        return out
    radius, decrease = 1e4, 2.0
    it = 0
    rr, JJ = corrected(r, jacobian(q, t, params))
    while True:
        g = JJ.T @ rr
        if np.abs(g).max() <= opt.gradient_tolerance or it >= opt.max_num_iterations:
            break
        it += 1
        scale = 1.0 / (1.0 + np.sqrt((JJ * JJ).sum(0)))
        Js = JJ * scale
        A = Js.T @ Js
        diag = np.clip(np.diag(A), 1e-6, 1e32)
        step_s = np.linalg.solve(A + np.diag(diag / radius), -(Js.T @ rr))
        step = step_s * scale
        model_change = -(rr @ (Js @ step_s) + 0.5 * (Js @ step_s) @ (Js @ step_s))
        xnorm = math.sqrt(float(q @ q + t @ t + sum(params[i] ** 2 for i in ridx)))
        if np.linalg.norm(step) <= 1e-8 * (xnorm + 1e-8):
            break
        qn, tn, pn = _qplus(q, step[:3]), t + step[3:6], params.copy()
        for k, i in enumerate(ridx):
            pn[i] += step[6 + k]
        rn = residuals(qn, tn, pn)
        cn = cost_of(rn)
        ratio = (cost - cn) / model_change if model_change > 0 else -1.0
        if np.isfinite(cn) and ratio > 1e-3:
            done = abs(cost - cn) <= 1e-6 * cost
            q, t, params, cost = qn, tn, pn, cn
            radius = min(1e16, radius / max(1.0 / 3.0, 1.0 - (2.0 * ratio - 1.0) ** 3))
            decrease = 2.0
            rr, JJ = corrected(rn, jacobian(q, t, params))
            if done:
                break
        else:
            radius /= decrease
            decrease *= 2.0
            if radius < 1e-32:
                break
    out.success, out.qvec, out.tvec, out.params, out.num_iterations = True, q, t, params, it
    if covariance:
        rr, JJ = corrected(residuals(q, t, params), jacobian(q, t, params))
        out.covariance = np.linalg.inv(JJ.T @ JJ)[:6, :6]
    return out


def robust_cost(qvec, tvec, points2D, points3D, inlier_mask, camera, loss_function_scale=1.0):
    sel = np.asarray(inlier_mask, bool)
    Xc = np.asarray(points3D, np.float64)[sel] @ quat_to_rotation(np.asarray(qvec, np.float64)).T + tvec
    r = R.img_from_cam(camera, Xc[:, :2] / Xc[:, 2:]) - np.asarray(points2D, np.float64)[sel]
    a2 = loss_function_scale ** 2
    return 0.5 * float((a2 * np.log1p((r * r).sum(1) / a2)).sum())


def absolute_pose_estimation(points2D, points3D, camera, estimation_options=None, refinement_options=None,
                             return_covariance=False, seed=0):
    """pycolmap.absolute_pose_estimation: dict(cam_from_world=(qvec, tvec), num_inliers, inliers[, covariance],
    camera=<parameters the caller's camera ends up with>) or None."""
    est = estimate_absolute_pose(points2D, points3D, camera, estimation_options, seed)
    if not est.success:
        return None
    q = rotation_to_quat(est.P[:, :3])
    ref = refine_absolute_pose(q, est.P[:, 3], points2D, points3D, est.inlier_mask, est.camera, refinement_options,
                               covariance=return_covariance)
    if not ref.success:
        return None
    cam = dict(est.camera)
    cam["params"] = list(ref.params)
    out = dict(qvec=ref.qvec, tvec=ref.tvec, num_inliers=est.num_inliers, inliers=est.inlier_mask, camera=cam,
               factor_index=est.factor_index)
    if return_covariance:
        out["covariance"] = ref.covariance
    return out


def planted_scene(rng, n, camera, outlier_ratio=0.0, noise_px=0.0, depth=(4.0, 10.0)):
    """A random cam_from_world, n world points in front of it, their projections with pixel noise and a fraction of
    uniformly random outliers.  Returns (qvec, tvec, points2D, points3D, inlier_mask)."""
    ang = rng.normal(size=3)
    ang *= rng.uniform(0.1, 0.6) / np.linalg.norm(ang)
    th = np.linalg.norm(ang)
    k = ang / th
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    Rm = np.eye(3) + math.sin(th) * K + (1 - math.cos(th)) * K @ K
    t = rng.uniform(-1, 1, 3)
    w, h = camera["width"], camera["height"]
    model, f, c, _ = R._intrinsics(camera)
    pix = np.c_[rng.uniform(0.05 * w, 0.95 * w, n), rng.uniform(0.05 * h, 0.95 * h, n)]
    uv = R.cam_from_img(camera, pix)
    z = rng.uniform(depth[0], depth[1], n)
    Xc = np.c_[uv * z[:, None], z]
    X = (Xc - t) @ Rm
    pts = R.img_from_cam(camera, uv) + rng.normal(scale=noise_px, size=(n, 2)) if noise_px > 0 else pix.copy()
    inl = np.ones(n, bool)
    m = int(round(outlier_ratio * n))
    if m:
        o = rng.choice(n, m, replace=False)
        pts[o] = np.c_[rng.uniform(0, w, m), rng.uniform(0, h, m)]
        inl[o] = False
    return rotation_to_quat(Rm), t, pts, X, inl
