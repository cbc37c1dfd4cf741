"""GPU: the pose-refinement kernel (b2m_abs_refine_kernel, csrc/abs_pose.cu) against an exact reference.

The kernel's Jacobians are forward-mode dual numbers through camera_models.h.  A wrong derivative still lets LM get
close to the optimum, so these tests read the Jacobian back through quantities that depend on it directly, for every
camera model (FOV twice: omega = 0.3 and omega = 1e-9) and for pose only, + focal length, + focal length and extra
parameters.  The reference is tests/helpers/exact_camera.py (sympy derivatives, checked on the CPU by
test_exact_camera_reference.py):

  covariance  inv(J^T J)[:6, :6] at the returned pose and camera, J from the reference;
  one step    pose_refinement with max_num_iterations = 1 from a perturbed start equals one restated LM step;
  optimum     pose_refinement with gradient_tolerance = 1e-10 ends at least as low, and as converged, as the restated
              LM iteration with the same stopping rules, and no lower than the true minimum.

Every scene carries edge geometry: points on and within 1e-9 of the optical axis, points with r just above machine
epsilon (the fisheye and thin-prism r <= eps switch), FOV points on both sides of the Taylor switch
|2 r tan(omega / 2)| = 1e-6, and points 4 px from the image border under strong distortion.  The edge points sit
exactly at their normalised coordinates at the identity pose, which is where the one-step test evaluates J, so that
test is the one that exercises the branch switches.  The observations come from a true pose about 0.008 rad away, so
at the pose the covariance and optimum tests evaluate J the same points are 5e-3 to 2e-2 off the axis.  Those two
tests still see them, but at ordinary radii.  The border points stay within about 15 px of the border in all three."""
import numpy as np
import pytest

from helpers import exact_camera as E
from helpers.native_import import load_native

pytestmark = pytest.mark.gpu
nat = load_native()

CASES = list(E.CASES)
CONFIGS = list(E.CONFIGS)
Q0, T0 = np.array([1.0, 0.0, 0.0, 0.0]), np.zeros(3)
# FULL_OPENCV's radial factor is (1 + k1 r^2 + k2 r^4 + k3 r^6) / (1 + k4 r^2 + k5 r^4 + k6 r^6): with all eight
# coefficients refined, numerator and denominator nearly cancel and the scaled J^T J has cond ~ 1e15, so a tolerance
# set from the conditioning cannot fail.  The model is covered by its pose and focal configurations, and this
# configuration by the optimum test.
NEAR_SINGULAR = {("FULL_OPENCV", "focal_extra")}


def skip_near_singular(case, config):
    if (case, config) in NEAR_SINGULAR:
        pytest.skip("J^T J near-singular (cond ~ 1e15): a conditioning-based tolerance cannot fail here")


def scene(case):
    return E.planted(case, np.random.default_rng(1000 + CASES.index(case)))


def options(config, **kw):
    f, e = E.CONFIGS[config]
    return dict(refine_focal_length=f, refine_extra_params=e, **kw)


def pose_of(res):
    g = res["cam_from_world"]
    x, y, z, w = g.rotation.quat
    return np.array([w, x, y, z]), np.asarray(g.translation, np.float64)


def rigid(q, t):
    return nat.Rigid3d(nat.Rotation3d([q[1], q[2], q[3], q[0]]), np.asarray(t, np.float64))


def refine_from_start(case, config, **kw):
    """pose_refinement from the identity pose and perturbed camera parameters over all points.
    Returns (problem, start parameters, result, the camera parameters after the call)."""
    cam, X, x2, q_true, t_true, ne = scene(case)
    model = cam["model"]
    ridx = E.refined_idxs(model, *E.CONFIGS[config])
    p0 = E.perturbed_params(case, ridx)
    mine = dict(cam, params=list(p0))
    out = nat.pose_refinement(rigid(Q0, T0), x2, X, np.ones(len(X), bool), mine, options(config, **kw))
    return E.Problem(model, X, x2, ridx), p0, out, np.array(mine["params"], np.float64)


def scaled_cond(A):
    """Condition number after unit-diagonal scaling, over the unknowns the cost depends on (a zero column of J, as
    omega's below |omega| = 1e-8, decouples and does not amplify rounding in the others)."""
    keep = np.diag(A) > 0
    s = np.sqrt(np.diag(A)[keep])
    return float(np.linalg.cond(A[np.ix_(keep, keep)] / np.outer(s, s)))


@pytest.mark.parametrize("config", CONFIGS)
@pytest.mark.parametrize("case", CASES)
def test_covariance_equals_the_exact_reference(case, config):
    skip_near_singular(case, config)
    cam, X, x2, q_true, t_true, ne = scene(case)
    model = cam["model"]
    ridx = E.refined_idxs(model, *E.CONFIGS[config])
    mine = dict(cam, params=list(cam["params"]))
    got = nat.absolute_pose_estimation(x2, X, mine, refinement_options=options(config), return_covariance=True)
    if case == "FOV_OMEGA_1E-9" and config == "focal_extra":
        # |omega| < 1e-8: the projection does not depend on omega, J^T J is singular and there is no covariance
        assert got is None
        return
    assert got is not None
    inl = np.asarray(got["inliers"], bool)
    assert inl.sum() >= 0.98 * len(X)
    q, t = pose_of(got)
    p = np.array(mine["params"], np.float64)
    assert all(p[i] == cam["params"][i] for i in range(len(p)) if i not in ridx)
    C_ref, A = E.Problem(model, X[inl], x2[inl], ridx).covariance(q, t, p)
    C = np.asarray(got["covariance"], np.float64)
    assert np.all(np.isfinite(C)) and np.all(np.isfinite(A))
    d = 1.0 / np.sqrt(np.diag(C_ref))
    err = float(np.abs((C - C_ref) * np.outer(d, d)).max())
    cond = scaled_cond(A)
    assert err <= max(1e-8, 1e-14 * cond), (err, cond)


@pytest.mark.parametrize("config", CONFIGS)
@pytest.mark.parametrize("case", CASES)
def test_one_lm_step_equals_the_exact_reference(case, config):
    skip_near_singular(case, config)
    prob, p0, out, p = refine_from_start(case, config, max_num_iterations=1, gradient_tolerance=0.0)
    assert out is not None
    q, t = pose_of(out)
    cost0, rr, JJ = prob.evaluate(Q0, T0, p0)
    assert np.all(np.isfinite(JJ))
    step, model_change, As = E.lm_step(rr, JJ, 1e4)
    assert model_change > 0
    assert (cost0 - prob.cost(*prob.apply(Q0, T0, p0, step))) / model_change > 1e-3   # the reference accepts it
    assert all(p[i] == p0[i] for i in range(len(p)) if i not in prob.ridx)
    got = np.r_[E.qminus(q, Q0), t - T0, (p - p0)[prob.ridx]]
    assert np.abs(got).max() > 0                                                      # the kernel accepted it
    # compared in the Jacobi-scaled coordinates the trust-region system is solved in
    scale = 1.0 / (1.0 + np.sqrt(np.diag(JJ.T @ JJ)))
    err = float(np.linalg.norm((got - step) / scale) / np.linalg.norm(step / scale))
    assert err <= max(1e-8, 1e-14 * scaled_cond(As)), err


def newton_decrement(rr, JJ):
    """1/2 g^T (J^T J)^+ g: the cost decrease a Gauss-Newton step from here would still predict."""
    g = JJ.T @ rr
    return 0.5 * float(g @ np.linalg.lstsq(JJ.T @ JJ, g, rcond=None)[0])


@pytest.mark.parametrize("config", CONFIGS)
@pytest.mark.parametrize("case", CASES)
def test_refinement_reaches_the_optimum(case, config):
    """Ceres' function tolerance stops LM once a step lowers the cost by <= 1e-6 of it, which leaves a gradient of
    1e-4 to 1e-3 of the initial one (and, for FULL_OPENCV with its eight coefficients, whose numerator and denominator
    nearly cancel, a cost about 1 % above the minimum).  So the kernel is held to the restated iteration, which has
    the same stopping rules and an exact Jacobian: its cost within 1 + 2e-6 of that iteration's, its Newton
    decrement no larger than 2e-6 of the cost or 10 x the iteration's, and its cost no lower than the minimum."""
    prob, p0, out, p = refine_from_start(case, config, gradient_tolerance=1e-10)
    assert out is not None
    q, t = pose_of(out)
    cost, rr, JJ = prob.evaluate(q, t, p)
    assert np.all(np.isfinite(JJ))
    qr, tr, pr, cost_r, steps = E.minimise(prob, Q0, T0, p0, gradient_tolerance=1e-10)
    *_, best, _ = E.minimise(prob, Q0, T0, p0, max_iterations=200, function_tolerance=0.0)
    assert steps >= 3
    assert best * (1 - 1e-9) <= cost <= (1 + 2e-6) * cost_r, (cost, cost_r, best)
    _, rr_r, JJ_r = prob.evaluate(qr, tr, pr)
    assert newton_decrement(rr, JJ) <= max(2e-6 * cost, 10 * newton_decrement(rr_r, JJ_r))
    g0 = np.abs(prob.gradient(Q0, T0, p0)).max()
    assert np.abs(JJ.T @ rr).max() <= 1e-2 * g0
