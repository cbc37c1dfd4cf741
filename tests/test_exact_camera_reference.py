"""CPU self-check of tests/helpers/exact_camera.py, the exact reference that test_zz_abs_pose_numerics_gpu.py holds the
refinement kernel to: its projections equal the oracle's ImgFromCam, its sympy derivatives (camera and pose chain rule)
equal Richardson-extrapolated central differences, its float64 evaluation equals a 40-digit mpmath evaluation, and
its LM restatement converges from the start the GPU tests use."""
import numpy as np
import pytest

from helpers import exact_camera as E
from oracle import ransac as R

CASES = list(E.CASES)


def scene_points(case, n=40):
    cam, X, x2, q, t, ne = E.planted(case, np.random.default_rng(7), n=n)
    return cam, X[:, :2] / X[:, 2:]   # normalised coordinates at the identity pose, edge points included


def richardson(f, x, h):
    d1 = (f(x + h) - f(x - h)) / (2 * h)
    d2 = (f(x + h / 2) - f(x - h / 2)) / h
    return (4 * d2 - d1) / 3


@pytest.mark.parametrize("case", CASES)
def test_projection_equals_the_oracle(case):
    cam, uv = scene_points(case)
    pix, _, _ = E.project(cam["model"], cam["params"], uv)
    want = R.img_from_cam(cam, uv)
    assert np.abs(pix - want).max() < 1e-9


@pytest.mark.parametrize("case", CASES)
def test_camera_derivatives_equal_richardson_differences(case):
    cam, uv = scene_points(case)
    model, params = cam["model"], np.array(cam["params"])
    _, duv, dp = E.project(model, params, uv)
    for a in range(2):
        e = np.zeros(2)
        e[a] = 1.0
        num = richardson(lambda s: E.project(model, params, uv + s * e)[0], 0.0, 1e-4)
        assert np.abs(num - duv[:, :, a]).max() <= 1e-8 * E.F, a
    for i in range(len(params)):
        if case == "FOV_OMEGA_1E-9" and i == 4:
            # |omega| < 1e-8: the model is the identity (factor 1), so d/d omega is exactly 0 there
            assert np.all(dp[:, :, i] == 0.0)
            continue
        e = np.zeros(len(params))
        h = 1e-4 * max(1.0, abs(params[i]))
        e[i] = 1.0
        num = richardson(lambda s: E.project(model, params + s * e, uv)[0], 0.0, h)
        assert np.abs(num - dp[:, :, i]).max() <= 1e-6, i


@pytest.mark.parametrize("case", CASES)
def test_pose_jacobian_equals_richardson_differences(case):
    cam, X, x2, q_true, t_true, ne = E.planted(case, np.random.default_rng(11), n=40)
    model, params = cam["model"], np.array(cam["params"])
    ridx = E.refined_idxs(model, True, case != "FOV_OMEGA_1E-9")
    q, t = q_true, t_true
    r0, J = E.residuals_and_jacobian(model, params, q, t, X, x2, ridx)
    assert np.all(np.isfinite(J))

    def res(d):
        qn, tn, pn = E.Problem(model, X, x2, ridx).apply(q, t, params, d)
        return E.residuals_and_jacobian(model, pn, qn, tn, X, x2, [])[0]
    for c in range(J.shape[2]):
        e = np.zeros(J.shape[2])
        e[c] = 1.0
        h = 1e-5 if c < 6 else 1e-4 * max(1.0, abs(params[ridx[c - 6]]))
        num = richardson(lambda s: res(s * e), 0.0, h)
        scale = max(1.0, np.abs(J[:, :, c]).max())
        assert np.abs(num - J[:, :, c]).max() <= 1e-7 * scale, c


@pytest.mark.parametrize("case", CASES)
def test_float64_evaluation_equals_mpmath(case):
    cam, uv = scene_points(case, n=4)
    model, params = cam["model"], cam["params"]
    pix, duv, dp = E.project(model, params, uv)
    n = len(params)
    for m in range(len(uv)):
        want = np.array([float(v) for v in E.project_mp(model, params, uv[m, 0], uv[m, 1])])
        got = np.r_[pix[m], duv[m].reshape(-1), dp[m, 0], dp[m, 1]]
        assert got.shape == want.shape == (6 + 2 * n,)
        assert np.all(np.abs(got - want) <= 1e-12 * (np.abs(want) + E.F)), m


def test_restated_lm_step_decreases_the_cost():
    """One step of the LM restatement from the perturbed start of the GPU tests is accepted and lowers the cost."""
    cam, X, x2, q_true, t_true, ne = E.planted("OPENCV", np.random.default_rng(3))
    ridx = E.refined_idxs(4, True, True)
    prob = E.Problem(4, X, x2, ridx)
    q0, t0, p0 = np.array([1.0, 0, 0, 0]), np.zeros(3), E.perturbed_params("OPENCV", ridx)
    cost0, rr, JJ = prob.evaluate(q0, t0, p0)
    step, mc, _ = E.lm_step(rr, JJ, 1e4)
    assert mc > 0 and (cost0 - prob.cost(*prob.apply(q0, t0, p0, step))) / mc > 0.5
    q, t, p, cost, acc = E.minimise(prob, q0, t0, p0, gradient_tolerance=1e-10)
    assert acc >= 3 and cost < 0.1 * cost0
    # within pixel noise of the true pose, which is 0.004 / 0.05 from the start
    assert np.linalg.norm(E.qminus(q, q_true)) < 1e-3 and np.linalg.norm(t - t_true) < 1e-2
