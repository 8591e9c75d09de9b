"""The camera-prior model (tests/camera_prior_model.py) on the CPU: its Jacobian against central differences through the
actual increment map, and the dense LM step of the total (reprojection + prior) problem against the true cost change."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import camera_prior_model as pm


def _camera_and_mean(angle, seed):
    """a camera whose rotation is `angle` rad away from the prior mean's"""
    rng = np.random.default_rng(seed)
    R0 = Rotation.from_rotvec(rng.uniform(-1, 1, 3))
    axis = rng.standard_normal(3)
    axis /= np.linalg.norm(axis)
    R = Rotation.from_rotvec(angle * axis) * R0
    cam = np.concatenate([R.as_quat(), rng.uniform(-2, 2, 3), [500.0 + rng.uniform(-5, 5), 0.05, -0.01]])
    mean = np.concatenate([R0.as_quat(), rng.uniform(-2, 2, 3), [505.0, 0.0, 0.0]])
    return cam, mean


@pytest.mark.parametrize("angle", [0.0, 1e-9, 1e-4, 0.3, 1.5, 2.5, 3.0])
@pytest.mark.parametrize("kind", ["dense", "centre", "intrinsics"])
def test_jacobian_matches_central_differences_through_the_increment_map(angle, kind):
    cam, mean = _camera_and_mean(angle, seed=int(angle * 1000) + 7)
    L = pm.sqrt_info_kind(kind, np.random.default_rng(3))
    e0 = pm.residual(cam, mean)
    assert abs(np.linalg.norm(e0[3:6]) - angle) < 1e-9
    J = L @ pm.jacobian(cam, mean)
    h = 1e-6
    Jfd = np.zeros((9, 9))
    for j in range(9):
        d = np.zeros(9)
        d[j] = h
        Jfd[:, j] = (L @ pm.residual(pm.apply_inc(cam, d), mean) - L @ pm.residual(pm.apply_inc(cam, -d), mean)) / (2 * h)
    assert np.max(np.abs(J - Jfd)) <= 1e-7 * max(1.0, np.max(np.abs(J))), (J - Jfd)
    # the structure: no centre dependence on the rotation increment, identity on the intrinsics
    Je = pm.jacobian(cam, mean)
    assert np.all(Je[0:3, 3:9] == 0) and np.array_equal(Je[6:9, 6:9], np.eye(3))


def test_cost_is_half_the_squared_whitened_residual():
    cam, mean = _camera_and_mean(0.7, seed=1)
    L = pm.sqrt_info_kind("dense", np.random.default_rng(5))
    e = pm.residual(cam, mean)
    assert pm.cost(cam[None], mean[None], L[None]) == pytest.approx(0.5 * np.sum((L @ e) ** 2), rel=1e-14)
    assert np.allclose(e[:3], pm.centre(cam) - mean[4:7]) and np.allclose(e[6:], cam[7:] - mean[7:])
    # a prior at the camera itself has zero residual
    assert np.allclose(pm.residual(cam, pm.mean_at(cam[None])[0]), 0, atol=1e-12)


def test_first_order_model_of_the_total_objective_predicts_the_true_cost_change():
    """the dense LM step of the total problem (scaling over reprojection + prior columns, H, b, inc, l_diff): for a heavily
    damped step the model decrease matches the true decrease of reprojection + prior cost"""
    from rootba_b200.synthetic import BalArrays
    from objective_checks import dense_system, total_cost
    from test_oracle_dense_numpy import _reduced
    prob, mean, L = pm.prior_case()
    Jp, Jl, r = dense_system(prob, camera=(mean, L))
    lam = 1e4
    D, sl, Jps, Jls, Minv, H, b = _reduced(Jp, Jl, r, lam, prob.nl, float(np.sqrt(1e-10)))
    assert np.all(D[-9:] < 1e3)  # the unobserved camera is scaled by its prior, not by 1 / eps
    inc = -np.linalg.solve(H, b)
    dl_s = -Minv @ (Jls.T @ r + Jls.T @ (Jps @ inc))
    l_diff = 0.5 * r @ r - 0.5 * np.sum((r + Jps @ inc + Jls @ dl_s) ** 2)
    e0 = total_cost(prob, camera=(mean, L))
    assert 0.5 * r @ r == pytest.approx(e0, rel=1e-12)
    d = (D * inc).reshape(-1, 9)
    cams1 = np.stack([pm.apply_inc(prob.cams[c], d[c]) for c in range(prob.nc)])
    lms1 = np.asarray(prob.lms) + (sl * dl_s).reshape(-1, 3)
    e1 = total_cost(BalArrays(cams1, lms1, prob.lm_off, prob.obs_cam, prob.obs_xy), camera=(mean, L))
    assert l_diff > 0 and e0 > e1
    assert (e0 - e1) / l_diff == pytest.approx(1.0, abs=5e-2)
