"""The pair-prior model (tests/pair_prior_model.py) on the CPU: its Jacobian against central differences through the actual
increment map, the dense LM step of the total (reprojection + absolute + pair prior) problem against the true cost change,
and the convergence argument of the power series on Hpp^-1 (E_0 - O) (DESIGN.md section 15)."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import camera_model as cm
import camera_prior_model as pm
import pair_prior_model as qm


def _pair_and_mean(angle, seed):
    """two cameras whose relative rotation is `angle` rad away from the mean's"""
    rng = np.random.default_rng(seed)
    Ri, Rj = Rotation.from_rotvec(rng.uniform(-1, 1, 3)), Rotation.from_rotvec(rng.uniform(-1, 1, 3))
    ci = np.concatenate([Ri.as_quat(), rng.uniform(-2, 2, 3), [500.0, 0.01, 0.0]])
    cj = np.concatenate([Rj.as_quat(), rng.uniform(-2, 2, 3), [510.0, 0.0, 0.02]])
    axis = rng.standard_normal(3)
    axis /= np.linalg.norm(axis)
    R0 = Rotation.from_rotvec(-angle * axis) * (Ri * Rj.inv())  # Log(Ri Rj^T R0^T) = angle * axis
    mean = np.concatenate([R0.as_quat(), rng.uniform(-1, 1, 3)])
    return ci, cj, mean


@pytest.mark.parametrize("angle", [0.0, 1e-9, 1e-4, 0.3, 1.5, 2.5, 3.0])
@pytest.mark.parametrize("kind", ["dense", "translation", "rotation"])
def test_jacobian_matches_central_differences_through_the_increment_map(angle, kind):
    ci, cj, mean = _pair_and_mean(angle, seed=int(angle * 1000) + 11)
    L = qm.sqrt_info_kind(kind, np.random.default_rng(4))
    e0 = qm.residual(ci, cj, mean)
    assert abs(np.linalg.norm(e0[3:6]) - angle) < 1e-9
    Ji, Jj = qm.jacobians(ci, cj, mean)
    h = 1e-6
    for J, which in ((L @ Ji, 0), (L @ Jj, 1)):
        Jfd = np.zeros((6, 9))
        for k in range(9):
            d = np.zeros(9)
            d[k] = h
            plus = [ci, cj]
            minus = [ci, cj]
            plus[which] = pm.apply_inc(plus[which], d)
            minus[which] = pm.apply_inc(minus[which], -d)
            Jfd[:, k] = (L @ qm.residual(*plus, mean) - L @ qm.residual(*minus, mean)) / (2 * h)
        assert np.max(np.abs(J - Jfd)) <= 1e-7 * max(1.0, np.max(np.abs(J))), (which, J - Jfd)
    # the structure: zero intrinsic columns, d e_t / d w_j = 0, d e_r / d v = 0
    assert np.all(Ji[:, 6:] == 0) and np.all(Jj[:, 6:] == 0)
    assert np.all(Jj[0:3, 3:6] == 0) and np.all(Ji[3:6, 0:3] == 0) and np.all(Jj[3:6, 0:3] == 0)


def test_cost_and_residual_at_the_relative_pose():
    ci, cj, mean = _pair_and_mean(0.7, seed=2)
    L = qm.sqrt_info_kind("dense", np.random.default_rng(5))
    e = qm.residual(ci, cj, mean)
    assert qm.cost(np.stack([ci, cj]), [(0, 1)], mean[None], L[None]) == pytest.approx(0.5 * np.sum((L @ e) ** 2), rel=1e-14)
    # e_t is the centre of j seen from camera i, minus t0
    Ri = cm.rotation(ci[:4])
    assert np.allclose(e[:3], Ri @ (pm.centre(cj) - pm.centre(ci)) - mean[4:7])
    # a prior at the cameras' own relative pose has zero residual
    assert np.allclose(qm.residual(ci, cj, qm.mean_at(np.stack([ci, cj]), [(0, 1)])[0]), 0, atol=1e-12)


def test_first_order_model_of_the_total_objective_predicts_the_true_cost_change():
    """the dense LM step of reprojection + absolute + pair rows (scaling over the whole Jacobian, H, b, inc, l_diff): for a
    heavily damped step the model decrease matches the true decrease of the total cost"""
    from rootba_b200.synthetic import BalArrays
    from objective_checks import dense_system, total_cost
    from test_oracle_dense_numpy import _reduced
    prob, pair = qm.pair_case()
    _, mean_a, L_a = pm.prior_case(7, 90)
    absp = (pm.mean_at(prob.cams), L_a)
    Jp, Jl, r = dense_system(prob, camera=absp, pairs=pair)
    lam = 1e4
    D, sl, Jps, Jls, Minv, H, b = _reduced(Jp, Jl, r, lam, prob.nl, float(np.sqrt(1e-10)))
    inc = -np.linalg.solve(H, b)
    dl_s = -Minv @ (Jls.T @ r + Jls.T @ (Jps @ inc))
    l_diff = 0.5 * r @ r - 0.5 * np.sum((r + Jps @ inc + Jls @ dl_s) ** 2)
    e0 = total_cost(prob, camera=absp, pairs=pair)
    assert 0.5 * r @ r == pytest.approx(e0, rel=1e-12)
    d = (D * inc).reshape(-1, 9)
    cams1 = np.stack([pm.apply_inc(prob.cams[c], d[c]) for c in range(prob.nc)])
    lms1 = np.asarray(prob.lms) + (sl * dl_s).reshape(-1, 3)
    e1 = total_cost(BalArrays(cams1, lms1, prob.lm_off, prob.obs_cam, prob.obs_xy), camera=absp, pairs=pair)
    assert l_diff > 0 and e0 > e1
    assert (e0 - e1) / l_diff == pytest.approx(1.0, abs=5e-2)


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("lam", [1e-6, 1e-2, 1.0])
def test_power_series_on_E0_minus_O_converges_to_the_direct_solve(seed, lam):
    """Hpp - (E_0 - O) and Hpp + (E_0 - O) are both positive definite, so the eigenvalues of Hpp^-1 (E_0 - O) lie in (-1, 1)
    and the series reaches the solve of the total reduced system"""
    from objective_checks import dense_system
    from test_oracle_dense_numpy import _reduced
    rng = np.random.default_rng(100 + seed)
    prob, (pairs, mean, L) = qm.pair_case(6 + seed % 3, 70, seed=200 + seed)
    L = L * rng.uniform(0.5, 20.0)  # weak to strong pair priors
    Jp, Jl, r = dense_system(prob, pairs=(pairs, mean, L))
    D, sl, Jps, Jls, Minv, H, b = _reduced(Jp, Jl, r, lam, prob.nl, float(np.sqrt(1e-10)))
    Hpp, O = qm.power_split(Jps, lam)
    assert np.max(np.abs(O)) > 0
    W = Jps.T @ Jls
    E0mO = W @ Minv @ W.T - O
    assert np.allclose(Hpp - E0mO, H, rtol=0, atol=1e-9 * np.max(np.abs(H)))
    assert np.min(np.linalg.eigvalsh(Hpp - E0mO)) > 0 and np.min(np.linalg.eigvalsh(Hpp + E0mO)) > 0
    rho = np.max(np.abs(np.linalg.eigvals(np.linalg.solve(Hpp, E0mO))))
    assert rho < 1
    if lam < 1e-2:  # the gauge freedom of BA puts rho within 1e-5 of 1: converges, in far more terms than this test runs
        return
    x = qm.power_series(Hpp, E0mO, b, order=200000, eta=1e-14)
    want = -np.linalg.solve(H, b)
    assert np.linalg.norm(x - want) <= 1e-6 * np.linalg.norm(want), rho
