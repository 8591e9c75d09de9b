"""The landmark-prior model (tests/landmark_prior_model.py) on the CPU: the total objective against central differences, the
dense LM step against the true cost change, the compression [L~; sqrt(lambda) I] -> C and its fold into the landmark's R
against dense elimination, and the checkers against planted faults."""
import numpy as np
import pytest

import landmark_prior_model as lp
from objective_checks import dense_system, total_cost

EPS = 1e-5  # the float64 Jacobi-scaling epsilon


@pytest.fixture(scope="module")
def case():
    from rootba_b200.synthetic import synth_bal
    prob = synth_bal(6, 40, 3.5, seed=11)
    return prob, lp.prior_case(prob.lms, every=2, seed=3)


def _cost_at(prob, lms, prior):
    from rootba_b200.synthetic import BalArrays
    return total_cost(BalArrays(prob.cams, lms, prob.lm_off, prob.obs_cam, prob.obs_xy), landmarks=prior)


def test_landmark_jacobian_of_the_total_objective_matches_central_differences(case):
    """the gradient J^T r of the dense system (reprojection + prior rows) in the landmark columns against central differences
    of the total cost"""
    prob, prior = case
    Jp, Jl, r = dense_system(prob, landmarks=prior)
    grad = Jl.T @ r
    h = 1e-6
    for l in list(prior[0][:4]) + [1, 3]:
        for k in range(3):
            lp_, lm_ = np.array(prob.lms, np.float64), np.array(prob.lms, np.float64)
            lp_[l, k] += h
            lm_[l, k] -= h
            fd = (_cost_at(prob, lp_, prior) - _cost_at(prob, lm_, prior)) / (2 * h)
            assert abs(fd - grad[3 * l + k]) <= 1e-6 * max(1.0, abs(fd)), (l, k, fd, grad[3 * l + k])


def test_cost_is_half_the_squared_whitened_residual(case):
    prob, (idx, mean, L) = case
    e = np.asarray(prob.lms, np.float64)[idx] - mean
    assert lp.cost(prob.lms, idx, mean, L) == pytest.approx(0.5 * sum(np.sum((L[p] @ e[p]) ** 2) for p in range(len(idx))), rel=1e-14)
    # a height-only prior sees nothing but the height
    p = 1
    assert np.count_nonzero(L[p]) == 1 and L[p][2, 2] != 0


def test_dense_lm_step_predicts_the_true_cost_change(case):
    """with a tiny lambda the model change l_diff of the scaled step equals the true change of the total cost to second order"""
    from rootba_b200.synthetic import BalArrays
    import camera_prior_model as pm
    prob, prior = case
    Jp, Jl, r = dense_system(prob, landmarks=prior)
    dp, dl, l_diff, D, sl = lp.lm_step(Jp, Jl, r, 1e-6, EPS)
    step = 1e-3
    cams = np.array([pm.apply_inc(prob.cams[c], step * D[9 * c:9 * c + 9] * dp[9 * c:9 * c + 9]) for c in range(prob.nc)])
    lms = np.asarray(prob.lms, np.float64) + step * (sl * dl).reshape(-1, 3)
    true = total_cost(prob, landmarks=prior) - total_cost(BalArrays(cams, lms, prob.lm_off, prob.obs_cam, prob.obs_xy), landmarks=prior)
    Js = np.hstack([Jp * D, Jl * sl])
    d = np.concatenate([dp, dl])
    model = -(step * (Js @ d) @ r + 0.5 * step ** 2 * np.sum((Js @ d) ** 2))
    assert abs(true - model) <= 1e-4 * abs(model), (true, model)
    assert l_diff > 0


def test_prior_columns_enter_the_jacobi_scaling(case):
    prob, prior = case
    Jp, Jl, r = dense_system(prob, landmarks=prior)
    from test_oracle_dense_numpy import _dense_system
    _, Jl0, _ = _dense_system(prob)
    idx, _, L = prior
    _, sl = lp.scaling(Jp, Jl, EPS)
    for p, l in enumerate(idx):
        want = 1.0 / (EPS + np.sqrt(np.sum(Jl0[:, 3 * l:3 * l + 3] ** 2, axis=0) + np.sum(L[p] ** 2, axis=0)))
        assert np.allclose(sl[3 * l:3 * l + 3], want, rtol=1e-14)


def _landmark_case(seed, kind="dense", lam=1e-3):
    """one landmark: Jl (2n x 3), r, a prior (L~, g) in its scaled space"""
    rng = np.random.default_rng(seed)
    n = 4
    Jl = rng.standard_normal((2 * n, 3))
    r = rng.standard_normal(2 * n)
    Lt = lp.sqrt_info_kind(kind, rng) * rng.uniform(0.5, 2.0, 3)
    g = rng.standard_normal(3)
    return Jl, r, Lt, g, lam


@pytest.mark.parametrize("lam", [0.0, 1e-3, 10.0])
@pytest.mark.parametrize("kind", ["dense", "height", "rank2", "none"])
def test_compression_preserves_the_gram_matrix_and_the_projected_residual(kind, lam):
    _, _, Lt, g, _ = _landmark_case(5, kind)
    C, c = lp.compress(Lt, g, lam)
    assert np.allclose(np.tril(C, -1), 0)
    assert np.allclose(C.T @ C, Lt.T @ Lt + lam * np.eye(3), atol=1e-12)
    assert np.allclose(C.T @ c, Lt.T @ g, atol=1e-12)


def _check_fold(Jl, r, Lt, g, lam, C, c):
    """the checker: R, rr after "QR of [Jl | r], then the 6 rotations with [C | c]" must be the dense elimination of the
    landmark, R^T R = Jl^T Jl + L~^T L~ + lam I and R^T rr = Jl^T r + L~^T g"""
    Q, R0 = np.linalg.qr(Jl)
    rr0 = Q.T @ r
    R, rr, Dw, _ = lp.fold_damping(R0, rr0, C, c)
    ok_rot = np.allclose(np.triu(Dw), 0, atol=1e-12) and np.allclose(np.tril(R, -1), 0, atol=1e-12)
    H = Jl.T @ Jl + Lt.T @ Lt + lam * np.eye(3)
    return ok_rot and np.allclose(R.T @ R, H, rtol=1e-10, atol=1e-12) and np.allclose(R.T @ rr, Jl.T @ r + Lt.T @ g, rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize("lam", [0.0, 1e-3, 10.0])
@pytest.mark.parametrize("kind", ["dense", "height", "rank2"])
def test_compress_then_fold_equals_dense_elimination(kind, lam):
    Jl, r, Lt, g, _ = _landmark_case(9, kind)
    C, c = lp.compress(Lt, g, lam)
    assert _check_fold(Jl, r, Lt, g, lam, C, c)
    # and the landmark step of the folded factors is that of the dense normal equations
    Q, R0 = np.linalg.qr(Jl)
    R, rr, _, _ = lp.fold_damping(R0, Q.T @ r, C, c)
    assert np.allclose(-np.linalg.solve(R, rr), -np.linalg.solve(Jl.T @ Jl + Lt.T @ Lt + lam * np.eye(3), Jl.T @ r + Lt.T @ g))


@pytest.mark.parametrize("fault", ["no_lambda", "g_sign"])
def test_fold_checker_rejects_planted_faults(fault):
    Jl, r, Lt, g, lam = _landmark_case(13, "dense", lam=0.5)
    assert not _check_fold(Jl, r, Lt, g, lam, *lp.compress(Lt, g, lam, fault=fault))


def test_scaling_checker_rejects_L_without_the_landmark_scaling(case):
    """the step from the prior rows scaled by diag(jls) is the model's; one with L taken as is in the scaled space is not"""
    prob, prior = case
    Jp, Jl, r = dense_system(prob, landmarks=prior)
    lam = 1e-3
    dp, dl, l_diff, D, sl = lp.lm_step(Jp, Jl, r, lam, EPS)
    # the faulty variant: the reprojection part scaled, the prior rows' landmark columns not
    nobs_rows = Jp.shape[0] - 3 * len(prior[0])
    Js = np.hstack([Jp * D, Jl * sl])
    Js[nobs_rows:, Jp.shape[1]:] = Jl[nobs_rows:]
    d_bad = -np.linalg.solve(Js.T @ Js + lam * np.eye(Js.shape[1]), Js.T @ r)
    d = np.concatenate([dp, dl])
    assert np.linalg.norm(d_bad - d) > 1e-3 * np.linalg.norm(d)


def test_cost_checker_rejects_the_prior_cost_counted_once_per_rank():
    reproj, priors = [10.0, 12.5], [0.75, 1.25]
    want = sum(reproj) + sum(priors)
    assert lp.sharded_cost(reproj, priors) == want
    assert abs(lp.sharded_cost(reproj, priors, per_rank_all_priors=True) - want) > 1e-9 * want
