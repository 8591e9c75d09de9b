"""Pin the oracle's linear algebra against an INDEPENDENT dense numpy derivation of the same LM inner step.

The reference cannot be built here and ships no golden vectors ("parity unpinned", DESIGN.md section 6). What can be
done without it: derive, from the per-observation Jacobians alone, what LinearizorQR must produce using nothing but
dense textbook algebra in float64 numpy (no QR, no landmark blocks, no PCG), with the per-observation Jacobians from the
independent camera model of tests/camera_model.py (on the benign stand-in and once with real lens distortion), and require the oracle's
stage 1 / stage 2 / PCG / back-substitution pipeline (Householder and Givens, both preconditioners, staged and
un-staged) to reproduce it.  The algebra (Demmel et al., "Square Root Bundle Adjustment", eq. 9-17; reference
qr/impl/landmark_block_base.ipp):

  Jp_s = Jp * D,  D = diag(1 / (eps + ||Jp[:, j]||))                    (linearizor_qr.cpp:130-132, ipp:589-614)
  Jl_s = Jl * diag(1 / (eps + ||Jl[:, j]||)) per landmark               (ipp:571-587)
  with landmark damping lambda:  M = Jl_s^T Jl_s + lambda I  (per landmark, 3x3)
  H   = Jp_s^T Jp_s - Jp_s^T Jl_s M^-1 Jl_s^T Jp_s + lambda I           ((Q2^T Jp)^T (Q2^T Jp) + pose damping)
  b   = Jp_s^T r    - Jp_s^T Jl_s M^-1 Jl_s^T r                         ((Q2^T Jp)^T Q2^T r)
  inc = -H^-1 b                                                         (PCG solves H (-x) = b, linearizor_base.cpp:81-103)
  dl_s = -M^-1 (Jl_s^T r + Jl_s^T Jp_s inc),  p_w += scale_l * dl_s     (ipp:212-284)
  l_diff = 1/2 |r|^2 - 1/2 |r + Jp_s inc + Jl_s dl_s|^2                 (ipp:255-262: model cost change, un-damped)
"""
import numpy as np
import pytest

import camera_model as cm
from conftest import rel_err
from oracle import oracle_py as orc


def _dense_system(prob):
    """dense Jacobians and residual (float64) of the whole problem from the independent camera model (tests/camera_model.py),
    so that neither side of the comparison takes its linearisation from the oracle"""
    nobs, nc, nl = prob.nobs, prob.nc, prob.nl
    jp, jl, res, _ = cm.weighted(prob)
    Jp = np.zeros((2 * nobs, 9 * nc))
    Jl = np.zeros((2 * nobs, 3 * nl))
    lm_of_obs = np.repeat(np.arange(nl), np.diff(prob.lm_off))
    for k in range(nobs):
        c, l = int(prob.obs_cam[k]), int(lm_of_obs[k])
        Jp[2 * k:2 * k + 2, 9 * c:9 * c + 9] = jp[k]
        Jl[2 * k:2 * k + 2, 3 * l:3 * l + 3] = jl[k]
    return Jp, Jl, res.ravel()


def _problem(kind):
    """the benign stand-in, or the same shape with real lens distortion and a wide field of view"""
    from rootba_b200.synthetic import synth_bal
    if kind == "distorted":
        return synth_bal(7, 90, 3.6, seed=21, k1_sigma=0.1, k2_sigma=0.02, max_tan=1.4)
    return synth_bal(7, 90, 3.6, seed=21)


def _reduced(Jp, Jl, r, lam, nl, eps):
    D = 1.0 / (eps + np.linalg.norm(Jp, axis=0))
    sl = 1.0 / (eps + np.linalg.norm(Jl, axis=0))
    Jps, Jls = Jp * D, Jl * sl
    Minv = np.zeros((3 * nl, 3 * nl))
    for l in range(nl):
        B = Jls[:, 3 * l:3 * l + 3]
        Minv[3 * l:3 * l + 3, 3 * l:3 * l + 3] = np.linalg.inv(B.T @ B + lam * np.eye(3))
    W = Jps.T @ Jls
    H = Jps.T @ Jps - W @ Minv @ W.T + lam * np.eye(Jp.shape[1])
    b = Jps.T @ r - W @ Minv @ (Jls.T @ r)
    return D, sl, Jps, Jls, Minv, H, b


@pytest.fixture(scope="module")
def dense_case():
    prob = _problem("benign")
    return prob, _dense_system(prob)


@pytest.fixture(scope="module")
def distorted_case():
    prob = _problem("distorted")
    return prob, _dense_system(prob)


@pytest.mark.parametrize("use_householder", [1, 0])
@pytest.mark.parametrize("precond", [1, 0])
@pytest.mark.parametrize("staged", [1, 0])
def test_lm_inner_step_matches_dense_normal_equations(dense_case, use_householder, precond, staged):
    _check_lm_inner_step(dense_case, use_householder, precond, staged)


@pytest.mark.parametrize("use_householder", [1, 0])
@pytest.mark.parametrize("precond", [1, 0])
@pytest.mark.parametrize("staged", [1, 0])
def test_lm_inner_step_matches_dense_normal_equations_with_distortion(distorted_case, use_householder, precond, staged):
    """the same derivation on a problem with real lens distortion (|k1| ~ 0.1, |x/z| <= 1.4)"""
    _check_lm_inner_step(distorted_case, use_householder, precond, staged)


def _check_lm_inner_step(case, use_householder, precond, staged):
    prob, (Jp, Jl, r) = case
    lam = 1e-3
    eps = float(np.sqrt(1e-10))  # Sophus::Constants<double>::epsilonSqrt(), linearizor_base.cpp:72-79
    D, sl, Jps, Jls, Minv, H, b = _reduced(Jp, Jl, r, lam, prob.nl, eps)
    # eta tiny + many iterations: PCG runs to the solution of the linear system instead of the truncated-Newton stop
    opts = orc.default_options(use_householder=use_householder, preconditioner_type=precond, staged_execution=staged,
                               eta=1e-15, max_linear_solver_iterations=4000, num_threads=1)
    o = orc.Oracle(prob, np.float64, opts)
    assert o.compute_error()["all"]["error"] == pytest.approx(0.5 * r @ r, rel=1e-13)
    assert o.linearize()
    assert rel_err(o.get_scaling(), D) < 1e-13
    inc, dbg = o.solve(lam, want_debug=True)
    assert rel_err(dbg["b"], b) < 1e-11
    x = np.random.default_rng(1).uniform(-1, 1, H.shape[0])
    assert rel_err(o.right_multiply(x), H @ x) < 1e-11
    # block-Jacobi preconditioner = inverse of the diagonal blocks of H (SCHUR_JACOBI) or of D Jp^T Jp D + lambda I (JACOBI)
    Hp = H if precond == 1 else Jps.T @ Jps + lam * np.eye(H.shape[0])
    for c in range(prob.nc):
        blk = Hp[9 * c:9 * c + 9, 9 * c:9 * c + 9]
        assert rel_err(dbg["inv_blocks"][c], np.linalg.inv(blk)) < 1e-8, c
    want_inc = -np.linalg.solve(H, b)
    assert rel_err(inc, want_inc) < 1e-8 * np.linalg.cond(H) ** 0.5
    # back substitution + state update with the SAME increment on both sides
    dl_s = -Minv @ (Jls.T @ r + Jls.T @ (Jps @ inc))
    want_l = 0.5 * r @ r - 0.5 * np.sum((r + Jps @ inc + Jls @ dl_s) ** 2)
    l_diff = o.apply(inc)
    assert l_diff == pytest.approx(want_l, rel=1e-9)
    cams_new, lms_new = o.get_state()
    assert rel_err(lms_new, prob.lms + (sl * dl_s).reshape(-1, 3)) < 1e-12
    # cameras: T <- se3_expd(inc_pose) * T, intrinsics += inc_intr with the UN-scaled increment (linearizor_qr.cpp:279-287)
    d = (D * inc).reshape(-1, 9)
    for c in range(prob.nc):
        assert np.allclose(cams_new[c, 7:10], prob.cams[c, 7:10] + d[c, 6:9], rtol=1e-13, atol=1e-15)
        assert rel_err(cams_new[c], orc.camera_apply_inc(prob.cams[c], d[c])) < 1e-14


def test_first_order_model_predicts_the_true_cost_change(dense_case):
    """ties the linear algebra to the nonlinear problem: for a small step the model decrease l_diff (ipp:255-262) must
    match the true decrease of the cost (bal_bundle_adjustment.cpp:430-446: step_quality = f_diff / l_diff -> 1)"""
    _check_first_order_model(dense_case)


def test_first_order_model_predicts_the_true_cost_change_with_distortion(distorted_case):
    _check_first_order_model(distorted_case)


def _check_first_order_model(case):
    prob, _ = case
    o = orc.Oracle(prob, np.float64, orc.default_options(num_threads=1))
    e0 = o.compute_error()["all"]["error"]
    assert o.linearize()
    inc, _ = o.solve(1e4)  # heavy damping = short gradient-like step: the quadratic model is accurate
    l_diff = o.apply(inc)
    e1 = o.compute_error()["all"]["error"]
    assert l_diff > 0 and e0 > e1
    assert (e0 - e1) / l_diff == pytest.approx(1.0, abs=5e-2)


def test_sc_and_power_sc_linearizors_match_dense_normal_equations(dense_case):
    _check_sc_and_power_sc(dense_case)


def test_sc_and_power_sc_linearizors_match_dense_normal_equations_with_distortion(distorted_case):
    _check_sc_and_power_sc(distorted_case)


def _check_sc_and_power_sc(case):
    """the Schur-complement and Power-SC restatements (the checkers of tests/test_gpu_sc.py; reference
    solver/linearizor_sc.cpp, solver/linearizor_power_sc.cpp, sc/linearization_power_sc.hpp:92-160) against the same dense
    derivation:  H = Hpp + lambda I - E0,  Hpp = Jp_s^T Jp_s (block diagonal),  E0 = W M^-1 W^T,
    power series  x_m = sum_{i=0..m} ((Hpp + lambda I)^-1 E0)^i (Hpp + lambda I)^-1 (-b)  ->  -H^-1 b
    These are the properties the reference's own tests check between its classes -- sc/linearization_power_sc.test.cpp:67-137
    (Hpp^-1 == inverted JACOBI blocks), :142-211 (b and the product of PowerSC == explicit SC), :214-300 (solve for m = 0 and
    m = 5 == the series written out), cg/preconditioner.test.cpp:59-136 -- here against dense numpy instead of against each other."""
    prob, (Jp, Jl, r) = case
    lam = 1e-3
    eps = float(np.sqrt(1e-10))
    D, sl, Jps, Jls, Minv, H, b = _reduced(Jp, Jl, r, lam, prob.nl, eps)
    N = H.shape[0]
    W = Jps.T @ Jls
    E0 = W @ Minv @ W.T
    Hpp_inv = np.linalg.inv(Jps.T @ Jps + lam * np.eye(N))  # block diagonal: one 9x9 block per camera
    opts = orc.default_options(eta=1e-15, max_linear_solver_iterations=4000, num_threads=1)
    o = orc.Oracle(prob, np.float64, opts)
    o.compute_error()
    o.scl_linearize()
    assert rel_err(o.scl_get_scaling(), D) < 1e-13
    x = np.random.default_rng(2).uniform(-1, 1, N)
    # Schur-complement solver: same b, same block-Jacobi preconditioner, same solution as the dense system
    inc, dbg = o.scl_solve(lam)
    assert rel_err(dbg["b"], b) < 1e-11
    for c in range(prob.nc):
        assert rel_err(dbg["inv_blocks"][c], np.linalg.inv(H[9 * c:9 * c + 9, 9 * c:9 * c + 9])) < 1e-8, c
    want_inc = -np.linalg.solve(H, b)
    assert rel_err(inc, want_inc) < 1e-8 * np.linalg.cond(H) ** 0.5
    # E0 alone (the operator of the power series)
    assert rel_err(o.scl_e0(lam, x), E0 @ x) < 1e-11
    # truncated power series, term by term
    term = Hpp_inv @ (-b)
    acc = term.copy()
    partial = {0: acc.copy()}
    for i in range(1, 41):
        term = Hpp_inv @ (E0 @ term)
        acc = acc + term
        partial[i] = acc.copy()
    for m in (0, 1, 5, 40):
        inc_m, d = o.scl_power_solve(lam, power_order=m, q_tolerance=0.0)
        assert rel_err(d["b"], b) < 1e-11
        assert rel_err(inc_m, partial[m]) < 1e-10, m
    # the series converges towards the exact solution (spectral radius of Hpp^-1 E0 < 1), monotonically in the H-norm
    errs = [np.sqrt((partial[m] - want_inc) @ H @ (partial[m] - want_inc)) for m in (0, 5, 40)]
    assert errs[0] > errs[1] > errs[2]
    # the reference's stopping rule  zeta = i |term_i| / |sum| < q_tolerance  (linearization_power_sc.hpp:147-156)
    inc_q, dq = o.scl_power_solve(lam, power_order=40, q_tolerance=0.1)
    term = Hpp_inv @ (-b); acc = term.copy(); stop = 40
    for i in range(1, 41):
        term = Hpp_inv @ (E0 @ term); acc = acc + term
        if i * np.linalg.norm(term) / np.linalg.norm(acc) < 0.1:
            stop = i
            break
    assert dq["power_order"] == stop and dq["termination"] == (1 if stop < 40 else 0)
    assert rel_err(inc_q, acc) < 1e-10
    # back substitution of the SC linearizor: model decrease and landmark update as in the dense derivation
    inc, _ = o.scl_solve(lam)
    dl_s = -Minv @ (Jls.T @ r + Jls.T @ (Jps @ inc))
    want_l = 0.5 * r @ r - 0.5 * np.sum((r + Jps @ inc + Jls @ dl_s) ** 2)
    assert o.scl_apply(inc) == pytest.approx(want_l, rel=1e-9)
    _, lms_new = o.get_state()
    assert rel_err(lms_new, prob.lms + (sl * dl_s).reshape(-1, 3)) < 1e-12
