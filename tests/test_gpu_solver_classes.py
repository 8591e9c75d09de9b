"""The Schur-complement solvers and the non-default square-root options at every track-length class of
test_gpu_kernel_classes (CASES, problem(n): W + 1 landmarks of ONE track length n), landmark by landmark and camera by camera.

  SCHUR_COMPLEMENT        k_sc_stage2 (Hll with G lanes per landmark, its Cholesky factor, q1d, rr, the gradient) and the
                          implicit kernels on its q1d, against the float64 model of tests/solver_model.py at its
                          componentwise bars (c u M, c = 2 n + m + 128 + 512 kappa, see that module): b, the SCHUR_JACOBI
                          blocks of get_preconditioner()[1] and their inverse, H x, every landmark's update of
                          rba_back_substitute and l_diff; the PCG count (+-2) and the termination of the oracle's
                          scl_solve.  float64 also runs the reference's own cross-check (qr/linearization_qr.test.cpp:
                          120-222) at every class: the square-root solver (dense, default options) equals SC per camera
                          (b, blocks, H x) and per landmark (update) at 1e-11
  POWER_SCHUR_COMPLEMENT  the inverse of Hpp + lam I per camera against the model at the same bars, then the series
                          truncated at 1, 2 and CONVERGED terms against power_replay on the handle's own get_rhs,
                          get_preconditioner and right_multiply at the bar of test_gpu_pcg_iterates (lam = LAM_POWER,
                          C_BAR k u kappa_b min(k, 1 / (1 - rho))): the e0_only implicit kernels on both sides of the
                          TMA / plain split (W n <= 64)
  SQUARE_ROOT options     stage2_form = IDENTITY (k_stage2<S, false> writing the damping rows into the panels, through
                          shared memory and, from n = 82, global scratch), preconditioner_type = JACOBI
                          (k_precond_partial<0>) and robust_norm = HUBER (a threshold between the residual norms, as
                          test_gpu_observation_model._huber_threshold picks it), each set on the handle and the oracle, with
                          the checks of test_dense_operator_class: every landmark's block incl. the damping rows, H x
                          componentwise from the kernel's own panels, the back-substitution bar, b, the inverse and inc
                          per camera.  The identity form keeps the one-decade-looser float32 bar of the inverse blocks that
                          test_option_branches_single_solve uses (it cancels Jp^T Jp - Q1d^T Q1d).  The JACOBI solve's inc
                          is compared as a whole vector at TOLS, like test_option_branches_single_solve does: with the
                          weaker preconditioner the float32 rounding of PCG reaches 1.3e-4 on single cameras (n = 57,
                          while b, the blocks and the iteration count agree).
  singular landmark block float32 SC at lam = 1e-9 on a landmark with one valid observation (Jl_s^T Jl_s + lam I singular
                          in working precision): NaN from k_sc_stage2's Cholesky reaches b, PCG runs to
                          max_linear_solver_iterations and reports NO_CONVERGENCE (as the reference's CG: is_zero_or_infinity
                          does not catch NaN), rba_apply reports a non-finite l_diff, rba_restore gives back the state bit
                          for bit, and rba_lm_run raises lam and reaches the float64 square-root solver's minimum
"""
import numpy as np
import pytest

import solver_model as sm
from conftest import rel_err
from pcg_replay import NO_CONVERGENCE, power_replay
from test_gpu_kernel_classes import CASES, _case_id, _check_back_substitution, _check_operator_componentwise, _per_camera, \
    problem
from test_gpu_parity import TOL1, TOLB, TOLS, make_pair

pytestmark = pytest.mark.gpu

LAM = 0.1
LAM_POWER = 0.1          # test_gpu_pcg_iterates
C_BAR = 10               # test_gpu_pcg_iterates: 2 u for each of five operations per term
U = {np.float32: 2.0 ** -24, np.float64: 2.0 ** -53}
BAR_MAX = {np.float32: 1e-2, np.float64: 1e-8}
# 60 terms: rho <= 0.9 on these problems, so the last term is below 2e-3 of the first.  Its float32 bar grows with the
# number of terms (~2e-2 at kappa_b ~ 60, rho ~ 0.9), so BAR_MAX guards the truncations at 1 and 2 terms and
# BAR_MAX_CONVERGED this one
CONVERGED = 60
BAR_MAX_CONVERGED = {np.float32: 3e-2, np.float64: 1e-8}


def _handle(arrays, dtype, **opt):
    import rootba_b200 as rb
    bp = rb.BalProblem.from_arrays(arrays, dtype)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(**opt))
    lin.linearize()
    return bp, lin


def _landmark_update(lin, bp, dp):
    lin.download_state()
    lms0 = bp.lms.astype(np.float64)
    l_diff = lin.back_substitute(dp)
    lin.download_state()
    lms1 = bp.lms.astype(np.float64)
    return lms1 - lms0, lms1, l_diff


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("n", CASES, ids=_case_id)
def test_schur_complement_class(n, dtype):
    from oracle import oracle_py as orc
    arrays = problem(n)
    nc = arrays.nc
    bp, lin = _handle(arrays, dtype, solver_type="SCHUR_COMPLEMENT")
    lin.solve(LAM)
    m = sm.SCModel(arrays, dtype, lin.get_jacobian_scaling()[0], LAM)
    if dtype == np.float64:
        assert m.c * m.u <= 1e-9, m.c
    b_g = lin.get_rhs()
    b, Mb = m.b()
    sm.check(b_g, b, Mb, m, "b")
    inv_g, blk_g = lin.get_preconditioner()
    B, MB = m.schur_blocks()
    sm.check(blk_g, B, MB, m, "SCHUR_JACOBI blocks")
    sm.check_inverse(inv_g, B, MB, m, "inverse")
    x = np.random.default_rng(n).uniform(-1, 1, 9 * nc).astype(dtype)
    y_g = lin.right_multiply(x)
    y, My = m.hx(x)
    sm.check(y_g, y, My, m, "H x")
    o = orc.Oracle(arrays, dtype, orc.default_options(num_threads=0))
    o.scl_linearize()
    _, dbg = o.scl_solve(LAM)
    assert abs(lin.last_cg.num_iterations - dbg["cg_iterations"]) <= 2
    assert lin.last_cg.termination_type == dbg["cg_termination"]
    dp = (np.random.default_rng(n + 1).uniform(-1, 1, 9 * nc) * 0.01).astype(dtype)
    got, lms1, l_g = _landmark_update(lin, bp, dp)
    _, _, dl, Mdl, l_diff, Ml = m.back_substitute(dp)
    sm.check_landmark_update(got, m, dl, Mdl, lms1)
    sm.check(l_g, l_diff, Ml, m, "l_diff")
    lin.close()
    if dtype == np.float64:
        # QR == SC (qr/linearization_qr.test.cpp:120-222) between the two CUDA solvers, per camera and per landmark
        bq, qr = _handle(arrays, dtype)
        qr.solve(LAM)
        _per_camera(qr.get_rhs(), b_g, nc, 1e-11, "b")
        _per_camera(qr.get_preconditioner()[1], blk_g, nc, 1e-11, "blocks")
        _per_camera(qr.right_multiply(x), y_g, nc, 1e-11, "H x")
        got_q, _, _ = _landmark_update(qr, bq, dp)
        for lm in range(arrays.nl):
            assert rel_err(got_q[lm], got[lm]) < 1e-11, ("landmark update", lm)
        qr.close()


def _power_solve(arrays, dtype, order):
    _, lin = _handle(arrays, dtype, solver_type="POWER_SCHUR_COMPLEMENT", power_order=order, eta=0.0)
    inc = lin.solve(LAM_POWER)
    out = (inc, lin.last_cg.termination_type, lin.last_cg.num_iterations, lin.get_rhs(), lin.get_preconditioner()[0])
    lin.close()
    return out


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("n", CASES, ids=_case_id)
def test_power_schur_complement_class(n, dtype):
    from test_gpu_pcg_iterates import operator_of
    arrays = problem(n)
    _, lin = _handle(arrays, dtype, solver_type="POWER_SCHUR_COMPLEMENT", power_order=CONVERGED, eta=0.0)
    lin.solve(LAM_POWER)
    b, inv = lin.get_rhs(), lin.get_preconditioner()[0]
    m = sm.SCModel(arrays, dtype, lin.get_jacobian_scaling()[0], LAM_POWER)
    J, MJ = m.jacobi_blocks()
    sm.check_inverse(inv, J, MJ, m, "inverse of Hpp + lam I")
    full = power_replay(operator_of(lin, dtype), inv, b, order=CONVERGED, eta=0.0)
    lin.close()
    sums = full["sums"]
    d1, d2 = np.linalg.norm(sums[-1] - sums[-2]), np.linalg.norm(sums[-2] - sums[-3])
    rho = d1 / d2 if d2 > 0 else 0.0
    assert rho < 1, rho
    kappa_b = max(np.linalg.cond(blk) for blk in inv.astype(np.float64))
    for k in (1, 2, CONVERGED):
        bar = C_BAR * k * U[dtype] * kappa_b * min(k, 1 / (1 - rho))
        assert bar <= (BAR_MAX_CONVERGED if k == CONVERGED else BAR_MAX)[dtype], (kappa_b, rho, bar)
        inc, term, it, b_k, inv_k = _power_solve(arrays, dtype, k)
        assert np.array_equal(b_k, b) and np.array_equal(inv_k, inv), k
        assert (term, it) == (NO_CONVERGENCE, k), k
        assert rel_err(inc, sums[k]) < bar, (k, rel_err(inc, sums[k]), bar)


OPTIONS = {"identity": {"stage2_form": "IDENTITY"}, "jacobi": {"preconditioner_type": "JACOBI"},
           "huber": {"robust_norm": "HUBER"}}


@pytest.mark.parametrize("option", list(OPTIONS))
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("n", CASES, ids=_case_id)
def test_square_root_option_class(n, dtype, option):
    from test_gpu_observation_model import _huber_threshold
    arrays = problem(n)
    kw = dict(OPTIONS[option])
    if option == "huber":
        kw["huber_parameter"] = _huber_threshold(arrays, dtype)
    bp, lin, o, _ = make_pair(arrays, dtype, **kw)
    tol, nc = TOL1[dtype], arrays.nc
    lin.linearize()
    assert o.linearize()
    inc_g = lin.solve(LAM)
    inc_c, dbg = o.solve(LAM, want_debug=True)
    _per_camera(lin.get_rhs(), dbg["b"], nc, 4 * tol, "b")
    inv_g, _ = lin.get_preconditioner()
    tb = TOLB[dtype] * (10 if option == "identity" and dtype == np.float32 else 1)
    _per_camera(inv_g, dbg["inv_blocks"], nc, tb, "preconditioner inverse")
    assert abs(lin.last_cg.num_iterations - dbg["cg_iterations"]) <= 2
    assert lin.last_cg.termination_type == dbg["cg_termination"]
    if option == "jacobi":  # see the module docstring
        assert rel_err(inc_g, inc_c) < TOLS[dtype]
    else:
        _per_camera(inc_g, inc_c, nc, TOLS[dtype], "inc")
    blocks = []
    for lm in range(arrays.nl):
        bg, lm_idx, res_idx, jls_g = lin.debug_get_block(lm)
        bc, li, ri, jls_c = o.get_block(lm)
        assert (li, ri) == (lm_idx, res_idx) and bg.shape == bc.shape
        assert rel_err(jls_g, jls_c) < tol, lm
        assert rel_err(bg[:3, :9 * n], bc[:3, :9 * n]) < tol * 4, lm
        assert rel_err(np.triu(bg[:3, lm_idx:lm_idx + 3]), np.triu(bc[:3, lm_idx:lm_idx + 3])) < tol * 4, lm
        assert rel_err(bg[:3, res_idx], bc[:3, res_idx]) < tol * 4, lm
        assert rel_err(bg[3:, :9 * n], bc[3:, :9 * n]) < tol * 4, lm  # the damping rows of rows 2n.. included
        blocks.append((bg, lm_idx, res_idx, jls_g))
    _check_operator_componentwise(lin, arrays, dtype, LAM, blocks, n)
    l_g = _check_back_substitution(lin, bp, arrays, dtype, blocks, n)
    l_c, ok = o.back_substitute((np.random.default_rng(n + 1).uniform(-1, 1, 9 * nc) * 0.01).astype(dtype))
    assert ok and abs(l_g - l_c) <= tol * 20 * abs(l_c)
    lin.close()


LAM_SINGULAR = 1e-9  # below the float32 resolution of Hll's unit diagonal: 1 + 1e-9 rounds to 1


def _singular_setup():
    """turned_problem of test_gpu_observation_model under ERROR_VALID: landmarks with exactly one valid observation, whose
    Jl_s^T Jl_s has rank 2 and unit diagonal"""
    import rootba_b200 as rb
    from test_gpu_observation_model import SPECIAL, _setup
    arrays, _, _, _ = _setup("valid", np.float32)
    assert any(v == 1 for _, v in SPECIAL)
    so = rb.SolverOptions(solver_type="SCHUR_COMPLEMENT")
    so.optimized_cost = "ERROR_VALID"
    return arrays, so


def test_schur_complement_with_a_singular_landmark_block():
    """float32 SC at a lam where Jl_s^T Jl_s + lam I of a one-observation landmark is singular in working precision: rba_solve
    returns, rba_apply reports the step as not finite (never an accepted finite step), rba_restore gives back the state bit
    for bit, and rba_lm_run starting at that lam raises it and reaches the float64 square-root solver's minimum"""
    import rootba_b200 as rb
    arrays, so = _singular_setup()
    bp = rb.BalProblem.from_arrays(arrays, np.float32)
    lin = rb.LinearizorQR.create(bp, so)
    lin.linearize()
    inc = lin.solve(LAM_SINGULAR)
    term, it = lin.last_cg.termination_type, lin.last_cg.num_iterations
    assert not np.isfinite(lin.get_rhs()).all() and not np.isfinite(inc).all()
    assert (term, it) == (NO_CONVERGENCE, so.max_linear_solver_iterations), (term, it)
    lin.download_state()
    cams0, lms0 = bp.cams.copy(), bp.lms.copy()
    bp.backup()
    l_diff = lin.apply(inc)
    assert not np.isfinite(l_diff), (l_diff, term, it, np.isfinite(inc).all())
    bp.restore()
    lin.download_state()
    assert np.array_equal(bp.cams, cams0) and np.array_equal(bp.lms, lms0)
    lin.close()
    # the native LM loop from that lam on, against the float64 square-root solver's minimum (same loop, default lam)
    so.max_num_iterations = 30
    so.initial_trust_region_radius = 1 / LAM_SINGULAR
    lin = rb.LinearizorQR.create(rb.BalProblem.from_arrays(arrays, np.float32), so)
    its, _, _ = lin.lm_run(64)
    lin.close()
    ref = rb.SolverOptions(max_num_iterations=30)
    ref.optimized_cost = "ERROR_VALID"
    lin = rb.LinearizorQR.create(rb.BalProblem.from_arrays(arrays, np.float64), ref)
    its_q, _, _ = lin.lm_run(64)
    lin.close()
    assert not its[0]["accepted"] and its[1]["lambda"] > its[0]["lambda"], its[:2]
    best = min(i["cost"] for i in its if i["accepted"])
    best_q = min(i["cost"] for i in its_q if i["accepted"])
    assert abs(best - best_q) <= 1e-4 * best_q, (best, best_q)
