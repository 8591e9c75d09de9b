"""Oracle-independent GPU parity check: the CUDA path (through the C ABI) against dense float64 numpy algebra built from
the Jacobians of the independent camera model (tests/camera_model.py) only.  tests/test_oracle_dense_numpy.py states the algebra and holds the oracle to the same bar."""
import numpy as np
import pytest

from conftest import rel_err

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("use_householder", [True, False])
def test_f64_against_dense_normal_equations(use_householder):
    """Oracle-independent check of the CUDA path: b, H x, the converged PCG solution, the model cost change and the landmark
    update against dense float64 numpy algebra built from the Jacobians of the independent camera model only
    (tests/test_oracle_dense_numpy.py states the algebra and holds the oracle to the same bar)."""
    _check_against_dense_normal_equations(use_householder, "benign")


@pytest.mark.parametrize("use_householder", [True, False])
def test_f64_against_dense_normal_equations_with_distortion(use_householder):
    """the same check on a problem with real lens distortion (|k1| ~ 0.1, |x/z| <= 1.4)"""
    _check_against_dense_normal_equations(use_householder, "distorted")


def _check_against_dense_normal_equations(use_householder, kind):
    import rootba_b200 as rb
    from test_oracle_dense_numpy import _dense_system, _problem, _reduced
    prob = _problem(kind)
    Jp, Jl, r = _dense_system(prob)
    lam = 1e-3
    D, sl, Jps, Jls, Minv, H, b = _reduced(Jp, Jl, r, lam, prob.nl, float(np.sqrt(1e-10)))
    so = rb.SolverOptions()
    so.eta = 1e-13  # run PCG (nearly) to the solution of the linear system: the oracle needs ~48 iterations here and is then
    #                 within 1e-8 of the direct solve; well above the 1e-16 round-off noise of the zeta stopping test
    so.use_householder_marginalization = use_householder
    bp = rb.BalProblem.from_arrays(prob, np.float64)
    lin = rb.LinearizorQR.create(bp, so)
    assert abs(lin.compute_error()["all"]["error"] - 0.5 * r @ r) <= 1e-12 * (0.5 * r @ r)
    lin.linearize()
    s_g, _ = lin.get_jacobian_scaling()
    assert rel_err(s_g, D) < 1e-12
    inc = lin.solve(lam)
    assert rel_err(lin.get_rhs(), b) < 1e-9
    x = np.random.default_rng(1).uniform(-1, 1, H.shape[0])
    assert rel_err(lin.right_multiply(x), H @ x) < 1e-9
    assert lin.last_cg.termination_type == 1 and lin.last_cg.num_iterations < 200
    assert rel_err(inc, -np.linalg.solve(H, b)) < 1e-6
    dl_s = -Minv @ (Jls.T @ r + Jls.T @ (Jps @ inc))
    want_l = 0.5 * r @ r - 0.5 * np.sum((r + Jps @ inc + Jls @ dl_s) ** 2)
    l_diff = lin.apply(inc)
    assert abs(l_diff - want_l) <= 1e-8 * abs(want_l)
    lin.download_state()
    assert rel_err(bp.lms, prob.lms + (sl * dl_s).reshape(-1, 3)) < 1e-10
    lin.close()
