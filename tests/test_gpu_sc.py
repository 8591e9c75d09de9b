"""GPU parity of the Schur-complement solvers on the same device data model (SURVEY 8f row 3):
  solver_type = SCHUR_COMPLEMENT        <-> LinearizorSC       (solver/linearizor_sc.cpp, sc/landmark_block.hpp, sc/linearization_sc.hpp)
  solver_type = POWER_SCHUR_COMPLEMENT  <-> LinearizorPowerSC  (solver/linearizor_power_sc.cpp, sc/linearization_power_sc.hpp:92-160)
against the oracle's restatement of those files, plus the reference's own cross-check QR == SC
(qr/linearization_qr.test.cpp:120-222), here between the two CUDA solvers.

Tolerances: f64 1e-9 (the device factorises Hll = R^T R and substitutes, the reference / oracle inverts the 3x3 explicitly:
different round-off, both of size eps * cond(Hll)); f32 1e-3 -- the Schur complement squares the condition number of the
landmark block, which is the reason the square-root solver exists (its own f32 bar is 1e-5)."""
import numpy as np
import pytest

from conftest import rel_err

pytestmark = pytest.mark.gpu

TOL = {np.float32: 1e-3, np.float64: 1e-9}


def _pair(arrays, dtype, solver_type, **kw):
    import rootba_b200 as rb
    from oracle import oracle_py as orc
    so = rb.SolverOptions(solver_type=solver_type, **kw)
    bp = rb.BalProblem.from_arrays(arrays, dtype)
    lin = rb.LinearizorQR.create(bp, so)
    okw = {k: v for k, v in kw.items() if k in ("eta", "max_linear_solver_iterations")}
    o = orc.Oracle(arrays, dtype, orc.default_options(num_threads=0, **okw))
    return bp, lin, o


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_schur_complement_solver_against_oracle(small_problem, dtype):
    bp, lin, o = _pair(small_problem, dtype, "SCHUR_COMPLEMENT")
    tol = TOL[dtype]
    lin.linearize(); o.scl_linearize()
    assert rel_err(lin.get_jacobian_scaling()[0], o.scl_get_scaling()) < (1e-5 if dtype == np.float32 else 1e-12)
    lam = 1e-2
    inc_g = lin.solve(lam)
    inc_c, dbg = o.scl_solve(lam)
    assert rel_err(lin.get_rhs(), dbg["b"]) < tol
    inv_g, _ = lin.get_preconditioner()
    assert max(rel_err(inv_g[c], dbg["inv_blocks"][c]) for c in range(lin.nc)) < 10 * tol
    # H x against the SC landmark blocks of the oracle (sc/landmark_block.hpp:238-279)
    x = np.random.default_rng(4).uniform(-1, 1, 9 * lin.nc).astype(dtype)
    o.sc_linearize(); o.sc_scale_Jp(o.scl_get_scaling())
    _, _, y_c = o.sc_get_Hb(lam, lam, x)
    assert rel_err(lin.right_multiply(x), y_c) < tol
    assert abs(lin.last_cg.num_iterations - dbg["cg_iterations"]) <= 2 and lin.last_cg.termination_type == dbg["cg_termination"]
    assert rel_err(inc_g, inc_c) < 10 * tol
    l_g, l_c = lin.apply(inc_g), o.scl_apply(inc_c)
    assert abs(l_g - l_c) <= 100 * tol * abs(l_c)
    lin.download_state()
    cams_c, lms_c = o.get_state()
    assert rel_err(bp.lms, lms_c) < 100 * tol and rel_err(bp.cams, cams_c) < 10 * tol
    import rootba_b200 as rb
    with pytest.raises(rb.RbaError):  # no Q2 panels exist for the Schur-complement solvers
        lin.debug_get_block(0)
    lin.close()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_power_schur_complement_solver_against_oracle(small_problem, dtype):
    bp, lin, o = _pair(small_problem, dtype, "POWER_SCHUR_COMPLEMENT", power_order=20)
    tol = TOL[dtype]
    lin.linearize(); o.scl_linearize()
    for lam, order, eta in ((1e-2, 20, 0.1), (1e-1, 40, 1e-3)):
        lin.options.power_order = order
        import rootba_b200 as rb
        bp2 = rb.BalProblem.from_arrays(small_problem, dtype)
        lin2 = rb.LinearizorQR.create(bp2, rb.SolverOptions(solver_type="POWER_SCHUR_COMPLEMENT", power_order=order, eta=eta))
        lin2.linearize()
        inc_g = lin2.solve(lam)
        inc_c, dbg = o.scl_power_solve(lam, order, eta)
        assert rel_err(lin2.get_rhs(), dbg["b"]) < tol
        assert abs(lin2.last_cg.num_iterations - dbg["power_order"]) <= 1, (lin2.last_cg.num_iterations, dbg)
        assert lin2.last_cg.termination_type == dbg["termination"]
        if lin2.last_cg.num_iterations == dbg["power_order"]:
            assert rel_err(inc_g, inc_c) < 10 * tol
        else:  # a zeta within rounding of eta: the float64 replay of the series on the handle's own inputs
            from pcg_replay import power_replay
            from test_gpu_pcg_iterates import operator_of
            rep = power_replay(operator_of(lin2, dtype), lin2.get_preconditioner()[0], lin2.get_rhs(), order=order, eta=eta)
            assert (rep["iterations"], rep["termination"]) == (lin2.last_cg.num_iterations, lin2.last_cg.termination_type)
            assert rel_err(inc_g, rep["sums"][-1]) < 10 * tol
        l_g, l_c = lin2.apply(inc_g), None
        assert np.isfinite(l_g) and l_g > 0
        lin2.close()
    lin.close()


def test_qr_equals_schur_complement_on_device(small_problem):
    """the reference's own cross-check (qr/linearization_qr.test.cpp:120-222: b, diagonal blocks, H x, l_diff, landmark update of
    the QR formulation against the SC formulation), here between the two CUDA solvers in float64"""
    import rootba_b200 as rb
    res = {}
    rng = np.random.default_rng(8)
    x = rng.uniform(-1, 1, 9 * small_problem.nc)
    dp = 0.01 * rng.uniform(-1, 1, 9 * small_problem.nc)
    for st in ("SQUARE_ROOT", "SCHUR_COMPLEMENT"):
        bp = rb.BalProblem.from_arrays(small_problem, np.float64)
        lin = rb.LinearizorQR.create(bp, rb.SolverOptions(solver_type=st, eta=1e-12, max_linear_solver_iterations=300))
        lin.linearize()
        inc = lin.solve(0.1)
        inv, blk = lin.get_preconditioner()
        r = {"b": lin.get_rhs(), "blocks": blk.copy(), "Hx": lin.right_multiply(x), "inc": inc, "it": lin.last_cg.num_iterations}
        r["l_diff"] = lin.back_substitute(dp)
        lin.download_state()
        r["lms"] = bp.lms.copy()
        res[st] = r
        lin.close()
    a, b = res["SQUARE_ROOT"], res["SCHUR_COMPLEMENT"]
    for k in ("b", "blocks", "Hx", "lms"):
        assert rel_err(a[k], b[k]) < 1e-11, k
    assert rel_err(a["inc"], b["inc"]) < 1e-8 and abs(a["l_diff"] - b["l_diff"]) <= 1e-10 * abs(a["l_diff"])


@pytest.mark.parametrize("solver_type", ["SCHUR_COMPLEMENT", "POWER_SCHUR_COMPLEMENT"])
def test_lm_loop_with_the_schur_complement_solvers(small_problem, solver_type):
    """the unchanged LM loop drives the other Linearizors through the same interface and reaches the QR solver's minimum"""
    import rootba_b200 as rb
    costs = {}
    for st in ("SQUARE_ROOT", solver_type):
        bp = rb.BalProblem.from_arrays(small_problem, np.float64)
        summ = rb.bundle_adjust_manual(bp, rb.SolverOptions(solver_type=st, max_num_iterations=12, power_order=40))
        costs[st] = min(it["cost"]["all"]["error"] for it in summ["iterations"] if it.get("step_is_successful"))
    assert abs(costs[solver_type] - costs["SQUARE_ROOT"]) <= 1e-4 * costs["SQUARE_ROOT"], costs
