"""Gaussian camera priors (rba_set_camera_prior) on the GPU: every solver against the dense float64 algebra of the total
(reprojection + prior) problem, truncated PCG iterates, priors with held parameters, no behaviour change without priors,
an observation-free camera, an end-to-end minimum against scipy, bad input and the sharded path."""
import ctypes as C

import numpy as np
import pytest

import camera_prior_model as pm
from conftest import rel_err
from objective_checks import CONFIGS, MASK, cfg_id, check_against_dense, check_two_rank_step, fixed_params

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def case7():
    return pm.prior_case(7, 90)


@pytest.fixture(scope="module")
def case120():
    return pm.prior_case(120, 500, seed=5)


@pytest.mark.parametrize("cfg", CONFIGS, ids=cfg_id)
def test_f64_against_dense_system_with_priors(cfg, case7):
    prob, mean, L = case7
    check_against_dense(cfg, prob, camera=(mean, L))


@pytest.mark.parametrize("env", [{"RBA_PCG_CLUSTER": "1"}, {"RBA_PCG_PARTIALS": "0"}], ids=["one-cta", "no-partials"])
@pytest.mark.parametrize("cfg", CONFIGS, ids=cfg_id)
def test_f64_120_cameras_against_dense_system_with_priors(cfg, env, case120):
    """RBA_PCG_CLUSTER=1: 120 cameras leave the register-resident layout of the vector step (its uncached path)"""
    prob, mean, L = case120
    check_against_dense(cfg, prob, camera=(mean, L), env=env)


@pytest.mark.parametrize("cfg", [CONFIGS[0], CONFIGS[2], CONFIGS[5], CONFIGS[8], CONFIGS[9]], ids=cfg_id)
def test_f32_against_dense_system_with_priors(cfg, case7):
    prob, mean, L = case7
    check_against_dense(cfg, prob, camera=(mean, L), dtype=np.float32)


@pytest.mark.parametrize("cfg", CONFIGS, ids=cfg_id)
def test_f64_priors_with_held_parameters_against_restricted_dense_system(cfg, case7):
    prob, mean, L = case7
    check_against_dense(cfg, prob, camera=(mean, L), mask=np.resize(MASK, prob.nc))


# ---- truncated PCG iterates -------------------------------------------------------------------------------------------
def _seq_case():
    from rootba_b200.synthetic import synth_config
    arrays = synth_config("ladybug-1723", scale=0.05)
    rng = np.random.default_rng(11)
    mean = pm.mean_at(arrays.cams)
    mean[:, 4:7] += rng.normal(0, 0.1, (arrays.nc, 3))
    kinds = ["centre", "dense", "intrinsics", "none"]
    L = np.stack([pm.sqrt_info_kind(kinds[c % 4], rng, 0.5) for c in range(arrays.nc)])
    return arrays, mean, L


@pytest.fixture(scope="module")
def seq_prior():
    return _seq_case()


@pytest.mark.parametrize("operator_form", ["DENSE", "IMPLICIT"])
@pytest.mark.parametrize("precond", ["JACOBI", "SCHUR_JACOBI"])
def test_pcg_truncated_iterates_with_priors(seq_prior, operator_form, precond):
    from objective_checks import check_truncated_pcg_iterates
    arrays, mean, L = seq_prior
    check_truncated_pcg_iterates(arrays, operator_form, precond, camera_prior=(mean, L))


# ---- held parameters through whole LM runs, no behaviour change without priors ------------------------------------------
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_held_parameters_stay_fixed_with_priors_through_lm_run(small_problem, dtype):
    import rootba_b200 as rb
    so = rb.SolverOptions(max_num_iterations=8)
    flags = np.full(small_problem.nc, rb.FIX_INTRINSICS, np.uint8)
    flags[[0, 1]] = rb.FIX_ALL
    prior = pm.small_prior(small_problem)
    bp = rb.BalProblem.from_arrays(small_problem, dtype)
    bp.camera_fixed = flags
    bp.camera_prior = prior
    cams0 = bp.cams.copy()
    lin = rb.LinearizorQR.create(bp, so)
    its, _, _ = lin.lm_run(64)
    lin.download_state()
    lin.close()
    fp = fixed_params(flags)
    assert np.array_equal(bp.cams[fp], cams0[fp])
    assert not np.array_equal(bp.cams[~fp], cams0[~fp])
    acc = [it["cost"] for it in its if it["accepted"]]
    assert len(acc) >= 1 and all(b < a for a, b in zip(acc, acc[1:])), its


@pytest.mark.parametrize("solver_type", ["SQUARE_ROOT", "SCHUR_COMPLEMENT"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_no_behaviour_change_without_priors(small_problem, dtype, solver_type):
    import rootba_b200 as rb
    from objective_checks import assert_identical_steps, lm_steps
    run = lambda mode: lm_steps(small_problem, dtype, dict(solver_type=solver_type), mode, rb.LinearizorQR.set_camera_prior,
                                pm.small_prior(small_problem))
    c0, ref = run("never")
    assert_identical_steps((c0, ref), run("set_then_none"), "set_then_none")
    if dtype == np.float64:
        c2, zeros = run("zeros")
        assert abs(c2 - c0) <= 1e-12 * c0
        for a, b in zip(ref, zeros):
            assert rel_err(b[0], a[0]) < 1e-12 and abs(b[1] - a[1]) <= 1e-12 * abs(a[1])
            assert rel_err(b[2], a[2]) < 1e-12 and rel_err(b[3], a[3]) < 1e-12


# ---- an observation-free camera ---------------------------------------------------------------------------------------
def test_unobserved_camera_with_intrinsics_prior_reaches_the_mean_in_one_step():
    """its prior residual is linear in f, k1, k2: one undamped step puts them at the prior mean.  The other cameras are held
    (rba_set_camera_fixed), so the reduced system is this camera's block alone, which the block preconditioner inverts
    exactly: the solve is exact rather than accurate to the PCG stopping rule of the whole problem."""
    import rootba_b200 as rb
    prob, _, _ = pm.prior_case(7, 90, unobserved=True)
    mean = pm.mean_at(prob.cams)
    mean[-1, 7:10] = prob.cams[-1, 7:10] + [12.5, 0.03, -0.004]
    L = np.zeros((prob.nc, 9, 9))
    L[-1, 6:9, 6:9] = np.diag([0.05, 2.0, 4.0])
    bp = rb.BalProblem.from_arrays(prob, np.float64)
    bp.camera_prior = (mean, L)
    flags = np.full(prob.nc, rb.FIX_ALL, np.uint8)
    flags[-1] = 0
    bp.camera_fixed = flags
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(eta=1e-13))
    lin.compute_error()
    lin.linearize()
    lin.solve(1e-12)
    lin.apply(None)
    lin.download_state()
    lin.close()
    assert np.allclose(bp.cams[-1, 7:10], mean[-1, 7:10], rtol=1e-9, atol=1e-12), bp.cams[-1, 7:10] - mean[-1, 7:10]
    assert np.array_equal(bp.cams[-1, :7], prob.cams[-1, :7])  # no information on its pose: zero pose increment


# ---- end to end against scipy -----------------------------------------------------------------------------------------
def _e2e_problem():
    from rootba_b200.synthetic import BalArrays, synth_bal
    prob = synth_bal(8, 150, 4.0, seed=31)
    rng = np.random.default_rng(32)
    truth = np.asarray(prob.cams, np.float64)
    mean = pm.mean_at(truth)
    mean[:, 4:7] += rng.normal(0, 0.02, (prob.nc, 3))
    L = np.zeros((prob.nc, 9, 9))
    L[:, 0:3, 0:3] = 20.0 * np.eye(3)   # centres to ~0.05
    L[:, 6, 6] = 0.02                  # f to ~50 pixels
    L[:, 7:9, 7:9] = 10.0 * np.eye(2)  # k1, k2 to ~0.1
    cams = truth.copy()
    from scipy.spatial.transform import Rotation
    for c in range(prob.nc):
        cams[c, :4] = (Rotation.from_rotvec(rng.normal(0, 0.01, 3)) * Rotation.from_quat(cams[c, :4])).as_quat()
        cams[c, 4:7] += rng.normal(0, 0.02, 3)
        cams[c, 7] *= 1 + rng.normal(0, 0.01)
    lms = np.asarray(prob.lms) + rng.normal(0, 0.02, np.shape(prob.lms))
    return BalArrays(cams, lms, prob.lm_off, prob.obs_cam, prob.obs_xy), mean, L


def test_lm_run_reaches_the_scipy_minimum_of_the_total_objective():
    import rootba_b200 as rb
    from objective_checks import scipy_minimum
    prob, mean, L = _e2e_problem()
    cams_s, lms_s, cost_s = scipy_minimum(prob, camera=(mean, L))
    so = rb.SolverOptions(max_num_iterations=60, function_tolerance=1e-15, eta=1e-10)
    runs = {}
    for dtype in (np.float64, np.float32):
        bp = rb.BalProblem.from_arrays(prob, dtype)
        bp.camera_prior = (mean, L)
        lin = rb.LinearizorQR.create(bp, so)
        its, _, _ = lin.lm_run(200)
        lin.download_state()
        cost = lin.compute_error()["all"]["error"]
        lin.close()
        runs[dtype] = (bp, its, cost)
    bp, its, cost = runs[np.float64]
    assert abs(cost - cost_s) <= 1e-9 * cost_s, (cost, cost_s)
    centres = np.stack([pm.centre(c) for c in bp.cams])
    assert rel_err(centres, np.stack([pm.centre(c) for c in cams_s])) < 1e-6
    assert rel_err(bp.cams[:, 7:10], cams_s[:, 7:10]) < 1e-6
    assert rel_err(bp.lms, lms_s) < 1e-6
    # float32 reaches the float64 minimum
    assert abs(runs[np.float32][2] - cost) <= 1e-4 * cost


def test_lm_run_with_priors_equals_the_python_host_loop():
    """rba_lm_run and bundle_adjust_manual on the same total objective: bit-identical trajectory (default LM options, under
    which test_native_lm_loop_equals_the_python_loop compares the two loops)"""
    import rootba_b200 as rb
    from objective_checks import check_lm_run_equals_host_loop
    prob, mean, L = _e2e_problem()
    check_lm_run_equals_host_loop(prob, rb.SolverOptions(max_num_iterations=10), camera_prior=(mean, L))


# ---- bad input --------------------------------------------------------------------------------------------------------
def test_bad_input_keeps_the_previous_priors(small_problem):
    import rootba_b200 as rb
    from rootba_b200 import _lib
    lib = _lib.lib()
    mean, L = pm.small_prior(small_problem)
    bp = rb.BalProblem.from_arrays(small_problem, np.float64)
    bp.camera_prior = (mean, L)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions())
    lin.compute_error()
    lin.linearize()
    inc_ref = lin.solve(1e-4)
    p = lambda a: C.c_void_p(a.ctypes.data)
    bad_nan = L.copy()
    bad_nan[3, 2, 2] = np.nan
    bad_q = mean.copy()
    bad_q[4, :4] *= 1.01
    for args in ((p(mean), p(bad_nan)), (p(mean), None), (None, p(L)), (p(bad_q), p(L))):
        assert lib.rba_set_camera_prior(lin.h, *args) == -1  # RBA_ERR_INVALID_ARGUMENT
        assert lib.rba_last_error()
    assert b"camera 4" in (lib.rba_set_camera_prior(lin.h, p(bad_q), p(L)), lib.rba_last_error())[1]
    # nothing changed: the same solve as before, and the handle is still linearised
    assert np.array_equal(lin.solve(1e-4), inc_ref)
    with pytest.raises(ValueError):
        lin.set_camera_prior((bad_q, L))
    assert bp.camera_prior[0] is not bad_q and np.array_equal(bp.camera_prior[0], mean)
    # a prior change needs a new linearisation
    lin.set_camera_prior((mean, L))
    with pytest.raises(rb.RbaError) as e:
        lin.solve(1e-4)
    assert e.value.code == -6  # RBA_ERR_STATE
    lin.linearize()
    assert np.array_equal(lin.solve(1e-4), inc_ref)
    lin.close()


# ---- two GPUs ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("peer", ["1", "0"])
@pytest.mark.parametrize("sfx", ["f32", "f64"])
def test_two_ranks_with_priors(tmp_path, peer, sfx):
    """every prior term is added once, after the sum over the shards: the sharded step equals the single-rank step"""
    check_two_rank_step(tmp_path, "camera", sfx, peer, 29500, (7 if peer == "1" else 0) + (13 if sfx == "f32" else 0))
