"""Relative pose priors between pairs of cameras (rba_set_camera_pair_prior) on the GPU: every solver against the dense
float64 algebra of the total (reprojection + pair prior) problem, with absolute priors and with held parameters, truncated
PCG iterates, no behaviour change without pair priors, an observation-free camera, an end-to-end minimum against scipy, bad
input and the sharded path."""
import ctypes as C

import numpy as np
import pytest

import camera_prior_model as pm
import pair_prior_model as qm
from objective_checks import CONFIGS, MASK, cfg_id, check_against_dense, check_two_rank_step

pytestmark = pytest.mark.gpu


def _check(cfg, prob, pair, **kw):
    """check_against_dense with pair priors: in float64 the PCG increment bar widens to sqrt(eta kappa)"""
    check_against_dense(cfg, prob, pairs=pair, inc_eta_kappa=True, **kw)


@pytest.fixture(scope="module")
def case7():
    return qm.pair_case(7, 90)


@pytest.fixture(scope="module")
def case120():
    return qm.pair_case(120, 500, seed=5)


@pytest.mark.parametrize("cfg", CONFIGS, ids=cfg_id)
def test_f64_against_dense_system_with_pair_priors(cfg, case7):
    _check(cfg, *case7)


@pytest.mark.parametrize("env", [{"RBA_PCG_CLUSTER": "1"}, {"RBA_PCG_PARTIALS": "0"}], ids=["one-cta", "no-partials"])
@pytest.mark.parametrize("cfg", CONFIGS, ids=cfg_id)
def test_f64_120_cameras_against_dense_system_with_pair_priors(cfg, env, case120):
    """RBA_PCG_CLUSTER=1: 120 cameras leave the register-resident layout of the vector step (its uncached path)"""
    _check(cfg, *case120, env=env)


@pytest.mark.parametrize("cfg", [CONFIGS[0], CONFIGS[2], CONFIGS[5], CONFIGS[8], CONFIGS[9]], ids=cfg_id)
def test_f32_against_dense_system_with_pair_priors(cfg, case7):
    _check(cfg, *case7, dtype=np.float32)


@pytest.mark.parametrize("cfg", CONFIGS, ids=cfg_id)
def test_f64_pair_and_absolute_priors_against_dense_system(cfg, case7):
    prob, pair = case7
    _, mean_a, L_a = pm.prior_case(7, 90)
    _check(cfg, prob, pair, camera=(mean_a, L_a))


@pytest.mark.parametrize("cfg", CONFIGS, ids=cfg_id)
def test_f64_pair_priors_with_held_parameters_against_restricted_dense_system(cfg, case7):
    """MASK holds every parameter of camera 3, which pairs (2, 3) and (3, 4) join to free cameras"""
    prob = case7[0]
    _check(cfg, *case7, mask=np.resize(MASK, prob.nc))


# ---- truncated PCG iterates -------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def seq_pairs():
    from rootba_b200.synthetic import synth_config
    arrays = synth_config("ladybug-1723", scale=0.05)
    rng = np.random.default_rng(12)
    pairs = np.array([(c, c + 1) for c in range(arrays.nc - 1)] + [(c + 5, c) for c in range(0, arrays.nc - 5, 3)], np.int32)
    mean = qm.mean_at(arrays.cams, pairs)
    mean[:, 4:7] += rng.normal(0, 0.1, (len(pairs), 3))
    kinds = ["dense", "translation", "rotation", "none"]
    L = np.stack([qm.sqrt_info_kind(kinds[p % 4], rng, 0.5) for p in range(len(pairs))])
    return arrays, (pairs, mean, L)


@pytest.mark.parametrize("operator_form", ["DENSE", "IMPLICIT"])
@pytest.mark.parametrize("precond", ["JACOBI", "SCHUR_JACOBI"])
def test_pcg_truncated_iterates_with_pair_priors(seq_pairs, operator_form, precond):
    """the replay's operator includes the off-diagonal pair blocks"""
    from objective_checks import check_truncated_pcg_iterates
    arrays, pair = seq_pairs
    check_truncated_pcg_iterates(arrays, operator_form, precond, camera_pair_prior=pair)


# ---- no behaviour change without pair priors ----------------------------------------------------------------------------
def _chain_pairs(problem, seed=4):
    rng = np.random.default_rng(seed)
    pairs = np.array([(c, c + 1) for c in range(problem.nc - 1)], np.int32)
    mean = qm.mean_at(problem.cams, pairs)
    mean[:, 4:7] += rng.normal(0, 0.05, (len(pairs), 3))
    L = np.stack([qm.sqrt_info_kind(["dense", "translation", "rotation"][p % 3], rng) for p in range(len(pairs))])
    return pairs, mean, L


@pytest.mark.parametrize("absolute", [False, True], ids=["no-priors", "absolute-priors"])
@pytest.mark.parametrize("solver_type", ["SQUARE_ROOT", "SCHUR_COMPLEMENT", "POWER_SCHUR_COMPLEMENT"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_no_behaviour_change_without_pair_priors(small_problem, dtype, solver_type, absolute):
    """pair priors set and cleared, or all with a zero L: the LM trajectory of a handle that never had any, bit for bit
    (with and without absolute priors)"""
    import rootba_b200 as rb
    from objective_checks import assert_identical_steps, lm_steps
    run = lambda mode: lm_steps(small_problem, dtype, dict(solver_type=solver_type), mode, rb.LinearizorQR.set_camera_pair_prior,
                                _chain_pairs(small_problem), camera_prior=pm.small_prior(small_problem) if absolute else None)
    ref = run("never")
    for mode in ("set_then_none", "zeros"):
        assert_identical_steps(ref, run(mode), mode)


# ---- an observation-free camera ---------------------------------------------------------------------------------------
def test_unobserved_camera_tied_by_a_strong_pair_prior_reaches_the_relative_pose_in_one_step():
    """the last camera has no observations; a strong dense pair prior ties it to camera 0 at a relative pose away from the
    current one.  The other cameras are held, so the reduced system is this camera's pose block, and one nearly undamped
    step puts T_last T_0^-1 at the prior mean (the residual is nearly linear in the pose of the last camera for a small move)"""
    import rootba_b200 as rb
    from scipy.spatial.transform import Rotation
    prob, _ = qm.pair_case(7, 90)
    n = prob.nc
    mean = qm.mean_at(prob.cams, [(n - 1, 0)])
    mean[0, 4:7] += [0.02, -0.01, 0.015]
    mean[0, :4] = (Rotation.from_rotvec([0.003, -0.002, 0.001]) * Rotation.from_quat(mean[0, :4])).as_quat()
    pair = (np.array([(n - 1, 0)], np.int32), mean, 1e3 * np.eye(6)[None])
    bp = rb.BalProblem.from_arrays(prob, np.float64)
    bp.camera_pair_prior = pair
    flags = np.full(n, rb.FIX_ALL, np.uint8)
    flags[-1] = rb.FIX_INTRINSICS
    bp.camera_fixed = flags
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(eta=1e-13))
    e0 = lin.compute_error()["all"]["error"]
    lin.linearize()
    lin.solve(1e-12)
    lin.apply(None)
    lin.download_state()
    lin.close()
    e = qm.residual(bp.cams[-1], bp.cams[0], mean[0])
    e_before = qm.residual(prob.cams[-1], prob.cams[0], mean[0])
    assert np.linalg.norm(e) < 1e-3 * np.linalg.norm(e_before), (e, e_before)
    assert np.array_equal(bp.cams[:-1], prob.cams[:-1])


# ---- end to end against scipy -----------------------------------------------------------------------------------------
def _e2e_problem():
    """a perturbed synthetic problem with pair priors between consecutive cameras and a loop closure (sigma 1 on translation,
    0.01 rad on rotation)"""
    from rootba_b200.synthetic import BalArrays, synth_bal
    from scipy.spatial.transform import Rotation
    prob = synth_bal(8, 150, 4.0, seed=31)
    rng = np.random.default_rng(33)
    truth = np.asarray(prob.cams, np.float64)
    pairs = np.array([(c, c + 1) for c in range(prob.nc - 1)] + [(prob.nc - 1, 0)], np.int32)
    mean = qm.mean_at(truth, pairs)
    mean[:, 4:7] += rng.normal(0, 0.01, (len(pairs), 3))
    L = np.tile(np.diag([1.0, 1.0, 1.0, 100.0, 100.0, 100.0]), (len(pairs), 1, 1))  # sigma 1 and 0.01 rad
    cams = truth.copy()
    for c in range(prob.nc):
        cams[c, :4] = (Rotation.from_rotvec(rng.normal(0, 0.01, 3)) * Rotation.from_quat(cams[c, :4])).as_quat()
        cams[c, 4:7] += rng.normal(0, 0.02, 3)
        cams[c, 7] *= 1 + rng.normal(0, 0.01)
    lms = np.asarray(prob.lms) + rng.normal(0, 0.02, np.shape(prob.lms))
    return BalArrays(cams, lms, prob.lm_off, prob.obs_cam, prob.obs_xy), (pairs, mean, L)


def test_lm_run_reaches_the_scipy_minimum_of_the_total_objective():
    """the cost at the minimum is gauge-free; the relative poses of the pairs are compared (the pair priors and reprojections
    leave the similarity gauge free, so absolute poses may differ between the two solvers)"""
    import rootba_b200 as rb
    from objective_checks import scipy_minimum
    prob, pair = _e2e_problem()
    cams_s, _, cost_s = scipy_minimum(prob, pairs=pair)
    so = rb.SolverOptions(max_num_iterations=60, function_tolerance=1e-15, eta=1e-10)
    runs = {}
    for dtype in (np.float64, np.float32):
        bp = rb.BalProblem.from_arrays(prob, dtype)
        bp.camera_pair_prior = pair
        lin = rb.LinearizorQR.create(bp, so)
        lin.lm_run(200)
        lin.download_state()
        cost = lin.compute_error()["all"]["error"]
        lin.close()
        runs[dtype] = (bp, cost)
    bp, cost = runs[np.float64]
    assert abs(cost - cost_s) <= 1e-8 * cost_s, (cost, cost_s)
    pairs, mean, L = pair
    e_gpu = np.stack([qm.residual(bp.cams[i], bp.cams[j], mean[p]) for p, (i, j) in enumerate(pairs)])
    e_ref = np.stack([qm.residual(cams_s[i], cams_s[j], mean[p]) for p, (i, j) in enumerate(pairs)])
    assert np.max(np.abs(e_gpu - e_ref)) < 1e-4 * max(1.0, np.max(np.abs(e_ref)))
    assert abs(runs[np.float32][1] - cost) <= 1e-4 * cost


def test_lm_run_with_pair_priors_equals_the_python_host_loop():
    import rootba_b200 as rb
    from objective_checks import check_lm_run_equals_host_loop
    prob, pair = _e2e_problem()
    check_lm_run_equals_host_loop(prob, rb.SolverOptions(max_num_iterations=10), camera_pair_prior=pair)


# ---- bad input --------------------------------------------------------------------------------------------------------
def test_bad_input_keeps_the_previous_pair_priors(small_problem):
    import rootba_b200 as rb
    from rootba_b200 import _lib
    lib = _lib.lib()
    pairs, mean, L = _chain_pairs(small_problem)
    bp = rb.BalProblem.from_arrays(small_problem, np.float64)
    bp.camera_pair_prior = (pairs, mean, L)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions())
    lin.compute_error()
    lin.linearize()
    inc_ref = lin.solve(1e-4)
    p = lambda a: C.c_void_p(a.ctypes.data)
    m = C.c_int32(len(pairs))
    bad_nan_L, bad_nan_m = L.copy(), mean.copy()
    bad_nan_L[3, 2, 2] = np.nan
    bad_nan_m[2, 5] = np.inf
    bad_q = mean.copy()
    bad_q[4, :4] *= 1.01
    out_of_range, self_pair, negative = pairs.copy(), pairs.copy(), pairs.copy()
    out_of_range[5, 1] = small_problem.nc
    self_pair[6, 1] = self_pair[6, 0]
    negative[7, 0] = -1
    cases = [(C.c_int32(-1), p(pairs), p(mean), p(L)), (m, None, p(mean), p(L)), (m, p(pairs), None, p(L)), (m, p(pairs), p(mean), None),
             (m, p(out_of_range), p(mean), p(L)), (m, p(self_pair), p(mean), p(L)), (m, p(negative), p(mean), p(L)),
             (m, p(pairs), p(mean), p(bad_nan_L)), (m, p(pairs), p(bad_nan_m), p(L)), (m, p(pairs), p(bad_q), p(L))]
    for args in cases:
        assert lib.rba_set_camera_pair_prior(lin.h, *args) == -1  # RBA_ERR_INVALID_ARGUMENT
        assert lib.rba_last_error()
    assert b"pair 4" in (lib.rba_set_camera_pair_prior(lin.h, m, p(pairs), p(bad_q), p(L)), lib.rba_last_error())[1]
    # nothing changed: the same solve as before, and the handle is still linearised
    assert np.array_equal(lin.solve(1e-4), inc_ref)
    for bad in ((pairs, bad_q, L), (out_of_range, mean, L), (self_pair, mean, L), (pairs, mean, bad_nan_L), (pairs[:, :1], mean, L)):
        with pytest.raises(ValueError):
            lin.set_camera_pair_prior(bad)
    assert np.array_equal(bp.camera_pair_prior[1], mean)
    # a change needs a new linearisation
    lin.set_camera_pair_prior((pairs, mean, L))
    with pytest.raises(rb.RbaError) as e:
        lin.solve(1e-4)
    assert e.value.code == -6  # RBA_ERR_STATE
    lin.linearize()
    assert np.array_equal(lin.solve(1e-4), inc_ref)
    lin.close()


# ---- two GPUs ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("peer", ["1", "0"])
@pytest.mark.parametrize("sfx", ["f32", "f64"])
def test_two_ranks_with_pair_priors(tmp_path, peer, sfx):
    """every pair term is added once, after the sum over the shards: the sharded step equals the single-rank step"""
    check_two_rank_step(tmp_path, "pair", sfx, peer, 29500, (11 if peer == "1" else 0) + (17 if sfx == "f32" else 0))
