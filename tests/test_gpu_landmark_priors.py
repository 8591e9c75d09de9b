"""Gaussian priors on landmark positions (rba_set_landmark_prior) on the GPU: every solver configuration against the dense
float64 algebra of the total (reprojection + landmark prior) problem in both precisions, every track-length class landmark by
landmark with prior and prior-free landmarks in one tile, lambda = 0, rank-deficient L, landmarks with one and with no valid
observation, no behaviour change without priors, bad input, an end-to-end minimum against scipy with every other prior
kind and held cameras, covariances with the gauge fixed by landmark priors, and the sharded path."""
import ctypes as C

import numpy as np
import pytest

import camera_model as cm
import camera_prior_model as pm
import landmark_prior_model as lp
import pair_prior_model as qm
from conftest import rel_err
from objective_checks import CONFIGS, cfg_id, check_against_dense, check_two_rank_step, dense_system, fixed_entries, reduced

pytestmark = pytest.mark.gpu

# CONFIGS of objective_checks (SQUARE_ROOT dense / implicit x Householder / Givens x JACOBI / SCHUR_JACOBI, SC, Power-SC)
# and the dense operator with stage2_form = IDENTITY (k_stage2<S, false>)
CONFIGS_LMP = CONFIGS + [dict(solver_type="SQUARE_ROOT", operator_form="DENSE", use_householder_marginalization=hh,
                              preconditioner_type=pc, stage2_form="IDENTITY") for hh in (True, False) for pc in ("JACOBI", "SCHUR_JACOBI")]


def _check(cfg, prob, prior, **kw):
    """check_against_dense with landmark priors: in float64 the PCG increment bar widens to sqrt(eta kappa)"""
    check_against_dense(cfg, prob, landmarks=prior, inc_eta_kappa=True, **kw)


@pytest.fixture(scope="module")
def case7():
    from rootba_b200.synthetic import synth_bal
    prob = synth_bal(7, 90, 3.6, seed=21)
    return prob, lp.prior_case(prob.lms, every=3, seed=5)


@pytest.mark.parametrize("cfg", CONFIGS_LMP, ids=cfg_id)
def test_f64_against_dense_system_with_landmark_priors(cfg, case7):
    _check(cfg, *case7)


@pytest.mark.parametrize("cfg", CONFIGS_LMP, ids=cfg_id)
def test_f32_against_dense_system_with_landmark_priors(cfg, case7):
    _check(cfg, *case7, dtype=np.float32)


@pytest.mark.parametrize("cfg", CONFIGS_LMP, ids=cfg_id)
def test_f64_landmark_and_camera_priors_with_held_parameters(cfg):
    """with the camera priors of test_camera_prior_model.prior_case (an unobserved camera held by its prior) and a held
    camera"""
    prob, mean_c, L_c = pm.prior_case(7, 90)
    mask = np.zeros(prob.nc, np.uint8)
    mask[2] = 15
    mask[4] = 14
    _check(cfg, prob, lp.prior_case(prob.lms, every=2, seed=8), camera=(mean_c, L_c), mask=mask)


@pytest.mark.parametrize("cfg", [CONFIGS_LMP[i] for i in (0, 3, 5, 8, 9, 10)], ids=cfg_id)
def test_lambda_zero_and_rank_one_priors(cfg):
    """lambda = 0: the prior landmarks' damping rows are [C | 0 | c] of L~ alone (the lambda = 0 shortcut must not skip
    them); height-only (rank-1) priors in the mix; the gauge fixed by camera priors"""
    prob, mean_c, L_c = pm.prior_case(7, 90)
    prior = lp.prior_case(prob.lms, every=2, seed=9, kinds=("height", "dense", "height", "rank2"))
    _check(cfg, prob, prior, camera=(mean_c, L_c), lam=0.0)


# ---- every track-length class, landmark by landmark ---------------------------------------------------------------------
def _class_ns():
    from test_gpu_kernel_classes import CASES, _signature
    return [n for n in CASES if n == 2 or _signature(n) != _signature(n - 1)]


@pytest.mark.parametrize("cfg", [CONFIGS_LMP[i] for i in (0, 4, 12, 8)], ids=cfg_id)
@pytest.mark.parametrize("n", _class_ns())
def test_every_track_length_class_landmark_by_landmark(n, cfg):
    """W + 1 landmarks of track length n (one full tile, one ragged tile) with priors on every other landmark, so prior and
    prior-free landmarks share a tile; each landmark's update against the dense model from the handle's own camera
    increment: |d - d^| <= 1e-7 (|d^| + max_l |d^_l|) per landmark"""
    import rootba_b200 as rb
    from test_gpu_kernel_classes import problem
    prob = problem(n)
    prior = lp.prior_case(prob.lms, every=2, seed=n, sigma=0.02)
    lam = 1e-3
    Jp, Jl, r = dense_system(prob, landmarks=prior)
    D, sl, Jps, Jls, Minv, H, b = reduced(Jp, Jl, r, lam, prob.nl)
    bp = rb.BalProblem.from_arrays(prob, np.float64)
    bp.landmark_prior = prior
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(eta=1e-13, **cfg))
    lin.linearize()
    inc = lin.solve(lam)
    assert rel_err(lin.get_rhs(), b) < 1e-9
    lin.apply(None)
    lin.download_state()
    lin.close()
    dl = (sl * (-Minv @ (Jls.T @ r + Jls.T @ (Jps @ np.asarray(inc, np.float64))))).reshape(-1, 3)
    got = bp.lms - np.asarray(prob.lms, np.float64)
    scale = np.max(np.linalg.norm(dl, axis=1))
    for l in range(prob.nl):
        assert np.linalg.norm(got[l] - dl[l]) <= 1e-7 * (np.linalg.norm(dl[l]) + scale), (l, got[l], dl[l])


# ---- landmarks with one valid observation and with none ----------------------------------------------------------------
def _two_turned():
    """10 cameras, cameras 0 and 1 turned around (their observations are invalid): landmark 0 is seen by cameras 0 and 5
    (one valid observation), landmark 1 by cameras 0 and 1 (none)"""
    from rootba_b200.synthetic import synth_bal, turn_cameras_around
    rng = np.random.default_rng(5)
    tracks = [np.array([0, 5]), np.array([0, 1])] + [rng.choice(np.arange(2, 10), int(rng.integers(2, 6)), replace=False) for _ in range(120)]
    a = synth_bal(10, len(tracks), 0.0, seed=6, tracks=tracks, lm_spread=0.5)
    return turn_cameras_around(a, [0, 1])


@pytest.mark.parametrize("cfg", [CONFIGS_LMP[i] for i in (0, 4, 8, 9)], ids=cfg_id)
def test_priors_on_landmarks_with_one_and_without_valid_observations(cfg):
    """ERROR_VALID: cameras 0 and 1 have no valid observation and are held; landmark 0 (rank-2 Jl) carries a height-only
    prior, landmark 1 (no valid row) a dense one.  Both are full rank only with their prior: the step is finite (no NaN
    from the SC solver's Cholesky) and equals the dense model's"""
    import rootba_b200 as rb
    prob = _two_turned()
    rng = np.random.default_rng(4)
    idx = np.array([0, 1, 7, 20], np.int32)
    mean = np.asarray(prob.lms, np.float64)[idx] + rng.normal(0, 0.02, (4, 3))
    L = np.stack([lp.sqrt_info_kind(k, rng) for k in ("height", "dense", "dense", "rank2")])
    mask = np.zeros(prob.nc, np.uint8)
    mask[[0, 1]] = 15
    jp, jl, res, keep = cm.weighted(prob, valid_only=True)
    assert keep[0:2].sum() == 1 and keep[2:4].sum() == 0
    nobs, nc, nl = len(keep), prob.nc, prob.nl
    lm_of_obs = np.repeat(np.arange(nl), np.diff(prob.lm_off))
    Jp, Jl = np.zeros((2 * nobs, 9 * nc)), np.zeros((2 * nobs, 3 * nl))
    for k in range(nobs):
        Jp[2 * k:2 * k + 2, 9 * prob.obs_cam[k]:9 * prob.obs_cam[k] + 9] = jp[k]
        Jl[2 * k:2 * k + 2, 3 * lm_of_obs[k]:3 * lm_of_obs[k] + 3] = jl[k]
    Jp, Jl, r = lp.append_rows((Jp, Jl, res.ravel()), nl, prob.lms, idx, mean, L)
    lam = 1e-3
    D, sl, Jps, Jls, Minv, H, b = reduced(Jp, Jl, r, lam, nl)
    free = ~fixed_entries(mask)
    bp = rb.BalProblem.from_arrays(prob, np.float64)
    bp.landmark_prior = (idx, mean, L)
    bp.camera_fixed = mask
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(eta=1e-13, optimized_cost="ERROR_VALID", **cfg))
    lin.linearize()
    inc = np.asarray(lin.solve(lam), np.float64)
    assert np.all(np.isfinite(inc)) and np.all(inc[~free] == 0)
    Hff = H[np.ix_(free, free)]
    if cfg.get("solver_type") != "POWER_SCHUR_COMPLEMENT":  # the truncated series is not the direct solve (it is finite)
        assert rel_err(inc[free], -np.linalg.solve(Hff, b[free])) < max(1e-6, np.sqrt(1e-13 * np.linalg.cond(Hff)))
    l_diff = lin.apply(None)
    lin.download_state()
    lin.close()
    dl = -Minv @ (Jls.T @ r + Jls.T @ (Jps @ inc))
    want_l = 0.5 * r @ r - 0.5 * np.sum((r + Jps @ inc + Jls @ dl) ** 2)
    assert np.isfinite(l_diff) and abs(l_diff - want_l) <= 1e-8 * abs(want_l)
    assert np.all(np.isfinite(bp.lms))
    assert rel_err(bp.lms[:2], np.asarray(prob.lms, np.float64)[:2] + (sl * dl).reshape(-1, 3)[:2]) < 1e-9


# ---- no behaviour change without priors, bad input ---------------------------------------------------------------------
@pytest.mark.parametrize("cfg", [CONFIGS_LMP[i] for i in (0, 4, 12, 8, 9)], ids=cfg_id)
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_no_behaviour_change_without_landmark_priors(small_problem, dtype, cfg):
    """priors set and cleared (None or num = 0), or all with a zero L: the LM trajectory of a handle that never had any, bit
    for bit"""
    import rootba_b200 as rb
    from objective_checks import assert_identical_steps, lm_steps
    run = lambda mode: lm_steps(small_problem, dtype, cfg, mode, rb.LinearizorQR.set_landmark_prior,
                                lp.prior_case(small_problem.lms, every=5, seed=2))
    ref = run("never")
    for mode in ("set_then_none", "set_then_empty", "zeros"):
        assert_identical_steps(ref, run(mode), mode)


def test_bad_input_keeps_the_previous_landmark_priors(small_problem):
    import rootba_b200 as rb
    from rootba_b200 import _lib
    lib = _lib.lib()
    idx, mean, L = lp.prior_case(small_problem.lms, every=5, seed=2)
    bp = rb.BalProblem.from_arrays(small_problem, np.float64)
    bp.landmark_prior = (idx, mean, L)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions())
    lin.compute_error()
    lin.linearize()
    inc_ref = lin.solve(1e-4)
    p = lambda a: C.c_void_p(a.ctypes.data)
    m = len(idx)
    bad_L, bad_m = L.copy(), mean.copy()
    bad_L[3, 1, 2] = np.nan
    bad_m[2, 0] = np.inf
    out_of_range, negative, dup = idx.copy(), idx.copy(), idx.copy()
    out_of_range[5] = small_problem.nl
    negative[6] = -1
    dup[7] = dup[8]
    cases = [(-1, p(idx), p(mean), p(L)), (m, None, p(mean), p(L)), (m, p(idx), None, p(L)), (m, p(idx), p(mean), None),
             (m, p(out_of_range), p(mean), p(L)), (m, p(negative), p(mean), p(L)), (m, p(dup), p(mean), p(L)),
             (m, p(idx), p(mean), p(bad_L)), (m, p(idx), p(bad_m), p(L))]
    for args in cases:
        assert lib.rba_set_landmark_prior(lin.h, *args) == -1  # RBA_ERR_INVALID_ARGUMENT
        assert lib.rba_last_error()
    assert np.array_equal(lin.solve(1e-4), inc_ref)  # nothing changed, still linearised
    for bad in ((out_of_range, mean, L), (dup, mean, L), (idx, mean, bad_L), (idx[:, None], mean, L), (idx, mean[:, :2], L)):
        with pytest.raises(ValueError):
            lin.set_landmark_prior(bad)
    assert np.array_equal(bp.landmark_prior[1], mean)
    lin.set_landmark_prior((idx, mean, L))  # a change needs a new linearisation
    with pytest.raises(rb.RbaError) as e:
        lin.solve(1e-4)
    assert e.value.code == -6  # RBA_ERR_STATE
    lin.linearize()
    assert np.array_equal(lin.solve(1e-4), inc_ref)
    lin.close()


# ---- end to end against scipy -------------------------------------------------------------------------------------------
def _e2e_problem():
    """a perturbed synthetic problem with ground control points (dense L, sigma 0.1, on every 6th landmark, a height-only
    one among them), pair priors between consecutive cameras, a centre prior on camera 1, and camera 0 held"""
    from rootba_b200.synthetic import BalArrays, synth_bal
    from scipy.spatial.transform import Rotation
    prob = synth_bal(8, 150, 4.0, seed=31)
    rng = np.random.default_rng(35)
    truth_c, truth_l = np.asarray(prob.cams, np.float64), np.asarray(prob.lms, np.float64)
    idx = np.arange(0, prob.nl, 6, dtype=np.int32)
    mean = truth_l[idx] + rng.normal(0, 0.01, (len(idx), 3))
    L = np.stack([10.0 * np.eye(3) if p % 5 else np.diag([0.0, 0.0, 10.0]) for p in range(len(idx))])
    pairs = np.array([(c, c + 1) for c in range(prob.nc - 1)], np.int32)
    pmean = qm.mean_at(truth_c, pairs)
    pmean[:, 4:7] += rng.normal(0, 0.01, (len(pairs), 3))
    pL = np.tile(np.diag([1.0, 1.0, 1.0, 100.0, 100.0, 100.0]), (len(pairs), 1, 1))
    cmean = pm.mean_at(truth_c)
    cL = np.zeros((prob.nc, 9, 9))
    cL[1, 0:3, 0:3] = 2.0 * np.eye(3)
    mask = np.zeros(prob.nc, np.uint8)
    mask[0] = 15
    cams = truth_c.copy()
    for c in range(1, prob.nc):
        cams[c, :4] = (Rotation.from_rotvec(rng.normal(0, 0.01, 3)) * Rotation.from_quat(cams[c, :4])).as_quat()
        cams[c, 4:7] += rng.normal(0, 0.02, 3)
        cams[c, 7] *= 1 + rng.normal(0, 0.01)
    lms = truth_l + rng.normal(0, 0.02, truth_l.shape)
    return BalArrays(cams, lms, prob.lm_off, prob.obs_cam, prob.obs_xy), (idx, mean, L), (pairs, pmean, pL), (cmean, cL), mask


def test_lm_run_reaches_the_scipy_minimum_with_every_prior_kind_and_held_cameras():
    """the ground control points, the held camera and the camera prior fix the gauge, so the landmarks themselves are
    compared"""
    import rootba_b200 as rb
    from objective_checks import scipy_minimum
    prob, lmp, pair, camp, mask = _e2e_problem()
    _, lms_s, cost_s = scipy_minimum(prob, camera=camp, pairs=pair, landmarks=lmp, mask=mask)
    so = rb.SolverOptions(max_num_iterations=60, function_tolerance=1e-15, eta=1e-10)
    runs = {}
    for dtype in (np.float64, np.float32):
        bp = rb.BalProblem.from_arrays(prob, dtype)
        bp.landmark_prior = lmp
        bp.camera_pair_prior = pair
        bp.camera_prior = camp
        bp.camera_fixed = mask
        lin = rb.LinearizorQR.create(bp, so)
        lin.lm_run(200)
        lin.download_state()
        cost = lin.compute_error()["all"]["error"]
        lin.close()
        runs[dtype] = (bp, cost)
    bp, cost = runs[np.float64]
    assert abs(cost - cost_s) <= 1e-8 * cost_s, (cost, cost_s)
    assert np.max(np.abs(bp.lms - lms_s)) < 1e-4 * max(1.0, np.max(np.abs(lms_s)))
    assert np.array_equal(bp.cams[0], np.asarray(prob.cams[0], np.float64))
    assert abs(runs[np.float32][1] - cost) <= 1e-4 * cost


# ---- covariances --------------------------------------------------------------------------------------------------------
def _dense_covariance_check(cam, lm, Jp, Jl, fixed):
    """cam / lm against the dense inverse of J^T J (unscaled, the held entries removed): componentwise
    |S - S^| <= 8 N kappa u sqrt(S^_ii S^_jj), kappa of the equilibrated matrix; returns the bar"""
    J = np.hstack([Jp[:, ~fixed], Jl])
    A = J.T @ J
    d = 1.0 / np.sqrt(np.diag(A))
    kappa = np.linalg.cond(d[:, None] * A * d[None, :])
    S = np.linalg.inv(A)
    N = A.shape[0]
    bar = 8 * N * kappa * 2.0 ** -53
    assert bar <= 1e-4, bar
    nf = int((~fixed).sum())
    Sc = np.zeros((len(fixed), len(fixed)))
    Sc[np.ix_(~fixed, ~fixed)] = S[:nf, :nf]
    sd = np.sqrt(np.abs(np.diag(Sc)))
    for c in range(len(cam)):
        sel = slice(9 * c, 9 * c + 9)
        assert np.all(np.abs(cam[c] - Sc[sel, sel]) <= bar * np.outer(sd[sel], sd[sel]) + 1e-300), c
    Sl = S[nf:, nf:]
    sdl = np.sqrt(np.diag(Sl))
    for l in range(len(lm)):
        sel = slice(3 * l, 3 * l + 3)
        assert np.all(np.abs(lm[l] - Sl[sel, sel]) <= bar * np.outer(sdl[sel], sdl[sel])), l
    return bar


def test_covariance_with_the_gauge_fixed_by_landmark_priors_alone():
    """no camera prior and no held camera: dense priors on every 3rd landmark fix the similarity gauge"""
    import rootba_b200 as rb
    from rootba_b200.synthetic import synth_bal
    prob = synth_bal(7, 90, 3.6, seed=21)
    prior = lp.prior_case(prob.lms, every=3, seed=6, kinds=("dense",), scale=5.0)
    bp = rb.BalProblem.from_arrays(prob, np.float64)
    bp.landmark_prior = prior
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions())
    cam, lm = lin.covariance()
    lin.close()
    Jp, Jl, _ = dense_system(prob, landmarks=prior)
    _dense_covariance_check(cam, lm, Jp, Jl, np.zeros(9 * prob.nc, bool))
    # without the priors the gauge is free
    bp2 = rb.BalProblem.from_arrays(prob, np.float64)
    lin2 = rb.LinearizorQR.create(bp2, rb.SolverOptions())
    with pytest.raises(rb.RbaError):
        lin2.covariance()
    lin2.close()


def test_covariance_of_a_rank2_landmark_with_a_prior_is_finite():
    """ERROR_VALID on the two-turned problem (cameras 0 and 1 held): landmark 0 (one valid observation) with a height-only
    prior and landmark 1 (none) with a dense one get finite blocks; landmark priors elsewhere fix the gauge"""
    import rootba_b200 as rb
    prob = _two_turned()
    rng = np.random.default_rng(12)
    idx = np.array([0, 1] + list(range(10, prob.nl, 9)), np.int32)
    mean = np.asarray(prob.lms, np.float64)[idx] + rng.normal(0, 0.02, (len(idx), 3))
    L = np.stack([np.diag([0.0, 0.0, 3.0]), 3.0 * np.eye(3)] + [lp.sqrt_info_kind("dense", rng, 3.0) for _ in idx[2:]])
    mask = np.zeros(prob.nc, np.uint8)
    mask[[0, 1]] = 15
    bp = rb.BalProblem.from_arrays(prob, np.float64)
    bp.landmark_prior = (idx, mean, L)
    bp.camera_fixed = mask
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(optimized_cost="ERROR_VALID"))
    cam, lm = lin.covariance()
    lin.close()
    assert np.all(np.isfinite(lm)) and np.all(np.isfinite(cam))
    jp, jl, res, keep = cm.weighted(prob, valid_only=True)
    nobs, nc, nl = len(keep), prob.nc, prob.nl
    lm_of_obs = np.repeat(np.arange(nl), np.diff(prob.lm_off))
    Jp, Jl = np.zeros((2 * nobs, 9 * nc)), np.zeros((2 * nobs, 3 * nl))
    for k in range(nobs):
        Jp[2 * k:2 * k + 2, 9 * prob.obs_cam[k]:9 * prob.obs_cam[k] + 9] = jp[k]
        Jl[2 * k:2 * k + 2, 3 * lm_of_obs[k]:3 * lm_of_obs[k] + 3] = jl[k]
    Jp, Jl, _ = lp.append_rows((Jp, Jl, res.ravel()), nl, prob.lms, idx, mean, L)
    _dense_covariance_check(cam, lm, Jp, Jl, fixed_entries(mask))


# ---- two GPUs ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("peer", ["1", "0"])
@pytest.mark.parametrize("sfx", ["f32", "f64"])
def test_two_ranks_with_landmark_priors(tmp_path, peer, sfx):
    """each shard adds its own landmark priors before the sum over the shards: the sharded step equals the single-rank step"""
    res = check_two_rank_step(tmp_path, "landmark", sfx, peer, 29500, (23 if peer == "1" else 0) + (29 if sfx == "f32" else 0))
    assert min(res["priors_per_shard"]) > 0, res
