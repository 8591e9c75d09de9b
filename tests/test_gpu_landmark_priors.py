"""Gaussian priors on landmark positions (rba_set_landmark_prior) on the GPU: every solver configuration against the dense
float64 algebra of the total (reprojection + landmark prior) problem in both precisions, every track-length class landmark by
landmark with prior and prior-free landmarks in one tile, lambda = 0, rank-deficient L, landmarks with one and with no valid
observation, no behaviour change without priors, bad input, an end-to-end minimum against scipy with every other prior
kind and held cameras, covariances with the gauge fixed by landmark priors, and the sharded path."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import camera_model as cm
import camera_prior_model as pm
import landmark_prior_model as lp
import pair_prior_model as qm
from conftest import ROOT, rel_err
from test_camera_prior_model import prior_case as camera_prior_case
from test_fixed_cameras import fixed_entries
from test_gpu_camera_priors import BARS, _ID, _ngpu, _reduced
from test_gpu_fixed_cameras import CONFIGS, fixed_params

pytestmark = pytest.mark.gpu

# CONFIGS of test_gpu_fixed_cameras (SQUARE_ROOT dense / implicit x Householder / Givens x JACOBI / SCHUR_JACOBI, SC, Power-SC)
# and the dense operator with stage2_form = IDENTITY (k_stage2<S, false>)
CONFIGS_LMP = CONFIGS + [dict(solver_type="SQUARE_ROOT", operator_form="DENSE", use_householder_marginalization=hh,
                              preconditioner_type=pc, stage2_form="IDENTITY") for hh in (True, False) for pc in ("JACOBI", "SCHUR_JACOBI")]


def _stored(prob, dtype):
    """prob with its state and observations rounded to the handle's scalar type (compared in float64 from there)"""
    from rootba_b200.synthetic import BalArrays
    f = lambda a: np.asarray(np.asarray(a, dtype), np.float64)
    return BalArrays(f(prob.cams), f(prob.lms), prob.lm_off, prob.obs_cam, f(prob.obs_xy))


def _check_against_dense(cfg, prob, prior, dtype=np.float64, cam_prior=None, mask=None, lam=1e-3, env=None, monkeypatch=None):
    import rootba_b200 as rb
    from rootba_b200.synthetic import BalArrays
    bars = BARS[dtype]
    idx, mean, L = prior
    sprior = (idx, np.asarray(np.asarray(mean, dtype), np.float64), np.asarray(np.asarray(L, dtype), np.float64))
    sprob = _stored(prob, dtype)
    Jp, Jl, r = lp.dense_system(sprob, sprior, cam_prior)
    D, sl, Jps, Jls, Minv, H, b = _reduced(Jp, Jl, r, lam, prob.nl, dtype)
    n = H.shape[0]
    fixed = fixed_entries(mask) if mask is not None else np.zeros(n, bool)
    free = ~fixed
    bp = rb.BalProblem.from_arrays(prob, dtype)
    bp.landmark_prior = prior
    if cam_prior is not None:
        bp.camera_prior = cam_prior
    if mask is not None:
        bp.camera_fixed = mask
    so = rb.SolverOptions(eta=1e-13, **cfg)
    if monkeypatch is not None:
        with monkeypatch.context() as m:
            for k, v in (env or {}).items():
                m.setenv(k, v)
            lin = rb.LinearizorQR.create(bp, so)
    else:
        lin = rb.LinearizorQR.create(bp, so)
    cams0 = bp.cams.copy()
    e0 = lin.compute_error()["all"]["error"]
    assert abs(e0 - lp.total_cost(sprob, sprior, cam_prior)) <= bars["cost"] * e0
    lin.linearize()
    inc = lin.solve(lam)
    s, _ = lin.get_jacobian_scaling()
    assert rel_err(s, D) < bars["scaling"]
    assert rel_err(lin.get_rhs(), np.where(fixed, 0.0, b)) < bars["b"]
    inv, blk = lin.get_preconditioner()
    power = cfg.get("solver_type") == "POWER_SCHUR_COMPLEMENT"
    jacobi = power or cfg.get("preconditioner_type") == "JACOBI"
    Hp = Jps.T @ Jps + lam * np.eye(n) if jacobi else H  # the landmark-prior rows have no camera columns
    for c in range(prob.nc):
        sel = slice(9 * c, 9 * c + 9)
        f = free[sel]
        want = np.zeros((9, 9))
        want[np.ix_(f, f)] = np.linalg.inv(Hp[sel, sel][np.ix_(f, f)])
        assert rel_err(inv[c], want) < bars["inv"], c
        if not jacobi:
            assert rel_err(blk[c], Hp[sel, sel]) < bars["blocks"], c
    x = np.random.default_rng(1).uniform(-1, 1, n)
    assert rel_err(lin.right_multiply(x), H @ x) < bars["op"]
    assert np.all(inc[fixed] == 0)
    Hff, bf = H[np.ix_(free, free)], b[free]
    tol_inc = bars["inc"]
    if dtype == np.float32:
        tol_inc = max(tol_inc, 100 * 2.0 ** -24 * np.linalg.cond(Hff))  # as test_gpu_camera_priors
    if power:
        W = Jps.T @ Jls
        E0 = (W @ Minv @ W.T)[np.ix_(free, free)]
        Hinv = np.linalg.inv((Jps.T @ Jps + lam * np.eye(n))[np.ix_(free, free)])
        tmp = -Hinv @ bf
        acc = tmp.copy()
        for i in range(1, so.power_order + 1):
            tmp = Hinv @ (E0 @ tmp)
            acc = acc + tmp
            if i * np.linalg.norm(tmp) / np.linalg.norm(acc) < so.eta:
                break
        assert rel_err(inc[free], acc) < (1e-9 if dtype == np.float64 else tol_inc)
    else:
        if dtype == np.float64:
            assert lin.last_cg.termination_type == 1
            tol_inc = max(tol_inc, np.sqrt(so.eta * np.linalg.cond(Hff)))  # as test_gpu_pair_priors
        assert rel_err(inc[free], -np.linalg.solve(Hff, bf)) < tol_inc
    inc64 = np.asarray(inc, np.float64)
    dl_s = -Minv @ (Jls.T @ r + Jls.T @ (Jps @ inc64))
    want_l = 0.5 * r @ r - 0.5 * np.sum((r + Jps @ inc64 + Jls @ dl_s) ** 2)
    l_diff = lin.apply(None)
    assert abs(l_diff - want_l) <= bars["l_diff"] * abs(want_l)
    lin.download_state()
    want_lms = sprob.lms + (sl * dl_s).reshape(-1, 3)
    assert rel_err(bp.lms, want_lms) < bars["lms"]
    e1 = lin.compute_error()["all"]["error"]
    new = BalArrays(bp.cams.astype(np.float64), bp.lms.astype(np.float64), prob.lm_off, prob.obs_cam, sprob.obs_xy)
    want_e1 = lp.total_cost(new, sprior, cam_prior)
    assert abs(e1 - want_e1) <= bars["cost"] * want_e1
    if mask is not None:
        fp = fixed_params(mask)
        assert np.array_equal(bp.cams[fp], cams0[fp])
    lin.close()
    return dl_s, sl


@pytest.fixture(scope="module")
def case7():
    from rootba_b200.synthetic import synth_bal
    prob = synth_bal(7, 90, 3.6, seed=21)
    return prob, lp.prior_case(prob.lms, every=3, seed=5)


@pytest.mark.parametrize("cfg", CONFIGS_LMP, ids=_ID)
def test_f64_against_dense_system_with_landmark_priors(cfg, case7):
    _check_against_dense(cfg, *case7)


@pytest.mark.parametrize("cfg", CONFIGS_LMP, ids=_ID)
def test_f32_against_dense_system_with_landmark_priors(cfg, case7):
    _check_against_dense(cfg, *case7, dtype=np.float32)


@pytest.mark.parametrize("cfg", CONFIGS_LMP, ids=_ID)
def test_f64_landmark_and_camera_priors_with_held_parameters(cfg):
    """with the camera priors of test_camera_prior_model.prior_case (an unobserved camera held by its prior) and a held
    camera"""
    prob, mean_c, L_c = camera_prior_case(7, 90)
    mask = np.zeros(prob.nc, np.uint8)
    mask[2] = 15
    mask[4] = 14
    _check_against_dense(cfg, prob, lp.prior_case(prob.lms, every=2, seed=8), cam_prior=(mean_c, L_c), mask=mask)


@pytest.mark.parametrize("cfg", [CONFIGS_LMP[i] for i in (0, 3, 5, 8, 9, 10)], ids=_ID)
def test_lambda_zero_and_rank_one_priors(cfg):
    """lambda = 0: the prior landmarks' damping rows are [C | 0 | c] of L~ alone (the lambda = 0 shortcut must not skip
    them); height-only (rank-1) priors in the mix; the gauge fixed by camera priors"""
    prob, mean_c, L_c = camera_prior_case(7, 90)
    prior = lp.prior_case(prob.lms, every=2, seed=9, kinds=("height", "dense", "height", "rank2"))
    _check_against_dense(cfg, prob, prior, cam_prior=(mean_c, L_c), lam=0.0)


# ---- every track-length class, landmark by landmark ---------------------------------------------------------------------
def _class_ns():
    from test_gpu_kernel_classes import CASES, _signature
    return [n for n in CASES if n == 2 or _signature(n) != _signature(n - 1)]


@pytest.mark.parametrize("cfg", [CONFIGS_LMP[i] for i in (0, 4, 12, 8)], ids=_ID)
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
    Jp, Jl, r = lp.dense_system(prob, prior)
    D, sl, Jps, Jls, Minv, H, b = _reduced(Jp, Jl, r, lam, prob.nl, np.float64)
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


@pytest.mark.parametrize("cfg", [CONFIGS_LMP[i] for i in (0, 4, 8, 9)], ids=_ID)
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
    D, sl, Jps, Jls, Minv, H, b = _reduced(Jp, Jl, r, lam, nl, np.float64)
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
def _lm_steps(arrays, dtype, cfg, mode, steps=3):
    import rootba_b200 as rb
    bp = rb.BalProblem.from_arrays(arrays, dtype)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(**cfg))
    prior = lp.prior_case(arrays.lms, every=5, seed=2)
    if mode == "set_then_none":
        lin.set_landmark_prior(prior)
        lin.set_landmark_prior(None)
    elif mode == "set_then_empty":
        lin.set_landmark_prior(prior)
        lin.set_landmark_prior((np.zeros(0, np.int32), np.zeros((0, 3)), np.zeros((0, 3, 3))))
    elif mode == "zeros":
        lin.set_landmark_prior((prior[0], prior[1], np.zeros_like(prior[2])))
    out = []
    cost = lin.compute_error()["all"]["error"]
    for _ in range(steps):
        lin.linearize()
        inc = lin.solve(1e-4)
        l_diff = lin.apply(None)
        lin.download_state()
        out.append((inc, l_diff, bp.cams.copy(), bp.lms.copy(), lin.compute_error()["all"]["error"]))
    lin.close()
    return cost, out


@pytest.mark.parametrize("cfg", [CONFIGS_LMP[i] for i in (0, 4, 12, 8, 9)], ids=_ID)
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_no_behaviour_change_without_landmark_priors(small_problem, dtype, cfg):
    """priors set and cleared (None or num = 0), or all with a zero L: the LM trajectory of a handle that never had any, bit
    for bit"""
    c0, ref = _lm_steps(small_problem, dtype, cfg, "never")
    for mode in ("set_then_none", "set_then_empty", "zeros"):
        c1, got = _lm_steps(small_problem, dtype, cfg, mode)
        assert c0 == c1, mode
        for a, b in zip(ref, got):
            assert np.array_equal(a[0], b[0]) and a[1] == b[1] and a[4] == b[4], mode
            assert np.array_equal(a[2], b[2]) and np.array_equal(a[3], b[3]), mode


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


def _scipy_minimum(prob, lmp, pair, camp, mask):
    from scipy.optimize import least_squares
    from scipy.spatial.transform import Rotation
    nc, nl = prob.nc, prob.nl
    free_c = np.flatnonzero(mask == 0)
    lm_of_obs = np.repeat(np.arange(nl), np.diff(prob.lm_off))
    base = np.asarray(prob.cams, np.float64)

    def unpack(x):
        pc = x[:9 * len(free_c)].reshape(-1, 9)
        cams = base.copy()
        cams[free_c, :4] = Rotation.from_rotvec(pc[:, :3]).as_quat()
        cams[free_c, 4:7], cams[free_c, 7:10] = pc[:, 3:6], pc[:, 6:9]
        return cams, x[9 * len(free_c):].reshape(nl, 3)

    def fun(x):
        cams, lms = unpack(x)
        res = cm.linearize(cams[prob.obs_cam], lms[lm_of_obs], prob.obs_xy)["res"].ravel()
        pri = [L @ (lms[i] - m) for i, m, L in zip(*lmp)]
        pri += [pair[2][p] @ qm.residual(cams[i], cams[j], pair[1][p]) for p, (i, j) in enumerate(pair[0])]
        pri += [camp[1][c] @ pm.residual(cams[c], camp[0][c]) for c in range(nc)]
        return np.concatenate([res, np.concatenate(pri)])

    x0 = np.concatenate([np.hstack([Rotation.from_quat(base[free_c, :4]).as_rotvec(), base[free_c, 4:10]]).ravel(), np.ravel(prob.lms)])
    sol = least_squares(fun, x0, method="trf", x_scale="jac", xtol=1e-15, ftol=1e-15, gtol=1e-15, max_nfev=200)
    cams, lms = unpack(sol.x)
    return cams, lms, float(sol.cost)


def test_lm_run_reaches_the_scipy_minimum_with_every_prior_kind_and_held_cameras():
    """the ground control points, the held camera and the camera prior fix the gauge, so the landmarks themselves are
    compared"""
    import rootba_b200 as rb
    prob, lmp, pair, camp, mask = _e2e_problem()
    _, lms_s, cost_s = _scipy_minimum(prob, lmp, pair, camp, mask)
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
    Jp, Jl, _ = lp.dense_system(prob, prior)
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
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    out = tmp_path / "res.json"
    env = dict(os.environ, RBA_PEER_AR=peer, MASTER_ADDR="127.0.0.1")
    port = 29500 + (os.getpid() + (23 if peer == "1" else 0) + (29 if sfx == "f32" else 0)) % 2000
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "tests", "multirank_landmark_prior_worker.py"), str(out), sfx]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    res = json.loads(out.read_text())
    tols = 1e-4 if sfx == "f32" else 1e-8  # the bars of test_gpu_multirank.py
    assert res["replicas_identical"] and min(res["priors_per_shard"]) > 0, res
    assert res["b"] < 4 * tols and res["inc"] < tols and res["l_diff"] < 20 * tols, res
    assert res["lms"] < 10 * tols and res["cams"] < tols and res["cost"] < tols and res["cost0"] < tols, res
