"""Robust losses on the priors (rba_set_prior_loss, rba_get_prior_residuals, DESIGN.md section 22) on the GPU, against the
float64 model of tests/prior_loss_model.py: one LM step of every solver configuration in both precisions against the dense
weighted total system, the unmodified path, TUKEY rejection, both covariance entry points, the read-back, the new kernels at
their thread-block edges, LM runs on a pose chain with false loop closures, the problem-term protocol and the example."""
import os
import subprocess
import sys

import numpy as np
import pytest

import camera_model as cm
import covariance_model as cvm
import objective_checks as oc
import observation_loss_model as olm
import pair_prior_model as qm
import prior_loss_model as plm
from conftest import ROOT, rel_err

pytestmark = pytest.mark.gpu

DTYPES = [np.float64, np.float32]
dt_id = lambda d: np.dtype(d).name
ALL = (olm.NONE, olm.HUBER, olm.CAUCHY, olm.SOFT_L1, olm.TUKEY)


def rounded(prob, priors, dtype):
    from rootba_b200.synthetic import BalArrays
    f = lambda a: np.asarray(np.asarray(a, dtype), np.float64)
    sprob = BalArrays(f(prob.cams), f(prob.lms), prob.lm_off, prob.obs_cam, f(prob.obs_xy))
    return sprob, {k: oc._stored(v, dtype) for k, v in priors.items()}


def make(prob, dtype, priors, losses, **opts):
    """a handle with the priors and their losses (losses: prior kind -> (kind, scale) or None) set on the BalProblem"""
    import rootba_b200 as rb
    bp = oc.bal_problem(prob, dtype, camera_prior=priors.get("camera"), camera_pair_prior=priors.get("pairs"),
                        landmark_prior=priors.get("landmarks"))
    for k, loss in losses.items():
        if loss is not None:
            bp._set_prior_loss(k, loss)
    return bp, rb.LinearizorQR.create(bp, rb.SolverOptions(**opts))


def robust_total_cost(prob, priors, losses):
    return float(cm.compute_error(prob)["all"]["error"]) + plm.prior_cost((prob.cams, prob.lms), priors, losses)


def check_robust_step(cfg, prob, priors, losses, dtype, lam=1e-3):
    """check_against_dense of tests/objective_checks.py for robust priors: the dense model is that of the priors with L
    replaced by sqrt(w) L, w at the (rounded) state of the linearisation, and the costs are the robust ones"""
    bars = oc.BARS[dtype]
    sprob, model = rounded(prob, priors, dtype)
    state = (sprob.cams, sprob.lms)
    Jp, Jl, r = oc.dense_system(sprob, **plm.weighted_all(state, model, losses))
    D, sl, Jps, Jls, Minv, H, b = oc.reduced(Jp, Jl, r, lam, prob.nl, dtype)
    import rootba_b200 as rb
    so = rb.SolverOptions(eta=1e-13, **cfg)
    bp, lin = make(prob, dtype, priors, losses, eta=1e-13, **cfg)
    e0 = lin.compute_error()["all"]["error"]
    assert abs(e0 - robust_total_cost(sprob, model, losses)) <= bars["cost"] * e0
    lin.linearize()
    inc = lin.solve(lam)
    # float32: w = rho'(s) carries the float32 error of s = |L e|^2, and the scaling sqrt(w) of it, so its bar is twice the
    # unweighted one
    assert rel_err(lin.get_jacobian_scaling()[0], D) < bars["scaling"] * (2 if dtype == np.float32 else 1)
    assert rel_err(lin.get_rhs(), b) < bars["b"]
    inv, blk = lin.get_preconditioner()
    power = cfg.get("solver_type") == "POWER_SCHUR_COMPLEMENT"
    jacobi = power or cfg.get("preconditioner_type") == "JACOBI"
    Hpp, O = qm.power_split(Jps, lam)
    for c in range(prob.nc):
        sel = slice(9 * c, 9 * c + 9)
        assert rel_err(inv[c], np.linalg.inv(Hpp[sel, sel] if jacobi else H[sel, sel])) < bars["inv"], c
    x = np.random.default_rng(1).uniform(-1, 1, H.shape[0])
    assert rel_err(lin.right_multiply(x), H @ x) < bars["op"]
    tol_inc = bars["inc"] if dtype == np.float64 else max(bars["inc"], 100 * 2.0 ** -24 * np.linalg.cond(H))
    if power:
        W = Jps.T @ Jls
        want = qm.power_series(Hpp, W @ Minv @ W.T - O, b, so.power_order, so.eta)
        assert rel_err(inc, want) < (1e-9 if dtype == np.float64 else tol_inc)
    else:
        if dtype == np.float64:
            assert lin.last_cg.termination_type == 1
        assert rel_err(inc, -np.linalg.solve(H, b)) < tol_inc
    inc64 = np.asarray(inc, np.float64)
    dl_s = -Minv @ (Jls.T @ r + Jls.T @ (Jps @ inc64))
    want_l = 0.5 * r @ r - 0.5 * np.sum((r + Jps @ inc64 + Jls @ dl_s) ** 2)
    l_diff = lin.apply(None)
    assert abs(l_diff - want_l) <= bars["l_diff"] * abs(want_l)
    lin.download_state()
    from rootba_b200.synthetic import BalArrays
    new = BalArrays(bp.cams.astype(np.float64), bp.lms.astype(np.float64), prob.lm_off, prob.obs_cam, sprob.obs_xy)
    e1 = lin.compute_error()["all"]["error"]
    assert abs(e1 - robust_total_cost(new, model, losses)) <= bars["cost"] * e1
    lin.close()


@pytest.fixture(scope="module")
def case():
    return plm.robust_case()


def losses_for(prob, priors, kinds, seed=0):
    state = (np.asarray(prob.cams, np.float64), np.asarray(prob.lms, np.float64))
    return {k: plm.losses_around(k, state, priors[plm.KINDS[k]], seed + k) for k in kinds}


@pytest.mark.parametrize("dtype", DTYPES, ids=dt_id)
@pytest.mark.parametrize("kind", [plm.CAMERA, plm.PAIR, plm.LANDMARK], ids=["camera", "pair", "landmark"])
@pytest.mark.parametrize("cfg", oc.CONFIGS, ids=oc.cfg_id)
def test_step_against_the_dense_weighted_system(case, cfg, kind, dtype):
    """every loss kind in turn over the priors of one kind (the others quadratic), every solver configuration"""
    prob, priors = case
    check_robust_step(cfg, prob, priors, losses_for(prob, priors, [kind]), dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=dt_id)
def test_all_three_kinds_together(case, dtype):
    prob, priors = case
    check_robust_step(oc.CONFIGS[0], prob, priors, losses_for(prob, priors, [0, 1, 2], seed=3), dtype)


def lm_steps(bp_lin, steps=3):
    bp, lin = bp_lin
    out = [lin.compute_error()["all"]["error"]]
    for _ in range(steps):
        lin.linearize()
        inc = lin.solve(1e-4)
        l_diff = lin.apply(None)
        lin.download_state()
        out.append((inc, l_diff, bp.cams.copy(), bp.lms.copy(), lin.compute_error()["all"]["error"]))
    lin.close()
    return out


def same_steps(a, b):
    assert a[0] == b[0]
    for x, y in zip(a[1:], b[1:]):
        assert np.array_equal(x[0], y[0]) and x[1] == y[1] and x[4] == y[4]
        assert np.array_equal(x[2], y[2]) and np.array_equal(x[3], y[3])


@pytest.mark.parametrize("dtype", DTYPES, ids=dt_id)
def test_none_set_explicitly_is_bit_identical_to_unset(case, dtype):
    prob, priors = case
    ref = lm_steps(make(prob, dtype, priors, {}))
    none = {k: (np.zeros(len(priors[n][-1]), np.uint8), np.full(len(priors[n][-1]), np.nan)) for k, n in enumerate(plm.KINDS)}
    same_steps(ref, lm_steps(make(prob, dtype, priors, none)))
    # set, then cleared with NULL
    bp, lin = make(prob, dtype, priors, losses_for(prob, priors, [0, 1, 2]))
    for k in range(3):
        lin.set_prior_loss(k, None)
    same_steps(ref, lm_steps((bp, lin)))


@pytest.mark.parametrize("dtype", DTYPES, ids=dt_id)
def test_tukey_beyond_its_scale_is_the_prior_removed(case, dtype):
    """a TUKEY pair with w = 0 (its rows zero) against the same pair with L = 0 (dropped): the same step; the cost differs by
    a^2/6, with a a quarter of the pair's |L e| so that the constant stands well above the bar in float64"""
    prob, priors = case
    pairs = priors["pairs"]
    m = len(pairs[0])
    sprob, model = rounded(prob, priors, dtype)
    k = np.zeros(m, np.uint8)
    a = np.full(m, np.nan)
    k[0], a[0] = olm.TUKEY, 0.25 * np.linalg.norm(plm.whitened(plm.PAIR, (sprob.cams, sprob.lms), model["pairs"])[0])
    removed = dict(priors, pairs=(pairs[0], pairs[1], pairs[2].copy()))
    removed["pairs"][2][0] = 0
    ref = lm_steps(make(prob, dtype, removed, {}))
    got = lm_steps(make(prob, dtype, priors, {plm.PAIR: (k, a)}))
    tol = 1e-10 if dtype == np.float64 else 1e-5
    const = float(np.asarray(a[0], dtype)) ** 2 / 6
    if dtype == np.float64:
        assert const > 100 * tol * ref[0]  # dropping the constant would fail the next line
    assert abs(got[0] - ref[0] - const) <= tol * ref[0]
    for x, y in zip(got[1:], ref[1:]):
        assert rel_err(x[0], y[0]) < tol and abs(x[1] - y[1]) <= tol * abs(y[1]) and rel_err(x[2], y[2]) < tol


@pytest.mark.parametrize("entry", ["covariance", "blocks"])
@pytest.mark.parametrize("when", ["linearized", "moved_after_linearize", "never_linearized"])
def test_covariance_uses_the_weights_at_the_current_state(case, when, entry):
    prob, priors = case
    losses = losses_for(prob, priors, [0, 1, 2], seed=7)
    losses[plm.CAMERA] = (np.where(losses[plm.CAMERA][0] == olm.TUKEY, olm.CAUCHY, losses[plm.CAMERA][0]).astype(np.uint8),
                          np.where(losses[plm.CAMERA][0] == olm.NONE, np.nan, np.nan_to_num(losses[plm.CAMERA][1], nan=1.0)))
    bp, lin = make(prob, np.float64, priors, losses)
    if when != "never_linearized":
        lin.linearize()
    if when == "moved_after_linearize":
        bp.cams[:, 4:7] += 0.05
        bp.lms += 0.02
        lin.upload_state()
    from rootba_b200.synthetic import BalArrays
    cur = BalArrays(bp.cams.copy(), bp.lms.copy(), prob.lm_off, prob.obs_cam, prob.obs_xy)
    Jp, Jl, _ = oc.dense_system(cur, **plm.weighted_all((cur.cams, cur.lms), priors, losses))
    cam_w, lm_w, kappa = cvm.dense_inverse(Jp, Jl, prob.nc, prob.nl)
    if entry == "covariance":
        cam, lm = lin.covariance()
    else:
        out = lin.covariance_blocks(marginals=True)
        cam, lm = out["cam"], out["lm"]
    bar = max(1e-9, 1e-14 * kappa)
    assert rel_err(cam, cam_w) < bar and rel_err(lm, lm_w) < bar
    # the unweighted inverse is far from it: the weights matter here
    Jp0, Jl0, _ = oc.dense_system(cur, **priors)
    assert rel_err(cam, cvm.dense_inverse(Jp0, Jl0, prob.nc, prob.nl)[0]) > 1e3 * bar
    lin.close()


@pytest.mark.parametrize("dtype", DTYPES, ids=dt_id)
def test_read_back_in_caller_order(case, dtype):
    prob, priors = case
    losses = losses_for(prob, priors, [0, 1, 2], seed=11)
    bp, lin = make(prob, dtype, priors, losses)
    bp.cams[:, 4:7] += 0.01  # a state the handle has not linearised
    lin.upload_state()
    sprob, model = rounded(BalProblemArrays(bp, prob), priors, dtype)
    tol = 1e-12 if dtype == np.float64 else 2e-4
    for k, name in enumerate(plm.KINDS):
        res, w = lin.prior_residuals(k)
        want_r = plm.whitened(k, (sprob.cams, sprob.lms), model[name])
        _, _, want_w = plm.weights(k, (sprob.cams, sprob.lms), model[name], losses[k])
        drop = plm.dropped(k, model[name])
        want_w = np.where(drop, 1.0, want_w)
        assert rel_err(res, want_r) < tol and np.max(np.abs(w - want_w)) < tol, name
        assert np.all(res[drop] == 0) and np.all(w[drop] == 1)
        if k == plm.CAMERA:
            assert np.all(res[3] == 0) and w[3] == 1  # camera 3 has an all-zero L
    lin.close()


def BalProblemArrays(bp, prob):
    from rootba_b200.synthetic import BalArrays
    return BalArrays(bp.cams.astype(np.float64), bp.lms.astype(np.float64), prob.lm_off, prob.obs_cam, prob.obs_xy)


@pytest.mark.parametrize("dtype", DTYPES, ids=dt_id)
@pytest.mark.parametrize("n", [127, 128, 129, 300])
def test_weighting_kernels_at_thread_block_edges(n, dtype):
    """n cameras with a prior each, n pairs (a ring) and n landmark priors (thread per item, 128 threads per block): every
    item's loss reaches its own rows, cost and read-back"""
    import camera_prior_model as pm
    from rootba_b200.synthetic import synth_bal
    prob = synth_bal(n, 2 * n, 3.0, seed=n)
    assert prob.nc == n and prob.nl >= n
    rng = np.random.default_rng(n)
    cams = np.asarray(prob.cams, np.float64)
    cmean = pm.mean_at(cams)
    cmean[:, 4:7] += rng.normal(0, 0.3, (n, 3))
    cL = np.stack([pm.sqrt_info_kind("dense", rng, 3.0) for _ in range(n)])
    pairs = np.stack([np.arange(n), (np.arange(n) + 1) % n], 1).astype(np.int32)
    pmean = qm.mean_at(cams, pairs)
    pmean[:, 4:7] += rng.normal(0, 0.3, (n, 3))
    pL = np.stack([np.eye(6) * 5.0 for _ in range(n)])
    idx = (np.arange(n) * (prob.nl // n)).astype(np.int32)
    lmean = np.asarray(prob.lms, np.float64)[idx] + rng.normal(0, 0.3, (n, 3))
    lL = np.stack([np.eye(3) * 5.0 for _ in range(n)])
    priors = dict(camera=(cmean, cL), pairs=(pairs, pmean, pL), landmarks=(idx, lmean, lL))
    sprob, model = rounded(prob, priors, dtype)
    state = (sprob.cams, sprob.lms)
    losses = {k: plm.losses_around(k, state, model[plm.KINDS[k]], seed=k) for k in range(3)}
    bars = oc.BARS[dtype]
    bp, lin = make(prob, dtype, priors, losses)
    e0 = lin.compute_error()["all"]["error"]
    assert abs(e0 - robust_total_cost(sprob, model, losses)) <= bars["cost"] * e0
    lin.linearize()
    lin.solve(1e-3)
    Jp, Jl, r = oc.dense_system(sprob, **plm.weighted_all(state, model, losses))
    _, _, _, _, _, H, b = oc.reduced(Jp, Jl, r, 1e-3, prob.nl, dtype)
    assert rel_err(lin.get_rhs(), b) < bars["b"]
    for k in range(3):
        res, w = lin.prior_residuals(k)
        # L e against the model; w against the model's loss on the handle's own s, which in float32 carries the rounding of
        # the centre c = -R^T t far from the origin
        assert rel_err(res, plm.whitened(k, state, model[plm.KINDS[k]])) < (1e-12 if dtype == np.float64 else bars["b"])
        want = olm.loss(losses[k][0], losses[k][1], np.sum(np.asarray(res, np.float64) ** 2, axis=1))[1]
        assert np.max(np.abs(w - want)) < (1e-12 if dtype == np.float64 else 1e-5)
    lin.close()


# ---- a pose chain with false loop closures ------------------------------------------------------------------------------
def chain_case(nc=12, seed=5):
    """synth_bal(nc) with odometry pair priors between consecutive cameras at their true relative poses, a centre prior on
    camera 0 (the gauge), and three false loop closures 30 degrees and 4 units per axis off their true relative poses"""
    from scipy.spatial.transform import Rotation
    from rootba_b200.synthetic import synth_bal
    import camera_prior_model as pm
    prob = synth_bal(nc, 150, 3.4, seed=seed)
    cams = np.asarray(prob.cams, np.float64)
    good = [(i, i + 1) for i in range(nc - 1)]
    bad = [(0, nc - 1), (2, nc - 3), (1, nc // 2)]
    pairs = np.asarray(good + bad, np.int32)
    mean = qm.mean_at(cams, pairs)
    rng = np.random.default_rng(seed)
    for p in range(len(good), len(pairs)):  # 30 degrees about a random axis; 4 units on every translation axis
        axis = rng.normal(size=3)
        mean[p, :4] = (Rotation.from_rotvec(np.radians(30) * axis / np.linalg.norm(axis)) * Rotation.from_quat(mean[p, :4])).as_quat()
        mean[p, 4:7] += rng.choice([-1, 1], 3) * 4.0
    L = np.stack([np.diag([20.0] * 3 + [100.0] * 3)] * len(pairs))
    cmean = pm.mean_at(cams)
    cL = np.zeros((nc, 9, 9))
    cL[0] = np.eye(9) * 100.0
    return prob, dict(camera=(cmean, cL), pairs=(pairs, mean, L)), len(good)


def run_lm(prob, priors, losses):
    import rootba_b200 as rb
    bp, lin = make(prob, np.float64, priors, losses, max_num_iterations=200, function_tolerance=1e-16)
    lin.lm_run(200)
    lin.download_state()
    lin.close()
    return bp.cams.copy(), bp.lms.copy()


def test_false_loop_closures_cauchy_and_tukey_recover_the_outlier_free_solution():
    prob, priors, ngood = chain_case()
    pairs = priors["pairs"]
    clean = dict(priors, pairs=tuple(a[:ngood] for a in pairs))
    ref_c, ref_l = run_lm(prob, clean, {})
    m = len(pairs[0])
    err = lambda cams: np.max(np.abs(cams[:, 4:7] - ref_c[:, 4:7]))
    none_c, _ = run_lm(prob, priors, {})
    assert err(none_c) > 1e-3  # the quadratic false closures pull the chain away
    # bars on the largest centre error against the outlier-free solution, as a share of NONE's: CAUCHY keeps a bounded pull
    # a^2 / |L e| per false closure, TUKEY none while a closure stays beyond its scale
    # TUKEY rejects whatever lies beyond its scale, so its scale must lie between the odometry pairs' largest |L e| at the
    # outlier-free solution (they disagree with the observations there) and the false closures' smallest at the start
    good = np.linalg.norm(plm.whitened(plm.PAIR, (ref_c, ref_l), clean["pairs"]), axis=1).max()
    false = np.linalg.norm(plm.whitened(plm.PAIR, (prob.cams, prob.lms), tuple(x[ngood:] for x in pairs)), axis=1).min()
    a_tukey = 2.0 * max(good, 3.55)
    assert a_tukey < 0.5 * false, (good, false)
    # measured on one H100: CAUCHY ends 0.04-0.1 and TUKEY 0.16 of NONE's error away (TUKEY reaches another stationary point
    # of its non-convex cost on this chain; why was not investigated)
    for kind, a, bar in ((olm.CAUCHY, 3.55, 0.1), (olm.TUKEY, a_tukey, 0.25)):
        got_c, _ = run_lm(prob, priors, {plm.PAIR: (np.full(m, kind, np.uint8), np.full(m, a))})
        assert err(got_c) < bar * err(none_c), (kind, a, err(got_c), err(none_c))


@pytest.mark.parametrize("kind", [olm.CAUCHY, olm.SOFT_L1], ids=["CAUCHY", "SOFT_L1"])
def test_robust_lm_ends_at_a_stationary_point_and_equals_the_host_loop(kind):
    import rootba_b200 as rb
    prob, priors, _ = chain_case()
    m = len(priors["pairs"][0])
    losses = {plm.PAIR: (np.full(m, kind, np.uint8), np.full(m, 3.55))}
    so = rb.SolverOptions(max_num_iterations=64, min_relative_decrease=0.0, function_tolerance=1e-16)
    bp = oc.bal_problem(prob, np.float64, camera_prior=priors["camera"], camera_pair_prior=priors["pairs"])
    bp.camera_pair_prior_loss = losses[plm.PAIR]
    lin = rb.LinearizorQR.create(bp, so)
    lin.lm_run(64)
    lin.download_state()
    lin.close()
    from rootba_b200.synthetic import BalArrays
    fin = BalArrays(bp.cams, bp.lms, prob.lm_off, prob.obs_cam, prob.obs_xy)
    Jp, Jl, r = oc.dense_system(fin, **plm.weighted_all((fin.cams, fin.lms), priors, losses))
    J = np.hstack([Jp, Jl])
    assert np.linalg.norm(J.T @ r) <= 1e-6 * np.linalg.norm(J, 2) * np.linalg.norm(r)
    oc.check_lm_run_equals_host_loop(prob, so, camera_prior=priors["camera"], camera_pair_prior=priors["pairs"],
                                     camera_pair_prior_loss=losses[plm.PAIR])


# ---- the problem-term protocol ------------------------------------------------------------------------------------------
def test_protocol(case):
    import rootba_b200 as rb
    from rootba_b200 import _lib
    prob, priors = case
    losses = losses_for(prob, priors, [0, 1, 2], seed=2)
    bp, lin = make(prob, np.float64, priors, {})
    L = _lib.lib()
    lin.linearize()
    lin.solve(1e-3)
    e_before = lin.compute_error()["all"]["error"]
    grown = {}
    for k, name in enumerate(plm.KINDS):
        before = lin.stats()["device_bytes"]
        lin.set_prior_loss(k, *losses[k])
        n = {plm.CAMERA: prob.nc, plm.PAIR: int((~plm.dropped(k, priors[name])).sum()),
             plm.LANDMARK: int((~plm.dropped(k, priors[name])).sum())}[k]
        nr = _lib.PRIOR_ROWS[k]
        grown[k] = (n + (n + 7) // 8) * 8 + nr * nr * n * 8  # records (scales + kinds) and sqrt(w) L
        assert lin.stats()["device_bytes"] - before == grown[k], name
        for call in (lambda: lin.solve(1e-3), lambda: lin.apply(None)):  # until the next linearize; the increment discarded
            with pytest.raises(_lib.RbaError) as e:
                call()
            assert e.value.code == -6  # RBA_ERR_STATE
        lin.linearize()
        lin.solve(1e-3)
    # the cached error was discarded: the robust cost is new
    assert lin.compute_error()["all"]["error"] != e_before
    # invalid input leaves the previous losses in force (the read-back's weights do not change)
    w0 = [lin.prior_residuals(k)[1] for k in range(3)]
    n = [prob.nc, len(priors["pairs"][0]), len(priors["landmarks"][0])]
    h = lin.h
    u8 = lambda a: np.ascontiguousarray(a, np.uint8)
    f64 = lambda a: np.ascontiguousarray(a, np.float64)
    bad = [(3, n[0], u8(np.zeros(n[0])), f64(np.ones(n[0]))), (-1, n[0], u8(np.zeros(n[0])), f64(np.ones(n[0])))]
    for k in range(3):
        bad += [(k, n[k] + 1, u8(np.zeros(n[k] + 1)), f64(np.ones(n[k] + 1))), (k, n[k], u8(np.zeros(n[k])), None),
                (k, n[k], None, f64(np.ones(n[k]))), (k, n[k], u8(np.full(n[k], 5)), f64(np.ones(n[k]))),
                (k, n[k], u8(np.full(n[k], 2)), f64(np.zeros(n[k]))), (k, n[k], u8(np.full(n[k], 4)), f64(np.full(n[k], np.inf)))]
    for which, num, kind, scale in bad:
        rc = L.rba_set_prior_loss(h, which, num, None if kind is None else kind.ctypes.data, None if scale is None else scale.ctypes.data)
        assert rc == -1, (which, num)
    lin.linearize()
    lin.solve(1e-3)  # the rejected calls changed nothing of the state protocol either
    for k in range(3):
        assert np.array_equal(lin.prior_residuals(k)[1], w0[k])
    assert L.rba_get_prior_residuals(h, 0, None, None) == -1 and L.rba_get_prior_residuals(h, 7, None, None) == -1
    # a setter of the kind clears its losses: the weights read back as 1 (and the same buffers serve the next loss)
    for k, (name, attr) in enumerate(zip(plm.KINDS, ("camera_prior", "camera_pair_prior", "landmark_prior"))):
        setattr(bp, attr, priors[name])
        assert np.all(lin.prior_residuals(k)[1] == 1)
    before = lin.stats()["device_bytes"]
    for k in range(3):
        lin.set_prior_loss(k, *losses[k])
    assert lin.stats()["device_bytes"] == before
    lin.close()


def test_example_flags(tmp_path, case):
    from rootba_b200.synthetic import write_bal
    prob, priors = case
    path = tmp_path / "p.txt"
    write_bal(prob, str(path))
    cp = tmp_path / "cam.npz"
    np.savez(cp, mean=priors["camera"][0], sqrt_info=priors["camera"][1])
    pp = tmp_path / "pairs.npz"
    np.savez(pp, pairs=priors["pairs"][0], mean=priors["pairs"][1], sqrt_info=priors["pairs"][2])
    lk = tmp_path / "lk.npz"
    m = len(priors["pairs"][0])
    np.savez(lk, kind=np.array(["CAUCHY"] * m), scale=np.full(m, 2.0))
    out = tmp_path / "res.npz"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "examples", "solve_bal.py"), str(path), "--max-num-iterations", "3",
                        "--camera-prior", str(cp), "--camera-pair-prior", str(pp), "--camera-prior-loss", "SOFT_L1:0.01",
                        "--pair-prior-loss", str(lk), "--prior-residuals", str(out)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    with np.load(out) as f:
        assert f["camera_residual"].shape == (prob.nc, 9) and f["pair_robust_weight"].shape == (m,)
        # NONE would give w = 1 everywhere: the losses of both flags reached the handle
        for kind in ("camera", "pair"):
            w = f[kind + "_robust_weight"]
            assert np.all(w <= 1) and np.min(w) < 0.9, kind
    r = subprocess.run([sys.executable, os.path.join(ROOT, "examples", "solve_bal.py"), str(path), "--pair-prior-loss", "CAUCHY"],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode != 0 and "--pair-prior-loss" in r.stderr


# ---- the C++ host -------------------------------------------------------------------------------------------------------
def test_cpp_host_forwards_the_prior_losses(tmp_path, case):
    """tests/host_prior_loss.cpp fills ProblemPriors' prior and loss fields and creates the handle through the C++
    LinearizorQR: its cost equals the Python host's with the same losses bit for bit, differs from the cost without them, and
    a loss array of the wrong length is refused"""
    prob, priors = case
    exe = str(tmp_path / "host_prior_loss")
    subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-Wall", "-pthread", "-I", os.path.join(ROOT, "rootba_b200", "host"), "-o", exe,
                    os.path.join(ROOT, "tests", "host_prior_loss.cpp"), "-L", os.path.join(ROOT, "rootba_b200"), "-lrootba_b200",
                    "-Wl,-rpath," + os.path.join(ROOT, "rootba_b200")], check=True)
    losses = losses_for(prob, priors, [0, 1, 2], seed=13)
    cm_, cL = priors["camera"]
    pairs, pm_, pL = priors["pairs"]
    lidx, lm_, lL = priors["landmarks"]
    files = dict(cams=prob.cams, lms=prob.lms, lm_off=np.asarray(prob.lm_off, np.int64), obs_cam=np.asarray(prob.obs_cam, np.int32),
                 obs_xy=prob.obs_xy, cmean=cm_, cL=cL, pairs=np.asarray(pairs, np.int32), pmean=pm_, pL=pL,
                 lidx=np.asarray(lidx, np.int32), lmean=lm_, lL=lL)
    for key, (k, a) in zip(("c", "p", "l"), (losses[0], losses[1], losses[2])):
        files[key + "k"], files[key + "s"] = np.asarray(k, np.uint8), np.nan_to_num(np.asarray(a, np.float64), nan=0.0)
    for name, a in files.items():
        arr = np.ascontiguousarray(a)
        (tmp_path / name).write_bytes((arr if arr.dtype != np.float32 else arr.astype(np.float64)).tobytes())
    args = [exe, str(tmp_path), str(prob.nc), str(prob.nl), str(len(prob.obs_cam)), str(len(pairs)), str(len(lidx))]
    r = subprocess.run(args, capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    cpp = float(r.stdout.strip())
    _, lin = make(prob, np.float64, priors, losses)
    py = lin.compute_error()["all"]["error"]
    lin.close()
    _, lin = make(prob, np.float64, priors, {})
    plain = lin.compute_error()["all"]["error"]
    lin.close()
    assert cpp == py and cpp != plain
    r = subprocess.run(args + ["short"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 3 and "camera_pair_prior_loss" in r.stdout, r.stdout + r.stderr


# ---- sharded handles ----------------------------------------------------------------------------------------------------
def raw_readback(lin, k, n):
    """rba_get_prior_residuals into NaN-filled buffers: entries the handle does not write stay NaN"""
    import ctypes as C
    from rootba_b200 import _lib
    res = np.full((n, _lib.PRIOR_ROWS[k]), np.nan, lin.dtype)
    w = np.full(n, np.nan, lin.dtype)
    _lib.check(_lib.lib().rba_get_prior_residuals(lin.h, k, C.c_void_p(res.ctypes.data), C.c_void_p(w.ctypes.data)))
    return res, w


@pytest.mark.parametrize("dtype", DTYPES, ids=dt_id)
def test_shard_maps_the_callers_landmark_losses_to_its_own_priors(dtype):
    """each rank's handle of a two-shard problem, one after the other on one GPU (the setters and the read-back need no
    communicator): landmark losses given in the caller's order over priors of both shards, zero-L ones among them, reach the
    shard's own priors -- the read-back writes exactly those, with the model's L e and w (0 and 1 for a zero L) -- and the
    losses' device memory is that of the shard's own kept priors"""
    import landmark_prior_model as lp
    import rootba_b200 as rb
    from rootba_b200 import _lib
    from rootba_b200.synthetic import synth_bal
    prob = synth_bal(20, 400, 3.5, seed=3)
    prior = lp.prior_case(prob.lms, every=5, seed=4)  # "dense", "height", "rank2", "none" in turn
    sprob, model = rounded(prob, {"landmarks": prior}, dtype)
    state = (sprob.cams, sprob.lms)
    loss = plm.losses_around(plm.LANDMARK, state, model["landmarks"], seed=6)
    want_r = plm.whitened(plm.LANDMARK, state, model["landmarks"])
    drop = plm.dropped(plm.LANDMARK, model["landmarks"])
    want_w = np.where(drop, 1.0, plm.weights(plm.LANDMARK, state, model["landmarks"], loss)[2])
    tol = 1e-12 if dtype == np.float64 else 1e-5
    seen = np.zeros(len(prior[0]), int)
    for rank in range(2):
        bp = rb.BalProblem.from_arrays(prob, dtype)
        bp.landmark_prior = prior
        lin = rb.LinearizorQR.create(bp, rb.SolverOptions(rank=rank, nranks=2))
        st = lin.stats()
        own = (prior[0] >= st["landmark_begin"]) & (prior[0] < st["landmark_end"])
        assert own.any() and (~own).any() and (own & drop).any() and (own & ~drop).any()
        before = st["device_bytes"]
        lin.set_prior_loss("landmark", *loss)
        n = int((own & ~drop).sum())  # the shard's kept priors: records (scales + kinds) and sqrt(w) L
        size = np.dtype(dtype).itemsize
        recs = 2 * n if dtype == np.float32 else n + (n + 7) // 8
        assert lin.stats()["device_bytes"] - before == (recs + 9 * n) * size
        res, w = raw_readback(lin, plm.LANDMARK, len(prior[0]))
        assert np.all(np.isnan(res[~own])) and np.all(np.isnan(w[~own]))
        assert rel_err(res[own], want_r[own]) < tol and np.max(np.abs(w[own] - want_w[own])) < tol
        assert np.all(res[own & drop] == 0) and np.all(w[own & drop] == 1)
        seen += own
        # a num that is not the caller's count is refused on every shard
        k = np.zeros(len(prior[0]) - 1, np.uint8)
        a = np.ones(len(prior[0]) - 1, dtype)
        assert _lib.lib().rba_set_prior_loss(lin.h, plm.LANDMARK, len(k), k.ctypes.data, a.ctypes.data) == -1
        lin.close()
    assert np.all(seen == 1)


@pytest.mark.parametrize("sfx", ["f32", "f64"])
def test_two_ranks_with_prior_losses(tmp_path, sfx):
    res = oc.run_two_ranks(tmp_path, "multirank_prior_loss_worker.py", sfx, "1", 31900, 53 + (37 if sfx == "f32" else 0))
    tols = 1e-4 if sfx == "f32" else 1e-8
    assert res["replicas_identical"] and res["landmark_readback_covers_own_shard_only"], res
    assert res["landmark_readback_model"] < (1e-4 if sfx == "f32" else 1e-12), res
    assert res["b"] < 4 * tols and res["inc"] < tols and res["l_diff"] < 20 * tols, res
    assert res["lms"] < 10 * tols and res["cams"] < tols and res["cost"] < tols and res["cost0"] < tols, res
    assert res["camera_readback"] < tols and res["pair_readback"] < tols and res["landmark_readback"] < tols, res
