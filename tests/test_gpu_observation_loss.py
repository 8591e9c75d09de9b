"""Robust losses per observation (rba_set_observation_loss, DESIGN.md section 21) on the GPU: every solver configuration against
the dense float64 model of the weighted problem (tests/observation_loss_model.py) in both precisions, mixed kinds, with
observation information, held cameras, every prior kind and intrinsics groups; the unmodified path and the flagged kernels bit
for bit; every track-length class landmark by landmark with Tukey-rejected observations; the read-back; covariances; LM runs
to the robust minimum and against scipy; the protocol; the example; two ranks."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import camera_model as cm
import objective_checks as oc
import observation_info_model as om
import observation_loss_model as lm
from conftest import ROOT, rel_err
from objective_checks import BARS, CONFIGS, cfg_id, fixed_entries, reduced

pytestmark = pytest.mark.gpu

DTYPES = [np.float32, np.float64]
PCG_CONFIGS = [c for c in CONFIGS if c["solver_type"] != "POWER_SCHUR_COMPLEMENT"]


def _rounded(a, dtype):
    return np.asarray(np.asarray(a, dtype), np.float64)


class loss_checks:
    """While active, the shared dense-objective checks of `module` run on the robustly weighted problem: the model's
    reprojection rows and cost are those of observation_loss_model with the scales and W rounded to the handle's scalar type,
    and every BalProblem they make carries the losses (and W)."""

    def __init__(self, module, kind, scale, dtype, W=None):
        self.module, self.kind, self.scale, self.dtype, self.W = module, kind, scale, dtype, W
        self.m = pytest.MonkeyPatch()

    def __enter__(self):
        kind, a, dtype = self.kind, _rounded(self.scale, self.dtype), self.dtype
        Wd = None if self.W is None else _rounded(self.W, dtype)
        dense, total, make = oc.dense_system, oc.total_cost, oc.bal_problem

        def dense_system(prob, **model):
            Jp, Jl, r = dense(prob, **model)
            Jw, Lw, rw = lm.dense_system(prob, kind, a, Wd, dtype=dtype)
            n = len(rw)
            Jp[:n], Jl[:n], r[:n] = Jw, Lw, rw  # the reprojection rows come first
            return Jp, Jl, r

        def total_cost(prob, **model):
            return total(prob, **model) - float(cm.compute_error(prob)["all"]["error"]) + lm.cost(prob, kind, a, Wd)

        def bal_problem(arrays, dt, **features):
            bp = make(arrays, dt, **features)
            bp.observation_loss = (self.kind, self.scale)
            if self.W is not None:
                bp.observation_sqrt_info = self.W
            return bp
        for name, fn in (("dense_system", dense_system), ("total_cost", total_cost), ("bal_problem", bal_problem)):
            self.m.setattr(self.module, name, fn)
        return self

    def __exit__(self, *exc):
        self.m.undo()


def check_loss_step(cfg, prob, kind, scale, dtype, W=None, **kw):
    with loss_checks(oc, kind, scale, dtype, W):
        oc.check_against_dense(cfg, prob, dtype=dtype, inc_eta_kappa=True, **kw)


@pytest.fixture(scope="module")
def case7():
    from rootba_b200.synthetic import synth_bal
    prob = synth_bal(7, 90, 3.6, seed=21)
    kind, scale = lm.mixed(prob.nobs, seed=5, lo=1.0, hi=4.0)
    return prob, kind, scale


# ---- every solver configuration against the dense model -----------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
@pytest.mark.parametrize("cfg", CONFIGS, ids=cfg_id)
def test_against_dense_system(cfg, dtype, case7):
    prob, kind, scale = case7
    w = lm.rows(prob, kind, scale)["w"]
    assert (w < 1).mean() > 0.2 and (w == 0).sum() > 0  # every kind active, Tukey rejecting some
    check_loss_step(cfg, prob, kind, scale, dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
@pytest.mark.parametrize("cfg", CONFIGS[:2], ids=cfg_id)
def test_with_switched_off_and_rank_one_information(cfg, dtype, case7):
    prob, kind, scale = case7
    W = om.random_info(prob.nobs, seed=3)
    W[::9] = 0.0
    W[4::9, 1] = 0.0
    check_loss_step(cfg, prob, kind, scale, dtype, W=W)


@pytest.mark.parametrize("cfg", PCG_CONFIGS[:4], ids=cfg_id)
def test_with_held_cameras_and_every_prior_kind(cfg):
    import camera_prior_model as pm
    import landmark_prior_model as lp
    import pair_prior_model as qm
    prob, mean_c, L_c = pm.prior_case(7, 90)
    mask = np.zeros(prob.nc, np.uint8)
    mask[2] = 15
    mask[4] = 14
    pairs = np.array([(0, 1), (3, 1), (5, 6)], np.int32)
    rng = np.random.default_rng(11)
    pmean = qm.mean_at(prob.cams, pairs)
    pmean[:, 4:7] += rng.normal(0, 0.05, (len(pairs), 3))
    pL = np.stack([qm.sqrt_info_kind(k, rng) for k in ("dense", "translation", "rotation")])
    kind, scale = lm.mixed(prob.nobs, seed=12, lo=0.5, hi=2.0)
    check_loss_step(cfg, prob, kind, scale, np.float64, W=om.random_info(prob.nobs, seed=5), camera=(mean_c, L_c),
                    pairs=(pairs, pmean, pL), landmarks=lp.prior_case(prob.lms, every=2, seed=8), mask=mask)


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
@pytest.mark.parametrize("cfg", [PCG_CONFIGS[i] for i in (0, 4)], ids=cfg_id)
def test_with_intrinsics_groups(cfg, dtype):
    import test_gpu_shared_intrinsics as ts
    from test_shared_intrinsics_model import GROUP, _case
    prob, _, model = _case(("camera",))
    kind, scale = lm.mixed(prob.nobs, seed=6, lo=0.5, hi=2.0)
    with loss_checks(ts, kind, scale, dtype):
        ts.check_tied_step(cfg, prob, GROUP, model, dtype)


# ---- the unmodified path and the flagged kernels, bit for bit ------------------------------------------------------------
def _steps(prob, dtype, opts):
    """three LM steps of a handle without a loss (oc.lm_steps)"""
    return oc.lm_steps(prob, dtype, opts, "never")


def _steps_with(prob, dtype, opts, setter, steps):
    """oc.lm_steps with `setter(lin)` applied before the first step"""
    import rootba_b200 as rb
    bp = rb.BalProblem.from_arrays(prob, dtype)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(**opts))
    setter(lin)
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


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
@pytest.mark.parametrize("qr", [True, False], ids=["householder", "givens"])
def test_the_handles_own_choice_is_the_unmodified_path(small_problem, dtype, qr):
    import rootba_b200 as rb
    n = small_problem.nobs
    huber = dict(use_householder_marginalization=qr, residual=rb.ResidualOptions(robust_norm="HUBER", huber_parameter=1.5))
    plain = dict(use_householder_marginalization=qr)
    ref_h = _steps(small_problem, dtype, huber)
    ref_n = _steps(small_problem, dtype, plain)
    oc.assert_identical_steps(ref_h, _steps_with(small_problem, dtype, huber, lambda l: l.set_observation_loss("HUBER", 1.5), 3),
                              "(HUBER, huber_parameter) everywhere")
    oc.assert_identical_steps(ref_n, _steps_with(small_problem, dtype, plain, lambda l: l.set_observation_loss("NONE", np.nan), 3),
                              "NONE everywhere with robust_norm NONE")
    kind, scale = lm.mixed(n, seed=1)

    def set_then_null(l):
        l.set_observation_loss(kind, scale)
        l.set_observation_loss(None)
    oc.assert_identical_steps(ref_n, _steps_with(small_problem, dtype, plain, set_then_null, 3), "NULL after a non-default loss")


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
@pytest.mark.parametrize("qr", [True, False], ids=["householder", "givens"])
def test_the_flagged_kernels_coincide_with_the_unflagged_ones(small_problem, dtype, qr):
    """(HUBER, a) everywhere but one observation that stays an inlier, given (HUBER, 2a): the OBSL instances run and give the
    unflagged handle's LM run bit for bit (w = 1 for that observation either way; the others use error_weight's arithmetic)"""
    import rootba_b200 as rb
    a = 1.5
    opts = dict(use_householder_marginalization=qr, residual=rb.ResidualOptions(robust_norm="HUBER", huber_parameter=a))
    lin = rb.LinearizorQR.create(rb.BalProblem.from_arrays(small_problem, dtype), rb.SolverOptions(**opts))
    res, hw, _ = lin.observation_residuals()
    lin.close()
    s = (np.asarray(res, np.float64) ** 2).sum(1)
    assert 0.05 < (hw < 1).mean() < 0.95
    o = int(np.argmin(s))
    assert s[o] < 0.01 * a * a  # stays below a over the three steps
    scale = np.full(small_problem.nobs, a)
    scale[o] = 2 * a
    stats = {}

    def setter(l):
        l.set_observation_loss("HUBER", scale)
        stats["bytes"] = l.stats()["device_bytes"]
    got = _steps_with(small_problem, dtype, opts, setter, 3)
    oc.assert_identical_steps(_steps(small_problem, dtype, opts), got, "flagged kernels at coinciding values")


# ---- every track-length class, landmark by landmark ---------------------------------------------------------------------
def _class_ns():
    from test_gpu_kernel_classes import CASES, _signature
    return [n for n in CASES if n <= 150 and (n == 2 or _signature(n) != _signature(n - 1))] + [150]


@pytest.mark.parametrize("qr", ["householder", "givens"])
@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
@pytest.mark.parametrize("n", sorted(set(_class_ns())))
def test_every_track_length_class_landmark_by_landmark(n, dtype, qr):
    """B^T B of each landmark's stored block against A^T A of the model's rows (with the damping rows), mixed kinds with
    Tukey-rejected observations first, in the middle and last in a track (landmark l mod 3), and landmark 1 rejected whole"""
    import rootba_b200 as rb
    from rootba_b200.synthetic import BalArrays
    from test_gpu_kernel_classes import problem
    prob = problem(n)
    f = lambda a: _rounded(a, dtype)
    sprob = BalArrays(f(prob.cams), f(prob.lms), prob.lm_off, prob.obs_cam, f(prob.obs_xy))
    lam, eps = 0.1, float(cm.EPS_SQRT[np.dtype(dtype)])
    tol = 1e-10 if dtype == np.float64 else 2e-4
    kind, scale = lm.mixed(prob.nobs, seed=n, kinds=(lm.NONE, lm.HUBER, lm.CAUCHY, lm.SOFT_L1), lo=0.5, hi=3.0)
    tiny = 1e-6  # Tukey at this scale rejects every observation with |W r| >= 1e-6
    for l in range(prob.nl):
        o = prob.lm_off[l] + (0, n // 2, n - 1)[l % 3]
        kind[o], scale[o] = lm.TUKEY, tiny
    kind[prob.lm_off[1]:prob.lm_off[2]], scale[prob.lm_off[1]:prob.lm_off[2]] = lm.TUKEY, tiny
    bp = rb.BalProblem.from_arrays(prob, dtype)
    bp.observation_loss = (kind, scale)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(use_householder_marginalization=(qr == "householder")))
    lin.linearize()
    lin.solve(lam)
    w = lm.rows(sprob, kind, f(scale), dtype=dtype)
    assert np.all(w["w"][prob.lm_off[1]:prob.lm_off[2]] == 0)
    s, _ = lin.get_jacobian_scaling()
    Jp, Jl, r = lm.dense_system(sprob, kind, f(scale), dtype=dtype)
    D, _, _, _, _, _, b = reduced(Jp, Jl, r, lam, prob.nl, dtype)
    assert rel_err(s, D) < BARS[dtype]["scaling"]
    assert rel_err(lin.get_rhs(), b) < BARS[dtype]["b"]
    sd = np.asarray(s, np.float64).reshape(-1, 9)
    for l in range(prob.nl):
        o0, o1 = int(prob.lm_off[l]), int(prob.lm_off[l + 1])
        B, lm_idx, res_idx, jls = lin.debug_get_block(l)
        B, jls = np.asarray(B, np.float64), np.asarray(jls, np.float64)
        want_jls = 1.0 / (eps + np.sqrt((w["Jl"][o0:o1] ** 2).sum((0, 1))))
        assert rel_err(jls, want_jls) < tol, (l, jls, want_jls)
        A = np.zeros((2 * n + 3, B.shape[1]))
        for i in range(n):
            A[2 * i:2 * i + 2, 9 * i:9 * i + 9] = w["Jp"][o0 + i] * sd[prob.obs_cam[o0 + i]]
        A[:2 * n, lm_idx:lm_idx + 3] = w["Jl"][o0:o1].reshape(2 * n, 3) * want_jls
        A[:2 * n, res_idx] = w["r"][o0:o1].ravel()
        A[2 * n:, lm_idx:lm_idx + 3] = np.sqrt(lam) * np.eye(3)
        cols = [c for c in range(B.shape[1]) if c != res_idx]
        G, Gw = B[:, cols].T @ B[:, cols], A[:, cols].T @ A[:, cols]
        assert rel_err(G, Gw) < tol, l
        g, gw = B[:, lm_idx:lm_idx + 3].T @ B[:, res_idx], A[:, lm_idx:lm_idx + 3].T @ A[:, res_idx]
        assert np.max(np.abs(g - gw)) <= tol * (1 + np.max(np.abs(gw))), l
    lin.close()


# ---- the read-back ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
def test_robust_weight_read_back(small_problem, dtype):
    """mixed kinds on mixed tracks, a camera turned around (invalid projections) and switched-off observations: each
    observation's own w against the model; the flags are those of section 19"""
    import rootba_b200 as rb
    from rootba_b200.synthetic import BalArrays, turn_cameras_around
    prob = turn_cameras_around(small_problem, [3])
    W = om.random_info(prob.nobs, seed=12)
    W[::11] = 0.0
    kind, scale = lm.mixed(prob.nobs, seed=13)
    f = lambda a: _rounded(a, dtype)
    sprob = BalArrays(f(prob.cams), f(prob.lms), prob.lm_off, prob.obs_cam, f(prob.obs_xy))
    w = lm.rows(sprob, kind, f(scale), f(W), dtype=dtype)
    bp = rb.BalProblem.from_arrays(prob, dtype)
    bp.observation_sqrt_info = W
    bp.observation_loss = (kind, scale)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(residual=rb.ResidualOptions(robust_norm="HUBER", huber_parameter=0.7)))
    res, hw, flags = lin.observation_residuals()
    lin.close()
    sq = np.sqrt(w["s"])
    far = np.abs(sq - f(scale)) > 1e-3 * np.maximum(1, f(scale))  # away from the kinks of Huber and Tukey
    far |= kind == lm.NONE
    # a float32 residual carries ~1e-4 of absolute rounding (it is the difference of ~1000-pixel coordinates), which moves w by
    # up to ~1e-3 near Tukey's scale
    assert np.allclose(hw[far], w["w"][far], rtol=1e-9 if dtype == np.float64 else 1e-2, atol=1e-12 if dtype == np.float64 else 2e-3)
    for k in (lm.NONE, lm.HUBER, lm.CAUCHY, lm.SOFT_L1, lm.TUKEY):
        assert (kind[w["on"]] == k).sum() > 10
    assert np.all(hw[kind == lm.NONE] == 1) and (hw[kind == lm.TUKEY] == 0).sum() > 0
    assert np.array_equal(flags, w["valid"].astype(np.uint8) | (w["on"].astype(np.uint8) << 1))


# ---- the cost and its counts --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
def test_compute_error_counts_tukey_rejections_as_valid(small_problem, dtype):
    import rootba_b200 as rb
    from rootba_b200.synthetic import BalArrays
    kind, scale = lm.mixed(small_problem.nobs, seed=14)
    W = np.ones(small_problem.nobs)
    W[::13] = 0.0
    f = lambda a: _rounded(a, dtype)
    sprob = BalArrays(f(small_problem.cams), f(small_problem.lms), small_problem.lm_off, small_problem.obs_cam, f(small_problem.obs_xy))
    want = lm.residual_info(sprob, kind, f(scale), W, dtype=dtype)
    bp = rb.BalProblem.from_arrays(small_problem, dtype)
    bp.observation_loss = (kind, scale)
    bp.observation_sqrt_info = W
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions())
    got = lin.compute_error()
    lin.close()
    bar = 1e-10 if dtype == np.float64 else 1e-5
    for key in ("all", "valid"):
        assert got[key]["num_obs"] == want[key]["num_obs"]
        assert abs(got[key]["error"] - want[key]["error"]) <= bar * want[key]["error"]
        assert abs(got[key]["residual_sum"] - want[key]["residual_sum"]) <= bar * want[key]["residual_sum"]


# ---- covariances ---------------------------------------------------------------------------------------------------------
def test_covariances_use_each_observations_weight(case7):
    import rootba_b200 as rb
    from test_gpu_landmark_priors import _dense_covariance_check
    prob, kind, scale = case7
    kind = kind.copy()
    kind[kind == lm.TUKEY] = lm.CAUCHY  # every landmark keeps rank 3
    mask = np.zeros(prob.nc, np.uint8)
    mask[[0, 3]] = 15
    bp = rb.BalProblem.from_arrays(prob, np.float64)
    bp.camera_fixed = mask
    bp.observation_loss = (kind, scale)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions())
    cam, lmc = lin.covariance()
    blocks = lin.covariance_blocks(marginals=True)
    lin.close()
    Jp, Jl, _ = lm.dense_system(prob, kind, scale)
    _dense_covariance_check(cam, lmc, Jp, Jl, fixed_entries(mask))
    assert np.array_equal(blocks["cam"], cam) and np.array_equal(blocks["lm"], lmc)


# ---- outliers end to end ------------------------------------------------------------------------------------------------
def _outlier_problem(frac, seed, truth=False):
    """keypoint noise sigma = 1 with a fraction `frac` of gross outliers of 20 to 100 sigma; cameras 0 and 6 held at their
    true poses (the gauge).  truth: also the true cameras (the same draw without noise and without the perturbed start)"""
    from rootba_b200.synthetic import BalArrays, synth_bal
    rng = np.random.default_rng(seed)
    kw = dict(seed=41, track_lengths=rng.integers(8, 12, 60), lm_spread=0.5)
    prob = synth_bal(12, 60, 0.0, obs_noise=1.0, **kw)
    true = synth_bal(12, 60, 0.0, obs_noise=0.0, perturb_lm=0.0, perturb_rot=0.0, perturb_trans=0.0, **kw)
    planted = rng.random(prob.nobs) < frac
    ang = rng.uniform(0, 2 * np.pi, prob.nobs)
    mag = rng.uniform(20, 100, prob.nobs)
    xy = prob.obs_xy + np.where(planted[:, None], mag[:, None] * np.stack([np.cos(ang), np.sin(ang)], 1), 0.0)
    mask = np.zeros(prob.nc, np.uint8)
    mask[[0, 6]] = 15
    cams = np.asarray(prob.cams, np.float64).copy()
    cams[[0, 6]] = true.cams[[0, 6]]
    out = BalArrays(cams, prob.lms, prob.lm_off, prob.obs_cam, xy), mask
    return out + (np.asarray(true.cams, np.float64),) if truth else out


def _robust_run(prob, mask, kind, a):
    import rootba_b200 as rb
    bp = rb.BalProblem.from_arrays(prob, np.float64)
    bp.camera_fixed = mask
    bp.observation_loss = (kind, a)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(max_num_iterations=100, function_tolerance=1e-15, eta=1e-10))
    lin.lm_run(300)
    lin.download_state()
    cost = lin.compute_error()["all"]["error"]
    lin.close()
    return bp, cost


@pytest.mark.parametrize("name", ["CAUCHY", "SOFT_L1"])
def test_lm_run_reaches_scipys_robust_minimum(name):
    """scipy least_squares(loss=..., f_scale=a) on the 1-D residual |r| per observation has the same cost as the 2-D norm
    loss only for one residual per observation, so scipy minimises sum a^2 rho(|r|^2 / a^2) / 2 with the residual
    f_o = |r_o| here (its Jacobian by finite differences); held cameras fix the gauge"""
    from scipy.optimize import least_squares
    from rootba_b200.synthetic import BalArrays
    prob, mask = _outlier_problem(0.1, 3)
    a = 2.0
    bp, cost = _robust_run(prob, mask, name, a)
    free = np.flatnonzero(mask == 0)
    x0 = np.concatenate([np.asarray(prob.cams, np.float64)[free].ravel(), np.asarray(prob.lms, np.float64).ravel()])

    def unpack(x):
        cams = np.asarray(prob.cams, np.float64).copy()
        cams[free] = x[:10 * len(free)].reshape(-1, 10)
        cams[:, :4] /= np.linalg.norm(cams[:, :4], axis=1, keepdims=True)
        return BalArrays(cams, x[10 * len(free):].reshape(-1, 3), prob.lm_off, prob.obs_cam, prob.obs_xy)

    def fun(x):
        res = cm.linearize(*cm.observations(unpack(x)))["res"]
        return np.sqrt((res ** 2).sum(1) + 1e-300)
    xs = np.concatenate([bp.cams[free].ravel(), bp.lms.ravel()])
    ls = least_squares(fun, xs, loss=name.lower(), f_scale=a, x_scale="jac", ftol=1e-15, xtol=1e-15, gtol=1e-15, max_nfev=200)
    assert ls.cost <= cost * (1 + 1e-9)  # scipy started at the handle's result
    assert abs(cost - ls.cost) <= 1e-8 * ls.cost, (cost, ls.cost)
    want = unpack(ls.x)
    assert np.max(np.abs(bp.lms - want.lms)) < 1e-4 * max(1.0, np.max(np.abs(want.lms)))


def test_lm_run_with_tukey_reaches_a_stationary_point_of_the_robust_cost():
    """the robust gradient sum w J^T W r of the model at the result is below 1e-5 of its value at the start"""
    import rootba_b200 as rb
    prob, mask = _outlier_problem(0.1, 4)
    bp, _ = _robust_run(prob, mask, "TUKEY", 5.0)
    from rootba_b200.synthetic import BalArrays
    fixed = fixed_entries(mask)

    def grad(arrays):
        Jp, Jl, r = lm.dense_system(arrays, lm.TUKEY, 5.0)
        return np.concatenate([(Jp.T @ r)[~fixed], Jl.T @ r])
    g0 = grad(prob)
    g1 = grad(BalArrays(bp.cams, bp.lms, prob.lm_off, prob.obs_cam, prob.obs_xy))
    assert np.linalg.norm(g1) < 1e-5 * np.linalg.norm(g0), (np.linalg.norm(g1), np.linalg.norm(g0))


def test_lm_run_equals_host_loop_with_a_loss():
    import rootba_b200 as rb
    prob, mask = _outlier_problem(0.1, 5)
    kind, scale = lm.mixed(prob.nobs, seed=15, lo=2.0, hi=6.0)
    oc.check_lm_run_equals_host_loop(prob, rb.SolverOptions(max_num_iterations=8), camera_fixed=mask, observation_loss=(kind, scale))


@pytest.mark.parametrize("frac", [0.05, 0.2])
def test_robust_losses_recover_the_cameras(frac):
    """camera-centre RMS error against the ground truth after rba_lm_run with each loss (the table of DESIGN.md section 21):
    every robust loss beats NONE by a wide margin"""
    prob, mask, truth = _outlier_problem(frac, 6, truth=True)

    def centres(cams):
        from scipy.spatial.transform import Rotation
        return -Rotation.from_quat(cams[:, :4]).inv().apply(cams[:, 4:7])
    rms = {}
    for name in ("NONE", "HUBER", "CAUCHY", "SOFT_L1", "TUKEY"):
        bp, _ = _robust_run(prob, mask, name, 3.0)
        rms[name] = float(np.sqrt(np.mean(np.sum((centres(bp.cams) - centres(truth)) ** 2, 1))))
    print("camera-centre RMS", frac, rms)
    assert all(rms[k] < rms["NONE"] for k in ("CAUCHY", "TUKEY"))


# ---- the protocol --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
def test_protocol_and_bad_input(small_problem, dtype):
    import rootba_b200 as rb
    from rootba_b200 import _lib
    lib = _lib.lib()
    kind, scale = lm.mixed(small_problem.nobs, seed=4)
    scale = np.asarray(scale, dtype)
    bp = rb.BalProblem.from_arrays(small_problem, dtype)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions())
    bytes0 = lin.stats()["device_bytes"]
    lin.set_observation_loss("NONE", 1.0)  # the handle's own choice: nothing allocated
    assert lin.stats()["device_bytes"] == bytes0
    lin.set_observation_loss(kind, scale)
    grown = lin.stats()["device_bytes"] - bytes0
    assert grown >= small_problem.nobs * (8 if dtype == np.float32 else 9)
    lin.compute_error()
    lin.linearize()
    inc_ref = lin.solve(1e-4)
    k, p = C.c_void_p(kind.ctypes.data), lambda a: C.c_void_p(a.ctypes.data)
    for bad_kind, bad_scale in [(5, 1.0), (lm.CAUCHY, 0.0), (lm.CAUCHY, -1.0), (lm.TUKEY, np.nan), (lm.HUBER, np.inf)]:
        kk, ss = kind.copy(), scale.copy()
        kk[17], ss[17] = bad_kind, bad_scale
        assert lib.rba_set_observation_loss(lin.h, p(kk), p(ss)) == -1
        assert lib.rba_last_error()
    assert lib.rba_set_observation_loss(lin.h, k, None) == -1 and lib.rba_set_observation_loss(lin.h, None, p(scale)) == -1
    assert np.array_equal(lin.solve(1e-4), inc_ref)  # nothing changed, still linearised
    lin.set_observation_loss(kind, scale)  # a change needs a new linearisation
    for call in (lambda: lin.solve(1e-4), lambda: lin.apply(None)):
        with pytest.raises(rb.RbaError) as e:
            call()
        assert e.value.code == -6  # RBA_ERR_STATE
    lin.linearize()
    assert np.array_equal(lin.solve(1e-4), inc_ref)  # the same losses: the same step
    assert lin.stats()["device_bytes"] - bytes0 == grown  # refilled in place
    lin.close()


# ---- the example ---------------------------------------------------------------------------------------------------------
def test_example_takes_observation_loss(tmp_path, small_problem):
    from rootba_b200.synthetic import write_bal
    path = tmp_path / "problem.txt"
    write_bal(small_problem, str(path))
    cmd = [sys.executable, os.path.join(ROOT, "examples", "solve_bal.py"), str(path), "--max-num-iterations", "3",
           "--log-path", str(tmp_path / "log.json"), "--residuals", str(tmp_path / "res.npz")]
    r = subprocess.run(cmd + ["--observation-loss", "TUKEY:0.5"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    with np.load(tmp_path / "res.npz") as f:
        hw = f["robust_weight"]
        assert hw.shape == (small_problem.nobs,) and (hw == 0).sum() > 0 and np.all(hw <= 1)
    kind, scale = lm.mixed(small_problem.nobs, seed=2)
    np.savez(tmp_path / "loss.npz", kind=kind, scale=scale)
    r = subprocess.run(cmd + ["--observation-loss", str(tmp_path / "loss.npz")], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    np.savez(tmp_path / "short.npz", kind=kind[:-1], scale=scale[:-1])
    r = subprocess.run(cmd + ["--observation-loss", str(tmp_path / "short.npz")], capture_output=True, text=True, timeout=300)
    assert r.returncode != 0 and "observation-loss" in r.stderr
    r = subprocess.run(cmd + ["--observation-loss", "CAUCHY:0"], capture_output=True, text=True, timeout=300)
    assert r.returncode != 0 and "observation-loss" in r.stderr


# ---- two GPUs ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sfx", ["f32", "f64"])
def test_two_ranks_with_observation_loss(tmp_path, sfx):
    res = oc.run_two_ranks(tmp_path, "multirank_observation_loss_worker.py", sfx, "1", 31700, 41 + (37 if sfx == "f32" else 0))
    tols = 1e-4 if sfx == "f32" else 1e-8
    assert res["replicas_identical"] and res["readback_covers_own_shard_only"], res
    assert res["b"] < 4 * tols and res["inc"] < tols and res["l_diff"] < 20 * tols, res
    assert res["lms"] < 10 * tols and res["cams"] < tols and res["cost"] < tols and res["cost0"] < tols, res
    assert res["residuals"] < tols, res
