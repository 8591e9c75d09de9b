"""Per-observation square-root information and the residual read-back (rba_set_observation_info,
rba_get_observation_residuals, DESIGN.md section 19) on the GPU: every solver configuration against the dense float64 model of
the whitened problem (tests/observation_info_model.py) in both precisions, with Huber, held cameras, every prior kind and
intrinsics groups; every track-length class landmark by landmark with switched-off observations; switched off = removed;
identity and NULL bit-identical to a handle without information; a switched-off observation that does not project; the
read-back in problem order; the outlier loop the feature exists for; covariances; the protocol; the example; two ranks."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import camera_model as cm
import objective_checks as oc
import observation_info_model as om
from conftest import ROOT, rel_err
from objective_checks import BARS, CONFIGS, cfg_id, fixed_entries, reduced

pytestmark = pytest.mark.gpu

DTYPES = [np.float32, np.float64]
PCG_CONFIGS = [c for c in CONFIGS if c["solver_type"] != "POWER_SCHUR_COMPLEMENT"]


def _rounded(a, dtype):
    return np.asarray(np.asarray(a, dtype), np.float64)


def _options(threshold=None, **kw):
    import rootba_b200 as rb
    if threshold is not None:
        kw["residual"] = rb.ResidualOptions(robust_norm="HUBER", huber_parameter=threshold)
    return kw


class whitened_checks:
    """While active, the shared dense-objective checks of `module` (objective_checks.check_against_dense,
    test_gpu_shared_intrinsics.check_tied_step) run on the whitened problem: the model's reprojection rows and cost are
    those of observation_info_model with W rounded to the handle's scalar type, and every BalProblem they make carries W."""

    def __init__(self, module, W, dtype, threshold):
        self.module, self.W, self.dtype, self.threshold = module, W, dtype, threshold
        self.m = pytest.MonkeyPatch()

    def __enter__(self):
        Wd, thr, dtype = _rounded(self.W, self.dtype), self.threshold, self.dtype
        dense, total, make = oc.dense_system, oc.total_cost, oc.bal_problem

        def dense_system(prob, **model):
            Jp, Jl, r = dense(prob, **model)
            Jw, Lw, rw = om.dense_system(prob, Wd, dtype=dtype, threshold=thr)
            n = len(rw)
            Jp[:n], Jl[:n], r[:n] = Jw, Lw, rw  # the reprojection rows come first
            return Jp, Jl, r

        def total_cost(prob, **model):
            return total(prob, **model) - float(cm.compute_error(prob)["all"]["error"]) + om.cost(prob, Wd, thr)

        def bal_problem(arrays, dt, **features):
            bp = make(arrays, dt, **features)
            bp.observation_sqrt_info = self.W
            return bp
        for name, fn in (("dense_system", dense_system), ("total_cost", total_cost), ("bal_problem", bal_problem)):
            self.m.setattr(self.module, name, fn)
        return self

    def __exit__(self, *exc):
        self.m.undo()


def check_whitened_step(cfg, prob, W, dtype, threshold=None, **kw):
    with whitened_checks(oc, W, dtype, threshold):
        oc.check_against_dense(_options(threshold, **cfg), prob, dtype=dtype, inc_eta_kappa=True, **kw)


@pytest.fixture(scope="module")
def case7():
    from rootba_b200.synthetic import synth_bal
    prob = synth_bal(7, 90, 3.6, seed=21)
    return prob, om.random_info(prob.nobs, seed=3)


# ---- every solver configuration against the dense model -----------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
@pytest.mark.parametrize("cfg", CONFIGS, ids=cfg_id)
def test_against_dense_system(cfg, dtype, case7):
    check_whitened_step(cfg, *case7, dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
@pytest.mark.parametrize("cfg", CONFIGS, ids=cfg_id)
def test_against_dense_system_with_huber(cfg, dtype, case7):
    prob, W = case7
    hw = om.whitened(prob, W, threshold=1.0)["hw"]
    assert 0.1 < (hw < 1).mean() < 0.9  # the Huber weight is active on part of the observations, at |W r|, not |r|
    check_whitened_step(cfg, prob, W, dtype, threshold=1.0)


@pytest.mark.parametrize("cfg", [dict(c, stage2_form=f) for c in CONFIGS[:2] for f in ("PANEL", "IDENTITY")], ids=cfg_id)
def test_both_stage2_forms_with_switched_off_and_rank_one_information(cfg, case7):
    prob, W = case7
    W = W.copy()
    W[::9] = 0.0
    W[4::9, 1] = 0.0  # rank 1: a constraint along one image direction
    check_whitened_step(cfg, prob, W, np.float64)


@pytest.mark.parametrize("cfg", PCG_CONFIGS, ids=cfg_id)
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
    check_whitened_step(cfg, prob, om.random_info(prob.nobs, seed=5), np.float64, camera=(mean_c, L_c), pairs=(pairs, pmean, pL),
                        landmarks=lp.prior_case(prob.lms, every=2, seed=8), mask=mask)


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
@pytest.mark.parametrize("cfg", [PCG_CONFIGS[i] for i in (0, 3, 4, 8)], ids=cfg_id)
def test_with_intrinsics_groups(cfg, dtype):
    import test_gpu_shared_intrinsics as ts
    from test_shared_intrinsics_model import GROUP, _case
    prob, _, model = _case(("camera",))
    with whitened_checks(ts, om.random_info(prob.nobs, seed=6), dtype, None):
        ts.check_tied_step(cfg, prob, GROUP, model, dtype)


# ---- every track-length class, landmark by landmark ---------------------------------------------------------------------
def _class_ns():
    from test_gpu_kernel_classes import CASES, _signature
    return [n for n in CASES if n <= 150 and (n == 2 or _signature(n) != _signature(n - 1))] + [150]


def _off_patterns(prob, n):
    """two sets of switched-off observations: (a) landmark l loses its first, a middle or its last observation (l mod 3);
    (b) landmark 0 keeps one observation, landmark 1 none"""
    a, b = np.zeros(prob.nobs, bool), np.zeros(prob.nobs, bool)
    for l in range(prob.nl):
        a[prob.lm_off[l] + (0, n // 2, n - 1)[l % 3]] = True
    b[prob.lm_off[0]:prob.lm_off[1]] = True
    b[prob.lm_off[0] + n // 2] = False
    b[prob.lm_off[1]:prob.lm_off[2]] = True
    return a, b


@pytest.mark.parametrize("qr", ["householder", "givens"])
@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
@pytest.mark.parametrize("n", sorted(set(_class_ns())))
def test_every_track_length_class_landmark_by_landmark(n, dtype, qr):
    """W + 1 landmarks of track length n (one full tile, one ragged tile).  A landmark's stored block B = Q^T [Jp | Jl | r] with
    the damping rows is fixed up to the orthogonal Q, so B^T B is compared with A^T A, A the float64 whitened, scaled rows
    and [0 | sqrt(lambda) I | 0]; jls, the pose scaling and b separately"""
    import rootba_b200 as rb
    from test_gpu_kernel_classes import problem
    prob = problem(n)
    f = lambda a: _rounded(a, dtype)
    from rootba_b200.synthetic import BalArrays
    sprob = BalArrays(f(prob.cams), f(prob.lms), prob.lm_off, prob.obs_cam, f(prob.obs_xy))
    lam, eps = 0.1, float(cm.EPS_SQRT[np.dtype(dtype)])
    tol = 1e-10 if dtype == np.float64 else 2e-4
    bp = rb.BalProblem.from_arrays(prob, dtype)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(use_householder_marginalization=(qr == "householder")))
    W0 = om.random_info(prob.nobs, seed=n)
    for off in _off_patterns(prob, n):
        W = W0.copy()
        W[off] = 0.0
        lin.set_observation_info(W)
        lin.linearize()
        lin.solve(lam)
        w = om.whitened(sprob, f(W), dtype=dtype)
        s, _ = lin.get_jacobian_scaling()
        Jp, Jl, r = om.dense_system(sprob, f(W), dtype=dtype)
        D, _, _, _, _, _, b = reduced(Jp, Jl, r, lam, prob.nl, dtype)
        assert rel_err(s, D) < BARS[dtype]["scaling"]
        assert rel_err(lin.get_rhs(), b) < BARS[dtype]["b"]
        sd = np.asarray(s, np.float64).reshape(-1, 9)
        for lm in range(prob.nl):
            o0, o1 = int(prob.lm_off[lm]), int(prob.lm_off[lm + 1])
            B, lm_idx, res_idx, jls = lin.debug_get_block(lm)
            B, jls = np.asarray(B, np.float64), np.asarray(jls, np.float64)
            want_jls = 1.0 / (eps + np.sqrt((w["Jl"][o0:o1] ** 2).sum((0, 1))))
            assert rel_err(jls, want_jls) < tol, (lm, jls, want_jls)
            A = np.zeros((2 * n + 3, B.shape[1]))
            for i in range(n):
                A[2 * i:2 * i + 2, 9 * i:9 * i + 9] = w["Jp"][o0 + i] * sd[prob.obs_cam[o0 + i]]
            A[:2 * n, lm_idx:lm_idx + 3] = w["Jl"][o0:o1].reshape(2 * n, 3) * want_jls
            A[:2 * n, res_idx] = w["r"][o0:o1].ravel()
            A[2 * n:, lm_idx:lm_idx + 3] = np.sqrt(lam) * np.eye(3)
            # the stored block keeps the residual column in its first 3 rows only (Q1^T r): of that column the products
            # with the landmark columns, R^T (Q1^T r) = Jl^T r, are compared
            cols = np.r_[0:9 * n, lm_idx:lm_idx + 3]
            G, Gw = B.T @ B, A.T @ A
            err = max(np.max(np.abs((G - Gw)[np.ix_(cols, cols)])), np.max(np.abs((G - Gw)[lm_idx:lm_idx + 3, res_idx])))
            assert err <= tol * np.max(np.abs(Gw)), (lm, err, np.max(np.abs(Gw)))
            kept = ~off[o0:o1]
            if kept.sum() == 0:  # nothing left: the damping rows alone
                assert np.all(B[:, :9 * n] == 0) and np.all(B[:, res_idx] == 0), lm
    lin.close()


# ---- switched off = removed ---------------------------------------------------------------------------------------------
def _random_off(prob, frac, seed):
    """a random `frac` of the observations, every landmark keeping at least 2 (a handle cannot be created on fewer)"""
    rng = np.random.default_rng(seed)
    off = rng.random(prob.nobs) < frac
    for l in np.flatnonzero(np.add.reduceat((~off).astype(int), prob.lm_off[:-1]) < 2):
        off[prob.lm_off[l]:prob.lm_off[l + 1]] = False
    return off


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
@pytest.mark.parametrize("cfg", [CONFIGS[i] for i in (0, 4, 8)], ids=cfg_id)
def test_switched_off_equals_removed(small_problem, dtype, cfg):
    """a handle on the full problem with W = 0 on a random 10 % against a handle created on the problem without them (their
    track-length classes differ, so not bit for bit: the bars of the dense checks)"""
    import rootba_b200 as rb
    bars, lam = BARS[dtype], 1e-3
    off = _random_off(small_problem, 0.1, seed=9)
    W = om.random_info(small_problem.nobs, seed=10)
    sub, kept = om.without(small_problem, off)
    assert 0.05 * small_problem.nobs < off.sum() and not np.array_equal(np.diff(sub.lm_off), np.diff(small_problem.lm_off))
    W0 = W.copy()
    W0[off] = 0.0
    out = []
    for arrays, info in ((small_problem, W0), (sub, W[kept])):
        bp = rb.BalProblem.from_arrays(arrays, dtype)
        bp.observation_sqrt_info = info
        lin = rb.LinearizorQR.create(bp, rb.SolverOptions(eta=1e-13, optimized_cost="ERROR_VALID", **cfg))
        ri = lin.compute_error()
        lin.linearize()
        inc = lin.solve(lam)
        b = lin.get_rhs()
        x = np.random.default_rng(1).uniform(-1, 1, 9 * arrays.nc).astype(dtype)
        y = lin.right_multiply(x)
        l_diff = lin.apply(None)
        lin.download_state()
        out.append((ri, b, y, inc, l_diff, bp.cams.copy(), bp.lms.copy(), lin.compute_error()))
        lin.close()
    (ri_a, b_a, y_a, inc_a, l_a, cams_a, lms_a, e_a), (ri_b, b_b, y_b, inc_b, l_b, cams_b, lms_b, e_b) = out
    assert ri_a["all"]["num_obs"] == small_problem.nobs and ri_b["all"]["num_obs"] == len(kept)
    assert ri_a["valid"]["num_obs"] == ri_b["valid"]["num_obs"] <= len(kept)  # the counting rule
    for key in ("error", "residual_sum"):
        assert abs(ri_a["all"][key] - ri_b["all"][key]) <= bars["cost"] * ri_b["all"][key]
        assert abs(ri_a["valid"][key] - ri_b["valid"][key]) <= bars["cost"] * ri_b["valid"][key]
    assert rel_err(b_a, b_b) < bars["b"] and rel_err(y_a, y_b) < bars["op"]
    assert rel_err(inc_a, inc_b) < (bars["inc"] if dtype == np.float64 else 5e-2)
    assert abs(l_a - l_b) <= bars["l_diff"] * abs(l_b)
    assert rel_err(lms_a, lms_b) < max(bars["lms"], 1e-8) and rel_err(cams_a, cams_b) < max(bars["lms"], 1e-8)
    # the two states agree to the increment's bar, so the cost after the step to that bar times the step's share of it
    assert abs(e_a["valid"]["error"] - e_b["valid"]["error"]) <= max(bars["cost"], 1e-8) * e_b["valid"]["error"]


# ---- identity and NULL ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
@pytest.mark.parametrize("cfg", [CONFIGS[0], CONFIGS[4], CONFIGS[8]], ids=cfg_id)
def test_identity_and_null_are_the_unmodified_path(small_problem, dtype, cfg):
    """after set(identity) and after set(W) then set(None): an LM run bit-identical to a fresh handle's"""
    import rootba_b200 as rb
    eye = np.tile(np.eye(2), (small_problem.nobs, 1, 1))

    def run(mode):
        bp = rb.BalProblem.from_arrays(small_problem, dtype)
        lin = rb.LinearizorQR.create(bp, rb.SolverOptions(max_num_iterations=6, **cfg))
        if mode == "identity":
            lin.set_observation_info(eye)
        elif mode == "set_then_none":
            lin.set_observation_info(om.random_info(small_problem.nobs, seed=2))
            lin.compute_error()
            lin.linearize()
            lin.set_observation_info(None)
        its, _, _ = lin.lm_run(6)
        lin.download_state()
        lin.close()
        return [{k: v for k, v in it.items() if k != "device_seconds"} for it in its], bp.cams.copy(), bp.lms.copy()
    ref = run("never")
    assert len(ref[0]) >= 3
    for mode in ("identity", "set_then_none"):
        got = run(mode)
        assert got[0] == ref[0], mode
        assert np.array_equal(got[1], ref[1]) and np.array_equal(got[2], ref[2]), mode


# ---- a switched-off observation that does not project --------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
def test_switched_off_observation_with_a_non_finite_projection(small_problem, dtype):
    """camera c at the identity pose and landmark l on its z = 0 plane: the projection of observation (c, l) divides by zero.
    With unit weights the error is numerically invalid and the linearisation fails; switched off it poisons nothing"""
    import rootba_b200 as rb
    from rootba_b200.synthetic import BalArrays
    o = int(small_problem.lm_off[40])
    c, l = int(small_problem.obs_cam[o]), 40
    cams, lms = small_problem.cams.copy(), small_problem.lms.copy()
    cams[c, :7] = (0, 0, 0, 1, 0, 0, 0)
    lms[l] = (0.5, -0.25, 0.0)
    prob = BalArrays(cams, lms, small_problem.lm_off, small_problem.obs_cam, small_problem.obs_xy)
    bp = rb.BalProblem.from_arrays(prob, dtype)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions())
    assert not lin.compute_error()["is_numerically_valid"]
    with pytest.raises(rb.RbaError):
        lin.linearize()
    W = np.ones(prob.nobs)
    W[o] = 0.0
    lin.set_observation_info(W)
    ri = lin.compute_error()
    assert ri["is_numerically_valid"] and np.isfinite(ri["all"]["error"])
    assert ri["all"]["num_obs"] == prob.nobs
    lin.linearize()
    inc = lin.solve(1e-3)
    assert np.all(np.isfinite(inc)) and np.isfinite(lin.apply(None))
    res, hw, flags = lin.observation_residuals()
    assert np.all(np.isfinite(res)) and np.all(res[o] == 0) and (flags[o] & 2) == 0
    lin.close()


# ---- the read-back -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
@pytest.mark.parametrize("with_info", [True, False])
def test_observation_residuals_in_problem_order(small_problem, dtype, with_info):
    """mixed track lengths (the slots are a permutation of the observations), a camera turned around (invalid projections),
    switched-off observations, Huber: residual, weight and flags against the model, and nothing of the handle changed"""
    import rootba_b200 as rb
    from rootba_b200 import _lib
    from rootba_b200.synthetic import BalArrays, turn_cameras_around
    prob = turn_cameras_around(small_problem, [3])
    assert len(np.unique(np.diff(prob.lm_off))) > 3
    W = om.random_info(prob.nobs, seed=12)
    W[::11] = 0.0
    f = lambda a: _rounded(a, dtype)
    sprob = BalArrays(f(prob.cams), f(prob.lms), prob.lm_off, prob.obs_cam, f(prob.obs_xy))
    Wm = f(W) if with_info else np.ones(prob.nobs)
    thr = 1.0 if with_info else 2.0
    w = om.whitened(sprob, Wm, dtype=dtype, threshold=thr)
    bp = rb.BalProblem.from_arrays(prob, dtype)
    if with_info:
        bp.observation_sqrt_info = W
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(**_options(thr)))
    lin.compute_error()
    lin.linearize()
    inc_ref = lin.solve(1e-4)
    res, hw, flags = lin.observation_residuals()
    assert res.dtype == dtype and res.shape == (prob.nobs, 2) and flags.dtype == np.uint8
    # the rounding of a projection scales with the focal length, that of the residual with the observed pixel too
    pixel = np.abs(sprob.obs_xy) + sprob.cams[prob.obs_cam, 7:8]
    scale = np.abs(w["wr"]) + np.einsum("oij,oj->oi", np.abs(om.expand(Wm, prob.nobs)), pixel)
    u = 1e-12 if dtype == np.float64 else 1e-5
    assert np.all(np.abs(res - w["wr"]) <= u * (1 + scale))
    far = np.abs(np.sqrt((w["wr"] ** 2).sum(1)) - thr) > 1e-3  # away from the kink of the Huber weight
    assert np.allclose(hw[far], w["hw"][far], rtol=1e-9 if dtype == np.float64 else 1e-2, atol=0)
    assert 0.05 < (hw < 1).mean() < 0.95
    assert np.array_equal(flags, w["valid"].astype(np.uint8) | (w["on"].astype(np.uint8) << 1))
    assert ((flags & 1) == 0).sum() > 0 and (((flags & 2) == 0).sum() > 0) == with_info
    assert np.array_equal(lin.solve(1e-4), inc_ref)  # still linearised, the same solve
    # any pointer may be NULL, not all
    only = np.zeros(prob.nobs, np.uint8)
    lib = _lib.lib()
    assert lib.rba_get_observation_residuals(lin.h, None, None, C.c_void_p(only.ctypes.data)) == 0
    assert np.array_equal(only, flags)
    assert lib.rba_get_observation_residuals(lin.h, None, None, None) == -1
    lin.close()


# ---- the loop the feature exists for ------------------------------------------------------------------------------------
def test_outlier_loop_reaches_the_minimum_of_the_problem_without_them():
    """2 % gross outliers (30 to 100 sigma) planted in a problem whose keypoint noise is sigma = 0.5: solve, read the
    residuals, switch off |W r| > 5, solve again on the same handle.  Every planted outlier is off, and the state is the
    scipy minimum of the problem without the switched-off observations (a uniform W = I / sigma scales the cost by
    1 / sigma^2 and leaves the minimiser), the gauge held by two fixed cameras."""
    import rootba_b200 as rb
    from objective_checks import scipy_minimum
    from rootba_b200.synthetic import BalArrays, synth_bal
    sigma = 0.5
    rng = np.random.default_rng(77)
    prob = synth_bal(16, 80, 0.0, seed=41, track_lengths=rng.integers(12, 17, 80), lm_spread=0.5, obs_noise=sigma)
    planted = rng.random(prob.nobs) < 0.02
    ang = rng.uniform(0, 2 * np.pi, prob.nobs)
    mag = rng.uniform(30, 100, prob.nobs) * sigma
    xy = prob.obs_xy + np.where(planted[:, None], mag[:, None] * np.stack([np.cos(ang), np.sin(ang)], 1), 0.0)
    prob = BalArrays(prob.cams, prob.lms, prob.lm_off, prob.obs_cam, xy)
    mask = np.zeros(prob.nc, np.uint8)
    mask[[0, 8]] = 15
    bp = rb.BalProblem.from_arrays(prob, np.float64)
    bp.camera_fixed = mask
    bp.observation_sqrt_info = np.full(prob.nobs, 1 / sigma)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(max_num_iterations=60, function_tolerance=1e-15, eta=1e-10))
    lin.lm_run(200)
    res, _, flags = lin.observation_residuals()
    off = np.sqrt((res ** 2).sum(1)) > 5.0
    assert planted.sum() >= 10 and np.all(off[planted])
    # without a robust norm an outlier also drags its landmark's other residuals over the bar: those go too
    assert off.sum() < 0.2 * prob.nobs and np.add.reduceat((~off).astype(int), prob.lm_off[:-1]).min() >= 2
    W = np.full(prob.nobs, 1 / sigma)
    W[off] = 0.0
    lin.set_observation_info(W)
    lin.lm_run(200)
    lin.download_state()
    ri = lin.compute_error()
    _, _, flags = lin.observation_residuals()
    lin.close()
    assert np.array_equal((flags & 2) == 0, off)
    assert ri["valid"]["num_obs"] == int((~off).sum()) and ri["all"]["num_obs"] == prob.nobs
    sub, _ = om.without(prob, off)
    _, lms_s, cost_s = scipy_minimum(sub, mask=mask)
    cost_s /= sigma ** 2
    assert abs(ri["all"]["error"] - cost_s) <= 1e-8 * cost_s, (ri["all"]["error"], cost_s)
    assert np.max(np.abs(bp.lms - lms_s)) < 1e-4 * max(1.0, np.max(np.abs(lms_s)))
    assert np.array_equal(bp.cams[[0, 8]], np.asarray(prob.cams, np.float64)[[0, 8]])


# ---- covariances ---------------------------------------------------------------------------------------------------------
def test_covariance_scales_with_sigma_squared_and_matches_the_whitened_inverse(case7):
    import rootba_b200 as rb
    from test_gpu_landmark_priors import _dense_covariance_check
    prob, W = case7
    mask = np.zeros(prob.nc, np.uint8)
    mask[[0, 3]] = 15

    def cov(info):
        bp = rb.BalProblem.from_arrays(prob, np.float64)
        bp.camera_fixed = mask
        bp.observation_sqrt_info = info
        lin = rb.LinearizorQR.create(bp, rb.SolverOptions())
        out = lin.covariance()
        lin.close()
        return out
    sigma = 0.4
    (cam1, lm1), (cam_s, lm_s) = cov(None), cov(np.full(prob.nobs, 1 / sigma))
    assert rel_err(cam_s, sigma ** 2 * cam1) < 1e-9 and rel_err(lm_s, sigma ** 2 * lm1) < 1e-9
    W = W.copy()
    long_tracks = np.repeat(np.diff(prob.lm_off) >= 4, np.diff(prob.lm_off))  # every landmark keeps rank 3
    W[np.flatnonzero(long_tracks)[::7]] = 0.0
    cam, lm = cov(W)
    Jp, Jl, _ = om.dense_system(prob, W)
    _dense_covariance_check(cam, lm, Jp, Jl, fixed_entries(mask))


# ---- the protocol --------------------------------------------------------------------------------------------------------
def test_protocol_and_bad_input(small_problem):
    import rootba_b200 as rb
    from rootba_b200 import _lib
    lib = _lib.lib()
    W = om.random_info(small_problem.nobs, seed=4)
    bp = rb.BalProblem.from_arrays(small_problem, np.float64)
    bp.observation_sqrt_info = W
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions())
    bytes_with = lin.stats()["device_bytes"]
    lin.compute_error()
    lin.linearize()
    inc_ref = lin.solve(1e-4)
    bad = W.copy()
    bad[17, 0, 1] = np.nan
    assert lib.rba_set_observation_info(lin.h, C.c_void_p(bad.ctypes.data)) == -1  # RBA_ERR_INVALID_ARGUMENT
    assert lib.rba_last_error()
    assert np.array_equal(lin.solve(1e-4), inc_ref)  # nothing changed, still linearised
    with pytest.raises(ValueError):
        lin.set_observation_info(bad)
    assert np.array_equal(bp.observation_sqrt_info, W)
    lin.set_observation_info(W)  # a change needs a new linearisation
    for call in (lambda: lin.solve(1e-4), lambda: lin.apply(None)):
        with pytest.raises(rb.RbaError) as e:
            call()
        assert e.value.code == -6  # RBA_ERR_STATE
    lin.linearize()
    assert np.array_equal(lin.solve(1e-4), inc_ref)
    lin.close()
    lin2 = rb.LinearizorQR.create(rb.BalProblem.from_arrays(small_problem, np.float64), rb.SolverOptions())
    assert bytes_with - lin2.stats()["device_bytes"] >= 32 * small_problem.nobs  # 4 Scalars per slot
    lin2.close()


# ---- the example ---------------------------------------------------------------------------------------------------------
def test_example_takes_observation_info_and_writes_residuals(tmp_path, small_problem):
    from rootba_b200.synthetic import write_bal
    path = tmp_path / "problem.txt"
    write_bal(small_problem, str(path))
    info = np.full(small_problem.nobs, 2.0)
    info[::50] = 0.0
    np.save(tmp_path / "info.npy", info)
    cmd = [sys.executable, os.path.join(ROOT, "examples", "solve_bal.py"), str(path), "--max-num-iterations", "3",
           "--log-path", str(tmp_path / "log.json"), "--residuals", str(tmp_path / "res.npz")]
    r = subprocess.run(cmd + ["--observation-info", str(tmp_path / "info.npy")], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    with np.load(tmp_path / "res.npz") as f:
        assert f["residual"].shape == (small_problem.nobs, 2) and f["robust_weight"].shape == (small_problem.nobs,)
        assert np.array_equal((f["flags"] & 2) == 0, info == 0)
    np.save(tmp_path / "short.npy", info[:-1])
    r = subprocess.run(cmd + ["--observation-info", str(tmp_path / "short.npy")], capture_output=True, text=True, timeout=300)
    assert r.returncode != 0 and "observations" in r.stderr


# ---- two GPUs ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("peer", ["1", "0"])
@pytest.mark.parametrize("sfx", ["f32", "f64"])
def test_two_ranks_with_observation_info(tmp_path, peer, sfx):
    """every rank passes the full array: the sharded step equals the single-rank step at the bars of test_gpu_multirank.py, and
    each rank's read-back covers exactly the observations of its landmark shard"""
    res = oc.run_two_ranks(tmp_path, "multirank_observation_info_worker.py", sfx, peer, 31500,
                           (31 if peer == "1" else 0) + (37 if sfx == "f32" else 0))
    tols = 1e-4 if sfx == "f32" else 1e-8
    assert res["replicas_identical"] and res["readback_covers_own_shard_only"], res
    assert res["b"] < 4 * tols and res["inc"] < tols and res["l_diff"] < 20 * tols, res
    assert res["lms"] < 10 * tols and res["cams"] < tols and res["cost"] < tols and res["cost0"] < tols, res
    assert res["residuals"] < tols, res
