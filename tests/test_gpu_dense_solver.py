"""linear_solver_type = DENSE_SCHUR (DESIGN.md section 27) on the GPU: the exact increment of the reduced camera system.

Every step is checked twice: by the existing one-step checkers of each feature (objective_checks.check_against_dense and the
tied, robust, whitened and loss variants, whose PCG bars it passes trivially), and by check_exact against -H_ff^-1 b_f of the
dense float64 model with the bar C kappa(H_ff) u, kappa computed here.  C = 1000 in float64: the handle's b and D come from
its own Scalar linearisation and the matrix from the float64 re-linearisation, each within a few u of the model, and the
solve turns a relative perturbation e of the system into at most about kappa e.  In float32 C = 100 with u of float32, the
bar of the float32 PCG checks (test_gpu_pcg_iterates)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import objective_checks as oc
from conftest import ROOT, rel_err

pytestmark = pytest.mark.gpu

DENSE = dict(linear_solver_type="DENSE_SCHUR")
CONFIGS = [dict(c, **DENSE) for c in oc.CONFIGS if c["solver_type"] != "POWER_SCHUR_COMPLEMENT"]
CONFIGS += [dict(solver_type="SQUARE_ROOT", operator_form=op, stage2_form="IDENTITY", **DENSE) for op in ("DENSE", "IMPLICIT")]
DTYPES = [np.float64, np.float32]
dt_id = lambda d: np.dtype(d).name
C_BAR = {np.float64: 1000.0, np.float32: 100.0}
U = {np.float64: 2.0 ** -53, np.float32: 2.0 ** -24}
SUCCESS, FAILURE, REASON_OK, REASON_PIVOT = 1, 2, 7, 8


def _prob(nc=7, nl=90, seed=21, mean_n=3.6, **kw):
    from rootba_b200.synthetic import synth_bal
    return synth_bal(nc, nl, mean_n, seed=seed, **kw)


def _rounded(prob, dtype):
    from rootba_b200.synthetic import BalArrays
    f = lambda a: np.asarray(np.asarray(a, dtype), np.float64)
    return BalArrays(f(prob.cams), f(prob.lms), prob.lm_off, prob.obs_cam, f(prob.obs_xy))


def model_step(prob, dtype, lam, mask=None, pinv=False, **model):
    """(H, b, free) of the dense float64 model at the state rounded to dtype; pinv: the landmark blocks pseudo-inverted
    (lambda = 0 with a rank-deficient landmark)"""
    sprob = _rounded(prob, dtype)
    Jp, Jl, r = oc.dense_system(sprob, **{k: oc._stored(v, dtype) for k, v in model.items()})
    D, sl, Jps, Jls, Minv, H, b = oc.reduced(Jp, Jl, r, 1.0 if pinv else lam, prob.nl, dtype)
    if pinv:
        Minv = np.zeros_like(Minv)
        for l in range(prob.nl):
            B = Jls[:, 3 * l:3 * l + 3]
            Minv[3 * l:3 * l + 3, 3 * l:3 * l + 3] = np.linalg.pinv(B.T @ B + lam * np.eye(3), rcond=1e-10, hermitian=True)
        W = Jps.T @ Jls
        H = Jps.T @ Jps - W @ Minv @ W.T + lam * np.eye(Jp.shape[1])
        b = Jps.T @ r - W @ Minv @ (Jls.T @ r)
    n = H.shape[0]
    fixed = oc.fixed_entries(mask) if mask is not None else np.zeros(n, bool)
    return H, b, ~fixed


def check_exact(lin, H, b, free, dtype, lam):
    """the handle's increment at lam against -H_ff^-1 b_f at C kappa u; held entries exactly 0; the summary of the dense path"""
    inc = lin.solve(lam)
    cg = lin.last_cg
    assert (cg.termination_type, cg.reason, cg.num_iterations, cg.num_matvecs) == (SUCCESS, REASON_OK, 0, 0)
    assert np.all(inc[~free] == 0)
    Hff = H[np.ix_(free, free)]
    kappa = np.linalg.cond(Hff)
    want = -np.linalg.solve(Hff, b[free])
    bar = C_BAR[dtype] * kappa * U[dtype]
    err = rel_err(inc[free].astype(np.float64), want)
    assert err < bar, (err, bar, kappa)
    return inc


def exact_step(prob, dtype, cfg, lam=1e-3, mask=None, **model):
    import rootba_b200 as rb
    H, b, free = model_step(prob, dtype, lam, mask, **model)
    bp = oc.bal_problem(prob, dtype, camera_fixed=mask, camera_prior=model.get("camera"), camera_pair_prior=model.get("pairs"),
                        landmark_prior=model.get("landmarks"))
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(**cfg))
    lin.compute_error()
    lin.linearize()
    check_exact(lin, H, b, free, dtype, lam)
    lin.close()


# ---- one step in every configuration ------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=dt_id)
@pytest.mark.parametrize("cfg", CONFIGS, ids=oc.cfg_id)
def test_step_in_every_configuration(cfg, dtype):
    prob = _prob()
    oc.check_against_dense(cfg, prob, dtype=dtype)
    exact_step(prob, dtype, cfg)


def _priors():
    """the prior case of tests/camera_prior_model.py with a pair prior of each kind and landmark priors on every second landmark"""
    import camera_prior_model as pm
    import landmark_prior_model as lp
    import pair_prior_model as qm
    prob, mean_c, L_c = pm.prior_case(7, 90)
    pairs = np.array([(0, 1), (3, 1), (5, 6)], np.int32)
    rng = np.random.default_rng(11)
    pmean = qm.mean_at(prob.cams, pairs)
    pmean[:, 4:7] += rng.normal(0, 0.05, (len(pairs), 3))
    pL = np.stack([qm.sqrt_info_kind(k, rng) for k in ("dense", "translation", "rotation")])
    return prob, dict(camera=(mean_c, L_c), pairs=(pairs, pmean, pL), landmarks=lp.prior_case(prob.lms, every=2, seed=8))


@pytest.mark.parametrize("dtype", DTYPES, ids=dt_id)
@pytest.mark.parametrize("kinds", [("camera",), ("pairs",), ("landmarks",), ("camera", "pairs", "landmarks")], ids="+".join)
def test_priors_without_losses(kinds, dtype):
    prob, model = _priors()
    model = {k: v for k, v in model.items() if k in kinds}
    oc.check_against_dense(CONFIGS[0], prob, dtype=dtype, **model)
    exact_step(prob, dtype, CONFIGS[0], **model)


@pytest.mark.parametrize("dtype", DTYPES, ids=dt_id)
@pytest.mark.parametrize("kinds", [[0], [1], [2], [0, 1, 2]], ids=["camera", "pair", "landmark", "all"])
def test_priors_with_losses(kinds, dtype):
    import prior_loss_model as plm
    import test_gpu_prior_loss as tpl
    prob, priors = plm.robust_case()
    tpl.check_robust_step(CONFIGS[0], prob, priors, tpl.losses_for(prob, priors, kinds, seed=3), dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=dt_id)
def test_observation_info_with_switched_off_observations(dtype):
    import observation_info_model as om
    import test_gpu_observation_info as toi
    prob = _prob()
    W = om.random_info(prob.nobs, seed=3)
    W[::9] = 0.0
    W[4::9, 1] = 0.0
    toi.check_whitened_step(CONFIGS[0], prob, W, dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=dt_id)
def test_every_observation_loss(dtype):
    import observation_loss_model as lm
    import test_gpu_observation_loss as tol
    prob = _prob()
    kind, scale = lm.mixed(prob.nobs, seed=5, lo=1.0, hi=4.0)
    assert set(np.unique(kind)) >= {lm.HUBER, lm.CAUCHY, lm.SOFT_L1, lm.TUKEY}
    tol.check_loss_step(CONFIGS[0], prob, kind, scale, dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=dt_id)
@pytest.mark.parametrize("cfg", [CONFIGS[0], CONFIGS[-3]], ids=oc.cfg_id)
def test_held_parameters(cfg, dtype):
    """oc.MASK holds every bit, combinations of intrinsics and one whole camera: those entries exactly 0"""
    prob = _prob()
    oc.check_against_dense(cfg, prob, dtype=dtype, mask=oc.MASK)
    exact_step(prob, dtype, cfg, mask=oc.MASK)


# ---- tied systems -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=dt_id)
def test_intrinsics_groups(dtype):
    import test_gpu_shared_intrinsics as ts
    from test_shared_intrinsics_model import GROUP, _case
    prob, _, model = _case(("camera",))
    ts.check_tied_step(CONFIGS[0], prob, GROUP, model, dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=dt_id)
def test_rigs(dtype):
    import test_gpu_camera_rigs as tr
    from test_camera_rig_model import RIG, rig_case
    prob, _, _, E, model = rig_case(("camera",))
    tr.check_rig_step(CONFIGS[0], prob, RIG, E, model, dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=dt_id)
def test_rigs_with_sensors(dtype):
    import test_gpu_rig_sensors as tz
    from test_camera_rig_model import rig_case
    prob, _, _, E, model = rig_case(("camera", "pairs"))
    tz.check_sensor_step(CONFIGS[0], prob, E, model, dtype)


# ---- shapes -------------------------------------------------------------------------------------------------------------
def test_every_track_length_class():
    """tracks of 2 .. 70 observations: the landmark pass's lanes stride over slots of long tracks"""
    prob = _prob(nc=72, nl=150, seed=5, mean_n=30.0, max_track=72)
    lengths = set(np.diff(prob.lm_off).tolist())
    assert min(lengths) <= 3 and max(lengths) > 64 and len(lengths) > 20
    exact_step(prob, np.float64, CONFIGS[0])


@pytest.mark.parametrize("nc", [3, 7, 57, 64], ids=["below_one_tile", "padding_1", "padding_63", "multiple_of_64"])
def test_camera_counts(nc):
    assert (-9 * nc) % 64 == {3: 37, 7: 1, 57: 63, 64: 0}[nc]
    exact_step(_prob(nc=nc, nl=12 * nc, seed=nc), np.float64, CONFIGS[0])


def test_lambda_zero_with_a_rank_deficient_landmark():
    """a landmark of track length 2 with one observation switched off (W = 0, DESIGN.md section 19), so that its Jl has rank 2,
    at lambda = 0: its null direction is dropped, as in the pseudo-inverse of the model, where the observation is removed;
    two whole cameras held fix the gauge"""
    import rootba_b200 as rb
    from rootba_b200.synthetic import BalArrays
    prob = _prob()
    n = np.diff(prob.lm_off)
    l = int(np.flatnonzero(n == 2)[0])
    off = int(prob.lm_off[l]) + 1
    W = np.tile(np.eye(2), (prob.nobs, 1, 1))
    W[off] = 0.0
    keep = np.arange(prob.nobs) != off
    lm_off = prob.lm_off.copy()
    lm_off[l + 1:] -= 1
    removed = BalArrays(prob.cams, prob.lms, lm_off, prob.obs_cam[keep], prob.obs_xy[keep])
    mask = np.zeros(prob.nc, np.uint8)
    mask[[0, 1]] = oc.FIX_POSE | oc.FIX_F | oc.FIX_K1 | oc.FIX_K2
    H, b, free = model_step(removed, np.float64, 0.0, mask, pinv=True)
    bp = oc.bal_problem(prob, np.float64, camera_fixed=mask, observation_sqrt_info=W)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(**CONFIGS[0]))
    lin.compute_error()
    lin.linearize()
    check_exact(lin, H, b, free, np.float64, 0.0)
    lin.close()


# ---- failure ------------------------------------------------------------------------------------------------------------
def _handle(prob, dtype=np.float64, cfg=None, **features):
    import rootba_b200 as rb
    bp = oc.bal_problem(prob, dtype, **features)
    return bp, rb.LinearizorQR.create(bp, rb.SolverOptions(**(CONFIGS[0] if cfg is None else cfg)))


@pytest.mark.parametrize("lam", [float("nan"), -1e3], ids=["nan", "negative"])
def test_failed_pivot(lam):
    """a non-finite or indefinite damped system: FAILURE / reason 8, NaN on the free entries, 0 on the held ones; rba_lm_step
    sets solve_failed"""
    prob = _prob()
    mask = np.zeros(prob.nc, np.uint8)
    mask[2] = oc.FIX_POSE
    bp, lin = _handle(prob, camera_fixed=mask)
    lin.compute_error()
    lin.linearize()
    inc = lin.solve(lam)
    assert (lin.last_cg.termination_type, lin.last_cg.reason, lin.last_cg.num_iterations) == (FAILURE, REASON_PIVOT, 0)
    held = oc.fixed_entries(mask)
    assert np.all(np.isnan(inc[~held])) and np.all(inc[held] == 0)
    r = lin.lm_step(lam, True)
    assert r["solve_failed"] and lin.last_cg.reason == REASON_PIVOT
    lin.close()


def test_lm_run_rejects_failed_steps_and_restores_the_state():
    """a negative initial lambda: every step fails, is rejected and undone; the state stays bit-identical"""
    import rootba_b200 as rb
    prob = _prob()
    bp, lin = _handle(prob)
    cams0, lms0 = bp.cams.copy(), bp.lms.copy()
    its, _, _ = lin.lm_run(4, rb.SolverOptions(initial_trust_region_radius=-1e-3, max_num_iterations=4, **DENSE))
    assert len(its) == 4
    assert all(not it["accepted"] and it["cg_termination"] == FAILURE for it in its)
    lin.download_state()
    assert np.array_equal(bp.cams, cams0) and np.array_equal(bp.lms, lms0)
    lin.close()


# ---- protocol -----------------------------------------------------------------------------------------------------------
def _create(prob, **fields):
    from rootba_b200 import _lib
    L = _lib.lib()
    o = _lib.SolverOpts()
    L.rba_default_solver_opts(C.byref(o))
    for k, v in fields.items():
        setattr(o, k, v)
    off = np.ascontiguousarray(prob.lm_off, np.int64)
    oc_ = np.ascontiguousarray(prob.obs_cam, np.int32)
    xy = np.ascontiguousarray(prob.obs_xy, np.float64)
    pv = _lib.ProblemView(prob.nc, prob.nl, prob.nobs, off.ctypes.data, oc_.ctypes.data, xy.ctypes.data)
    h = C.c_void_p(12345)
    rc = L.rba_create_f64(C.byref(pv), C.byref(o), C.byref(h))
    msg = L.rba_last_error().decode() if rc else ""
    if rc == 0:
        L.rba_destroy(h)
    return rc, h.value, msg


@pytest.mark.parametrize("fields,code", [(dict(linear_solver_type=2), -1), (dict(linear_solver_type=-1), -1),
                                         (dict(linear_solver_type=1, solver_type=2), -1),
                                         (dict(linear_solver_type=1, nranks=2, rank=0), -4)],
                         ids=["value_2", "value_-1", "power_series", "two_ranks"])
def test_rejected_options(fields, code):
    rc, h, _ = _create(_prob(), **fields)
    assert rc == code and h == 12345


@pytest.mark.parametrize("fields", [dict(), dict(solver_type=1), dict(use_householder_marginalization=0, operator_form=1),
                                    dict(stage2_form=1)], ids=["default", "sc", "givens_implicit", "identity"])
def test_accepted_options(fields):
    assert _create(_prob(), linear_solver_type=1, **fields)[0] == 0


def test_memory_check_on_13682_cameras():
    """the Final-13682 camera count needs a (9 * 13682 -> 123 136)^2 float64 matrix, about 121 GB: RBA_ERR_UNSUPPORTED with the
    byte count, the output handle untouched; a default handle on the same problem is unaffected"""
    from rootba_b200.synthetic import BalArrays
    nc = 13682
    rng = np.random.default_rng(0)
    nl = nc
    obs_cam = np.sort(np.stack([np.arange(nc), (np.arange(nc) + 1) % nc], 1), axis=1).ravel().astype(np.int32)
    cams = np.zeros((nc, 10))
    cams[:, 3] = 1.0
    cams[:, 6] = -5.0
    cams[:, 7] = 1.0
    lms = rng.normal(0, 0.1, (nl, 3))
    prob = BalArrays(cams, lms, np.arange(0, 2 * nl + 1, 2, dtype=np.int64), obs_cam, rng.normal(0, 0.01, (2 * nl, 2)))
    rc, h, msg = _create(prob, linear_solver_type=1)
    np_ = (9 * nc + 63) // 64 * 64
    assert rc == -4 and h == 12345
    need = int(msg.split("needs ")[1].split(" bytes")[0])
    assert need >= 8 * np_ * np_ > 120e9
    assert _create(prob)[0] == 0


def test_device_bytes_grow_by_the_dense_buffers():
    prob = _prob(nc=20, nl=200)
    stats = []
    for cfg in (dict(), DENSE):
        _, lin = _handle(prob, cfg=cfg)
        stats.append(lin.stats()["device_bytes"])
        lin.close()
    np_ = (9 * prob.nc + 63) // 64 * 64
    fixed = 8 * (np_ * np_ + 64 * np_ + 64 * 64 + 3 * np_) + 4
    extra = stats[1] - stats[0] - fixed
    assert extra >= 45 * 8 * prob.nobs and extra % (45 * 8) == 0, (stats, fixed)


# ---- determinism and the unchanged parts of the solve ---------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=dt_id)
def test_bit_identical_repeats_and_unchanged_solve_outputs(dtype):
    prob = _prob(nc=20, nl=200)
    x = np.random.default_rng(1).uniform(-1, 1, 9 * prob.nc)
    out = []
    for cfg in (DENSE, DENSE, dict()):
        _, lin = _handle(prob, dtype, cfg=cfg)
        lin.compute_error()
        lin.linearize()
        incs = [lin.solve(1e-3) for _ in range(2)]
        out.append((incs, lin.get_rhs(), lin.get_preconditioner(), lin.right_multiply(x)))
        lin.close()
    (a, b, it) = out
    assert np.array_equal(a[0][0], a[0][1]) and np.array_equal(a[0][0], b[0][0])
    for d in (a, b):
        assert np.array_equal(d[1], it[1])
        assert all(np.array_equal(p, q) for p, q in zip(d[2], it[2]))
        assert np.array_equal(d[3], it[3])


# ---- end to end ---------------------------------------------------------------------------------------------------------
def test_lm_run_equals_the_host_loop():
    import rootba_b200 as rb
    oc.check_lm_run_equals_host_loop(_prob(nc=20, nl=200), rb.SolverOptions(max_num_iterations=12, **DENSE))


def test_lm_run_against_converged_pcg():
    """DENSE_SCHUR against PCG at eta = 1e-13: the same accepted steps and costs to 1e-9"""
    import rootba_b200 as rb
    prob = _prob(nc=20, nl=200)
    runs = []
    for cfg in (DENSE, dict(eta=1e-13, max_linear_solver_iterations=2000)):
        _, lin = _handle(prob, cfg=cfg)
        runs.append(lin.lm_run(12, rb.SolverOptions(max_num_iterations=12, **cfg))[0])
        lin.close()
    assert len(runs[0]) == len(runs[1]) >= 3
    for d, p in zip(*runs):
        assert d["accepted"] == p["accepted"] and d["cg_iterations"] == 0
        assert abs(d["cost"] - p["cost"]) <= 1e-9 * p["cost"]


def test_minimum_with_every_prior_kind():
    """a held camera and every prior kind: rba_lm_run with DENSE_SCHUR reaches scipy's minimum of the total objective"""
    import rootba_b200 as rb
    from rootba_b200.synthetic import BalArrays
    prob, model = _priors()
    mask = np.zeros(prob.nc, np.uint8)
    mask[0] = oc.FIX_POSE | oc.FIX_F | oc.FIX_K1 | oc.FIX_K2
    cams, lms, cost = oc.scipy_minimum(prob, mask=mask, **model)
    bp, lin = _handle(prob, camera_fixed=mask, camera_prior=model["camera"], camera_pair_prior=model["pairs"],
                      landmark_prior=model["landmarks"])
    its, _, _ = lin.lm_run(60, rb.SolverOptions(max_num_iterations=60, function_tolerance=1e-15, **DENSE))
    lin.download_state()
    lin.close()
    got = oc.total_cost(BalArrays(bp.cams, bp.lms, prob.lm_off, prob.obs_cam, prob.obs_xy), **model)
    assert abs(got - cost) <= 1e-8 * cost, (got, cost, len(its))


def test_example_runs_and_writes_its_log(tmp_path):
    from rootba_b200.synthetic import write_bal
    path = tmp_path / "p.txt"
    write_bal(_prob(nc=20, nl=200), str(path))
    log = tmp_path / "log.json"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "examples", "solve_bal.py"), str(path), "--max-num-iterations", "3",
                        "--linear-solver-type", "DENSE_SCHUR", "--log-path", str(log)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert log.exists() and log.stat().st_size > 0
