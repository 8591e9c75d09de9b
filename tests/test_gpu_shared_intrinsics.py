"""Intrinsics shared across groups of cameras (rba_set_intrinsics_groups) on the GPU: every PCG solver configuration against
the dense float64 model of the tied problem (tests/shared_intrinsics_model.py), with held flags and every prior kind, the
assembled operator, members bit-identical through LM runs, groups of one and cleared groups bit-identical to no groups,
and the rejected calls."""
import ctypes as C

import numpy as np
import pytest

import shared_intrinsics_model as sm
from conftest import rel_err
from objective_checks import BARS, CONFIGS, bal_problem, cfg_id, dense_system, fixed_entries, total_cost
from test_shared_intrinsics_model import GROUP, _case

pytestmark = pytest.mark.gpu

PCG_CONFIGS = [c for c in CONFIGS if c["solver_type"] != "POWER_SCHUR_COMPLEMENT"]
PCG_CONFIGS += [dict(solver_type="SQUARE_ROOT", stage2_form="IDENTITY")]


def check_tied_step(cfg, prob, group, model, dtype=np.float64, mask=None, lam=1e-3, env=None):
    """one LM step of a handle with intrinsics groups against the dense model of the tied problem: the scaling, b, the
    inverse preconditioner, the increment, l_diff and the state after apply (members bit-identical to their lead)"""
    import rootba_b200 as rb
    from rootba_b200.synthetic import BalArrays
    bars = BARS[dtype]
    f = lambda a: np.asarray(np.asarray(a, dtype), np.float64)
    sprob = BalArrays(f(prob.cams), f(prob.lms), prob.lm_off, prob.obs_cam, f(prob.obs_xy))
    smodel = {k: (tuple(v[:-2]) + (f(v[-2]), f(v[-1]))) for k, v in model.items()}
    lead = sm.leads(group)
    Jp, Jl, r = dense_system(sprob, **smodel)
    D, sl, Jls, Minv, Hu, bu, P, E = sm.tied_step(Jp, Jl, r, lam, prob.nl, lead, dtype)
    Jps = Jp * D
    W = Jps.T @ Jls
    Hfull = Jps.T @ Jps - W @ Minv @ W.T
    jacobi = cfg.get("preconditioner_type") == "JACOBI"
    src = Jps.T @ Jps if jacobi else Hfull
    blocks = np.stack([src[9 * c:9 * c + 9, 9 * c:9 * c + 9] for c in range(prob.nc)])
    fixed9 = fixed_entries(mask) if mask is not None else np.zeros(9 * prob.nc, bool)
    keep = np.flatnonzero(~sm.members(lead))
    fu = ~fixed9[keep]
    names = {"camera": "camera_prior", "pairs": "camera_pair_prior", "landmarks": "landmark_prior"}
    bp = bal_problem(prob, dtype, camera_fixed=mask, **{names[k]: v for k, v in model.items()})
    bp.intrinsics_group = group
    with pytest.MonkeyPatch.context() as m:
        for k, v in (env or {}).items():
            m.setenv(k, v)
        lin = rb.LinearizorQR.create(bp, rb.SolverOptions(eta=1e-13, **cfg))
    e0 = lin.compute_error()["all"]["error"]
    assert abs(e0 - total_cost(sprob, **smodel)) <= bars["cost"] * e0
    lin.linearize()
    inc = lin.solve(lam)
    s, _ = lin.get_jacobian_scaling()
    assert rel_err(s, D) < bars["scaling"]
    assert rel_err(lin.get_rhs(), np.where(fixed9, 0.0, E @ bu)) < bars["b"]
    inv, _ = lin.get_preconditioner()
    want_inv = sm.device_blocks(blocks, lam, lead, fixed9)
    for c in range(prob.nc):
        assert rel_err(inv[c], want_inv[c]) < bars["inv"], c
    Hff = Hu[np.ix_(fu, fu)]
    u = np.zeros(len(bu))
    u[fu] = -np.linalg.solve(Hff, bu[fu])
    tol = bars["inc"] if dtype == np.float64 else max(bars["inc"], 100 * 2.0 ** -24 * np.linalg.cond(Hff))
    assert rel_err(inc, P @ u) < tol
    inc64 = np.asarray(inc, np.float64)
    g = lead >= 0
    assert np.array_equal(inc.reshape(-1, 9)[g, 6:], inc.reshape(-1, 9)[lead[g], 6:])
    dl_s = -Minv @ (Jls.T @ r + Jls.T @ (Jps @ inc64))
    want_l = 0.5 * r @ r - 0.5 * np.sum((r + Jps @ inc64 + Jls @ dl_s) ** 2)
    l_diff = lin.apply(None)
    assert abs(l_diff - want_l) <= bars["l_diff"] * abs(want_l)
    lin.download_state()
    assert np.array_equal(bp.cams[g, 7:], bp.cams[lead[g], 7:])
    want_cams = sm.apply_tied(sprob.cams, D * inc64)
    assert rel_err(bp.cams[:, 4:], want_cams[:, 4:]) < (1e-10 if dtype == np.float64 else 1e-5)
    assert rel_err(bp.lms, sprob.lms + (sl * dl_s).reshape(-1, 3)) < bars["lms"]
    lin.close()


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("cfg", PCG_CONFIGS, ids=cfg_id)
def test_every_solver_against_the_tied_model(cfg, dtype):
    prob, _, model = _case(("camera",))
    check_tied_step(cfg, prob, GROUP, model, dtype)


@pytest.mark.parametrize("grouping", ["all_one_group", "lead_without_observations"])
def test_groupings(grouping):
    prob, _, model = _case(())
    nc = prob.nc
    # camera nc - 1 has no observations: the lead of a group of its own and camera 2
    group = np.zeros(nc, np.int32) if grouping == "all_one_group" else np.where(np.isin(np.arange(nc), [2]), 0, -1).astype(np.int32)
    if grouping == "lead_without_observations":
        from rootba_b200.synthetic import BalArrays
        cams = np.vstack([prob.cams[-1:], prob.cams[:-1]])  # the camera without observations first: the lead
        oc = np.asarray(prob.obs_cam) + 1
        prob = BalArrays(cams, prob.lms, prob.lm_off, oc.astype(np.int32), prob.obs_xy)
        group = np.full(nc, -1, np.int32)
        group[[0, 3, 5]] = 2
        cams[[3, 5], 7:] = cams[0, 7:]
    else:
        prob.cams[:, 7:] = prob.cams[0, 7:]
    for cfg in (PCG_CONFIGS[0], PCG_CONFIGS[-2]):
        check_tied_step(cfg, prob, group, model={"camera": _case(("camera",))[2]["camera"]} if grouping == "all_one_group" else {})


def test_assembled_operator_with_damping():
    """RBA_ASSEMBLED_AT=2: S is built and the solve switches to it from iteration 2 (lambda > 0: its damping part)"""
    import rootba_b200 as rb
    prob, _, model = _case(("camera",))
    check_tied_step(PCG_CONFIGS[0], prob, GROUP, model, lam=1e-2, env={"RBA_ASSEMBLED_AT": "2"})
    # the same solve did switch: more than 2 iterations, and the operator it ended with is S (its algorithmic bytes)
    bytes_of = {}
    for at in ("2", None):
        with pytest.MonkeyPatch.context() as m:
            if at:
                m.setenv("RBA_ASSEMBLED_AT", at)
            else:
                m.setenv("RBA_ASSEMBLED_RCS", "0")
            bp = bal_problem(prob, np.float64, camera_prior=model["camera"])
            bp.intrinsics_group = GROUP
            lin = rb.LinearizorQR.create(bp, rb.SolverOptions(eta=1e-13, **PCG_CONFIGS[0]))
        lin.linearize()
        lin.solve(1e-2)
        assert lin.last_cg.num_iterations > 2
        bytes_of[at] = lin.stats()["matvec_algorithmic_bytes"]
        lin.close()
    assert bytes_of["2"] != bytes_of[None]


def test_covariance_is_that_of_the_tied_problem():
    """rba_compute_covariance against the dense inverse of the tied system, the gauge fixed by the camera priors (and a
    held pose)"""
    import rootba_b200 as rb
    from objective_checks import FIX_POSE
    prob, lead, model = _case(("camera", "landmarks"))
    Jp, Jl, _ = dense_system(prob, **model)
    for held in (False, True):
        mask = None
        if held:
            mask = np.zeros(prob.nc, np.uint8)
            mask[3] = FIX_POSE
        want_cam, want_lm = sm.tied_covariance(Jp, Jl, lead, fixed_entries(mask) if held else None)
        bp = bal_problem(prob, np.float64, camera_prior=model["camera"], landmark_prior=model["landmarks"], camera_fixed=mask)
        bp.intrinsics_group = GROUP
        lin = rb.LinearizorQR.create(bp, rb.SolverOptions())
        cam, lm = lin.covariance()
        lin.close()
        assert rel_err(cam, want_cam) < 1e-7, held
        assert rel_err(lm, want_lm) < 1e-7, held
        g = lead >= 0
        assert np.array_equal(cam[g][:, 6:, 6:], cam[lead[g]][:, 6:, 6:])


def _tied_scipy_minimum(prob, group, camera):
    """scipy's least-squares minimum of the tied objective (a pose per camera, f, k1, k2 per group): (cams, lms, cost)"""
    from scipy.optimize import least_squares
    from scipy.spatial.transform import Rotation
    import camera_model as cm
    import camera_prior_model as pm
    lead = sm.leads(group)
    nc, nl = prob.nc, prob.nl
    own = np.flatnonzero((lead < 0) | (lead == np.arange(nc)))  # cameras that carry intrinsics parameters
    slot = {c: k for k, c in enumerate(own)}
    lm_of_obs = np.repeat(np.arange(nl), np.diff(prob.lm_off))
    base = np.asarray(prob.cams, np.float64)

    def unpack(x):
        pose = x[:6 * nc].reshape(nc, 6)
        intr = x[6 * nc:6 * nc + 3 * len(own)].reshape(-1, 3)
        cams = base.copy()
        cams[:, :4] = Rotation.from_rotvec(pose[:, :3]).as_quat()
        cams[:, 4:7] = pose[:, 3:]
        for c in range(nc):
            cams[c, 7:] = intr[slot[c if lead[c] < 0 else lead[c]]]
        return cams, x[6 * nc + 3 * len(own):].reshape(nl, 3)

    def fun(x):
        cams, lms = unpack(x)
        out = [cm.linearize(cams[prob.obs_cam], lms[lm_of_obs], prob.obs_xy)["res"].ravel()]
        out += [camera[1][c] @ pm.residual(cams[c], camera[0][c]) for c in range(nc)]
        return np.concatenate(out)

    x0 = np.concatenate([np.hstack([Rotation.from_quat(base[:, :4]).as_rotvec(), base[:, 4:7]]).ravel(), base[own, 7:].ravel(),
                         np.ravel(prob.lms)])
    sol = least_squares(fun, x0, method="trf", x_scale="jac", xtol=1e-15, ftol=1e-15, gtol=1e-15, max_nfev=300)
    cams, lms = unpack(sol.x)
    return cams, lms, float(sol.cost)


def test_lm_run_reaches_the_scipy_minimum_of_the_tied_objective():
    import rootba_b200 as rb
    from test_gpu_camera_priors import _e2e_problem
    from rootba_b200.synthetic import BalArrays, project
    prob, mean, L = _e2e_problem()
    group = (np.arange(prob.nc) % 3).astype(np.int32)
    lead = sm.leads(group)
    # observations of a scene whose cameras really share intrinsics per group (pixel noise), then a perturbed start
    rng = np.random.default_rng(12)
    truth = np.array(prob.cams, np.float64)
    truth[:, 7:] = truth[lead, 7:]
    lm_of_obs = np.repeat(np.arange(prob.nl), np.diff(prob.lm_off))
    xy, _ = project(truth[prob.obs_cam], np.asarray(prob.lms, np.float64)[lm_of_obs])
    cams = truth.copy()
    cams[:, 4:7] += rng.normal(0, 0.01, (prob.nc, 3))
    cams[:, 7] *= (1 + rng.normal(0, 0.01, prob.nc))[lead]
    prob = BalArrays(cams, np.asarray(prob.lms) + rng.normal(0, 0.01, np.shape(prob.lms)), prob.lm_off, prob.obs_cam,
                     xy + rng.normal(0, 0.5, xy.shape))
    cams_s, lms_s, cost_s = _tied_scipy_minimum(prob, group, (mean, L))
    bp = rb.BalProblem.from_arrays(prob, np.float64)
    bp.camera_prior = (mean, L)
    bp.intrinsics_group = group
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(max_num_iterations=60, function_tolerance=1e-15, eta=1e-10))
    lin.lm_run(200)
    lin.download_state()
    cost = lin.compute_error()["all"]["error"]
    lin.close()
    assert abs(cost - cost_s) <= 1e-9 * cost_s, (cost, cost_s)
    assert np.array_equal(bp.cams[:, 7:], bp.cams[lead, 7:])
    assert rel_err(bp.cams[:, 7:10], cams_s[:, 7:10]) < 1e-6
    assert rel_err(bp.lms, lms_s) < 1e-6


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_more_than_1808_cameras(dtype):
    """1900 cameras in 5 groups and ungrouped ones (several blocks of the per-camera grids of the group kernels): the solve
    satisfies the tied system P^T (H P u) + lambda u = -b_u, with H P u from rba_right_multiply (the full operator, whose
    damping lambda P u is taken out again)"""
    import rootba_b200 as rb
    from rootba_b200.synthetic import synth_bal
    prob = synth_bal(1900, 6000, 4.0, seed=7)
    nc = prob.nc
    group = np.where(np.arange(nc) % 7 == 0, -1, np.arange(nc) % 5).astype(np.int32)
    lead = sm.leads(group)
    bp = rb.BalProblem.from_arrays(prob, dtype)
    bp.intrinsics_group = group
    lam = 1e-2
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(eta=1e-12, max_linear_solver_iterations=2000))
    lin.linearize()
    inc = np.asarray(lin.solve(lam), np.float64)
    b = np.asarray(lin.get_rhs(), np.float64)
    u = np.where(sm.members(lead), 0.0, inc)  # the 9 nc layout of u
    Hx = np.asarray(lin.right_multiply(inc), np.float64)  # (H + lambda I) P u
    res = sm.contract(Hx - lam * inc, lead) + lam * u + b
    assert rel_err(res + b, b) < (1e-5 if dtype == np.float64 else 2e-2), rel_err(res + b, b)
    inc2 = inc.reshape(-1, 9)
    g = lead >= 0
    assert np.array_equal(inc2[g, 6:], inc2[lead[g], 6:])
    assert np.all(b.reshape(-1, 9)[g & (lead != np.arange(nc)), 6:] == 0)
    lin.close()


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_held_flags_and_every_prior_kind(dtype):
    from objective_checks import FIX_F, FIX_K1, FIX_K2, FIX_POSE
    prob, _, model = _case(("camera", "pairs", "landmarks"))
    mask = np.zeros(prob.nc, np.uint8)
    mask[[2, 4, 7]] = FIX_K1 | FIX_K2  # one whole group holds k1, k2
    mask[3] = FIX_POSE | FIX_F
    mask[1] = FIX_POSE
    check_tied_step(PCG_CONFIGS[1], prob, GROUP, model, dtype, mask=mask)


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_members_stay_identical_through_lm_run(small_problem, dtype):
    import rootba_b200 as rb
    nc = small_problem.nc
    group = (np.arange(nc) % 3).astype(np.int32)
    bp = rb.BalProblem.from_arrays(small_problem, dtype)
    bp.intrinsics_group = group
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(max_num_iterations=8))
    its, _, _ = lin.lm_run(64)
    lin.download_state()
    lin.close()
    lead = sm.leads(group)
    assert np.array_equal(bp.cams[:, 7:], bp.cams[lead, 7:])
    acc = [it["cost"] for it in its if it["accepted"]]
    assert len(acc) >= 1 and all(b < a for a, b in zip(acc, acc[1:])), its
    assert not np.array_equal(bp.cams[:, 7:], np.asarray(small_problem.cams, dtype)[:, 7:])


@pytest.mark.parametrize("mode", ["groups_of_one", "set_then_none"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_groups_of_one_and_cleared_groups_change_nothing(small_problem, dtype, mode):
    import rootba_b200 as rb
    from objective_checks import assert_identical_steps, lm_steps
    ref = lm_steps(small_problem, dtype, {}, "never")
    nc = small_problem.nc
    if mode == "groups_of_one":
        got = lm_steps(small_problem, dtype, {}, "zeros", lambda lin, v: lin.set_intrinsics_groups(np.arange(nc, dtype=np.int32)),
                       np.zeros(nc, np.int32))
    else:
        def setter(lin, v):  # setting the groups tied the state; the caller's state is set again after clearing them
            lin.set_intrinsics_groups(v)
            if v is None:
                lin.upload_state()
        got = lm_steps(small_problem, dtype, {}, "set_then_none", setter, np.zeros(nc, np.int32))
    assert_identical_steps(ref, got, mode)


def test_rejected_calls(small_problem):
    import rootba_b200 as rb
    from rootba_b200 import _lib
    L = _lib.lib()
    nc = small_problem.nc
    ptr = lambda a: C.c_void_p(a.ctypes.data)
    lin = rb.LinearizorQR.create(rb.BalProblem.from_arrays(small_problem, np.float64), rb.SolverOptions(solver_type="POWER_SCHUR_COMPLEMENT"))
    g = np.zeros(nc, np.int32)
    assert L.rba_set_intrinsics_groups(lin.h, ptr(g)) == -4  # RBA_ERR_UNSUPPORTED
    assert L.rba_set_intrinsics_groups(lin.h, ptr(np.arange(nc, dtype=np.int32))) == 0  # groups of one are fine
    lin.close()
    bp = rb.BalProblem.from_arrays(small_problem, np.float64)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions())
    group = (np.arange(nc) % 2).astype(np.int32)
    lin.set_intrinsics_groups(group)
    lin.compute_error()
    lin.linearize()
    inc_ref = lin.solve(1e-4)
    for bad in (np.full(nc, nc, np.int32), np.full(nc, -2, np.int32)):
        assert L.rba_set_intrinsics_groups(lin.h, ptr(bad)) == -1  # RBA_ERR_INVALID_ARGUMENT
    flags = np.zeros(nc, np.uint8)
    flags[0] = rb.FIX_F  # camera 0 leads group 0; camera 2 is a member without the bit
    assert L.rba_set_camera_fixed(lin.h, ptr(flags)) == -1
    assert b"camera 2" in L.rba_last_error()
    lin.linearize()  # the failed calls left the groups (and no flags) in force
    assert np.array_equal(lin.solve(1e-4), inc_ref)
    flags[group == 0] = rb.FIX_F
    assert L.rba_set_camera_fixed(lin.h, ptr(flags)) == 0
    assert L.rba_set_intrinsics_groups(lin.h, ptr((np.arange(nc) % 3).astype(np.int32))) == -1  # groups that split the bits
    lin.close()


@pytest.mark.parametrize("sfx", ["f32", "f64"])
def test_two_ranks_with_groups(tmp_path, sfx):
    """two GPUs (skipped with fewer): with groups the hand-over is NCCL whether or not the peers are mapped"""
    from objective_checks import run_two_ranks
    res = run_two_ranks(tmp_path, "multirank_groups_worker.py", sfx, "1", 29500, 3 if sfx == "f32" else 11)
    tols = 1e-4 if sfx == "f32" else 1e-8
    assert res["replicas_identical"] and res["members_identical"] and res["inc_tied"], res
    assert res["b"] < 4 * tols and res["inc"] < tols and res["l_diff"] < 20 * tols, res
    assert res["lms"] < 10 * tols and res["cams"] < tols and res["cost"] < tols and res["cost0"] < tols, res


@pytest.mark.parametrize("use_double", [True, False])
def test_bal_qr_shared_intrinsics_matches_python_host(tmp_path, use_double):
    """bal_qr --shared-intrinsics (C++ BalProblem::intrinsics_group) against the Python host with every camera in one group"""
    import subprocess
    import rootba_b200 as rb
    from oracle import oracle_py as orc
    from rootba_b200.synthetic import BalArrays, synth_bal, write_bal
    from test_host_cpp import BAL_QR, _build, _load_ba_log
    _build()
    prob = synth_bal(20, 400, 4.0, seed=9, normalize_scale=None)
    path = str(tmp_path / "p.txt")
    write_bal(prob, path)
    log = str(tmp_path / "ba_log.json")
    args = [BAL_QR, "--input", path, "--max-num-iterations", "4", "--log-path", log, "--shared-intrinsics"]
    subprocess.check_call(args + ([] if use_double else ["--no-use-double"]), stdout=subprocess.DEVNULL)
    cols, _ = _load_ba_log(log)
    d = orc.load_bal(path, normalize=True)
    arrays = BalArrays(d["cams"], d["lms"], d["lm_off"], d["obs_cam"], d["obs_xy"])
    bp = rb.BalProblem.from_arrays(arrays, np.float64 if use_double else np.float32)
    bp.intrinsics_group = np.zeros(arrays.nc, np.int32)
    summ = rb.bundle_adjust_manual(bp, rb.SolverOptions(max_num_iterations=4))
    assert len(cols["iteration"]) == len(summ["iterations"])
    prev = None
    for k, it in enumerate(summ["iterations"]):
        cb = it["cost"]["all"]["error"] if (it["step_is_successful"] or prev is None) else prev
        prev = cb
        assert abs(cols["cost"][k] - cb) <= (1e-6 if use_double else 5e-3) * cb + 1e-12 * cols["cost"][0]
    free = rb.bundle_adjust_manual(rb.BalProblem.from_arrays(arrays, bp.dtype), rb.SolverOptions(max_num_iterations=4))
    assert free["iterations"][-1]["cost"]["all"]["error"] != summ["iterations"][-1]["cost"]["all"]["error"]
