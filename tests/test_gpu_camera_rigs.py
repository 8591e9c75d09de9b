"""Rigid camera rigs (rba_set_camera_rigs) on the GPU: every PCG solver configuration against the dense float64 model of the
tied problem (tests/camera_rig_model.py), with held rigs, every prior kind and intrinsics groups,
the assembled operator, the members exactly rigid through LM runs, rigs of one and cleared rigs bit-identical to no rigs,
and the rejected calls."""
import numpy as np
import pytest

import camera_rig_model as rm
import shared_intrinsics_model as sm
from conftest import rel_err
from objective_checks import BARS, CONFIGS, FIX_POSE, bal_problem, cfg_id, dense_system, fixed_entries, reduced
from test_camera_rig_model import RIG, rig_case

pytestmark = pytest.mark.gpu

# the C ABI's return codes (include/rootba_b200.h)
INVALID, UNSUPPORTED = -1, -4

PCG_CONFIGS = [c for c in CONFIGS if c["solver_type"] != "POWER_SCHUR_COMPLEMENT"]
PCG_CONFIGS += [dict(solver_type="SQUARE_ROOT", stage2_form="IDENTITY")]
NAMES = {"camera": "camera_prior", "pairs": "camera_pair_prior", "landmarks": "landmark_prior"}


def check_rig_step(cfg, prob, rig, E, model, dtype=np.float64, mask=None, group=None, lam=1e-3, env=None, obs=None):
    """one LM step of a handle with rigs against the dense model of the tied problem, evaluated at the state the handle
    re-tied: the scaling, b, the preconditioner inverse (without intrinsics groups), the increment, l_diff and the state
    after apply (members at M_j T_lead).  obs: (loss kind, loss scale, sqrt_info) per observation"""
    import rootba_b200 as rb
    from rootba_b200.synthetic import BalArrays
    bars = BARS[dtype]
    f = lambda a: np.asarray(np.asarray(a, dtype), np.float64)
    bp = bal_problem(prob, dtype, camera_fixed=mask, **{NAMES[k]: v for k, v in model.items()})
    if group is not None:
        bp.intrinsics_group = group
    if obs is not None:
        bp.observation_sqrt_info = obs[2]
        bp.observation_loss = (obs[0], obs[1])
    bp.camera_rig = (rig, E)
    with pytest.MonkeyPatch.context() as m:
        for k, v in (env or {}).items():
            m.setenv(k, v)
        lin = rb.LinearizorQR.create(bp, rb.SolverOptions(eta=1e-13, **cfg))
    lin.download_state()
    lead = rm.leads(rig)
    glead = None if group is None else sm.leads(group)
    M = rm.maps(f(E), lead)
    cams0 = np.array(bp.cams, np.float64)
    for c in np.flatnonzero((lead >= 0) & (lead != np.arange(len(lead)))):  # the call re-tied the members
        assert rel_err(rm.compose(M[c], cams0[lead[c]], cams0[c]), cams0[c]) < (1e-14 if dtype == np.float64 else 1e-6), c
    sprob = BalArrays(cams0, f(prob.lms), prob.lm_off, prob.obs_cam, f(prob.obs_xy))
    smodel = {k: (tuple(v[:-2]) + (f(v[-2]), f(v[-1]))) for k, v in model.items()}
    Jp, Jl, r = dense_system(sprob, **smodel)
    if obs is not None:  # the reprojection rows weighted by each observation's information and loss
        import observation_loss_model as lm
        Jp, Jl, r = Jp.copy(), Jl.copy(), r.copy()
        Jpo, Jlo, ro = lm.dense_system(sprob, obs[0], obs[1], obs[2])
        no = len(ro)
        Jp[:no], Jl[:no], r[:no] = Jpo, Jlo, ro
    Dcam = sm.tied_step(Jp, Jl, r, lam, prob.nl, glead if glead is not None else np.full(prob.nc, -1), dtype)[0]
    P = rm.expansion(lead, M, glead)
    Du, sl, _, Jls, Minv, Hu, bu = reduced(Jp @ P, Jl, r, lam, prob.nl, dtype)
    fixed9 = fixed_entries(mask) if mask is not None else np.zeros(9 * prob.nc, bool)
    keep = np.flatnonzero(~rm.held(lead, glead))
    fu = ~fixed9[keep]
    e0 = lin.compute_error()["all"]["error"]
    lin.linearize()
    inc = lin.solve(lam)
    s, _ = lin.get_jacobian_scaling()
    assert rel_err(s, Dcam) < bars["scaling"]
    assert rel_err(lin.get_rhs(), np.where(fixed9, 0.0, rm.embed(lead, glead) @ bu)) < bars["b"]
    if group is None:  # the merged blocks sum_j P~_j^T B_j P~_j: the device's inverse against the model's
        Jps = Jp * Dcam
        jacobi = cfg.get("preconditioner_type") == "JACOBI"
        if jacobi:
            src = Jps.T @ Jps
        else:
            W = Jps.T @ Jls
            src = Jps.T @ Jps - W @ Minv @ W.T
        blocks = np.stack([src[9 * c:9 * c + 9, 9 * c:9 * c + 9] for c in range(prob.nc)])
        want_inv = rm.device_blocks(blocks, lam, lead, rm.scaled_map(P, Dcam, Du), fixed9)
        inv, _ = lin.get_preconditioner()
        for c in range(prob.nc):
            assert rel_err(inv[c], want_inv[c]) < bars["inv"], c
    Hff = Hu[np.ix_(fu, fu)]
    u = np.zeros(len(bu))
    u[fu] = -np.linalg.solve(Hff, bu[fu])
    tol = bars["inc"] if dtype == np.float64 else max(bars["inc"], 100 * 2.0 ** -24 * np.linalg.cond(Hff))
    want_inc = (P @ (Du * u)) / Dcam
    assert rel_err(inc, want_inc) < tol
    inc64 = np.asarray(inc, np.float64)
    Jps = Jp * Dcam
    dl_s = -Minv @ (Jls.T @ r + Jls.T @ (Jps @ inc64))
    want_l = 0.5 * r @ r - 0.5 * np.sum((r + Jps @ inc64 + Jls @ dl_s) ** 2)
    l_diff = lin.apply(None)
    assert abs(l_diff - want_l) <= bars["l_diff"] * abs(want_l)
    lin.download_state()
    want_cams = rm.apply_tied(cams0, Dcam * inc64, lead, M)
    sgn = lambda c: np.c_[c[:, :4] * np.sign(c[:, 3:4]), c[:, 4:]]  # q and -q are one rotation
    assert rel_err(sgn(np.asarray(bp.cams, np.float64)), sgn(want_cams)) < (1e-9 if dtype == np.float64 else 2e-4)
    check_rigid(bp.cams, lead, M, dtype)
    assert rel_err(bp.lms, sprob.lms + (sl * dl_s).reshape(-1, 3)) < bars["lms"]
    assert e0 > 0
    lin.close()


def check_rigid(cams, lead, M, dtype):
    """every member's pose relative to its lead equals M_j at the scalar's rounding"""
    u = 1e-15 if dtype == np.float64 else 1e-6
    cams = np.asarray(cams, np.float64)
    for c in np.flatnonzero((lead >= 0) & (lead != np.arange(len(lead)))):
        q, t = rm.relative(cams[c], cams[lead[c]])
        q *= np.sign(q[3]) * np.sign(M[c, 3])
        scale = 1.0 + np.linalg.norm(cams[lead[c], 4:7])
        assert np.max(np.abs(q - M[c, :4])) < 20 * u and np.max(np.abs(t - M[c, 4:])) < 20 * u * scale, c


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("cfg", PCG_CONFIGS, ids=cfg_id)
def test_every_solver_against_the_tied_model(cfg, dtype):
    prob, _, _, E, model = rig_case(("camera",))
    check_rig_step(cfg, prob, RIG, E, model, dtype)


@pytest.mark.parametrize("layout", ["two", "six", "all_in_one", "lead_without_observations"])
def test_rig_layouts(layout):
    prob, _, _, E, model = rig_case(("camera",))
    nc = prob.nc
    if layout == "two":
        rig = (np.arange(nc) // 2).astype(np.int32)
    elif layout == "six":
        rig = np.where(np.arange(nc) < 6, 0, -1).astype(np.int32)
    elif layout == "all_in_one":
        rig = np.zeros(nc, np.int32)
    else:  # camera 7 (no observations) leads rig {7 -> first, 1, 2} after a reorder
        from rootba_b200.synthetic import BalArrays
        cams = np.vstack([prob.cams[-1:], prob.cams[:-1]])
        prob = BalArrays(cams, prob.lms, prob.lm_off, (np.asarray(prob.obs_cam) + 1).astype(np.int32), prob.obs_xy)
        model = {"camera": (np.vstack([model["camera"][0][-1:], model["camera"][0][:-1]]),
                            np.concatenate([model["camera"][1][-1:], model["camera"][1][:-1]]))}
        rig = np.full(nc, -1, np.int32)
        rig[[0, 2, 5]] = 4
    for cfg in (PCG_CONFIGS[0], PCG_CONFIGS[-2]):
        check_rig_step(cfg, prob, rig, E, model)


def test_assembled_operator_with_damping():
    """RBA_ASSEMBLED_AT=2: S is built and the solve switches to it from iteration 2"""
    prob, _, _, E, model = rig_case(("camera",))
    check_rig_step(PCG_CONFIGS[0], prob, RIG, E, model, lam=1e-2, env={"RBA_ASSEMBLED_AT": "2"})


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("with_obs", [False, True], ids=["priors", "priors-obs-info-loss"])
def test_held_rig_as_gauge_with_every_prior(dtype, with_obs):
    """a held rig as the gauge with camera, pair (inside and across rigs) and landmark priors, and with observation
    information and robust losses per observation"""
    import observation_info_model as om
    import observation_loss_model as lm
    prob, _, _, E, model = rig_case(("camera", "pairs", "landmarks"))
    mask = np.zeros(prob.nc, np.uint8)
    mask[[2, 3, 4]] = FIX_POSE
    nobs = len(prob.obs_cam)
    obs = None
    if with_obs:
        kind, scale = lm.mixed(nobs, 8, kinds=(lm.NONE, lm.HUBER, lm.CAUCHY, lm.SOFT_L1), lo=20.0, hi=60.0)
        obs = (kind, scale, om.random_info(nobs, 9))
    for cfg in (PCG_CONFIGS[0], PCG_CONFIGS[3], PCG_CONFIGS[-2]):
        check_rig_step(cfg, prob, RIG, E, model, dtype, mask=mask, obs=obs)


def test_rigs_with_intrinsics_groups():
    prob, _, _, E, model = rig_case(("camera", "pairs"))
    group = np.array([0, 0, -1, 0, 5, 5, -1, 5], np.int32)
    glead = sm.leads(group)
    cams = np.array(prob.cams)
    g = glead >= 0
    cams[g, 7:] = cams[glead[g], 7:]
    from rootba_b200.synthetic import BalArrays
    prob = BalArrays(cams, prob.lms, prob.lm_off, prob.obs_cam, prob.obs_xy)
    for cfg in (PCG_CONFIGS[0], PCG_CONFIGS[1], PCG_CONFIGS[-2]):
        check_rig_step(cfg, prob, RIG, E, model, group=group)


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_members_stay_rigid_through_lm_runs(dtype):
    """the relative pose of every member to its lead is M_j at the scalar's rounding after 1 and after 20 iterations"""
    import rootba_b200 as rb
    from rootba_b200.synthetic import synth_bal
    arrays = synth_bal(60, 1500, 4.0, seed=11)
    nc = arrays.cams.shape[0]
    rig = (np.arange(nc) // 3).astype(np.int32)
    E = rm.extrinsics_from_state(arrays.cams, rig)
    lead = rm.leads(rig)
    M = rm.maps(np.asarray(np.asarray(E, dtype), np.float64), lead)
    for its in (1, 20):
        bp = rb.BalProblem.from_arrays(arrays, dtype)
        bp.camera_rig = (rig, E)
        lin = rb.LinearizorQR.create(bp, rb.SolverOptions())
        e0 = lin.compute_error()["all"]["error"]
        lin.lm_run(its)
        lin.download_state()
        check_rigid(bp.cams, lead, M, dtype)
        assert lin.compute_error()["all"]["error"] < e0
        lin.close()


def test_many_cameras():
    """> 1808 cameras (the counter hand-over of the plain path): the step is finite and lowers the cost, members rigid"""
    import rootba_b200 as rb
    from rootba_b200.synthetic import synth_bal
    arrays = synth_bal(1900, 6000, 3.0, seed=5)
    nc = arrays.cams.shape[0]
    rig = (np.arange(nc) // 4).astype(np.int32)
    E = rm.extrinsics_from_state(arrays.cams, rig)
    bp = rb.BalProblem.from_arrays(arrays, np.float64)
    bp.camera_rig = (rig, E)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions())
    e0 = lin.compute_error()["all"]["error"]
    lin.lm_run(3)
    lin.download_state()
    check_rigid(bp.cams, rm.leads(rig), rm.maps(E, rm.leads(rig)), np.float64)
    assert lin.compute_error()["all"]["error"] < e0
    lin.close()


def _steps(arrays, dtype, setup, steps=3):
    import rootba_b200 as rb
    bp = rb.BalProblem.from_arrays(arrays, dtype)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions())
    setup(lin)
    out = []
    for _ in range(steps):
        before = lin.timings()["kernel_launches"]  # the handle's total: the launches of this step
        lin.linearize()
        inc = lin.solve(1e-4)
        l_diff = lin.apply(None)
        launches = lin.timings()["kernel_launches"] - before
        lin.download_state()
        out.append((inc.copy(), l_diff, bp.cams.copy(), bp.lms.copy(), launches, lin.compute_error()["all"]["error"]))
    lin.close()
    return out


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_rigs_of_one_and_cleared_rigs_are_bit_identical(dtype):
    from rootba_b200.synthetic import synth_bal
    arrays = synth_bal(30, 800, 4.0, seed=3)
    nc = arrays.cams.shape[0]
    E = rm.rig_case(nc)
    ref = _steps(arrays, dtype, lambda lin: None)
    for what, setup in [("one", lambda lin: lin.set_camera_rigs(np.arange(nc, dtype=np.int32), E)),
                        ("free", lambda lin: lin.set_camera_rigs(np.full(nc, -1, np.int32), E)),
                        ("cleared", lambda lin: (lin.set_camera_rigs((np.arange(nc) // 2).astype(np.int32), E),
                                                 lin.set_camera_rigs(None), lin.upload_state()))]:
        got = _steps(arrays, dtype, setup)
        for a, b in zip(ref, got):
            assert np.array_equal(a[0], b[0]) and a[1] == b[1] and a[4] == b[4] and a[5] == b[5], what
            assert np.array_equal(a[2], b[2]) and np.array_equal(a[3], b[3]), what


def test_rejected_calls():
    import ctypes as C
    import rootba_b200 as rb
    from rootba_b200 import _lib
    prob, _, _, E, _ = rig_case()
    bp = rb.BalProblem.from_arrays(prob, np.float64)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions())
    L = _lib.lib()
    rig = np.ascontiguousarray(RIG)
    e = np.ascontiguousarray(E, np.float64)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    assert L.rba_set_camera_rigs(lin.h, p(rig), None) == INVALID
    assert L.rba_set_camera_rigs(lin.h, None, p(e)) == INVALID
    bad = rig.copy(); bad[1] = prob.nc
    assert L.rba_set_camera_rigs(lin.h, p(bad), p(e)) == INVALID
    bad = rig.copy(); bad[1] = -2
    assert L.rba_set_camera_rigs(lin.h, p(bad), p(e)) == INVALID
    be = e.copy(); be[1, 5] = np.inf
    assert L.rba_set_camera_rigs(lin.h, p(rig), p(be)) == INVALID
    be = e.copy(); be[1, :4] *= 1.01
    assert L.rba_set_camera_rigs(lin.h, p(rig), p(be)) == INVALID
    be = e.copy(); be[5, :] = np.nan  # a free camera's entries are ignored
    assert L.rba_set_camera_rigs(lin.h, p(rig), p(be)) == _lib.RBA_OK
    # differing RBA_FIX_POSE bits within a rig, in both orders
    mask = np.zeros(prob.nc, np.uint8); mask[2] = FIX_POSE
    with pytest.raises(_lib.RbaError):
        lin.set_camera_fixed(mask)
    lin.set_camera_rigs(None)
    lin.set_camera_fixed(mask)
    with pytest.raises(_lib.RbaError):
        lin.set_camera_rigs(RIG, E)
    lin.set_camera_fixed(None)
    # a call after a set needs a new linearize
    lin.linearize(); lin.solve(1e-3)
    lin.set_camera_rigs(RIG, E)
    with pytest.raises(_lib.RbaError, match="error -6"):
        lin.solve(1e-3)
    lin.close()
    bp = rb.BalProblem.from_arrays(prob, np.float64)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(solver_type="POWER_SCHUR_COMPLEMENT"))
    assert L.rba_set_camera_rigs(lin.h, p(rig), p(e)) == UNSUPPORTED
    lin.close()


@pytest.mark.parametrize("precond", ["JACOBI", "SCHUR_JACOBI"])
@pytest.mark.parametrize("sfx", ["f32", "f64"])
def test_two_ranks_with_rigs(tmp_path, sfx, precond):
    """two GPUs (skipped with fewer): the NCCL hand-over with the rig contraction, and with SCHUR_JACOBI the cross-rank sum of
    the blocks D_u is built from; the sharded step equals the single-rank one, the cameras are bit-identical on both ranks and
    every member is at M_j T_lead"""
    from objective_checks import run_two_ranks
    res = run_two_ranks(tmp_path, "multirank_camera_rigs_worker.py", sfx, "1", 29500, (5 if sfx == "f32" else 13) + (0 if precond == "JACOBI" else 2),
                        precond)
    tols = 1e-4 if sfx == "f32" else 1e-8
    assert res["replicas_identical"] and res["rigid"] < 20, res
    assert res["b"] < 4 * tols and res["inc"] < tols and res["l_diff"] < 20 * tols, res
    assert res["lms"] < 10 * tols and res["cams"] < tols and res["cost"] < tols and res["cost0"] < tols, res


def test_lm_run_reaches_a_stationary_point_of_the_tied_objective():
    """rba_lm_run to convergence: the gradient of the tied objective, P^T J^T r of the dense model at the final state, is zero
    relative to its start (the first-order condition of the tied minimum), and the members are rigid"""
    import rootba_b200 as rb
    from rootba_b200.synthetic import BalArrays
    import camera_prior_model as pm
    prob, mean, L = pm.prior_case()
    model = {"camera": (mean, L)}
    E = rm.extrinsics_from_state(prob.cams, RIG)  # rigs consistent with the start: LM converges in a few steps
    lead = rm.leads(RIG)
    M = rm.maps(E, lead)
    bp = bal_problem(prob, np.float64, camera_prior=model["camera"])
    bp.camera_rig = (RIG, E)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(max_num_iterations=60, function_tolerance=1e-15, eta=1e-10))
    lin.download_state()

    def gradient(b):
        p = BalArrays(np.array(b.cams, np.float64), np.array(b.lms, np.float64), prob.lm_off, prob.obs_cam, prob.obs_xy)
        Jp, Jl, r = dense_system(p, **model)
        return np.r_[rm.expansion(lead, M).T @ (Jp.T @ r), Jl.T @ r]
    g0 = np.linalg.norm(gradient(bp))
    lin.lm_run(200)
    lin.download_state()
    check_rigid(bp.cams, lead, M, np.float64)
    assert np.linalg.norm(gradient(bp)) < 1e-6 * g0
    lin.close()


def test_covariance_is_that_of_the_tied_problem():
    """rba_compute_covariance and rba_compute_covariance_blocks against the dense inverse of the tied system, the gauge fixed
    by the camera priors (and a held rig); the relative-pose covariance of two members of one rig is 0 to rounding"""
    import rootba_b200 as rb
    prob, lead, M, E, model = rig_case(("camera", "landmarks"))
    Jp, Jl, _ = dense_system(prob, **model)
    for held in (False, True):
        mask = None
        if held:
            mask = np.zeros(prob.nc, np.uint8)
            mask[[0, 1]] = FIX_POSE
        want_cam, want_lm, _ = rm.tied_covariance(Jp, Jl, lead, M, fixed_entries(mask) if held else None)
        bp = bal_problem(prob, np.float64, camera_prior=model["camera"], landmark_prior=model["landmarks"], camera_fixed=mask)
        bp.camera_rig = (RIG, E)
        lin = rb.LinearizorQR.create(bp, rb.SolverOptions())
        cam, lm_ = lin.covariance()
        assert rel_err(cam, want_cam) < 1e-7, held
        assert rel_err(lm_, want_lm) < 1e-7, held
        got = lin.covariance_blocks(cameras=[[2, 4], [0, 5]], relative=[[2, 4], [3, 2], [1, 5]])
        _, _, full = rm.tied_covariance(Jp, Jl, lead, M, fixed_entries(mask) if held else None)
        assert rel_err(got["cameras"][0], full[18:27, 36:45]) < 1e-7 and rel_err(got["cameras"][1], full[0:9, 45:54]) < 1e-7
        scale = np.max(np.abs(got["relative"][2]))
        assert scale > 0 and np.max(np.abs(got["relative"][:2])) < 1e-9 * max(scale, np.max(np.abs(cam))), got["relative"][:2]
        lin.close()
