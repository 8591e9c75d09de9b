"""Estimated rig extrinsics (rba_set_rig_sensors) on the GPU: every PCG configuration in both precisions and the assembled
operator against the dense float64 model of the tied problem (tests/rig_sensor_model.py), with every prior kind, observation
information and losses, held rigs and intrinsics groups; rba_get_rig_extrinsics; the inc_out round trip; backup / restore;
the cameras of a sensor tied through LM runs at 8 and 1900 cameras; NULL and cleared sensors bit-identical to rigs alone;
the rejected calls; both covariance entry points; and the recovery of true extrinsics from a perturbed start."""
import numpy as np
import pytest

import camera_rig_model as rm
import rig_sensor_model as sn
import shared_intrinsics_model as sm
from conftest import rel_err
from objective_checks import BARS, CONFIGS, FIX_POSE, bal_problem, cfg_id, dense_system, fixed_entries, reduced
from test_camera_rig_model import RIG
from test_rig_sensor_model import SENSOR, _with_cams
from test_camera_rig_model import rig_case

pytestmark = pytest.mark.gpu

INVALID = -1
PCG_CONFIGS = [c for c in CONFIGS if c["solver_type"] != "POWER_SCHUR_COMPLEMENT"]
PCG_CONFIGS += [dict(solver_type="SQUARE_ROOT", stage2_form="IDENTITY")]
NAMES = {"camera": "camera_prior", "pairs": "camera_pair_prior", "landmarks": "landmark_prior"}
sgn = lambda c: np.c_[c[:, :4] * np.sign(c[:, 3:4]), c[:, 4:]]  # q and -q are one rotation


def _handle(cfg, prob, E, model, dtype, sensor=SENSOR, mask=None, group=None, obs=None, env=None):
    import rootba_b200 as rb
    bp = bal_problem(prob, dtype, camera_fixed=mask, **{NAMES[k]: v for k, v in model.items()})
    if group is not None:
        bp.intrinsics_group = group
    if obs is not None:
        bp.observation_sqrt_info = obs[2]
        bp.observation_loss = (obs[0], obs[1])
    bp.camera_rig = (RIG, E)
    bp.rig_sensor = sensor
    with pytest.MonkeyPatch.context() as m:
        for k, v in (env or {}).items():
            m.setenv(k, v)
        lin = rb.LinearizorQR.create(bp, rb.SolverOptions(eta=1e-13, **cfg))
    return bp, lin


def check_sensor_step(cfg, prob, E, model, dtype=np.float64, sensor=SENSOR, mask=None, group=None, lam=1e-3, env=None,
                      obs=None, move_home=True):
    """one LM step with sensors against the dense model of the tied problem at the state the handle tied: the scaling, b,
    the preconditioner inverse (without intrinsics groups: the sensors' blocks sum_j Q~_j B_j Q~_j in their homes' slots,
    the homes free under a held rig), the increment, l_diff, the state after apply (re-tied), the landmarks and
    rba_get_rig_extrinsics"""
    bars = BARS[dtype]
    f = lambda a: np.asarray(np.asarray(a, dtype), np.float64)
    bp, lin = _handle(cfg, prob, E, model, dtype, sensor, mask, group, obs, env)
    lead, home = sn.structure(RIG, sensor)
    E64 = f(E)
    lin.download_state()
    cams0 = np.array(bp.cams, np.float64)
    want0 = sn.tie_at_call(f(prob.cams), lead, home, E64)
    assert rel_err(sgn(cams0[:, :7]), sgn(want0[:, :7])) < (1e-13 if dtype == np.float64 else 1e-6)
    if move_home:  # E_s away from the given extrinsics: the sensors' homes turned and shifted, then re-tied by set_state
        import camera_prior_model as pm
        for h in np.unique(home[home >= 0]):
            cams0[h] = pm.apply_inc(cams0[h], np.r_[0.01, -0.02, 0.005, 0.02, -0.01, 0.015, 0, 0, 0])
        bp.cams[:] = cams0
        lin.upload_state()
        lin.download_state()
        cams0 = np.array(bp.cams, np.float64)
        assert rel_err(sgn(cams0[:, :7]), sgn(sn.retie(cams0, lead, home, E64)[:, :7])) < (1e-13 if dtype == np.float64 else 1e-6)
    glead = None if group is None else sm.leads(group)
    sprob = _with_cams(prob, cams0)
    sprob.lms = f(prob.lms)
    sprob.obs_xy = f(prob.obs_xy)
    smodel = {k: (tuple(v[:-2]) + (f(v[-2]), f(v[-1]))) for k, v in model.items()}
    Jp, Jl, r = dense_system(sprob, **smodel)
    if obs is not None:
        import observation_loss_model as lm
        Jp, Jl, r = Jp.copy(), Jl.copy(), r.copy()
        Jpo, Jlo, ro = lm.dense_system(sprob, obs[0], obs[1], obs[2])
        no = len(ro)
        Jp[:no], Jl[:no], r[:no] = Jpo, Jlo, ro
    Dcam = sm.tied_step(Jp, Jl, r, lam, prob.nl, glead if glead is not None else np.full(prob.nc, -1), dtype)[0]
    M = sn.maps(cams0, lead, home, E64)
    P = sn.expansion(lead, home, M, glead)
    Du, sl, _, Jls, Minv, Hu, bu = reduced(Jp @ P, Jl, r, lam, prob.nl, dtype)
    fixed9 = fixed_entries(mask) if mask is not None else np.zeros(9 * prob.nc, bool)
    fixed9 = fixed9.reshape(-1, 9)
    fixed9[home >= 0, :6] = False  # a held rig does not hold its sensor cameras
    fixed9 = fixed9.ravel()
    keep = np.flatnonzero(~sn.held(lead, home, glead))
    fu = ~fixed9[keep]
    lin.linearize()
    inc = lin.solve(lam)
    s, _ = lin.get_jacobian_scaling()
    assert rel_err(s, Dcam) < bars["scaling"]
    assert rel_err(lin.get_rhs(), np.where(fixed9, 0.0, sn.embed(lead, home, glead) @ bu)) < bars["b"]
    if group is None:
        Jps = Jp * Dcam
        if cfg.get("preconditioner_type") == "JACOBI":
            src = Jps.T @ Jps
        else:
            W = Jps.T @ Jls
            src = Jps.T @ Jps - W @ Minv @ W.T
        blocks = np.stack([src[9 * c:9 * c + 9, 9 * c:9 * c + 9] for c in range(prob.nc)])
        want_inv = sn.device_blocks(blocks, lam, lead, home, (P * Du[None, :]) / Dcam[:, None], fixed9)
        inv, _ = lin.get_preconditioner()
        for c in range(prob.nc):
            assert rel_err(inv[c], want_inv[c]) < bars["inv"], c
        assert np.max(np.abs(want_inv[home[home >= 0]][:, :6, :6])) > 0  # the homes' slots carry their sensors' blocks
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
    want_cams = sn.apply_tied(cams0, Dcam * inc64, lead, home, E64)
    got = np.asarray(bp.cams, np.float64)
    assert rel_err(sgn(got), sgn(want_cams)) < (1e-9 if dtype == np.float64 else 2e-4)
    check_tied(got, lead, home, E64, dtype)
    assert rel_err(bp.lms, sprob.lms + (sl * dl_s).reshape(-1, 3)) < bars["lms"]
    ext = np.asarray(lin.rig_extrinsics(), np.float64)
    want_ext = sn.sensor_extrinsics(got, lead, home, E64)
    assert rel_err(sgn(ext), sgn(want_ext)) < (1e-12 if dtype == np.float64 else 1e-5)
    lin.close()
    return inc


def check_tied(cams, lead, home, E, dtype):
    """every held member at M_j T_lead and every sensor camera at E_s E_lead^-1 T_lead, at the scalar's rounding"""
    u = 1e-15 if dtype == np.float64 else 1e-6
    cams = np.asarray(cams, np.float64)
    M = sn.maps(cams, lead, home, E)
    for c in np.flatnonzero((lead >= 0) & (lead != np.arange(len(lead))) & (home != np.arange(len(lead)))):
        q, t = rm.relative(cams[c], cams[lead[c]])
        q *= np.sign(q[3]) * np.sign(M[c, 3])
        scale = 1.0 + np.linalg.norm(cams[lead[c], 4:7]) + np.linalg.norm(cams[home[c], 4:7]) if home[c] >= 0 else \
            1.0 + np.linalg.norm(cams[lead[c], 4:7])
        assert np.max(np.abs(q - M[c, :4])) < 50 * u and np.max(np.abs(t - M[c, 4:])) < 50 * u * scale, c


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("cfg", PCG_CONFIGS, ids=cfg_id)
def test_every_solver_against_the_tied_model(cfg, dtype):
    prob, _, _, E, model = rig_case(("camera", "pairs"))
    check_sensor_step(cfg, prob, E, model, dtype)


def test_assembled_operator_with_damping():
    prob, _, _, E, model = rig_case(("camera",))
    check_sensor_step(PCG_CONFIGS[0], prob, E, model, lam=1e-2, env={"RBA_ASSEMBLED_AT": "2"})


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("with_obs", [False, True], ids=["priors", "priors-obs-info-loss"])
def test_held_rig_with_every_prior(dtype, with_obs):
    """rig {2, 3, 4} held (its sensor cameras still move with their sensors) with camera, pair (a lead and a sensor camera
    among them) and landmark priors, and with observation information and robust losses"""
    import observation_info_model as om
    import observation_loss_model as lm
    prob, _, _, E, model = rig_case(("camera", "pairs", "landmarks"))
    mask = np.zeros(prob.nc, np.uint8)
    mask[[2, 3, 4]] = FIX_POSE
    obs = None
    if with_obs:
        nobs = len(prob.obs_cam)
        kind, scale = lm.mixed(nobs, 8, kinds=(lm.NONE, lm.HUBER, lm.CAUCHY, lm.SOFT_L1), lo=20.0, hi=60.0)
        obs = (kind, scale, om.random_info(nobs, 9))
    for cfg in (PCG_CONFIGS[0], PCG_CONFIGS[3], PCG_CONFIGS[-2]):
        check_sensor_step(cfg, prob, E, model, dtype, mask=mask, obs=obs)


@pytest.mark.parametrize("layout", ["one_capture_without_observations", "home_in_the_last_rig", "captures_in_every_rig"])
def test_sensor_layouts(layout):
    prob, _, _, E, model = rig_case(("camera",))
    sensor = {"one_capture_without_observations": np.array([-1, -1, -1, -1, -1, -1, -1, 4], np.int32),
              "home_in_the_last_rig": np.array([-1, 2, -1, -1, -1, -1, 2, -1], np.int32),  # rig {6, 7} led by camera 7
              "captures_in_every_rig": np.array([-1, 0, -1, 0, 1, -1, -1, 0], np.int32)}[layout]
    for cfg in (PCG_CONFIGS[0], PCG_CONFIGS[-2]):
        check_sensor_step(cfg, prob, E, model, sensor=sensor)


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_pair_priors_between_captures_of_one_sensor(dtype):
    """pair priors between two captures of sensor 0 (their cross terms in D_s), a lead and a capture, and two rigs, for both
    block-Jacobi preconditioners"""
    from test_rig_sensor_model import _pair_model
    prob, _, _, E, _ = rig_case()
    model = _pair_model(prob, ("camera", "pairs"))
    for cfg in (PCG_CONFIGS[0], PCG_CONFIGS[1], PCG_CONFIGS[3]):
        check_sensor_step(cfg, prob, E, model, dtype)


def test_sensors_with_intrinsics_groups():
    prob, _, _, E, model = rig_case(("camera", "pairs"))
    group = np.array([0, 0, -1, 0, 5, 5, -1, 5], np.int32)
    glead = sm.leads(group)
    cams = np.array(prob.cams)
    g = glead >= 0
    cams[g, 7:] = cams[glead[g], 7:]
    prob = _with_cams(prob, cams)
    for cfg in (PCG_CONFIGS[0], PCG_CONFIGS[1], PCG_CONFIGS[-2]):
        check_sensor_step(cfg, prob, E, model, group=group)


def test_inc_out_round_trip_and_backup_restore():
    """the increment rba_solve returns, given back to rba_apply, gives the device-resident step bit for bit; backup / restore
    brings the state back bit for bit"""
    prob, _, _, E, model = rig_case(("camera", "pairs"))
    outs = []
    for host in (False, True):
        bp, lin = _handle(PCG_CONFIGS[0], prob, E, model, np.float64)
        lin.linearize()
        inc = lin.solve(1e-3)
        lin._backup()
        lin.download_state()
        before = bp.cams.copy()
        l_diff = lin.apply(inc if host else None)
        lin.download_state()
        outs.append((l_diff, bp.cams.copy()))
        lin._restore()
        lin.download_state()
        assert np.array_equal(bp.cams, before)
        lin.close()
    assert abs(outs[0][0] - outs[1][0]) <= 1e-12 * abs(outs[0][0])
    assert rel_err(outs[0][1], outs[1][1]) < 1e-13


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_sensor_cameras_stay_tied_through_lm_runs(dtype):
    import rootba_b200 as rb
    cap = _capture(4, 15, 1500, seed=11)
    for its in (1, 20):
        bp = rb.BalProblem.from_arrays(cap.prob, dtype)
        bp.camera_rig = (cap.rig, cap.cam_from_rig)
        sensor = np.where(cap.sensor == 0, -1, cap.sensor).astype(np.int32)
        bp.rig_sensor = sensor
        lin = rb.LinearizorQR.create(bp, rb.SolverOptions())
        e0 = lin.compute_error()["all"]["error"]
        lin.lm_run(its)
        lin.download_state()
        lead, home = sn.structure(cap.rig, sensor)
        check_tied(bp.cams, lead, home, np.asarray(np.asarray(cap.cam_from_rig, dtype), np.float64), dtype)
        assert lin.compute_error()["all"]["error"] <= e0
        lin.close()


def _capture(K, F, nl, seed, perturb=True):
    """a rig capture with perturbed landmarks and rig poses (so that LM has work to do)"""
    from rootba_b200.synthetic import synth_rig_capture
    cap = synth_rig_capture(K, F, nl, seed=seed, max_depth=8.0)
    if perturb:
        rng = np.random.default_rng(seed)
        cap.prob.lms += rng.normal(0, 0.01, cap.prob.lms.shape)
    return cap


def test_many_cameras():
    """1900 cameras (the counter hand-over): the step lowers the cost and the sensor cameras stay tied"""
    import rootba_b200 as rb
    cap = _capture(5, 380, 20000, seed=5)
    bp = rb.BalProblem.from_arrays(cap.prob, np.float64)
    bp.camera_rig = (cap.rig, cap.cam_from_rig)
    sensor = np.where(cap.sensor == 0, -1, cap.sensor).astype(np.int32)
    bp.rig_sensor = sensor
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions())
    e0 = lin.compute_error()["all"]["error"]
    lin.lm_run(3)
    lin.download_state()
    lead, home = sn.structure(cap.rig, sensor)
    check_tied(bp.cams, lead, home, cap.cam_from_rig, np.float64)
    assert lin.compute_error()["all"]["error"] < e0
    lin.close()


def _steps(arrays, rig, E, dtype, setup, steps=3):
    import rootba_b200 as rb
    bp = rb.BalProblem.from_arrays(arrays, dtype)
    bp.camera_rig = (rig, E)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions())
    setup(lin)
    out = []
    for _ in range(steps):
        before = lin.timings()["kernel_launches"]
        lin.linearize()
        inc = lin.solve(1e-4)
        l_diff = lin.apply(None)
        launches = lin.timings()["kernel_launches"] - before
        lin.download_state()
        out.append((inc.copy(), l_diff, bp.cams.copy(), bp.lms.copy(), launches, lin.compute_error()["all"]["error"]))
    lin.close()
    return out


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_null_and_cleared_sensors_are_bit_identical_to_rigs_alone(dtype):
    cap = _capture(3, 10, 800, seed=3)
    nc = cap.prob.nc
    ref = _steps(cap.prob, cap.rig, cap.cam_from_rig, dtype, lambda lin: None)
    sensor = np.where(cap.sensor == 0, -1, cap.sensor).astype(np.int32)
    for what, setup in [("null", lambda lin: lin.set_rig_sensors(None)),
                        ("all_held", lambda lin: lin.set_rig_sensors(np.full(nc, -1, np.int32))),
                        ("cleared", lambda lin: (lin.set_rig_sensors(sensor), lin.set_rig_sensors(None)))]:
        got = _steps(cap.prob, cap.rig, cap.cam_from_rig, dtype, setup)
        for a, b in zip(ref, got):
            assert np.array_equal(a[0], b[0]) and a[1] == b[1] and a[4] == b[4] and a[5] == b[5], what
            assert np.array_equal(a[2], b[2]) and np.array_equal(a[3], b[3]), what


def test_rejected_calls_keep_the_previous_sensors():
    import ctypes as C
    import rootba_b200 as rb
    from rootba_b200 import _lib
    prob, _, _, E, model = rig_case(("camera",))
    bp, lin = _handle(PCG_CONFIGS[0], prob, E, model, np.float64)
    L = _lib.lib()
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    ext0 = lin.rig_extrinsics()
    lin.download_state()
    cams0 = bp.cams.copy()
    for bad in (np.r_[SENSOR[:7], 8], np.r_[SENSOR[:7], -2], np.array([-1, 0, -1, 0, 1, 3, -1, 1]),
                np.array([-1, 0, -1, 0, 0, -1, -1, 1]), np.array([2, 0, -1, 0, 1, -1, -1, 1])):
        assert L.rba_set_rig_sensors(lin.h, p(np.ascontiguousarray(bad, np.int32))) == INVALID
    assert np.array_equal(lin.rig_extrinsics(), ext0)
    lin.download_state()
    assert np.array_equal(bp.cams, cams0)
    lin.linearize()
    lin.solve(1e-3)  # the sensors are still in force: a solve works
    assert L.rba_get_rig_extrinsics(lin.h, None) == INVALID
    lin.close()
    # sensors without rigs, and a later rba_set_camera_rigs clears them
    bp = rb.BalProblem.from_arrays(prob, np.float64)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions())
    assert L.rba_set_rig_sensors(lin.h, p(np.ascontiguousarray(SENSOR))) == INVALID
    assert L.rba_set_rig_sensors(lin.h, None) == _lib.RBA_OK
    lin.set_camera_rigs(RIG, E)
    lin.set_rig_sensors(SENSOR)
    lin.set_camera_rigs(RIG, E)  # the extrinsics are the given ones again
    given = np.c_[E[:, :4] / np.linalg.norm(E[:, :4], axis=1, keepdims=True), E[:, 4:]]
    given[RIG < 0] = [0, 0, 0, 1, 0, 0, 0]  # a free camera's are the identity
    assert rel_err(sgn(np.asarray(lin.rig_extrinsics(), np.float64)), sgn(given)) < 1e-15
    assert bp.rig_sensor is None
    lin.close()


def test_covariance_is_that_of_the_tied_problem():
    """both covariance entry points against the dense inverse of the tied system (gauge fixed by the camera priors), with
    sensor 0 captured in all three rigs whose leads share one held extrinsics: the relative covariance of a lead and a
    capture of sensor 0 is the model's, not 0, and equal to rounding across the three rigs"""
    import pair_prior_model as qm
    prob, _, _, E, model = rig_case(("camera", "landmarks"))
    E = E.copy()
    E[[2, 6]] = E[0]
    sensor = np.array([-1, 0, -1, 0, 1, -1, -1, 0], np.int32)
    for held in (False, True):
        mask = None
        if held:
            mask = np.zeros(prob.nc, np.uint8)
            mask[[0, 1]] = FIX_POSE
        bp, lin = _handle(PCG_CONFIGS[0], prob, E, model, np.float64, sensor=sensor, mask=mask)
        lin.download_state()
        lead, home = sn.structure(RIG, sensor)
        cams = np.array(bp.cams, np.float64)
        Jp, Jl, _ = dense_system(_with_cams(prob, cams), **model)
        M = sn.maps(cams, lead, home, E)
        fixed9 = None
        if held:
            fixed9 = fixed_entries(mask).reshape(-1, 9)
            fixed9[home >= 0, :6] = False
            fixed9 = fixed9.ravel()
        want_cam, want_lm, full = sn.tied_covariance(Jp, Jl, lead, home, M, fixed9)
        cam, lm_ = lin.covariance()
        assert rel_err(cam, want_cam) < 1e-7, held
        assert rel_err(lm_, want_lm) < 1e-7, held
        pairs = np.array([[1, 0], [3, 2], [7, 6], [4, 2]])
        got = lin.covariance_blocks(cameras=[[2, 4], [0, 3]], relative=pairs)
        assert rel_err(got["cameras"][0], full[18:27, 36:45]) < 1e-7 and rel_err(got["cameras"][1], full[0:9, 27:36]) < 1e-7
        for k, (i, j) in enumerate(pairs):  # the relative pose T_i T_j^-1 linearised as the pair-prior residual
            Jr = qm.jacobians(cams[i], cams[j], qm.mean_at(cams, np.array([[i, j]]))[0])
            Jij = np.zeros((6, 9 * prob.nc))
            Jij[:, 9 * i:9 * i + 9], Jij[:, 9 * j:9 * j + 9] = Jr
            want = Jij @ full @ Jij.T
            assert rel_err(got["relative"][k], want) < 1e-7, (held, k)
        rel = got["relative"]
        assert np.max(np.abs(rel[0])) > 0
        assert rel_err(rel[1], rel[0]) < 1e-9 and rel_err(rel[2], rel[0]) < 1e-9, held
        lin.close()


def test_recovers_true_extrinsics_from_a_perturbed_start():
    """a noise-free capture, extrinsics of every sensor but the held one perturbed by a few degrees and centimetres, the
    gauge fixed by centre priors at the true camera centres of the held sensor: rba_lm_run in f64 recovers the truth"""
    import rootba_b200 as rb
    import camera_prior_model as pm
    from rootba_b200.synthetic import synth_rig_capture
    cap = synth_rig_capture(4, 12, 3000, seed=21, max_depth=8.0)
    rng = np.random.default_rng(4)
    E = cap.cam_from_rig.copy()
    sensor = np.where(cap.sensor == 0, -1, cap.sensor).astype(np.int32)
    for k in range(1, 4):
        d = np.r_[rng.normal(0, 0.03, 3), np.deg2rad(rng.normal(0, 2.0, 3)), 0, 0, 0]
        e = pm.apply_inc(np.r_[E[cap.sensor == k][0], 0, 0, 0], d)[:7]
        E[cap.sensor == k] = e
    nc = cap.prob.nc
    held = np.flatnonzero(sensor < 0)
    mean = pm.mean_at(cap.prob.cams)  # the true cameras; only their centres are weighted
    Lc = np.zeros((nc, 9, 9))
    Lc[held, 0, 0] = Lc[held, 1, 1] = Lc[held, 2, 2] = 1e3
    bp = rb.BalProblem.from_arrays(cap.prob, np.float64)
    bp.camera_prior = (mean, Lc)
    bp.camera_rig = (cap.rig, E)
    bp.rig_sensor = sensor
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(max_num_iterations=100, function_tolerance=1e-20, eta=1e-12))
    ext0 = np.asarray(lin.rig_extrinsics(), np.float64)
    err0 = np.max(np.abs(sgn(ext0) - sgn(cap.cam_from_rig)))
    lin.lm_run(100)
    ext = np.asarray(lin.rig_extrinsics(), np.float64)
    err = np.max(np.abs(sgn(ext) - sgn(cap.cam_from_rig)))
    assert err0 > 1e-2 and err < 1e-9, (err0, err)
    lin.close()


@pytest.mark.parametrize("precond", ["JACOBI", "SCHUR_JACOBI"])
@pytest.mark.parametrize("sfx", ["f32", "f64"])
def test_two_ranks_with_sensors(tmp_path, sfx, precond):
    """two GPUs (skipped with fewer): the NCCL hand-over with the sensor contraction; the sharded step equals the single-rank
    one and the cameras are bit-identical on both ranks"""
    from objective_checks import run_two_ranks
    res = run_two_ranks(tmp_path, "multirank_rig_sensors_worker.py", sfx, "1", 29700, (5 if sfx == "f32" else 13) + (0 if precond == "JACOBI" else 2),
                        precond)
    tols = 1e-4 if sfx == "f32" else 1e-8
    assert res["replicas_identical"], res
    assert res["inc"] < tols and res["l_diff"] < 20 * tols and res["cams"] < tols and res["cost"] < tols, res


def test_example_flags(tmp_path):
    """examples/solve_bal.py --camera-rigs with a `sensor` array and --rig-extrinsics: the held cameras' extrinsics come back
    as given, every capture of a sensor reports the same refined extrinsics, and the covariance handle built after the solve
    ties the sensors to them"""
    import os
    import subprocess
    import sys
    from rootba_b200.synthetic import write_bal
    cap = _capture(3, 6, 800, seed=8, perturb=False)
    path = tmp_path / "p.txt"
    write_bal(cap.prob, str(path))
    nc = cap.prob.nc
    E = rm.rig_case(nc, seed=2)
    sensor = np.where(cap.sensor == 0, -1, cap.sensor).astype(np.int32)
    rp = tmp_path / "rigs.npz"
    np.savez(rp, rig=cap.rig, cam_from_rig=E, sensor=sensor)
    out = tmp_path / "ext.npy"
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, os.path.join(root, "examples", "solve_bal.py"), str(path), "--max-num-iterations", "3",
                        "--camera-rigs", str(rp), "--rig-extrinsics", str(out), "--log-path", str(tmp_path / "log.json")],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    ext = np.load(out)
    assert ext.shape == (nc, 7)
    given = np.c_[E[:, :4] / np.linalg.norm(E[:, :4], axis=1, keepdims=True), E[:, 4:]]
    held = sensor < 0
    assert rel_err(sgn(ext[held]), sgn(given[held])) < 1e-15
    for k in (1, 2):
        m = sgn(ext[cap.sensor == k])
        assert np.max(np.abs(m - m[0])) == 0.0
        assert np.max(np.abs(m[0] - sgn(given[cap.sensor == k])[0])) > 0  # refined away from the given start
