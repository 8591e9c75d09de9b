"""The float64 model of estimated rig extrinsics (tests/rig_sensor_model.py) on the CPU: a sensor camera's first-order move
against central differences of the exact composition, the tied Jacobian (every prior kind, a pair prior between a lead and a
sensor camera among them) against central differences of the re-tied problem, the tied step against the true cost change,
the contracted covariance against the tied inverse, the planted faults the GPU checks must catch, the public header, the
library's exports and the Python host's validation."""
import re

import numpy as np
import pytest

import camera_prior_model as pm
import camera_rig_model as rm
import rig_sensor_model as sn
import shared_intrinsics_model as sm
from objective_checks import dense_system, reduced, total_cost
from test_camera_rig_model import RIG, rig_case

# rigs {0, 1}, {2, 3, 4}, {6, 7}: sensor 0 = cameras 1 (home) and 3, sensor 1 = cameras 4 (home) and 7 (no observations)
SENSOR = np.array([-1, 0, -1, 0, 1, -1, -1, 1], np.int32)


def _with_cams(prob, cams):
    from rootba_b200.synthetic import BalArrays
    return BalArrays(cams, prob.lms, prob.lm_off, prob.obs_cam, prob.obs_xy)


def sensor_case(priors=(), sensor=SENSOR):
    """rig_case tied as rba_set_rig_sensors leaves it, and moved off the given extrinsics: sensor 0's home turned by 0.02 rad
    and shifted, so that E_s differs from every given E.  Returns prob, lead, home, E, model"""
    prob, _, _, E, model = rig_case(priors)
    lead, home = sn.structure(RIG, sensor)
    cams = sn.tie_at_call(prob.cams, lead, home, E)
    h = home[np.flatnonzero(home >= 0)[0]]
    cams[h] = pm.apply_inc(cams[h], np.r_[0.01, -0.02, 0.005, 0.02, -0.01, 0.015, 0, 0, 0])
    cams = sn.retie(cams, lead, home, E)
    return _with_cams(prob, cams), lead, home, E, model


def _inc_of(c, ref):
    """the left increment (v, w) that maps the pose ref to c"""
    q, t = rm.relative(c, ref)
    return np.r_[t, pm.log_so3(rm.rot(q))]


def test_sensor_camera_moves_by_the_adjoint_plus_the_sensor_increment():
    """d_j = A_j d_lead + d_s to first order against the exact composition T_j = Exp(d_s) E_s E_lead^-1 Exp(d_lead) T_lead;
    the planted right-multiplied sensor increment (A_j d_s) is far outside the bar"""
    rng = np.random.default_rng(3)
    E = rm.rig_case(3, spread=0.4)
    lead_cam = np.r_[rng.standard_normal(4), rng.standard_normal(3), 1.0, 0.0, 0.0]
    lead_cam[:4] /= np.linalg.norm(lead_cam[:4])
    Es = np.r_[E[1, :4] / np.linalg.norm(E[1, :4]), E[1, 4:]]
    def member(dl, ds):
        lc = pm.apply_inc(lead_cam, np.r_[dl, 0, 0, 0])
        es = pm.apply_inc(np.r_[Es, 0, 0, 0], np.r_[ds, 0, 0, 0])[:7]
        return rm.compose(sn.pose_mul(es, sn.pose_inv(E[0])), lc, lc)
    T = member(np.zeros(6), np.zeros(6))
    A = rm.adjoint(sn.pose_mul(Es, sn.pose_inv(E[0])))
    h = 1e-6
    for k in range(6):
        d = np.zeros(6)
        d[k] = h
        fd_l = (_inc_of(member(d, 0 * d), T) - _inc_of(member(-d, 0 * d), T)) / (2 * h)
        fd_s = (_inc_of(member(0 * d, d), T) - _inc_of(member(0 * d, -d), T)) / (2 * h)
        assert np.max(np.abs(fd_l - A[:, k])) < 1e-6, k
        assert np.max(np.abs(fd_s - np.eye(6)[:, k])) < 1e-6, k
    assert np.max(np.abs(A - np.eye(6))) > 1e-2  # the "right" fault would differ


PRIORS = [(), ("camera",), ("camera", "pairs", "landmarks")]


@pytest.mark.parametrize("priors", PRIORS, ids=lambda p: "-".join(p) or "none")
def test_tied_jacobian_against_central_differences(priors):
    """J P against central differences of the residual of the re-tied problem; the pair prior (0, 1) joins a lead and a
    sensor camera.  The planted faults (right-multiplied sensor increment, homes masked, A_j stale after E_s moved) do not
    match"""
    prob, lead, home, E, model = sensor_case(priors)
    Jp, _, _ = dense_system(prob, **model)
    M = sn.maps(prob.cams, lead, home, E)
    P = sn.expansion(lead, home, M)
    Ju = Jp @ P
    h = 1e-6
    fd = np.zeros_like(Ju)
    for k in range(P.shape[1]):
        e = np.zeros(P.shape[1])
        e[k] = h
        rp = dense_system(_with_cams(prob, sn.apply_tied(prob.cams, P @ e, lead, home, E)), **model)[2]
        rmi = dense_system(_with_cams(prob, sn.apply_tied(prob.cams, -P @ e, lead, home, E)), **model)[2]
        fd[:, k] = (rp - rmi) / (2 * h)
    bar = lambda J: np.max(np.abs(fd - J)) / max(1.0, np.max(np.abs(fd)))
    assert bar(Ju) <= 1e-5
    stale = sn.maps(sn.tie_at_call(prob.cams, lead, home, E), lead, home, E)  # M of the given E, not the state's
    assert bar(Jp @ sn.expansion(lead, home, stale)) > 1e-3
    assert bar(Jp @ sn.expansion(lead, home, M, fault="right")) > 1e-3
    # the homes masked: the sensor cameras move with their rig alone, so no column of that Jacobian reproduces a sensor
    # column of the finite differences (the recurrence check below rejects the same fault in the solve)
    no_home = Jp @ sn.expansion(lead, home, M, fault="no_sensor")
    scols = sn.reduced_cols(lead, home)[np.unique(home[home >= 0])][:, :6].ravel()
    resid = fd[:, scols] - no_home @ np.linalg.lstsq(no_home, fd[:, scols], rcond=None)[0]
    assert np.max(np.abs(resid)) > 1e-3 * np.max(np.abs(fd[:, scols]))


def test_pair_prior_between_a_lead_and_a_sensor_camera_acts_on_the_sensor():
    """a pair prior inside a rig between the lead and a sensor camera: zero on the rig's columns, non-zero on the sensor's"""
    import pair_prior_model as qm
    prob, lead, home, E, _ = sensor_case()
    rng = np.random.default_rng(9)
    pairs = np.array([[2, 3]], np.int32)
    model = {"pairs": (pairs, qm.mean_at(prob.cams, pairs), np.stack([qm.sqrt_info_kind("dense", rng)]))}
    Jp, _, _ = dense_system(prob, **model)
    P = sn.expansion(lead, home, sn.maps(prob.cams, lead, home, E))
    E9 = sn.embed(lead, home)
    rows = (Jp @ P)[-6:]
    rig_cols = [np.flatnonzero(E9[18 + k])[0] for k in range(6)]
    sen_cols = [np.flatnonzero(E9[9 + k])[0] for k in range(6)]  # sensor 0's home: camera 1
    assert np.max(np.abs(rows[:, rig_cols])) < 1e-12 * np.max(np.abs(Jp[-6:]))
    assert np.max(np.abs(rows[:, sen_cols])) > 1e-3


@pytest.mark.parametrize("groups", [False, True], ids=["sensors", "sensors-and-groups"])
def test_tied_step_decreases_the_true_cost_as_the_model_predicts(groups):
    """the LM step of J P with every prior kind: the model cost change matches the true change of the re-tied problem, and
    the sensor cameras stay at E_s E_lead^-1 T_lead"""
    prob, lead, home, E, model = sensor_case(("camera", "pairs", "landmarks"))
    glead = sm.leads(np.array([0, 0, -1, 0, 5, 5, -1, 5])) if groups else None
    if groups:
        cams = np.array(prob.cams)
        g = glead >= 0
        cams[g, 7:] = cams[glead[g], 7:]
        prob = _with_cams(prob, cams)
    Jp, Jl, r = dense_system(prob, **model)
    P = sn.expansion(lead, home, sn.maps(prob.cams, lead, home, E), glead)
    lam = 1e-4
    Du, sl, _, Jls, Minv, Hu, bu = reduced(Jp @ P, Jl, r, lam, prob.nl)
    u = -np.linalg.solve(Hu, bu)
    x = P @ (Du * u)
    W = (Jp @ P * Du).T @ Jls
    dl = -Minv @ (Jls.T @ r + W.T @ u)
    step = 1e-4
    lin = r + step * ((Jp @ P * Du) @ u + Jls @ dl)
    l_diff = 0.5 * r @ r - 0.5 * lin @ lin
    cams = sn.apply_tied(prob.cams, step * x, lead, home, E)
    from rootba_b200.synthetic import BalArrays
    new = BalArrays(cams, prob.lms + step * (sl * dl).reshape(-1, 3), prob.lm_off, prob.obs_cam, prob.obs_xy)
    true = total_cost(prob, **model) - total_cost(new, **model)
    assert l_diff > 0 and abs(true - l_diff) <= 1e-3 * l_diff
    Es = sn.sensor_extrinsics(cams, lead, home, E)
    for c in np.flatnonzero(home >= 0):  # every camera of a sensor reports its home's extrinsics
        q = Es[c, :4] * np.sign(Es[c, 3])
        qh = Es[home[c], :4] * np.sign(Es[home[c], 3])
        assert np.allclose(q, qh, atol=1e-12) and np.allclose(Es[c, 4:], Es[home[c], 4:], atol=1e-12), c


def test_contracted_covariance_is_the_tied_inverse():
    """P (P^T A P)^-1 P^T of the full reduced camera matrix equals the camera blocks of inv(J_u^T J_u); the relative
    covariance of a lead and a sensor camera is not zero, unlike that of a lead and a held member"""
    prob, lead, home, E, model = sensor_case(("camera", "landmarks"))
    Jp, Jl, _ = dense_system(prob, **model)
    M = sn.maps(prob.cams, lead, home, E)
    want, _, full = sn.tied_covariance(Jp, Jl, lead, home, M)
    Hll_inv = np.linalg.inv(Jl.T @ Jl)
    A = Jp.T @ Jp - Jp.T @ Jl @ Hll_inv @ Jl.T @ Jp
    got = sn.contracted_covariance(A, lead, home, M)
    assert np.max(np.abs(got - want)) <= 1e-8 * np.max(np.abs(want))
    def rel(i, j):  # the covariance of d_i - A d_j, the relative motion of camera i against camera j's frame
        Aij = rm.adjoint(sn.pose_mul(prob.cams[i, :7], sn.pose_inv(prob.cams[j, :7])))
        Tm = np.zeros((6, 9 * len(lead)))
        Tm[:, 9 * i:9 * i + 6] = np.eye(6)
        Tm[:, 9 * j:9 * j + 6] = -Aij
        return Tm @ full @ Tm.T
    assert np.max(np.abs(rel(3, 2))) > 1e-6 * np.max(np.abs(full))
    # without sensors the same pair is a held member and its lead: 0 to rounding
    prob0, lead0, M0, _, _ = rig_case(("camera", "landmarks"))
    Jp0, Jl0, _ = dense_system(prob0, **model)
    full0 = rm.tied_covariance(Jp0, Jl0, lead0, M0)[2]
    Aij = rm.adjoint(M0[3])
    Tm = np.zeros((6, 72))
    Tm[:, 27:33] = np.eye(6)
    Tm[:, 18:24] = -Aij
    assert np.max(np.abs(Tm @ full0 @ Tm.T)) < 1e-9 * np.max(np.abs(full0))


def test_python_validation():
    import rootba_b200 as rb
    from rootba_b200.linearizor import _rig_sensor_array
    prob, _, _, E, _ = rig_case()
    rig = (RIG, E)
    assert _rig_sensor_array(None, rig, 8) is None
    assert np.array_equal(_rig_sensor_array(SENSOR, rig, 8), SENSOR)
    for bad, what in [(SENSOR[:7], "one entry"), (SENSOR.astype(float), "integers"), (np.r_[SENSOR[:7], 8], "integers"),
                      (np.r_[SENSOR[:7], -2], "integers"), (np.array([-1, 0, -1, 0, 1, 3, -1, 1]), "not in a rig"),
                      (np.array([-1, 0, -1, 0, 0, -1, -1, 1]), "same sensor"), (np.array([2, 0, -1, 0, 1, -1, -1, 1]), "every camera")]:
        with pytest.raises(ValueError, match=what):
            _rig_sensor_array(bad, rig, 8)
    with pytest.raises(ValueError, match="not in a rig"):
        _rig_sensor_array(SENSOR, None, 8)
    bp = rb.BalProblem.from_arrays(prob, np.float64)
    bp.camera_rig = rig
    bp.rig_sensor = SENSOR
    assert np.array_equal(bp.rig_sensor, SENSOR)
    bp.camera_rig = rig  # a new camera_rig clears the sensors
    assert bp.rig_sensor is None


def test_header_and_exports():
    from rootba_b200 import _lib
    txt = open(_lib.HEADER_PATH).read()
    assert re.search(r"int32_t rba_set_rig_sensors\(rba_handle\* h, const int32_t\* sensor\);", txt)
    assert re.search(r"int32_t rba_get_rig_extrinsics\(rba_handle\* h, void\* cam_from_rig\);", txt)
    assert "DESIGN.md section 24" in txt
    assert {"rba_set_rig_sensors", "rba_get_rig_extrinsics"} <= set(_lib.declared_symbols())
    import os
    if os.path.exists(_lib.LIB_PATH):
        out = __import__("subprocess").run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True).stdout
        assert " rba_set_rig_sensors" in out and " rba_get_rig_extrinsics" in out


# ---- the device's recurrence and preconditioner against the tied system ---------------------------------------------
K, PERIOD = 8, 5  # iterations compared, one residual refresh included


def _pair_model(prob, priors):
    """the priors of `priors` with pair priors joining a lead and a sensor capture (0, 1), two captures of sensor 0 (1, 3),
    a lead and a capture of sensor 1 (2, 4) and two rigs' cameras (3, 5)"""
    import pair_prior_model as qm
    _, _, _, _, model = rig_case(tuple(p for p in priors if p != "pairs"))
    if "pairs" in priors:
        rng = np.random.default_rng(5)
        pairs = np.array([[0, 1], [1, 3], [2, 4], [3, 5]], np.int32)
        model["pairs"] = (pairs, qm.mean_at(prob.cams, pairs), np.stack([qm.sqrt_info_kind("dense", rng) for _ in pairs]))
    return model


def _systems(priors, lam, jacobi, fault=None):
    """(Hfull without the pose damping, b_full, per-camera blocks) of the full x-space system under the per-camera scaling D,
    and (P~, H_u, b_u, lead, home) of the tied model in the device's scaling (D_u, D_s of the merged columns).  Planted faults
    of P~: "q_without_ds" (a sensor's columns scaled by D_j^-1 alone), "ds_without_pair_terms" (D_s from the captures' own
    column norms, without the cross terms of the pair priors between two captures of the sensor)"""
    import camera_model as cm
    prob, lead, home, E, _ = sensor_case()
    model = _pair_model(prob, priors)
    Jp, Jl, r = dense_system(prob, **model)
    P = sn.expansion(lead, home, sn.maps(prob.cams, lead, home, E))
    D, sl, _, Jls, Minv, _, _ = reduced(Jp, Jl, r, lam, prob.nl)
    Du = reduced(Jp @ P, Jl, r, lam, prob.nl)[0]
    Jps = Jp * D
    W = Jps.T @ Jls
    Hfull = Jps.T @ Jps - W @ Minv @ W.T
    b_full = Jps.T @ r - W @ Minv @ (Jls.T @ r)
    src = Jps.T @ Jps if jacobi else Hfull
    blocks = np.stack([src[9 * c:9 * c + 9, 9 * c:9 * c + 9] for c in range(prob.nc)])
    Pt = (P * Du[None, :]) / D[:, None]
    Hu = Pt.T @ Hfull @ Pt + lam * np.eye(P.shape[1])
    bad = Pt
    if fault is not None:
        col = sn.reduced_cols(lead, home)
        scol = np.concatenate([col[h, :6] for h in np.unique(home[home >= 0])])
        Du_bad = Du.copy()
        if fault == "q_without_ds":
            Du_bad[scol] = 1.0
        else:
            eps = float(cm.EPS_SQRT[np.dtype(np.float64)])
            for h in np.unique(home[home >= 0]):
                for k in range(6):
                    n2 = sum(float(Jp[:, 9 * j + k] @ Jp[:, 9 * j + k]) for j in np.flatnonzero(home == h))
                    Du_bad[col[h, k]] = 1.0 / (eps + np.sqrt(n2))
        bad = (P * Du_bad[None, :]) / D[:, None]
    return Hfull, b_full, blocks, Pt, Hu, Pt.T @ b_full, lead, home, bad


def _pcg_ref(Hu, bu, blocks, lam, lead, home, Pt):
    from pcg_replay import pcg_replay
    Mu = sn.reduced_block_jacobi(blocks, lam, lead, home, Pt)
    return pcg_replay(lambda v: Hu @ v, bu, lambda v: Mu @ v, eta=-1.0, max_it=K, period=PERIOD)


def _max_iterate_err(ref, got, lead, home):
    E = sn.embed(lead, home)
    n = min(len(ref["xs"]), len(got["xs"]))
    assert n == K + 1, n
    return max(float(np.linalg.norm(got["xs"][k] - E @ ref["xs"][k]) / np.linalg.norm(E @ ref["xs"][k])) for k in range(1, n))


@pytest.mark.parametrize("jacobi", [False, True], ids=["SCHUR_JACOBI", "JACOBI"])
@pytest.mark.parametrize("priors", PRIORS, ids=lambda p: "-".join(p) or "none")
def test_device_recurrence_equals_pcg_on_the_tied_system(priors, jacobi):
    """the 9 nc recurrence (b contracted into the leads and homes, P~ expand / contract around K, lambda on the contracted v,
    the device's blocks with the sensors' in their homes' slots) is PCG on the tied system in the device's scaling, iterate
    by iterate through a residual refresh; the device's blocks are M_u^-1 of the tied system in the 9 nc layout"""
    from pcg_replay import block_apply
    lam = 1e-3
    Hfull, b_full, blocks, Pt, Hu, bu, lead, home, _ = _systems(priors, lam, jacobi)
    E = sn.embed(lead, home)
    inv = sn.device_blocks(blocks, lam, lead, home, Pt)
    Mu = sn.reduced_block_jacobi(blocks, lam, lead, home, Pt)
    x = np.random.default_rng(2).standard_normal(len(bu))
    assert np.linalg.norm(block_apply(inv, E @ x) - E @ (Mu @ x)) < 1e-13 * np.linalg.norm(E @ (Mu @ x))
    got = sn.replay_9nc(Hfull, b_full, blocks, lam, lead, home, Pt, eta=-1.0, max_it=K, period=PERIOD)
    assert _max_iterate_err(_pcg_ref(Hu, bu, blocks, lam, lead, home, Pt), got, lead, home) < 1e-12


@pytest.mark.parametrize("fault", ["lambda_per_member", "home_masked", "q_without_ds", "ds_without_pair_terms"])
def test_the_recurrence_check_catches_planted_faults(fault):
    """each planted fault, run through the same iterate comparison as the correct replay, lies far outside its bar"""
    lam = 1e-3
    Hfull, b_full, blocks, Pt, Hu, bu, lead, home, bad = _systems(("camera", "pairs"), lam, False,
                                                                  fault if fault in ("q_without_ds", "ds_without_pair_terms") else None)
    ref = _pcg_ref(Hu, bu, blocks, lam, lead, home, Pt)
    got = sn.replay_9nc(Hfull, b_full, blocks, lam, lead, home, bad, eta=-1.0, max_it=K, period=PERIOD,
                        fault=fault if fault in ("lambda_per_member", "home_masked") else None)
    assert _max_iterate_err(ref, got, lead, home) > 1e-6
    ok = sn.replay_9nc(Hfull, b_full, blocks, lam, lead, home, Pt, eta=-1.0, max_it=K, period=PERIOD)
    assert _max_iterate_err(ref, ok, lead, home) < 1e-8


def test_held_rig_tied_step_decreases_the_true_cost_as_the_model_predicts():
    """RBA_FIX_POSE on rig {2, 3, 4}: its lead's pose is held, its captures still move with their sensors (the homes' entries
    free); the step of the tied system without the held entries matches the true cost change, and the lead stays put"""
    from objective_checks import fixed_entries
    prob, lead, home, E, model = sensor_case(("camera", "pairs", "landmarks"))
    mask = np.zeros(prob.nc, np.uint8)
    mask[[2, 3, 4]] = 1  # RBA_FIX_POSE
    fixed9 = fixed_entries(mask).reshape(-1, 9)
    fixed9[home >= 0, :6] = False
    keep = np.flatnonzero(~sn.held(lead, home))
    fu = ~fixed9.ravel()[keep]
    Jp, Jl, r = dense_system(prob, **model)
    P = sn.expansion(lead, home, sn.maps(prob.cams, lead, home, E))
    lam = 1e-4
    Du, sl, _, Jls, Minv, Hu, bu = reduced(Jp @ P, Jl, r, lam, prob.nl)
    u = np.zeros(len(bu))
    u[fu] = -np.linalg.solve(Hu[np.ix_(fu, fu)], bu[fu])
    assert np.all(u[~fu] == 0) and np.max(np.abs(u[sn.reduced_cols(lead, home)[4, :6]])) > 0  # home 4 moves in the held rig
    x = P @ (Du * u)
    W = (Jp @ P * Du).T @ Jls
    dl = -Minv @ (Jls.T @ r + W.T @ u)
    step = 1e-4
    lin = r + step * ((Jp @ P * Du) @ u + Jls @ dl)
    l_diff = 0.5 * r @ r - 0.5 * lin @ lin
    cams = sn.apply_tied(prob.cams, step * x, lead, home, E)
    from rootba_b200.synthetic import BalArrays
    new = BalArrays(cams, prob.lms + step * (sl * dl).reshape(-1, 3), prob.lm_off, prob.obs_cam, prob.obs_xy)
    true = total_cost(prob, **model) - total_cost(new, **model)
    assert l_diff > 0 and abs(true - l_diff) <= 1e-3 * l_diff
    assert np.max(np.abs(cams[2, :7] - np.asarray(prob.cams, np.float64)[2, :7])) < 1e-12  # a zero increment, to rounding
