"""The float64 model of rigid camera rigs (tests/camera_rig_model.py) on the CPU: the adjoint against central differences of
the exact composition, the tied LM step against the true cost change with every prior kind and with intrinsics groups, a
pair prior inside a rig, rigs of one, the planted faults the GPU checks must catch, and the public header."""
import re

import numpy as np
import pytest

import camera_prior_model as pm
import camera_rig_model as rm
import landmark_prior_model as lp
import pair_prior_model as qm
import shared_intrinsics_model as sm
from objective_checks import dense_system, reduced, total_cost

# rigs {0, 1}, {2, 3, 4} and {6, 7} (camera 7 has no observations), camera 5 free
RIG = np.array([0, 0, 3, 3, 3, -1, 7, 7], np.int32)


def _with_cams(prob, cams):
    from rootba_b200.synthetic import BalArrays
    return BalArrays(cams, prob.lms, prob.lm_off, prob.obs_cam, prob.obs_xy)


def rig_case(priors=(), rig=RIG):
    """camera_prior_model.prior_case (8 cameras, the last without observations) re-tied to the rigs of `rig`, and the prior
    kinds `priors` names (the pair priors join cameras inside and across rigs).  Returns prob, lead, M, cam_from_rig, model."""
    prob, mean, L = pm.prior_case()
    E = rm.rig_case(prob.nc)
    lead = rm.leads(rig)
    M = rm.maps(E, lead)
    prob = _with_cams(prob, rm.retie(prob.cams, lead, M))
    model = {}
    if "camera" in priors:
        model["camera"] = (mean, L)
    if "pairs" in priors:
        rng = np.random.default_rng(5)
        pairs = np.array([[0, 1], [2, 4], [3, 5], [1, 2]], np.int32)
        model["pairs"] = (pairs, qm.mean_at(prob.cams, pairs), np.stack([qm.sqrt_info_kind("dense", rng) for _ in pairs]))
    if "landmarks" in priors:
        model["landmarks"] = lp.prior_case(prob.lms)
    return prob, lead, M, E, model


def test_adjoint_against_the_exact_composition():
    """a lead increment d moves member j by A_j d to first order; the error of the linear map is O(|d|^2)"""
    rng = np.random.default_rng(3)
    E = rm.rig_case(2, spread=0.4)
    m = rm.maps(E, np.array([0, 0]))[1]
    lead = np.r_[rng.standard_normal(4), rng.standard_normal(3), 1.0, 0.0, 0.0]
    lead[:4] /= np.linalg.norm(lead[:4])
    member = rm.compose(m, lead, lead)
    A = rm.adjoint(m)
    h = 1e-6
    for k in range(6):
        d = np.zeros(9)
        d[k] = h
        plus = rm.compose(m, pm.apply_inc(lead, d), lead)
        minus = rm.compose(m, pm.apply_inc(lead, -d), lead)
        # the member increment (v, w) that maps member to plus / minus, by the same convention
        def inc_of(c):
            q, t = rm.relative(c, member)  # T_c T_member^-1 = [Exp(w) | v']
            w = pm.log_so3(rm.rot(q))
            return np.r_[t, w]
        fd = (inc_of(plus) - inc_of(minus)) / (2 * h)
        assert np.max(np.abs(fd - A[:, k])) < 1e-6, k
    # the planted sign flip of [t_m]x is far outside that bar
    bad = rm.expansion(np.array([0, 0]), np.stack([np.r_[0, 0, 0, 1.0, 0, 0, 0], m]), fault="tx_sign")[9:15, :6]
    assert np.max(np.abs(bad - A)) > 1e-2


PRIORS = [(), ("camera",), ("camera", "pairs", "landmarks")]


@pytest.mark.parametrize("priors", PRIORS, ids=lambda p: "-".join(p) or "none")
def test_tied_jacobian_against_central_differences(priors):
    prob, lead, M, _, model = rig_case(priors)
    Jp, _, _ = dense_system(prob, **model)
    P = rm.expansion(lead, M)
    Ju = Jp @ P
    h = 1e-6
    for k in range(P.shape[1]):
        e = np.zeros(P.shape[1])
        e[k] = h
        rp = dense_system(_with_cams(prob, rm.apply_tied(prob.cams, P @ e, lead, M)), **model)[2]
        rmi = dense_system(_with_cams(prob, rm.apply_tied(prob.cams, -P @ e, lead, M)), **model)[2]
        fd = (rp - rmi) / (2 * h)
        assert np.max(np.abs(fd - Ju[:, k])) <= 1e-5 * max(1.0, np.max(np.abs(Ju[:, k]))), k


@pytest.mark.parametrize("groups", [False, True], ids=["rigs", "rigs-and-groups"])
def test_tied_step_decreases_the_true_cost_as_the_model_predicts(groups):
    """the LM step of J P with every prior kind: the model cost change matches the true change of the re-tied problem at a
    small lambda and a small step, and the members stay rigid"""
    prob, lead, M, _, model = rig_case(("camera", "pairs", "landmarks"))
    glead = sm.leads(np.array([0, 0, -1, 0, 5, 5, -1, 5])) if groups else None
    if groups:
        cams = np.array(prob.cams)
        g = glead >= 0
        cams[g, 7:] = cams[glead[g], 7:]
        prob = _with_cams(prob, cams)
    Jp, Jl, r = dense_system(prob, **model)
    P = rm.expansion(lead, M, glead)
    lam = 1e-4
    Du, sl, _, Jls, Minv, Hu, bu = reduced(Jp @ P, Jl, r, lam, prob.nl)
    u = -np.linalg.solve(Hu, bu)
    x = P @ (Du * u)
    W = (Jp @ P * Du).T @ Jls
    dl = -Minv @ (Jls.T @ r + W.T @ u)
    step = 1e-4
    lin = r + step * ((Jp @ P * Du) @ u + Jls @ dl)
    l_diff = 0.5 * r @ r - 0.5 * lin @ lin
    cams = rm.apply_tied(prob.cams, step * x, lead, M)
    from rootba_b200.synthetic import BalArrays
    new = BalArrays(cams, prob.lms + step * (sl * dl).reshape(-1, 3), prob.lm_off, prob.obs_cam, prob.obs_xy)
    true = total_cost(prob, **model) - total_cost(new, **model)
    assert l_diff > 0 and abs(true - l_diff) <= 1e-3 * l_diff
    # the members stay exactly rigid
    for c in np.flatnonzero((lead >= 0) & (lead != np.arange(len(lead)))):
        q, t = rm.relative(cams[c], cams[lead[c]])
        assert np.allclose(np.r_[q * np.sign(q[3]), t], M[c] * np.r_[np.sign(M[c, 3]) * np.ones(4), np.ones(3)], atol=1e-12)


def test_pair_prior_inside_a_rig_has_a_zero_tied_jacobian():
    prob, lead, M, _, _ = rig_case()
    rng = np.random.default_rng(9)
    pairs = np.array([[2, 4]], np.int32)
    model = {"pairs": (pairs, qm.mean_at(prob.cams, pairs), np.stack([qm.sqrt_info_kind("dense", rng)]))}
    Jp, _, _ = dense_system(prob, **model)
    Ju = Jp @ rm.expansion(lead, M)
    rows = Ju[-6:]
    assert np.max(np.abs(rows)) < 1e-12 * max(1.0, np.max(np.abs(Jp[-6:])))
    # and across two rigs it is not
    pairs = np.array([[1, 2]], np.int32)
    model = {"pairs": (pairs, qm.mean_at(prob.cams, pairs), np.stack([qm.sqrt_info_kind("dense", rng)]))}
    Jp, _, _ = dense_system(prob, **model)
    assert np.max(np.abs((Jp @ rm.expansion(lead, M))[-6:])) > 1e-3


def test_rigs_of_one_give_the_free_system():
    prob, _, _, E, _ = rig_case()
    lead = rm.leads(np.arange(prob.nc))
    assert np.all(lead == -1)
    assert np.array_equal(rm.expansion(lead, rm.maps(E, lead)), np.eye(9 * prob.nc))


def test_planted_faults_move_the_step():
    """the faults the GPU checks must catch move the increment far beyond the float64 bars: a missing D_j^-1 or D_u in P~,
    D_u from the diagonal of the members' blocks only (no Gram, no pair cross terms), and the members updated linearly
    without a re-tie (drift after 20 steps)"""
    prob, lead, M, _, model = rig_case(("camera", "pairs"))
    Jp, Jl, r = dense_system(prob, **model)
    P = rm.expansion(lead, M)
    D = reduced(Jp, Jl, r, 1e-3, prob.nl)[0]
    Du = reduced(Jp @ P, Jl, r, 1e-3, prob.nl)[0]
    good = rm.scaled_map(P, D, Du)
    assert np.max(np.abs(good - (P * Du[None, :]))) > 1e-2 * np.max(np.abs(good))       # missing D_j^-1
    assert np.max(np.abs(good - P / D[:, None])) > 1e-2 * np.max(np.abs(good))           # missing D_u
    G = Jp.T @ Jp
    n_diag = np.sqrt(np.maximum(P.T ** 2 @ np.diag(G), 0))
    n_gram = np.sqrt(np.diag(P.T @ G @ P))
    assert np.max(np.abs(n_diag - n_gram) / n_gram) > 1e-3
    # linear member updates drift: 20 steps of a rotation of 0.05 on the lead
    cams = np.array(prob.cams)
    lin_cams = cams.copy()
    x = np.zeros(9 * prob.nc)
    x[3:6] = [0.05, -0.02, 0.03]
    for _ in range(20):
        step = P @ np.linalg.lstsq(P, x, rcond=None)[0]
        lin_cams = np.stack([pm.apply_inc(c, d) for c, d in zip(lin_cams, step.reshape(-1, 9))])
        cams = rm.apply_tied(cams, step, lead, M)
    q, t = rm.relative(lin_cams[1], lin_cams[0])
    assert np.linalg.norm(t - M[1, 4:]) > 1e-6
    q, t = rm.relative(cams[1], cams[0])
    assert np.linalg.norm(t - M[1, 4:]) < 1e-12


def test_header_declares_the_setter():
    import os
    from rootba_b200 import _lib
    assert "rba_set_camera_rigs" in _lib.declared_symbols()
    if os.path.exists(_lib.LIB_PATH):  # the built library exports it and the binding sets its argument types
        L = _lib.lib()
        assert hasattr(L, "rba_set_camera_rigs") and L.rba_set_camera_rigs.argtypes is not None
    txt = open(_lib.HEADER_PATH).read()
    assert re.search(r"int32_t rba_set_camera_rigs\(rba_handle\* h, const int32_t\* rig, const void\* cam_from_rig\);", txt)
    assert "DESIGN.md section 23" in txt


def test_python_host_validation():
    import rootba_b200 as rb
    prob, _, _, E, _ = rig_case()
    bp = rb.BalProblem.from_arrays(prob, np.float64)
    for rig, e, what in [(np.full(prob.nc + 1, -1), E, "one entry per camera"), (np.full(prob.nc, prob.nc), E, "in \\[-1"),
                         (RIG, E[:, :6], "shape"), (RIG, np.where(np.arange(8)[:, None] == 0, np.nan, E), "finite"),
                         (RIG, E * np.r_[1.1, 1.1, 1.1, 1.1, 1, 1, 1], "norm 1")]:
        with pytest.raises(ValueError, match=what):
            bp.camera_rig = (rig, e)
    assert bp.camera_rig is None
    free = np.where(RIG[:, None] >= 0, E, np.nan)  # a free camera's entries are ignored
    bp.camera_rig = (RIG, free)
    assert bp.camera_rig[0].dtype == np.int32


# ---- the device's recurrence, preconditioner and covariance against the tied system -----------------------------------
K, PERIOD = 8, 5  # iterations compared, one residual refresh included


def _systems(priors, lam, jacobi):
    """(Hfull without the pose damping, b_full, per-camera blocks) of the full x-space system under the per-camera scaling D,
    and (P~, H_u, b_u, lead) of the tied model in the device's scaling (D_u of the merged columns)"""
    prob, lead, M, _, model = rig_case(priors)
    Jp, Jl, r = dense_system(prob, **model)
    P = rm.expansion(lead, M)
    D, sl, _, Jls, Minv, _, _ = reduced(Jp, Jl, r, lam, prob.nl)
    Du = reduced(Jp @ P, Jl, r, lam, prob.nl)[0]
    Jps = Jp * D
    W = Jps.T @ Jls
    Hfull = Jps.T @ Jps - W @ Minv @ W.T
    b_full = Jps.T @ r - W @ Minv @ (Jls.T @ r)
    src = Jps.T @ Jps if jacobi else Hfull
    blocks = np.stack([src[9 * c:9 * c + 9, 9 * c:9 * c + 9] for c in range(prob.nc)])
    Pt = rm.scaled_map(P, D, Du)
    Hu = Pt.T @ Hfull @ Pt + lam * np.eye(P.shape[1])
    return Hfull, b_full, blocks, Pt, Hu, Pt.T @ b_full, lead


def _pcg_ref(Hu, bu, blocks, lam, lead, Pt):
    from pcg_replay import pcg_replay
    Mu = rm.reduced_block_jacobi(blocks, lam, lead, Pt)
    return pcg_replay(lambda v: Hu @ v, bu, lambda v: Mu @ v, eta=-1.0, max_it=K, period=PERIOD)


def _max_iterate_err(ref, got, lead):
    E = rm.embed(lead)
    n = min(len(ref["xs"]), len(got["xs"]))
    assert n == K + 1, n
    return max(float(np.linalg.norm(got["xs"][k] - E @ ref["xs"][k]) / np.linalg.norm(E @ ref["xs"][k])) for k in range(1, n))


@pytest.mark.parametrize("jacobi", [False, True], ids=["SCHUR_JACOBI", "JACOBI"])
@pytest.mark.parametrize("priors", PRIORS, ids=lambda p: "-".join(p) or "none")
def test_device_recurrence_equals_pcg_on_the_tied_system(priors, jacobi):
    """the 9 nc recurrence (contracted b, P~ expand / contract around K, lambda on the contracted v, the device's blocks) is
    PCG on the tied system in the device's scaling, iterate by iterate through a residual refresh; the device's blocks are
    M_u^-1 of the tied system in the 9 nc layout"""
    from pcg_replay import block_apply
    lam = 1e-3
    Hfull, b_full, blocks, Pt, Hu, bu, lead = _systems(priors, lam, jacobi)
    E = rm.embed(lead)
    inv = rm.device_blocks(blocks, lam, lead, Pt)
    Mu = rm.reduced_block_jacobi(blocks, lam, lead, Pt)
    x = np.random.default_rng(2).standard_normal(len(bu))
    assert np.linalg.norm(block_apply(inv, E @ x) - E @ (Mu @ x)) < 1e-13 * np.linalg.norm(E @ (Mu @ x))
    got = rm.replay_9nc(Hfull, b_full, blocks, lam, lead, Pt, eta=-1.0, max_it=K, period=PERIOD)
    assert _max_iterate_err(_pcg_ref(Hu, bu, blocks, lam, lead, Pt), got, lead) < 1e-12


@pytest.mark.parametrize("fault", ["lambda_per_member", "b_not_contracted", "no_pt", "no_Dj", "no_Du", "Du_diagonal", "tx_sign"])
def test_the_recurrence_check_catches_planted_faults(fault):
    """each planted fault, run through the same iterate comparison as the correct replay, lies far outside its bar"""
    lam = 1e-3
    Hfull, b_full, blocks, Pt, Hu, bu, lead = _systems(("camera", "pairs"), lam, False)
    ref = _pcg_ref(Hu, bu, blocks, lam, lead, Pt)
    bad_Pt = Pt
    if fault in ("no_Dj", "no_Du", "Du_diagonal", "tx_sign"):
        prob, _, M, _, model = rig_case(("camera", "pairs"))
        Jp, Jl, r = dense_system(prob, **model)
        P = rm.expansion(lead, M, fault="tx_sign" if fault == "tx_sign" else None)
        D = reduced(Jp, Jl, r, lam, prob.nl)[0]
        Du = reduced(Jp @ rm.expansion(lead, M), Jl, r, lam, prob.nl)[0]
        if fault == "Du_diagonal":  # the members' column norms from the diagonal of their Gram only, without the cross terms
            G = Jp.T @ Jp
            Du = 1.0 / (np.sqrt(np.finfo(np.float64).eps) + np.sqrt((P ** 2).T @ np.diag(G)))
        bad_Pt = (P * Du[None, :]) if fault == "no_Dj" else (P / D[:, None]) if fault == "no_Du" else rm.scaled_map(P, D, Du)
    got = rm.replay_9nc(Hfull, b_full, blocks, lam, lead, bad_Pt, eta=-1.0, max_it=K, period=PERIOD,
                        fault=fault if fault in ("lambda_per_member", "b_not_contracted", "no_pt") else None)
    assert _max_iterate_err(ref, got, lead) > 1e-6
    ok = rm.replay_9nc(Hfull, b_full, blocks, lam, lead, Pt, eta=-1.0, max_it=K, period=PERIOD)
    assert _max_iterate_err(ref, ok, lead) < 1e-8


def test_contracted_covariance_is_that_of_the_tied_problem():
    """the device's order (contract P^T A P, hold the members, invert, expand) equals the tied covariance; the planted
    row-only contraction does not; two members of one rig have a zero relative-pose covariance"""
    from conftest import rel_err
    prob, lead, M, _, model = rig_case(("camera", "landmarks"))
    Jp, Jl, _ = dense_system(prob, **model)
    want, _, full = rm.tied_covariance(Jp, Jl, lead, M)
    A = Jp.T @ Jp - Jp.T @ Jl @ np.linalg.solve(Jl.T @ Jl, Jl.T @ Jp)
    assert rel_err(rm.contracted_covariance(A, lead, M), want) < 1e-9
    assert rel_err(rm.contracted_covariance(A, lead, M, fault="rows_only"), want) > 1e-3
    # the relative pose T_i T_j^-1 of two members is constant, so its linearisation maps P Sigma_u P^T to 0
    i, j = 2, 4
    Jr = qm.jacobians(prob.cams[i], prob.cams[j], qm.mean_at(prob.cams, np.array([[i, j]]))[0])
    Jij = np.zeros((6, 9 * prob.nc))
    Jij[:, 9 * i:9 * i + 9], Jij[:, 9 * j:9 * j + 9] = Jr
    rel = Jij @ full @ Jij.T
    assert np.max(np.abs(rel)) < 1e-12 * np.max(np.abs(full))
