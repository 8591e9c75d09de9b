"""The float64 model of intrinsics shared across groups of cameras (tests/shared_intrinsics_model.py) on the CPU: the tied
model against central differences and the true cost change, the device's 9 nc recurrence against PCG on the tied system
iterate by iterate (and the planted faults that check must catch), and groups of one camera."""
import numpy as np
import pytest

import camera_prior_model as pm
import landmark_prior_model as lp
import pair_prior_model as qm
import shared_intrinsics_model as sm
from conftest import rel_err
from objective_checks import dense_system, reduced, total_cost

GROUP = np.array([0, 0, 5, -1, 5, 0, 3, 5])  # groups {0, 1, 5} and {2, 4, 7}, camera 3 on its own, 6 a group of one


def _case(priors):
    """camera_prior_model.prior_case (8 cameras, the last without observations) with the members' intrinsics tied to their
    leads', and the prior kinds `priors` names"""
    from rootba_b200.synthetic import BalArrays
    prob, mean, L = pm.prior_case()
    lead = sm.leads(GROUP)
    cams = np.array(prob.cams, np.float64)
    g = lead >= 0
    cams[g, 7:] = cams[lead[g], 7:]
    prob = BalArrays(cams, np.asarray(prob.lms, np.float64), prob.lm_off, prob.obs_cam, np.asarray(prob.obs_xy, np.float64))
    model = {}
    if "camera" in priors:
        model["camera"] = (mean, L)
    if "pairs" in priors:
        rng = np.random.default_rng(5)
        pairs = np.array([[0, 1], [2, 4], [3, 5]], np.int32)
        model["pairs"] = (pairs, qm.mean_at(cams, pairs), np.stack([qm.sqrt_info_kind("dense", rng) for _ in pairs]))
    if "landmarks" in priors:
        model["landmarks"] = lp.prior_case(prob.lms)
    return prob, lead, model


def _with_cams(prob, cams):
    from rootba_b200.synthetic import BalArrays
    return BalArrays(cams, prob.lms, prob.lm_off, prob.obs_cam, prob.obs_xy)


PRIORS = [(), ("camera",), ("camera", "pairs", "landmarks")]


@pytest.mark.parametrize("priors", PRIORS, ids=lambda p: "-".join(p) or "none")
def test_tied_jacobian_against_central_differences(priors):
    prob, lead, model = _case(priors)
    Jp, _, _ = dense_system(prob, **model)
    P = sm.expansion(lead)
    Ju = Jp @ P
    h = 1e-6
    for k in range(P.shape[1]):
        e = np.zeros(P.shape[1])
        e[k] = h
        rp = dense_system(_with_cams(prob, sm.apply_tied(prob.cams, P @ e)), **model)[2]
        rm = dense_system(_with_cams(prob, sm.apply_tied(prob.cams, -P @ e)), **model)[2]
        fd = (rp - rm) / (2 * h)
        assert np.max(np.abs(fd - Ju[:, k])) <= 1e-5 * max(1.0, np.max(np.abs(Ju[:, k]))), k


@pytest.mark.parametrize("priors", PRIORS, ids=lambda p: "-".join(p) or "none")
def test_tied_lm_step_against_the_true_cost_change(priors):
    prob, lead, model = _case(priors)
    Jp, Jl, r = dense_system(prob, **model)
    lam = 1e-3
    D, sl, Jls, Minv, Hu, bu, P, E = sm.tied_step(Jp, Jl, r, lam, prob.nl, lead)
    u = -np.linalg.solve(Hu, bu)
    x_s = P @ u  # scaled increment in the 9 nc layout, members equal to their lead
    dl_s = -Minv @ (Jls.T @ r + Jls.T @ ((Jp * D) @ x_s))
    c0 = total_cost(prob, **model)
    for t in (1e-2, 1e-3):
        x, dl = t * D * x_s, t * sl * dl_s
        l_diff = 0.5 * r @ r - 0.5 * np.sum((r + Jp @ x + Jl @ dl) ** 2)
        from rootba_b200.synthetic import BalArrays
        new = BalArrays(sm.apply_tied(prob.cams, x), prob.lms + dl.reshape(-1, 3), prob.lm_off, prob.obs_cam, prob.obs_xy)
        true = c0 - total_cost(new, **model)
        assert abs(true - l_diff) <= 20 * t * abs(l_diff), (t, true, l_diff)
        # the members stay tied
        g = lead >= 0
        assert np.array_equal(new.cams[g, 7:], new.cams[lead[g], 7:])


def _systems(priors, lam, jacobi, summed_scaling=True):
    """(Hfull without the pose damping, b_full, per-camera blocks) of the full system under the group-summed scaling (or,
    planted fault, the per-camera scaling), and (H_u, b_u, lead, E) of the tied model"""
    prob, lead, model = _case(priors)
    Jp, Jl, r = dense_system(prob, **model)
    D, sl, Jls, Minv, Hu, bu, P, E = sm.tied_step(Jp, Jl, r, lam, prob.nl, lead)
    if not summed_scaling:
        D = reduced(Jp, Jl, r, lam, prob.nl)[0]
    Jps = Jp * D
    W = Jps.T @ Jls
    Hfull = Jps.T @ Jps - W @ Minv @ W.T
    b_full = Jps.T @ r - W @ Minv @ (Jls.T @ r)
    src = Jps.T @ Jps if jacobi else Hfull
    blocks = np.stack([src[9 * c:9 * c + 9, 9 * c:9 * c + 9] for c in range(prob.nc)])
    return Hfull, b_full, blocks, Hu, bu, lead, P, E


K, PERIOD = 8, 5  # iterations compared, one residual refresh included (before the rounding of either recurrence has grown)


def _reduced_pcg(Hu, bu, blocks, lam, lead):
    Mu = sm.reduced_block_jacobi(blocks, lam, lead)
    return pcg_run(lambda v: Hu @ v, bu, lambda v: Mu @ v)


def pcg_run(op, b, minv):
    from pcg_replay import pcg_replay
    return pcg_replay(op, b, minv, eta=-1.0, max_it=K, period=PERIOD)


def _max_iterate_err(ref, got, E):
    n = min(len(ref["xs"]), len(got["xs"]))
    assert n == K + 1, n
    return max(rel_err(got["xs"][k], E @ ref["xs"][k]) for k in range(1, n))


@pytest.mark.parametrize("jacobi", [False, True], ids=["SCHUR_JACOBI", "JACOBI"])
@pytest.mark.parametrize("priors", PRIORS, ids=lambda p: "-".join(p) or "none")
def test_device_recurrence_equals_pcg_on_the_tied_system(priors, jacobi):
    lam = 1e-3
    Hfull, b_full, blocks, Hu, bu, lead, P, E = _systems(priors, lam, jacobi)
    # the contraction of the full operator and gradient is the tied system
    assert rel_err(P.T @ Hfull @ P + lam * np.eye(len(bu)), Hu) < 1e-13
    assert rel_err(P.T @ b_full, bu) < 1e-13
    # the device's inverse blocks are M_u^-1 in the 9 nc layout
    inv = sm.device_blocks(blocks, lam, lead)
    Mu = sm.reduced_block_jacobi(blocks, lam, lead)
    x = np.random.default_rng(2).standard_normal(len(bu))
    from pcg_replay import block_apply
    assert rel_err(block_apply(inv, E @ x), E @ (Mu @ x)) < 1e-13
    # PCG on the tied system with its operator applied as P^T (H (P u)) + lambda u and M_u^-1 as the blocks just checked
    # (both equal to H_u and M_u above; the same products as the 9 nc replay, so that the iterates agree to rounding
    # rather than to kappa times it)
    ref = pcg_run(lambda v: P.T @ (Hfull @ (P @ v)) + lam * v, P.T @ b_full, lambda v: E.T @ block_apply(inv, E @ v))
    got = sm.replay_9nc(Hfull, b_full, blocks, lam, lead, eta=-1.0, max_it=K, period=PERIOD)
    assert _max_iterate_err(ref, got, E) < 1e-12
    assert np.allclose(got["alphas"], ref["alphas"], rtol=1e-12, atol=0) and np.allclose(got["zetas"], ref["zetas"], rtol=1e-10, atol=0)


@pytest.mark.parametrize("fault", ["lambda_per_member", "b_not_contracted", "x_not_expanded", "scaling_not_summed"])
def test_the_recurrence_check_catches_planted_faults(fault):
    lam = 1e-3
    summed = fault != "scaling_not_summed"
    Hfull, b_full, blocks, Hu, bu, lead, P, E = _systems(("camera",), lam, False, summed_scaling=summed)
    ref = _reduced_pcg(Hu, bu, *_systems(("camera",), lam, False)[2:3], lam, lead)
    got = sm.replay_9nc(Hfull, b_full, blocks, lam, lead, eta=-1.0, max_it=K, period=PERIOD, fault=None if fault == "scaling_not_summed" else fault)
    assert _max_iterate_err(ref, got, E) > 1e-6
    # the control: the correct replay is within the bar of the same comparison
    Hfull, b_full, blocks = _systems(("camera",), lam, False)[:3]
    ok = sm.replay_9nc(Hfull, b_full, blocks, lam, lead, eta=-1.0, max_it=K, period=PERIOD)
    assert _max_iterate_err(ref, ok, E) < 1e-8


def test_groups_of_one_camera_are_the_ungrouped_system():
    prob, _, model = _case(("camera",))
    lead = sm.leads(np.arange(prob.nc))
    assert np.all(lead == -1) and np.array_equal(sm.expansion(lead), np.eye(9 * prob.nc))
    Jp, Jl, r = dense_system(prob, **model)
    want = reduced(Jp, Jl, r, 1e-3, prob.nl)
    got = sm.tied_step(Jp, Jl, r, 1e-3, prob.nl, lead)
    for a, b in zip((want[0], want[1], want[3], want[4], want[5], want[6]), got[:6]):
        assert np.array_equal(a, b)
    # and a group id that only one camera carries is a group of one
    assert np.array_equal(sm.leads(np.array([4, -1, 0, 0])), np.array([-1, -1, 2, 2]))


def _reduced_camera_matrix(Jp, Jl):
    """the full reduced camera matrix of the covariance (unscaled, lambda = 0): Jp^T Jp - Jp^T Jl (Jl^T Jl)^+ Jl^T Jp"""
    W = Jp.T @ Jl
    return Jp.T @ Jp - W @ np.linalg.pinv(Jl.T @ Jl) @ W.T


@pytest.mark.parametrize("held", [False, True], ids=["priors", "priors-held-pose"])
def test_contracted_covariance_is_the_tied_covariance(held):
    from objective_checks import FIX_POSE, fixed_entries
    prob, lead, model = _case(("camera", "landmarks"))
    Jp, Jl, _ = dense_system(prob, **model)
    fixed9 = None
    if held:
        mask = np.zeros(prob.nc, np.uint8)
        mask[3] = FIX_POSE
        fixed9 = fixed_entries(mask)
    want, _ = sm.tied_covariance(Jp, Jl, lead, fixed9)
    A = _reduced_camera_matrix(Jp, Jl)
    assert rel_err(sm.contracted_covariance(A, lead, fixed9), want) < 1e-8
    # every member's block carries the group's intrinsics covariance
    g = lead >= 0
    assert np.array_equal(want[g][:, 6:, 6:], want[lead[g]][:, 6:, 6:])
    # the planted fault: contracted on rows only
    assert rel_err(sm.contracted_covariance(A, lead, fixed9, fault="rows_only"), want) > 1e-3
