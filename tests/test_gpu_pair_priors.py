"""Relative pose priors between pairs of cameras (rba_set_camera_pair_prior) on the GPU: every solver against the dense
float64 algebra of the total (reprojection + pair prior) problem, with absolute priors and with held parameters, truncated
PCG iterates, no behaviour change without pair priors, an observation-free camera, an end-to-end minimum against scipy, bad
input and the sharded path."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import camera_model as cm
import camera_prior_model as pm
import pair_prior_model as qm
from conftest import ROOT, rel_err
from test_camera_prior_model import prior_case
from test_fixed_cameras import MASK, fixed_entries
from test_gpu_camera_priors import BARS, _ID, _ngpu, _reduced, _small_prior
from test_gpu_fixed_cameras import CONFIGS, fixed_params

pytestmark = pytest.mark.gpu


def _check_against_dense(cfg, prob, pair, env, monkeypatch, dtype=np.float64, mask=None, absp=None):
    import rootba_b200 as rb
    from rootba_b200.synthetic import BalArrays
    bars = BARS[dtype]
    lam = 1e-3
    Jp, Jl, r = qm.dense_system_with_pairs(prob, pair, absp)
    D, sl, Jps, Jls, Minv, H, b = _reduced(Jp, Jl, r, lam, prob.nl, dtype)
    n = H.shape[0]
    fixed = fixed_entries(mask) if mask is not None else np.zeros(n, bool)
    free = ~fixed
    bp = rb.BalProblem.from_arrays(prob, dtype)
    bp.camera_pair_prior = pair
    if absp is not None:
        bp.camera_prior = absp
    if mask is not None:
        bp.camera_fixed = mask
    so = rb.SolverOptions(eta=1e-13, **cfg)
    with monkeypatch.context() as m:
        for k, v in env.items():
            m.setenv(k, v)
        lin = rb.LinearizorQR.create(bp, so)
    cams0 = bp.cams.copy()
    e0 = lin.compute_error()["all"]["error"]
    assert abs(e0 - qm.total_cost(prob, pair, absp)) <= bars["cost"] * e0
    lin.linearize()
    inc = lin.solve(lam)
    s, _ = lin.get_jacobian_scaling()
    assert rel_err(s, D) < bars["scaling"]
    assert rel_err(lin.get_rhs(), np.where(fixed, 0.0, b)) < bars["b"]
    inv, blk = lin.get_preconditioner()
    power = cfg.get("solver_type") == "POWER_SCHUR_COMPLEMENT"
    jacobi = power or cfg.get("preconditioner_type") == "JACOBI"
    Hpp, O = qm.power_split(Jps, lam)  # Hpp: the JACOBI blocks with the pairs' diagonal blocks
    for c in range(prob.nc):
        sel = slice(9 * c, 9 * c + 9)
        Hc = Hpp[sel, sel] if jacobi else H[sel, sel]
        f = free[sel]
        want = np.zeros((9, 9))
        want[np.ix_(f, f)] = np.linalg.inv(Hc[np.ix_(f, f)])
        assert rel_err(inv[c], want) < bars["inv"], c
        if not jacobi:  # the blocks are written with SCHUR_JACOBI (rba_get_preconditioner)
            assert rel_err(blk[c], H[sel, sel]) < bars["blocks"], c
    # the full operator, off-diagonal pair blocks included
    assert np.max(np.abs(O)) > 0
    x = np.random.default_rng(1).uniform(-1, 1, n)
    assert rel_err(lin.right_multiply(x), H @ x) < bars["op"]
    assert np.all(inc[fixed] == 0)
    Hff, bf = H[np.ix_(free, free)], b[free]
    tol_inc = bars["inc"]
    if dtype == np.float32:
        tol_inc = max(tol_inc, 100 * 2.0 ** -24 * np.linalg.cond(Hff))  # as test_gpu_camera_priors
    if power:
        # the series of k_power_vec on Hpp^-1 (E_0 - O), E_0 - O = Hpp - H, on the free entries
        acc = qm.power_series(Hpp[np.ix_(free, free)], (Hpp - H)[np.ix_(free, free)], bf, so.power_order, so.eta)
        assert rel_err(inc[free], acc) < (1e-9 if dtype == np.float64 else tol_inc)
    else:
        if dtype == np.float64:
            assert lin.last_cg.termination_type == 1
            # the stopping test bounds the change of the quadratic model, which is second order in the error of the
            # iterate: a converged increment is accurate to about sqrt(eta kappa), above the bar for some configurations
            tol_inc = max(tol_inc, np.sqrt(so.eta * np.linalg.cond(Hff)))
        assert rel_err(inc[free], -np.linalg.solve(Hff, bf)) < tol_inc
    inc64 = np.asarray(inc, np.float64)
    dl_s = -Minv @ (Jls.T @ r + Jls.T @ (Jps @ inc64))
    want_l = 0.5 * r @ r - 0.5 * np.sum((r + Jps @ inc64 + Jls @ dl_s) ** 2)
    l_diff = lin.apply(None)
    assert abs(l_diff - want_l) <= bars["l_diff"] * abs(want_l)
    lin.download_state()
    assert rel_err(bp.lms, prob.lms + (sl * dl_s).reshape(-1, 3)) < bars["lms"]
    e1 = lin.compute_error()["all"]["error"]
    want_e1 = qm.total_cost(BalArrays(bp.cams.astype(np.float64), bp.lms.astype(np.float64), prob.lm_off, prob.obs_cam, prob.obs_xy),
                            pair, absp)
    assert abs(e1 - want_e1) <= bars["cost"] * want_e1
    if mask is not None:
        fp = fixed_params(mask)
        assert np.array_equal(bp.cams[fp], cams0[fp])
    lin.close()


@pytest.fixture(scope="module")
def case7():
    return qm.pair_case(7, 90)


@pytest.fixture(scope="module")
def case120():
    return qm.pair_case(120, 500, seed=5)


@pytest.mark.parametrize("cfg", CONFIGS, ids=_ID)
def test_f64_against_dense_system_with_pair_priors(cfg, case7, monkeypatch):
    _check_against_dense(cfg, *case7, {}, monkeypatch)


@pytest.mark.parametrize("env", [{"RBA_PCG_CLUSTER": "1"}, {"RBA_PCG_PARTIALS": "0"}], ids=["one-cta", "no-partials"])
@pytest.mark.parametrize("cfg", CONFIGS, ids=_ID)
def test_f64_120_cameras_against_dense_system_with_pair_priors(cfg, env, case120, monkeypatch):
    """RBA_PCG_CLUSTER=1: 120 cameras leave the register-resident layout of the vector step (its uncached path)"""
    _check_against_dense(cfg, *case120, env, monkeypatch)


@pytest.mark.parametrize("cfg", [CONFIGS[0], CONFIGS[2], CONFIGS[5], CONFIGS[8], CONFIGS[9]], ids=_ID)
def test_f32_against_dense_system_with_pair_priors(cfg, case7, monkeypatch):
    _check_against_dense(cfg, *case7, {}, monkeypatch, dtype=np.float32)


@pytest.mark.parametrize("cfg", CONFIGS, ids=_ID)
def test_f64_pair_and_absolute_priors_against_dense_system(cfg, case7, monkeypatch):
    prob, pair = case7
    _, mean_a, L_a = prior_case(7, 90)
    _check_against_dense(cfg, prob, pair, {}, monkeypatch, absp=(mean_a, L_a))


@pytest.mark.parametrize("cfg", CONFIGS, ids=_ID)
def test_f64_pair_priors_with_held_parameters_against_restricted_dense_system(cfg, case7, monkeypatch):
    """MASK holds every parameter of camera 3, which pairs (2, 3) and (3, 4) join to free cameras"""
    prob = case7[0]
    _check_against_dense(cfg, *case7, {}, monkeypatch, mask=np.resize(MASK, prob.nc))


# ---- truncated PCG iterates -------------------------------------------------------------------------------------------
K_TRUNC = 8


@pytest.fixture(scope="module")
def seq_pairs():
    from rootba_b200.synthetic import synth_config
    arrays = synth_config("ladybug-1723", scale=0.05)
    rng = np.random.default_rng(12)
    pairs = np.array([(c, c + 1) for c in range(arrays.nc - 1)] + [(c + 5, c) for c in range(0, arrays.nc - 5, 3)], np.int32)
    mean = qm.mean_at(arrays.cams, pairs)
    mean[:, 4:7] += rng.normal(0, 0.1, (len(pairs), 3))
    kinds = ["dense", "translation", "rotation", "none"]
    L = np.stack([qm.sqrt_info_kind(kinds[p % 4], rng, 0.5) for p in range(len(pairs))])
    return arrays, (pairs, mean, L)


def _pair_handle(arrays, pair, dtype, **opt):
    import rootba_b200 as rb
    bp = rb.BalProblem.from_arrays(arrays, dtype)
    bp.camera_pair_prior = pair
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(**opt))
    lin.linearize()
    return lin


@pytest.mark.parametrize("operator_form", ["DENSE", "IMPLICIT"])
@pytest.mark.parametrize("precond", ["JACOBI", "SCHUR_JACOBI"])
def test_pcg_truncated_iterates_with_pair_priors(seq_pairs, operator_form, precond):
    """pcg_replay on the handle's own b, M^-1 and right_multiply (which includes the off-diagonal pair blocks): iterates
    k = 1..8 at the bar of test_gpu_pcg_iterates (10 k u kappa)"""
    from pcg_replay import NO_CONVERGENCE, lanczos_condition, pcg_replay
    from test_gpu_pcg_iterates import C_BAR, NEVER, U
    arrays, pair = seq_pairs
    opt = dict(operator_form=operator_form, preconditioner_type=precond)
    lam = 1e-3
    lin = _pair_handle(arrays, pair, np.float64, **opt)
    lin.solve(lam)
    b, inv = lin.get_rhs(), lin.get_preconditioner()[0]
    op = lambda v: lin.right_multiply(np.asarray(v, np.float64))
    full = pcg_replay(op, b, inv, eta=0.0, max_it=600)
    lmin, lmax = lanczos_condition(full["alphas"], full["betas"])
    bars = [C_BAR * max(k, 1) * U[np.float64] * lmax / lmin for k in range(K_TRUNC + 1)]
    assert full["iterations"] >= K_TRUNC and bars[K_TRUNC] <= 1e-8
    ref = pcg_replay(op, b, inv, eta=NEVER, max_it=K_TRUNC)
    lin.close()
    for k in range(1, K_TRUNC + 1):
        assert rel_err(ref["xs"][k], ref["xs"][k - 1]) > 100 * bars[k], k
        h = _pair_handle(arrays, pair, np.float64, eta=NEVER, max_linear_solver_iterations=k, **opt)
        inc = h.solve(lam)
        assert np.array_equal(h.get_rhs(), b) and np.array_equal(h.get_preconditioner()[0], inv), k
        assert (h.last_cg.termination_type, h.last_cg.num_iterations) == (NO_CONVERGENCE, k)
        assert rel_err(inc, -ref["xs"][k]) < bars[k], (k, rel_err(inc, -ref["xs"][k]), bars[k])
        h.close()


# ---- no behaviour change without pair priors ----------------------------------------------------------------------------
def _chain_pairs(problem, seed=4):
    rng = np.random.default_rng(seed)
    pairs = np.array([(c, c + 1) for c in range(problem.nc - 1)], np.int32)
    mean = qm.mean_at(problem.cams, pairs)
    mean[:, 4:7] += rng.normal(0, 0.05, (len(pairs), 3))
    L = np.stack([qm.sqrt_info_kind(["dense", "translation", "rotation"][p % 3], rng) for p in range(len(pairs))])
    return pairs, mean, L


def _lm_steps(arrays, dtype, solver_type, mode, absolute=False, steps=3):
    import rootba_b200 as rb
    bp = rb.BalProblem.from_arrays(arrays, dtype)
    if absolute:
        bp.camera_prior = _small_prior(arrays)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(solver_type=solver_type))
    if mode == "set_then_none":
        lin.set_camera_pair_prior(_chain_pairs(arrays))
        lin.set_camera_pair_prior(None)
    elif mode == "zeros":
        pairs, mean, L = _chain_pairs(arrays)
        lin.set_camera_pair_prior((pairs, mean, np.zeros_like(L)))
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


@pytest.mark.parametrize("absolute", [False, True], ids=["no-priors", "absolute-priors"])
@pytest.mark.parametrize("solver_type", ["SQUARE_ROOT", "SCHUR_COMPLEMENT", "POWER_SCHUR_COMPLEMENT"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_no_behaviour_change_without_pair_priors(small_problem, dtype, solver_type, absolute):
    """pair priors set and cleared, or all with a zero L: the LM trajectory of a handle that never had any, bit for bit
    (with and without absolute priors)"""
    c0, ref = _lm_steps(small_problem, dtype, solver_type, "never", absolute)
    for mode in ("set_then_none", "zeros"):
        c1, got = _lm_steps(small_problem, dtype, solver_type, mode, absolute)
        assert c0 == c1, mode
        for a, b in zip(ref, got):
            assert np.array_equal(a[0], b[0]) and a[1] == b[1] and a[4] == b[4], mode
            assert np.array_equal(a[2], b[2]) and np.array_equal(a[3], b[3]), mode


# ---- an observation-free camera ---------------------------------------------------------------------------------------
def test_unobserved_camera_tied_by_a_strong_pair_prior_reaches_the_relative_pose_in_one_step():
    """the last camera has no observations; a strong dense pair prior ties it to camera 0 at a relative pose away from the
    current one.  The other cameras are held, so the reduced system is this camera's pose block, and one nearly undamped
    step puts T_last T_0^-1 at the prior mean (the residual is nearly linear in the pose of the last camera for a small move)"""
    import rootba_b200 as rb
    from scipy.spatial.transform import Rotation
    prob, _ = qm.pair_case(7, 90)
    n = prob.nc
    mean = qm.mean_at(prob.cams, [(n - 1, 0)])
    mean[0, 4:7] += [0.02, -0.01, 0.015]
    mean[0, :4] = (Rotation.from_rotvec([0.003, -0.002, 0.001]) * Rotation.from_quat(mean[0, :4])).as_quat()
    pair = (np.array([(n - 1, 0)], np.int32), mean, 1e3 * np.eye(6)[None])
    bp = rb.BalProblem.from_arrays(prob, np.float64)
    bp.camera_pair_prior = pair
    flags = np.full(n, rb.FIX_ALL, np.uint8)
    flags[-1] = rb.FIX_INTRINSICS
    bp.camera_fixed = flags
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(eta=1e-13))
    e0 = lin.compute_error()["all"]["error"]
    lin.linearize()
    lin.solve(1e-12)
    lin.apply(None)
    lin.download_state()
    lin.close()
    e = qm.residual(bp.cams[-1], bp.cams[0], mean[0])
    e_before = qm.residual(prob.cams[-1], prob.cams[0], mean[0])
    assert np.linalg.norm(e) < 1e-3 * np.linalg.norm(e_before), (e, e_before)
    assert np.array_equal(bp.cams[:-1], prob.cams[:-1])


# ---- end to end against scipy -----------------------------------------------------------------------------------------
def _e2e_problem():
    """a perturbed synthetic problem with pair priors between consecutive cameras and a loop closure (sigma 1 on translation,
    0.01 rad on rotation)"""
    from rootba_b200.synthetic import BalArrays, synth_bal
    from scipy.spatial.transform import Rotation
    prob = synth_bal(8, 150, 4.0, seed=31)
    rng = np.random.default_rng(33)
    truth = np.asarray(prob.cams, np.float64)
    pairs = np.array([(c, c + 1) for c in range(prob.nc - 1)] + [(prob.nc - 1, 0)], np.int32)
    mean = qm.mean_at(truth, pairs)
    mean[:, 4:7] += rng.normal(0, 0.01, (len(pairs), 3))
    L = np.tile(np.diag([1.0, 1.0, 1.0, 100.0, 100.0, 100.0]), (len(pairs), 1, 1))  # sigma 1 and 0.01 rad
    cams = truth.copy()
    for c in range(prob.nc):
        cams[c, :4] = (Rotation.from_rotvec(rng.normal(0, 0.01, 3)) * Rotation.from_quat(cams[c, :4])).as_quat()
        cams[c, 4:7] += rng.normal(0, 0.02, 3)
        cams[c, 7] *= 1 + rng.normal(0, 0.01)
    lms = np.asarray(prob.lms) + rng.normal(0, 0.02, np.shape(prob.lms))
    return BalArrays(cams, lms, prob.lm_off, prob.obs_cam, prob.obs_xy), (pairs, mean, L)


def _scipy_minimum(prob, pair):
    from scipy.optimize import least_squares
    from scipy.spatial.transform import Rotation
    nc, nl = prob.nc, prob.nl
    pairs, mean, L = pair
    lm_of_obs = np.repeat(np.arange(nl), np.diff(prob.lm_off))

    def unpack(x):
        pc = x[:9 * nc].reshape(nc, 9)
        cams = np.zeros((nc, 10))
        cams[:, :4] = Rotation.from_rotvec(pc[:, :3]).as_quat()
        cams[:, 4:7], cams[:, 7:10] = pc[:, 3:6], pc[:, 6:9]
        return cams, x[9 * nc:].reshape(nl, 3)

    def fun(x):
        cams, lms = unpack(x)
        res = cm.linearize(cams[prob.obs_cam], lms[lm_of_obs], prob.obs_xy)["res"].ravel()
        pri = np.concatenate([L[p] @ qm.residual(cams[i], cams[j], mean[p]) for p, (i, j) in enumerate(pairs)])
        return np.concatenate([res, pri])

    x0 = np.concatenate([np.hstack([Rotation.from_quat(prob.cams[:, :4]).as_rotvec(), prob.cams[:, 4:10]]).ravel(), np.ravel(prob.lms)])
    sol = least_squares(fun, x0, method="trf", x_scale="jac", xtol=1e-15, ftol=1e-15, gtol=1e-15, max_nfev=200)
    cams, lms = unpack(sol.x)
    return cams, lms, float(sol.cost)


def test_lm_run_reaches_the_scipy_minimum_of_the_total_objective():
    """the cost at the minimum is gauge-free; the relative poses of the pairs are compared (the pair priors and reprojections
    leave the similarity gauge free, so absolute poses may differ between the two solvers)"""
    import rootba_b200 as rb
    prob, pair = _e2e_problem()
    cams_s, _, cost_s = _scipy_minimum(prob, pair)
    so = rb.SolverOptions(max_num_iterations=60, function_tolerance=1e-15, eta=1e-10)
    runs = {}
    for dtype in (np.float64, np.float32):
        bp = rb.BalProblem.from_arrays(prob, dtype)
        bp.camera_pair_prior = pair
        lin = rb.LinearizorQR.create(bp, so)
        lin.lm_run(200)
        lin.download_state()
        cost = lin.compute_error()["all"]["error"]
        lin.close()
        runs[dtype] = (bp, cost)
    bp, cost = runs[np.float64]
    assert abs(cost - cost_s) <= 1e-8 * cost_s, (cost, cost_s)
    pairs, mean, L = pair
    e_gpu = np.stack([qm.residual(bp.cams[i], bp.cams[j], mean[p]) for p, (i, j) in enumerate(pairs)])
    e_ref = np.stack([qm.residual(cams_s[i], cams_s[j], mean[p]) for p, (i, j) in enumerate(pairs)])
    assert np.max(np.abs(e_gpu - e_ref)) < 1e-4 * max(1.0, np.max(np.abs(e_ref)))
    assert abs(runs[np.float32][1] - cost) <= 1e-4 * cost


def test_lm_run_with_pair_priors_equals_the_python_host_loop():
    import rootba_b200 as rb
    prob, pair = _e2e_problem()
    so = rb.SolverOptions(max_num_iterations=10)
    bp = rb.BalProblem.from_arrays(prob, np.float64)
    bp.camera_pair_prior = pair
    lin = rb.LinearizorQR.create(bp, so)
    its, _, _ = lin.lm_run(64)
    lin.download_state()
    lin.close()
    bp2 = rb.BalProblem.from_arrays(prob, np.float64)
    bp2.camera_pair_prior = pair
    summ = rb.bundle_adjust_manual(bp2, so)
    host = summ["iterations"][1:]
    assert len(host) == len(its) and len(its) >= 2
    for h, n in zip(host, its):
        assert bool(h["step_is_successful"]) == n["accepted"] and h["lam"] == n["lambda"]
        assert h["linear_solver_iterations"] == n["cg_iterations"] and h["cost"]["all"]["error"] == n["cost"]
    assert np.array_equal(bp2.cams, bp.cams) and np.array_equal(bp2.lms, bp.lms)


# ---- bad input --------------------------------------------------------------------------------------------------------
def test_bad_input_keeps_the_previous_pair_priors(small_problem):
    import rootba_b200 as rb
    from rootba_b200 import _lib
    lib = _lib.lib()
    pairs, mean, L = _chain_pairs(small_problem)
    bp = rb.BalProblem.from_arrays(small_problem, np.float64)
    bp.camera_pair_prior = (pairs, mean, L)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions())
    lin.compute_error()
    lin.linearize()
    inc_ref = lin.solve(1e-4)
    p = lambda a: C.c_void_p(a.ctypes.data)
    m = C.c_int32(len(pairs))
    bad_nan_L, bad_nan_m = L.copy(), mean.copy()
    bad_nan_L[3, 2, 2] = np.nan
    bad_nan_m[2, 5] = np.inf
    bad_q = mean.copy()
    bad_q[4, :4] *= 1.01
    out_of_range, self_pair, negative = pairs.copy(), pairs.copy(), pairs.copy()
    out_of_range[5, 1] = small_problem.nc
    self_pair[6, 1] = self_pair[6, 0]
    negative[7, 0] = -1
    cases = [(C.c_int32(-1), p(pairs), p(mean), p(L)), (m, None, p(mean), p(L)), (m, p(pairs), None, p(L)), (m, p(pairs), p(mean), None),
             (m, p(out_of_range), p(mean), p(L)), (m, p(self_pair), p(mean), p(L)), (m, p(negative), p(mean), p(L)),
             (m, p(pairs), p(mean), p(bad_nan_L)), (m, p(pairs), p(bad_nan_m), p(L)), (m, p(pairs), p(bad_q), p(L))]
    for args in cases:
        assert lib.rba_set_camera_pair_prior(lin.h, *args) == -1  # RBA_ERR_INVALID_ARGUMENT
        assert lib.rba_last_error()
    assert b"pair 4" in (lib.rba_set_camera_pair_prior(lin.h, m, p(pairs), p(bad_q), p(L)), lib.rba_last_error())[1]
    # nothing changed: the same solve as before, and the handle is still linearised
    assert np.array_equal(lin.solve(1e-4), inc_ref)
    for bad in ((pairs, bad_q, L), (out_of_range, mean, L), (self_pair, mean, L), (pairs, mean, bad_nan_L), (pairs[:, :1], mean, L)):
        with pytest.raises(ValueError):
            lin.set_camera_pair_prior(bad)
    assert np.array_equal(bp.camera_pair_prior[1], mean)
    # a change needs a new linearisation
    lin.set_camera_pair_prior((pairs, mean, L))
    with pytest.raises(rb.RbaError) as e:
        lin.solve(1e-4)
    assert e.value.code == -6  # RBA_ERR_STATE
    lin.linearize()
    assert np.array_equal(lin.solve(1e-4), inc_ref)
    lin.close()


# ---- two GPUs ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("peer", ["1", "0"])
@pytest.mark.parametrize("sfx", ["f32", "f64"])
def test_two_ranks_with_pair_priors(tmp_path, peer, sfx):
    """every pair term is added once, after the sum over the shards: the sharded step equals the single-rank step"""
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    out = tmp_path / "res.json"
    env = dict(os.environ, RBA_PEER_AR=peer, MASTER_ADDR="127.0.0.1")
    port = 29500 + (os.getpid() + (11 if peer == "1" else 0) + (17 if sfx == "f32" else 0)) % 2000
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "tests", "multirank_pair_worker.py"), str(out), sfx]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    res = json.loads(out.read_text())
    tols = 1e-4 if sfx == "f32" else 1e-8  # the bars of test_gpu_multirank.py
    assert res["replicas_identical"], res
    assert res["b"] < 4 * tols and res["inc"] < tols and res["l_diff"] < 20 * tols, res
    assert res["lms"] < 10 * tols and res["cams"] < tols and res["cost"] < tols and res["cost0"] < tols, res
