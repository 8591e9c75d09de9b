"""Gaussian camera priors (rba_set_camera_prior) on the GPU: every solver against the dense float64 algebra of the total
(reprojection + prior) problem, truncated PCG iterates, priors with held parameters, no behaviour change without priors,
an observation-free camera, an end-to-end minimum against scipy, bad input and the sharded path."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import camera_model as cm
import camera_prior_model as pm
from conftest import ROOT, rel_err
from test_camera_prior_model import prior_case, total_cost
from test_fixed_cameras import MASK, fixed_entries
from test_gpu_fixed_cameras import CONFIGS, fixed_params

pytestmark = pytest.mark.gpu

# bars: those of test_gpu_fixed_cameras (float64) and test_gpu_sc / test_gpu_unobserved_cameras (float32)
BARS = {np.float64: dict(scaling=1e-12, b=1e-9, blocks=1e-9, inv=1e-8, op=1e-9, inc=1e-6, l_diff=1e-8, lms=1e-10, cost=1e-10),
        np.float32: dict(scaling=1e-5, b=1e-3, blocks=1e-3, inv=1e-3, op=1e-3, inc=1e-3, l_diff=1e-3, lms=1e-3, cost=1e-3)}


def _reduced(Jp, Jl, r, lam, nl, dtype=np.float64):
    """the dense derivation with the Jacobi-scaling epsilon of the handle's scalar type (sqrt of Sophus' epsilon)"""
    from test_oracle_dense_numpy import _reduced as red
    return red(Jp, Jl, r, lam, nl, float(cm.EPS_SQRT[np.dtype(dtype)]))


def _check_against_dense(cfg, prob, mean, L, env, monkeypatch, dtype=np.float64, mask=None):
    import rootba_b200 as rb
    bars = BARS[dtype]
    lam = 1e-3
    Jp, Jl, r = pm.dense_system_with_prior(prob, mean, L)
    D, sl, Jps, Jls, Minv, H, b = _reduced(Jp, Jl, r, lam, prob.nl, dtype)
    n = H.shape[0]
    fixed = fixed_entries(mask) if mask is not None else np.zeros(n, bool)
    free = ~fixed
    bp = rb.BalProblem.from_arrays(prob, dtype)
    bp.camera_prior = (mean, L)
    if mask is not None:
        bp.camera_fixed = mask
    so = rb.SolverOptions(eta=1e-13, **cfg)
    with monkeypatch.context() as m:
        for k, v in env.items():
            m.setenv(k, v)
        lin = rb.LinearizorQR.create(bp, so)
    cams0 = bp.cams.copy()
    e0 = lin.compute_error()["all"]["error"]
    assert abs(e0 - total_cost(prob, mean, L)) <= bars["cost"] * e0
    lin.linearize()
    inc = lin.solve(lam)
    s, d2 = lin.get_jacobian_scaling()
    assert rel_err(s, D) < bars["scaling"]
    assert rel_err(lin.get_rhs(), np.where(fixed, 0.0, b)) < bars["b"]
    inv, blk = lin.get_preconditioner()
    power = cfg.get("solver_type") == "POWER_SCHUR_COMPLEMENT"
    jacobi = power or cfg.get("preconditioner_type") == "JACOBI"
    Hp = Jps.T @ Jps + lam * np.eye(n) if jacobi else H  # Jps holds the prior rows: Hpp + A^T A
    for c in range(prob.nc):
        sel = slice(9 * c, 9 * c + 9)
        f = free[sel]
        want = np.zeros((9, 9))
        want[np.ix_(f, f)] = np.linalg.inv(Hp[sel, sel][np.ix_(f, f)])
        assert rel_err(inv[c], want) < bars["inv"], c
        if not jacobi:  # the blocks are written with SCHUR_JACOBI (rba_get_preconditioner)
            assert rel_err(blk[c], Hp[sel, sel]) < bars["blocks"], c
    x = np.random.default_rng(1).uniform(-1, 1, n)
    assert rel_err(lin.right_multiply(x), H @ x) < bars["op"]
    assert np.all(inc[fixed] == 0)
    Hff, bf = H[np.ix_(free, free)], b[free]
    tol_inc = bars["inc"]
    if dtype == np.float32:
        # against the exact float64 solve a float32 PCG iterate carries ~ c k u kappa (test_gpu_pcg_iterates); c k = 100 covers
        # the ~20 iterations these solves run
        tol_inc = max(tol_inc, 100 * 2.0 ** -24 * np.linalg.cond(H[np.ix_(free, free)]))
    if power:
        # the series of k_power_vec on Hpp + A^T A (the JACOBI blocks) with E0 unchanged
        W = Jps.T @ Jls
        E0 = (W @ Minv @ W.T)[np.ix_(free, free)]
        Hinv = np.linalg.inv((Jps.T @ Jps + lam * np.eye(n))[np.ix_(free, free)])
        tmp = -Hinv @ bf
        acc = tmp.copy()
        for i in range(1, so.power_order + 1):
            tmp = Hinv @ (E0 @ tmp)
            acc = acc + tmp
            if i * np.linalg.norm(tmp) / np.linalg.norm(acc) < so.eta:
                break
        assert rel_err(inc[free], acc) < (1e-9 if dtype == np.float64 else tol_inc)
    else:
        if dtype == np.float64:
            assert lin.last_cg.termination_type == 1
        assert rel_err(inc[free], -np.linalg.solve(Hff, bf)) < tol_inc
    inc64 = np.asarray(inc, np.float64)
    dl_s = -Minv @ (Jls.T @ r + Jls.T @ (Jps @ inc64))
    want_l = 0.5 * r @ r - 0.5 * np.sum((r + Jps @ inc64 + Jls @ dl_s) ** 2)
    l_diff = lin.apply(None)
    assert abs(l_diff - want_l) <= bars["l_diff"] * abs(want_l)
    lin.download_state()
    assert rel_err(bp.lms, prob.lms + (sl * dl_s).reshape(-1, 3)) < bars["lms"]
    # the exact total cost at the new state
    from rootba_b200.synthetic import BalArrays
    e1 = lin.compute_error()["all"]["error"]
    want_e1 = total_cost(BalArrays(bp.cams.astype(np.float64), bp.lms.astype(np.float64), prob.lm_off, prob.obs_cam, prob.obs_xy), mean, L)
    assert abs(e1 - want_e1) <= bars["cost"] * want_e1
    if mask is not None:
        fp = fixed_params(mask)
        assert np.array_equal(bp.cams[fp], cams0[fp])
    lin.close()


_ID = lambda c: "-".join(str(v) for v in c.values())


@pytest.fixture(scope="module")
def case7():
    return prior_case(7, 90)


@pytest.fixture(scope="module")
def case120():
    return prior_case(120, 500, seed=5)


@pytest.mark.parametrize("cfg", CONFIGS, ids=_ID)
def test_f64_against_dense_system_with_priors(cfg, case7, monkeypatch):
    _check_against_dense(cfg, *case7, {}, monkeypatch)


@pytest.mark.parametrize("env", [{"RBA_PCG_CLUSTER": "1"}, {"RBA_PCG_PARTIALS": "0"}], ids=["one-cta", "no-partials"])
@pytest.mark.parametrize("cfg", CONFIGS, ids=_ID)
def test_f64_120_cameras_against_dense_system_with_priors(cfg, env, case120, monkeypatch):
    """RBA_PCG_CLUSTER=1: 120 cameras leave the register-resident layout of the vector step (its uncached path)"""
    _check_against_dense(cfg, *case120, env, monkeypatch)


@pytest.mark.parametrize("cfg", [CONFIGS[0], CONFIGS[2], CONFIGS[5], CONFIGS[8], CONFIGS[9]], ids=_ID)
def test_f32_against_dense_system_with_priors(cfg, case7, monkeypatch):
    _check_against_dense(cfg, *case7, {}, monkeypatch, dtype=np.float32)


@pytest.mark.parametrize("cfg", CONFIGS, ids=_ID)
def test_f64_priors_with_held_parameters_against_restricted_dense_system(cfg, case7, monkeypatch):
    prob = case7[0]
    _check_against_dense(cfg, *case7, {}, monkeypatch, mask=np.resize(MASK, prob.nc))


# ---- truncated PCG iterates -------------------------------------------------------------------------------------------
K_TRUNC = 8


def _seq_case():
    from rootba_b200.synthetic import synth_config
    arrays = synth_config("ladybug-1723", scale=0.05)
    rng = np.random.default_rng(11)
    mean = pm.mean_at(arrays.cams)
    mean[:, 4:7] += rng.normal(0, 0.1, (arrays.nc, 3))
    kinds = ["centre", "dense", "intrinsics", "none"]
    L = np.stack([pm.sqrt_info_kind(kinds[c % 4], rng, 0.5) for c in range(arrays.nc)])
    return arrays, mean, L


@pytest.fixture(scope="module")
def seq_prior():
    return _seq_case()


def _prior_handle(arrays, mean, L, dtype, **opt):
    import rootba_b200 as rb
    bp = rb.BalProblem.from_arrays(arrays, dtype)
    bp.camera_prior = (mean, L)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(**opt))
    lin.linearize()
    return lin


@pytest.mark.parametrize("operator_form", ["DENSE", "IMPLICIT"])
@pytest.mark.parametrize("precond", ["JACOBI", "SCHUR_JACOBI"])
def test_pcg_truncated_iterates_with_priors(seq_prior, operator_form, precond):
    """pcg_replay on the handle's own b, M^-1 and right_multiply (which includes A^T A): iterates k = 1..8 at the bar of
    test_gpu_pcg_iterates (10 k u kappa)"""
    from pcg_replay import NO_CONVERGENCE, lanczos_condition, pcg_replay
    from test_gpu_pcg_iterates import C_BAR, NEVER, U
    arrays, mean, L = seq_prior
    opt = dict(operator_form=operator_form, preconditioner_type=precond)
    lam = 1e-3
    lin = _prior_handle(arrays, mean, L, np.float64, **opt)
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
        h = _prior_handle(arrays, mean, L, np.float64, eta=NEVER, max_linear_solver_iterations=k, **opt)
        inc = h.solve(lam)
        assert np.array_equal(h.get_rhs(), b) and np.array_equal(h.get_preconditioner()[0], inv), k
        assert (h.last_cg.termination_type, h.last_cg.num_iterations) == (NO_CONVERGENCE, k)
        assert rel_err(inc, -ref["xs"][k]) < bars[k], (k, rel_err(inc, -ref["xs"][k]), bars[k])
        h.close()


# ---- held parameters through whole LM runs, no behaviour change without priors ------------------------------------------
def _small_prior(problem, seed=3):
    rng = np.random.default_rng(seed)
    mean = pm.mean_at(problem.cams)
    mean[:, 4:7] += rng.normal(0, 0.05, (problem.nc, 3))
    L = np.stack([pm.sqrt_info_kind(["centre", "dense", "intrinsics"][c % 3], rng) for c in range(problem.nc)])
    return mean, L


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_held_parameters_stay_fixed_with_priors_through_lm_run(small_problem, dtype):
    import rootba_b200 as rb
    so = rb.SolverOptions(max_num_iterations=8)
    flags = np.full(small_problem.nc, rb.FIX_INTRINSICS, np.uint8)
    flags[[0, 1]] = rb.FIX_ALL
    prior = _small_prior(small_problem)
    bp = rb.BalProblem.from_arrays(small_problem, dtype)
    bp.camera_fixed = flags
    bp.camera_prior = prior
    cams0 = bp.cams.copy()
    lin = rb.LinearizorQR.create(bp, so)
    its, _, _ = lin.lm_run(64)
    lin.download_state()
    lin.close()
    fp = fixed_params(flags)
    assert np.array_equal(bp.cams[fp], cams0[fp])
    assert not np.array_equal(bp.cams[~fp], cams0[~fp])
    acc = [it["cost"] for it in its if it["accepted"]]
    assert len(acc) >= 1 and all(b < a for a, b in zip(acc, acc[1:])), its


def _lm_steps(arrays, dtype, solver_type, mode, steps=3):
    import rootba_b200 as rb
    bp = rb.BalProblem.from_arrays(arrays, dtype)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(solver_type=solver_type))
    if mode == "set_then_none":
        lin.set_camera_prior(_small_prior(arrays))
        lin.set_camera_prior(None)
    elif mode == "zeros":
        lin.set_camera_prior((pm.mean_at(arrays.cams), np.zeros((arrays.nc, 9, 9))))
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


@pytest.mark.parametrize("solver_type", ["SQUARE_ROOT", "SCHUR_COMPLEMENT"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_no_behaviour_change_without_priors(small_problem, dtype, solver_type):
    c0, ref = _lm_steps(small_problem, dtype, solver_type, "never")
    c1, got = _lm_steps(small_problem, dtype, solver_type, "set_then_none")
    assert c0 == c1
    for a, b in zip(ref, got):
        assert np.array_equal(a[0], b[0]) and a[1] == b[1] and a[4] == b[4]
        assert np.array_equal(a[2], b[2]) and np.array_equal(a[3], b[3])
    if dtype == np.float64:
        c2, zeros = _lm_steps(small_problem, dtype, solver_type, "zeros")
        assert abs(c2 - c0) <= 1e-12 * c0
        for a, b in zip(ref, zeros):
            assert rel_err(b[0], a[0]) < 1e-12 and abs(b[1] - a[1]) <= 1e-12 * abs(a[1])
            assert rel_err(b[2], a[2]) < 1e-12 and rel_err(b[3], a[3]) < 1e-12


# ---- an observation-free camera ---------------------------------------------------------------------------------------
def test_unobserved_camera_with_intrinsics_prior_reaches_the_mean_in_one_step():
    """its prior residual is linear in f, k1, k2: one undamped step puts them at the prior mean.  The other cameras are held
    (rba_set_camera_fixed), so the reduced system is this camera's block alone, which the block preconditioner inverts
    exactly: the solve is exact rather than accurate to the PCG stopping rule of the whole problem."""
    import rootba_b200 as rb
    prob, _, _ = prior_case(7, 90, unobserved=True)
    mean = pm.mean_at(prob.cams)
    mean[-1, 7:10] = prob.cams[-1, 7:10] + [12.5, 0.03, -0.004]
    L = np.zeros((prob.nc, 9, 9))
    L[-1, 6:9, 6:9] = np.diag([0.05, 2.0, 4.0])
    bp = rb.BalProblem.from_arrays(prob, np.float64)
    bp.camera_prior = (mean, L)
    flags = np.full(prob.nc, rb.FIX_ALL, np.uint8)
    flags[-1] = 0
    bp.camera_fixed = flags
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(eta=1e-13))
    lin.compute_error()
    lin.linearize()
    lin.solve(1e-12)
    lin.apply(None)
    lin.download_state()
    lin.close()
    assert np.allclose(bp.cams[-1, 7:10], mean[-1, 7:10], rtol=1e-9, atol=1e-12), bp.cams[-1, 7:10] - mean[-1, 7:10]
    assert np.array_equal(bp.cams[-1, :7], prob.cams[-1, :7])  # no information on its pose: zero pose increment


# ---- end to end against scipy -----------------------------------------------------------------------------------------
def _e2e_problem():
    from rootba_b200.synthetic import BalArrays, synth_bal
    prob = synth_bal(8, 150, 4.0, seed=31)
    rng = np.random.default_rng(32)
    truth = np.asarray(prob.cams, np.float64)
    mean = pm.mean_at(truth)
    mean[:, 4:7] += rng.normal(0, 0.02, (prob.nc, 3))
    L = np.zeros((prob.nc, 9, 9))
    L[:, 0:3, 0:3] = 20.0 * np.eye(3)   # centres to ~0.05
    L[:, 6, 6] = 0.02                  # f to ~50 pixels
    L[:, 7:9, 7:9] = 10.0 * np.eye(2)  # k1, k2 to ~0.1
    cams = truth.copy()
    from scipy.spatial.transform import Rotation
    for c in range(prob.nc):
        cams[c, :4] = (Rotation.from_rotvec(rng.normal(0, 0.01, 3)) * Rotation.from_quat(cams[c, :4])).as_quat()
        cams[c, 4:7] += rng.normal(0, 0.02, 3)
        cams[c, 7] *= 1 + rng.normal(0, 0.01)
    lms = np.asarray(prob.lms) + rng.normal(0, 0.02, np.shape(prob.lms))
    return BalArrays(cams, lms, prob.lm_off, prob.obs_cam, prob.obs_xy), mean, L


def _scipy_minimum(prob, mean, L):
    from scipy.optimize import least_squares
    from scipy.spatial.transform import Rotation
    nc, nl = prob.nc, prob.nl
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
        pri = np.concatenate([L[c] @ pm.residual(cams[c], mean[c]) for c in range(nc)])
        return np.concatenate([res, pri])

    x0 = np.concatenate([np.hstack([Rotation.from_quat(prob.cams[:, :4]).as_rotvec(), prob.cams[:, 4:10]]).ravel(), np.ravel(prob.lms)])
    sol = least_squares(fun, x0, method="trf", x_scale="jac", xtol=1e-15, ftol=1e-15, gtol=1e-15, max_nfev=200)
    cams, lms = unpack(sol.x)
    return cams, lms, float(sol.cost)


def test_lm_run_reaches_the_scipy_minimum_of_the_total_objective():
    import rootba_b200 as rb
    prob, mean, L = _e2e_problem()
    cams_s, lms_s, cost_s = _scipy_minimum(prob, mean, L)
    so = rb.SolverOptions(max_num_iterations=60, function_tolerance=1e-15, eta=1e-10)
    runs = {}
    for dtype in (np.float64, np.float32):
        bp = rb.BalProblem.from_arrays(prob, dtype)
        bp.camera_prior = (mean, L)
        lin = rb.LinearizorQR.create(bp, so)
        its, _, _ = lin.lm_run(200)
        lin.download_state()
        cost = lin.compute_error()["all"]["error"]
        lin.close()
        runs[dtype] = (bp, its, cost)
    bp, its, cost = runs[np.float64]
    assert abs(cost - cost_s) <= 1e-9 * cost_s, (cost, cost_s)
    centres = np.stack([pm.centre(c) for c in bp.cams])
    assert rel_err(centres, np.stack([pm.centre(c) for c in cams_s])) < 1e-6
    assert rel_err(bp.cams[:, 7:10], cams_s[:, 7:10]) < 1e-6
    assert rel_err(bp.lms, lms_s) < 1e-6
    # float32 reaches the float64 minimum
    assert abs(runs[np.float32][2] - cost) <= 1e-4 * cost


def test_lm_run_with_priors_equals_the_python_host_loop():
    """rba_lm_run and bundle_adjust_manual on the same total objective: bit-identical trajectory (default LM options, under
    which test_native_lm_loop_equals_the_python_loop compares the two loops)"""
    import rootba_b200 as rb
    prob, mean, L = _e2e_problem()
    so = rb.SolverOptions(max_num_iterations=10)
    bp = rb.BalProblem.from_arrays(prob, np.float64)
    bp.camera_prior = (mean, L)
    lin = rb.LinearizorQR.create(bp, so)
    its, _, _ = lin.lm_run(64)
    lin.download_state()
    lin.close()
    bp2 = rb.BalProblem.from_arrays(prob, np.float64)
    bp2.camera_prior = (mean, L)
    summ = rb.bundle_adjust_manual(bp2, so)
    host = summ["iterations"][1:]
    assert len(host) == len(its) and len(its) >= 2
    for h, n in zip(host, its):
        assert bool(h["step_is_successful"]) == n["accepted"] and h["lam"] == n["lambda"]
        assert h["linear_solver_iterations"] == n["cg_iterations"] and h["cost"]["all"]["error"] == n["cost"]
    assert np.array_equal(bp2.cams, bp.cams) and np.array_equal(bp2.lms, bp.lms)


# ---- bad input --------------------------------------------------------------------------------------------------------
def test_bad_input_keeps_the_previous_priors(small_problem):
    import rootba_b200 as rb
    from rootba_b200 import _lib
    lib = _lib.lib()
    mean, L = _small_prior(small_problem)
    bp = rb.BalProblem.from_arrays(small_problem, np.float64)
    bp.camera_prior = (mean, L)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions())
    lin.compute_error()
    lin.linearize()
    inc_ref = lin.solve(1e-4)
    p = lambda a: C.c_void_p(a.ctypes.data)
    bad_nan = L.copy()
    bad_nan[3, 2, 2] = np.nan
    bad_q = mean.copy()
    bad_q[4, :4] *= 1.01
    for args in ((p(mean), p(bad_nan)), (p(mean), None), (None, p(L)), (p(bad_q), p(L))):
        assert lib.rba_set_camera_prior(lin.h, *args) == -1  # RBA_ERR_INVALID_ARGUMENT
        assert lib.rba_last_error()
    assert b"camera 4" in (lib.rba_set_camera_prior(lin.h, p(bad_q), p(L)), lib.rba_last_error())[1]
    # nothing changed: the same solve as before, and the handle is still linearised
    assert np.array_equal(lin.solve(1e-4), inc_ref)
    with pytest.raises(ValueError):
        lin.set_camera_prior((bad_q, L))
    assert bp.camera_prior[0] is not bad_q and np.array_equal(bp.camera_prior[0], mean)
    # a prior change needs a new linearisation
    lin.set_camera_prior((mean, L))
    with pytest.raises(rb.RbaError) as e:
        lin.solve(1e-4)
    assert e.value.code == -6  # RBA_ERR_STATE
    lin.linearize()
    assert np.array_equal(lin.solve(1e-4), inc_ref)
    lin.close()


# ---- two GPUs ---------------------------------------------------------------------------------------------------------
def _ngpu():
    import torch
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.parametrize("peer", ["1", "0"])
@pytest.mark.parametrize("sfx", ["f32", "f64"])
def test_two_ranks_with_priors(tmp_path, peer, sfx):
    """every prior term is added once, after the sum over the shards: the sharded step equals the single-rank step"""
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    out = tmp_path / "res.json"
    env = dict(os.environ, RBA_PEER_AR=peer, MASTER_ADDR="127.0.0.1")
    port = 29500 + (os.getpid() + (7 if peer == "1" else 0) + (13 if sfx == "f32" else 0)) % 2000
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "tests", "multirank_prior_worker.py"), str(out), sfx]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    res = json.loads(out.read_text())
    tols = 1e-4 if sfx == "f32" else 1e-8  # the bars of test_gpu_multirank.py
    assert res["replicas_identical"], res
    assert res["b"] < 4 * tols and res["inc"] < tols and res["l_diff"] < 20 * tols, res
    assert res["lms"] < 10 * tols and res["cams"] < tols and res["cost"] < tols and res["cost0"] < tols, res
