"""preconditioner_type = CLUSTER_JACOBI (DESIGN.md section 28) on the GPU.

The cluster blocks read back (rba_get_cluster_preconditioner) are checked against the dense float64 model of the scaled,
damped reduced camera matrix restricted to each cluster, at the blocks bar of objective_checks.BARS.  The PCG recurrence is
replayed here in float64 with M^-1 as a callable built from the read-back blocks and S from rba_right_multiply, iterate by
iterate, at the bar of test_gpu_pcg_iterates (C k kappa u)."""
import ctypes as C

import numpy as np
import pytest

import objective_checks as oc
from conftest import rel_err

pytestmark = pytest.mark.gpu

U = {np.float64: 2.0 ** -53, np.float32: 2.0 ** -24}
DTYPES = [np.float64, np.float32]
dt_id = lambda d: np.dtype(d).name
CJ = dict(preconditioner_type="CLUSTER_JACOBI")
CONFIGS = [dict(solver_type="SQUARE_ROOT", operator_form=op, use_householder_marginalization=hh, **CJ)
           for op in ("DENSE", "IMPLICIT") for hh in (True, False)]
CONFIGS += [dict(solver_type="SCHUR_COMPLEMENT", **CJ)]
# nc = 8 (camera_prior_model.prior_case): clusters {0, 1, 2}, {3, 4}, {5}, {6, 7}; the pair (0, 1) inside a cluster,
# (3, 1) and (5, 6) across
CLUSTERS8 = np.array([0, 0, 0, 1, 1, 2, 3, 3], np.int32)
# every RBA_FIX_* bit, a fully held camera (3), free cameras
MASK = np.append(oc.MASK, 0).astype(np.uint8)


def _priors():
    import camera_prior_model as pm
    import landmark_prior_model as lp
    import pair_prior_model as qm
    prob, mean_c, L_c = pm.prior_case(7, 90)
    pairs = np.array([(0, 1), (3, 1), (5, 6)], np.int32)
    rng = np.random.default_rng(11)
    pmean = qm.mean_at(prob.cams, pairs)
    pmean[:, 4:7] += rng.normal(0, 0.05, (len(pairs), 3))
    pL = np.stack([qm.sqrt_info_kind("dense", rng) for _ in pairs])
    return prob, dict(camera=(mean_c, L_c), pairs=(pairs, pmean, pL), landmarks=lp.prior_case(prob.lms, every=2, seed=8))


def _rounded(prob, dtype):
    from rootba_b200.synthetic import BalArrays
    f = lambda a: np.asarray(np.asarray(a, dtype), np.float64)
    return BalArrays(f(prob.cams), f(prob.lms), prob.lm_off, prob.obs_cam, f(prob.obs_xy))


def _handle(prob, dtype, cfg, clusters=None, mask=None, **model):
    import rootba_b200 as rb
    bp = oc.bal_problem(prob, dtype, camera_fixed=mask, camera_prior=model.get("camera"), camera_pair_prior=model.get("pairs"),
                        landmark_prior=model.get("landmarks"))
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(**cfg))
    if clusters is not None:
        lin.set_camera_clusters(clusters)
    return bp, lin


def _masked(H, mask, nc):
    H = H.copy()
    if mask is not None:
        fx = oc.fixed_entries(mask)
        H[fx, :] = 0
        H[:, fx] = 0
        H[fx, fx] = 1
    return H


def _model_H(prob, dtype, lam, **model):
    Jp, Jl, r = oc.dense_system(_rounded(prob, dtype), **{k: oc._stored(v, dtype) for k, v in model.items()})
    return oc.reduced(Jp, Jl, r, lam, prob.nl, dtype)[5]


def _cluster_index(c):
    return [np.concatenate([np.arange(9 * cam, 9 * cam + 9) for cam in np.flatnonzero(c == k)]) for k in range(c.max() + 1)]


# ---- the cluster blocks ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=dt_id)
@pytest.mark.parametrize("cfg", CONFIGS, ids=oc.cfg_id)
def test_cluster_blocks_against_the_dense_model(cfg, dtype):
    """priors of every kind, a pair inside a cluster and two across (absent), held parameters with a fully held camera;
    clusters of 3, 2 and 1 cameras"""
    prob, model = _priors()
    lam = 1e-3
    H = _masked(_model_H(prob, dtype, lam, **model), MASK, prob.nc)
    bp, lin = _handle(prob, dtype, cfg, CLUSTERS8, MASK, **model)
    lin.compute_error()
    lin.linearize()
    lin.solve(lam)
    c, blocks, status = lin.cluster_preconditioner()
    assert np.array_equal(c, CLUSTERS8) and np.all(status == 0) and len(blocks) == 4
    for B, idx in zip(blocks, _cluster_index(c)):
        want = H[np.ix_(idx, idx)]
        assert np.array_equal(B, B.T)
        assert rel_err(B, want) < oc.BARS[dtype]["blocks"], (rel_err(B, want), idx[0] // 9)
    lin.close()


@pytest.mark.parametrize("dtype", DTYPES, ids=dt_id)
@pytest.mark.parametrize("k", [2, 15, 16])
def test_large_clusters_and_long_tracks(k, dtype):
    """clusters of 2, 15 and 16 cameras on an 18-camera problem with tracks up to 72 and two cameras without observations"""
    from rootba_b200.synthetic import BalArrays, synth_bal
    base = synth_bal(16, 160, 5.0, seed=7, max_track=72)
    cams = np.vstack([base.cams, base.cams[:2]])  # cameras 16 and 17 observe nothing
    prob = BalArrays(cams, base.lms, base.lm_off, base.obs_cam, base.obs_xy)
    assert np.diff(prob.lm_off).max() <= 72
    lam = 1e-3
    H = _model_H(prob, dtype, lam)
    c = (np.arange(prob.nc) // k).astype(np.int32)
    _, lin = _handle(prob, dtype, dict(CJ), c)
    lin.compute_error()
    lin.linearize()
    lin.solve(lam)
    c2, blocks, status = lin.cluster_preconditioner()
    assert np.array_equal(c2, c) and np.all(status == 0)
    for B, idx in zip(blocks, _cluster_index(c)):
        assert rel_err(B, H[np.ix_(idx, idx)]) < oc.BARS[dtype]["blocks"]
    lin.close()


# ---- singletons: SCHUR_JACOBI -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=dt_id)
def test_singleton_clusters_are_schur_jacobi(dtype):
    prob, model = _priors()
    lam = 1e-3
    single = np.arange(prob.nc, dtype=np.int32)
    _, lin = _handle(prob, dtype, dict(CJ), single, MASK, **model)
    _, ref = _handle(prob, dtype, dict(preconditioner_type="SCHUR_JACOBI"), None, MASK, **model)
    for h in (lin, ref):
        h.compute_error()
        h.linearize()
    inc, inc_ref = lin.solve(lam), ref.solve(lam)
    _, blocks, status = lin.cluster_preconditioner()
    _, sj = ref.get_preconditioner()
    sj = np.asarray(sj, np.float64)
    fx = oc.fixed_entries(MASK).reshape(prob.nc, 9)
    for cam, B in enumerate(blocks):
        want = sj[cam].copy()
        want[fx[cam], :] = 0
        want[:, fx[cam]] = 0
        want[fx[cam], fx[cam]] = 1
        assert np.array_equal(B, want), cam
    assert np.all(status == 0)
    assert lin.last_cg.num_iterations == ref.last_cg.num_iterations
    assert rel_err(inc, inc_ref) < 100 * lin.last_cg.num_iterations * 1e3 * U[dtype]
    lin.close(); ref.close()


# ---- one cluster of all cameras: M = S --------------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg", [CONFIGS[0], CONFIGS[3], CONFIGS[4]], ids=oc.cfg_id)
def test_one_cluster_is_the_exact_step(cfg):
    prob, model = _priors()
    lam = 1e-3
    dtype = np.float64
    cfg = dict(cfg, max_linear_solver_iterations=1)
    bp, lin = _handle(prob, dtype, cfg, np.zeros(prob.nc, np.int32), MASK, **model)
    lin.compute_error()
    lin.linearize()
    inc = lin.solve(lam)
    assert lin.last_cg.num_iterations == 1
    b = lin.get_rhs()
    H = _masked(_model_H(prob, dtype, lam, **model), MASK, prob.nc)
    kappa = np.linalg.cond(H)
    assert rel_err(inc, -np.linalg.solve(H, b)) < 1000 * kappa * U[dtype]
    dense = {k: v for k, v in cfg.items() if k != "preconditioner_type"}
    _, dl = _handle(prob, dtype, dict(dense, linear_solver_type="DENSE_SCHUR"), None, MASK, **model)
    dl.compute_error()
    dl.linearize()
    assert rel_err(inc, dl.solve(lam)) < 1000 * kappa * U[dtype]
    lin.close(); dl.close()


# ---- the PCG recurrence, replayed ------------------------------------------------------------------------------------------
def _replay(S, b, Minv, k):
    x = np.zeros_like(b); r = b.copy(); z = Minv(r); p = z.copy(); rho = r @ z
    for _ in range(k):
        q = S @ p
        a = rho / (p @ q)
        x += a * p; r -= a * q
        z = Minv(r)
        rho, rho0 = r @ z, rho
        p = z + rho / rho0 * p
    return x


@pytest.mark.parametrize("env", [{}, {"RBA_PCG_PARTIALS": "0"}, {"RBA_ASSEMBLED_AT": "3"}], ids=["partials", "counter", "assembled"])
def test_pcg_iterates_against_a_float64_replay(env, monkeypatch):
    """x_k of the handle (max = min = k iterations) against the replay on S (rba_right_multiply) and M (read back), k = 1..6"""
    for k_, v in env.items():
        monkeypatch.setenv(k_, v)
    prob, model = _priors()
    lam, dtype = 1e-3, np.float64
    n = 9 * prob.nc
    S = b = Minv = None
    for k in range(1, 7):
        cfg = dict(CJ, min_linear_solver_iterations=k, max_linear_solver_iterations=k, eta=1e-300)
        _, lin = _handle(prob, dtype, cfg, CLUSTERS8, MASK, **model)
        lin.compute_error()
        lin.linearize()
        inc = lin.solve(lam)
        if S is None:
            S = np.stack([lin.right_multiply(e) for e in np.eye(n)], axis=1)
            fx = oc.fixed_entries(MASK)
            b = lin.get_rhs().astype(np.float64)
            c, blocks, _ = lin.cluster_preconditioner()
            M = np.zeros((n, n))
            for B, idx in zip(blocks, _cluster_index(c)):
                M[np.ix_(idx, idx)] = B
            Mi = np.linalg.inv(M)
            Minv = lambda r: np.where(fx, 0.0, Mi @ np.where(fx, 0.0, r))
            kappa = np.linalg.cond(_masked(S, MASK, prob.nc))
        assert lin.last_cg.num_iterations == k
        want = -_replay(S, b, Minv, k)
        assert rel_err(inc, want) < 10 * k * kappa * U[dtype], (k, rel_err(inc, want))
        lin.close()


# ---- fallback ---------------------------------------------------------------------------------------------------------------
def test_fallback_at_lambda_zero_with_a_rank_deficient_cluster():
    """one cluster of all cameras at lambda = 0 without priors: the cluster block has the 7-dimensional gauge null space, a
    pivot fails, the cluster falls back to its cameras' SCHUR_JACOBI blocks, and PCG runs"""
    from rootba_b200.synthetic import synth_bal
    prob = synth_bal(6, 120, 4.0, seed=3)
    _, lin = _handle(prob, np.float64, dict(CJ, max_linear_solver_iterations=20), np.zeros(prob.nc, np.int32))
    lin.compute_error()
    lin.linearize()
    inc = lin.solve(0.0)
    _, _, status = lin.cluster_preconditioner()
    assert status.tolist() == [1]
    assert lin.last_cg.num_iterations >= 1 and np.all(np.isfinite(inc))
    lin.close()


# ---- determinism ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=dt_id)
def test_bit_identical_increments(dtype):
    import rootba_b200 as rb
    prob, model = _priors()
    runs = []
    for _ in range(2):
        bp, lin = _handle(prob, dtype, dict(CJ), None, **model)
        lin.compute_error()
        lin.linearize()
        runs += [lin.solve(1e-3), lin.solve(1e-3)]
        lin.set_camera_clusters(CLUSTERS8)
        other = lin.solve(1e-3)
        lin.set_camera_clusters(rb.cluster_cameras(bp, 4))  # the default clustering (RBA_CLUSTER_DEFAULT_CAMERAS), given explicitly
        runs.append(lin.solve(1e-3))
        lin.set_camera_clusters(CLUSTERS8)
        assert np.array_equal(lin.solve(1e-3), other)
        lin.close()
    assert all(np.array_equal(r, runs[0]) for r in runs)


# ---- protocol ---------------------------------------------------------------------------------------------------------------
def test_rejected_calls_leave_the_handle_untouched():
    from rootba_b200 import _lib
    L = _lib.lib()
    prob, model = _priors()
    bp, lin = _handle(prob, np.float64, dict(CJ), CLUSTERS8, **model)
    lin.compute_error()
    lin.linearize()
    inc = lin.solve(1e-3)
    bad = [np.array([0, 0, 0, 1, 1, 2, 8, 3], np.int32), np.array([0, 0, 0, 2, 2, 3, 4, 4], np.int32),
           np.array([0, 0, 0, 1, 1, -1, 2, 2], np.int32)]
    for c in bad:
        assert L.rba_set_camera_clusters(lin.h, c.ctypes.data_as(C.c_void_p)) == -1
    assert L.rba_set_intrinsics_groups(lin.h, np.array([0, 0, -1, -1, -1, -1, -1, -1], np.int32).ctypes.data_as(C.c_void_p)) == -4
    rig = np.array([0, 0, -1, -1, -1, -1, -1, -1], np.int32)
    E = np.tile(np.array([0, 0, 0, 1, 0, 0, 0], np.float64), (prob.nc, 1))
    assert L.rba_set_camera_rigs(lin.h, rig.ctypes.data, E.ctypes.data) == -4
    assert L.rba_set_rig_sensors(lin.h, np.array([0, -1, -1, -1, -1, -1, -1, -1], np.int32).ctypes.data) == -4
    # a trivial tie is accepted
    assert L.rba_set_intrinsics_groups(lin.h, np.full(prob.nc, -1, np.int32).ctypes.data_as(C.c_void_p)) == 0
    c, _, _ = lin.cluster_preconditioner()
    assert np.array_equal(c, CLUSTERS8)
    lin.linearize()
    assert np.array_equal(lin.solve(1e-3), inc)
    _, ref = _handle(prob, np.float64, dict(preconditioner_type="SCHUR_JACOBI"))
    assert L.rba_set_camera_clusters(ref.h, None) == -6
    assert L.rba_get_cluster_preconditioner(ref.h, None, None, None) == -6
    lin.close(); ref.close()


# ---- end to end -------------------------------------------------------------------------------------------------------------
def test_lm_run_reaches_the_scipy_minimum():
    import pair_prior_model as qm
    import rootba_b200 as rb
    from rootba_b200.synthetic import synth_bal
    prob = synth_bal(8, 100, 4.0, seed=5)
    pairs = np.array([(i + 1, i) for i in range(prob.nc - 1)], np.int32)
    mean = qm.mean_at(prob.cams, pairs)
    mean[:, 4:7] += np.random.default_rng(2).normal(0, 0.05, (len(pairs), 3))
    pr = (pairs, mean, np.tile(np.eye(6) * 3.0, (len(pairs), 1, 1)))
    from rootba_b200.synthetic import BalArrays
    so = rb.SolverOptions(max_num_iterations=60, function_tolerance=1e-15, **CJ)
    bp = oc.bal_problem(prob, np.float64, camera_pair_prior=pr)
    lin = rb.LinearizorQR.create(bp, so)
    lin.set_camera_clusters(rb.cluster_cameras(bp, 4))
    its, _, _ = lin.lm_run(60, so)
    lin.download_state()
    lin.close()
    _, _, want = oc.scipy_minimum(prob, pairs=pr)
    got = oc.total_cost(BalArrays(bp.cams, bp.lms, prob.lm_off, prob.obs_cam, prob.obs_xy), pairs=pr)
    assert abs(got - want) <= 1e-8 * want, (got, want, len(its))
