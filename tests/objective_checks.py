"""Shared by the held-camera and prior tests: the held-camera flags, the dense float64 model of the total objective
(reprojection + camera priors + pair priors + landmark priors), one check of a handle's LM step against that model, an LM-step
harness, the scipy minimum of the total objective, and the two-rank launcher.  Not collected by pytest (no test_ prefix)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import camera_model as cm
import camera_prior_model as pm
import landmark_prior_model as lp
import pair_prior_model as qm
from conftest import ROOT, rel_err

# ---- held camera parameters (rba_set_camera_fixed) ----------------------------------------------------------------------
FIX_POSE, FIX_F, FIX_K1, FIX_K2 = 1, 2, 4, 8
# every bit, a combination of intrinsics, one fully fixed camera, free cameras
MASK = np.array([FIX_POSE, FIX_F, FIX_K1 | FIX_K2, FIX_POSE | FIX_F | FIX_K1 | FIX_K2, 0, FIX_F | FIX_K1 | FIX_K2, FIX_K2], np.uint8)
# camera parameter columns (quat xyzw, t, f, k1, k2) held by each RBA_FIX_* bit
_PARAM_COLS = {FIX_POSE: [0, 1, 2, 3, 4, 5, 6], FIX_F: [7], FIX_K1: [8], FIX_K2: [9]}


def fixed_entries(flags):
    """[9 nc] bool: increment entries (t, r, f, k1, k2 per camera) held by the RBA_FIX_* bits"""
    fx = np.zeros((len(flags), 9), bool)
    fx[:, :6] = (flags & FIX_POSE)[:, None] != 0
    fx[:, 6] = (flags & FIX_F) != 0
    fx[:, 7] = (flags & FIX_K1) != 0
    fx[:, 8] = (flags & FIX_K2) != 0
    return fx.ravel()


def fixed_params(flags):
    """[nc, 10] bool: camera parameters that must stay bit-identical"""
    out = np.zeros((len(flags), 10), bool)
    for bit, cols in _PARAM_COLS.items():
        out[np.ix_((flags & bit) != 0, cols)] = True
    return out


# ---- the dense model of the total objective -----------------------------------------------------------------------------
def dense_system(prob, camera=None, pairs=None, landmarks=None):
    """the dense (Jp, Jl, r) of the total objective, unscaled: the reprojection rows of
    tests/test_oracle_dense_numpy.py::_dense_system, then the rows of each prior kind given, camera (mean, L) ->
    pairs (pairs, mean, L) -> landmarks (idx, mean, L).  reduced() of it is the total LM step: the Jacobi scaling over the
    whole Jacobian, H, b, inc = -H^-1 b, l_diff."""
    from scipy.linalg import block_diag
    from test_oracle_dense_numpy import _dense_system
    Jp, Jl, r = _dense_system(prob)
    cam_rows = []
    if camera is not None:
        A, rc = pm.rows(prob.cams, *camera)
        cam_rows.append((block_diag(*A), rc.ravel()))
    if pairs is not None:
        cam_rows.append(qm.rows(prob.cams, *pairs))
    for Jq, rq in cam_rows:  # camera columns only
        Jp, Jl, r = np.vstack([Jp, Jq]), np.vstack([Jl, np.zeros((len(rq), Jl.shape[1]))]), np.concatenate([r, rq])
    if landmarks is not None:
        Jp, Jl, r = lp.append_rows((Jp, Jl, r), prob.nl, prob.lms, *landmarks)
    return Jp, Jl, r


def total_cost(prob, camera=None, pairs=None, landmarks=None):
    """reprojection (camera_model, no robust loss) + the cost of each prior kind given"""
    c = float(cm.compute_error(prob)["all"]["error"])
    if camera is not None:
        c += pm.cost(prob.cams, *camera)
    if pairs is not None:
        c += qm.cost(prob.cams, *pairs)
    if landmarks is not None:
        c += lp.cost(prob.lms, *landmarks)
    return c


def reduced(Jp, Jl, r, lam, nl, dtype=np.float64):
    """the dense derivation with the Jacobi-scaling epsilon of the handle's scalar type (sqrt of Sophus' epsilon)"""
    from test_oracle_dense_numpy import _reduced
    return _reduced(Jp, Jl, r, lam, nl, float(cm.EPS_SQRT[np.dtype(dtype)]))


# ---- one LM step of a handle against the dense model --------------------------------------------------------------------
CONFIGS = [dict(solver_type="SQUARE_ROOT", operator_form=op, use_householder_marginalization=hh, preconditioner_type=pc)
           for op in ("DENSE", "IMPLICIT") for hh in (True, False) for pc in ("JACOBI", "SCHUR_JACOBI")]
CONFIGS += [dict(solver_type="SCHUR_COMPLEMENT"), dict(solver_type="POWER_SCHUR_COMPLEMENT")]

cfg_id = lambda c: "-".join(str(v) for v in c.values())

# bars: those of test_gpu_fixed_cameras (float64) and test_gpu_sc / test_gpu_unobserved_cameras (float32)
BARS = {np.float64: dict(scaling=1e-12, b=1e-9, blocks=1e-9, inv=1e-8, op=1e-9, inc=1e-6, l_diff=1e-8, lms=1e-10, cost=1e-10),
        np.float32: dict(scaling=1e-5, b=1e-3, blocks=1e-3, inv=1e-3, op=1e-3, inc=1e-3, l_diff=1e-3, lms=1e-3, cost=1e-3)}


def bal_problem(arrays, dtype, **features):
    """a BalProblem of `arrays` with the features given that are not None (camera_fixed, camera_prior, camera_pair_prior,
    landmark_prior)"""
    import rootba_b200 as rb
    bp = rb.BalProblem.from_arrays(arrays, dtype)
    for name, value in features.items():
        if value is not None:
            setattr(bp, name, value)
    return bp


def _stored(prior, dtype):
    """a prior tuple (..., mean, L) with mean and L rounded to the handle's scalar type, in float64"""
    f = lambda a: np.asarray(np.asarray(a, dtype), np.float64)
    return None if prior is None else tuple(prior[:-2]) + (f(prior[-2]), f(prior[-1]))


def check_against_dense(cfg, prob, camera=None, pairs=None, landmarks=None, mask=None, dtype=np.float64, lam=1e-3, env=None,
                        inc_eta_kappa=False):
    """one LM step (compute_error, linearize, solve, apply) of a handle with the given priors and held-camera flags `mask`
    against the dense float64 model: the cost before and after, the Jacobi scaling, b, the block preconditioner, H x, the
    increment (by PCG or the power series), l_diff and the landmarks; held parameters bit-identical, the others moved.  The
    model is evaluated at the state, observations and prior arrays rounded to `dtype`, as the handle stores them.  `env`:
    test-hook variables in force while the handle is made.  inc_eta_kappa: in float64 the PCG increment bar is widened to
    sqrt(eta kappa(H_ff)), since the stopping test bounds the change of the quadratic model, which is second order in the
    error of the iterate."""
    import rootba_b200 as rb
    from rootba_b200.synthetic import BalArrays
    bars = BARS[dtype]
    f = lambda a: np.asarray(np.asarray(a, dtype), np.float64)
    sprob = BalArrays(f(prob.cams), f(prob.lms), prob.lm_off, prob.obs_cam, f(prob.obs_xy))
    model = dict(camera=_stored(camera, dtype), pairs=_stored(pairs, dtype), landmarks=_stored(landmarks, dtype))
    Jp, Jl, r = dense_system(sprob, **model)
    D, sl, Jps, Jls, Minv, H, b = reduced(Jp, Jl, r, lam, prob.nl, dtype)
    n = H.shape[0]
    fixed = fixed_entries(mask) if mask is not None else np.zeros(n, bool)
    free = ~fixed
    bp = bal_problem(prob, dtype, landmark_prior=landmarks, camera_pair_prior=pairs, camera_prior=camera, camera_fixed=mask)
    so = rb.SolverOptions(eta=1e-13, **cfg)
    with pytest.MonkeyPatch.context() as m:
        for k, v in (env or {}).items():
            m.setenv(k, v)
        lin = rb.LinearizorQR.create(bp, so)
    cams0 = bp.cams.copy()
    e0 = lin.compute_error()["all"]["error"]
    assert abs(e0 - total_cost(sprob, **model)) <= bars["cost"] * e0
    lin.linearize()
    inc = lin.solve(lam)
    s, _ = lin.get_jacobian_scaling()
    assert rel_err(s, D) < bars["scaling"]
    assert rel_err(lin.get_rhs(), np.where(fixed, 0.0, b)) < bars["b"]
    inv, blk = lin.get_preconditioner()
    power = cfg.get("solver_type") == "POWER_SCHUR_COMPLEMENT"
    jacobi = power or cfg.get("preconditioner_type") == "JACOBI"
    Hpp, O = qm.power_split(Jps, lam)  # Hpp: the JACOBI blocks, prior rows and pair diagonals included; O: the pair blocks
    if pairs is not None:
        assert np.max(np.abs(O)) > 0
    for c in range(prob.nc):
        sel = slice(9 * c, 9 * c + 9)
        Hc = Hpp[sel, sel] if jacobi else H[sel, sel]
        fc = free[sel]
        want = np.zeros((9, 9))
        want[np.ix_(fc, fc)] = np.linalg.inv(Hc[np.ix_(fc, fc)])
        assert rel_err(inv[c], want) < bars["inv"], c
        if not jacobi:  # the blocks are written with SCHUR_JACOBI (rba_get_preconditioner)
            assert rel_err(blk[c], H[sel, sel]) < bars["blocks"], c
    x = np.random.default_rng(1).uniform(-1, 1, n)
    assert rel_err(lin.right_multiply(x), H @ x) < bars["op"]
    assert np.all(inc[fixed] == 0)
    Hff, bf = H[np.ix_(free, free)], b[free]
    tol_inc = bars["inc"]
    if dtype == np.float32:
        # against the exact float64 solve a float32 PCG iterate carries ~ c k u kappa (test_gpu_pcg_iterates); c k = 100 covers
        # the ~20 iterations these solves run
        tol_inc = max(tol_inc, 100 * 2.0 ** -24 * np.linalg.cond(Hff))
    if power:
        # the series of k_power_vec on Hpp^-1 (E_0 - O) on the free entries
        W = Jps.T @ Jls
        E0mO = (W @ Minv @ W.T - O)[np.ix_(free, free)]
        acc = qm.power_series(Hpp[np.ix_(free, free)], E0mO, bf, so.power_order, so.eta)
        assert rel_err(inc[free], acc) < (1e-9 if dtype == np.float64 else tol_inc)
    else:
        if dtype == np.float64:
            assert lin.last_cg.termination_type == 1
            if inc_eta_kappa:
                tol_inc = max(tol_inc, np.sqrt(so.eta * np.linalg.cond(Hff)))
        assert rel_err(inc[free], -np.linalg.solve(Hff, bf)) < tol_inc
    inc64 = np.asarray(inc, np.float64)
    dl_s = -Minv @ (Jls.T @ r + Jls.T @ (Jps @ inc64))
    want_l = 0.5 * r @ r - 0.5 * np.sum((r + Jps @ inc64 + Jls @ dl_s) ** 2)
    l_diff = lin.apply(None)  # the device-resident increment
    assert abs(l_diff - want_l) <= bars["l_diff"] * abs(want_l)
    lin.download_state()
    assert rel_err(bp.lms, sprob.lms + (sl * dl_s).reshape(-1, 3)) < bars["lms"]
    # the exact total cost at the new state
    e1 = lin.compute_error()["all"]["error"]
    new = BalArrays(bp.cams.astype(np.float64), bp.lms.astype(np.float64), prob.lm_off, prob.obs_cam, sprob.obs_xy)
    want_e1 = total_cost(new, **model)
    assert abs(e1 - want_e1) <= bars["cost"] * want_e1
    fp = fixed_params(mask) if mask is not None else np.zeros(bp.cams.shape, bool)
    assert np.array_equal(bp.cams[fp], cams0[fp])
    assert not np.array_equal(bp.cams[~fp], cams0[~fp])
    lin.close()


# ---- no behaviour change without a feature ------------------------------------------------------------------------------
def lm_steps(arrays, dtype, options, mode, setter=None, value=None, camera_prior=None, steps=3):
    """`steps` LM steps (linearize, solve at lambda 1e-4, apply, download) of a handle whose feature was never set (mode
    "never"), or set by `setter(lin, ...)` before the first step: `value` then None ("set_then_none"), `value` then an empty
    one ("set_then_empty"), or `value` with a zero last array, the flags or the sqrt_info ("zeros").  camera_prior is set on
    the problem before the handle is made.  Returns the initial cost and per step (inc, l_diff, cams, lms, cost)."""
    import rootba_b200 as rb
    bp = bal_problem(arrays, dtype, camera_prior=camera_prior)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(**options))
    if mode in ("set_then_none", "set_then_empty"):
        setter(lin, value)
        setter(lin, None if mode == "set_then_none" else tuple(a[:0] for a in value))
    elif mode == "zeros":
        setter(lin, np.zeros_like(value) if isinstance(value, np.ndarray) else (*value[:-1], np.zeros_like(value[-1])))
    else:
        assert mode == "never", mode
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


def assert_identical_steps(ref, got, what):
    """two results of lm_steps bit for bit"""
    assert ref[0] == got[0], what
    for a, b in zip(ref[1], got[1]):
        assert np.array_equal(a[0], b[0]) and a[1] == b[1] and a[4] == b[4], what
        assert np.array_equal(a[2], b[2]) and np.array_equal(a[3], b[3]), what


# ---- LM runs ------------------------------------------------------------------------------------------------------------
def check_lm_run_equals_host_loop(arrays, so, **features):
    """rba_lm_run and bundle_adjust_manual on the same float64 problem: bit-identical trajectory (compared as
    test_native_lm_loop_equals_the_python_loop compares the two loops)"""
    import rootba_b200 as rb
    bp = bal_problem(arrays, np.float64, **features)
    lin = rb.LinearizorQR.create(bp, so)
    its, _, _ = lin.lm_run(64)
    lin.download_state()
    lin.close()
    bp2 = bal_problem(arrays, np.float64, **features)
    summ = rb.bundle_adjust_manual(bp2, so)
    host = summ["iterations"][1:]
    assert len(host) == len(its) and len(its) >= 2
    for h, n in zip(host, its):
        assert bool(h["step_is_successful"]) == n["accepted"] and h["lam"] == n["lambda"]
        assert h["linear_solver_iterations"] == n["cg_iterations"] and h["cost"]["all"]["error"] == n["cost"]
    assert np.array_equal(bp2.cams, bp.cams) and np.array_equal(bp2.lms, bp.lms)


def scipy_minimum(prob, camera=None, pairs=None, landmarks=None, mask=None):
    """scipy's least-squares minimum of the total objective over the cameras not held by `mask` (any flag holds the whole
    camera) and every landmark: (cams, lms, cost)"""
    from scipy.optimize import least_squares
    from scipy.spatial.transform import Rotation
    nc, nl = prob.nc, prob.nl
    free_c = np.arange(nc) if mask is None else np.flatnonzero(mask == 0)
    lm_of_obs = np.repeat(np.arange(nl), np.diff(prob.lm_off))
    base = np.asarray(prob.cams, np.float64)

    def unpack(x):
        pc = x[:9 * len(free_c)].reshape(-1, 9)
        cams = base.copy()
        cams[free_c, :4] = Rotation.from_rotvec(pc[:, :3]).as_quat()
        cams[free_c, 4:7], cams[free_c, 7:10] = pc[:, 3:6], pc[:, 6:9]
        return cams, x[9 * len(free_c):].reshape(nl, 3)

    def fun(x):
        cams, lms = unpack(x)
        out = [cm.linearize(cams[prob.obs_cam], lms[lm_of_obs], prob.obs_xy)["res"].ravel()]
        if landmarks is not None:
            out += [L @ (lms[i] - m) for i, m, L in zip(*landmarks)]
        if pairs is not None:
            out += [pairs[2][p] @ qm.residual(cams[i], cams[j], pairs[1][p]) for p, (i, j) in enumerate(pairs[0])]
        if camera is not None:
            out += [camera[1][c] @ pm.residual(cams[c], camera[0][c]) for c in range(nc)]
        return np.concatenate(out)

    x0 = np.concatenate([np.hstack([Rotation.from_quat(base[free_c, :4]).as_rotvec(), base[free_c, 4:10]]).ravel(), np.ravel(prob.lms)])
    sol = least_squares(fun, x0, method="trf", x_scale="jac", xtol=1e-15, ftol=1e-15, gtol=1e-15, max_nfev=200)
    cams, lms = unpack(sol.x)
    return cams, lms, float(sol.cost)


# ---- truncated PCG iterates ---------------------------------------------------------------------------------------------
K_TRUNC = 8


def check_truncated_pcg_iterates(arrays, operator_form, precond, **features):
    """pcg_replay on the handle's own b, M^-1 and right_multiply (which includes every prior term): iterates k = 1..8 at the
    bar of test_gpu_pcg_iterates (10 k u kappa)"""
    import rootba_b200 as rb
    from pcg_replay import NO_CONVERGENCE, lanczos_condition, pcg_replay
    from test_gpu_pcg_iterates import C_BAR, NEVER, U

    def handle(**opt):
        lin = rb.LinearizorQR.create(bal_problem(arrays, np.float64, **features),
                                     rb.SolverOptions(operator_form=operator_form, preconditioner_type=precond, **opt))
        lin.linearize()
        return lin

    lam = 1e-3
    lin = handle()
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
        h = handle(eta=NEVER, max_linear_solver_iterations=k)
        inc = h.solve(lam)
        assert np.array_equal(h.get_rhs(), b) and np.array_equal(h.get_preconditioner()[0], inv), k
        assert (h.last_cg.termination_type, h.last_cg.num_iterations) == (NO_CONVERGENCE, k)
        assert rel_err(inc, -ref["xs"][k]) < bars[k], (k, rel_err(inc, -ref["xs"][k]), bars[k])
        h.close()


# ---- two GPUs -----------------------------------------------------------------------------------------------------------
def ngpu():
    import torch
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


def run_two_ranks(tmp_path, worker, sfx, peer, port, offset, *args):
    """tests/<worker> <out.json> <sfx> <args> on 2 GPUs under torchrun with RBA_PEER_AR=peer (skipped with fewer): its JSON.
    The master port is port + (pid + offset) mod 2000, so that tests running side by side do not collide."""
    if ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    out = tmp_path / "res.json"
    env = dict(os.environ, RBA_PEER_AR=peer, MASTER_ADDR="127.0.0.1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(port + (os.getpid() + offset) % 2000), os.path.join(ROOT, "tests", worker), str(out), sfx, *args]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return json.loads(out.read_text())


def check_two_rank_step(tmp_path, kind, sfx, peer, port, offset):
    """multirank_step_worker.py: the sharded step of `kind` against the single-rank step, at the bars of
    test_gpu_multirank.py; the cost, which carries every prior term, for the prior kinds.  Returns the JSON."""
    res = run_two_ranks(tmp_path, "multirank_step_worker.py", sfx, peer, port, offset, kind)
    tols = 1e-4 if sfx == "f32" else 1e-8
    assert res["replicas_identical"], res
    assert res["b"] < 4 * tols and res["inc"] < tols and res["l_diff"] < 20 * tols, res
    assert res["lms"] < 10 * tols and res["cams"] < tols, res
    if kind != "fixed":
        assert res["cost"] < tols and res["cost0"] < tols, res
    return res
