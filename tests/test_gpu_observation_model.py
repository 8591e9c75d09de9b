"""The observation linearisation on the GPU against the independent float64 camera model (tests/camera_model.py) on inputs
the benign stand-ins never produce: real lens distortion, Huber weights on both sides of the threshold, invalid projections
(turned-around cameras, landmarks with 0, 1 or 2 valid observations) and points behind a camera with validity ignored.

Inputs (every problem has landmarks of track lengths 2..40: lanes per landmark G = 1..32 and row-chunked tracks, see
paths() of test_gpu_kernel_classes):
  distorted   k1 ~ N(0, 0.1^2), k2 ~ N(0, 0.02^2), field of view +-56 degrees (|x/z| <= 1.5)
  huber       the same with the Huber threshold between the two residual norms around the median
  valid       ERROR_VALID, cameras 0..3 turned around (every observation they have is invalid) and landmarks with exactly
              0, 1 or 2 valid observations
  behind      ERROR (validity ignored) on the same problem: points behind a camera, z < 0, are linearised like any other

Per-landmark Gram invariant (independent of the oracle).  Q is orthogonal, so the damped block B = Q^T [Jp_s Jl_s r; 0 sqrt(lam) I
0] of debug_get_block satisfies, column pair by column pair,
    B_Jp^T B_Jp = Jp_s^T Jp_s,  B_Jp^T B_Jl = Jp_s^T Jl_s,  B_Jl^T B_Jl = Jl_s^T Jl_s + lam I,  B_Jl^T B_r = Jl_s^T r
(the Jl and r columns of rows 3.. are reported as 0, so the last three use rows 0..2).  ||r|| in the bar is the norm of
the residual's rounding scale sqrt(w) (|proj| + |obs|): a residual is the difference of two pixel positions.  The model side is built from the
model's Jacobians, weighted with the model's Huber weight, scaled with the kernel's own D and jls (cast exactly) and with the
rows of invalid observations zeroed.  This holds however the Householder vectors of a rank-deficient landmark came out, which
is why such landmarks are checked through it and not entry by entry.  Bar, normwise per column pair:
    |G - G^|_ab <= c u ||a|| ||b||,   c = 2 (c_qr + c_lin),   c_qr = 6 (2 n + 3) + 36,   c_lin = 256 kappa
u the unit round-off of the kernel's type.  Householder QR and a sequence of Givens rotations applied to a matrix with m rows
are columnwise backward stable: Q^T (A + dA) with ||dA_j|| <= gamma_{c m} ||A_j||, c a small constant (Higham, Accuracy and
Stability of Numerical Algorithms, 2nd ed., Thm 19.4 and 19.10); 6 (2 n + 3) covers the 3 reflectors or the chains of
rotations on the 2 n rows, 36 the 6 damping rotations.  c_lin is the bar of the per-observation linearisation against the
model (tests/test_camera_model.py), kappa the largest camera_model.condition() of the landmark's observations (it adds the
Huber weight's division by the residual to the bar of the linearisation).  D and jls are held to (300 + 4 m) u kappa
relative, m the observations in the column sum.  ||a|| of a Jp column is the norm of its rows' largest entries times the
column's scaling, because the linearisation bar is relative to the largest entry of a row.  The factor 2 is the Gram of a perturbed pair,
(a + da)^T (b + db) - a^T b <= (||da|| ||b|| + ||a|| ||db||).
"""
import functools

import numpy as np
import pytest

import camera_model as cm
from conftest import rel_err
from test_gpu_kernel_classes import _per_camera, paths
from test_gpu_parity import TOL1, TOLB, TOLS, make_pair

pytestmark = pytest.mark.gpu

NS = (2, 3, 4, 7, 12, 20, 30, 40)        # G = 1, 2, 2, 4, 8, 16, 16 (chunked), 32 (chunked)
TURNED = (0, 1, 2, 3)
SPECIAL = ((2, 0), (3, 0), (4, 0), (2, 1), (3, 1), (5, 1), (3, 2), (6, 2))  # (track length, valid observations)
LAM = 0.1
assert {paths(n)["G"] for n in NS} == {1, 2, 4, 8, 16, 32} and paths(40)["chunks"] > 1


def _u(dtype):
    return float(np.finfo(dtype).eps) / 2


@functools.lru_cache(maxsize=None)
def turned_problem():
    """cameras 0..3 turned around; SPECIAL landmarks first (their valid count is exact), then 12 landmarks per length in NS
    on random cameras (some of them turned)"""
    from rootba_b200.synthetic import synth_bal, turn_cameras_around
    rng = np.random.default_rng(77)
    nc = 48
    rest = np.arange(len(TURNED), nc)
    tracks = [np.concatenate([rng.choice(TURNED, n - v, replace=False), rng.choice(rest, v, replace=False)]) for n, v in SPECIAL]
    tracks += [rng.choice(nc, n, replace=False) for n in NS for _ in range(12)]
    a = synth_bal(nc, len(tracks), 0.0, seed=78, tracks=tracks, lm_spread=0.5, k1_sigma=0.05, k2_sigma=0.01)
    return turn_cameras_around(a, TURNED)


@functools.lru_cache(maxsize=None)
def distorted_problem():
    from rootba_b200.synthetic import synth_bal
    a = synth_bal(60, 300, 9.0, seed=79, max_track=40, max_tan=1.5, k1_sigma=0.1, k2_sigma=0.02)
    n = a.track_lengths()
    assert {paths(k)["G"] for k in np.unique(n)} == {1, 2, 4, 8, 16, 32} and n.max() >= 25
    return a


def _huber_threshold(arrays, dtype):
    """a threshold between the two residual norms around the median, at least 1e-3 relative away from both"""
    L = cm.linearize(*cm.observations(arrays.cast(dtype)), dtype=dtype)
    r = np.sort(np.sqrt((L["res"] ** 2).sum(1)))
    k = len(r) // 2
    while r[k + 1] - r[k] < 2e-3 * r[k]:
        k += 1
    return float(0.5 * (r[k] + r[k + 1]))


INPUTS = {
    "distorted": (distorted_problem, {}),
    "huber": (distorted_problem, {"robust_norm": "HUBER"}),
    "valid": (turned_problem, {"optimized_cost": "ERROR_VALID"}),
    "behind": (turned_problem, {"optimized_cost": "ERROR"}),
}


def _setup(which, dtype, **kw):
    make, opts = INPUTS[which]
    arrays = make()
    opts = dict(opts, **kw)
    th = None
    if opts.get("robust_norm") == "HUBER":
        th = _huber_threshold(arrays, dtype)
        opts["huber_parameter"] = th
    valid_only = opts.get("optimized_cost", "ERROR") != "ERROR"
    if which == "valid":
        L = cm.linearize(*cm.observations(arrays.cast(dtype)), dtype=dtype)
        lm_of_obs = np.repeat(np.arange(arrays.nl), arrays.track_lengths())
        nvalid = np.bincount(lm_of_obs, weights=L["valid"], minlength=arrays.nl)
        assert [int(v) for v in nvalid[:len(SPECIAL)]] == [v for _, v in SPECIAL]
        assert not np.any(L["valid"][np.isin(arrays.obs_cam, TURNED)]) and np.all(L["valid"][~np.isin(arrays.obs_cam, TURNED)])
    if which == "behind":
        z = cm.linearize(*cm.observations(arrays))["pc"][:, 2]
        assert np.sum(z < 0) > 50 and np.abs(z).min() > 1.0
    return arrays, opts, th, valid_only


def _model_rows(arrays, dtype, th, valid_only):
    """per observation: weighted Jp (2 x 9), Jl (2 x 3), r (2) in float64 from the dtype-cast state, the kept mask and the
    rounding scale of r"""
    return cm.weighted(arrays.cast(dtype), dtype=dtype, threshold=th, valid_only=valid_only, magnitude=True)


def _model_scaling(arrays, jp, jl, dtype):
    eps = float(cm.EPS_SQRT[np.dtype(dtype)])
    d2 = np.zeros((arrays.nc, 9))
    np.add.at(d2, arrays.obs_cam, (jp ** 2).sum(1))
    lm_of_obs = np.repeat(np.arange(arrays.nl), arrays.track_lengths())
    l2 = np.zeros((arrays.nl, 3))
    np.add.at(l2, lm_of_obs, (jl ** 2).sum(1))
    return 1 / (eps + np.sqrt(d2)), 1 / (eps + np.sqrt(l2))


@pytest.mark.parametrize("qr", ["householder", "givens"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("which", list(INPUTS))
def test_landmark_blocks_against_the_model(which, dtype, qr):
    arrays, opts, th, valid_only = _setup(which, dtype)
    bp, lin, o, _ = make_pair(arrays, dtype, use_householder_marginalization=(qr == "householder"), **opts)
    u = _u(dtype)
    lin.linearize()
    assert o.linearize()
    lin.solve(LAM)
    o.solve(LAM)
    D = lin.get_jacobian_scaling()[0].astype(np.float64).reshape(-1, 9)
    jp, jl, r, keep, rmag = _model_rows(arrays, dtype, th, valid_only)
    D_m, jls_m = _model_scaling(arrays, jp, jl, dtype)
    m_cam = np.bincount(arrays.obs_cam, minlength=arrays.nc).max()
    kap = cm.condition(arrays.cast(dtype), dtype, th)
    k_cam = np.ones(arrays.nc)
    np.maximum.at(k_cam, arrays.obs_cam, kap)
    assert np.all(np.abs(D - D_m) <= (300 + 4 * m_cam) * u * k_cam[:, None] * D_m), np.max(np.abs(D - D_m) / D_m)
    exact = 0
    for lm in range(arrays.nl):
        s, e = int(arrays.lm_off[lm]), int(arrays.lm_off[lm + 1])
        n, cams = e - s, arrays.obs_cam[s:e]
        bg, lm_idx, res_idx, jls_g = lin.debug_get_block(lm)
        jls = jls_g.astype(np.float64)
        k_lm = kap[s:e].max()
        assert np.all(np.abs(jls - jls_m[lm]) <= (300 + 4 * n) * u * k_lm * jls_m[lm]), (lm, jls, jls_m[lm], k_lm)
        # structure: R upper triangular, the Jl and r columns of rows 3.. zero
        B = bg.astype(np.float64)
        assert np.all(np.tril(B[:3, lm_idx:lm_idx + 3], -1) == 0) and np.all(B[3:, lm_idx:] == 0), lm
        # model side
        Jps_full = np.zeros((2 * n, 9 * n))
        for i in range(n):
            Jps_full[2 * i:2 * i + 2, 9 * i:9 * i + 9] = jp[s + i] * D[cams[i]]
        Jls = (jl[s:e] * jls).reshape(2 * n, 3)
        rw = r[s:e].reshape(2 * n)
        A, R, q = B[:, :9 * n], B[:3, lm_idx:lm_idx + 3], B[:3, res_idx]
        # the linearisation bar is per row (relative to the row's largest entry), so the Jp column scale is the norm of the
        # row maxima times the column's scaling
        na = (np.linalg.norm(np.abs(jp[s:e]).max(axis=2), axis=1)[:, None] * D[cams]).ravel()
        nl_, nr = np.sqrt((Jls ** 2).sum(0) + LAM), np.linalg.norm(rmag[s:e])
        c = 2 * (6 * (2 * n + 3) + 36 + 256 * k_lm)
        for got, want, bound, what in (
                (A.T @ A, Jps_full.T @ Jps_full, np.outer(na, na), "JpJp"),
                (A[:3].T @ R, Jps_full.T @ Jls, np.outer(na, nl_), "JpJl"),
                (R.T @ R, Jls.T @ Jls + LAM * np.eye(3), np.outer(nl_, nl_), "JlJl"),
                (R.T @ q, Jls.T @ rw, nl_ * nr, "Jlr")):
            err = np.abs(got - want)
            assert np.all(err <= c * u * bound), (what, lm, n, float(np.max(err / np.maximum(bound, 1e-300))) / u)
        nvalid = int(keep[s:e].sum())
        bc, _, _, jls_c = o.get_block(lm)
        if nvalid == 0:
            # no valid observation: R_d = sqrt(lam) I (sign from make_givens), everything else 0, jls = 1 / eps
            assert np.array_equal(bg, bc) and np.array_equal(jls_g, jls_c), lm
            assert np.all(jls_g == dtype(1) / cm.EPS_SQRT[np.dtype(dtype)])
            exact += 1
            continue
        sv = np.linalg.svd(Jls, compute_uv=False)
        if sv[-1] > 1e-3 * sv[0] and k_lm < 10:  # well conditioned: a unique factorisation, compared at the single-stage bars
            tol = TOL1[dtype]
            assert rel_err(jls_g, jls_c) < tol, lm
            assert rel_err(bg[:3, :9 * n], bc[:3, :9 * n]) < tol * 4, lm
            assert rel_err(np.triu(bg[:3, lm_idx:lm_idx + 3]), np.triu(bc[:3, lm_idx:lm_idx + 3])) < tol * 4, lm
            assert rel_err(bg[:3, res_idx], bc[:3, res_idx]) < tol * 4, lm
            assert rel_err(bg[3:, :9 * n], bc[3:, :9 * n]) < tol * 4, lm
    assert exact == (3 if which == "valid" else 0)
    lin.close()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("which", list(INPUTS))
def test_compute_error_against_the_model(which, dtype):
    arrays, opts, th, _ = _setup(which, dtype)
    bp, lin, o, _ = make_pair(arrays, dtype, **opts)
    g, c = lin.compute_error(), o.compute_error()
    want = cm.compute_error(arrays.cast(dtype), dtype=dtype, threshold=th)
    assert g["is_numerically_valid"]
    for key in ("all", "valid"):
        assert g[key]["num_obs"] == c[key]["num_obs"] == want[key]["num_obs"], key
        for q in ("error", "residual_sum"):
            if dtype == np.float64:
                tol = 1e-12 * want[key][q]
            else:  # test_gpu_parity.py::test_compute_error: 3x the distance of the float32 oracle from float64, + 1e-5
                tol = 3 * abs(c[key][q] - want[key][q]) + 1e-5 * want[key][q]
            assert abs(g[key][q] - want[key][q]) <= tol, (key, q, g[key][q], want[key][q])
    if which in ("valid", "behind"):
        assert 0 < g["valid"]["num_obs"] < g["all"]["num_obs"]
    lin.close()


def _boundary_problem(dtype, z_far):
    """two identical cameras with the identity rotation and t = 0 (pc = p exactly); landmark 0 at z = sqrt(eps), landmark 1
    one ulp below, landmark 2 at `z_far`"""
    from rootba_b200.synthetic import BalArrays
    e = cm.EPS_SQRT[np.dtype(dtype)]
    zs = np.array([e, np.nextafter(e, dtype(0)), z_far], dtype=dtype)
    cams = np.tile(np.array([0, 0, 0, 1, 0, 0, 0, 500, 0, 0], dtype=np.float64), (2, 1))
    lms = np.stack([0.1 * zs, -0.05 * zs, zs], axis=1).astype(dtype)
    obs = np.array([[50.0, -25.0]] * 6) + np.arange(12).reshape(6, 2)
    return BalArrays(cams, lms.astype(np.float64), np.array([0, 2, 4, 6]), np.array([0, 1] * 3, np.int32), obs)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_validity_threshold_is_inclusive(dtype):
    """z = sqrt(eps) exactly is valid, one ulp below is not (the >= rule on both sides; pc is exact with the identity camera)"""
    import rootba_b200 as rb
    a = _boundary_problem(dtype, 10.0)
    assert np.array_equal(a.cast(dtype).lms.astype(np.float64), a.lms)
    bp, lin, o, _ = make_pair(a, dtype, optimized_cost="ERROR_VALID")
    g, c = lin.compute_error(), o.compute_error()
    want = cm.compute_error(a, dtype=dtype)
    assert g["valid"]["num_obs"] == c["valid"]["num_obs"] == want["valid"]["num_obs"] == 4
    assert g["all"]["num_obs"] == 6
    lin.close()
    # z = 0 exactly with validity ignored: the projection is not finite, compute_error says so and linearize raises
    bp, lin, o, _ = make_pair(_boundary_problem(dtype, 0.0), dtype, optimized_cost="ERROR")
    assert not lin.compute_error()["is_numerically_valid"] and not o.compute_error()["is_numerically_valid"]
    with pytest.raises(rb.RbaError):
        lin.linearize()
    assert not o.linearize()
    lin.close()


SOLVERS = {"qr-dense": dict(solver_type="SQUARE_ROOT"), "qr-implicit": dict(solver_type="SQUARE_ROOT", operator_form="IMPLICIT"),
           "sc": dict(solver_type="SCHUR_COMPLEMENT"), "power-sc": dict(solver_type="POWER_SCHUR_COMPLEMENT")}
SC_TOL = {np.float32: 1e-3, np.float64: 1e-9}  # test_gpu_sc


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("which", ["valid", "behind"])
@pytest.mark.parametrize("solver", list(SOLVERS))
def test_solvers_downstream(solver, which, dtype):
    import rootba_b200 as rb
    from oracle import oracle_py as orc
    arrays, opts, th, valid_only = _setup(which, dtype)
    so = rb.SolverOptions(**SOLVERS[solver])
    so.optimized_cost = opts["optimized_cost"]
    bp = rb.BalProblem.from_arrays(arrays, dtype)
    lin = rb.LinearizorQR.create(bp, so)
    o = orc.Oracle(arrays, dtype, orc.default_options(num_threads=0, use_valid_projections_only=int(valid_only),
                                                      optimized_cost=1 if valid_only else 0))
    nc, u = arrays.nc, _u(dtype)
    lin.linearize()
    inc = lin.solve(LAM)
    b, (inv, _) = lin.get_rhs(), lin.get_preconditioner()
    if so.solver_type == "SQUARE_ROOT":
        assert o.linearize()
        inc_c, dbg = o.solve(LAM, want_debug=True)
        imp = so.operator_form == "IMPLICIT" and dtype == np.float32
        _per_camera(b, dbg["b"], nc, 4 * TOL1[dtype] * (10 if imp else 1), "b")
        _per_camera(inv, dbg["inv_blocks"], nc, TOLB[dtype] * (10 if imp else 1), "preconditioner inverse")
        _per_camera(inc, inc_c, nc, TOLS[dtype] * (5 if imp else 1), "inc")
    else:
        o.scl_linearize()
        if so.solver_type == "SCHUR_COMPLEMENT":
            inc_c, dbg = o.scl_solve(LAM)
            _per_camera(inv, dbg["inv_blocks"], nc, 10 * SC_TOL[dtype], "preconditioner inverse")
            _per_camera(inc, inc_c, nc, 10 * SC_TOL[dtype], "inc")
        else:
            inc_c, dbg = o.scl_power_solve(LAM, so.power_order, so.eta)
            assert abs(lin.last_cg.num_iterations - dbg["power_order"]) <= 1
            if lin.last_cg.num_iterations == dbg["power_order"]:
                _per_camera(inc, inc_c, nc, 10 * SC_TOL[dtype], "inc")
        _per_camera(b, dbg["b"], nc, SC_TOL[dtype], "b")
    if valid_only:  # the turned cameras have no valid observation: nothing reaches their gradient or their increment
        assert np.all(b.reshape(nc, 9)[list(TURNED)] == 0) and np.all(inc.reshape(nc, 9)[list(TURNED)] == 0)
        assert np.all(inc_c.reshape(nc, 9)[list(TURNED)] == 0)
    # back substitution landmark by landmark against the model's dense formula
    D = lin.get_jacobian_scaling()[0].astype(np.float64).reshape(nc, 9)
    jp, jl, r, keep, rmag = _model_rows(arrays, dtype, th, valid_only)
    _, jls_m = _model_scaling(arrays, jp, jl, dtype)
    dp = (np.random.default_rng(3).uniform(-1, 1, 9 * nc) * 0.01).astype(dtype)
    lin.download_state()
    lms0 = bp.lms.astype(np.float64)
    lin.back_substitute(dp)
    lin.download_state()
    lms1 = bp.lms.astype(np.float64)
    dpd = dp.astype(np.float64).reshape(nc, 9)
    for lm in range(arrays.nl):
        s, e = int(arrays.lm_off[lm]), int(arrays.lm_off[lm + 1])
        n, cams = e - s, arrays.obs_cam[s:e]
        got = lms1[lm] - lms0[lm]
        if not keep[s:e].any():
            assert np.all(got == 0), (lm, got)
            continue
        jls = jls_m[lm]
        Jls = (jl[s:e] * jls).reshape(2 * n, 3)
        Jpdp = np.einsum("kij,kj->ki", jp[s:e] * D[cams][:, None, :], dpd[cams]).reshape(2 * n)
        rhs = r[s:e].reshape(2 * n) + Jpdp
        M = Jls.T @ Jls + LAM * np.eye(3)
        sol = np.linalg.solve(M, Jls.T @ rhs)
        want = -jls * sol
        Minv = np.abs(np.linalg.inv(M))
        mag = np.abs(Jls).T @ (rmag[s:e].reshape(2 * n) + np.abs(Jpdp)) + np.abs(M) @ np.abs(sol)
        allow = 2 * (9 * n + 4 + 256) * u * jls * (Minv @ mag) + u * (np.abs(want) + np.abs(lms1[lm]))
        if so.solver_type != "SQUARE_ROOT":  # the Schur complement forms the normal equations: the condition enters squared
            allow *= 1 + np.linalg.cond(M)
        assert np.all(np.abs(got - want) <= allow), (lm, n, got, want, allow)
    lin.close()


def test_lm_with_invalid_projections_f64():
    """ERROR_VALID with turned-around cameras in float64: bundle_adjust_manual against the oracle's loop (every decision and the
    iteration count exact, cost at 1e-9) and rba_lm_run against bundle_adjust_manual bit for bit"""
    import rootba_b200 as rb
    arrays, opts, _, _ = _setup("valid", np.float64)
    bp, lin, o, so = make_pair(arrays, np.float64, max_num_iterations=8, **opts)
    e = float(cm.EPS_SQRT[np.dtype(np.float64)])

    def margin(cams, lms):
        z = cm.linearize(*cm.observations(type(arrays)(cams, lms, arrays.lm_off, arrays.obs_cam, arrays.obs_xy)))["pc"][:, 2]
        return np.min(np.abs(z - e)) / e
    assert margin(arrays.cams, arrays.lms) > 1e-6
    summ = rb.bundle_adjust_manual(bp, so, linearizor=lin)
    rows, _ = o.optimize()
    g_it = summ["iterations"]
    assert len(g_it) == len(rows) and len(rows) >= 4
    for a, b in zip(g_it, rows):
        assert a["iteration"] == int(b["iteration"])
        assert bool(a["step_is_successful"]) == bool(b["step_is_successful"]), a["iteration"]
        assert abs(a["cost"]["valid"]["error"] - b["cost_valid"]) <= 1e-9 * b["cost_valid"], a["iteration"]
        assert a["cost"]["valid"]["num_obs"] == int(b["num_obs_valid"])
    lin.download_state()
    # validity never came near the threshold: the state at the end is as far from it as at the start
    assert margin(bp.cams, bp.lms) > 1e-6 and margin(*o.get_state()) > 1e-6
    lin.close()
    # native loop against the Python loop, bit for bit
    bpa, bpb = rb.BalProblem.from_arrays(arrays, np.float64), rb.BalProblem.from_arrays(arrays, np.float64)
    summ = rb.bundle_adjust_manual(bpa, so)
    lin = rb.LinearizorQR.create(bpb, so)
    its, _, _ = lin.lm_run(64)
    py = summ["iterations"][1:]
    assert len(its) == len(py)
    for a, b in zip(py, its):
        assert bool(a["step_is_successful"]) == b["accepted"] and a["cost"]["valid"]["error"] == b["cost"]
        assert a["linear_solver_iterations"] == b["cg_iterations"] and a["lam"] == b["lambda"]
    lin.download_state()
    assert np.array_equal(bpa.cams, bpb.cams) and np.array_equal(bpa.lms, bpb.lms)
    lin.close()
