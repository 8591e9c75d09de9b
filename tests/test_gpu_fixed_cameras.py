"""Held camera parameters (rba_set_camera_fixed) on the GPU: every solver against the dense float64 algebra of the restricted
system, no behaviour change without flags, fixed parameters bit-identical through whole LM runs, the no-free-parameter
case, bad input, the C++ host and the sharded path."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from conftest import rel_err
from objective_checks import CONFIGS, MASK, cfg_id, check_against_dense, check_two_rank_step, dense_system, fixed_entries, \
    fixed_params, reduced

pytestmark = pytest.mark.gpu


def _dense_case(nc=7, nl=90):
    from rootba_b200.synthetic import synth_bal
    prob = synth_bal(nc, nl, 3.6, seed=21)
    Jp, Jl, r = dense_system(prob)
    lam = 1e-3
    return prob, lam, r, reduced(Jp, Jl, r, lam, prob.nl)


@pytest.mark.parametrize("cfg", CONFIGS, ids=cfg_id)
def test_f64_against_restricted_dense_system(cfg):
    _check_restricted(cfg, 7, 90, {})


@pytest.mark.parametrize("cfg", CONFIGS, ids=cfg_id)
def test_f64_uncached_vector_step_against_restricted_dense_system(cfg):
    """120 cameras with a one-CTA PCG vector kernel (RBA_PCG_CLUSTER=1): from 114 cameras on, its share of the vectors is no
    longer register-resident and it reads the camera-reduced operator output (DESIGN.md section 13)"""
    _check_restricted(cfg, 120, 500, {"RBA_PCG_CLUSTER": "1"})


def _check_restricted(cfg, nc, nl, env):
    from rootba_b200.synthetic import synth_bal
    check_against_dense(cfg, synth_bal(nc, nl, 3.6, seed=21), mask=np.resize(MASK, nc), env=env)


@pytest.mark.parametrize("solver_type", ["SQUARE_ROOT", "SCHUR_COMPLEMENT"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_no_behaviour_change_without_flags(small_problem, dtype, solver_type):
    import rootba_b200 as rb
    from objective_checks import assert_identical_steps, lm_steps
    opt = dict(solver_type=solver_type)
    ref = lm_steps(small_problem, dtype, opt, "never")
    for mode in ("zeros", "set_then_none"):
        got = lm_steps(small_problem, dtype, opt, mode, rb.LinearizorQR.set_camera_fixed,
                       np.full(small_problem.nc, rb.FIX_ALL, np.uint8))
        assert_identical_steps(ref, got, mode)


def _run_flags(nc):
    import rootba_b200 as rb
    flags = np.full(nc, rb.FIX_INTRINSICS, np.uint8)
    flags[[0, 1]] = rb.FIX_ALL
    return flags


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_fixed_parameters_stay_fixed_through_lm_run(small_problem, dtype):
    import rootba_b200 as rb
    so = rb.SolverOptions(max_num_iterations=8)
    flags = _run_flags(small_problem.nc)
    bp = rb.BalProblem.from_arrays(small_problem, dtype)
    bp.camera_fixed = flags
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
    # the Python host loop with the same flags: bit-identical trajectory
    bp2 = rb.BalProblem.from_arrays(small_problem, dtype)
    bp2.camera_fixed = flags
    summ = rb.bundle_adjust_manual(bp2, so)
    host = summ["iterations"][1:]
    assert len(host) == len(its)
    for h, n in zip(host, its):  # compared as test_native_lm_loop_equals_the_python_loop compares them
        assert bool(h["step_is_successful"]) == n["accepted"] and h["lam"] == n["lambda"]
        assert h["linear_solver_iterations"] == n["cg_iterations"] and h["cost"]["all"]["error"] == n["cost"]
    assert np.array_equal(bp2.cams, bp.cams) and np.array_equal(bp2.lms, bp.lms)


@pytest.mark.parametrize("solver_type", ["SQUARE_ROOT", "SCHUR_COMPLEMENT", "POWER_SCHUR_COMPLEMENT"])
def test_every_camera_fixed_is_landmark_gauss_newton(solver_type):
    import rootba_b200 as rb
    prob, lam, r, (D, sl, Jps, Jls, Minv, H, b) = _dense_case()
    bp = rb.BalProblem.from_arrays(prob, np.float64)
    bp.camera_fixed = np.full(prob.nc, rb.FIX_ALL, np.uint8)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(solver_type=solver_type))
    lin.compute_error()
    lin.linearize()
    inc = lin.solve(lam)
    assert np.all(inc == 0) and np.all(lin.get_rhs() == 0)
    assert (lin.last_cg.termination_type, lin.last_cg.num_iterations, lin.last_cg.num_matvecs) == (1, 0, 0)
    dl_s = -Minv @ (Jls.T @ r)
    want_l = 0.5 * r @ r - 0.5 * np.sum((r + Jls @ dl_s) ** 2)
    l_diff = lin.apply(None)
    assert abs(l_diff - want_l) <= 1e-8 * abs(want_l)
    lin.download_state()
    assert np.array_equal(bp.cams, prob.cams)
    assert rel_err(bp.lms, prob.lms + (sl * dl_s).reshape(-1, 3)) < 1e-10
    lin.close()


def test_bad_input_and_host_increments(small_problem):
    import rootba_b200 as rb
    from rootba_b200 import _lib
    L = _lib.lib()
    flags = _run_flags(small_problem.nc)
    fixed = fixed_entries(flags)
    bp = rb.BalProblem.from_arrays(small_problem, np.float64)
    bp.camera_fixed = flags
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions())
    lin.compute_error()
    lin.linearize()
    bad = flags.copy()
    bad[5] = 0x10
    assert L.rba_set_camera_fixed(lin.h, C.c_void_p(bad.ctypes.data)) == -1  # RBA_ERR_INVALID_ARGUMENT
    assert b"camera 5" in L.rba_last_error()
    inc = lin.solve(1e-4)  # the earlier flags are still in force
    assert np.all(inc[fixed] == 0) and np.any(inc[~fixed] != 0)
    # a flag change discards the device-resident increment
    lin.set_camera_fixed(flags)
    with pytest.raises(rb.RbaError) as e:
        lin.apply(None)
    assert e.value.code == -6  # RBA_ERR_STATE
    # a host increment with non-zero fixed entries: those parameters stay, l_diff is that of the zeroed increment
    lin.download_state()
    cams0, lms0 = bp.cams.copy(), bp.lms.copy()
    noisy = inc.copy()
    noisy[fixed] = np.random.default_rng(4).uniform(-1, 1, int(fixed.sum()))
    bp.backup()
    l_noisy = lin.apply(noisy)
    lin.download_state()
    cams1, lms1 = bp.cams.copy(), bp.lms.copy()
    fp = fixed_params(flags)
    assert np.array_equal(cams1[fp], cams0[fp])
    bp.restore()
    l_zero = lin.apply(np.where(fixed, 0.0, noisy))
    lin.download_state()
    assert l_noisy == l_zero
    assert np.array_equal(bp.cams, cams1) and np.array_equal(bp.lms, lms1)
    assert not np.array_equal(lms1, lms0)
    lin.close()


@pytest.mark.parametrize("use_double", [True, False])
def test_bal_qr_fixed_matches_python_host(tmp_path, use_double):
    import rootba_b200 as rb
    from oracle import oracle_py as orc
    from rootba_b200.synthetic import BalArrays, synth_bal, write_bal
    from test_host_cpp import BAL_QR, _build, _load_ba_log
    _build()
    prob = synth_bal(20, 400, 4.0, seed=9, normalize_scale=None)
    path = str(tmp_path / "p.txt")
    write_bal(prob, path)
    log = str(tmp_path / "ba_log.json")
    args = [BAL_QR, "--input", path, "--max-num-iterations", "4", "--log-path", log, "--fix-intrinsics", "--fix-cameras", "0"]
    subprocess.check_call(args + ([] if use_double else ["--no-use-double"]), stdout=subprocess.DEVNULL)
    cols, _ = _load_ba_log(log)
    d = orc.load_bal(path, normalize=True)
    arrays = BalArrays(d["cams"], d["lms"], d["lm_off"], d["obs_cam"], d["obs_xy"])
    bp = rb.BalProblem.from_arrays(arrays, np.float64 if use_double else np.float32)
    flags = np.full(arrays.nc, rb.FIX_INTRINSICS, np.uint8)
    flags[0] = rb.FIX_ALL
    bp.camera_fixed = flags
    summ = rb.bundle_adjust_manual(bp, rb.SolverOptions(max_num_iterations=4))
    assert len(cols["iteration"]) == len(summ["iterations"])
    prev = None
    for k, it in enumerate(summ["iterations"]):
        cb = it["cost"]["all"]["error"] if (it["step_is_successful"] or prev is None) else prev
        prev = cb
        # as test_bal_qr_matches_python_host: independent loaders, inputs differ in the last ulp
        assert abs(cols["cost"][k] - cb) <= (1e-6 if use_double else 5e-3) * cb + 1e-12 * cols["cost"][0]
    # and the flags took effect: the run differs from the unflagged one
    free = rb.bundle_adjust_manual(rb.BalProblem.from_arrays(arrays, bp.dtype), rb.SolverOptions(max_num_iterations=4))
    assert free["iterations"][-1]["cost"]["all"]["error"] != summ["iterations"][-1]["cost"]["all"]["error"]


@pytest.mark.parametrize("peer", ["1", "0"])
@pytest.mark.parametrize("sfx", ["f32", "f64"])
def test_two_ranks_with_fixed_cameras(tmp_path, peer, sfx):
    res = check_two_rank_step(tmp_path, "fixed", sfx, peer, 27500, (7 if peer == "1" else 0) + (13 if sfx == "f32" else 0))
    assert res["fixed_inc_zero"] and res["fixed_params_identical"], res
