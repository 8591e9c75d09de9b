"""Every track-length class and fallback path of the tile kernels, checked landmark by landmark and camera by camera.

The kernels branch on per-landmark properties (rootba_b200/csrc/layout.hpp, solver.cu, kernels.cuh): lanes per landmark G,
column pairs per lane KP, row chunks of long tracks, the register-resident or shared-memory large-KP matvec, global scratch
of k_linearize_qr / k_stage2, the streamed or plain implicit operator.  A whole-vector norm can hide an error confined to
one class or one tile, so each case here is a problem whose landmarks all have ONE track length n -- one full tile of
W = 32 / G landmarks plus a ragged tile holding one -- and every landmark and camera is compared on its own:

  blocks      debug_get_block against the oracle's get_block for every landmark (Q1 rows, R, Q1^T r, Q2 panel incl. the
              damping rows) at the single-stage bars of test_gpu_parity
  operator    y = H x against the float64 product of the kernel's OWN panels (downloaded, cast exactly), componentwise:
                |y - y^| <= c u (sum_l |P_l|^T (|P_l| |x|) + lam |x|),  c = 11 n + m + 4
              u the unit round-off of the kernel's scalar type, n the track length (9 n products per panel row, 2 n rows
              per landmark), m the landmarks of the camera (their sum, in segments), + 4 for lam x, its addition and the
              final sum of the segment partials (Higham's gamma_k bound for any summation order, DESIGN.md section 6)
  back-subst. the landmark update of rba_back_substitute against float64 from the kernel's damped block (the oracle's
              back_substitute formula): |d - d^| <= 2 (9 n + 4) u |jls| |R^-1| (|Q1^T r| + |A| |dp| + |R| |s|)
                                                        + u (|d^| + |p_new|)
              (the Skeel condition of the damped R enters through |R^-1| |R|)
  per camera  b, the preconditioner inverse and inc against the oracle at the bars of test_gpu_parity
"""
import functools
import math

import numpy as np
import pytest

from conftest import rel_err
from test_gpu_parity import TOL1, TOLB, TOLS, make_pair

pytestmark = pytest.mark.gpu

# ---- mirror of the class formulas (layout.hpp, solver.cu, kernels.cuh) ----
ROWS_PER_ITEM = 32                      # layout.hpp
KP_SMALL_MAX = 9                        # layout.hpp: KP > 9 goes to k_matvec_large
KPMAX = {np.float32: 16, np.float64: 10}  # solver.cu: largest register-resident KP of k_matvec_large
K1_CAP, K2_CAP = 3904, 3072             # solver.cu: shared-memory scalars per warp of k_linearize_qr / k_stage2
IMP_MAXSLOTS = 64                       # solver.cu: slots per tile of the streamed implicit operator


def group_size_for(n):
    for lim, g in ((2, 1), (4, 2), (8, 4), (16, 8), (32, 16)):
        if n <= lim:
            return g
    return 32


def kp_for(n, g):
    kp = (9 * n + 2 * g - 1) // (2 * g)
    return (kp + 1) & ~1 if kp > 9 else kp


def row_chunks(n):
    rows = 2 * n
    return 1 if rows <= ROWS_PER_ITEM + ROWS_PER_ITEM // 2 else (rows + ROWS_PER_ITEM - 1) // ROWS_PER_ITEM


def stage2_need(n, g, kp):
    w = 32 // g
    return 3 * w * ((2 * g * kp) | 1) + w * n * 9 + w * 20 + 8


def paths(n):
    """the kernel variants a tile of track length n takes"""
    g = group_size_for(n)
    w, kp = 32 // g, kp_for(n, g)

    def matvec(dt):
        return "small" if kp <= KP_SMALL_MAX else ("large-reg" if kp <= KPMAX[dt] else "large-smem")
    return {"G": g, "KP": kp, "chunks": row_chunks(n),
            "matvec_f32": matvec(np.float32), "matvec_f64": matvec(np.float64),
            "k1_global": w * n * 60 + 64 > K1_CAP, "k2_global": stage2_need(n, g, kp) > K2_CAP,
            "implicit": "tma" if w * n <= IMP_MAXSLOTS else "plain"}


def _signature(n):
    p = paths(n)
    return (p["G"], p["KP"] if p["KP"] <= max(KPMAX.values()) + 6 else "smem", p["chunks"] > 1, p["matvec_f32"],
            p["matvec_f64"], p["k1_global"], p["k2_global"], p["implicit"])


def _cases():
    ns = set(range(2, 41)) | {150, 300}
    for n in range(3, 301):  # both sides of every change of the class signature
        if _signature(n) != _signature(n - 1):
            ns |= {n - 1, n}
    return sorted(ns)


CASES = _cases()
# the boundaries named in layout.hpp / solver.cu must be among them
assert {24, 25, 64, 65, 71, 72, 85, 86, 113, 114}.issubset(CASES)


def _case_id(n):
    p = paths(n)
    return f"n{n}-G{p['G']}-KP{p['KP']}-c{p['chunks']}-{p['matvec_f32']}-{p['matvec_f64']}" + \
        ("-k1g" if p["k1_global"] else "") + ("-k2g" if p["k2_global"] else "") + f"-imp_{p['implicit']}"


@functools.lru_cache(maxsize=None)
def problem(n):
    """W + 1 landmarks of track length n (one full tile, one ragged tile), all inside every camera's field of view"""
    from rootba_b200.synthetic import synth_bal
    w = 32 // group_size_for(n)
    nc = max(12, n + 6)
    return synth_bal(nc, w + 1, 0.0, seed=1000 + n, track_lengths=np.full(w + 1, n), lm_spread=0.5)


def _unit_roundoff(dtype):
    return float(np.finfo(dtype).eps) / 2


def _cams_of(arrays, lm):
    return arrays.obs_cam[arrays.lm_off[lm]:arrays.lm_off[lm + 1]]


def _per_camera(a, b, nc, bar, what):
    a, b = np.asarray(a).reshape(nc, -1), np.asarray(b).reshape(nc, -1)
    worst = max(range(nc), key=lambda c: rel_err(a[c], b[c]))
    assert rel_err(a[worst], b[worst]) < bar, (what, worst, rel_err(a[worst], b[worst]))


def _check_operator_componentwise(lin, arrays, dtype, lam, blocks, n):
    """y = H x against the float64 sum of the kernel's own panels (see the module docstring for c)"""
    nc = arrays.nc
    x = np.random.default_rng(n).uniform(-1, 1, 9 * nc).astype(dtype)
    y = lin.right_multiply(x).astype(np.float64)
    xd = x.astype(np.float64).reshape(nc, 9)
    lam_s = float(dtype(lam))
    yhat, bound = lam_s * xd, lam_s * np.abs(xd)
    for lm, (bg, _, _, _) in enumerate(blocks):
        cams = _cams_of(arrays, lm)
        P = bg[3:, :9 * n].astype(np.float64)  # the 2n panel rows incl. the damping rows
        xs = xd[cams].ravel()
        yhat[cams] += (P.T @ (P @ xs)).reshape(n, 9)
        bound[cams] += (np.abs(P).T @ (np.abs(P) @ np.abs(xs))).reshape(n, 9)
    m = np.bincount(arrays.obs_cam, minlength=nc).max()
    c = 11 * n + m + 4
    err = np.abs(y.reshape(nc, 9) - yhat)
    worst = np.unravel_index(np.argmax(err - c * _unit_roundoff(dtype) * bound), err.shape)
    assert np.all(err <= c * _unit_roundoff(dtype) * bound), ("H x", worst, err[worst], bound[worst])


def _check_back_substitution(lin, bp, arrays, dtype, blocks, n):
    nc = arrays.nc
    dp = (np.random.default_rng(n + 1).uniform(-1, 1, 9 * nc) * 0.01).astype(dtype)
    lin.download_state()
    lms0 = bp.lms.astype(np.float64)
    l_g = lin.back_substitute(dp)
    lin.download_state()
    lms1 = bp.lms.astype(np.float64)
    u = _unit_roundoff(dtype)
    dpd = dp.astype(np.float64).reshape(nc, 9)
    for lm, (bg, lm_idx, res_idx, jls) in enumerate(blocks):
        bd = bg.astype(np.float64)
        A, R, q = bd[:3, :9 * n], np.triu(bd[:3, lm_idx:lm_idx + 3]), bd[:3, res_idx]
        pr = dpd[_cams_of(arrays, lm)].ravel()
        s = np.linalg.solve(R, q + A @ pr)
        jl = jls.astype(np.float64)
        want = -s * jl
        Rinv = np.abs(np.linalg.inv(R))
        allow = 2 * (9 * n + 4) * u * np.abs(jl) * (Rinv @ (np.abs(q) + np.abs(A) @ np.abs(pr) + np.abs(R) @ np.abs(s)))
        allow += u * (np.abs(want) + np.abs(lms1[lm]))
        got = lms1[lm] - lms0[lm]
        assert np.all(np.abs(got - want) <= allow), ("landmark update", lm, got, want, allow)
    return l_g


@pytest.mark.parametrize("qr", ["householder", "givens"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("n", CASES, ids=_case_id)
def test_dense_operator_class(n, dtype, qr):
    arrays = problem(n)
    assert np.all(arrays.track_lengths() == n)
    bp, lin, o, _ = make_pair(arrays, dtype, use_householder_marginalization=(qr == "householder"))
    tol, lam, nc = TOL1[dtype], 0.1, arrays.nc
    lin.linearize()
    assert o.linearize()
    inc_g = lin.solve(lam)
    inc_c, dbg = o.solve(lam, want_debug=True)
    _per_camera(lin.get_rhs(), dbg["b"], nc, 4 * tol, "b")
    inv_g, _ = lin.get_preconditioner()
    _per_camera(inv_g, dbg["inv_blocks"], nc, TOLB[dtype], "preconditioner inverse")
    assert abs(lin.last_cg.num_iterations - dbg["cg_iterations"]) <= 2
    assert lin.last_cg.termination_type == dbg["cg_termination"]
    _per_camera(inc_g, inc_c, nc, TOLS[dtype], "inc")
    # blocks of every landmark, in the reference storage layout
    blocks = []
    for lm in range(arrays.nl):
        bg, lm_idx, res_idx, jls_g = lin.debug_get_block(lm)
        bc, li, ri, jls_c = o.get_block(lm)
        assert (li, ri) == (lm_idx, res_idx) and bg.shape == bc.shape
        assert rel_err(jls_g, jls_c) < tol, lm
        assert rel_err(bg[:3, :9 * n], bc[:3, :9 * n]) < tol * 4, lm
        assert rel_err(np.triu(bg[:3, lm_idx:lm_idx + 3]), np.triu(bc[:3, lm_idx:lm_idx + 3])) < tol * 4, lm
        assert rel_err(bg[:3, res_idx], bc[:3, res_idx]) < tol * 4, lm
        assert rel_err(bg[3:, :9 * n], bc[3:, :9 * n]) < tol * 4, lm
        blocks.append((bg, lm_idx, res_idx, jls_g))
    _check_operator_componentwise(lin, arrays, dtype, lam, blocks, n)
    l_g = _check_back_substitution(lin, bp, arrays, dtype, blocks, n)
    l_c, ok = o.back_substitute((np.random.default_rng(n + 1).uniform(-1, 1, 9 * nc) * 0.01).astype(dtype))
    assert ok and abs(l_g - l_c) <= tol * 20 * abs(l_c)
    lin.close()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("n", CASES, ids=_case_id)
def test_implicit_operator_class(n, dtype):
    """operator_form = IMPLICIT stores no panels: H x per camera against the float64 product of the oracle's panels, at the
    bars of DESIGN.md section 9 (f64 1e-11, f32 1e-4: the implicit form subtracts two positive terms), x4 like test_gpu_parity"""
    arrays = problem(n)
    bp, lin, o, _ = make_pair(arrays, dtype, operator_form="IMPLICIT")
    tol, lam, nc = TOL1[dtype] * (10 if dtype == np.float32 else 1), 0.1, arrays.nc
    lin.linearize()
    assert o.linearize()
    inc_g = lin.solve(lam)
    inc_c, dbg = o.solve(lam, want_debug=True)
    _per_camera(lin.get_rhs(), dbg["b"], nc, 4 * tol, "b")
    inv_g, _ = lin.get_preconditioner()
    _per_camera(inv_g, dbg["inv_blocks"], nc, 10 * TOLB[dtype] if dtype == np.float32 else TOLB[dtype], "preconditioner inverse")
    x = np.random.default_rng(n).uniform(-1, 1, 9 * nc).astype(dtype)
    xd = x.astype(np.float64).reshape(nc, 9)
    yhat = float(dtype(lam)) * xd
    for lm in range(arrays.nl):
        bc = o.get_block(lm)[0].astype(np.float64)
        cams = _cams_of(arrays, lm)
        P = bc[3:, :9 * n]
        yhat[cams] += (P.T @ (P @ xd[cams].ravel())).reshape(n, 9)
    _per_camera(lin.right_multiply(x), yhat, nc, 4 * tol, "H x")
    assert lin.last_cg.termination_type == dbg["cg_termination"]
    assert abs(lin.last_cg.num_iterations - dbg["cg_iterations"]) <= 2
    _per_camera(inc_g, inc_c, nc, TOLS[dtype] * (5 if dtype == np.float32 else 1), "inc")
    lin.close()
