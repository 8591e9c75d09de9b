"""The float64 Schur-complement model (tests/solver_model.py) and its bars, on the CPU, before a GPU test relies on them:

  equality    in float64 the model equals the oracle's restatement of the reference's SC code (scl_solve, sc_get_Hb,
              scl_e0, scl_apply): b, the SCHUR_JACOBI blocks and their inverse, E0 x, H x, the landmark update and l_diff
              per camera / landmark at 1e-12 relative
  acceptance  the checkers the GPU test uses accept the float32 and the float64 oracle: a correct implementation at the
              same precision must pass, else a bar is too tight
  rejection   the same checkers reject errors planted in the model's float64 values, each on at least one track length:
              an observation left out of Hll (a lost lane of the group sum), lam missing from one diagonal entry of
              Hll, the rr part of b with the wrong sign, jls applied twice in the landmark update, one camera's 9-vector
              shifted by one entry, one landmark's contribution to E0 x dropped; else a bar is too loose
on problem(n) of test_gpu_kernel_classes (every landmark of track length n) for lengths with G = 1, 4, 8, 16, 32 lanes per
landmark, row-chunked (n >= 25) and a 2-landmark tile (n = 72).
"""
import numpy as np
import pytest

import solver_model as sm
from conftest import rel_err
from test_gpu_kernel_classes import _per_camera, paths, problem

NS = (2, 7, 12, 24, 40, 72)
LAM = 0.1
assert {paths(n)["G"] for n in NS} >= {1, 4, 8, 16, 32} and any(paths(n)["chunks"] > 1 for n in NS)


def _vectors(nc, seed):
    rng = np.random.default_rng(seed)
    return rng.uniform(-1, 1, 9 * nc), 0.01 * rng.uniform(-1, 1, 9 * nc)


def oracle_sc(arrays, dtype, lam, x, dp):
    """the oracle's SC outputs in `dtype` and its Jacobi scaling"""
    from oracle import oracle_py as orc
    o = orc.Oracle(arrays, dtype, orc.default_options(num_threads=0))
    o.scl_linearize()
    D = o.scl_get_scaling()
    inc, dbg = o.scl_solve(lam)
    o.sc_linearize()
    o.sc_scale_Jp(D)
    b, blocks, y = o.sc_get_Hb(lam, lam, x.astype(dtype))
    e0 = o.scl_e0(lam, x.astype(dtype))
    lms0 = o.get_state()[1].astype(np.float64)
    l_diff = o.scl_apply(dp.astype(dtype).copy())
    lms1 = o.get_state()[1].astype(np.float64)
    return {"D": D, "b": dbg["b"], "b_hb": b, "blocks": blocks, "inv": dbg["inv_blocks"], "hx": y, "e0": e0,
            "dl": lms1 - lms0, "lms1": lms1, "l_diff": l_diff}


def _model(n, dtype, D):
    return sm.SCModel(problem(n), dtype, D, LAM)


@pytest.mark.parametrize("n", NS)
def test_model_equals_the_oracle_f64(n):
    arrays = problem(n)
    nc = arrays.nc
    x, dp = _vectors(nc, n)
    ref = oracle_sc(arrays, np.float64, LAM, x, dp)
    m = _model(n, np.float64, ref["D"])
    b, _ = m.b()
    _per_camera(b, ref["b"], nc, 1e-12, "b")
    _per_camera(b, ref["b_hb"], nc, 1e-12, "b of get_Hb")
    B, MB = m.schur_blocks()
    _per_camera(B, ref["blocks"], nc, 1e-12, "SCHUR_JACOBI blocks")
    _per_camera(np.linalg.inv(B), ref["inv"], nc, 1e-12, "inverse")
    _per_camera(m.e0(x)[0], ref["e0"], nc, 1e-12, "E0 x")
    _per_camera(m.hx(x)[0], ref["hx"], nc, 1e-12, "H x")
    _, _, dl, _, l_diff, _ = m.back_substitute(dp)
    for lm in range(arrays.nl):
        assert rel_err(dl[lm], ref["dl"][lm]) < 1e-12, lm
    assert abs(l_diff - ref["l_diff"]) <= 1e-12 * abs(l_diff)


def check_all(m, got, x, dp):
    """every checker of the GPU test on one set of outputs (got: b, blocks, inv, hx, dl, lms1, l_diff)"""
    b, Mb = m.b()
    sm.check(got["b"], b, Mb, m, "b")
    B, MB = m.schur_blocks()
    sm.check(got["blocks"], B, MB, m, "SCHUR_JACOBI blocks")
    sm.check_inverse(got["inv"], B, MB, m, "inverse")
    y, My = m.hx(x)
    sm.check(got["hx"], y, My, m, "H x")
    if "e0" in got:
        e0, Me0 = m.e0(x)
        sm.check(got["e0"], e0, Me0, m, "E0 x")
    _, _, dl, Mdl, l_diff, Ml = m.back_substitute(dp)
    sm.check_landmark_update(got["dl"], m, dl, Mdl, got["lms1"])
    sm.check(got["l_diff"], l_diff, Ml, m, "l_diff")


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("n", NS)
def test_checkers_accept_the_oracle(n, dtype):
    arrays = problem(n)
    x, dp = _vectors(arrays.nc, n)
    ref = oracle_sc(arrays, dtype, LAM, x, dp)
    m = _model(n, dtype, ref["D"])
    if dtype == np.float64:
        assert m.c * m.u <= 1e-9, m.c
    check_all(m, ref, x, dp)


def _rejects(got, want, mag, m):
    return sm.excess(got, want, mag, m.c, m.u)[0] > 1


def _planted(n, dtype):
    """which planted errors the checkers of `dtype` reject on problem(n)"""
    arrays = problem(n)
    x, dp = _vectors(arrays.nc, n)
    from oracle import oracle_py as orc
    o = orc.Oracle(arrays, np.float64, orc.default_options(num_threads=0))
    o.scl_linearize()
    D = o.scl_get_scaling().astype(dtype)
    m = _model(n, dtype, D)
    b, Mb = m.b()
    B, MB = m.schur_blocks()
    y, My = m.hx(x)
    e0, Me0 = m.e0(x)
    _, _, dl, Mdl, _, _ = m.back_substitute(dp)
    out = {}
    # an observation left out of Hll, a diagonal entry of Hll without lam: seen in b and in the SCHUR_JACOBI blocks
    for name, lm in (("lost lane", 0), ("missing lam", arrays.nl - 1)):
        p = _model(n, dtype, D)
        H = p.Hll[lm].copy()
        if name == "lost lane":
            i = p.off[lm] + (n - 1)
            H -= p.Jl[i].T @ p.Jl[i]
        else:
            H[2, 2] -= p.lam
        p.set_hll(lm, H)
        out[name] = _rejects(p.b()[0], b, Mb, m) or _rejects(p.schur_blocks()[0], B, MB, m)
    p1, p2, _ = m.gradient_parts()
    out["rr sign"] = _rejects(p1 + p2, b, Mb, m)
    mag = Mdl + np.abs(dl) / m.c
    out["jls twice"] = _rejects(dl * m.jls, dl, mag, m)
    c = int(m.cam[0])
    for name, v, M in (("shifted b", b, Mb), ("shifted H x", y, My)):
        w = v.copy()
        w[c] = np.roll(w[c], 1)
        out[name] = _rejects(w, v, M, m)
    others = [lm for lm in range(arrays.nl) if lm != arrays.nl // 2]
    out["dropped E0 landmark"] = _rejects(m.e0(x, others)[0], e0, Me0, m) or _rejects(y + (e0 - m.e0(x, others)[0]), y, My, m)
    return out


# float32: the bar of H x and E0 x stays above one landmark's share of E0 x and above a shift within one camera's
# vector: for a random x the terms of E0 x have random signs, and the magnitude sums them without cancellation
F32_BLIND = {"shifted H x", "dropped E0 landmark"}


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_checkers_reject_planted_errors(dtype):
    """float64: every planted error on every n; float32: every one outside F32_BLIND on at least one n"""
    seen = {n: _planted(n, dtype) for n in NS}
    for name in seen[NS[0]]:
        hits = [n for n in NS if seen[n][name]]
        if dtype == np.float64:
            assert hits == list(NS), (name, hits)
        elif name not in F32_BLIND:
            assert hits, name
