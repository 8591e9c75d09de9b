"""Cameras without any observation on one GPU (first, middle and last camera index): their increment is exactly 0 in every
solver and on every hand-over path of the operator output, the observed cameras match the oracle, and an rba_right_multiply
between two solves leaves nothing behind (it writes lambda x into the operator-output vector for every camera, which the
vector kernels that read that vector would otherwise take as the operator's value for such a camera)."""
import numpy as np
import pytest

from conftest import rel_err
from test_gpu_parity import TOLS

pytestmark = pytest.mark.gpu

UNOBSERVED = (0, 66, 132)
SC_TOL = {np.float32: 1e-3, np.float64: 1e-9}  # test_gpu_sc


@pytest.fixture(scope="module")
def gappy_problem():
    """133 cameras (>= 114: one CTA of the PCG vector kernel leaves the register-resident layout), three of them unobserved"""
    from rootba_b200.synthetic import BalArrays, synth_bal
    a = synth_bal(130, 2000, 4.1, seed=31)
    nc = a.nc + len(UNOBSERVED)
    seen = np.setdiff1d(np.arange(nc), UNOBSERVED)
    cams = np.empty((nc, 10))
    cams[seen] = a.cams
    cams[list(UNOBSERVED)] = a.cams[[3, 60, 120]]  # plausible cameras that simply see nothing
    b = BalArrays(cams, a.lms, a.lm_off, seen[a.obs_cam].astype(np.int32), a.obs_xy)
    assert np.array_equal(np.setdiff1d(np.arange(nc), b.obs_cam), UNOBSERVED)
    return b


SOLVERS = {"qr-dense": dict(solver_type="SQUARE_ROOT"), "qr-implicit": dict(solver_type="SQUARE_ROOT", operator_form="IMPLICIT"),
           "sc": dict(solver_type="SCHUR_COMPLEMENT"), "power-sc": dict(solver_type="POWER_SCHUR_COMPLEMENT")}
PATHS = {"partials": {}, "no-partials": {"RBA_PCG_PARTIALS": "0"}, "one-cta": {"RBA_PCG_CLUSTER": "1"}}


def _create(arrays, dtype, opts, env, monkeypatch):
    import rootba_b200 as rb
    with monkeypatch.context() as m:
        for k, v in env.items():
            m.setenv(k, v)
        return rb.LinearizorQR.create(rb.BalProblem.from_arrays(arrays, dtype), rb.SolverOptions(**opts))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("solver", SOLVERS)
def test_unobserved_cameras(gappy_problem, dtype, solver, path, monkeypatch):
    from oracle import oracle_py as orc
    a, opts, lam = gappy_problem, SOLVERS[solver], 1e-3
    x = np.random.default_rng(5).uniform(-1, 1, 9 * a.nc).astype(dtype)
    # solve -> right_multiply -> solve
    lin = _create(a, dtype, opts, PATHS[path], monkeypatch)
    lin.linearize()
    first = lin.solve(lam)
    it_first = lin.last_cg.num_iterations
    lin.right_multiply(x)
    second = lin.solve(lam)
    lin.close()
    # solve -> solve
    lin = _create(a, dtype, opts, PATHS[path], monkeypatch)
    lin.linearize()
    lin.solve(lam)
    plain = lin.solve(lam)
    lin.close()
    for inc in (first, second):
        assert np.all(inc.reshape(a.nc, 9)[list(UNOBSERVED)] == 0), inc.reshape(a.nc, 9)[list(UNOBSERVED)]
    assert np.array_equal(second, plain)
    assert np.array_equal(first, plain)
    # the observed cameras against the oracle
    o = orc.Oracle(a, dtype, orc.default_options(num_threads=0))
    if opts["solver_type"] == "SQUARE_ROOT":
        assert o.linearize()
        inc_c, dbg = o.solve(lam, want_debug=True)
        assert abs(it_first - dbg["cg_iterations"]) <= 2
        tol = TOLS[dtype] * (5 if opts.get("operator_form") == "IMPLICIT" and dtype == np.float32 else 1)
        assert rel_err(first, inc_c) < tol
    elif opts["solver_type"] == "SCHUR_COMPLEMENT":
        o.scl_linearize()
        inc_c, dbg = o.scl_solve(lam)
        assert abs(it_first - dbg["cg_iterations"]) <= 2
        assert rel_err(first, inc_c) < 10 * SC_TOL[dtype]
    else:
        o.scl_linearize()
        inc_c, dbg = o.scl_power_solve(lam, 20, 0.1)
        assert abs(it_first - dbg["power_order"]) <= 1
        if it_first == dbg["power_order"]:
            assert rel_err(first, inc_c) < 10 * SC_TOL[dtype]
    assert np.all(inc_c.reshape(a.nc, 9)[list(UNOBSERVED)] == 0)
