"""The PCG and power-series solves of the reduced camera system (RCS), iterate by iterate, against the float64 replays of
tests/pcg_replay.py run on the solver's own inputs: b from get_rhs, M^-1 from get_preconditioner and the operator from
right_multiply.  Linearisation noise stays out of the comparison, so only the loop is under test (k_pcg_vec / k_power_vec
and the host enqueue loops of Solver::solve_enqueue / power_enqueue): the refresh every residual_reset_period iterations,
the rho / q0 slots, the zeta rule and its min_linear_solver_iterations gate, is_last, and how far ahead the host enqueues
(pcg_check_period).

Options are fixed when a handle is created, so every truncation is a fresh handle on the same problem; b and M^-1 are first
checked to be bit-identical across handles.  Operator of the replay: float64 handles call right_multiply once per replay
iteration; float32 handles assemble H once in float64 from right_multiply of the 9 nc unit vectors (the kernel's own
float32 operator, exactly).

Bars.  Iterate k of PCG in precision u differs from the exact-arithmetic iterate by roughly c k u kappa (Greenbaum,
"Iterative Methods for Solving Linear Systems", ch. 4: every iteration adds rounding of relative size O(u) in the operator
product, the 9-term preconditioner product and three vector updates, and the recurrences amplify it by at most the
condition number kappa of M^-1 H).  c = 10 allows 2u for each of those five operations.  kappa is lanczos_condition of the
replay run to convergence.  The power series adds one term per step: term i carries the relative rounding of one operator
product and one 9x9 product, amplified by the condition number kappa_b of the damped camera blocks it inverts, and the
partial sums keep the error of every earlier term, carried on by later terms with factors rho^j (rho < 1 the spectral radius
of Hpp^-1 E0, estimated from the ratio of the last two terms of a long replay), so the bar is c k u kappa_b min(k, 1 / (1 - rho)),
held cameras' zero rows and columns left out of kappa_b.  The power series runs at LAM_POWER = 0.1: at LAM its spectral
radius is ~0.98 and the float32 bar would exceed 1e-2.  Each test asserts its bar is <= 1e-8 in float64 and <= 1e-2 in float32 (else the problem would
be too ill-conditioned to tell iterates apart), and in float64 that consecutive iterates differ by more than 100 times the
bar, so that an off-by-one iterate cannot pass.  In float32 the bar is ~1e-3, larger than the late PCG steps, so there the
exact counts (iterations, termination, operator applications) carry the discrimination and the values are checked at the bar.
"""
import contextlib
import os

import numpy as np
import pytest

from conftest import rel_err
from pcg_replay import NO_CONVERGENCE, SUCCESS, lanczos_condition, pcg_replay, power_replay
from objective_checks import MASK, fixed_entries
from test_pcg_replay import zeta_gap

pytestmark = pytest.mark.gpu

LAM = 1e-3
LAM_POWER = 0.1
K = 25
NEVER = -1e30  # k_pcg_vec tests zeta < eta: a negative eta no rounding can undercut, unlike 0
U = {np.float32: 2.0 ** -24, np.float64: 2.0 ** -53}
C_BAR = 10
BAR_MAX = {np.float32: 1e-2, np.float64: 1e-8}
MARGIN = {np.float32: 2.0, np.float64: 1 + 1e-6}


@pytest.fixture(scope="module")
def seq_problem():
    """sequence-like visibility, 86 cameras: PCG needs ~110 iterations at LAM"""
    from rootba_b200.synthetic import synth_config
    return synth_config("ladybug-1723", scale=0.05)


@pytest.fixture(scope="module")
def one_cta_problem():
    """120 cameras: with RBA_PCG_CLUSTER=1 the vector step leaves the register-resident layout"""
    from rootba_b200.synthetic import synth_bal
    return synth_bal(120, 1500, 4.1, seed=12)


@pytest.fixture(scope="module")
def many_cameras():
    from test_gpu_kernel_paths import vec_cached
    from rootba_b200.synthetic import synth_bal
    a = synth_bal(2200, 16000, 4.5, seed=13)
    assert not vec_cached(a.nc, 16)
    return a


@contextlib.contextmanager
def _env(env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _handle(arrays, dtype, env, mask=None, **opt):
    import rootba_b200 as rb
    with _env(env):
        bp = rb.BalProblem.from_arrays(arrays, dtype)
        bp.camera_fixed = mask
        lin = rb.LinearizorQR.create(bp, rb.SolverOptions(**opt))
    lin.linearize()
    return lin


def _lam(opt):
    return LAM_POWER if opt.get("solver_type") == "POWER_SCHUR_COMPLEMENT" else LAM


def _solve(arrays, dtype, env, mask=None, **opt):
    lin = _handle(arrays, dtype, env, mask, **opt)
    inc = lin.solve(_lam(opt))
    cg = lin.last_cg
    out = {"inc": inc, "term": cg.termination_type, "it": cg.num_iterations, "matvecs": cg.num_matvecs,
           "b": lin.get_rhs(), "inv": lin.get_preconditioner()[0], "matvec_launches": lin.timings()["matvec_launches"]}
    lin.close()
    return out


def operator_of(lin, dtype):
    """the handle's RCS operator for a replay: right_multiply itself (float64), or assembled once in float64 from the
    unit vectors (float32: the kernel's float32 operator, exactly)"""
    if dtype == np.float64:
        return lambda v: lin.right_multiply(np.asarray(v, np.float64))
    n = 9 * lin.nc
    H = np.empty((n, n))
    for j in range(n):
        e = np.zeros(n, np.float32)
        e[j] = 1
        H[:, j] = lin.right_multiply(e)
    return lambda v: H @ v


class Inputs:
    """b, M^-1 and the operator of one handle, after a solve; the handle stays open for the float64 operator"""

    def __init__(self, arrays, dtype, env, mask=None, **opt):
        self.dtype = dtype
        self.lin = _handle(arrays, dtype, env, mask, **opt)
        self.lin.solve(_lam(opt))
        self.b, self.inv = self.lin.get_rhs(), self.lin.get_preconditioner()[0]
        self.op = operator_of(self.lin, dtype)

    def close(self):
        self.lin.close()


def _pcg_bars(inp, period=10):
    full = pcg_replay(inp.op, inp.b, inp.inv, eta=0.0, max_it=600, period=period)
    lmin, lmax = lanczos_condition(full["alphas"], full["betas"])
    kappa = lmax / lmin
    bars = [C_BAR * max(k, 1) * U[inp.dtype] * kappa for k in range(K + 1)]
    assert full["iterations"] >= K, "the replay converges before K iterations: the problem cannot tell iterates apart"
    assert bars[K] <= BAR_MAX[inp.dtype], (kappa, bars[K])
    return full, bars


def _separated(xs, bars, dtype):
    if dtype == np.float64:  # float32: see the module docstring
        for k in range(1, K + 1):
            assert rel_err(xs[k], xs[k - 1]) > 100 * bars[k], k


PCG_CONFIGS = {
    # id: (problem fixture, dtype, env, options)
    "sqrt-dense-f64": ("seq_problem", np.float64, {}, {}),
    "sqrt-dense-f32": ("seq_problem", np.float32, {}, {}),
    "sqrt-implicit-f64": ("seq_problem", np.float64, {}, {"operator_form": "IMPLICIT"}),
    "sqrt-implicit-f32": ("seq_problem", np.float32, {}, {"operator_form": "IMPLICIT"}),
    "sqrt-jacobi-f64": ("seq_problem", np.float64, {}, {"preconditioner_type": "JACOBI"}),
    "sqrt-jacobi-f32": ("seq_problem", np.float32, {}, {"preconditioner_type": "JACOBI"}),
    "sc-f64": ("seq_problem", np.float64, {}, {"solver_type": "SCHUR_COMPLEMENT"}),
    "sc-f32": ("seq_problem", np.float32, {}, {"solver_type": "SCHUR_COMPLEMENT"}),
    "no-partials-f64": ("seq_problem", np.float64, {"RBA_PCG_PARTIALS": "0"}, {}),
    "no-partials-f32": ("seq_problem", np.float32, {"RBA_PCG_PARTIALS": "0"}, {}),
    "one-cta-f64": ("one_cta_problem", np.float64, {"RBA_PCG_CLUSTER": "1"}, {}),
    "many-cameras-f64": ("many_cameras", np.float64, {}, {}),
    "many-cameras-sc-f64": ("many_cameras", np.float64, {}, {"solver_type": "SCHUR_COMPLEMENT"}),
    "check1-period3-f64": ("seq_problem", np.float64, {}, {"pcg_check_period": 1, "residual_reset_period": 3}),
    "check7-period1-f64": ("seq_problem", np.float64, {}, {"pcg_check_period": 7, "residual_reset_period": 1}),
    "check4-period3-f32": ("seq_problem", np.float32, {}, {"pcg_check_period": 4, "residual_reset_period": 3}),
    "check7-period10-f32": ("seq_problem", np.float32, {}, {"pcg_check_period": 7}),
}


@pytest.mark.parametrize("cfg", list(PCG_CONFIGS))
def test_pcg_truncation_sweep(cfg, request):
    """max_linear_solver_iterations = k for k = 1..K with an eta no zeta undercuts: inc = -x_k, NO_CONVERGENCE, k iterations,
    k + k // period operator applications.  K = 25 covers k = period, period +- 1 and both sides of every chunk of
    pcg_check_period in {1, 4, 7}"""
    name, dtype, env, opt = PCG_CONFIGS[cfg]
    arrays = request.getfixturevalue(name)
    period = opt.get("residual_reset_period", 10)
    inp = Inputs(arrays, dtype, env, **opt)
    try:
        _, bars = _pcg_bars(inp, period)
        ref = pcg_replay(inp.op, inp.b, inp.inv, eta=NEVER, max_it=K, period=period)
    finally:
        inp.close()
    _separated(ref["xs"], bars, dtype)
    for k in range(1, K + 1):
        r = _solve(arrays, dtype, env, eta=NEVER, max_linear_solver_iterations=k, **opt)
        assert np.array_equal(r["b"], inp.b) and np.array_equal(r["inv"], inp.inv), k  # bit-reproducible inputs
        assert (r["term"], r["it"], r["matvecs"]) == (NO_CONVERGENCE, k, k + k // period), k
        # operator applications actually enqueued (num_matvecs is computed from the count): the refresh falls on
        # iterations period, 2 period, ...
        assert r["matvec_launches"] == k + k // period, (k, r["matvec_launches"])
        assert rel_err(r["inc"], -ref["xs"][k]) < bars[k], (k, rel_err(r["inc"], -ref["xs"][k]), bars[k])


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("period", [3, 10])
@pytest.mark.parametrize("which", ["1", "2", "period-1", "period", "period+1", "2period"])
def test_pcg_zeta_stop(seq_problem, dtype, period, which):
    """an eta in a gap of the replay's zeta sequence stops the solve at exactly k with SUCCESS and inc = -x_k"""
    k = {"1": 1, "2": 2, "period-1": period - 1, "period": period, "period+1": period + 1, "2period": 2 * period}[which]
    opt = {"residual_reset_period": period}
    inp = Inputs(seq_problem, dtype, {}, **opt)
    try:
        full, bars = _pcg_bars(inp, period)
    finally:
        inp.close()
    eta = zeta_gap(full["zetas"], k, MARGIN[dtype])
    if eta is None:
        pytest.skip(f"no eta stops exactly at iteration {k}: zeta_{k} is not below every earlier zeta by the factor "
                    f"{MARGIN[dtype]} (the margin float{8 * np.dtype(dtype).itemsize} rounding needs)")
    r = _solve(seq_problem, dtype, {}, eta=eta, **opt)
    assert (r["term"], r["it"]) == (SUCCESS, k)
    assert rel_err(r["inc"], -full["xs"][k]) < bars[k]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("m", [0, 1, 3, 10, 11])
def test_pcg_min_iterations(seq_problem, dtype, m):
    """an eta every zeta satisfies: the solve stops at exactly max(m, 1) with SUCCESS"""
    inp = Inputs(seq_problem, dtype, {})
    try:
        full, bars = _pcg_bars(inp)
    finally:
        inp.close()
    r = _solve(seq_problem, dtype, {}, eta=1e30, min_linear_solver_iterations=m)
    k = max(m, 1)
    assert (r["term"], r["it"]) == (SUCCESS, k)
    assert rel_err(r["inc"], -full["xs"][k]) < bars[k]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("solver_type", ["SQUARE_ROOT", "POWER_SCHUR_COMPLEMENT"])
def test_check_period_does_not_change_results(seq_problem, dtype, solver_type):
    """how far the host enqueues ahead is invisible: inc and the summary are bit-identical for pcg_check_period 1, 4, 7 in
    the truncated, the zeta-stopped and the converged solve"""
    power = solver_type == "POWER_SCHUR_COMPLEMENT"
    cases = ([{"power_order": 13, "eta": 0.0}, {"power_order": 40, "eta": 0.25}, {"power_order": 200, "eta": 1e-6}] if power else
             [{"max_linear_solver_iterations": 13, "eta": NEVER}, {"eta": 1e-3}, {"eta": 1e-12}])
    for case in cases:
        runs = [_solve(seq_problem, dtype, {}, solver_type=solver_type, pcg_check_period=c, **case) for c in (1, 4, 7)]
        for r in runs[1:]:
            assert np.array_equal(r["inc"], runs[0]["inc"]), case
            assert (r["term"], r["it"], r["matvecs"]) == (runs[0]["term"], runs[0]["it"], runs[0]["matvecs"]), case


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_pcg_with_held_cameras(seq_problem, dtype):
    """the replay on the masked b and M^-1 of objective_checks.MASK (on the first cameras); held entries exactly 0"""
    mask = np.zeros(seq_problem.nc, np.uint8)
    mask[:MASK.size] = MASK
    fixed = fixed_entries(mask)
    inp = Inputs(seq_problem, dtype, {}, mask=mask)
    try:
        assert np.all(inp.b[fixed] == 0) and np.all(inp.inv.reshape(-1, 9)[fixed] == 0)
        _, bars = _pcg_bars(inp)
        ref = pcg_replay(inp.op, inp.b, inp.inv, eta=NEVER, max_it=K)
    finally:
        inp.close()
    for k in (1, 9, 10, 11, K):
        r = _solve(seq_problem, dtype, {}, mask=mask, eta=NEVER, max_linear_solver_iterations=k)
        assert (r["term"], r["it"]) == (NO_CONVERGENCE, k)
        assert np.all(r["inc"][fixed] == 0)
        assert rel_err(r["inc"], -ref["xs"][k]) < bars[k]


def _power_bars(inp):
    full = power_replay(inp.op, inp.inv, inp.b, order=4 * K, eta=0.0)
    sums = full["sums"]
    d1, d2 = np.linalg.norm(sums[-1] - sums[-2]), np.linalg.norm(sums[-2] - sums[-3])
    rho = d1 / d2  # ratio of consecutive terms: the spectral radius of Hpp^-1 E0
    assert rho < 1
    kappa_b = max(np.linalg.cond(blk[np.ix_(nz, nz)]) for blk in inp.inv for nz in [np.any(blk != 0, axis=1)] if nz.any())
    bars = [C_BAR * max(k, 1) * U[inp.dtype] * kappa_b * min(max(k, 1), 1 / (1 - rho)) for k in range(len(sums))]
    assert bars[K] <= BAR_MAX[inp.dtype], (kappa_b, rho, bars[K])
    return full, bars


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("masked", [False, True], ids=["free", "held"])
def test_power_series_terms(seq_problem, dtype, masked):
    """power_order = k for k = 1..K at eta = 0: inc is the k-th partial sum, termination 0, k terms; a zeta stop at chosen
    terms, among them k == power_order (convergence and is_last on the same term)"""
    mask = None
    if masked:
        mask = np.zeros(seq_problem.nc, np.uint8)
        mask[:MASK.size] = MASK
    opt = {"solver_type": "POWER_SCHUR_COMPLEMENT"}
    inp = Inputs(seq_problem, dtype, {}, mask=mask, **opt)
    try:
        full, bars = _power_bars(inp)
    finally:
        inp.close()
    sums = full["sums"]
    _separated(sums, bars, dtype)
    for k in range(1, K + 1):
        r = _solve(seq_problem, dtype, {}, mask=mask, power_order=k, eta=0.0, **opt)
        assert np.array_equal(r["b"], inp.b) and np.array_equal(r["inv"], inp.inv), k
        assert (r["term"], r["it"]) == (NO_CONVERGENCE, k), k
        assert rel_err(r["inc"], sums[k]) < bars[k], (k, rel_err(r["inc"], sums[k]), bars[k])
        if mask is not None:
            assert np.all(r["inc"][fixed_entries(mask)] == 0)
    ks = [k for k in range(1, K + 1) if zeta_gap(full["zetas"], k, MARGIN[dtype]) is not None]
    assert ks
    for k in ks[:4]:
        eta = zeta_gap(full["zetas"], k, MARGIN[dtype])
        for order in (K, k):
            r = _solve(seq_problem, dtype, {}, mask=mask, power_order=order, eta=eta, **opt)
            assert (r["term"], r["it"]) == (SUCCESS, k), (k, order)
            assert rel_err(r["inc"], sums[k]) < bars[k]
