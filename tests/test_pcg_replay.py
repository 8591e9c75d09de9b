"""The float64 replays of tests/pcg_replay.py against the oracle's restatement of the same recurrences, iterate by iterate, and
against the dense solution they converge to.  No GPU.

The PCG replay runs on the oracle's own inputs -- b and the block-Jacobi inverse of the same solve (the oracle's damping
round trip makes them differ in the last bits from solve to solve), its right_multiply as the operator -- so the two sides
differ only in the order of float64 sums (bar 1e-12).  The power-series replay runs on the
dense float64 Hpp and E0 of test_oracle_dense_numpy, derived from the independent camera model, and takes E0 through
apply_S = Hpp_d - E0 like it does on the GPU; the oracle linearises on its own, so the bar is the 1e-10 that
test_oracle_dense_numpy allows for the partial sums."""
import numpy as np
import pytest

from conftest import rel_err
from oracle import oracle_py as orc
from pcg_replay import NO_CONVERGENCE, SUCCESS, block_apply, lanczos_condition, pcg_replay, power_replay

LAM = 1e-3
K = 25
NEVER = -1e30  # an eta no zeta can undercut: only max_linear_solver_iterations ends the solve


def zeta_gap(zetas, k, margin):
    """an eta with min(zeta_1..zeta_{k-1}) > margin * eta and eta > margin * zeta_k (zeta_k > 0), or None"""
    lo, hi = zetas[k - 1] * margin, min(zetas[:k - 1], default=np.inf) / margin
    if not 0 < lo < hi:
        return None
    return float(np.sqrt(lo * hi)) if np.isfinite(hi) else 2 * lo


@pytest.fixture(scope="module")
def oracle_case():
    """a sequence-like problem on which PCG is far from convergence after K iterations at LAM"""
    from rootba_b200.synthetic import synth_config
    a = synth_config("ladybug-49", scale=0.4)
    o = orc.Oracle(a, np.float64, orc.default_options(num_threads=1))
    assert o.linearize()
    _, dbg = o.solve(LAM, want_debug=True)
    ref = pcg_replay(o.right_multiply, dbg["b"], dbg["inv_blocks"], eta=NEVER, max_it=K)
    return o, dbg, ref


def _oracle_solve(o, **kw):
    o.set_options(orc.default_options(num_threads=1, **kw))
    inc, dbg = o.solve(LAM, want_debug=True)
    return inc, dbg


def _replay(o, d, **kw):
    return pcg_replay(o.right_multiply, d["b"], d["inv_blocks"], **kw)


def test_replay_problem_is_far_from_convergence(oracle_case):
    o, dbg, ref = oracle_case
    full = pcg_replay(o.right_multiply, dbg["b"], dbg["inv_blocks"], eta=0.0, max_it=500)
    assert full["iterations"] > K
    xs = ref["xs"]
    assert min(rel_err(xs[k], xs[k - 1]) for k in range(1, K + 1)) > 1e-6
    lmin, lmax = lanczos_condition(full["alphas"], full["betas"])
    assert 0 < lmin < lmax


@pytest.mark.parametrize("k", range(1, K + 1))
def test_truncated_oracle_solve_is_the_kth_iterate(oracle_case, k):
    o, dbg, ref = oracle_case
    inc, d = _oracle_solve(o, eta=NEVER, max_linear_solver_iterations=k)
    assert d["cg_iterations"] == k and d["cg_termination"] == NO_CONVERGENCE
    assert rel_err(inc, -_replay(o, d, eta=NEVER, max_it=k)["xs"][k]) < 1e-12


def test_zeta_stop_at_every_reachable_iteration(oracle_case):
    """zeta_k is not monotone in k: an eta stops exactly at k only where zeta_k is below every earlier zeta.  Every such k
    up to K is taken; they include k before and after the residual refresh at iteration 10."""
    o, dbg, ref = oracle_case
    ks = [k for k in range(1, K + 1) if zeta_gap(ref["zetas"], k, 1 + 1e-6) is not None]
    assert min(ks) == 1 and max(ks) > 10
    for k in ks:
        eta = zeta_gap(ref["zetas"], k, 1 + 1e-6)
        inc, d = _oracle_solve(o, eta=eta, max_linear_solver_iterations=500)
        rep = _replay(o, d, eta=eta, max_it=500)
        assert rep["iterations"] == k and rep["termination"] == SUCCESS
        assert d["cg_iterations"] == k and d["cg_termination"] == SUCCESS
        assert rel_err(inc, -rep["xs"][k]) < 1e-12


@pytest.mark.parametrize("m", [3, 10])
def test_min_iterations_gate(oracle_case, m):
    """an eta every zeta satisfies: the solve ends at exactly min_linear_solver_iterations"""
    o, dbg, ref = oracle_case
    rep = pcg_replay(o.right_multiply, dbg["b"], dbg["inv_blocks"], eta=1e30, max_it=500, min_it=m)
    assert rep["iterations"] == m and rep["termination"] == SUCCESS
    inc, d = _oracle_solve(o, eta=1e30, max_linear_solver_iterations=500, min_linear_solver_iterations=m)
    assert d["cg_iterations"] == m and d["cg_termination"] == SUCCESS
    assert rel_err(inc, -_replay(o, d, eta=1e30, max_it=500, min_it=m)["xs"][m]) < 1e-12
    # and max_linear_solver_iterations wins over the gate, like in the reference loop
    inc, d = _oracle_solve(o, eta=1e30, max_linear_solver_iterations=m - 1, min_linear_solver_iterations=m)
    assert d["cg_iterations"] == m - 1 and d["cg_termination"] == NO_CONVERGENCE
    rep = _replay(o, d, eta=1e30, max_it=m - 1, min_it=m)
    assert rep["iterations"] == m - 1 and rep["termination"] == NO_CONVERGENCE
    assert rel_err(inc, -rep["xs"][m - 1]) < 1e-12


def test_residual_refresh_changes_the_iterates(oracle_case):
    """the period is observable: without the refresh at iteration 10 the iterates after it differ (beyond the bar used
    above), so a replay with the wrong period could not pass the truncation sweep"""
    o, dbg, ref = oracle_case
    other = pcg_replay(o.right_multiply, dbg["b"], dbg["inv_blocks"], eta=NEVER, max_it=K, period=1000)
    assert all(rel_err(ref["xs"][k], other["xs"][k]) < 1e-13 for k in range(1, 10))
    assert rel_err(ref["xs"][K], other["xs"][K]) > 1e-12


@pytest.fixture(scope="module")
def dense_case():
    from test_oracle_dense_numpy import _dense_system, _problem, _reduced
    prob = _problem("benign")
    Jp, Jl, r = _dense_system(prob)
    D, sl, Jps, Jls, Minv, H, b = _reduced(Jp, Jl, r, LAM, prob.nl, float(np.sqrt(1e-10)))
    N = H.shape[0]
    W = Jps.T @ Jls
    E0 = W @ Minv @ W.T
    Hpp_d = Jps.T @ Jps + LAM * np.eye(N)
    inv = np.array([np.linalg.inv(Hpp_d[9 * c:9 * c + 9, 9 * c:9 * c + 9]) for c in range(prob.nc)])
    o = orc.Oracle(prob, np.float64, orc.default_options(num_threads=1))
    o.compute_error()
    o.scl_linearize()
    return prob, H, b, Hpp_d, E0, inv, o


@pytest.mark.parametrize("k", range(0, K + 1))
def test_power_series_partial_sums(dense_case, k):
    prob, H, b, Hpp_d, E0, inv, o = dense_case
    S = Hpp_d - E0
    rep = power_replay(lambda v: S @ v, inv, b, order=k, eta=0.0)
    assert rep["iterations"] == k and rep["termination"] == NO_CONVERGENCE and len(rep["sums"]) == k + 1
    inc, d = o.scl_power_solve(LAM, power_order=k, q_tolerance=0.0)
    assert d["power_order"] == k and d["termination"] == NO_CONVERGENCE
    assert rel_err(inc, rep["sums"][k]) < 1e-10
    # the E0 route through S is the series written with E0 itself
    direct = block_apply(inv, -b)
    acc = direct.copy()
    for _ in range(k):
        direct = block_apply(inv, E0 @ direct)
        acc = acc + direct
    assert rel_err(rep["sums"][k], acc) < 1e-12


def test_power_series_zeta_stop(dense_case):
    prob, H, b, Hpp_d, E0, inv, o = dense_case
    S = Hpp_d - E0
    full = power_replay(lambda v: S @ v, inv, b, order=K, eta=0.0)
    ks = [k for k in range(1, K + 1) if zeta_gap(full["zetas"], k, 1 + 1e-6) is not None]
    assert len(ks) >= 3
    for k in ks:
        eta = zeta_gap(full["zetas"], k, 1 + 1e-6)
        rep = power_replay(lambda v: S @ v, inv, b, order=K, eta=eta)
        assert rep["iterations"] == k and rep["termination"] == SUCCESS
        inc, d = o.scl_power_solve(LAM, power_order=K, q_tolerance=eta)
        assert d["power_order"] == k and d["termination"] == SUCCESS
        assert rel_err(inc, full["sums"][k]) < 1e-10


def test_replays_converge_to_the_dense_solution(dense_case):
    prob, H, b, Hpp_d, E0, inv, o = dense_case
    want = -np.linalg.solve(H, b)
    blocks = np.array([np.linalg.inv(H[9 * c:9 * c + 9, 9 * c:9 * c + 9]) for c in range(prob.nc)])
    rep = pcg_replay(lambda v: H @ v, b, blocks, eta=1e-15, max_it=1000)
    assert rep["termination"] == SUCCESS
    assert rel_err(-rep["xs"][-1], want) < 1e-8 * np.linalg.cond(H) ** 0.5  # the bar of test_oracle_dense_numpy.py
    S = Hpp_d - E0
    # spectral radius of Hpp_d^-1 E0 < 1: the series converges, its terms shrink geometrically
    rho = max(abs(np.linalg.eigvals(np.linalg.solve(Hpp_d, E0))))
    assert rho < 1
    order = int(np.ceil(np.log(1e-13) / np.log(rho)))
    pw = power_replay(lambda v: S @ v, inv, b, order=order, eta=0.0)
    assert rel_err(pw["sums"][-1], want) < 1e-10
    # the Lanczos estimate lies inside the spectrum of M^-1 H and approaches its ends
    ev = np.sort(np.linalg.eigvals(np.linalg.solve(np.linalg.inv(np.vstack([np.hstack(
        [blocks[c] if c == d else np.zeros((9, 9)) for d in range(prob.nc)]) for c in range(prob.nc)])), H)).real)
    lmin, lmax = lanczos_condition(rep["alphas"], rep["betas"])
    assert ev[0] * (1 - 1e-8) <= lmin and lmax <= ev[-1] * (1 + 1e-8)
    assert lmax / lmin > 0.5 * ev[-1] / ev[0]
