"""The assembled reduced camera matrix S = sum_l P_l^T P_l (assembled.cuh: k_rcs_terms + k_rcs_combine) block by block
against float64, its product k_rcs_spmv camera by camera at row-length edges, and the switch from the panel product to S
inside a PCG solve iterate by iterate (DESIGN.md section 4, "Assembled operator").  test_gpu_assembled_operator compares
whole vectors; a whole-vector norm can hide an error confined to one block, one row or one class of terms.

Every case asserts that S was taken: matvec_algorithmic_bytes equals the bytes of S (from the pair structure) and is below
that of an RBA_ASSEMBLED_RCS=0 handle of the same problem.  Problems qualify for S by the size rule of plan_assembled
(restated in test_pairs_cpu: S at most a quarter of the panel bytes).

Reading S.  right_multiply(e_j) for the 9 nc unit vectors gives column j of S + lambda I exactly: in k_rcs_spmv every
product but the one with the 1 is an exact zero and the partial sums add zeros, and k_pcg_q adds lambda x with one rounding
(on the diagonal only).

Bars (Higham's gamma_k = k u / (1 - k u)), M = sum_l |P_l|^T |P_l| from the kernel's own panels (rba_debug_get_block rows
3..2n+2, the damping rows included):
  S       |S - S^| <= gamma_k M per entry of the pair (ca, cb), k = 2 n_ab + 2 m_ab + 2 (m_ab common landmarks, n_ab the
          longest of their tracks: 2n - 3 fmas per undamped term, 3 per damping term, the two list-order sums, S_u + damping),
          + gamma_1 (M + lambda) on the diagonal (lambda added by right_multiply)
  S x     |y - S^ x - lambda x| <= (gamma_a + gamma_k + gamma_a gamma_k) M |x| + gamma_1 (|y^| + lambda |x|),
          a = ceil(nnz_row / 4) + 37 (each lane's fma chain over its warp's blocks, the 4 x 9 sum in shared memory and
          lambda x), k the largest of the row's pairs
  PCG     the iterate bars of test_gpu_pcg_iterates (10 k u kappa) against the float64 replay
"""
import contextlib
import functools
import math
import os

import numpy as np
import pytest

from conftest import rel_err
from objective_checks import MASK
from pcg_replay import NO_CONVERGENCE, SUCCESS, lanczos_condition, pcg_replay
from test_gpu_pcg_iterates import BAR_MAX, C_BAR, NEVER, U, operator_of
from test_pairs_cpu import lm_major, nnzb_of, panel_scalars, switch_iteration

SPMV_WARPS, SPMV_UNROLL = 4, 4  # assembled.cuh
TERMS_PER_SWEEP_PER_SM = 16 * 8 * 3  # k_rcs_terms: sm_count * 16 blocks of 8 warps, 3 terms per warp
ASM, PANEL = {"RBA_ASSEMBLED_AT": "1"}, {"RBA_ASSEMBLED_RCS": "0"}
LAM1, LAM2 = 1e-4, 1e2


def gamma(k, u):
    k = np.asarray(k, np.float64)
    return k * u / (1 - k * u)


# ---- problems ----
N_SWEEP = (2, 3, 4, 5, 8, 9, 16, 17, 32, 33, 40, 64, 150)  # every G, odd and even KP, the KP limits, row-chunked tracks


def _odd_nl(nc, n):
    """landmarks enough for S to be at most an eighth of the panels (nl n^2 >= 36 nc^2), odd: a ragged last tile"""
    return math.ceil(36 * nc * nc / (n * n)) | 1


@functools.lru_cache(maxsize=None)
def one_length(n):
    from rootba_b200.synthetic import synth_bal
    nc = max(6, n + 4)
    return synth_bal(nc, _odd_nl(nc, n), 0.0, seed=900 + n, track_lengths=[n] * _odd_nl(nc, n), lm_spread=0.5)


@functools.lru_cache(maxsize=None)
def mixed_unobserved():
    """every track-length class up to 150 and three cameras at the end that no landmark sees"""
    from rootba_b200.synthetic import BalArrays, synth_bal
    a = synth_bal(150, 6000, 9.0, seed=11, max_track=150)
    return BalArrays(np.concatenate([a.cams, a.cams[:3]]), a.lms, a.lm_off, a.obs_cam, a.obs_xy)


@functools.lru_cache(maxsize=None)
def seq_arrays():
    """sequence-like visibility, 86 cameras (test_gpu_pcg_iterates): qualifies for S, PCG needs ~110 iterations"""
    from rootba_b200.synthetic import synth_config
    return synth_config("ladybug-1723", scale=0.05)


@functools.lru_cache(maxsize=None)
def small():
    from rootba_b200.synthetic import synth_bal
    return synth_bal(30, 3000, 4.1, seed=5)


@functools.lru_cache(maxsize=None)
def chain_problem():
    """48 cameras in a row; per camera i, 12 landmarks seen by (i, i+1), 12 by (i, i+1, i+2) and 4 by i..i+4: cameras more
    than 4 apart share no landmark, so most blocks of S are zero by structure"""
    from rootba_b200.synthetic import synth_bal
    nc = 48
    tracks = [np.arange(i, i + n) for i in range(nc) for n, c in ((2, 12), (3, 12), (5, 4)) if i + n <= nc for _ in range(c)]
    rng = np.random.default_rng(31)
    tracks = [tracks[i] for i in rng.permutation(len(tracks))]
    return synth_bal(nc, len(tracks), 0.0, seed=31, tracks=tracks, lm_spread=0.5)


ROW_BLOCKS = (2, 3, 4, 5, 8, 15, 16, 17, 31, 32, 33, 64, 65, 400)
PER_PAIR = 24  # landmarks (n = 2) per co-visible pair


@functools.lru_cache(maxsize=None)
def row_problem():
    """hub camera h has ROW_BLOCKS[h] - 1 partners (its block row holds ROW_BLOCKS[h] blocks, the diagonal included); every
    partner is a filler camera seen with its hub only (rows of 2 blocks); PER_PAIR landmarks of n = 2 per pair, shuffled"""
    from rootba_b200.synthetic import synth_bal
    nh = len(ROW_BLOCKS)
    tracks, f = [], nh
    for h, d in enumerate(ROW_BLOCKS):
        for _ in range(d - 1):
            tracks += [np.array([h, f])] * PER_PAIR
            f += 1
    rng = np.random.default_rng(77)
    tracks = [tracks[i] for i in rng.permutation(len(tracks))]
    return synth_bal(f, len(tracks), 0.0, seed=77, tracks=tracks, lm_spread=0.5)


def structure(arrays):
    """the pair structure in float64-friendly form: per camera pair (dense nc x nc) the number of common landmarks and the
    longest of their tracks; nt, nnzb, the panel scalars (test_pairs_cpu's restatements)"""
    nc = arrays.nc
    m, nmax = np.zeros((nc, nc), np.int64), np.zeros((nc, nc), np.int64)
    for lm in range(arrays.nl):
        cams = arrays.obs_cam[arrays.lm_off[lm]:arrays.lm_off[lm + 1]]
        ix = np.ix_(cams, cams)
        m[ix] += 1
        nmax[ix] = np.maximum(nmax[ix], cams.size)
    lmi, oa, ob, _, _ = lm_major(arrays, 0, arrays.nl)
    return {"m": m, "nmax": nmax, "nt": int(lmi.size), "nnzb": int(nnzb_of(arrays, oa, ob)),
            "panel": int(panel_scalars(arrays, 0, arrays.nl))}


def s_bytes(st, nc, s):
    """matvec_algorithmic_bytes of S (Solver::get_stats)"""
    return (81 * st["nnzb"] + 18 * nc) * s + 4 * (st["nnzb"] + nc + 1)


def default_switch(st, s):
    return switch_iteration(st["nt"], st["panel"], st["nnzb"] * 81 * s, s)


def test_cases_reach_the_edges():
    """(CPU) the one-length cases reach every nt mod 3 (k_rcs_terms' tail warp), qualify for S, and one has more terms than
    one sweep of the grid on twice 132 SMs; the chain case has observed camera pairs without a common landmark"""
    st = {n: _structure(str(n)) for n in N_SWEEP}
    assert {s["nt"] % 3 for s in st.values()} == {0, 1, 2}
    assert all(4 * s["nnzb"] * 81 <= s["panel"] for s in st.values())
    assert max(s["nt"] for s in st.values()) > 132 * TERMS_PER_SWEEP_PER_SM * 2
    ch = _structure("chain")
    assert 4 * ch["nnzb"] * 81 <= ch["panel"] and np.count_nonzero(ch["m"] == 0) > ch["m"].size // 2
    assert set(np.diff(chain_problem().lm_off).tolist()) == {2, 3, 5}


# ---- GPU helpers ----
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


def _handle(arrays, dtype, env, prior=None, mask=None, linearize=True, **opt):
    import rootba_b200 as rb
    with _env(env):
        bp = rb.BalProblem.from_arrays(arrays, dtype)
        bp.camera_fixed = mask
        lin = rb.LinearizorQR.create(bp, rb.SolverOptions(use_double=dtype == np.float64, **opt))
    if prior:
        _prior(lin, arrays, dtype, prior)
    if linearize:
        lin.linearize()
    return lin


def _prior(lin, arrays, dtype, which):
    if which == "landmark":
        idx = np.arange(0, arrays.nl, 7, dtype=np.int32)
        L = np.tile(np.eye(3), (idx.size, 1, 1)) * 1.5
        lin.set_landmark_prior((idx, arrays.lms[idx].astype(dtype), L.astype(dtype)))
    elif which == "camera":
        rng = np.random.default_rng(3)
        mean = arrays.cams.astype(np.float64).copy()
        mean[:, :4] /= np.linalg.norm(mean[:, :4], axis=1, keepdims=True)
        L = np.zeros((arrays.nc, 9, 9))
        L[:, range(9), range(9)] = rng.uniform(0.5, 2.0, (arrays.nc, 9))
        lin.set_camera_prior((mean.astype(dtype), L.astype(dtype)))
    elif which == "pair":
        pairs = np.array([[0, 1], [2, 5], [7, 3]], np.int32)
        mean = np.zeros((3, 7)); mean[:, 0] = 1.0
        lin.set_camera_pair_prior((pairs, mean.astype(dtype), (np.tile(np.eye(6), (3, 1, 1)) * 0.7).astype(dtype)))


def _panel_bytes_of(arrays, dtype):
    """matvec_algorithmic_bytes of an RBA_ASSEMBLED_RCS=0 handle of the problem (the panel product)"""
    lin = _handle(arrays, dtype, PANEL, linearize=False)
    b = lin.stats()["matvec_algorithmic_bytes"]
    lin.close()
    return b


@functools.lru_cache(maxsize=None)
def _panel_bytes(key, dtype):
    return _panel_bytes_of(PROBLEMS[key](), dtype)


def assert_took_s(lin, key, st, dtype):
    got = lin.stats()["matvec_algorithmic_bytes"]
    assert got == s_bytes(st, lin.nc, np.dtype(dtype).itemsize) and got < _panel_bytes(key, dtype), (got, _panel_bytes(key, dtype))


def assert_took_panels(lin, key, dtype):
    assert lin.stats()["matvec_algorithmic_bytes"] == _panel_bytes(key, dtype)


def extract(lin):
    """S + lambda I of the handle, exactly, in float64 (column j = right_multiply(e_j))"""
    n = 9 * lin.nc
    Y = np.empty((n, n))
    e = np.zeros(n, lin.dtype)
    for j in range(n):
        e[j] = 1
        Y[:, j] = lin.right_multiply(e)
        e[j] = 0
    return Y


def reference(lin, arrays):
    """S^ = sum_l P_l^T P_l and M = sum_l |P_l|^T |P_l| in float64 from the handle's own panels (damping rows included)"""
    n9 = 9 * arrays.nc
    S, M = np.zeros((n9, n9)), np.zeros((n9, n9))
    for lm in range(arrays.nl):
        k0, k1 = int(arrays.lm_off[lm]), int(arrays.lm_off[lm + 1])
        n = k1 - k0
        P = lin.debug_get_block(lm)[0][3:3 + 2 * n, :9 * n].astype(np.float64)
        idx = (9 * arrays.obs_cam[k0:k1][:, None] + np.arange(9)).ravel()
        ix = np.ix_(idx, idx)
        S[ix] += P.T @ P
        A = np.abs(P)
        M[ix] += A.T @ A
    return S, M


def check_s(Y, lin, arrays, st, lam, dtype, what):
    """every entry of every block against S^ + lambda I at the module's bar; the exact properties"""
    u, lam_s = U[dtype], float(dtype(lam))
    nc = arrays.nc
    S, M = reference(lin, arrays)
    k = np.kron(2 * st["nmax"] + 2 * st["m"] + 2, np.ones((9, 9)))
    bar = gamma(k, u) * M
    d = np.arange(9 * nc)
    bar[d, d] += gamma(1, u) * (M[d, d] * (1 + gamma(k[d, d], u)) + lam_s)
    want = S.copy()
    want[d, d] += lam_s
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.where(Y == want, 0.0, np.abs(Y - want) / bar)
    worst = np.unravel_index(np.argmax(ratio), ratio.shape)
    assert ratio[worst] <= 1, (what, "entry", worst, "cameras", (worst[0] // 9, worst[1] // 9), "error / bar", ratio[worst])
    assert np.array_equal(Y, Y.T), what  # S bitwise symmetric: diagonal blocks by fma commuting, upper = lower transposed
    none = np.kron(st["m"] == 0, np.ones((9, 9), bool))
    seen = np.bincount(arrays.obs_cam, minlength=nc) > 0
    unseen = np.repeat(~seen, 9)
    assert np.all(Y[none & ~np.eye(9 * nc, dtype=bool)] == 0), what  # pairs without a common landmark: exactly 0
    if unseen.any():  # rows of cameras without observations: exactly lambda x
        assert np.array_equal(Y[unseen], lam_s * np.eye(9 * nc)[unseen]), what


PROBLEMS = {**{str(n): functools.partial(one_length, n) for n in N_SWEEP}, "mixed-unobserved": mixed_unobserved,
            "small": small, "rows": row_problem, "chain": chain_problem, "seq": seq_arrays}

S_CASES = {  # id: (problem, options, prior)
    **{str(n): (str(n), {}, None) for n in N_SWEEP},
    "mixed-unobserved": ("mixed-unobserved", {}, None),
    "chain": ("chain", {}, None),
    "seq": ("seq", {}, None),  # the problem of the switch tests below
    "givens": ("small", {"use_householder_marginalization": False}, None),
    "identity": ("9", {"stage2_form": "IDENTITY"}, None),
    "landmark-prior": ("small", {}, "landmark"),
}


@functools.lru_cache(maxsize=None)
def _structure(key):
    return structure(PROBLEMS[key]())


def _dtypes():
    return [pytest.param(d, id=np.dtype(d).name) for d in (np.float32, np.float64)]


# ---- 1. S block by block ----
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", _dtypes())
@pytest.mark.parametrize("case", list(S_CASES))
def test_s_blocks(case, dtype):
    """S at LAM1, then at LAM2 on the same linearisation (S_u reused), both against float64 block by block; S at LAM1
    bit-identical to a fresh handle's built at iteration 2 instead of 1, S at LAM2 to a fresh handle's that solves at LAM2
    only"""
    key, opt, prior = S_CASES[case]
    arrays, st = PROBLEMS[key](), _structure(key)
    lin = _handle(arrays, dtype, ASM, prior, **opt)
    for lam in (LAM1, LAM2):
        lin.solve(lam)
        assert_took_s(lin, key, st, dtype)
        Y = extract(lin)
        check_s(Y, lin, arrays, st, lam, dtype, (case, lam))
        if lam == LAM1:
            Y1 = Y
    lin.close()
    for env, lam, want in (({"RBA_ASSEMBLED_AT": "2"}, LAM1, Y1), (ASM, LAM2, Y)):
        fresh = _handle(arrays, dtype, env, prior, **opt)
        fresh.solve(lam)
        assert fresh.last_cg.num_iterations >= 2
        assert_took_s(fresh, key, st, dtype)
        assert np.array_equal(extract(fresh), want), ("S depends on the handle, on when it is built or on the lambda before", lam)
        fresh.close()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", _dtypes())
@pytest.mark.parametrize("key", ["9", "mixed-unobserved"])
def test_s_cache_across_states(key, dtype):
    """S after apply + linearize (S_u rebuilt) and after backup / apply / restore (S_u kept) bit-identical to fresh handles
    at the same state bits, and correct against float64"""
    from rootba_b200.synthetic import BalArrays
    arrays, st = PROBLEMS[key](), _structure(key)
    a = _handle(arrays, dtype, ASM)
    a._backup()
    a.apply(a.solve(LAM1))
    a._restore()
    a.solve(3.0)
    b = _handle(arrays, dtype, ASM)
    b.solve(3.0)
    assert_took_s(a, key, st, dtype)
    assert np.array_equal(extract(a), extract(b)), "S after a restore"
    b.close()
    a.apply(a.solve(LAM1))
    a.download_state()
    moved = BalArrays(a.bal_problem.cams.astype(np.float64), a.bal_problem.lms.astype(np.float64), arrays.lm_off,
                      arrays.obs_cam, arrays.obs_xy)
    a.linearize()
    a.solve(LAM2)
    c = _handle(moved, dtype, ASM)
    assert np.array_equal(c.bal_problem.cams, a.bal_problem.cams) and np.array_equal(c.bal_problem.lms, a.bal_problem.lms)
    c.solve(LAM2)
    Y = extract(a)
    assert np.array_equal(Y, extract(c)), "S after apply + linearize: S_u of the old linearisation reused?"
    check_s(Y, a, moved, st, LAM2, dtype, "after apply + linearize")
    a.close(); c.close()


# ---- 2. k_rcs_spmv at row-length edges ----
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", _dtypes())
def test_spmv_rows(dtype):
    """y = S x camera by camera, rows of 2 .. 400 blocks, against the float64 product of the kernel's panels"""
    arrays, st = row_problem(), _structure("rows")
    nc, u = arrays.nc, U[dtype]
    nnz_row = np.count_nonzero(st["m"], axis=1)
    assert set(ROW_BLOCKS) | {2} == set(nnz_row.tolist())
    lin = _handle(arrays, dtype, ASM)
    for lam in (LAM1, LAM2):
        lin.solve(lam)
        assert_took_s(lin, "rows", st, dtype)
        x = np.random.default_rng(5).uniform(-1, 1, 9 * nc).astype(dtype)
        xd, ax = x.astype(np.float64), np.abs(x.astype(np.float64))
        y = lin.right_multiply(x).astype(np.float64)
        want, mag = np.zeros(9 * nc), np.zeros(9 * nc)
        for lm in range(arrays.nl):
            k0, k1 = int(arrays.lm_off[lm]), int(arrays.lm_off[lm + 1])
            n = k1 - k0
            P = lin.debug_get_block(lm)[0][3:3 + 2 * n, :9 * n].astype(np.float64)
            idx = (9 * arrays.obs_cam[k0:k1][:, None] + np.arange(9)).ravel()
            want[idx] += P.T @ (P @ xd[idx])
            mag[idx] += np.abs(P).T @ (np.abs(P) @ ax[idx])
        lam_s = float(dtype(lam))
        want += lam_s * xd
        a = np.repeat(-(-nnz_row // SPMV_WARPS) + 37, 9)
        k = np.repeat(np.max(np.where(st["m"] > 0, 2 * st["nmax"] + 2 * st["m"] + 2, 0), axis=1), 9)
        ga, gk = gamma(a, u), gamma(k, u)
        bar = (ga + gk + ga * gk) * mag + gamma(1, u) * (np.abs(want) + lam_s * ax)
        ratio = np.where(y == want, 0.0, np.abs(y - want) / bar)
        worst = int(np.argmax(ratio))
        assert ratio[worst] <= 1, ("camera", worst // 9, "row blocks", nnz_row[worst // 9], "error / bar", ratio[worst])
    lin.close()


# ---- 3. the switch inside a solve ----
@pytest.fixture(scope="module")
def seq_problem():
    return seq_arrays()


LAM = 1e-3


def _solve_counts(lin, lam, **_):
    k0 = lin.timings()["kernel_launches"]
    inc = lin.solve(lam)
    t = lin.timings()
    cg = lin.last_cg
    return {"inc": inc, "term": cg.termination_type, "it": cg.num_iterations, "matvecs": cg.num_matvecs,
            "matvec_launches": t["matvec_launches"], "launches": t["kernel_launches"] - k0,
            "bytes": lin.stats()["matvec_algorithmic_bytes"]}


def _one_solve(arrays, dtype, env, prior=None, mask=None, lam=LAM, **opt):
    lin = _handle(arrays, dtype, env, prior, mask, **opt)
    r = _solve_counts(lin, lam)
    r["b"], r["inv"] = lin.get_rhs(), lin.get_preconditioner()[0]
    lin.close()
    return r


def _bars(op, b, inv, dtype, period, kmax):
    full = pcg_replay(op, b, inv, eta=0.0, max_it=600, period=period)
    lmin, lmax = lanczos_condition(full["alphas"], full["betas"])
    bars = [C_BAR * max(k, 1) * U[dtype] * lmax / lmin for k in range(kmax + 1)]
    # as in test_gpu_pcg_iterates up to its K = 25; beyond, the float32 bar passes 1e-2 and the exact counts carry the
    # discrimination
    assert full["iterations"] >= kmax and bars[min(kmax, 25)] <= BAR_MAX[dtype], (full["iterations"], bars[min(kmax, 25)])
    return full, bars


class Replay:
    """b, M^-1 and the operator of one converged solve on the problem, the replay to convergence and the bars"""

    def __init__(self, arrays, dtype, prior=None, mask=None, kmax=40, **opt):
        lin = _handle(arrays, dtype, ASM, prior, mask, **opt)
        lin.solve(LAM)
        self.b, self.inv = lin.get_rhs(), lin.get_preconditioner()[0]
        op = operator_of(lin, dtype)
        self.period = opt.get("residual_reset_period", 10)
        self.full, self.bars = _bars(op, self.b, self.inv, dtype, self.period, kmax)
        self.xs = pcg_replay(op, self.b, self.inv, eta=NEVER, max_it=kmax, period=self.period)["xs"]
        lin.close()


SWEEP = {  # id: dtype, residual_reset_period, pcg_check_period
    "f64-p10-c4": (np.float64, 10, 4),
    "f32-p10-c4": (np.float32, 10, 4),
    "f64-p3-c1": (np.float64, 3, 1),
    "f32-p3-c7": (np.float32, 3, 7),
    "f64-p10-c7": (np.float64, 10, 7),
    "f32-p10-c1": (np.float32, 10, 1),
}


def _apps(k, period):
    return k + k // period


def _check_switch_sweep(arrays, dtype, period, check, prior=None, mask=None, **opt):
    st = structure(arrays)
    size = np.dtype(dtype).itemsize
    s_def = default_switch(st, size)
    rep = Replay(arrays, dtype, prior, mask, kmax=s_def + period + 1, residual_reset_period=period, **opt)
    base = dict(eta=NEVER, residual_reset_period=period, pcg_check_period=check, **opt)
    panel = {}

    def panel_solve(k):  # the same truncation with the panel product throughout
        if k not in panel:
            panel[k] = _one_solve(arrays, dtype, PANEL, prior, mask, max_linear_solver_iterations=k, **base)
        return panel[k]
    # operator kernels + vector step (+ k_pair_ov) of one iteration without a refresh
    per_app = panel_solve(period + 1)["launches"] - panel_solve(period)["launches"]
    panel_b = panel_solve(period)["bytes"]
    assert panel_b == _panel_bytes_of(arrays, dtype)
    for s in sorted({1, 2, period - 1, period, period + 1, s_def} - {0}):
        env = {} if s == s_def else {"RBA_ASSEMBLED_AT": str(s)}
        for k in sorted({s - 1, s, s + 1, s + period} - {0}):
            r = _one_solve(arrays, dtype, env, prior, mask, max_linear_solver_iterations=k, **base)
            p = panel_solve(k)
            tag = (s, k)
            assert np.array_equal(r["b"], rep.b) and np.array_equal(r["inv"], rep.inv), tag
            assert (r["term"], r["it"], r["matvecs"], r["matvec_launches"]) == (NO_CONVERGENCE, k, _apps(k, period), _apps(k, period)), tag
            # S iff the solve reached iteration s (eta = NEVER: the host enqueues no iteration beyond k)
            assert (r["bytes"] == s_bytes(st, arrays.nc, size)) == (s <= k) and (r["bytes"] == panel_b) == (s > k), (tag, r["bytes"])
            # launches: the panel product's, the assembly (S_u + S: 4) once, and every application from iteration s on with
            # k_rcs_spmv (1 launch) instead of the panel kernels and their reduction
            after = _apps(k, period) - _apps(s - 1, period) if s <= k else 0
            op_panel = per_app - 1 - (1 if prior == "pair" else 0)
            assert r["launches"] == p["launches"] + (4 if s <= k else 0) - after * (op_panel - 1), (tag, r["launches"], p["launches"])
            assert rel_err(r["inc"], -rep.xs[k]) < rep.bars[k], (tag, rel_err(r["inc"], -rep.xs[k]), rep.bars[k])


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", list(SWEEP))
def test_switch_sweep(seq_problem, cfg):
    """RBA_ASSEMBLED_AT = s for s in {1, 2, period - 1, period, period + 1, the default}, max_linear_solver_iterations = k for
    k in {s - 1, s, s + 1, s + period} at an eta no zeta undercuts: inc = -x_k, the exact counts, the operator the solve
    ended with and the launches of the assembly"""
    dtype, period, check = SWEEP[cfg]
    _check_switch_sweep(seq_problem, dtype, period, check)


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["held", "camera-prior", "pair-prior"])
def test_switch_sweep_outside_s(seq_problem, which):
    """held cameras and the camera / pair priors are applied outside S"""
    mask = None
    if which == "held":
        mask = np.zeros(seq_problem.nc, np.uint8)
        mask[:MASK.size] = MASK
    _check_switch_sweep(seq_problem, np.float64, 10, 4, prior={"held": None, "camera-prior": "camera", "pair-prior": "pair"}[which],
                        mask=mask)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", _dtypes())
def test_assembly_once_per_linearisation(seq_problem, dtype):
    """S_u once per linearisation, S once per solve that reaches the switch (2 or 4 launches), nothing for a solve that
    stops before it is enqueued (test_s_after_a_solve_that_ended_before_the_switch: one that stops after)"""
    s, k = 5, 8
    st = structure(seq_problem)
    size = np.dtype(dtype).itemsize
    opt = dict(eta=NEVER, max_linear_solver_iterations=k)
    env = {"RBA_ASSEMBLED_AT": str(s)}
    a = _handle(seq_problem, dtype, env, **opt)
    b = _handle(seq_problem, dtype, PANEL, **opt)
    short = _handle(seq_problem, dtype, env, eta=NEVER, max_linear_solver_iterations=s - 1)
    short_p = _handle(seq_problem, dtype, PANEL, eta=NEVER, max_linear_solver_iterations=s - 1)
    extra = _apps(k, 10) - _apps(s - 1, 10)
    per_app = None
    for lam, su in ((LAM, 4), (1e-2, 2), (1.0, 2)):
        ra, rb_ = _solve_counts(a, lam), _solve_counts(b, lam)
        if per_app is None:
            per_app = (ra["launches"] - su - rb_["launches"]) // extra  # (1 - panel operator launches)
        assert ra["launches"] == rb_["launches"] + su + per_app * extra, (lam, ra["launches"], rb_["launches"])
        assert ra["bytes"] == s_bytes(st, seq_problem.nc, size) < rb_["bytes"], lam
        rs, rsp = _solve_counts(short, lam), _solve_counts(short_p, lam)
        assert rs["launches"] == rsp["launches"] and rs["bytes"] == rsp["bytes"] == rb_["bytes"], lam
    assert per_app < 0
    for lin in (a, b):
        lin.linearize()
    ra, rb_ = _solve_counts(a, LAM), _solve_counts(b, LAM)
    assert ra["launches"] == rb_["launches"] + 4 + per_app * extra
    assert ra["bytes"] == s_bytes(st, seq_problem.nc, size)
    for lin in (a, b, short, short_p):
        lin.close()


ETAS = (1e-1, 1e-2, 1e-3, 1e-4, 1e-6)
LAM_HI = 1e2  # a solve that ends after a few iterations at the same eta


@functools.lru_cache(maxsize=None)
def _eta_window(dtype, check):
    """the first eta of ETAS at which the panel-product solve at LAM ends past the first residual refresh (11 <= e <= 30,
    within the replay below), with e and the iteration e_hi at which the same eta ends the solve at LAM_HI"""
    arrays = seq_arrays()
    for eta in ETAS:
        p = _handle(arrays, dtype, PANEL, eta=eta, pcg_check_period=check)
        r, r_hi = _solve_counts(p, LAM), _solve_counts(p, LAM_HI)
        p.close()
        assert r["term"] == SUCCESS and r_hi["term"] == SUCCESS
        if 11 <= r["it"] <= 30:
            assert r_hi["it"] + check < r["it"], (eta, r_hi["it"], r["it"])
            return eta, r["it"], r_hi["it"]
    raise AssertionError("no eta of ETAS ends the solve at LAM between 11 and 30 iterations")


@pytest.mark.gpu
@pytest.mark.parametrize("check", [1, 4, 7])
@pytest.mark.parametrize("dtype", _dtypes())
def test_switch_after_the_end(seq_problem, dtype, check):
    """a solve stopped by eta at e (past a residual refresh), with the switch at e + 1, e + pcg_check_period (both enqueued
    among the no-op iterations that follow the end) and e + pcg_check_period + 1: the solve ended with the panel product, so
    inc, right_multiply and matvec_algorithmic_bytes are those of an RBA_ASSEMBLED_RCS=0 handle, bit for bit, and inc is
    the replay's -x_e"""
    eta, e, _ = _eta_window(dtype, check)
    rep = Replay(seq_problem, dtype, kmax=30)
    x = np.random.default_rng(9).uniform(-1, 1, 9 * seq_problem.nc).astype(dtype)
    p = _handle(seq_problem, dtype, PANEL, eta=eta, pcg_check_period=check)
    rp = _solve_counts(p, LAM)
    assert (rp["term"], rp["it"]) == (SUCCESS, e)
    assert rel_err(rp["inc"], -rep.xs[e]) < rep.bars[e]
    yp = p.right_multiply(x)
    for s in sorted({e + 1, e + check, e + check + 1}):
        env = {"RBA_ASSEMBLED_AT": str(s)}
        a = _handle(seq_problem, dtype, env, eta=eta, pcg_check_period=check)
        ra = _solve_counts(a, LAM)
        assert (ra["term"], ra["it"]) == (SUCCESS, e), s
        assert np.array_equal(ra["inc"], rp["inc"]), s
        assert ra["bytes"] == rp["bytes"], ("the solve ended before the switch, the handle reports S", s, ra["bytes"], rp["bytes"])
        assert np.array_equal(a.right_multiply(x), yp), ("right_multiply after a solve that ended before the switch", s)
        a.close()
    p.close()


@pytest.mark.gpu
@pytest.mark.parametrize("check", [1, 4, 7])
@pytest.mark.parametrize("dtype", _dtypes())
def test_s_after_a_solve_that_ended_before_the_switch(seq_problem, dtype, check):
    """one handle, one linearisation, a fixed eta: a solve at LAM_HI ends at e_hi, and the switch s = e_hi + 1 or
    e_hi + pcg_check_period is enqueued after its end, so its assembly does nothing.  The next solve, at LAM, runs past s:
    it must build S_u as well as S (the launches of a fresh handle's first solve, 4 for the assembly) and equal the fresh
    handle bit for bit (inc, S).  A handle whose S_u was built by an earlier solve keeps it across such a solve: S alone
    (2 launches fewer), the same S"""
    eta, e, e_hi = _eta_window(dtype, check)
    st = structure(seq_problem)
    size = np.dtype(dtype).itemsize
    panel_b = _panel_bytes_of(seq_problem, dtype)
    for s in sorted({e_hi + 1, e_hi + check}):
        env = {"RBA_ASSEMBLED_AT": str(s)}
        fresh = _handle(seq_problem, dtype, env, eta=eta, pcg_check_period=check)
        rf = _solve_counts(fresh, LAM)
        assert rf["it"] == e >= s and rf["bytes"] == s_bytes(st, seq_problem.nc, size) < panel_b, (s, rf["it"])
        Yf = extract(fresh)
        fresh.close()
        a = _handle(seq_problem, dtype, env, eta=eta, pcg_check_period=check)
        r1 = _solve_counts(a, LAM_HI)
        assert (r1["it"], r1["bytes"]) == (e_hi, panel_b), (s, r1["it"])
        r2 = _solve_counts(a, LAM)
        assert r2["launches"] == rf["launches"], ("S_u not rebuilt after an assembly that did nothing", s, r2["launches"], rf["launches"])
        assert r2["bytes"] == rf["bytes"] and r2["it"] == rf["it"] and np.array_equal(r2["inc"], rf["inc"]), s
        assert np.array_equal(extract(a), Yf), ("S after a solve whose assembly came after its end", s)
        a.close()
        b = _handle(seq_problem, dtype, env, eta=eta, pcg_check_period=check)
        _solve_counts(b, LAM)
        assert _solve_counts(b, LAM_HI)["bytes"] == panel_b
        r3 = _solve_counts(b, LAM)
        assert r3["launches"] == rf["launches"] - 2, ("S_u rebuilt although it was valid", s, r3["launches"], rf["launches"])
        assert np.array_equal(r3["inc"], rf["inc"]) and np.array_equal(extract(b), Yf), s
        b.close()
