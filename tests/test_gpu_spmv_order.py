"""The summation order of the assembled product k_rcs_spmv (assembled.cuh, layout.hpp), bit for bit.  Entry e = 9 p + q of
block row r is fixed as: SPMV_CLASSES = 4 fma chains, chain c over the row's blocks k with k - (row start) = c mod 4 in
ascending order, each from 0 with the terms S_k[e] x[col_k][q]; then the 4 x 9 partials of output p added from 0, chain by
chain, q ascending.  y = right_multiply(x) after the switch to S is compared with an exact restatement of that order: every
fma and add evaluated in integers and rounded once, to nearest even, to the target type (no float64 detour for float32,
which could round twice).

The problem has block rows across every stage and chunk edge of both types (16 or 32 blocks per stage, 3 stages in the
ring), a hub row of 130 blocks (5 float32 chunks, 9 float64 chunks), rows of 2 and cameras without observations (rows without blocks, y = 0).  It runs with the
grid of the device and with the rows dealt over 1 and 3 CTAs (RBA_SPMV_CTAS), so that a CTA takes many rows and wraps its
stage ring inside and across rows; all three give the same y.

Reading S.  right_multiply(e_j) gives column j of S + lambda I, exactly off the diagonal (every other product is an exact
zero).  A diagonal entry carries lambda, so x is zero on a set of cameras and only the rows of those cameras are checked:
there the diagonal entries multiply zeros, and right_multiply's lambda x adds zero.  Two complementary sets cover every row."""
import contextlib
import functools
import math
import os

import numpy as np
import pytest
import scipy.sparse as sp

SPMV_CLASSES = 4
HUB_ROWS = (2, 15, 16, 17, 31, 32, 33, 47, 48, 49, 63, 64, 65, 95, 96, 97, 127, 128, 129, 130)
PER_PAIR = 24    # landmarks (n = 2) per co-visible pair
UNOBSERVED = 3   # cameras at the end that no landmark sees
LAM = 1e-3


@functools.lru_cache(maxsize=None)
def problem():
    """hub h shares landmarks with the fillers 0 .. HUB_ROWS[h] - 2 (its row holds HUB_ROWS[h] blocks, the diagonal
    included); filler f's row holds 1 + the number of hubs that see it; PER_PAIR landmarks of n = 2 per pair, shuffled"""
    from rootba_b200.synthetic import BalArrays, synth_bal
    nh, nf = len(HUB_ROWS), max(HUB_ROWS) - 1
    tracks = [np.array([h, nh + f]) for h, d in enumerate(HUB_ROWS) for f in range(d - 1) for _ in range(PER_PAIR)]
    rng = np.random.default_rng(1723)
    tracks = [tracks[i] for i in rng.permutation(len(tracks))]
    a = synth_bal(nh + nf, len(tracks), 0.0, seed=1723, tracks=tracks, lm_spread=0.5)
    return BalArrays(np.concatenate([a.cams, a.cams[:UNOBSERVED]]), a.lms, a.lm_off, a.obs_cam, a.obs_xy)


def block_rows(arrays):
    """the camera-major block-row CSR of S (both triangles, columns ascending)"""
    A = sp.csr_matrix((np.ones(arrays.obs_cam.size, np.int32), arrays.obs_cam, arrays.lm_off), shape=(arrays.nl, arrays.nc))
    S = (A.T @ A).tocsr()
    S.sort_indices()
    return S.indptr.astype(np.int64), S.indices.astype(np.int64)


# ---- exact arithmetic ----
FMT = {np.float32: (24, -126), np.float64: (53, -1022)}  # significand bits, least normal exponent


def _exact(v):
    """v = n 2^e exactly"""
    m, e = math.frexp(v)
    return int(m * (1 << 53)), e - 53


def _round(n, e, fmt):
    """n 2^e rounded to nearest even in the format (subnormals included; no overflow in these problems)"""
    if n == 0:
        return 0.0
    bits, emin = fmt
    sign, n = (-1, -n) if n < 0 else (1, n)
    sh = max(n.bit_length() - bits, (emin - bits + 1) - e)
    if sh > 0:
        q, r, half = n >> sh, n & ((1 << sh) - 1), 1 << (sh - 1)
        if r > half or (r == half and q & 1):
            q += 1
        n, e = q, e + sh
    return sign * math.ldexp(n, e)


def fma(a, b, c, fmt):
    na, ea = _exact(a)
    nb, eb = _exact(b)
    nc, ec = _exact(c)
    n1, e1 = na * nb, ea + eb
    e = min(e1, ec)
    return _round((n1 << (e1 - e)) + (nc << (ec - e)), e, fmt)


def spmv_restated(row_ptr, col, blocks, x, rows, fmt):
    """y of the listed block rows in k_rcs_spmv's order; blocks[k] = the 9 x 9 block k of the CSR as Python floats"""
    y = {}
    for r in rows:
        k0, k1 = int(row_ptr[r]), int(row_ptr[r + 1])
        for p in range(9):
            t = 0.0
            for c in range(SPMV_CLASSES):
                for q in range(9):
                    acc = 0.0
                    for k in range(k0 + c, k1, SPMV_CLASSES):
                        acc = fma(blocks[k][p][q], x[9 * int(col[k]) + q], acc, fmt)
                    t = fma(1.0, acc, t, fmt)
            y[9 * r + p] = t
    return y


# ---- GPU ----
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


def _handle(arrays, dtype, ctas):
    import rootba_b200 as rb
    env = {"RBA_ASSEMBLED_AT": "1"}
    if ctas:
        env["RBA_SPMV_CTAS"] = str(ctas)
    with _env(env):
        bp = rb.BalProblem.from_arrays(arrays, dtype)
        lin = rb.LinearizorQR.create(bp, rb.SolverOptions(use_double=dtype == np.float64))
    lin.linearize()
    lin.solve(LAM)
    # S was taken (Solver::get_stats: the bytes of S and of x and y, and its CSR)
    row_ptr, col = block_rows(arrays)
    s, nnzb, nc = np.dtype(dtype).itemsize, col.size, arrays.nc
    assert lin.stats()["matvec_algorithmic_bytes"] == (81 * nnzb + 18 * nc) * s + 4 * (nnzb + nc + 1)
    return lin


def extract_blocks(lin, row_ptr, col, nc):
    """the blocks of S + lambda I in CSR order, from right_multiply of the 9 nc unit vectors"""
    Y = np.empty((9 * nc, 9 * nc))
    e = np.zeros(9 * nc, lin.dtype)
    for j in range(9 * nc):
        e[j] = 1
        Y[:, j] = lin.right_multiply(e)
        e[j] = 0
    rows = np.repeat(np.arange(nc), np.diff(row_ptr))
    return [Y[9 * r:9 * r + 9, 9 * c:9 * c + 9].tolist() for r, c in zip(rows.tolist(), col.tolist())]


def test_problem_reaches_the_edges():
    """(CPU) the rows cross every stage edge of both types and the ring of 3 stages, and cameras without blocks exist"""
    arrays = problem()
    row_ptr, _ = block_rows(arrays)
    n = set(np.diff(row_ptr).tolist())
    for stage in (16, 32):
        for m in (1, 2, 3, 4):
            assert {m * stage - 1, m * stage, m * stage + 1} <= n
    assert 0 in n and max(n) > 3 * 32  # rows without blocks, and a row longer than the float32 ring (3 stages of 32 blocks)
    assert np.count_nonzero(np.diff(row_ptr) == 0) == UNOBSERVED


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [pytest.param(np.float32, id="float32"), pytest.param(np.float64, id="float64")])
def test_spmv_order_exact(dtype):
    arrays = problem()
    nc = arrays.nc
    row_ptr, col = block_rows(arrays)
    fmt = FMT[dtype]
    lins = {ctas: _handle(arrays, dtype, ctas) for ctas in (0, 1, 3)}
    blocks = extract_blocks(lins[0], row_ptr, col, nc)
    rng = np.random.default_rng(38401)
    zero_cams = rng.permutation(nc) < nc // 2
    for half in (zero_cams, ~zero_cams):
        x = rng.uniform(-1, 1, 9 * nc).astype(dtype)
        x[np.repeat(half, 9)] = 0
        ys = {ctas: lin.right_multiply(x) for ctas, lin in lins.items()}
        for ctas in (1, 3):
            assert ys[ctas].tobytes() == ys[0].tobytes(), ("rows dealt over", ctas, "CTAs")
        rows = np.flatnonzero(half)
        want = spmv_restated(row_ptr, col, blocks, x.astype(np.float64).tolist(), rows.tolist(), fmt)
        got = ys[0].astype(np.float64)
        bad = [(i // 9, int(np.diff(row_ptr)[i // 9]), i % 9, got[i], w) for i, w in want.items() if got[i] != w]
        assert not bad, bad[:5]
    for lin in lins.values():
        lin.close()
