"""Held camera parameters (rba_set_camera_fixed) without a GPU: the exactness argument of DESIGN.md ("Fixed camera
parameters") restated in float64 numpy, and bal_qr's argument checks.

The device masks only the block-Jacobi inverse M^-1 (fixed rows and columns zero) and b (fixed entries zero), once per solve.
The PCG recurrences of k_pcg_vec (tests/pcg_replay.py) then never move a fixed entry of x, and the free entries follow PCG on the restricted
system H_ff x_f = -b_f iteration for iteration.  Same for the power series with the masked Hpp^-1."""
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT, rel_err
from objective_checks import MASK, fixed_entries
from pcg_replay import pcg_replay

def masked_block_inverse(blocks, fixed):
    """k_precond_invert with flags: fixed rows / columns of each 9x9 block -> identity, invert, zero them in the inverse"""
    out = np.zeros_like(blocks)
    for c, blk in enumerate(blocks):
        f = fixed[9 * c:9 * c + 9]
        a = blk.copy()
        a[f, :] = 0
        a[:, f] = 0
        a[f, f] = 1
        inv = np.linalg.inv(a)
        inv[f, :] = 0
        inv[:, f] = 0
        out[c] = inv
    return out


def block_apply(inv_blocks, v):
    return np.einsum("cij,cj->ci", inv_blocks, v.reshape(-1, 9)).ravel()


@pytest.fixture(scope="module")
def system():
    from rootba_b200.synthetic import synth_bal
    from test_oracle_dense_numpy import _dense_system, _reduced
    prob = synth_bal(7, 90, 3.6, seed=21)
    Jp, Jl, r = _dense_system(prob)
    lam = 1e-3
    D, sl, Jps, Jls, Minv, H, b = _reduced(Jp, Jl, r, lam, prob.nl, float(np.sqrt(1e-10)))
    W = Jps.T @ Jls
    return prob, lam, Jps, H, b, W @ Minv @ W.T


def test_masked_inverse_is_the_inverse_of_the_free_sub_block(system):
    prob, lam, Jps, H, b, E0 = system
    fixed = fixed_entries(MASK)
    blocks = np.array([H[9 * c:9 * c + 9, 9 * c:9 * c + 9] for c in range(prob.nc)])
    inv = masked_block_inverse(blocks, fixed)
    for c in range(prob.nc):
        f = fixed[9 * c:9 * c + 9]
        assert np.all(inv[c][f, :] == 0) and np.all(inv[c][:, f] == 0)
        if (~f).any():
            want = np.linalg.inv(blocks[c][np.ix_(~f, ~f)])
            assert rel_err(inv[c][np.ix_(~f, ~f)], want) < 1e-13
    # the fully fixed camera contributes nothing
    assert np.all(inv[3] == 0)


def test_pcg_with_masked_preconditioner_is_pcg_on_the_restricted_system(system):
    prob, lam, Jps, H, b, E0 = system
    fixed = fixed_entries(MASK)
    free = ~fixed
    blocks = np.array([H[9 * c:9 * c + 9, 9 * c:9 * c + 9] for c in range(prob.nc)])
    inv = masked_block_inverse(blocks, fixed)
    bm = np.where(fixed, 0.0, b)
    xs = pcg_replay(lambda v: H @ v, bm, inv, eta=1e-13, max_it=300)["xs"]
    # restricted problem: fixed rows and columns deleted, block-Jacobi on the free sub-blocks
    Hff, bf = H[np.ix_(free, free)], b[free]
    sizes = [int(free[9 * c:9 * c + 9].sum()) for c in range(prob.nc)]
    starts = np.concatenate([[0], np.cumsum(sizes)])
    inv_f = [np.linalg.inv(Hff[starts[c]:starts[c + 1], starts[c]:starts[c + 1]]) if sizes[c] else None for c in range(prob.nc)]

    def minv_f(v):
        return np.concatenate([inv_f[c] @ v[starts[c]:starts[c + 1]] for c in range(prob.nc) if sizes[c]])
    xs_f = pcg_replay(lambda v: Hff @ v, bf, minv_f, eta=1e-13, max_it=300)["xs"]
    assert len(xs) == len(xs_f) > 10  # same iteration count: same zeta history
    for x, xf in zip(xs, xs_f):
        assert np.all(x[fixed] == 0)
        assert rel_err(x[free], xf) < 1e-12
    want = -np.linalg.solve(Hff, bf)
    assert rel_err(-xs[-1][free], want) < 1e-8 * np.linalg.cond(Hff) ** 0.5  # the bar of test_oracle_dense_numpy.py


def test_power_series_with_masked_hpp_inverse_is_the_restricted_series(system):
    prob, lam, Jps, H, b, E0 = system
    fixed = fixed_entries(MASK)
    free = ~fixed
    N = H.shape[0]
    Hpp = Jps.T @ Jps + lam * np.eye(N)
    inv = masked_block_inverse(np.array([Hpp[9 * c:9 * c + 9, 9 * c:9 * c + 9] for c in range(prob.nc)]), fixed)
    bm = np.where(fixed, 0.0, b)
    Hpp_ff_inv = np.linalg.inv(Hpp[np.ix_(free, free)])  # block diagonal
    E0_ff, bf = E0[np.ix_(free, free)], b[free]

    def series(apply_inv, E, rhs, eta, order):  # k_power_vec: accum = Hpp^-1 (-b); tmp = Hpp^-1 (E0 tmp); zeta rule
        tmp = -apply_inv(rhs)
        acc = tmp.copy()
        out = [acc.copy()]
        for i in range(1, order + 1):
            tmp = apply_inv(E @ tmp)
            acc = acc + tmp
            out.append(acc.copy())
            if i * np.linalg.norm(tmp) / np.linalg.norm(acc) < eta:
                break
        return out
    full = series(lambda v: block_apply(inv, v), E0, bm, 1e-13, 40)
    restricted = series(lambda v: Hpp_ff_inv @ v, E0_ff, bf, 1e-13, 40)
    assert len(full) == len(restricted)
    for a, af in zip(full, restricted):
        assert np.all(a[fixed] == 0)
        assert rel_err(a[free], af) < 1e-12
    # and it approaches the restricted solution
    want = -np.linalg.solve(H[np.ix_(free, free)], bf)
    errs = [rel_err(full[m][free], want) for m in (0, 5, len(full) - 1)]
    assert errs[0] > errs[1] > errs[2]


BAL_QR = os.path.join(ROOT, "rootba_b200", "host", "bal_qr")


@pytest.mark.parametrize("arg", ["1,,2", "-1", "a", "", "0,3x", "99"])
def test_bal_qr_rejects_a_bad_camera_list(tmp_path, arg):
    """a malformed list fails while parsing the arguments, an index past the loaded problem right after loading it: both
    before any GPU work, with exit code 2"""
    from test_host_cpp import _build
    from rootba_b200.synthetic import synth_bal, write_bal
    _build()
    path = str(tmp_path / "p.txt")
    write_bal(synth_bal(5, 40, 3.0, seed=2, normalize_scale=None), path)
    r = subprocess.run([BAL_QR, "--input", path, "--fix-cameras", arg, "--log-path", str(tmp_path / "log.json")],
                       capture_output=True, text=True, timeout=120)
    assert r.returncode == 2, (r.stdout, r.stderr)
    assert "--fix-cameras" in r.stderr
    assert not (tmp_path / "log.json").exists()
