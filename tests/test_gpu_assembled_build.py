"""The damping pass of the assembled reduced camera matrix (assembled.cuh: k_rcs_damping + k_rcs_mirror): S = S_u + the
damping rows' part with every term formed from the two slots' dmp records, a warp per camera pair fetching DMP_BATCH terms
at a time.  test_gpu_assembled_classes checks S at every track-length class; here

  * pair lists of every length around the batch sizes (6 .. 100 terms, and a diagonal pair of several hundred), against
    float64 block by block, for two lambdas in a row on one linearisation (the second solve runs the damping pass alone)
    and bit for bit against a fresh handle;
  * the dmp records of stage2_form = IDENTITY (k_stage2<S, false> writes them from shared memory, the panel form from
    registers): the same S bit for bit at every track-length class, with cameras that no landmark sees.

A landmark seen twice by one camera cannot be generated (synth_bal makes the cameras of a track distinct).
"""
import functools

import numpy as np
import pytest

from test_gpu_assembled_classes import (ASM, LAM1, LAM2, _dtypes, _handle, _panel_bytes_of, check_s, extract, mixed_unobserved,
                                        s_bytes, structure)

DMP_BATCH = 16  # assembled.cuh
LIST_LENGTHS = (6, 7, 15, 16, 17, 31, 32, 33, 47, 48, 49, 64, 65, 100)


@functools.lru_cache(maxsize=None)
def hub_problem():
    """camera 0 shares LIST_LENGTHS[i] landmarks (n = 2) with camera i + 1 and with no other: the pairs (i + 1, 0) and
    (i + 1, i + 1) have lists of that length, the pair (0, 0) one of their sum; landmarks shuffled"""
    from rootba_b200.synthetic import synth_bal
    tracks = [np.array([0, i + 1]) for i, m in enumerate(LIST_LENGTHS) for _ in range(m)]
    rng = np.random.default_rng(41)
    tracks = [tracks[i] for i in rng.permutation(len(tracks))]
    return synth_bal(len(LIST_LENGTHS) + 1, len(tracks), 0.0, seed=41, tracks=tracks, lm_spread=0.5)


def test_hub_problem_reaches_the_batch_edges():
    """(CPU) list lengths around one, two and four batches, a list of more than twenty batches, and S qualifies"""
    arrays, st = hub_problem(), structure(hub_problem())
    m = st["m"]
    assert sorted(m[0, 1:].tolist()) == sorted(LIST_LENGTHS) and np.array_equal(np.diag(m)[1:], m[0, 1:])
    b = DMP_BATCH
    assert {b - 1, b, b + 1, 2 * b - 1, 2 * b, 2 * b + 1, 4 * b + 1} <= set(LIST_LENGTHS)
    assert m[0, 0] == sum(LIST_LENGTHS) > 20 * b
    assert np.count_nonzero(m[1:, 1:] - np.diag(np.diag(m)[1:])) == 0
    assert 4 * st["nnzb"] * 81 <= st["panel"] and arrays.nc == len(LIST_LENGTHS) + 1


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", _dtypes())
def test_pair_list_lengths(dtype):
    arrays, st = hub_problem(), structure(hub_problem())
    size = np.dtype(dtype).itemsize
    panel_b = _panel_bytes_of(arrays, dtype)
    lin = _handle(arrays, dtype, ASM)
    for lam in (LAM1, LAM2, 3.0):
        k0 = lin.timings()["kernel_launches"]
        lin.solve(lam)
        launches = lin.timings()["kernel_launches"] - k0
        assert lin.stats()["matvec_algorithmic_bytes"] == s_bytes(st, arrays.nc, size) < panel_b
        Y = extract(lin)
        check_s(Y, lin, arrays, st, lam, dtype, ("hub", lam))
        fresh = _handle(arrays, dtype, ASM)
        k0 = fresh.timings()["kernel_launches"]
        fresh.solve(lam)
        # the fresh handle builds S_u as well: two launches more for the same number of PCG iterations
        assert fresh.last_cg.num_iterations == lin.last_cg.num_iterations, lam
        assert fresh.timings()["kernel_launches"] - k0 == launches + (0 if lam == LAM1 else 2), lam
        assert np.array_equal(extract(fresh), Y), ("S depends on the lambda before", lam)
        fresh.close()
    lin.close()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", _dtypes())
def test_identity_form_builds_the_same_s(dtype):
    arrays = mixed_unobserved()
    got = {}
    for form in ("PANEL", "IDENTITY"):
        lin = _handle(arrays, dtype, ASM, stage2_form=form)
        got[form] = []
        for lam in (LAM1, LAM2):
            lin.solve(lam)
            assert lin.stats()["matvec_algorithmic_bytes"] < _panel_bytes_of(arrays, dtype)
            got[form].append(extract(lin))
        lin.close()
    for lam, a, b in zip((LAM1, LAM2), got["PANEL"], got["IDENTITY"]):
        assert np.array_equal(a, b), ("S differs between the stage-2 forms", lam)
        seen = np.repeat(np.bincount(arrays.obs_cam, minlength=arrays.nc) > 0, 9)
        assert not seen.all() and np.array_equal(a[~seen], float(dtype(lam)) * np.eye(9 * arrays.nc)[~seen])
