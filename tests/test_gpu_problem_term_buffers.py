"""The device buffers of every problem term across replacements (rootba_b200/csrc/solver.cu: the setters' term structs).
Each term kind is set with a larger list, a smaller one, cleared and set again on one handle.  After every set, one
compute_error, linearize, solve and apply is bit-identical to a fresh handle created with that term; device_bytes grows only
when a list outgrows its buffers, by exactly the bytes of the new ones (max(count, 1) entries each, never freed from the
count); and a call rejected after the list has grown leaves the grown term in force."""
import ctypes as C

import numpy as np
import pytest

import camera_prior_model as pm
import landmark_prior_model as lp
import observation_info_model as oi
import pair_prior_model as qm
from test_gpu_kernel_classes import group_size_for

pytestmark = pytest.mark.gpu

LAM = 1e-4
DTYPES = [np.float32, np.float64]


def _p(a):
    return C.c_void_p(a.ctypes.data)


def _layout_sizes(arrays):
    """(sorted landmarks, slots) of the one-rank tile layout: each track-length class n is cut into tiles of 32 / G(n)
    landmarks, padding included"""
    n = np.diff(arrays.lm_off)
    nsorted = nslots = 0
    for length, count in zip(*np.unique(n, return_counts=True)):
        w = 32 // group_size_for(int(length))
        padded = -(-int(count) // w) * w
        nsorted += padded
        nslots += padded * int(length)
    return nsorted, nslots


def _pairs(arrays, m, seed):
    rng = np.random.default_rng(seed)
    nc = arrays.nc
    pairs = np.array([(k % nc, (k + 1 + k // nc) % nc) for k in range(m)], np.int32)
    mean = qm.mean_at(arrays.cams, pairs)
    mean[:, 4:7] += rng.normal(0, 0.05, (m, 3))
    return pairs, mean, np.stack([qm.sqrt_info_kind("dense", rng, 0.5) for _ in range(m)])


def _groups(nc, sizes):
    g = np.full(nc, -1, np.int32)
    c = 0
    for k, s in enumerate(sizes):
        g[c:c + s] = k
        c += s
    return g


# per kind: the BalProblem attribute, the values in turn (None = cleared), the bytes the k-th value's new buffers add for
# scalar size s (given the previous values), and a rejected raw call on the handle
def _kinds(arrays):
    nc, nl, nobs = arrays.nc, arrays.nl, len(arrays.obs_cam)
    nsorted, nslots = _layout_sizes(arrays)
    held = [np.array([1 if c % 3 == 0 else 0 for c in range(nc)], np.uint8), np.array([15] + [2] * (nc - 1), np.uint8),
            None, np.array([1 if c % 3 == 0 else 0 for c in range(nc)], np.uint8)]
    cam = [pm.small_prior(arrays, 3), pm.small_prior(arrays, 4), None, pm.small_prior(arrays, 3)]
    pair = [_pairs(arrays, 5, 1), _pairs(arrays, 2 * nc + 3, 2), _pairs(arrays, 8, 3), None, _pairs(arrays, 2 * nc + 3, 2)]
    lmk = [lp.prior_case(arrays.lms, every=e, seed=e, kinds=("dense",)) for e in (30, 5, 15)]
    lmk = lmk + [None, lmk[1]]
    grp = [_groups(nc, [2, 3]), _groups(nc, [4, 3, nc - 7]), _groups(nc, [2]), None, _groups(nc, [4, 3, nc - 7])]
    obs = [oi.random_info(nobs, 1), oi.random_info(nobs, 2), None, oi.random_info(nobs, 1)]

    def pair_bytes(m, s):
        return m * (6 * 4 + 193 * s)

    def grp_bytes(g):
        members = [np.count_nonzero(g == k) for k in range(nc)]
        ng = sum(1 for x in members if x >= 2)
        return 4 * (nc + ng + 1 + sum(x for x in members if x >= 2))

    def bad_held(lib, h, bp):
        f = bp.camera_fixed.copy()
        f[1] = 16
        return lib.rba_set_camera_fixed(h, _p(f))

    def bad_prior(fn, attr):
        def call(lib, h, bp):
            v = getattr(bp, attr)
            L = v[-1].copy()
            L[1].flat[0] = np.nan
            head = (C.c_int32(len(v[0])), _p(v[0])) if len(v) == 3 else ()
            return getattr(lib, fn)(h, *head, _p(v[-2]), _p(L))
        return call

    def bad_groups(lib, h, bp):
        g = bp.intrinsics_group.copy()
        g[0] = nc
        return lib.rba_set_intrinsics_groups(h, _p(g))

    def bad_obs(lib, h, bp):
        W = bp.observation_sqrt_info.copy()
        W[3, 1, 0] = np.inf
        return lib.rba_set_observation_info(h, _p(W))

    return {
        "held": ("camera_fixed", held, lambda k, s: nc if k == 0 else 0, bad_held),
        "camera_prior": ("camera_prior", cam, lambda k, s: 271 * nc * s if k == 0 else 0,
                         bad_prior("rba_set_camera_prior", "camera_prior")),
        "pair_prior": ("camera_pair_prior", pair,
                       lambda k, s: {0: pair_bytes(5, s) + 4 * (nc + 1) + 99 * nc * s, 1: pair_bytes(2 * nc + 3, s)}.get(k, 0),
                       bad_prior("rba_set_camera_pair_prior", "camera_pair_prior")),
        "landmark_prior": ("landmark_prior", lmk,
                           lambda k, s: {0: len(lmk[0][0]) * (4 + 24 * s) + 4 * (nsorted + nl),
                                         1: len(lmk[1][0]) * (4 + 24 * s)}.get(k, 0),
                           bad_prior("rba_set_landmark_prior", "landmark_prior")),
        "groups": ("intrinsics_group", grp,
                   lambda k, s: 0 if grp[k] is None else grp_bytes(grp[k]) + (18 * nc * s + nc if k == 0 else 0), bad_groups),
        "observation_info": ("observation_sqrt_info", obs, lambda k, s: 4 * nslots * s if k == 0 else 0, bad_obs),
    }


def _step(lin, arrays):
    """compute_error, linearize, solve, apply from the problem's initial state; everything the caller sees"""
    bp = lin.bal_problem
    bp.cams[:] = arrays.cams
    bp.lms[:] = arrays.lms
    lin.upload_state()
    e = lin.compute_error()
    lin.linearize()
    inc = lin.solve(LAM)
    l_diff = lin.apply(inc)
    lin.download_state()
    return e, inc, l_diff, bp.cams.copy(), bp.lms.copy()


def _assert_identical(got, ref, what):
    assert got[0] == ref[0], what
    assert np.array_equal(got[1], ref[1]), what
    assert got[2] == ref[2] or (np.isnan(got[2]) and np.isnan(ref[2])), what
    assert np.array_equal(got[3], ref[3]) and np.array_equal(got[4], ref[4]), what


def _fresh(arrays, dtype, attr, value):
    import rootba_b200 as rb
    bp = rb.BalProblem.from_arrays(arrays, dtype)
    if value is not None:
        setattr(bp, attr, value)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions())
    try:
        return _step(lin, arrays)
    finally:
        lin.close()


@pytest.mark.parametrize("kind", ["held", "camera_prior", "pair_prior", "landmark_prior", "groups", "observation_info"])
@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
def test_replaced_term_matches_a_fresh_handle(tiny_problem, dtype, kind):
    import rootba_b200 as rb
    from rootba_b200 import _lib
    lib = _lib.lib()
    arrays = tiny_problem
    attr, values, grown, bad = _kinds(arrays)[kind]
    s = np.dtype(dtype).itemsize
    bp = rb.BalProblem.from_arrays(arrays, dtype)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions())
    try:
        for k, value in enumerate(values):
            before = lin.stats()["device_bytes"]
            setattr(bp, attr, value)
            assert lin.stats()["device_bytes"] - before == grown(k, s), (kind, k)
            ref = _fresh(arrays, dtype, attr, value)
            _assert_identical(_step(lin, arrays), ref, (kind, k))
            if k == 1:  # the term has grown: a rejected call keeps it and allocates nothing
                after = lin.stats()["device_bytes"]
                assert bad(lib, lin.h, bp) == -1 and lib.rba_last_error()  # RBA_ERR_INVALID_ARGUMENT
                assert lin.stats()["device_bytes"] == after
                _assert_identical(_step(lin, arrays), ref, (kind, k, "after a rejected call"))
    finally:
        lin.close()
