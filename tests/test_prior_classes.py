"""CPU side of tests/test_gpu_prior_classes.py.  At import: the GPU cases reach both sides of every boundary of the prior and
intrinsics-group kernels (tests/prior_classes.py reads the launch geometry from the sources).  The tests: the per-camera and
per-item checkers accept a float64 and a float32 restatement of the kernels' loops and reject, at every shape where the fault
applies, a camera's prior terms written to its neighbour, the last camera of a 128-thread block dropped, one incident pair side
dropped or doubled, O_ij applied to v_i instead of v_j, the 257th item of the cost or l_diff sum dropped, a group's 129th
member left out of its sum, and (with the replay) the camera-prior term missing on the strided path of k_pcg_vec.
"""
import numpy as np
import pytest

import prior_classes as pc
from conftest import rel_err
from pcg_replay import lanczos_condition, pcg_replay
from prior_classes import (C_LIN, GROUP_SIZES, GROUP_THREADS, HUB, HUB_33, HUB_ISOLATED, HUB_NC, HUB_SIDES, PER_THREAD,
                           SUM_THREADS, PriorTerms, check_b, check_bar, check_inverse_blocks, check_item_sum, check_scaling,
                           group_k, group_layout, group_sum_model, hub_pairs, kernel_group_sum, kernel_hx, kernel_item_sum,
                           landmark_cost_items, side_counts)
from test_gpu_camera_classes import CLUSTERS, UNOBSERVED_LAST, VEC_CASES, vec_partition, vec_problem
from test_gpu_prior_classes import P3_CASES, _items, _p3_case, _vec_params

# ---- part 1: the GPU cases sit on both sides of every boundary ----------------------------------------------------------
# thread per camera / per pair, <<<ceil(n / 128), 128>>>: a full block (128), one camera short of it (127), one thread in a
# further block (129, 257), and more than 113 cameras per CTA of 16 (1900)
_P3 = {name: _p3_case(name) for name in P3_CASES}
_NC = {a.nc for a, *_ in _P3.values()}
_M = {len(p[0]) for _, _, p, _ in _P3.values()}
assert {127, 128, 129, 257} <= _NC and max(_NC) == HUB_NC > 113 * 16, _NC
assert {n % PER_THREAD for n in _NC} >= {127, 0, 1} and {pc.blocks_of(n) for n in _NC} >= {1, 2, 3, 15}
assert {127, 128, 129} <= _M and max(_M) >= 3000, _M                        # pairs: k_pair_linearize, k_pair_scale
# one block of 256 strided over the items: fewer than a round, a full round, one and two items more per thread
_ITEMS = {(p.values[0], p.values[1]) for p in _items("camera") + _items("pair") + _items("landmark")}
for _kind in ("camera", "pair", "landmark"):
    _n = {n for k, n in _ITEMS if k == _kind}
    assert {255, 256, 257, 511, 512, 513} <= _n and max(_n) > 4000 and min(_n) <= 2, (_kind, _n)
    assert {-(-n // SUM_THREADS) for n in _n} >= {1, 2, 3} and any(n % SUM_THREADS == 1 for n in _n)
assert 1 in {n for k, n in _ITEMS if k == "pair"} and 1 in {n for k, n in _ITEMS if k == "landmark"}
# incident pair sides per camera: 0, 1, 2, 33, >= 300 at the hub, which holds a repeated pair, a reversed pair, a pair to the
# unobserved last camera and one to camera 5 (held in test_pcg_iterates_at_the_hub_with_a_held_neighbour)
_HP = hub_pairs()
_SIDES = side_counts(HUB_NC, _HP)
assert {0, 1, 2} <= set(_SIDES) and _SIDES[HUB_33] == 33 and _SIDES[HUB] == HUB_SIDES >= 300
assert np.all(_SIDES[list(HUB_ISOLATED)] == 0)
_AT_HUB = [tuple(p) for p in _HP if HUB in p]
assert _AT_HUB.count((HUB, 5)) >= 2 and (5, HUB) in _AT_HUB and (HUB_NC - 1, HUB) in _AT_HUB
assert np.bincount(vec_problem(HUB_NC, True).obs_cam, minlength=HUB_NC)[-1] == 0
# groups: the strided member loop with 1, 2, 3 and 4 members per thread, the tree; a lead at the end of a 128-camera block;
# grouped and ungrouped cameras in the last camera block (next to the group blocks of the grid ncb + ng)
_G = group_layout()
_SIZES = sorted(np.bincount(_G[_G >= 0]))
_SIZES_ID = {int(np.sum(_G == k)): k for k in range(len(GROUP_SIZES))}
assert set(GROUP_SIZES) <= set(_SIZES) and {2, 127, 128, 129, 256, 257} <= set(_SIZES) and max(_SIZES) > 3 * GROUP_THREADS
assert {-(-s // GROUP_THREADS) for s in _SIZES} >= {1, 2, 3, 4}
assert _G[127] >= 0 and np.flatnonzero(_G == _G[127])[0] == 127 and 127 % GROUP_THREADS == GROUP_THREADS - 1
_LAST = _G[(HUB_NC - 1) // GROUP_THREADS * GROUP_THREADS:]
assert np.any(_LAST >= 0) and np.any(_LAST < 0)
# k_pcg_vec<S, true, *> / k_power_vec<S, true>: the iterate tests run over VEC_CASES with pair priors ((b), and (c) with
# groups), and with camera priors only at clusters 1 and 16 ((a)): every property _reached() of test_gpu_camera_classes
# asserts for the kernel without priors
_B = {(p.values[0], p.values[1]) for p in _vec_params()}
_A = {(p.values[0], p.values[1]) for p in _vec_params(clusters=(1, 16))}
assert _B == set(VEC_CASES)
for _cases in (_B, _A):
    _parts = [vec_partition(nc, c) for c, nc in _cases]
    assert {p["cached"] for p in _parts} == {True, False} and {p["straddle"] for p in _parts} == {True, False}
    assert any(p["empty"] > 0 for p in _parts) and any(p["empty"] == 0 for p in _parts)
    assert {p["ragged"] for p in _parts} == {True, False}
    assert any(vec_partition(nc, c)["last_range"][1] == nc and (c, nc) in UNOBSERVED_LAST for c, nc in _cases)
assert all((c, 113 * c) in _B and (c, 113 * c + 1) in _B for c in CLUSTERS)
assert (16, 113 * 16 + 1) in _A and (1, 114) in _A  # the strided path with camera priors only: 1809 and 114 cameras


# ---- part 5: the checkers accept the restatement and reject planted faults ------------------------------------------------
U = {np.float64: 2.0 ** -53, np.float32: 2.0 ** -24}
DTYPES = [np.float64, np.float32]


@pytest.fixture(scope="module")
def terms():
    out = {}
    for name in P3_CASES:
        arrays, camera, pairs, _ = _P3[name]
        rng = np.random.default_rng(arrays.nc)
        D = rng.uniform(0.3, 3.0, 9 * arrays.nc)
        x = rng.uniform(-1, 1, 9 * arrays.nc)
        out[name] = (PriorTerms(arrays.cams, camera, pairs), D, x)
    return out


def _check_hx(t, D, x, dtype, **fault):
    want, My = t.hx(D, x)
    got = kernel_hx(t, D, x, dtype=dtype, **fault)
    check_bar(got, want, U[dtype] * (t.k() + C_LIN)[:, None] * My, "prior H x")


def _fault_sites(name, t):
    """(fault, camera) of every fault that applies at this case"""
    nc, sc = t.nc, side_counts(t.nc, t.pairs)
    ends = [min(c, nc - 1) for c in range(PER_THREAD - 1, nc + PER_THREAD - 1, PER_THREAD)]  # the last camera of every block
    out = [("neighbour", c) for c in sorted({nc - 2, 127, 128}) if c + 1 < nc]
    out += [("drop_block_last", [c]) for c in ends]
    cams = [HUB, HUB_33] if name == "hub" else []
    cams += [int(np.flatnonzero(sc == k)[0]) for k in (1, 2) if np.any(sc == k)]
    out += [(f, c) for f in ("side_dropped", "side_doubled", "O_on_vi") for c in cams]
    return out


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: np.dtype(d).name)
@pytest.mark.parametrize("name", P3_CASES)
def test_prior_hx_checker_accepts_the_restatement_and_rejects_faults(terms, name, dtype):
    t, D, x = terms[name]
    _check_hx(t, D, x, dtype)
    for fault, at in _fault_sites(name, t):
        with pytest.raises(AssertionError):
            _check_hx(t, D, x, dtype, fault=fault, at=at)


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: np.dtype(d).name)
@pytest.mark.parametrize("kind", ["camera", "pair", "landmark"])
def test_item_sum_checker_rejects_a_dropped_257th_item(kind, dtype):
    """the cost and l_diff items of one prior kind at every item count: accepted as the kernel sums them (Scalar items,
    double sums), rejected in float64 with item 257 dropped wherever there is one.  float32 cannot see that fault: each
    item carries the float32 rounding of its residual (a centre or translation difference of operands ~100 times larger),
    and the sum of those bars exceeds one item at most counts (0.006 .. 14 bars); the GPU item checks run in float64"""
    from test_gpu_prior_classes import _item_case
    for n in (pc.CAMERA_ITEM_COUNTS if kind == "camera" else pc.ITEM_COUNTS):
        arrays, feats = _item_case(kind, n)
        if kind == "landmark":  # cost only: a landmark prior's share of l_diff is summed per landmark in k_back_substitute
            sums = (("cost", landmark_cost_items(arrays.lms, *feats["landmarks"])),)
        else:
            t = PriorTerms(arrays.cams, feats.get("camera"), feats.get("pairs"))
            d = np.random.default_rng(n).uniform(-1, 1, 9 * arrays.nc) * 1e-2
            sums = (("cost", t.cost_items(kind)), ("l_diff", t.ldiff_items(kind, d)))
        for what, (items, mag) in sums:
            assert len(items) == n
            check_item_sum(kernel_item_sum(items, dtype=dtype), items, mag, U[dtype], what)
            if n > SUM_THREADS and dtype == np.float64:
                assert items[SUM_THREADS] != 0
                with pytest.raises(AssertionError):
                    check_item_sum(kernel_item_sum(items, "item_257_dropped", dtype=dtype), items, mag, U[dtype], what)


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: np.dtype(d).name)
def test_group_sum_checker_rejects_a_dropped_129th_member(dtype):
    g = group_layout()
    nc = len(g)
    d2 = np.random.default_rng(5).uniform(0.5, 2.0, (nc, 9)).astype(dtype).astype(np.float64)
    want = group_sum_model(d2, g)
    bar = U[dtype] * (group_k(g, nc) + 2)[:, None] * want
    check_bar(kernel_group_sum(d2, g, dtype=dtype), want, bar, "group diag2")
    for size in GROUP_SIZES:
        gid = _SIZES_ID[size]
        sel = g == gid
        got = kernel_group_sum(d2, np.where(sel, g, -1), "member_129_dropped", dtype)
        w = group_sum_model(d2, np.where(sel, g, -1))
        b = U[dtype] * (group_k(np.where(sel, g, -1), nc) + 2)[:, None] * w
        if size > GROUP_THREADS:
            with pytest.raises(AssertionError):
                check_bar(got, w, b, "group diag2")
        else:
            check_bar(got, w, b, "group diag2")



def test_replay_rejects_a_missing_camera_prior_term_on_the_strided_path():
    """k_pcg_vec without A^T A v on its strided path (more than 113 cameras per CTA): the operator the solve applies lacks
    the camera-prior term.  Iterate 1 of that solve against the replay of the right operator is off by far more than the bar
    10 k u kappa of the iterate tests, in float64 and float32"""
    c, nc = 1, 114
    assert not vec_partition(nc, c)["cached"]
    arrays = vec_problem(nc, False)
    t = PriorTerms(arrays.cams, pc.camera_prior(arrays.cams, seed=nc))
    n = 9 * nc
    rng = np.random.default_rng(1)
    G = rng.standard_normal((2 * n, n)) * (rng.uniform(size=(2 * n, n)) < 0.02)
    B, _ = t.blocks(np.ones(n))
    Hp = np.zeros((n, n))
    for k in range(nc):
        Hp[9 * k:9 * k + 9, 9 * k:9 * k + 9] = B[k]
    lam = 0.1
    H = G.T @ G + Hp + lam * np.eye(n)
    inv = np.stack([np.linalg.inv(H[9 * k:9 * k + 9, 9 * k:9 * k + 9]) for k in range(nc)])
    b = rng.standard_normal(n)
    good = pcg_replay(lambda v: H @ v, b, inv, eta=0.0, max_it=400)
    lmin, lmax = lanczos_condition(good["alphas"], good["betas"])
    bad = pcg_replay(lambda v: (H - Hp) @ v, b, inv, eta=-1e30, max_it=1)
    for dtype in DTYPES:
        bar = 10 * 1 * U[dtype] * lmax / lmin
        assert bar < 1e-2
        assert rel_err(bad["xs"][1], good["xs"][1]) > 10 * bar, dtype


# ---- the scaling, b and inverse-block checkers of the per-camera GPU test against a camera's prior terms misplaced ------------
def _misplace(v, fault, at):
    """v [nc, ...] of the prior part with camera `at`'s entry written to the next camera ("neighbour") or dropped
    ("drop_block_last")"""
    out = np.array(v, np.float64)
    if fault == "neighbour":
        out[at + 1] = v[at]
    out[at] = 0
    return out


@pytest.mark.parametrize("name", ["nc127", "nc128", "nc129", "nc257", "groups"])
def test_scaling_b_and_inverse_checkers_reject_a_misplaced_camera(terms, name):
    """the checkers of test_prior_terms_per_camera at their own bars, on a float64 restatement: the reprojection parts
    stand in random (diag2, b, SPD blocks with lam I), the prior parts from the models; accepted as they are, rejected with a
    camera's prior column norms, A^T r or prior block written to its neighbour, or dropped at the end of a 128-block"""
    import shared_intrinsics_model as sm
    from test_gpu_camera_classes import bar_constants
    arrays, camera, pairs, groups = _P3[name]
    t = PriorTerms(arrays.cams, camera, pairs) if name == "groups" else terms[name][0]
    nc, lam, eps = t.nc, 0.1, 1e-8
    rng = np.random.default_rng(nc)
    s = rng.uniform(0.3, 3.0, (nc, 9))
    d_rep = rng.uniform(0.5, 2.0, (nc, 9))
    s0 = 1 / (eps + np.sqrt(d_rep))
    b_rep = rng.uniform(-1, 1, (nc, 9))
    G = rng.standard_normal((nc, 12, 9))
    B_rep = np.einsum("cij,cik->cjk", G, G) + lam * np.eye(9)
    MB_rep = np.einsum("cij,cik->cjk", np.abs(G), np.abs(G)) + lam * np.eye(9)
    cb = bar_constants(arrays)[0] + 128
    d_pri, g_pri, B_pri = t.diag2()[0], t.g(s)[0], t.blocks(s)[0]
    gsum = (lambda v: group_sum_model(v, groups)) if groups is not None else (lambda v: v)
    lead = sm.leads(groups) if groups is not None else None
    contract = (lambda v: sm.contract(v, lead).reshape(nc, 9)) if groups is not None else (lambda v: v)
    cc = np.full(nc, 50.0)

    def run(dp, gp, Bp):
        Bd, _, free = pc.grouped_blocks(B_rep + Bp, MB_rep, lam, groups)
        inv = np.zeros((nc, 9, 9))
        for c in range(nc):
            f = free[c]
            inv[c][np.ix_(f, f)] = np.linalg.inv(Bd[c][np.ix_(f, f)])
        return [lambda: check_scaling(gsum(d_rep + dp), d_rep, s0, s, t, groups),
                lambda: check_b(contract(b_rep + gp), b_rep, np.abs(b_rep), cc, s, t, groups),
                lambda: check_inverse_blocks(inv, B_rep, MB_rep, cb, s, lam, t, groups, "inverse")]

    for check in run(d_pri, g_pri, B_pri):
        check()
    ends = [min(c, nc - 1) for c in range(PER_THREAD - 1, nc + PER_THREAD - 1, PER_THREAD)]
    sites = [("neighbour", c) for c in sorted({nc - 2, 127}) if c + 1 < nc] + [("drop_block_last", c) for c in ends]
    for fault, at in sites:
        for which, check in enumerate(run(_misplace(d_pri, fault, at), _misplace(g_pri, fault, at), _misplace(B_pri, fault, at))):
            with pytest.raises(AssertionError):
                check()
