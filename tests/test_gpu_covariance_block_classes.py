"""The covariance-block kernels (rba_compute_covariance_blocks, DESIGN.md section 20) request by request at the edges of
their launches (tests/covariance_block_classes.py): landmark pairs and camera-landmark requests on tracks longer than a warp
and of unequal lengths, landmarks whose rank comes from their prior or is 2, every instance of the elimination with Huber
weights active, every grid-stride edge at the device's SM count, intrinsics groups of 2, 65 and 129 members, and relative
poses at rotations up to pi, both quaternion signs and translations of 1e3.

Every block is compared componentwise with the float64 model at the handle's stored state (covariance_blocks_model.check:
8 (N kappa + n_l kappa_l) u of the entrywise bound, each bar asserted <= 1e-4 and printed on failure); the identities that
hold exactly are asserted bit for bit."""
import numpy as np
import pytest

import covariance_block_classes as cbc
import covariance_blocks_model as cbm
import covariance_model as cvm

pytestmark = pytest.mark.gpu

DTYPES = pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _held_rows_zero(got, req, mask, nc):
    fixed = cvm.fixed_mask(mask, nc).reshape(nc, 9)
    for k, (a, b) in enumerate(req["cameras"]):
        assert (got["cameras"][k][fixed[a], :] == 0).all() and (got["cameras"][k][:, fixed[b]] == 0).all(), (a, b)
    for k, (c, _) in enumerate(req["camera_landmark"]):
        assert (got["camera_landmark"][k][fixed[c], :] == 0).all(), c


@DTYPES
def test_long_and_unequal_tracks(dtype):
    """landmark pairs of tracks 2 .. 300 in both orders (up to 90 000 slot pairs, n_l != n_m both above a warp), camera-
    landmark requests whose slot loop takes up to 10 passes, with cameras at the start, middle and end of the track, outside
    it, held and across a tile"""
    prob, absp, mask = cbc.long_case()
    req = cbc.long_requests(prob)
    lin = cbc.handle(prob, dtype, absp=absp, mask=mask)
    got = lin.covariance_blocks(**req, marginals=True)
    lin.close()
    lq = req["landmarks"]
    same = lq[:, 0] == lq[:, 1]
    assert same.sum() == len(cbc.LONG)
    assert np.array_equal(got["landmarks"][same], got["lm"][lq[same, 0]])  # k_cov_lm_cross<false> (l, l) = <true>
    _held_rows_zero(got, req, mask, len(prob.cams))
    cbc.check(got, cbc.model(prob, dtype, absp=absp, mask=mask), req, f"long tracks {np.dtype(dtype).name}")


@DTYPES
def test_rank_classes_in_cross_requests(dtype):
    """landmark priors and observation information on one handle (k_cov_landmark<S, true, true>): landmarks of full rank,
    of rank 3 only through their prior (one observation left) and of rank 2, each in both positions of a landmark pair with
    short and long partners and in camera-landmark requests; NaN exactly where the model has it"""
    prob, absp, W, lmp, classes = cbc.rank_case()
    req = cbc.rank_requests(prob, classes)
    lin = cbc.handle(prob, dtype, absp=absp, lm_prior=lmp, W=W)
    got = lin.covariance_blocks(**req)
    lin.close()
    ref = cbc.model(prob, dtype, absp=absp, lm_prior=lmp, W=W)
    assert (ref["rank"][classes["prior"]] == 3).all() and (ref["rank"][classes["r2"]] == 2).all()
    r2 = np.asarray(classes["r2"])
    bad_cl = np.isin(req["camera_landmark"][:, 1], r2)
    bad_lm = np.isin(req["landmarks"], r2).any(1)
    assert bad_cl.any() and (~bad_cl).any() and bad_lm.any()
    assert np.isnan(got["camera_landmark"][bad_cl]).all() and np.isfinite(got["camera_landmark"][~bad_cl]).all()
    assert np.isnan(got["landmarks"][bad_lm]).all() and np.isfinite(got["landmarks"][~bad_lm]).all()
    cbc.check(got, ref, req, f"rank classes {np.dtype(dtype).name}")


@DTYPES
@pytest.mark.parametrize("instance", list(cbc.INSTANCES))
def test_every_elimination_instance(instance, dtype):
    """the dispatch of cov_factor_inverse: plain -> k_cov_landmark<S>, lmp -> <S, true> (landmark priors), obsw ->
    <S, false, true> (observation information), lmp_obsw -> <S, true, true>; each with the Huber weight active on about half
    the observations, W of rank 1 and 0 on long and short tracks"""
    prob, absp, W, lmp, classes = cbc.rank_case()
    kw = cbc.instance_inputs(instance, W, lmp)
    th = cbc.huber_threshold(prob, kw["W"])
    req = cbc.rank_requests(prob, classes)
    lin = cbc.handle(prob, dtype, absp=absp, threshold=th, **kw)
    got = lin.covariance_blocks(**req)
    lin.close()
    cbc.check(got, cbc.model(prob, dtype, absp=absp, threshold=th, **kw), req, f"{instance} {np.dtype(dtype).name}")


@DTYPES
@pytest.mark.parametrize("instance", list(cbc.INSTANCES))
def test_every_elimination_instance_against_the_dense_inverse(instance, dtype):
    """7 cameras: every kind against the full inverse of the stacked dense rows (reprojection, camera priors, landmark
    priors), 8 N kappa u of the largest entry of each kind"""
    prob, absp, W, lmp, _ = cbc.rank_case(**cbc.SMALL_RANK)
    kw = cbc.instance_inputs(instance, W, lmp)
    th = cbc.huber_threshold(prob, kw["W"])
    req = cbm.random_requests(np.random.default_rng(3), 7, len(prob.lm_off) - 1, 60)
    lin = cbc.handle(prob, dtype, absp=absp, threshold=th, **kw)
    got = lin.covariance_blocks(**req)
    lin.close()
    cbc.dense_check(got, prob, dtype, absp, th, req, **kw)


def test_grid_stride_edges():
    """per kind the request counts at every edge of the launch at this device's SM count (1, per CTA -1 / 0 / +1, the CTA
    cap, the stride -1 / 0 / +1, 2 stride + 1), all four kinds in one call per count, prefixes of one request list: every
    count gives the same blocks for its prefix, a permuted list the permuted blocks, and every request next to an edge the
    block it gets alone, all bit for bit; those requests against the model"""
    sms = _sm_count()
    prob, absp = cbc.edge_case()
    master = cbc.edge_master(prob, sms)
    counts = {k: cbc.edge_counts(k, sms) for k in cbc.LAUNCH}
    ncall = len(counts["cameras"])
    assert all(len(c) == ncall for c in counts.values())
    rng = np.random.default_rng(7)
    lin = cbc.handle(prob, np.float64, absp=absp)
    full = None
    edges = {k: set() for k in cbc.LAUNCH}
    for i in reversed(range(ncall)):
        req = {k: master[k][:counts[k][i]] for k in cbc.LAUNCH}
        got = lin.covariance_blocks(**req)
        if full is None:
            full = got
        for k in cbc.LAUNCH:
            m = counts[k][i]
            assert np.array_equal(got[k], full[k][:m]), (k, m)
            edges[k] |= set(cbc.edge_requests(k, m, sms).tolist())
        perm = {k: rng.permutation(counts[k][i]) for k in cbc.LAUNCH}
        gp = lin.covariance_blocks(**{k: req[k][perm[k]] for k in cbc.LAUNCH})
        for k in cbc.LAUNCH:
            assert np.array_equal(gp[k], got[k][perm[k]]), (k, counts[k][i])
    edges = {k: np.array(sorted(v)) for k, v in edges.items()}
    for j in range(max(len(v) for v in edges.values())):
        one = {k: master[k][v[j]][None] for k, v in edges.items() if j < len(v)}
        alone = lin.covariance_blocks(**one)
        for k in one:
            assert np.array_equal(alone[k][0], full[k][edges[k][j]]), (k, edges[k][j])
    lin.close()
    req = {k: master[k][v] for k, v in edges.items()}
    cbc.check({k: full[k][v] for k, v in edges.items()}, cbc.model(prob, np.float64, absp=absp), req, f"grid edges ({sms} SMs)")


def test_intrinsics_groups_in_the_blocks():
    """groups of 2, 65 and 129 members among non-members, a member across a tile, a member's pose held: two members' camera
    block [6:, 6:] is the lead's marginal [6:, 6:] and a member's camera-landmark rows 6..8 are the lead's, bit for bit (the
    members' rows of the inverse and their equilibration are copies of the lead's); every block against the model"""
    prob, absp, group, lead, mask, held = cbc.group_case()
    req = cbc.group_requests(prob, group, lead, held)
    lin = cbc.handle(prob, np.float64, absp=absp, mask=mask, group=group)
    got = lin.covariance_blocks(**req, marginals=True)
    lin.close()
    n = 0
    for k, (a, b) in enumerate(req["cameras"]):
        if group[a] >= 0 and group[a] == group[b]:
            assert np.array_equal(got["cameras"][k][6:, 6:], got["cam"][lead[a]][6:, 6:]), (a, b)
            n += 1
    assert n >= 3 * 9
    cl = req["camera_landmark"]
    where = {(int(c), int(l)): k for k, (c, l) in enumerate(cl)}
    m = 0
    for k, (c, l) in enumerate(cl):
        if lead[c] >= 0 and lead[c] != c and (int(lead[c]), int(l)) in where:
            assert np.array_equal(got["camera_landmark"][k][6:], got["camera_landmark"][where[int(lead[c]), int(l)]][6:]), (c, l)
            m += 1
    assert m >= 20
    _held_rows_zero(got, req, mask, len(prob.cams))
    cbc.check(got, cbc.model(prob, np.float64, absp=absp, mask=mask, lead=lead), req, "intrinsics groups")


@DTYPES
def test_relative_poses(dtype):
    """relative rotations 0, pi/2, pi - 1e-3 and pi, both signs of the stored quaternion, translations of 1e3, every pair in
    both orders, a held pose on one side, a camera across a tile: exactly symmetric, and against the model"""
    prob, absp, pair, mask, pairs = cbc.relative_case()
    req = cbc.relative_requests(prob, pairs)
    lin = cbc.handle(prob, dtype, absp=absp, pair=pair, mask=mask)
    got = lin.covariance_blocks(**req)
    lin.close()
    rel = got["relative"]
    assert np.array_equal(rel, rel.transpose(0, 2, 1))
    assert np.isfinite(rel).all()
    cbc.check(got, cbc.model(prob, dtype, absp=absp, pair=pair, mask=mask), req, f"relative poses {np.dtype(dtype).name}")
