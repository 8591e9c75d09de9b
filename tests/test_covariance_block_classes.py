"""CPU side of tests/test_gpu_covariance_block_classes.py: the launch geometry of the covariance-block kernels read from the
sources reaches both sides of every edge at the SM counts of the H100 SXM and PCIe (asserted at import), the problems and
requests of the GPU cases are what they claim to be, the model of the elimination instances equals the dense inverse, and
the float64 check of every GPU case rejects each planted fault of covariance_blocks_model.CLASS_FAULTS wherever it changes
a block, at that case's own bars."""
import numpy as np
import pytest

import camera_model as cm
import covariance_block_classes as cbc
import covariance_blocks_model as cbm
import covariance_model as cvm


def _adjacent(counts, kind, sms, f, a, b):
    """some count m and m + 1 both in counts with f(m) == a and f(m + 1) == b"""
    return any(m + 1 in counts and f(kind, m, sms) == a and f(kind, m + 1, sms) == b for m in counts)


for _name, _sms in cbc.SM_COUNTS.items():
    _cap = cbc.CAP_PER_SM * _sms
    for _kind, (_w, _per) in cbc.LAUNCH.items():
        _c = cbc.edge_counts(_kind, _sms)
        assert _c[0] == 1, (_name, _kind)
        assert _adjacent(_c, _kind, _sms, cbc.grid, 1, 2), (_name, _kind, "one CTA / two")
        assert _adjacent(_c, _kind, _sms, cbc.grid, _cap - 1, _cap), (_name, _kind, "below the CTA cap / at it")
        assert _adjacent(_c, _kind, _sms, cbc.sweeps, 1, 2), (_name, _kind, "one sweep / two")
        assert {cbc.sweeps(_kind, m, _sms) for m in _c} == {1, 2, 3}, (_name, _kind)
        if _w == 1:  # a full CTA and a full first sweep: every thread or warp of the grid has exactly one request
            assert _per in _c and cbc.stride_items(_kind, _sms) in _c, (_name, _kind)
        else:  # camera pairs: a request across two CTAs, and across two sweeps (81 does not divide the stride)
            assert any((_w * k) // _per != (_w * k + _w - 1) // _per for m in _c for k in range(min(m, 8))), _name
            assert all(len(cbc.straddles(_kind, m, _sms)) == cbc.sweeps(_kind, m, _sms) - 1 for m in _c), _name
            assert all(set(cbc.straddles(_kind, m, _sms).tolist()) <= set(cbc.edge_requests(_kind, m, _sms).tolist()) for m in _c)
assert cbc.COV_REL_THREADS in cbc.edge_counts("relative", 132)  # a CTA whose 64 threads all use their column of As
# the slot loops: 32 (one pass) and 33 (two), up to 300 (ten) slots; slot pairs up to 90 000
assert {cbc.SLOT_PASS, cbc.SLOT_PASS + 1} <= set(cbc.LONG) and max(cbc.LONG) > 9 * cbc.SLOT_PASS


def test_long_case_reaches_both_sides_of_the_slot_loops():
    prob, _, mask = cbc.long_case()
    req = cbc.long_requests(prob)
    n = np.diff(prob.lm_off)
    lq = req["landmarks"]
    nl_, nm_ = n[lq[:, 0]], n[lq[:, 1]]
    pairs = nl_ * nm_
    assert (pairs <= cbc.SLOT_PASS).any() and (pairs > cbc.SLOT_PASS).any() and pairs.max() == 300 * 300
    unequal = (nl_ != nm_) & (nl_ > cbc.SLOT_PASS) & (nm_ > cbc.SLOT_PASS)
    assert unequal.sum() == 6 * 5  # every ordered pair of the 6 landmarks above 32 (33, 63, 64, 65, 150, 300)
    assert ((nl_ > cbc.SLOT_PASS) & (nm_ <= 6)).any() and ((nl_ <= 6) & (nm_ > cbc.SLOT_PASS)).any()
    cl = req["camera_landmark"]
    passes = -(-n[cl[:, 1]] // cbc.SLOT_PASS)
    assert set(passes.tolist()) >= {1, 2, 3, 5, 10}
    straddle = set(cvm.straddling_cameras(cbc.LONG_NC))
    for l in range(len(cbc.LONG)):
        cams = cl[cl[:, 1] == l, 0]
        track = set(prob.obs_cam[prob.lm_off[l]:prob.lm_off[l + 1]].tolist())
        assert set(cbc.LONG_HELD) <= set(cams.tolist()) and any(c not in track for c in cams)
        assert any(c in straddle for c in cams)
    assert (mask[list(cbc.LONG_HELD)] != 0).all()


def test_rank_case_classes_in_every_instance():
    prob, absp, W, lmp, classes = cbc.rank_case()
    n = np.diff(prob.lm_off)
    off = np.asarray(prob.lm_off)
    rank1 = np.linalg.matrix_rank(W) == 1
    zero = ~W.reshape(-1, 4).any(1)
    lm_of = np.repeat(np.arange(len(n)), n)
    special = set(classes["prior"] + classes["r2"])
    alone = np.array([l not in special for l in lm_of])
    for sel in (rank1 & alone, zero & alone):  # on long and short tracks of full-rank landmarks
        assert (n[lm_of[sel]] > cbc.SLOT_PASS).any() and (n[lm_of[sel]] <= 6).any()
    assert n[classes["prior"]].max() > cbc.SLOT_PASS and n[classes["r2"]].max() > cbc.SLOT_PASS
    assert set(classes["prior"]) <= set(lmp[0].tolist()) and not set(classes["r2"]) & set(lmp[0].tolist())
    want = {"plain": (3, 3), "lmp": (3, 3), "obsw": (2, 2), "lmp_obsw": (3, 2)}  # ranks of the classes prior, r2
    for name, (rp, r2) in want.items():
        kw = cbc.instance_inputs(name, W, lmp)
        ref = cbc.model(prob, absp=absp, threshold=cbc.huber_threshold(prob, kw["W"]), **kw)
        assert (ref["rank"][classes["prior"]] == rp).all() and (ref["rank"][classes["r2"]] == r2).all(), name
        assert (ref["rank"][classes["r3"]] == 3).all()
    assert off[-1] == len(prob.obs_cam)


@pytest.mark.parametrize("instance", list(cbc.INSTANCES))
def test_instance_model_equals_the_dense_inverse(instance):
    """the model the GPU cases use (elimination with lm_info, whitened rows, Huber weights) equals the blocks of the full
    inverse of the stacked dense rows on the 7-camera version"""
    prob, absp, W, lmp, _ = cbc.rank_case(**cbc.SMALL_RANK)
    kw = cbc.instance_inputs(instance, W, lmp)
    th = cbc.huber_threshold(prob, kw["W"])
    req = cbm.random_requests(np.random.default_rng(3), 7, len(prob.lm_off) - 1, 60)
    ref = cbc.model(prob, absp=absp, threshold=th, **kw)
    assert (ref["rank"] == 3).all()
    cbc.dense_check(cbm.blocks(ref, **req), prob, np.float64, absp, th, req, **kw)
    F, _, _ = cbm.full_covariance(*cbc.dense_total(prob, np.float64, absp, threshold=th, **kw))
    want = cbm.dense_blocks(F, 7, np.asarray(prob.cams, np.float64), **req)
    got = cbm.blocks(ref, **req)
    for key in want:
        assert np.abs(got[key] - want[key]).max() <= 1e-9 * np.abs(want[key]).max(), key


def test_group_and_relative_cases():
    prob, _, group, lead, mask, held = cbc.group_case()
    assert sorted(np.bincount(group[group >= 0]).tolist()) == sorted(cbc.GROUP_SIZES)
    runs = np.flatnonzero(np.diff((group >= 0).astype(int)))  # members and non-members alternate along the cameras
    assert len(runs) >= 20
    assert lead[7] not in (-1, 7) and lead[held] not in (-1, held) and mask[held] != 0
    assert np.array_equal(prob.cams[lead >= 0, 7:], prob.cams[lead[lead >= 0], 7:])
    prob, absp, pair, mask, pairs = cbc.relative_case()
    req = cbc.relative_requests(prob, pairs)
    cams = np.asarray(prob.cams, np.float64)
    angles = []
    for e, o in pairs:
        M = cm.rotation(cams[e, :4]) @ cm.rotation(cams[o, :4]).T
        angles.append(np.arccos(np.clip((np.trace(M) - 1) / 2, -1, 1)))
        assert abs(np.linalg.norm(cams[e, 4:7]) - cbc.REL_T) < 1e-9
    assert np.allclose(angles, np.repeat(cbc.REL_ANGLES, 2), atol=1e-7)
    w = cams[pairs[:, 0], 3]
    assert (w < 0).sum() >= 3 and (w > 0).sum() >= 3
    rel = {tuple(r) for r in req["relative"].tolist()}
    assert all((int(a), int(b)) in rel and (int(b), int(a)) in rel for a, b in pairs)
    assert any(7 in r for r in rel) and 7 in cvm.straddling_cameras(len(cams))
    assert any(mask[a] or mask[b] for a, b in rel)


def _cases():
    """(name, ref, requests, faults that must apply) of every GPU case, float64"""
    prob, absp, mask = cbc.long_case()
    yield "long", cbc.model(prob, absp=absp, mask=mask), cbc.long_requests(prob), {"slot_pair_order", "first_pass_only", "w_swapped"}
    prob, absp, W, lmp, classes = cbc.rank_case()
    req = cbc.rank_requests(prob, classes)
    yield "rank classes", cbc.model(prob, absp=absp, lm_prior=lmp, W=W), req, \
        {"slot_pair_order", "first_pass_only", "w_swapped", "lm_prior_dropped"}
    for name in cbc.INSTANCES:
        kw = cbc.instance_inputs(name, W, lmp)
        th = cbc.huber_threshold(prob, kw["W"])
        yield name, cbc.model(prob, absp=absp, threshold=th, **kw), req, \
            {"w_swapped"} | ({"lm_prior_dropped"} if kw["lm_prior"] is not None else set())
    prob, absp = cbc.edge_case()
    ref = cbc.model(prob, absp=absp)
    for gpu, sms in cbc.SM_COUNTS.items():
        master = cbc.edge_master(prob, sms)
        idx = {k: sorted(set().union(*(cbc.edge_requests(k, m, sms).tolist() for m in cbc.edge_counts(k, sms))))
               for k in cbc.LAUNCH}
        yield f"edges {gpu}", ref, {k: master[k][v] for k, v in idx.items()}, {"w_swapped"}
    prob, absp, group, lead, mask, held = cbc.group_case()
    yield "groups", cbc.model(prob, absp=absp, mask=mask, lead=lead), cbc.group_requests(prob, group, lead, held), \
        {"member_not_expanded"}
    prob, absp, pair, mask, pairs = cbc.relative_case()
    yield "relative", cbc.model(prob, absp=absp, pair=pair, mask=mask), cbc.relative_requests(prob, pairs), set()


def test_class_faults_are_rejected_in_every_case():
    seen = set()
    for name, ref, req, must in _cases():
        cbc.check(cbm.blocks(ref, **req), ref, req, name)  # the unfaulted blocks pass at this case's bars
        for fault in cbm.CLASS_FAULTS:
            r = cbc.fault_rejected(ref, req, fault)
            assert r is not False, f"{name}: {fault} changes the blocks but passes the check"
            assert r or fault not in must, f"{name}: {fault} does not change any block"
            if r:
                seen.add(fault)
    assert seen == set(cbm.CLASS_FAULTS)
