"""Shared by tests/test_covariance_block_classes.py (CPU) and tests/test_gpu_covariance_block_classes.py: the launch geometry
of the covariance-block kernels (rba_compute_covariance_blocks, DESIGN.md section 20) read from the sources, the problems and
requests that sit on both sides of every boundary of it, and the float64 model of a handle's blocks at its stored state
(covariance_blocks_model.reference with the priors, observation information, held entries and intrinsics groups of the
handle).  Not collected by pytest.

Boundaries (rootba_b200/csrc/covariance.cuh section 5, solver.cu Solver::cov_compute):
  grid          every extraction kernel runs a grid-stride loop over its items on min(ceil(items / per CTA), 16 sm_count) CTAs:
                k_cov_cam_cross  a thread per entry, 81 entries per request, 256 per CTA (a request can straddle two CTAs
                                 or two sweeps);
                k_cov_cam_lm, k_cov_lm_cross<false>  a warp per request, 4 per CTA;
                k_cov_rel_pose   a thread per request, COV_REL_THREADS per CTA, its A in As[72][COV_REL_THREADS] by thread
  slot loops    k_cov_cam_lm: lanes over the n_l slots of the landmark, 32 at a time; cov_lm_block: lanes over the n_l n_m
                slot pairs, 32 at a time, pair t = (t / n_m, t % n_m)
  elimination   k_cov_landmark<S, LMP, OBSW>: four instances, chosen by cov_factor_inverse from the landmark priors (LMP) and
                the observation information (OBSW)
  tiles         the 64 tile of the dense inverse (covariance_model.TILE): a camera's 9 rows can straddle two tiles
"""
import os
import re

import numpy as np

import camera_model as cm
import camera_prior_model as pm
import covariance_blocks_model as cbm
import covariance_model as cvm
import observation_info_model as om
import pair_prior_model as qm
import shared_intrinsics_model as sim
from conftest import ROOT


def _source(name):
    with open(os.path.join(ROOT, "rootba_b200", "csrc", name)) as f:
        return f.read()


_SOLVER, _COV = _source("solver.cu"), _source("covariance.cuh")
COV_REL_THREADS = int(re.search(r"constexpr int COV_REL_THREADS = (\d+);", _COV).group(1))
CAP_PER_SM = int(re.search(r"\(items \+ per_block - 1\) / per_block, \(long long\)sm_count \* (\d+)\)", _SOLVER).group(1))
CAM_CROSS_THREADS = int(re.search(r"k_cov_cam_cross<<<grid\(81LL \* m, (\d+)\), \1,", _SOLVER).group(1))
_lm = re.search(r"k_cov_lm_cross<true>\)<<<grid\(m, (\d+)\), (\d+),", _SOLVER)
_clm = re.search(r"k_cov_cam_lm<<<grid\(kinds\[1\]\.m, (\d+)\), (\d+),", _SOLVER)
WARPS_PER_CTA = int(_lm.group(1))
assert int(_lm.group(2)) == int(_clm.group(2)) == 32 * WARPS_PER_CTA and int(_clm.group(1)) == WARPS_PER_CTA
assert re.search(r"k_cov_rel_pose<S><<<grid\(kinds\[3\]\.m, COV_REL_THREADS\), COV_REL_THREADS,", _SOLVER)
assert "__shared__ double As[72][COV_REL_THREADS];" in _COV and "As[12 * r + q][tid]" in _COV
assert f"__launch_bounds__({CAM_CROSS_THREADS}) k_cov_cam_cross" in _COV
assert "for (int i = lane; i < n; i += 32)" in _COV and "for (int t = lane; t < n * nm; t += 32)" in _COV
assert "const int a = t / nm, b = t % nm;" in _COV
assert (CAM_CROSS_THREADS, WARPS_PER_CTA, COV_REL_THREADS, CAP_PER_SM) == (256, 4, 64, 16)
SLOT_PASS = 32
# the dispatch of cov_factor_inverse: <LMP, OBSW> by (landmark priors set, observation information set)
assert re.search(r"auto kcov = n_lmp > 0 \? \(D\.obs_W \? k_cov_landmark<S, true, true> : k_cov_landmark<S, true>\)\s*"
                 r": \(D\.obs_W \? k_cov_landmark<S, false, true> : k_cov_landmark<S>\);", _SOLVER)

SM_COUNTS = {"H100 SXM": 132, "H100 PCIe": 114}

# per kind (items per request, items per CTA)
LAUNCH = {"cameras": (81, CAM_CROSS_THREADS), "camera_landmark": (1, WARPS_PER_CTA), "landmarks": (1, WARPS_PER_CTA),
          "relative": (1, COV_REL_THREADS)}


def grid(kind, m, sms):
    w, per = LAUNCH[kind]
    return max(1, min(-(-w * m // per), CAP_PER_SM * sms))


def sweeps(kind, m, sms):
    """passes of the grid-stride loop that run at least one item"""
    w, per = LAUNCH[kind]
    return -(-w * m // (grid(kind, m, sms) * per))


def stride_items(kind, sms):
    return LAUNCH[kind][1] * CAP_PER_SM * sms


def edge_counts(kind, sms):
    """request counts of one kind at every edge of its launch: 1; one CTA full and one more (per CTA -1, 0, +1); the last
    count below the CTA cap and the first at it; the last count of one sweep -1, 0, +1 (the stride); the first of a third
    sweep (2 stride + 1)"""
    w, per = LAUNCH[kind]
    T = stride_items(kind, sms)
    one, below, full = per // w, per * (CAP_PER_SM * sms - 1) // w, T // w
    return sorted({1, max(1, one - 1), one, one + 1, below, below + 1, full - 1, full, full + 1, 2 * T // w + 1})


def straddles(kind, m, sms):
    """request indices whose items lie in two sweeps"""
    w, per = LAUNCH[kind]
    g = grid(kind, m, sms) * per
    k = np.arange(m)
    return k[(w * k) // g != (w * k + w - 1) // g]


def edge_requests(kind, m, sms):
    """indices of the requests next to every edge of the launch of m requests: the first two and the last two, those at the
    start and end of every CTA of the first sweep's first and last two, and of every sweep"""
    w, per = LAUNCH[kind]
    g = grid(kind, m, sms)
    edges = {0, w * m}
    edges |= {per * c for c in (1, 2, g - 1, g) if 0 < per * c < w * m}
    edges |= {g * per * s for s in range(1, sweeps(kind, m, sms))}
    out = set()
    for e in edges:
        for item in (e - 2, e - 1, e, e + 1):
            if 0 <= item < w * m:
                out.add(item // w)
    return np.array(sorted(out))


# ---- the model of a handle ------------------------------------------------------------------------------------------
def stored(a, dtype):
    """an input array as a handle of `dtype` holds it, in float64"""
    return np.asarray(np.asarray(a, dtype), np.float64)


def model(prob, dtype=np.float64, absp=None, pair=None, lm_prior=None, W=None, threshold=None, mask=None, lead=None):
    """covariance_blocks_model.reference of a handle of `dtype` on `prob` at its stored state: the reprojection rows
    (whitened by W when given, Huber weight at `threshold`), the camera and pair priors' A^T A in H_extra, the landmark priors'
    L^T L in lm_info, the held entries of `mask`, the intrinsics groups `lead`; rotations as the kernels build them"""
    sprob, sabsp, spair = cvm.as_stored(prob, dtype, absp, pair)
    cams = np.asarray(sprob.cams, np.float64)
    nc, nl = len(cams), len(sprob.lm_off) - 1
    if W is None:
        jp, jl, _, _ = cm.weighted(sprob, dtype=dtype, threshold=threshold, device_rot=True)
    else:
        w = om.whitened(sprob, stored(W, dtype), dtype=dtype, threshold=threshold, device_rot=True)
        jp, jl = w["Jp"], w["Jl"]
    H = np.zeros((9 * nc, 9 * nc))
    if sabsp is not None:
        A, _ = pm.rows(cams, *sabsp, device_rot=True)
        for c in range(nc):
            H[9 * c:9 * c + 9, 9 * c:9 * c + 9] += A[c].T @ A[c]
    if spair is not None:
        Jq, _ = qm.rows(cams, *spair, device_rot=True)
        H += Jq.T @ Jq
    lm_info = None
    if lm_prior is not None:
        L = stored(lm_prior[2], dtype)
        lm_info = np.zeros((nl, 3, 3))
        lm_info[np.asarray(lm_prior[0])] = np.einsum("mki,mkj->mij", L, L)
    fixed = None if mask is None else cvm.fixed_mask(mask, nc)
    return cbm.reference(jp, jl, sprob.obs_cam, sprob.lm_off, cams, H, lm_info, fixed, lead)


def handle(prob, dtype, absp=None, pair=None, lm_prior=None, W=None, threshold=None, mask=None, group=None):
    import rootba_b200 as rb
    from rootba_b200.linearizor import ResidualOptions
    bp = rb.BalProblem.from_arrays(prob, dtype)
    if absp is not None:
        bp.camera_prior = absp
    if pair is not None:
        bp.camera_pair_prior = pair
    if lm_prior is not None:
        bp.landmark_prior = lm_prior
    if W is not None:
        bp.observation_sqrt_info = W
    if mask is not None:
        bp.camera_fixed = mask
    if group is not None:
        bp.intrinsics_group = group
    kw = {} if threshold is None else dict(residual=ResidualOptions("HUBER", threshold))
    return rb.LinearizorQR.create(bp, rb.SolverOptions(use_double=dtype == np.float64, **kw))


def check(got, ref, req, what):
    """every requested kind componentwise against the model (bars <= 1e-4, printed on failure)"""
    req = {k: v for k, v in req.items() if v is not None and len(v)}
    cbm.check({k: got[k] for k in req}, cbm.blocks(ref, **req), ref, req, what=what)


def fault_rejected(ref, req, fault):
    """None when the fault leaves the blocks of these requests unchanged (it does not apply), else whether check rejects it"""
    if (fault == "lm_prior_dropped" and ref["inputs"]["lm_info"] is None) or (fault == "member_not_expanded" and ref["lead"] is None):
        return None
    req = {k: v for k, v in req.items() if v is not None and len(v)}
    good, bad = cbm.blocks(ref, **req), cbm.blocks(ref, **req, fault=fault)
    if all(np.array_equal(good[k], bad[k], equal_nan=True) for k in good):
        return None
    try:
        cbm.check(bad, good, ref, req, what=fault)
    except AssertionError:
        return True
    return False


# ---- A. long and unequal tracks -------------------------------------------------------------------------------------
LONG = [2, 3, 31, 32, 33, 63, 64, 65, 150, 300]
LONG_NC = 320
LONG_HELD = {5: 0x01, 211: 0x0F}  # camera -> RBA_FIX_* (FIX_POSE; everything)


def long_case():
    """the problem of test_gpu_covariance_shapes.test_long_tracks: landmarks 0..9 on LONG named cameras, 3000 short ones,
    centre priors; two held cameras"""
    from rootba_b200.synthetic import synth_bal
    import rootba_b200 as rb
    rng = np.random.default_rng(17)
    tracks = [rng.choice(LONG_NC, n, replace=False) for n in LONG]
    tracks += [rng.choice(LONG_NC, int(rng.integers(2, 7)), replace=False) for _ in range(3000)]
    prob = synth_bal(LONG_NC, len(tracks), 0.0, seed=18, tracks=tracks, lm_spread=0.5)
    assert np.array_equal(np.diff(prob.lm_off)[:len(LONG)], LONG)
    mask = np.zeros(LONG_NC, np.uint8)
    for c, f in LONG_HELD.items():
        mask[c] = f
    assert LONG_HELD[5] == rb.FIX_POSE and LONG_HELD[211] == rb.FIX_ALL
    return prob, cvm.centre_priors(prob, 19), mask


def long_requests(prob):
    """every ordered pair of the long landmarks; each with three short partners in both orders; camera-landmark requests of
    each long landmark with the first, a middle and the last camera of its track, a camera outside it, both held cameras and
    a camera whose rows straddle a 64 tile (one of its track when it has one)"""
    rng = np.random.default_rng(20)
    nl, nlong = len(prob.lm_off) - 1, len(LONG)
    lm = [[l, m] for l in range(nlong) for m in range(nlong)]
    for l in range(nlong):
        for s in rng.choice(np.arange(nlong, nl), 3, replace=False):
            lm += [[l, int(s)], [int(s), l]]
    straddle = np.array(cvm.straddling_cameras(LONG_NC))
    cl = []
    for l in range(nlong):
        track = np.asarray(prob.obs_cam[prob.lm_off[l]:prob.lm_off[l + 1]])
        outside = np.setdiff1d(np.arange(LONG_NC), track)
        inside = np.intersect1d(straddle, track)
        st = inside[0] if len(inside) else straddle[l % len(straddle)]
        for c in (track[0], track[len(track) // 2], track[-1], outside[len(outside) // 2], *LONG_HELD, st):
            cl.append([int(c), l])
    cams = rng.integers(0, LONG_NC, (40, 2))
    cams[:2] = [[5, 211], [211, 7]]
    rel = np.array([[5, 9], [9, 211], [7, 300], [13, 14]])
    return dict(cameras=cams, camera_landmark=np.array(cl), landmarks=np.array(lm), relative=rel)


# ---- B, C. rank classes and the elimination instances ------------------------------------------------------------------
RANK_NC = 96
RANK_LONG = [33, 40, 64, 70]


def rank_case(nc=RANK_NC, long=RANK_LONG, nshort=700, seed=31, switch_off=True):
    """nc cameras with centre priors; landmarks 0.. on the `long` tracks, then short ones.  Returns (prob, absp, W, lm_prior,
    classes): W random with some observations rank 1 and some 0 on long and short tracks; classes: 'r3' (full rank from its
    observations), 'prior' (every observation but the first switched off, a dense landmark prior: rank 3 only through it),
    'r2' (every observation but the first switched off, no prior).  The landmark priors: the 'prior' class and every 5th
    landmark.  switch_off=False: no 'prior' and 'r2' classes (every landmark has full rank in every instance)."""
    from rootba_b200.synthetic import synth_bal
    import landmark_prior_model as lp
    rng = np.random.default_rng(seed)
    tracks = [rng.choice(nc, n, replace=False) for n in long]
    tracks += [rng.choice(nc, int(rng.integers(2, 7)), replace=False) for _ in range(nshort)]
    prob = synth_bal(nc, len(tracks), 0.0, seed=seed + 1, tracks=tracks, lm_spread=0.5)
    absp = cvm.centre_priors(prob, seed + 2)
    nl, off = len(tracks), np.asarray(prob.lm_off)
    n = np.diff(off)
    W = om.random_info(len(prob.obs_cam), seed + 3)
    nlong = len(long)
    short = np.arange(nlong, nl)
    classes = {"prior": [1] + [int(l) for l in short[n[short] >= 3][:6]],
               "r2": [0] + [int(l) for l in short[n[short] >= 3][6:12]]} if switch_off else {"prior": [], "r2": []}
    for l in classes["prior"] + classes["r2"]:
        W[off[l] + 1:off[l + 1]] = 0.0
    special = set(classes["prior"] + classes["r2"])
    classes["r3"] = [l for l in range(nl) if l not in special][:12]
    # rank-1 and zero W on single observations of full-rank landmarks (tracks >= 4 keep >= 2 full observations)
    for k, l in enumerate(l for l in range(nl) if l not in special and n[l] >= 4):
        u, v = rng.standard_normal(2), rng.standard_normal(2)
        if k % 3 == 0:
            W[off[l] + 1] = np.outer(u, v)
        elif k % 3 == 1:
            W[off[l + 1] - 1] = 0.0
    idx = np.array(sorted(set(classes["prior"]) | set(range(0, nl, 5)) - set(classes["r2"])), np.int32)
    mean = np.asarray(prob.lms, np.float64)[idx] + rng.normal(0, 0.05, (len(idx), 3))
    L = np.stack([lp.sqrt_info_kind("dense" if i % 4 else "height", rng) for i in range(len(idx))])
    for k in np.flatnonzero(np.isin(idx, classes["prior"])):
        L[k] = lp.sqrt_info_kind("dense", rng)
    return prob, absp, W, (idx, mean, L), classes


def rank_requests(prob, classes, seed=32):
    """every class landmark in both positions of a landmark pair with short and long partners and with each other, in
    camera-landmark requests with a camera of its track and one outside; random requests of every kind besides"""
    nc, nl = len(prob.cams), len(prob.lm_off) - 1
    rng = np.random.default_rng(seed)
    cls = classes["r3"][:4] + classes["prior"] + classes["r2"]
    partners = [0, 1, 2, 3] + [int(l) for l in rng.choice(np.arange(len(RANK_LONG), nl), 4, replace=False)]
    lm = [[l, p] for l in cls for p in partners] + [[p, l] for l in cls for p in partners] + [[l, l] for l in cls]
    lm += [[a, b] for a in cls[::3] for b in cls[1::3]]
    cl = []
    for l in cls:
        track = np.asarray(prob.obs_cam[prob.lm_off[l]:prob.lm_off[l + 1]])
        cl += [[int(track[0]), l], [int(track[-1]), l], [int(np.setdiff1d(np.arange(nc), track)[0]), l]]
    r = cbm.random_requests(rng, nc, nl, 60)
    return dict(cameras=r["cameras"], camera_landmark=np.r_[np.array(cl), r["camera_landmark"]],
                landmarks=np.r_[np.array(lm), r["landmarks"]], relative=r["relative"])


# the 7-camera version of rank_case, every landmark of full rank in every instance (the dense inverse exists)
SMALL_RANK = dict(nc=7, long=[7, 6], nshort=60, switch_off=False)

# the four instances of k_cov_landmark<S, LMP, OBSW> and what each sets on the handle
INSTANCES = {"plain": (False, False), "lmp": (True, False), "obsw": (False, True), "lmp_obsw": (True, True)}


def huber_threshold(prob, W=None):
    """the median |W r| (|r| without W) over the observations in use: about half of the Huber weights are active"""
    if W is None:
        L = cm.linearize(*cm.observations(prob))
        return float(np.median(np.sqrt((L["res"] ** 2).sum(1))))
    w = om.whitened(prob, W)
    return float(np.median(np.sqrt((w["wr"][w["on"]] ** 2).sum(1))))


def instance_inputs(name, W, lm_prior):
    lmp, obsw = INSTANCES[name]
    return dict(lm_prior=lm_prior if lmp else None, W=W if obsw else None)


def dense_total(prob, dtype=np.float64, absp=None, lm_prior=None, W=None, threshold=None):
    """(Jp, Jl) of the dense total system at the stored state: the reprojection rows (whitened by W, Huber weight at
    `threshold`), the camera priors' rows and the landmark priors' rows L in their landmark's columns"""
    sprob, sabsp, _ = cvm.as_stored(prob, dtype, absp)
    cams = np.asarray(sprob.cams, np.float64)
    nc, nl = len(cams), len(sprob.lm_off) - 1
    if W is None:
        jp, jl, _, _ = cm.weighted(sprob, dtype=dtype, threshold=threshold, device_rot=True)
    else:
        w = om.whitened(sprob, stored(W, dtype), dtype=dtype, threshold=threshold, device_rot=True)
        jp, jl = w["Jp"], w["Jl"]
    Jp, Jl = cbm.dense_rows(jp, jl, np.asarray(sprob.obs_cam), np.asarray(sprob.lm_off), nc)
    rows_p, rows_l = [Jp], [Jl]
    if sabsp is not None:
        A, _ = pm.rows(cams, *sabsp, device_rot=True)
        Ja = np.zeros((9 * nc, 9 * nc))
        for c in range(nc):
            Ja[9 * c:9 * c + 9, 9 * c:9 * c + 9] = A[c]
        rows_p.append(Ja)
        rows_l.append(np.zeros((9 * nc, 3 * nl)))
    if lm_prior is not None:
        idx, L = np.asarray(lm_prior[0]), stored(lm_prior[2], dtype)
        R = np.zeros((3 * len(idx), 3 * nl))
        for k, l in enumerate(idx):
            R[3 * k:3 * k + 3, 3 * l:3 * l + 3] = L[k]
        rows_p.append(np.zeros((3 * len(idx), 9 * nc)))
        rows_l.append(R)
    return np.vstack(rows_p), np.vstack(rows_l)


# ---- D. grid-stride edges ---------------------------------------------------------------------------------------------
def edge_case():
    from rootba_b200.synthetic import synth_bal
    prob = synth_bal(120, 500, 3.6, seed=5)
    return prob, cvm.centre_priors(prob, 5)


def edge_master(prob, sms, seed=41):
    """per kind a random request list as long as the largest edge count: every count takes a prefix of it"""
    nc, nl = len(prob.cams), len(prob.lm_off) - 1
    m = max(max(edge_counts(k, sms)) for k in LAUNCH)
    return cbm.random_requests(np.random.default_rng(seed), nc, nl, m)


# ---- E. intrinsics groups ----------------------------------------------------------------------------------------------
GROUP_NC = 240
GROUP_SIZES = (2, 65, 129)


def group_case(seed=51):
    """GROUP_NC cameras (random tracks, centre priors), groups of GROUP_SIZES members at random positions among the
    non-members; camera 7 (rows 63..71, across the first tile boundary) is a member that is not its group's lead, and another
    such member's pose is held.  The members start at their lead's intrinsics.  Returns (prob, absp, group, lead, mask,
    held member)"""
    import rootba_b200 as rb
    from rootba_b200.synthetic import BalArrays
    prob, absp = cvm.tile_case(GROUP_NC, seed=seed, per_camera=12)
    rng = np.random.default_rng(seed)
    perm = rng.permutation(GROUP_NC)
    group = np.full(GROUP_NC, -1, np.int32)
    start = 0
    for g, size in enumerate(GROUP_SIZES):
        group[perm[start:start + size]] = g
        start += size
    g7 = np.flatnonzero(group == group[7])
    if group[7] < 0 or g7[0] == 7:  # make camera 7 a non-lead member of the largest group
        other = [c for c in np.flatnonzero(group == 2) if c > 7][-1]
        group[other], group[7] = group[7], 2
    lead = sim.leads(group)
    assert lead[7] >= 0 and lead[7] != 7 and (9 * 7) // cvm.TILE != (9 * 7 + 8) // cvm.TILE
    held = int([c for c in np.flatnonzero(group == 1) if lead[c] != c][1])
    mask = np.zeros(GROUP_NC, np.uint8)
    mask[held] = rb.FIX_POSE
    cams = np.array(prob.cams, np.float64)
    cams[lead >= 0, 7:] = cams[lead[lead >= 0], 7:]
    prob = BalArrays(cams, prob.lms, prob.lm_off, prob.obs_cam, prob.obs_xy)
    return prob, absp, group, lead, mask, held


def group_requests(prob, group, lead, held, seed=52):
    """member pairs of every group (the lead, camera 7 and the held member among them), member / non-member pairs,
    camera-landmark requests of members and the same landmarks with their lead, random requests of every kind"""
    rng = np.random.default_rng(seed)
    nc, nl = len(prob.cams), len(prob.lm_off) - 1
    cams = []
    for g in range(len(GROUP_SIZES)):
        mem = np.flatnonzero(group == g)
        pick = np.unique(np.r_[mem[:2], mem[-1], rng.choice(mem, min(len(mem), 6), replace=False),
                               [c for c in (7, held) if group[c] == g]])
        cams += [[int(a), int(b)] for a in pick for b in pick]
    non = np.flatnonzero(group < 0)
    cams += [[int(a), int(b)] for a, b in zip(rng.choice(np.flatnonzero(group >= 0), 20), rng.choice(non, 20))]
    members = np.flatnonzero((lead >= 0) & (lead != np.arange(nc)))
    mem = np.unique(np.r_[7, held, rng.choice(members, 20, replace=False)])
    ls = rng.integers(0, nl, len(mem))
    cl = np.r_[np.c_[mem, ls], np.c_[lead[mem], ls]]
    r = cbm.random_requests(rng, nc, nl, 60)
    r["relative"][:3] = [[7, held], [held, int(lead[held])], [int(lead[7]), 7]]
    return dict(cameras=np.array(cams), camera_landmark=np.r_[cl, r["camera_landmark"]], landmarks=r["landmarks"],
                relative=r["relative"])


# ---- F. relative poses -------------------------------------------------------------------------------------------------
REL_ANGLES = (0.0, np.pi / 2, np.pi - 1e-3, np.pi)
REL_BASE = 12  # observed cameras; camera 7 straddles the first tile boundary
REL_T = 1e3


def relative_case(seed=61):
    """REL_BASE observed cameras with centre priors, then for every angle of REL_ANGLES and both signs of the stored
    quaternion one unobserved camera at that rotation from observed camera k % REL_BASE and at distance REL_T, held by a
    dense absolute prior and a dense pair prior to that camera (means at the current poses).  The first extra camera's pose
    is held.  Returns (prob, absp, pair, mask, pairs (extra, observed))"""
    import rootba_b200 as rb
    from scipy.spatial.transform import Rotation
    from rootba_b200.synthetic import BalArrays, synth_bal
    base = synth_bal(REL_BASE, 160, 3.6, seed=seed)
    rng = np.random.default_rng(seed)
    cams = [np.asarray(c, np.float64) for c in base.cams]
    pairs = []
    for k, (th, neg) in enumerate((th, neg) for th in REL_ANGLES for neg in (False, True)):
        o = (3 * k + 1) % REL_BASE
        axis = rng.standard_normal(3)
        axis /= np.linalg.norm(axis)
        Ro = cm.rotation(cams[o][:4])
        q = Rotation.from_matrix(Rotation.from_rotvec(th * axis).as_matrix() @ Ro).as_quat()
        q = q * (1.0 if q[3] >= 0 else -1.0) * (-1.0 if neg else 1.0)
        c = cams[o].copy()
        c[:4] = q
        d = rng.standard_normal(3)
        c[4:7] = REL_T * d / np.linalg.norm(d)
        cams.append(c)
        pairs.append((REL_BASE + k, o))
    cams = np.array(cams)
    nc = len(cams)
    prob = BalArrays(cams, base.lms, base.lm_off, base.obs_cam, base.obs_xy)
    mean, L = cvm.centre_priors(prob, seed)
    for e, _ in pairs:
        L[e] = pm.sqrt_info_kind("dense", rng)
    pairs = np.array(pairs, np.int32)
    pair = (pairs, qm.mean_at(cams, pairs), np.stack([qm.sqrt_info_kind("dense", rng) for _ in pairs]))
    mask = np.zeros(nc, np.uint8)
    mask[REL_BASE] = rb.FIX_POSE
    return prob, (mean, L), pair, mask, pairs


def relative_requests(prob, pairs, seed=62):
    """every (extra, observed) pair, every pair of consecutive extra cameras and camera 7 with every extra camera, all in
    both orders; random requests of the other kinds"""
    nc, nl = len(prob.cams), len(prob.lm_off) - 1
    extra = [int(e) for e in pairs[:, 0]]
    rel = [[int(a), int(b)] for a, b in pairs] + [[a, b] for a, b in zip(extra[:-1], extra[1:])] + [[7, e] for e in extra]
    rel = np.array(rel)
    r = cbm.random_requests(np.random.default_rng(seed), nc, nl, 30)
    return dict(cameras=r["cameras"], camera_landmark=r["camera_landmark"], landmarks=r["landmarks"],
                relative=np.r_[rel, rel[:, ::-1]])


def dense_check(got, prob, dtype, absp, threshold, req, lm_prior=None, W=None, c=8):
    """every kind against the blocks of the full inverse of the dense total system (dense_total), 8 N kappa u of the largest
    entry of each kind"""
    Jp, Jl = dense_total(prob, dtype, absp, lm_prior, W, threshold)
    F, kappa, N = cbm.full_covariance(Jp, Jl)
    cams = np.asarray(cvm.as_stored(prob, dtype)[0].cams, np.float64)
    want = cbm.dense_blocks(F, len(cams), cams, **req)
    bar = c * N * kappa * cbm.U
    assert bar <= 1e-4, f"dense bar {bar:.3g} above 1e-4 (kappa {kappa:.3g})"
    for key in want:
        scale = np.abs(want[key]).max()
        err = np.abs(np.asarray(got[key]) - want[key]).max()
        assert err <= bar * scale, f"{key}: off by {err / scale:.3g} of its largest entry, bar {bar:.3g}"
