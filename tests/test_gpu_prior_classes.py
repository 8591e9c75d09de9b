"""The prior and intrinsics-group kernels at every boundary of their launch geometry (tests/prior_classes.py), camera by
camera and item by item, against float64:

  iterates      the PCG and power-series solves at 1, 2, 3 iterations and at convergence against pcg_replay / power_replay
                on the handle's own b, M^-1 and rba_right_multiply, at the bars of test_gpu_camera_classes (10 k u kappa, and on
                at most 33 cameras no less than 4 times the replay's own sensitivity to rounding),
                over VEC_CASES with (a) camera priors of every kind, (b) (a) + pair priors, among them one that ties the
                unobserved last camera, (c) (b) + intrinsics groups (PCG only: Power-SC rejects groups), whose replay runs
                the tied operator u -> P^T (right_multiply(P u) - lam P u) + lam u.  (b) reaches k_pcg_vec<S, true, true>
                and k_power_vec<S, true>; with groups the prior terms move into k_group_contract and the vector step runs
                without them, so (c) does not replace (b).  (a) (k_pcg_vec<S, true, false>) runs at clusters 1 and 16.
  per camera    float64 handles at nc = 127, 128, 129, 257 (m = nc pairs) and at 1900 cameras with a hub of 320 incident
                pair sides, or with groups of 2 .. 400 members: the scaling, rba_right_multiply, b, and the SCHUR_JACOBI and
                JACOBI inverse blocks, each at gamma_k of its magnitudes with k counted from the camera's own terms (+ 9
                for its absolute prior, + 12 per incident pair side, + C_LIN units of the prior rows' linearisation).
                float32 is covered by the iterates, which use only the handle's own data: its prior rows are linearised
                in float32, and no componentwise bar of that linearisation is derived here.
  per item      the cost (rba_compute_error minus that of a twin handle without priors) and the model-cost change
                (rba_apply's l_diff minus the twin's for the same unscaled increment) against the float64 sums over the
                items, for every prior kind at 1 (2 cameras for the camera kind), 255, 256, 257, 511, 512, 513 and 4100 items.
"""
import numpy as np
import pytest

import landmark_prior_model as lp
import shared_intrinsics_model as sm
import solver_model as smod
from objective_checks import FIX_POSE, bal_problem
from prior_classes import (C_LIN, SUM_THREADS, U64, CAMERA_ITEM_COUNTS, HUB_NC, ITEM_COUNTS, LM_ITEM_CAMERAS, PAIR_ITEM_CAMERAS,
                           PriorTerms, camera_prior, chain_pairs, check_b, check_bar, check_inverse_blocks, check_item_sum,
                           check_scaling, group_layout, landmark_cost_items,
                           hub_pairs, item_problem, pair_prior, random_pairs, vec_groups)
from test_gpu_camera_classes import (F32_MAX_CAMERAS, LAM_PCG, UNOBSERVED_LAST, VEC_CASES, _env, _plain_operator,
                                     bar_constants, model_constants, panel_sums, pcg_edge_sweep, power_edge_sweep, vec_problem)

pytestmark = pytest.mark.gpu
F64 = np.float64


def _handle(arrays, dtype, env=None, camera=None, pairs=None, groups=None, landmarks=None, mask=None, solve=None, **opt):
    import rootba_b200 as rb
    bp = bal_problem(arrays, dtype, camera_prior=camera, camera_pair_prior=pairs, landmark_prior=landmarks, camera_fixed=mask)
    if groups is not None:
        bp.intrinsics_group = groups
    with _env(env or {}):
        lin = rb.LinearizorQR.create(bp, rb.SolverOptions(**opt))
    lin.linearize()
    if solve is not None:
        lin.solve(solve)
    return lin


def _ids(v):
    return v if isinstance(v, str) else np.dtype(v).name


# ---- part 2: the iterates at the camera-count edges, with priors ---------------------------------------------------------
def vec_features(kind, arrays):
    nc = arrays.nc
    out = {"camera": camera_prior(arrays.cams, seed=nc)}
    if kind in ("b", "c"):
        out["pairs"] = pair_prior(arrays.cams, chain_pairs(nc), seed=nc + 1)
    if kind == "c":
        out["groups"] = vec_groups(nc)
    return out


def _tied_operator(groups):
    """the replay's operator of a handle with intrinsics groups: u -> P^T (right_multiply(P u) - lam P u) + lam u (the
    full operator less its damping, contracted, plus the damping of the tied problem), and u -> P u"""
    from test_gpu_pcg_iterates import operator_of
    lead = sm.leads(groups)
    expand = lambda u: sm.expand(u, lead)

    def operator(lin, dtype):
        op, lam = operator_of(lin, dtype), float(dtype(LAM_PCG))
        return (lambda u: sm.contract(op(expand(u)) - lam * expand(u), lead) + lam * np.asarray(u, np.float64)), expand
    return operator


def _with(feats):
    """a handle maker for the sweeps of test_gpu_camera_classes with the priors, groups and held flags of feats"""
    return lambda arrays, dtype, env, **opt: _handle(arrays, dtype, env, **feats, **opt)


# On at most 33 cameras the replay's sensitivity to rounding (test_gpu_camera_classes.replay_sensitivity) enters the bar.
# The case that needs it: 3 cameras with a group of 2 (clusters 2 and 4, float64), whose solve is still converging at
# k = 13.  There the iterates of float64 replays of the handle's own operator, perturbed by C_BAR u of its magnitudes,
# spread by 2e-13 at k = 10 and 1.1e-12 at k = 13, growing about 2.3 times per iteration; the handle's iterate stays within
# that spread at every k (1.1e-12 at k = 13), while C_BAR k u kappa, linear in k, is 2.4e-13.
SENSITIVITY_CAMERAS = 33


def pcg_sweep(arrays, dtype, env, feats):
    groups = feats.get("groups")
    pcg_edge_sweep(arrays, dtype, env, _with(feats), _tied_operator(groups) if groups is not None else _plain_operator,
                   sensitivity=arrays.nc <= SENSITIVITY_CAMERAS)


def power_sweep(arrays, dtype, env, feats):
    power_edge_sweep(arrays, dtype, env, _with(feats))


def _vec_params(clusters=None):
    out = []
    for c, nc in VEC_CASES:
        if clusters is not None and c not in clusters:
            continue
        for dtype in (np.float32, np.float64) if nc <= F32_MAX_CAMERAS else (np.float64,):
            out.append(pytest.param(c, nc, dtype, id=f"c{c}-nc{nc}-{np.dtype(dtype).name}"))
    return out


def _vec(c, nc):
    return vec_problem(nc, (c, nc) in UNOBSERVED_LAST), {"RBA_PCG_CLUSTER": str(c)}


@pytest.mark.parametrize("c,nc,dtype", _vec_params())
def test_pcg_iterates_with_pair_priors(c, nc, dtype):
    arrays, env = _vec(c, nc)
    pcg_sweep(arrays, dtype, env, vec_features("b", arrays))


@pytest.mark.parametrize("c,nc,dtype", _vec_params())
def test_pcg_iterates_with_priors_and_groups(c, nc, dtype):
    arrays, env = _vec(c, nc)
    pcg_sweep(arrays, dtype, env, vec_features("c", arrays))


@pytest.mark.parametrize("c,nc,dtype", _vec_params())
def test_power_series_with_pair_priors(c, nc, dtype):
    arrays, env = _vec(c, nc)
    power_sweep(arrays, dtype, env, vec_features("b", arrays))


@pytest.mark.parametrize("solver", ["pcg", "power"])
@pytest.mark.parametrize("c,nc,dtype", _vec_params(clusters=(1, 16)))
def test_iterates_with_camera_priors_only(c, nc, dtype, solver):
    arrays, env = _vec(c, nc)
    (pcg_sweep if solver == "pcg" else power_sweep)(arrays, dtype, env, vec_features("a", arrays))


def test_pcg_iterates_at_the_hub_with_a_held_neighbour():
    """the hub of HUB_SIDES pair sides (a repeated, a reversed pair, a pair to the unobserved last camera) whose neighbour
    camera 5 has its pose held, at the default cluster (more than 113 cameras per CTA: the strided vector step).  float64:
    a float32 replay needs the operator assembled from 9 nc unit vectors"""
    arrays = vec_problem(HUB_NC, True)
    mask = np.zeros(HUB_NC, np.uint8)
    mask[5] = FIX_POSE
    feats = {"camera": camera_prior(arrays.cams, seed=3), "pairs": pair_prior(arrays.cams, hub_pairs(), seed=4), "mask": mask}
    pcg_sweep(arrays, F64, {}, feats)


# ---- part 3: every camera's prior terms (float64) --------------------------------------------------------------------------
LAM = 0.1


def _p3_case(name):
    if name in ("hub", "groups"):
        arrays = vec_problem(HUB_NC, True)
        pairs = hub_pairs() if name == "hub" else chain_pairs(HUB_NC)
        groups = group_layout() if name == "groups" else None
        if groups is not None:  # the members take their lead's intrinsics when the groups are set: so does the twin
            from rootba_b200.synthetic import BalArrays
            lead = sm.leads(groups)
            cams = np.array(arrays.cams, np.float64)
            cams[lead >= 0, 7:] = cams[lead[lead >= 0], 7:]
            arrays = BalArrays(cams, arrays.lms, arrays.lm_off, arrays.obs_cam, arrays.obs_xy)
    else:
        nc = int(name[2:])
        arrays = vec_problem(nc, True)
        pairs, groups = chain_pairs(nc, None if nc == 257 else nc), None
    return arrays, camera_prior(arrays.cams, seed=arrays.nc + 5), pair_prior(arrays.cams, pairs, seed=arrays.nc + 6), groups


P3_CASES = ["nc127", "nc128", "nc129", "nc257", "hub", "groups"]


@pytest.mark.parametrize("case", P3_CASES)
def test_prior_terms_per_camera(case):
    import camera_model as cm
    arrays, camera, pairs, groups = _p3_case(case)
    nc = arrays.nc
    lin = _handle(arrays, F64, camera=camera, pairs=pairs, groups=groups, solve=LAM)
    twin = _handle(arrays, F64, solve=LAM)
    try:
        terms = PriorTerms(arrays.cams, camera, pairs)
        kp = terms.k()
        # scaling: diag2 = (1 / s - eps)^2 = the twin's reprojection column norms + the prior rows', summed over a group
        eps = float(cm.EPS_SQRT[np.dtype(F64)])
        s = np.asarray(lin.get_jacobian_scaling()[0], np.float64)
        s0 = np.asarray(twin.get_jacobian_scaling()[0], np.float64).reshape(nc, 9)
        check_scaling(((1 / s - eps) ** 2).reshape(nc, 9), (1 / s0 - eps) ** 2, s0, s, terms, groups)
        # b: the reprojection part from solver_model with the handle's scaling, + sum A^T r of the priors (contracted)
        model = smod.SCModel(arrays, F64, s, LAM)
        b_rep, Mb = model.b()
        check_b(lin.get_rhs(), b_rep, Mb, model_constants(arrays, model), s, terms, groups)
        # SCHUR_JACOBI inverse blocks: sum P_c^T P_c + lam I of the kernel's own panels + the prior blocks
        x = np.random.default_rng(3).uniform(-1, 1, 9 * nc)
        ref = panel_sums(arrays, lin.debug_get_block, LAM, x).result()
        cb, cy = bar_constants(arrays)
        check_inverse_blocks(lin.get_preconditioner()[0], ref["B"], ref["MB"], cb + smod.C_FIXED, s, LAM, terms, groups,
                             "SCHUR_JACOBI inverse")
        if groups is None:
            # H x = sum P^T (P x) + the prior terms at the handle's scaling + lam x
            y, My = terms.hx(s, x)
            bar = U64 * (cy[:, None] * ref["My"] + (kp + C_LIN)[:, None] * My)
            check_bar(lin.right_multiply(x), ref["y"] + y, bar, "H x")
            # JACOBI inverse blocks: solver_model's blocks + the prior blocks
            jac = _handle(arrays, F64, camera=camera, pairs=pairs, solve=LAM, preconditioner_type="JACOBI")
            sj = np.asarray(jac.get_jacobian_scaling()[0], np.float64)
            mj = smod.SCModel(arrays, F64, sj, LAM)
            J, MJ = mj.jacobi_blocks()
            check_inverse_blocks(jac.get_preconditioner()[0], J, MJ, model_constants(arrays, mj), sj, LAM, terms, None,
                                 "JACOBI inverse")
            jac.close()
    finally:
        lin.close()
        twin.close()


# ---- part 4: the cost and the model-cost change at the item-count edges -------------------------------------------------------
def _item_case(kind, n):
    if kind == "camera":
        arrays = item_problem(n)
        return arrays, {"camera": camera_prior(arrays.cams, seed=n)}
    if kind == "pair":
        arrays = item_problem(PAIR_ITEM_CAMERAS)
        return arrays, {"pairs": pair_prior(arrays.cams, random_pairs(arrays.nc, n, seed=n), seed=n)}
    arrays = item_problem(LM_ITEM_CAMERAS)
    rng = np.random.default_rng(n)
    idx = np.sort(rng.choice(arrays.nl, n, replace=False)).astype(np.int32)
    mean = np.asarray(arrays.lms, np.float64)[idx] + rng.normal(0, 0.05, (n, 3))
    L = np.stack([lp.sqrt_info_kind(("dense", "height", "rank2", "none")[p % 4], rng) for p in range(n)])
    return arrays, {"landmarks": (idx, mean, L)}


def _items(kind):
    counts = CAMERA_ITEM_COUNTS if kind == "camera" else ITEM_COUNTS
    return [pytest.param(kind, c, id=f"{kind}-{c}") for c in counts]


@pytest.mark.parametrize("kind,n", _items("camera") + _items("pair") + _items("landmark"))
def test_prior_cost_per_item_count(kind, n):
    arrays, feats = _item_case(kind, n)
    lin, twin = _handle(arrays, F64, **feats), _handle(arrays, F64)
    e, e0 = lin.compute_error()["all"]["error"], twin.compute_error()["all"]["error"]
    lin.close()
    twin.close()
    if kind == "landmark":
        items, mag = landmark_cost_items(arrays.lms, *feats["landmarks"])
    else:
        items, mag = PriorTerms(arrays.cams, feats.get("camera"), feats.get("pairs")).cost_items(kind)
    assert len(items) == n
    bar = check_item_sum(e - e0, items, mag, U64, f"{kind} cost", extra=2 * U64 * (abs(e) + abs(e0)))
    if n > SUM_THREADS:  # the prior part is not swamped: the 257th item alone exceeds the bar
        assert abs(items[SUM_THREADS]) > 2 * bar, (kind, n, items[SUM_THREADS], bar)


@pytest.mark.parametrize("kind,n", _items("camera") + _items("pair"))
def test_prior_model_cost_change_per_item_count(kind, n):
    """l_diff of rba_apply(h, x) minus the twin's l_diff for x' = D x / D' (the same unscaled increment d = D x): the prior
    part -sum_p (A_p d)^T (1/2 A_p d + r_p).  The two reprojection parts agree to rounding, bounded by c_rep u M_rep with
    M_rep = q / 2 + sqrt(2 cost q), q = x'^T (H' x') >= |J d|^2 from the twin's operator, c_rep = the observation count + 1000"""
    arrays, feats = _item_case(kind, n)
    lin, twin = _handle(arrays, F64, solve=LAM, **feats), _handle(arrays, F64, solve=LAM)
    try:
        s = np.asarray(lin.get_jacobian_scaling()[0], np.float64)
        s0 = np.asarray(twin.get_jacobian_scaling()[0], np.float64)
        x = np.random.default_rng(n).uniform(-1, 1, 9 * arrays.nc) * 1e-2
        x0 = s * x / s0
        q = float(x0 @ twin.right_multiply(x0))
        cost0 = twin.compute_error()["all"]["error"]
        ld, ld0 = lin.apply(x), twin.apply(x0)
    finally:
        lin.close()
        twin.close()
    items, mag = PriorTerms(arrays.cams, feats.get("camera"), feats.get("pairs")).ldiff_items(kind, s * x)
    m_rep = 0.5 * q + np.sqrt(2 * cost0 * q)
    extra = (arrays.nobs + 1000) * U64 * m_rep + 2 * U64 * (abs(ld) + abs(ld0))
    assert len(items) == n
    bar = check_item_sum(ld - ld0, -items, mag, U64, f"{kind} l_diff", extra=extra)
    if n > SUM_THREADS:  # the prior part is not swamped: the 257th item alone exceeds the bar
        assert abs(items[SUM_THREADS]) > 2 * bar, (kind, n, items[SUM_THREADS], bar)
