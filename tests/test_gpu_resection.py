"""Resection of cameras from the current landmarks (rba_resect_cameras, DESIGN.md section 26) on the GPU: every mode in both
precisions against the float64 model of tests/resection_model.py camera by camera; cameras with 0, 2, 5 and 6 usable
points, planar points and points behind the camera; held, partially fixed and grouped cameras; rigs with and without
estimated sensors; switched-off observations, every loss, camera and pair priors with and without losses; the costs;
determinism across calls, solver configurations and subsets; the protocol and the rejected arguments; an LM run from
perturbed cameras; and the example's flags.

Bars, per unit from its own conditioning (u the unit roundoff of float64, eps_S that of the handle's Scalar, t the pose's
translation):
  LINEAR   |R - R_model|_F, |t - t_model| <= 1e3 kappa u (1 + |t| + |Xbar| + s) + 8 eps_S (1 + |t|), kappa = lambda_12 /
           lambda_2 of the model's 12x12 M (the gap that bounds the eigenvector's rounding, Jacobi against LAPACK)
  REFINE   the same differences <= 1e3 sqrt(u) (1 + |t|) sqrt(cond H) + 8 eps_S (1 + |t|), H the free block of the unit's
           normal equations, both converged (max_iterations = 100)
  cost     relative 1e-9 against the model's share at the cameras the handle stored."""
import os
import subprocess
import sys

import numpy as np
import pytest

import observation_loss_model as olm
import resection_model as rm
from rootba_b200 import _lib
from rootba_b200.synthetic import BalArrays, synth_bal, synth_rig_capture, write_bal

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = np.finfo(np.float64).eps
MODES = {"linear": rm.LINEAR, "refine": rm.REFINE, "linear+refine": rm.LINEAR | rm.REFINE}
STATUS_MASK = rm.WRITTEN | rm.FEW_POINTS | rm.DEGENERATE | rm.BEHIND | rm.HELD


def _f(a, dtype):
    return np.asarray(np.asarray(a, dtype), np.float64)


def _obs_lm(prob):
    return np.repeat(np.arange(prob.nl), np.diff(prob.lm_off))


def _problem(seed=3, nc=24, nl=900, rot=0.05, trans=0.5, k1=0.02, noise=0.5):
    """cameras perturbed by several degrees and tenths of units, landmarks exact, moderate distortion"""
    return synth_bal(nc, nl, 5.0, seed=seed, obs_noise=noise, perturb_lm=0.0, perturb_rot=rot, perturb_trans=trans,
                     k1_sigma=k1, k2_sigma=0.001 if k1 else 1e-13)


def _handle(prob, dtype, W=None, loss=None, cprior=None, pprior=None, cprior_loss=None, pprior_loss=None, fixed=None,
            groups=None, rigs=None, sensors=None, **opts):
    import rootba_b200 as rb
    bp = rb.BalProblem.from_arrays(prob, dtype)
    if W is not None:
        bp.observation_sqrt_info = W
    if loss is not None:
        bp.observation_loss = loss
    if cprior is not None:
        bp.camera_prior = cprior
    if pprior is not None:
        bp.camera_pair_prior = pprior
    if fixed is not None:
        bp.camera_fixed = fixed
    if groups is not None:
        bp.intrinsics_group = groups
    if rigs is not None:
        bp.camera_rig = rigs
    if sensors is not None:
        bp.rig_sensor = sensors
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(**opts))
    if cprior_loss is not None:
        lin.set_prior_loss("camera", *cprior_loss)
    if pprior_loss is not None:
        lin.set_prior_loss("pair", *pprior_loss)
    lin.download_state()  # the cameras as stored (rigs re-tied)
    return bp, lin


def _model(prob, dtype, cams, W=None, kind=None, a=None, cprior=None, pprior=None, **kw):
    """the model of the handle's stored inputs; cprior (mean, L, kind, a), pprior (pairs, mean, L, kind, a) rounded likewise"""
    if cprior is not None:
        mean = _f(cprior[0], dtype)
        cprior = (mean, _f(cprior[1], dtype), np.asarray(cprior[2]), _f(cprior[3], dtype))
    if pprior is not None:
        pprior = (np.asarray(pprior[0]), _f(pprior[1], dtype), _f(pprior[2], dtype), np.asarray(pprior[3]), _f(pprior[4], dtype))
    return rm.Problem(np.asarray(cams, np.float64), _f(prob.lms, dtype), prob.obs_cam, _obs_lm(prob), _f(prob.obs_xy, dtype),
                      W=None if W is None else _f(W, dtype), kind=kind, a=None if a is None else _f(a, dtype),
                      cprior=cprior, pprior=pprior, dtype=dtype, **kw)


def _rot(c):
    q = np.asarray(c[:4], np.float64)
    return rm.rot(q / np.linalg.norm(q))


def _compare(model, cams_in, cams_out, status, points, cost, cams_list, mode, max_iterations, dtype):
    """camera cams_list[p] against the model started from cams_in; returns the number of written units compared"""
    eps_s = np.finfo(dtype).eps
    seen = 0
    for p, c in enumerate(cams_list):
        out, st, pts, co = model.resect(int(c), mode, max_iterations)
        assert (status[p] & STATUS_MASK) == (st & STATUS_MASK), (c, status[p], st)
        assert points[p] == pts, (c, points[p], pts)
        ld, mem = model.unit(int(c))
        if not status[p] & rm.WRITTEN:
            assert np.array_equal(cams_out[mem], cams_in[mem]), c  # untouched, bit for bit
            continue
        t = np.linalg.norm(out[ld][4:7])
        rnd = 8 * eps_s * (1 + t)
        if status[p] & rm.REFINED and status[p] & rm.CONVERGED and st & rm.CONVERGED and st & rm.REFINED:
            _, H, _, _ = model.cost(out[ld], ld, mem, with_normal=True)
            fi = np.flatnonzero(model.free(int(c), mode))
            ev = np.linalg.eigvalsh(H[np.ix_(fi, fi)])
            bar = 1e3 * np.sqrt(U) * (1 + t) * np.sqrt(ev[-1] / max(ev[0], 1e-300)) + rnd
        elif not status[p] & rm.REFINED and not st & rm.REFINED:
            ev, s, xb = model.linear_condition(ld, mem)
            bar = 1e3 * ev[-1] / ev[1] * U * (1 + t + np.linalg.norm(xb) + s) + rnd
        else:
            continue  # refined on one side only: the paths may part
        for j in mem:
            assert np.linalg.norm(_rot(cams_out[j]) - _rot(out[j])) <= bar, (c, j, bar)
            assert np.linalg.norm(cams_out[j, 4:7] - out[j][4:7]) <= bar * (1 + t), (c, j, bar)
            assert np.array_equal(cams_out[j, 7:10], np.asarray(out[j][7:10], dtype)) or mode & rm.INTRINSICS
        cg = model.cost(cams_out[ld], ld, mem, start=cams_in, member_cams={j: cams_out[j] for j in mem})
        assert abs(cost[p] - cg) <= 1e-9 * max(cg, 1e-12) + 1e-12, (c, cost[p], cg)
        seen += 1
    return seen


def _run(prob, dtype, mode="linear+refine", cameras=None, intrinsics=False, max_iterations=100, model_kw=None, **hk):
    bp, lin = _handle(prob, dtype, **hk)
    cams_in = np.array(bp.cams, np.float64)
    status, points, cost = lin.resect(cameras, mode=mode, intrinsics=intrinsics, max_iterations=max_iterations)
    cams_out = np.array(bp.cams, np.float64)
    lin.close()
    model = _model(prob, dtype, cams_in, **(model_kw or {}))
    lst = np.arange(prob.nc) if cameras is None else np.asarray(cameras)
    m = MODES[mode] | (rm.INTRINSICS if intrinsics else 0)
    return _compare(model, cams_in, cams_out, status, points, cost, lst, m, max_iterations, dtype), status, cams_in, cams_out


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("mode", list(MODES))
def test_modes_against_model(dtype, mode):
    prob = _problem()
    seen, status, _, _ = _run(prob, dtype, mode)
    assert seen > 0.8 * prob.nc and np.all(status & rm.WRITTEN)


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_intrinsics_against_model(dtype):
    prob = _problem(seed=5)
    seen, status, cams_in, cams_out = _run(prob, dtype, "refine", intrinsics=True)
    assert seen > 0.8 * prob.nc
    assert np.any(cams_out[:, 7] != cams_in[:, 7])


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_point_counts(dtype):
    """0, 2, 5 and 6 usable points: FEW_POINTS untouched, DEGENERATE then refined, the linear estimate from 6"""
    prob = _problem(seed=6)
    W = np.broadcast_to(np.eye(2), (prob.nobs, 2, 2)).copy()
    keep = {0: 0, 1: 2, 2: 5, 3: 6}
    for c, n in keep.items():
        o = np.flatnonzero(prob.obs_cam == c)
        W[o[n:]] = 0.0
    cams = list(keep)
    for mode in MODES:
        _, status, cams_in, cams_out = _run(prob, dtype, mode, cameras=cams, W=W, model_kw=dict(W=W))
        assert np.all(status[:2] == rm.FEW_POINTS) and np.array_equal(cams_out[:2], cams_in[:2])
        if mode != "refine":
            assert status[2] & rm.DEGENERATE and not status[3] & rm.DEGENERATE


def _two_cams(X):
    """camera 0 at the origin looking along +z, camera 1 at z = 30 looking back; every landmark seen by both"""
    c0 = np.array([0, 0, 0, 1, 0, 0, 0, 500.0, 0, 0])
    c1 = np.array([0, 1, 0, 0, 0, 0, 30, 500.0, 0, 0])  # 180 degrees about y, centre (0, 0, 30)
    cams = np.stack([c0, c1])
    n = len(X)
    obs_cam = np.tile([0, 1], n).astype(np.int32)
    xy = np.zeros((2 * n, 2))
    for c in range(2):
        R = rm.rot(cams[c, :4])
        pc = X @ R.T + cams[c, 4:7]
        xy[c::2] = 500.0 * pc[:, :2] / pc[:, 2:]
    prob = BalArrays(cams, np.asarray(X, np.float64), np.arange(0, 2 * n + 1, 2, dtype=np.int64), obs_cam, xy)
    return prob


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_planar_and_behind(dtype):
    rng = np.random.default_rng(7)
    planar = np.column_stack([rng.uniform(-3, 3, 40), rng.uniform(-3, 3, 40), np.full(40, 12.0)])
    prob = _two_cams(planar)
    prob.cams = prob.cams.copy()
    prob.cams[0, 4:7] += [0.2, -0.1, 0.3]
    _, status, cams_in, cams_out = _run(prob, dtype, "linear", cameras=[0])
    assert status[0] == rm.DEGENERATE and np.array_equal(cams_out, cams_in)
    # most points behind camera 0 (in front of camera 1): the estimate is rejected
    X = np.column_stack([rng.uniform(-3, 3, 40), rng.uniform(-3, 3, 40), rng.uniform(-14, -8, 40)])
    prob = _two_cams(X)
    _, status, cams_in, cams_out = _run(prob, dtype, "linear", cameras=[0])
    assert status[0] == rm.BEHIND and np.array_equal(cams_out, cams_in)


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_held_partially_fixed_and_grouped(dtype):
    prob = _problem(seed=8)
    fixed = np.zeros(prob.nc, np.uint8)
    fixed[0:3] = rm.FIX_POSE
    fixed[3:6] = rm.FIX_F | rm.FIX_K2
    fixed[6] = rm.FIX_POSE | rm.FIX_F | rm.FIX_K1 | rm.FIX_K2
    groups = np.full(prob.nc, -1, np.int32)
    groups[10:14] = 0  # one intrinsics group: its cameras resect their pose only
    seen, status, cams_in, cams_out = _run(prob, dtype, "linear+refine", intrinsics=True, fixed=fixed, groups=groups,
                                           model_kw=dict(fixed=fixed, grouped=groups >= 0))
    assert np.all(status[0:3] & rm.WRITTEN) and not np.any(status[0:3] & rm.HELD)  # intrinsics free
    assert np.array_equal(cams_out[0:3, :7], cams_in[0:3, :7])
    assert np.array_equal(cams_out[3:6, [7, 9]], cams_in[3:6, [7, 9]])
    assert status[6] == rm.HELD and np.array_equal(cams_out[6], cams_in[6])
    assert np.array_equal(cams_out[10:14, 7:], cams_in[10:14, 7:])
    _, status, _, _ = _run(prob, dtype, "refine", fixed=fixed, model_kw=dict(fixed=fixed))  # pose held, no INTRINSICS
    assert np.all(status[0:3] == rm.HELD)


def _rig_problem(seed=4, perturb=True):
    cap = synth_rig_capture(3, 10, 250, seed=seed)
    prob = cap.prob
    rng = np.random.default_rng(seed)
    prob.obs_xy = prob.obs_xy + rng.normal(0, 0.3, prob.obs_xy.shape)
    if perturb:
        cams = prob.cams.copy()
        from scipy.spatial.transform import Rotation
        for f in range(10):  # move every placement: the re-tie at the handle's set-up carries it to the members
            d = Rotation.from_rotvec(rng.normal(0, 0.03, 3))
            lead = 3 * f
            R = d.as_matrix() @ rm.rot(cams[lead, :4])
            cams[lead, :4] = Rotation.from_matrix(R).as_quat()
            cams[lead, 4:7] += rng.normal(0, 0.2, 3)
        prob.cams = cams
    return cap, prob


def _maps(cams, lead):
    """M_j = T_j T_lead^-1 of the stored cameras (the identity for a lead)"""
    M = np.tile([0, 0, 0, 1.0, 0, 0, 0], (len(cams), 1))
    for j in range(len(cams)):
        if lead[j] >= 0 and lead[j] != j:
            M[j] = rm.tie(cams[j, :7], rm.pose_inv(cams[lead[j], :7]))
    return M


@pytest.mark.parametrize("sensors", [False, True], ids=["held", "sensors"])
def test_rigs_against_model(sensors):
    dtype = np.float64
    cap, prob = _rig_problem()
    rig = (cap.rig, cap.cam_from_rig)
    sens = np.where(cap.sensor == 0, -1, cap.sensor).astype(np.int32) if sensors else None
    bp, lin = _handle(prob, dtype, rigs=rig, sensors=sens)
    cams_in = np.array(bp.cams, np.float64)
    ext_in = lin.rig_extrinsics()
    lead = np.array([3 * (c // 3) for c in range(prob.nc)])  # sensor 0 is held: it leads every placement
    lst = np.array([1, 4, 5, 9, 20], np.int32)  # placements 0, 1 (two members listed), 3, 6
    status, points, cost = lin.resect(lst, max_iterations=100)
    cams_out = np.array(bp.cams, np.float64)
    ext_out = lin.rig_extrinsics()
    lin.close()
    units = {3 * (c // 3) + k for c in lst for k in range(3)}
    others = np.setdiff1d(np.arange(prob.nc), sorted(units))
    assert np.array_equal(cams_out[others], cams_in[others])  # unlisted cameras bit-identical
    assert np.allclose(ext_out, ext_in, rtol=0, atol=1e-12) or np.allclose(np.abs(ext_out), np.abs(ext_in), atol=1e-12)
    assert status[1] == status[2] and points[1] == points[2] and cost[1] == cost[2]  # one unit, listed twice
    model = _model(prob, dtype, cams_in, lead=lead, M=_maps(cams_in, lead))
    assert _compare(model, cams_in, cams_out, status, points, cost, lst, rm.LINEAR | rm.REFINE, 100, dtype) >= 3
    for c in sorted(units):  # members tied to their lead after the call
        if lead[c] != c:
            want = rm.tie(model.M[c], cams_out[lead[c], :7])
            assert np.allclose(cams_out[c, :7], want, rtol=0, atol=1e-12), c


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_held_rig_in_float32_and_float64(dtype):
    cap, prob = _rig_problem(seed=9)
    bp, lin = _handle(prob, dtype, rigs=(cap.rig, cap.cam_from_rig))
    cams_in = np.array(bp.cams, np.float64)
    status, points, cost = lin.resect(max_iterations=100)
    cams_out = np.array(bp.cams, np.float64)
    lin.close()
    lead = np.array([3 * (c // 3) for c in range(prob.nc)])
    E = _f(cap.cam_from_rig, dtype)  # the extrinsics as the handle stores them
    M = np.tile([0, 0, 0, 1.0, 0, 0, 0], (prob.nc, 1))
    for j in range(prob.nc):
        if lead[j] != j:
            e = E[j] / np.r_[np.linalg.norm(E[j, :4]) * np.ones(4), np.ones(3)]
            el = E[lead[j]] / np.r_[np.linalg.norm(E[lead[j], :4]) * np.ones(4), np.ones(3)]
            M[j] = rm.tie(e, rm.pose_inv(el))
    model = _model(prob, dtype, cams_in, lead=lead, M=M)
    assert _compare(model, cams_in, cams_out, status, points, cost, np.arange(prob.nc), rm.LINEAR | rm.REFINE, 100,
                    dtype) > 0.5 * prob.nc
    assert np.all(status == status[lead])


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("prior_loss", [False, True], ids=["no_prior_loss", "prior_loss"])
def test_information_losses_and_priors_against_model(dtype, prior_loss):
    prob = _problem(seed=9, nc=20, nl=700)
    rng = np.random.default_rng(2)
    W = rng.normal(0, 0.2, (prob.nobs, 2, 2)) + np.eye(2)
    W[rng.random(prob.nobs) < 0.1] = 0.0
    kind, scale = olm.mixed(prob.nobs, seed=6)
    nc = prob.nc
    mean = np.array(prob.cams, np.float64)
    mean[:, 4:7] = -np.einsum("nji,nj->ni", rm.rot(mean[:, :4]), mean[:, 4:7]) + rng.normal(0, 0.2, (nc, 3))
    L = np.zeros((nc, 9, 9))
    L[::3] = np.diag([2.0, 2.0, 2.0, 30.0, 30.0, 30.0, 0.0, 0.0, 0.0])
    pairs = np.array([[1, 2], [4, 7], [10, 5], [12, 13]], np.int32)
    from pair_prior_model import mean_at
    pmean = mean_at(prob.cams, pairs)
    pmean[:, 4:7] += rng.normal(0, 0.1, (len(pairs), 3))
    pL = np.broadcast_to(np.diag([4.0, 4.0, 4.0, 40.0, 40.0, 40.0]), (len(pairs), 6, 6)).copy()
    kinds5 = np.array([olm.NONE, olm.HUBER, olm.CAUCHY, olm.SOFT_L1, olm.TUKEY])
    ck = kinds5[np.arange(nc) % 5].astype(np.uint8) if prior_loss else np.zeros(nc, np.uint8)
    pk = kinds5[np.arange(len(pairs)) % 5].astype(np.uint8) if prior_loss else np.zeros(len(pairs), np.uint8)
    cs, ps = np.full(nc, 2.5), np.full(len(pairs), 2.5)
    bp, lin = _handle(prob, dtype, W=W, loss=(kind, scale), cprior=(mean, L), pprior=(pairs, pmean, pL),
                      cprior_loss=(ck, cs) if prior_loss else None, pprior_loss=(pk, ps) if prior_loss else None)
    cams_in = np.array(bp.cams, np.float64)
    # a unit's result does not depend on which other cameras are listed: resect half, then compare with the model
    lst = np.arange(0, nc, 2, dtype=np.int32)
    status, points, cost = lin.resect(lst, max_iterations=100)
    cams_out = np.array(bp.cams, np.float64)
    lin.close()
    qn = mean[:, :4] / np.linalg.norm(mean[:, :4], axis=1, keepdims=True)
    model = _model(prob, dtype, cams_in, W=W, kind=kind.astype(int), a=scale,
                   cprior=(np.column_stack([qn, mean[:, 4:]]), L, ck.astype(int), cs),
                   pprior=(pairs, pmean, pL, pk.astype(int), ps))
    assert _compare(model, cams_in, cams_out, status, points, cost, lst, rm.LINEAR | rm.REFINE, 100, dtype) > 0.5 * len(lst)


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_huber_refinement_lowers_every_cost(dtype):
    import rootba_b200 as rb
    prob = _problem(seed=12)
    bp = rb.BalProblem.from_arrays(prob, dtype)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(residual=rb.ResidualOptions(robust_norm="HUBER", huber_parameter=2.0)))
    e0 = lin.compute_error()["all"]["error"]
    _, _, c0 = lin.resect(mode="refine", max_iterations=0)  # no step: the share at the stored pose, nothing written
    assert np.array_equal(np.array(bp.cams), np.asarray(prob.cams, dtype))
    status, _, c1 = lin.resect(mode="refine")
    assert np.all(c1 <= c0)
    assert np.all(c1[(status & rm.WRITTEN) > 0] < c0[(status & rm.WRITTEN) > 0])
    e1 = lin.compute_error()["all"]["error"]
    assert e1 < e0
    cams_in = np.asarray(np.asarray(prob.cams, dtype), np.float64)
    model = _model(prob, dtype, cams_in, kind=olm.HUBER, a=2.0)
    for c in range(prob.nc):
        ld, mem = model.unit(c)
        cg = model.cost_stored(ld, mem)
        assert abs(c0[c] - cg) <= 1e-9 * cg
    lin.close()


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_bit_identical_across_calls_configurations_and_subsets(dtype):
    prob = _problem(seed=13)
    outs = []
    for cfg in (dict(), dict(solver_type="SCHUR_COMPLEMENT"), dict(operator_form="IMPLICIT", stage2_form="IDENTITY")):
        for _ in range(2):
            bp, lin = _handle(prob, dtype, **cfg)
            r = lin.resect()
            outs.append((np.array(bp.cams),) + r)
            lin.close()
    for o in outs[1:]:
        for a, b in zip(outs[0], o):
            assert np.array_equal(a, b)
    sub = np.random.default_rng(0).permutation(prob.nc)[: prob.nc // 3].astype(np.int32)
    bp, lin = _handle(prob, dtype)
    st, pt, co = lin.resect(sub)
    cams = np.array(bp.cams)
    lin.close()
    others = np.setdiff1d(np.arange(prob.nc), sub)
    assert np.array_equal(cams[others], np.asarray(prob.cams, dtype)[others])
    assert np.array_equal(cams[sub], outs[0][0][sub])
    assert np.array_equal(st, outs[0][1][sub]) and np.array_equal(pt, outs[0][2][sub]) and np.array_equal(co, outs[0][3][sub])


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_protocol_and_rejected_arguments(dtype):
    import ctypes as C
    import rootba_b200 as rb
    from rootba_b200.linearizor import _p
    prob = _problem(seed=14, nc=10, nl=300)
    bp, lin = _handle(prob, dtype)
    lin.linearize()
    lin._backup()
    before = np.array(bp.cams)
    lin.resect()
    assert not np.array_equal(np.array(bp.cams), before)
    with pytest.raises(_lib.RbaError) as e:
        lin.solve(1e-4)
    assert e.value.code == -6
    lin._restore()
    lin.download_state()
    assert np.array_equal(np.array(bp.cams), before)
    lin.linearize()
    lin.solve(1e-4)
    L = _lib.lib()
    o = _lib.ResectOpts()
    L.rba_default_resect_opts(C.byref(o))
    assert (o.mode, o.max_iterations, o.function_tolerance) == (3, 20, 1e-10)
    lin.download_state()
    ref = np.array(bp.cams)
    st = np.full(prob.nc, 255, np.uint8)
    idx_ok = np.arange(5, dtype=np.int32)

    def call(h, opts, num, idx):
        return L.rba_resect_cameras(h, None if opts is None else C.byref(opts), num, None if idx is None else _p(idx), _p(st),
                                    None, None)

    def opts(**kw):
        x = _lib.ResectOpts()
        L.rba_default_resect_opts(C.byref(x))
        for k, v in kw.items():
            setattr(x, k, v)
        return x

    nc = prob.nc
    cases = [(None, nc, None), (opts(mode=0), nc, None), (opts(mode=4), nc, None), (opts(mode=5), nc, None),
             (opts(mode=8), nc, None), (opts(mode=11), nc, None), (opts(max_iterations=-1), nc, None),
             (opts(function_tolerance=float("nan")), nc, None), (opts(function_tolerance=float("inf")), nc, None),
             (opts(function_tolerance=-1.0), nc, None), (opts(), -1, idx_ok), (opts(), nc - 1, None),
             (opts(), 2, np.array([0, nc], np.int32)), (opts(), 2, np.array([-1, 0], np.int32)),
             (opts(), 3, np.array([4, 1, 4], np.int32))]
    for k, (op, num, idx) in enumerate(cases):
        assert call(lin.h, op, num, idx) == -1, k
        assert np.all(st == 255), k
    lin.download_state()
    assert np.array_equal(np.array(bp.cams), ref)
    lin.solve(1e-4)  # still linearised: nothing changed
    lin.close()
    bp2 = rb.BalProblem.from_arrays(prob, dtype)
    sh = rb.LinearizorQR.create(bp2, rb.SolverOptions(nranks=2, rank=0))  # no communicator is made before rba_comm_init
    assert call(sh.h, opts(), nc, None) == -4 and np.all(st == 255)
    sh.close()


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_lm_run_from_perturbed_cameras_reaches_the_true_start(dtype):
    import rootba_b200 as rb
    prob = synth_bal(30, 2000, 5.0, seed=15, obs_noise=0.5, perturb_lm=0.0, perturb_rot=0.0, perturb_trans=0.0)
    opts = rb.SolverOptions(max_num_iterations=50, function_tolerance=1e-12)
    bp, lin = _handle(prob, dtype)
    lin.lm_run(50, opts)
    ref = lin.compute_error()["all"]["error"]
    lin.close()
    rng = np.random.default_rng(3)
    from scipy.spatial.transform import Rotation
    cams = np.array(prob.cams, np.float64)
    for c in range(prob.nc):  # several degrees and several units off
        d = Rotation.from_rotvec(np.deg2rad(5.0) * rng.normal(size=3) / np.sqrt(3))
        cams[c, :4] = (d * Rotation.from_quat(cams[c, :4])).as_quat()
        cams[c, 4:7] += rng.normal(0, 3.0, 3)
    bad = BalArrays(cams, prob.lms, prob.lm_off, prob.obs_cam, prob.obs_xy)
    bp, lin = _handle(bad, dtype)
    status, _, _ = lin.resect()
    assert np.count_nonzero(status & rm.WRITTEN) == prob.nc
    lin.lm_run(50, opts)
    got = lin.compute_error()["all"]["error"]
    lin.close()
    assert abs(got - ref) <= (1e-5 if dtype == np.float32 else 1e-6) * ref, (got, ref)


def test_example_flags(tmp_path):
    prob = _problem(seed=16, nc=10, nl=300)
    path = str(tmp_path / "problem.txt")
    write_bal(prob, path)
    out = str(tmp_path / "res.npz")
    base = [sys.executable, os.path.join(ROOT, "examples", "solve_bal.py"), path, "--max-num-iterations", "3",
            "--log-path", str(tmp_path / "log.json")]
    cmd = base + ["--resect", "linear+refine", "--resect-intrinsics", "--triangulate", "refine", "--resection", out]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "resected (linear+refine, intrinsics)" in r.stdout
    assert r.stdout.index("resected") < r.stdout.index("triangulated")  # resection first
    with np.load(out) as f:
        assert f["status"].shape == (prob.nc,) and np.all(f["status"] & rm.WRITTEN) and np.all(f["cost"] >= 0)
        assert np.all(f["points"] > 0)
    r = subprocess.run(base + ["--resection", out], capture_output=True, text=True, timeout=300)
    assert r.returncode != 0 and "--resection requires --resect" in r.stderr
    r = subprocess.run(base + ["--resect-intrinsics"], capture_output=True, text=True, timeout=300)
    assert r.returncode != 0 and "--resect-intrinsics requires --resect" in r.stderr
