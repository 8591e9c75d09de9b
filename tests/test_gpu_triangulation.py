"""Triangulation of landmarks from the current cameras (rba_triangulate_landmarks, DESIGN.md section 25) on the GPU: every
mode in both precisions against the float64 model of tests/triangulation_model.py landmark by landmark (track lengths of
every class up to 300 cameras; switched-off observations, every loss, landmark priors with and without losses; rigs with
estimated sensors); the skipped and rejected landmarks untouched bit for bit; the refinement's costs; determinism across
calls and solver configurations; subsets; the protocol and the rejected arguments; an LM run from scrambled landmarks; the
example's flags; and two ranks.

Bars, per landmark from its own conditioning (u the unit roundoff of float64, eps_S that of the handle's Scalar):
  LINEAR   |X - X_model| <= 100 kappa u (s + |X - cbar|) + 4 eps_S |X|, kappa = lambda_4 / lambda_2 of the model's M
  REFINE   |X - X_model| <= 1e3 sqrt(u) (1 + |X|) sqrt(cond H) + 4 eps_S |X|, both converged (max_iterations = 100)
  cost     relative 1e-9 against the model's share at the position the handle stored; the angle relative 1e-12 / 1e-5."""
import os
import subprocess
import sys

import numpy as np
import pytest

import objective_checks as oc
import observation_loss_model as olm
import triangulation_model as tm
from rootba_b200 import _lib
from rootba_b200.synthetic import BalArrays, synth_bal, synth_rig_capture, write_bal

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = np.finfo(np.float64).eps
CLASSES = [2, 3, 4, 5, 8, 9, 16, 17, 32, 33, 64, 65, 300]
MODES = {"linear": tm.LINEAR, "refine": tm.REFINE, "linear+refine": tm.LINEAR | tm.REFINE}
STATUS_MASK = tm.WRITTEN | tm.FEW_RAYS | tm.SMALL_ANGLE | tm.AT_INFINITY | tm.BEHIND


def _f(a, dtype):
    return np.asarray(np.asarray(a, dtype), np.float64)


def _stored(prob, dtype):
    return BalArrays(_f(prob.cams, dtype), _f(prob.lms, dtype), prob.lm_off, prob.obs_cam, _f(prob.obs_xy, dtype))


def _handle(prob, dtype, W=None, loss=None, prior=None, prior_loss=None, **opts):
    import rootba_b200 as rb
    bp = rb.BalProblem.from_arrays(prob, dtype)
    if W is not None:
        bp.observation_sqrt_info = W
    if loss is not None:
        bp.observation_loss = loss
    if prior is not None:
        bp.landmark_prior = prior
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(**opts))
    if prior_loss is not None:
        lin.set_prior_loss("landmark", *prior_loss)
    return bp, lin


@pytest.fixture(scope="module")
def classes():
    """one problem with tracks of every length class (several passes of the lane loop at 65 and 300), noisy, the landmarks
    perturbed, moderate distortion"""
    lengths = np.repeat(CLASSES, 6)
    return synth_bal(310, len(lengths), 4.0, seed=3, track_lengths=lengths, lm_spread=0.8, obs_noise=0.5, perturb_lm=0.5,
                     k1_sigma=0.02, k2_sigma=0.001)


def _model_tracks(prob, dtype, W=None, kind=None, a=None, prior=None, valid_only=False, cams=None):
    """the model's tracks of the handle's stored inputs; cams: the cameras the handle holds (bp.cams after the call's
    read-back), else prob's rounded to Scalar; prior (idx, mean, L, kind, a) rounded likewise"""
    sp = _stored(prob, dtype)
    if cams is not None:
        sp.cams = np.asarray(cams, np.float64)
    if W is not None:
        W = _f(W, dtype)
    if prior is not None:
        prior = (prior[0], _f(prior[1], dtype), _f(prior[2], dtype), prior[3], _f(prior[4], dtype))
    return sp, tm.tracks(sp, W, kind, None if a is None else _f(a, dtype), prior, valid_only, dtype)


def _compare(prob, dtype, mode, status, angle, cost, lms_out, trs, sp, max_iterations, min_angle=0.0, check_cost=True,
             lms_in=None):
    """landmark l of trs against the model started from sp.lms[l]; lms_in the stored positions before the call"""
    eps_s = np.finfo(dtype).eps
    lms_in = np.asarray(prob.lms, dtype) if lms_in is None else lms_in
    seen = 0
    for l, tr in enumerate(trs):
        X, st, ang, c = tr.triangulate(sp.lms[l], MODES[mode], max_iterations, min_angle, dtype=dtype)
        assert (status[l] & STATUS_MASK) == (st & STATUS_MASK), (l, status[l], st)
        assert abs(angle[l] - ang) <= (1e-12 if dtype == np.float64 else 1e-5) * max(ang, 1e-300), (l, angle[l], ang)
        Xg = np.asarray(lms_out[l], np.float64)
        if not status[l] & tm.WRITTEN:
            assert np.array_equal(lms_out[l], lms_in[l]), l  # untouched, bit for bit
            continue
        round_bar = 4 * eps_s * np.linalg.norm(X)
        if status[l] & (tm.REFINED | tm.CONVERGED) and st & tm.CONVERGED and status[l] & tm.CONVERGED:
            _, H, _ = tr.cost(X, with_normal=True)
            ev = np.linalg.eigvalsh(H)
            bar = 1e3 * np.sqrt(U) * (1 + np.linalg.norm(X)) * np.sqrt(ev[2] / max(ev[0], 1e-300)) + round_bar
        elif mode == "linear" or not status[l] & tm.REFINED:
            d, ok = tr.rays()
            c0 = tr.centres[ok]
            cb = c0.mean(0)
            s = np.sqrt(((c0 - cb) ** 2).sum(1).mean())
            M = np.zeros((4, 4))
            for i in np.flatnonzero(ok):
                R, t = tr.R[i], tr.cams[i, 4:7]
                B = np.hstack([R, ((R @ cb + t) / s)[:, None]])
                v = R @ d[i]
                v /= np.linalg.norm(v)
                M += B.T @ (np.eye(3) - np.outer(v, v)) @ B
            e = np.linalg.eigvalsh(M)
            bar = 100 * e[3] / e[1] * U * (s + np.linalg.norm(X - cb)) + round_bar
        else:
            continue  # refined without converging on one side: the paths may part
        assert np.linalg.norm(Xg - X) <= bar, (l, Xg, X, bar)
        if check_cost:  # the share at the position the handle stored
            cg = tr.cost(Xg)
            assert abs(cost[l] - cg) <= 1e-9 * max(cg, 1e-12) + 1e-12, (l, cost[l], cg)
        seen += 1
    return seen


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("mode", list(MODES))
def test_modes_against_model_at_every_track_length(classes, dtype, mode):
    bp, lin = _handle(classes, dtype)
    status, angle, cost = lin.triangulate(mode=mode, max_iterations=100)
    lms_out = np.array(bp.lms)
    lin.close()
    sp, trs = _model_tracks(classes, dtype, cams=bp.cams)
    seen = _compare(classes, dtype, mode, status, angle, cost, lms_out, trs, sp, 100)
    assert seen > 0.8 * classes.nl
    assert np.all(status & tm.WRITTEN)


def _planted(dtype):
    """FEW_RAYS (one observation in use), SMALL_ANGLE (a near-parallel pair under min_angle), AT_INFINITY (rays of a point
    1e12 away), BEHIND (a point behind the second camera) next to ordinary landmarks"""
    prob = synth_bal(12, 80, 3.0, seed=8, obs_noise=0.3, perturb_lm=0.2)
    prob.lms = prob.lms.copy()
    W = np.broadcast_to(np.eye(2), (prob.nobs, 2, 2)).copy()
    from rootba_b200.synthetic import project
    few = list(range(0, 8))
    for l in few:
        o0, o1 = prob.lm_off[l], prob.lm_off[l + 1]
        W[o0 + 1:o1] = 0.0
    far = list(range(8, 16))
    for l in far:
        o0, o1 = prob.lm_off[l], prob.lm_off[l + 1]
        X = np.array([1.0, 0.3, 0.2]) * 1e12
        prob.obs_xy[o0:o1] = project(prob.cams[prob.obs_cam[o0:o1]], np.broadcast_to(X, (o1 - o0, 3)))[0]
    behind = []
    for l in range(16, prob.nl):
        o0, o1 = prob.lm_off[l], prob.lm_off[l + 1]
        if o1 - o0 != 2:
            continue
        cams = prob.cams[prob.obs_cam[o0:o1]]
        R = tm.cm.rotation(cams[:, :4])
        c = -np.einsum("nji,nj->ni", R, cams[:, 4:7])
        Xb = c[1] + 0.5 * (c[1] - prob.lms[l])  # behind camera 1 along its line of sight
        z = np.einsum("nij,j->ni", R, Xb)[:, 2] + cams[:, 6]
        if z[0] > 1.0 and z[1] < -0.1:
            prob.obs_xy[o0:o1] = project(cams, np.broadcast_to(Xb, (2, 3)))[0]
            behind.append(l)
        if len(behind) == 6:
            break
    return prob, W, few, far, behind


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_skipped_and_rejected_landmarks_untouched(dtype):
    prob, W, few, far, behind = _planted(dtype)
    assert len(behind) >= 3
    bp, lin = _handle(prob, dtype, W=W)
    before = np.array(bp.lms)
    status, angle, cost = lin.triangulate(mode="linear", min_angle_deg=0.0)
    after = np.array(bp.lms)
    assert np.all(status[few] & tm.FEW_RAYS) and np.all(status[behind] & tm.BEHIND)
    # rays of a point 1e12 away: parallel up to the rounding of the observations, so at infinity in f64; in f32 the rounding
    # gives them a finite crossing, which is written or rejected like any other
    if dtype == np.float64:
        assert np.count_nonzero(status[far] & tm.AT_INFINITY) >= len(far) // 2
    skipped = (status & tm.WRITTEN) == 0
    assert skipped[few].all() and skipped[behind].all() and np.array_equal(before[skipped], after[skipped])
    sp, trs = _model_tracks(prob, dtype, W=W, cams=bp.cams)
    rest = np.setdiff1d(np.arange(prob.nl), far)
    _compare(prob, dtype, "linear", status[rest], angle[rest], cost[rest], after[rest], [trs[l] for l in rest],
             BalArrays(sp.cams, sp.lms[rest], None, None, None), 20, lms_in=before[rest])
    # SMALL_ANGLE: a threshold between the landmarks' angles skips the lower ones in every mode
    thr = float(np.median(angle[angle > 0]))
    bp2, lin2 = _handle(prob, dtype, W=W)
    st2, ang2, _ = lin2.triangulate(min_angle_deg=np.rad2deg(thr))
    small = (ang2 < thr) & (ang2 > 0) & ((st2 & tm.FEW_RAYS) == 0)
    assert small.sum() > 5 and np.all(st2[small] & tm.SMALL_ANGLE) and not np.any(st2[small] & tm.WRITTEN)
    assert np.array_equal(np.array(bp2.lms)[small], before[small])
    lin.close(); lin2.close()


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_information_losses_and_priors_against_model(dtype):
    prob = synth_bal(14, 300, 4.5, seed=9, obs_noise=1.0, perturb_lm=0.5, k1_sigma=0.02)
    rng = np.random.default_rng(2)
    W = rng.normal(0, 0.2, (prob.nobs, 2, 2)) + np.eye(2)
    W[rng.random(prob.nobs) < 0.1] = 0.0
    kind, scale = olm.mixed(prob.nobs, seed=6)
    idx = np.arange(0, prob.nl, 3, dtype=np.int32)
    mean = prob.lms[idx] + rng.normal(0, 0.1, (len(idx), 3))
    L = np.broadcast_to(np.diag([2.0, 3.0, 1.5]), (len(idx), 3, 3)).copy()
    pkind = np.array([olm.NONE, olm.HUBER, olm.CAUCHY, olm.SOFT_L1, olm.TUKEY])[np.arange(len(idx)) % 5].astype(np.uint8)
    pscale = np.full(len(idx), 2.8)
    for with_prior_loss in (False, True):
        bp, lin = _handle(prob, dtype, W=W, loss=(kind, scale), prior=(idx, mean, L),
                          prior_loss=(pkind, pscale) if with_prior_loss else None)
        status, angle, cost = lin.triangulate(max_iterations=100)
        lms_out = np.array(bp.lms)
        lin.close()
        pk = pkind if with_prior_loss else np.zeros(len(idx), int)
        sp, trs = _model_tracks(prob, dtype, W=W, kind=kind.astype(int), a=scale, prior=(idx, mean, L, pk, pscale), cams=bp.cams)
        seen = _compare(prob, dtype, "linear+refine", status, angle, cost, lms_out, trs, sp, 100)
        assert seen > 0.5 * prob.nl


def test_rigs_with_estimated_sensors_against_model():
    cap = synth_rig_capture(3, 12, 200, seed=4)
    prob = cap.prob
    prob.lms = prob.lms + np.random.default_rng(1).normal(0, 0.3, prob.lms.shape)
    import rootba_b200 as rb
    bp = rb.BalProblem.from_arrays(prob, np.float64)
    bp.camera_rig = (cap.rig, cap.cam_from_rig)
    bp.rig_sensor = np.where(cap.sensor == 0, -1, cap.sensor).astype(np.int32)  # sensor 0 held: it carries the rigs' poses
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions())
    lin.download_state()
    tied = BalArrays(np.array(bp.cams), prob.lms, prob.lm_off, prob.obs_cam, prob.obs_xy)
    status, angle, cost = lin.triangulate(max_iterations=100)
    sp, trs = _model_tracks(tied, np.float64)
    assert _compare(tied, np.float64, "linear+refine", status, angle, cost, np.array(bp.lms), trs, sp, 100) > 0.8 * prob.nl
    lin.close()


def _share_from_readback(lin, prob, huber, dtype):
    """each landmark's share of the cost from rba_get_observation_residuals: rho(|W r|^2)/2 of the handle's Huber over the
    observations in use, and its bar: the read-back residual is f rp m - obs in Scalar, so each carries an error of about
    delta = 16 eps_S (|obs| + 1), which moves the share by |r| delta + delta^2 per observation"""
    res, hw, flags = lin.observation_residuals()
    r = np.asarray(res, np.float64)
    s = (r ** 2).sum(1)
    err, _ = olm.loss(olm.HUBER, huber, s)
    err = np.where(flags & 2, err, 0.0)
    delta = 16 * np.finfo(dtype).eps * (np.abs(np.asarray(prob.obs_xy, np.float64)).max(1) + 1)
    share = np.add.reduceat(err, prob.lm_off[:-1])
    return share, np.add.reduceat(np.sqrt(s) * delta + delta * delta, prob.lm_off[:-1]) + 1e-9 * share


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_refinement_lowers_every_cost_and_matches_the_readback(dtype):
    prob = synth_bal(20, 600, 4.0, seed=12, obs_noise=1.0, perturb_lm=0.3)
    huber = 2.0
    import rootba_b200 as rb
    bp = rb.BalProblem.from_arrays(prob, dtype)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(residual=rb.ResidualOptions(robust_norm="HUBER", huber_parameter=huber)))
    e0 = lin.compute_error()["all"]["error"]
    _, _, c0 = lin.triangulate(mode="refine", max_iterations=0)  # no step: the cost at the stored position, nothing written
    assert np.array_equal(np.array(bp.lms), np.asarray(prob.lms, dtype))
    status, _, c1 = lin.triangulate(mode="refine")
    assert np.all(c1 <= c0), np.flatnonzero(c1 > c0)
    assert np.all((status & tm.WRITTEN) == 0) or np.all(c1[(status & tm.WRITTEN) > 0] < c0[(status & tm.WRITTEN) > 0])
    share, bar = _share_from_readback(lin, prob, huber, dtype)
    assert np.all(np.abs(share - c1) <= bar), np.max(np.abs(share - c1) / bar)
    e1 = lin.compute_error()["all"]["error"]
    assert e1 <= e0 * (1 + (1e-6 if dtype == np.float32 else 1e-12))
    assert e1 < e0
    lin.close()


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_bit_identical_across_calls_configurations_and_subsets(classes, dtype):
    outs = []
    for cfg in (dict(), dict(solver_type="SCHUR_COMPLEMENT"), dict(operator_form="IMPLICIT", stage2_form="IDENTITY")):
        for _ in range(2):
            bp, lin = _handle(classes, dtype, **cfg)
            r = lin.triangulate()
            outs.append((np.array(bp.lms),) + r)
            lin.close()
    for o in outs[1:]:
        for a, b in zip(outs[0], o):
            assert np.array_equal(a, b)
    # a subset, in any order: the listed landmarks as in the full call, the others bit-identical
    rng = np.random.default_rng(0)
    sub = rng.permutation(classes.nl)[: classes.nl // 3].astype(np.int32)
    bp, lin = _handle(classes, dtype)
    st, an, co = lin.triangulate(sub)
    lms = np.array(bp.lms)
    lin.close()
    others = np.setdiff1d(np.arange(classes.nl), sub)
    assert np.array_equal(lms[others], np.asarray(classes.lms, dtype)[others])
    assert np.array_equal(lms[sub], outs[0][0][sub])
    assert np.array_equal(st, outs[0][1][sub]) and np.array_equal(an, outs[0][2][sub]) and np.array_equal(co, outs[0][3][sub])


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_protocol_and_rejected_arguments(dtype):
    import ctypes as C
    from rootba_b200.linearizor import _p
    prob = synth_bal(10, 200, 4.0, seed=13, perturb_lm=0.3)
    bp, lin = _handle(prob, dtype)
    lin.linearize()
    lin._backup()
    before = np.array(bp.lms)
    lin.triangulate()
    with pytest.raises(_lib.RbaError) as e:
        lin.solve(1e-4)
    assert e.value.code == -6
    lin._restore()
    lin.download_state()
    assert np.array_equal(np.array(bp.lms), before)
    lin.linearize()
    lin.solve(1e-4)  # re-linearised: the solve runs again
    L = _lib.lib()
    o = _lib.TriangulateOpts()
    L.rba_default_triangulate_opts(C.byref(o))
    assert (o.mode, o.max_iterations, o.min_angle, o.function_tolerance) == (3, 20, 0.0, 1e-10)
    lin.download_state()
    ref = np.array(bp.lms)
    st = np.full(prob.nl, 255, np.uint8)
    idx_ok = np.arange(5, dtype=np.int32)

    def call(opts, num, idx):
        return L.rba_triangulate_landmarks(lin.h, None if opts is None else C.byref(opts), num, None if idx is None else _p(idx),
                                           _p(st), None, None)

    def opts(**kw):
        x = _lib.TriangulateOpts()
        L.rba_default_triangulate_opts(C.byref(x))
        for k, v in kw.items():
            setattr(x, k, v)
        return x

    cases = [(None, prob.nl, None), (opts(mode=0), prob.nl, None), (opts(mode=4), prob.nl, None),
             (opts(max_iterations=-1), prob.nl, None), (opts(min_angle=-1e-3), prob.nl, None),
             (opts(min_angle=float("nan")), prob.nl, None), (opts(function_tolerance=float("inf")), prob.nl, None),
             (opts(function_tolerance=-1.0), prob.nl, None), (opts(), -1, idx_ok), (opts(), prob.nl - 1, None),
             (opts(), 2, np.array([0, prob.nl], np.int32)), (opts(), 2, np.array([-1, 0], np.int32)),
             (opts(), 3, np.array([4, 1, 4], np.int32))]
    for k, (op, num, idx) in enumerate(cases):
        assert call(op, num, idx) == -1, k
        assert np.all(st == 255), k
    lin.download_state()
    assert np.array_equal(np.array(bp.lms), ref)
    lin.solve(1e-4)  # still linearised: nothing changed
    lin.close()


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_lm_run_from_scrambled_landmarks_reaches_the_true_start(dtype):
    import rootba_b200 as rb
    prob = synth_bal(30, 2000, 5.0, seed=14, obs_noise=0.5, perturb_lm=0.0, perturb_rot=0.0, perturb_trans=0.0)
    opts = rb.SolverOptions(max_num_iterations=50, function_tolerance=1e-12)
    bp, lin = _handle(prob, dtype)
    lin.lm_run(50, opts)
    ref = lin.compute_error()["all"]["error"]
    lin.close()
    bad = BalArrays(prob.cams, prob.lms + np.random.default_rng(3).normal(0, 20.0, prob.lms.shape), prob.lm_off, prob.obs_cam,
                    prob.obs_xy)
    bp, lin = _handle(bad, dtype)
    status, _, _ = lin.triangulate()
    assert np.count_nonzero(status & tm.WRITTEN) == prob.nl
    lin.lm_run(50, opts)
    got = lin.compute_error()["all"]["error"]
    lin.close()
    assert abs(got - ref) <= (1e-5 if dtype == np.float32 else 1e-6) * ref, (got, ref)


def test_example_flags(tmp_path):
    prob = synth_bal(10, 300, 4.0, seed=15, perturb_lm=2.0)
    path = str(tmp_path / "problem.txt")
    write_bal(prob, path)
    out = str(tmp_path / "tri.npz")
    cmd = [sys.executable, os.path.join(ROOT, "examples", "solve_bal.py"), path, "--max-num-iterations", "3",
           "--log-path", str(tmp_path / "log.json"), "--triangulate", "linear+refine", "--triangulation", out]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "triangulated (linear+refine)" in r.stdout
    with np.load(out) as f:
        assert f["status"].shape == (prob.nl,) and np.all(f["status"] & tm.WRITTEN) and np.all(f["cost"] >= 0)
    r = subprocess.run(cmd[:-4] + ["--triangulation", out], capture_output=True, text=True, timeout=300)
    assert r.returncode != 0 and "--triangulation requires --triangulate" in r.stderr


@pytest.mark.parametrize("sfx", ["f32", "f64"])
def test_two_ranks_union_equals_single_rank(tmp_path, sfx):
    res = oc.run_two_ranks(tmp_path, "multirank_triangulation_worker.py", sfx, "1", 33700, 53 + (31 if sfx == "f32" else 0))
    assert res["covers_own_shard_only"] and res["lms_identical"] and all(res["outputs_identical"]), res
    assert res["written"] > 0
