"""Marginal covariances (rba_compute_covariance, DESIGN.md section 16) on the GPU against the float64 inverse of J^T J of the
total objective: every solver configuration in both precisions (bit-identical within one), pair and absolute priors, held
parameters, a gauge fixed by held poses only, Huber weights, dropped invalid observations, a rank-2 landmark, the dense
kernels at 500 cameras and below one tile, singular systems, and the absence of side effects.

Bars are c * kappa * u with u the float64 unit roundoff and kappa the condition number of the Jacobi-equilibrated matrix
the test inverts; c = 8 * (number of unknowns) covers the rounding of the Cholesky-based inverse on both sides.  A float32
handle is compared with the reference at its float32 state and prior arrays, the rotation matrices built from the stored
quaternions as the kernels build them (camera_model.rotation(device=True)): the device widens those values to float64 and
computes in float64, so the float32 bars are the float64 ones.  Larger shapes, long tracks, the benchmark size and large
prior rotations are in test_gpu_covariance_shapes.py."""


import numpy as np
import pytest

import camera_model as cm
import camera_prior_model as pm
import covariance_model as cvm
import pair_prior_model as qm
from objective_checks import CONFIGS, MASK
from rootba_b200._lib import RBA_NUMERICAL_FAILURE

pytestmark = pytest.mark.gpu

U = 2.0 ** -53


_centre_priors = cvm.centre_priors


def _dense(prob, absp=None, pair=None, threshold=None, valid_only=False, dtype=np.float64):
    """[Jp | Jl] of the total objective: weighted reprojection rows (camera_model), absolute and pair prior rows, rotations
    as the kernels build them; `dtype` is the handle's (its validity threshold)"""
    nobs, nc, nl = len(prob.obs_cam), len(prob.cams), len(prob.lm_off) - 1
    jp, jl, _, _ = cm.weighted(prob, dtype=dtype, threshold=threshold, valid_only=valid_only, device_rot=True)
    Jp, Jl = np.zeros((2 * nobs, 9 * nc)), np.zeros((2 * nobs, 3 * nl))
    lm_of_obs = np.repeat(np.arange(nl), np.diff(prob.lm_off))
    for k in range(nobs):
        c, l = int(prob.obs_cam[k]), int(lm_of_obs[k])
        Jp[2 * k:2 * k + 2, 9 * c:9 * c + 9] = jp[k]
        Jl[2 * k:2 * k + 2, 3 * l:3 * l + 3] = jl[k]
    rows = [Jp]
    if absp is not None:
        A, _ = pm.rows(np.asarray(prob.cams, np.float64), *absp, device_rot=True)
        Ja = np.zeros((9 * nc, 9 * nc))
        for c in range(nc):
            Ja[9 * c:9 * c + 9, 9 * c:9 * c + 9] = A[c]
        rows.append(Ja)
    if pair is not None:
        Jq, _ = qm.rows(np.asarray(prob.cams, np.float64), *pair, device_rot=True)
        rows.append(Jq)
    Jp = np.vstack(rows)
    return Jp, np.vstack([Jl, np.zeros((Jp.shape[0] - Jl.shape[0], Jl.shape[1]))])


def _handle(prob, dtype, cfg=None, absp=None, pair=None, mask=None, **so_kw):
    import rootba_b200 as rb
    bp = rb.BalProblem.from_arrays(prob, dtype)
    if absp is not None:
        bp.camera_prior = absp
    if pair is not None:
        bp.camera_pair_prior = pair
    if mask is not None:
        bp.camera_fixed = mask
    return rb.LinearizorQR.create(bp, rb.SolverOptions(**(cfg or {}), **so_kw))


def _check(cam, lm, prob, dtype, absp=None, pair=None, mask=None, threshold=None, valid_only=False):
    nc, nl = len(prob.cams), len(prob.lm_off) - 1
    prob, absp, pair = cvm.as_stored(prob, dtype, absp, pair)
    Jp, Jl = _dense(prob, absp, pair, threshold, valid_only, dtype)
    fixed = cvm.fixed_mask(mask, nc)
    cam_ref, lm_ref, kappa = cvm.dense_inverse(Jp, Jl, nc, nl, fixed)
    bar = 8 * (int((~fixed).sum()) + 3 * nl) * kappa * U
    assert np.abs(cam - cam_ref).max() <= bar * np.abs(cam_ref).max(), (np.abs(cam - cam_ref).max() / np.abs(cam_ref).max(), bar)
    if lm is not None:
        assert np.abs(lm - lm_ref).max() <= bar * np.abs(lm_ref).max(), (np.abs(lm - lm_ref).max() / np.abs(lm_ref).max(), bar)
    if mask is not None:
        c2 = cam.reshape(nc, 9, 9)
        for c in range(nc):
            f = fixed[9 * c:9 * c + 9]
            assert (c2[c][f, :] == 0).all() and (c2[c][:, f] == 0).all()
    return kappa


def _case(nc, nl, seed):
    from rootba_b200.synthetic import synth_bal
    prob = synth_bal(nc, nl, 3.6, seed=seed)
    return prob, _centre_priors(prob, seed)


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("size", [(7, 90, 21), (120, 500, 5)], ids=["nc7", "nc120"])
def test_every_configuration_against_dense_inverse(size, dtype):
    prob, absp = _case(*size)
    first = None
    for cfg in CONFIGS:
        lin = _handle(prob, dtype, cfg, absp=absp)
        cam, lm = lin.covariance()
        lin.close()
        if first is None:
            first = (cam, lm)
            _check(cam, lm, prob, dtype, absp=absp)
        else:  # the result does not depend on the solver: bit-identical
            assert np.array_equal(cam, first[0]) and np.array_equal(lm, first[1]), cfg


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
def test_pair_and_absolute_priors(dtype):
    prob, pair = qm.pair_case(7, 90)  # + camera 7 without observations, tied to camera 0 by a pair prior
    absp = _centre_priors(prob, 9)
    absp[1][-1] = pm.sqrt_info_kind("dense", np.random.default_rng(9))  # its intrinsics need a prior
    lin = _handle(prob, dtype, absp=absp, pair=pair)
    cam, lm = lin.covariance()
    lin.close()
    _check(cam, lm, prob, dtype, absp=absp, pair=pair)


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
def test_held_parameters(dtype):
    prob, absp = _case(7, 90, 21)
    lin = _handle(prob, dtype, absp=absp, mask=MASK)
    cam, lm = lin.covariance()
    lin.close()
    _check(cam, lm, prob, dtype, absp=absp, mask=MASK)
    assert (cam[3] == 0).all()  # camera 3 is held entirely


def test_gauge_fixed_by_two_held_poses():
    import rootba_b200 as rb
    prob, _ = _case(7, 90, 21)
    mask = np.zeros(7, np.uint8)
    mask[[0, 4]] = rb.FIX_POSE
    lin = _handle(prob, np.float64, mask=mask)
    cam, lm = lin.covariance()
    lin.close()
    _check(cam, lm, prob, np.float64, mask=mask)


def test_huber_with_active_weights():
    _huber_with_active_weights(np.float64)


def test_huber_with_active_weights_float32():
    _huber_with_active_weights(np.float32)


def _huber_with_active_weights(dtype):
    prob, absp = _case(7, 90, 21)
    L = cm.linearize(*cm.observations(prob))
    rn = np.sqrt((L["res"] ** 2).sum(1))
    th = float(np.median(rn))
    assert (rn > th).sum() > 10
    from rootba_b200.linearizor import ResidualOptions
    lin = _handle(prob, dtype, absp=absp, residual=ResidualOptions("HUBER", th))
    cam, lm = lin.covariance()
    lin.close()
    _check(cam, lm, prob, dtype, absp=absp, threshold=th)


def _turned():
    """10 cameras, camera 0 turned around (its observations are invalid); landmark 0 is seen by cameras 0 and 5 only"""
    from rootba_b200.synthetic import synth_bal, turn_cameras_around
    rng = np.random.default_rng(5)
    tracks = [np.array([0, 5])] + [rng.choice(np.arange(1, 10), int(rng.integers(2, 6)), replace=False) for _ in range(120)]
    a = synth_bal(10, len(tracks), 0.0, seed=6, tracks=tracks, lm_spread=0.5)
    return turn_cameras_around(a, [0])


def _with_shallow_observation(prob, depth=1e-3):
    """prob + one landmark seen by camera 1 at `depth` in front of it (between float64's validity threshold sqrt(1e-10)
    and float32's sqrt(1e-5)) and by every other camera 2..9 that has it at least 1 in front"""
    from rootba_b200.synthetic import BalArrays
    cams = np.asarray(prob.cams, np.float64)
    R1 = cm.rotation(cams[1, :4])
    p = R1.T @ (np.array([0.1, -0.1, 1.0]) * depth - cams[1, 4:7])
    z = np.einsum("mij,j->mi", cm.rotation(cams[:, :4]), p)[:, 2] + cams[:, 6]
    obs_cam = np.array([1] + [c for c in range(2, len(cams)) if z[c] >= 1.0], np.int32)
    assert len(obs_cam) >= 3
    proj = cm.linearize(cams[obs_cam], np.broadcast_to(p, (len(obs_cam), 3)), np.zeros((len(obs_cam), 2)))["res"]
    xy = proj + np.random.default_rng(8).normal(0, 0.5, proj.shape)
    return BalArrays(cams, np.vstack([prob.lms, p]), np.append(prob.lm_off, prob.lm_off[-1] + len(obs_cam)),
                     np.concatenate([prob.obs_cam, obs_cam]), np.vstack([prob.obs_xy, xy]))


def test_invalid_observations_dropped_and_rank2_landmark():
    _invalid_observations_dropped_and_rank2_landmark(np.float64)


def test_invalid_observations_dropped_and_rank2_landmark_float32():
    _invalid_observations_dropped_and_rank2_landmark(np.float32)


def _invalid_observations_dropped_and_rank2_landmark(dtype):
    """use_valid_projections_only (optimized_cost ERROR_VALID): camera 0's rows are zero, so it is held by its prior alone;
    landmark 0 keeps one valid observation: NaN block, cameras against the pinv elimination.  The float32 handle also holds
    an observation at depth 1e-3, which float32's validity threshold (the one the handle's own scalar uses) drops and
    float64's would keep."""
    prob = _turned()
    if dtype == np.float32:
        prob = _with_shallow_observation(prob)
    absp = _centre_priors(prob, 4)
    absp[1][0] = pm.sqrt_info_kind("dense", np.random.default_rng(1))  # camera 0 has no valid observation
    nc, nl = len(prob.cams), len(prob.lm_off) - 1
    lin = _handle(prob, dtype, absp=absp, optimized_cost="ERROR_VALID")
    cam, lm = lin.covariance()
    lin.close()
    assert np.isnan(lm[0]).all() and np.isfinite(lm[1:]).all()
    sprob, sabsp, _ = cvm.as_stored(prob, dtype, absp)
    jp, jl, _, keep = cm.weighted(sprob, dtype=dtype, valid_only=True, device_rot=True)
    assert keep.sum() < len(keep) and keep[prob.lm_off[0]:prob.lm_off[1]].sum() == 1
    if dtype == np.float32:
        _, _, _, keep64 = cm.weighted(sprob, dtype=np.float64, valid_only=True, device_rot=True)
        assert not keep[prob.lm_off[-2]] and keep64[prob.lm_off[-2]] and (keep64 != keep).sum() == 1
    S = cvm.schur_reduced(jp, jl, np.asarray(prob.obs_cam), np.asarray(prob.lm_off), nc)
    A, _ = pm.rows(np.asarray(sprob.cams, np.float64), *sabsp, device_rot=True)
    for c in range(nc):
        S[9 * c:9 * c + 9, 9 * c:9 * c + 9] += A[c].T @ A[c]
    d = 1 / np.sqrt(np.diag(S))
    kappa = cvm.spd_cond(S * d[:, None] * d[None, :])
    ref = np.linalg.inv(S)
    ref_cam = np.stack([ref[9 * c:9 * c + 9, 9 * c:9 * c + 9] for c in range(nc)])
    assert np.abs(cam - ref_cam).max() <= 8 * 9 * nc * kappa * U * np.abs(ref_cam).max()
    # the other landmarks against the model's elimination formula (the pinv form for landmark 0)
    P = np.zeros_like(S)
    for c in range(nc):
        P[9 * c:9 * c + 9, 9 * c:9 * c + 9] = A[c].T @ A[c]
    _, lm_m = cvm.eigen_form(jp, jl, np.asarray(prob.obs_cam), np.asarray(prob.lm_off), nc, P)
    assert np.abs(lm[1:] - lm_m[1:]).max() <= 8 * (9 * nc + 3 * nl) * kappa * U * np.abs(lm_m[1:]).max()


@pytest.mark.parametrize("nc, nl", [(500, 5000), (2, 40), (7, 90)], ids=["nc500", "nc2", "nc7"])
def test_dense_kernels_against_schur_reduced(nc, nl):
    """N = 4500 (not a multiple of the 64 tile), N = 18 and N = 63 (below one tile).  One camera cannot hold a landmark (a
    landmark needs two observations by distinct cameras), so two is the smallest problem.  Every camera and landmark block
    is also compared componentwise with the vectorised reference (covariance_model.check)."""
    from rootba_b200.synthetic import synth_bal
    prob = synth_bal(nc, nl, 4.1 if nc > 2 else 2.0, seed=11)
    absp = _centre_priors(prob, 12)
    if nc == 2:
        absp[1][:] = pm.sqrt_info_kind("dense", np.random.default_rng(2))
    lin = _handle(prob, np.float64, absp=absp)
    cam, _ = lin.covariance(landmarks=False)
    cam2, lm2 = lin.covariance()
    lin.close()
    assert np.array_equal(cam, cam2)
    jp, jl, _, _ = cm.weighted(prob)
    S = cvm.schur_reduced(jp, jl, np.asarray(prob.obs_cam), np.asarray(prob.lm_off), nc)
    A, _ = pm.rows(np.asarray(prob.cams, np.float64), *absp)
    for c in range(nc):
        S[9 * c:9 * c + 9, 9 * c:9 * c + 9] += A[c].T @ A[c]
    d = 1 / np.sqrt(np.diag(S))
    kappa = cvm.spd_cond(S * d[:, None] * d[None, :])
    ref = np.linalg.inv(S)
    ref_cam = np.stack([ref[9 * c:9 * c + 9, 9 * c:9 * c + 9] for c in range(nc)])
    assert np.abs(cam - ref_cam).max() <= 8 * 9 * nc * kappa * U * np.abs(ref_cam).max()
    assert np.isfinite(lm2).all()
    cvm.check(cam2, lm2, cvm.reference(prob, absp=absp), what=f"nc {nc}")


@pytest.mark.parametrize("size", [(7, 90, 21), (120, 500, 5)], ids=["nc7", "nc120"])
def test_gauge_not_fixed(size):
    import rootba_b200 as rb
    from rootba_b200.synthetic import synth_bal
    prob = synth_bal(size[0], size[1], 3.6, seed=size[2])
    lin = _handle(prob, np.float64)
    with pytest.raises(rb.RbaError) as e:
        lin.covariance()
    assert e.value.code == RBA_NUMERICAL_FAILURE and "camera" in str(e.value) and "rba_set_camera_prior" in str(e.value)
    lin.set_camera_prior(_centre_priors(prob))
    cam, lm = lin.covariance()
    assert np.isfinite(cam).all() and np.isfinite(lm).all()
    lin.close()


def test_free_camera_without_observations():
    import rootba_b200 as rb
    prob, _, _ = pm.prior_case(7, 90)  # camera 7 has no observation
    mean, L = _centre_priors(prob)
    L[-1] = 0.0
    lin = _handle(prob, np.float64, absp=(mean, L))
    with pytest.raises(rb.RbaError) as e:
        lin.covariance()
    assert e.value.code == RBA_NUMERICAL_FAILURE and "camera 7" in str(e.value)
    L[-1] = pm.sqrt_info_kind("dense", np.random.default_rng(0))
    lin.set_camera_prior((mean, L))
    cam, lm = lin.covariance()
    lin.close()
    _check(cam, lm, prob, np.float64, absp=(mean, L))


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
def test_no_side_effects(dtype):
    prob, absp = _case(49, 1800, 38401)
    a = _handle(prob, dtype, absp=absp)
    b = _handle(prob, dtype, absp=absp)
    c1 = a.covariance()
    c2 = a.covariance()
    assert np.array_equal(c1[0], c2[0]) and np.array_equal(c1[1], c2[1])
    ia, _, _ = a.lm_run(2)
    a.covariance()
    ja, _, _ = a.lm_run(2)
    ib, _, _ = b.lm_run(2)
    jb, _, _ = b.lm_run(2)
    strip = lambda its: [{k: v for k, v in it.items() if k != "device_seconds"} for it in its]
    assert strip(ia + ja) == strip(ib + jb)
    for lin in (a, b):
        lin.download_state()
    assert np.array_equal(a.bal_problem.cams, b.bal_problem.cams) and np.array_equal(a.bal_problem.lms, b.bal_problem.lms)
    # the device-resident increment survives the call
    for lin in (a, b):
        lin.linearize()
        lin.solve(1e-3, to_host=False)
    a.covariance(landmarks=False)
    la, lb = a.apply(None), b.apply(None)
    assert la == lb
    for lin in (a, b):
        lin.download_state()
    assert np.array_equal(a.bal_problem.cams, b.bal_problem.cams) and np.array_equal(a.bal_problem.lms, b.bal_problem.lms)
    assert a.timings()["kernel_launches"] == b.timings()["kernel_launches"]
    a.close()
    b.close()


def test_unsupported_and_invalid():
    import rootba_b200 as rb
    from rootba_b200 import _lib
    prob, absp = _case(7, 90, 21)
    lin = _handle(prob, np.float64, absp=absp)
    assert _lib.lib().rba_compute_covariance(lin.h, None, None) == -1
    lin.close()
    lin = _handle(prob, np.float64, absp=absp, nranks=2, rank=0)  # no communicator is made before rba_comm_init
    with pytest.raises(rb.RbaError) as e:
        lin.covariance()
    assert e.value.code == -4 and "nranks" in str(e.value)
    lin.close()
