"""Marginal covariances (rba_compute_covariance, DESIGN.md section 16) against the float64 reference of
tests/covariance_model.py at the shapes where the dense kernels go wrong: every tile pair of the blocked inverse read by some
landmark, N a multiple of the 64 tile and not (paddings 0, 1, 2, 57, 63), tracks longer than a warp (up to 300 cameras), the
benchmark stand-in (N = 15 507), prior rotations up to pi through both series branches and the w < 0 flip, a state moved
by lm_run, by new priors and held flags and by restore, and a matrix larger than the device.

Every camera block and every landmark block is compared componentwise (covariance_model.check): an entry of a camera block
against c N kappa u sigma_i sigma_j, a landmark block against c (N kappa + n_l kappa_l) u |W| (I + g g^T) |W|^T (g =
sum_a |K_a| sigma_a, n_l its track length), c = 8, kappa the dpocon estimate of the equilibrated reduced matrix, kappa_l that of the landmark's Hll, sigma the
square roots of the reference inverse's diagonal.  Each bar is asserted to be <= 1e-4 and printed in the assertion message.
A float32 handle is compared with the reference at its stored (float32) state, rotations built from the stored quaternions
as the kernels build them: its covariance is computed in float64 from those values, so the bars are the same."""
import importlib.util
import os
import re

import numpy as np
import pytest

import camera_prior_model as pm
import covariance_model as cvm
import pair_prior_model as qm
from conftest import ROOT

pytestmark = pytest.mark.gpu

TILE_SHAPES = [14, 15, 57, 64, 71, 128]
# N = 9 nc and its padding to the 64 tile: 126 (2), 135 (57), 513 (63), 576 (0), 639 (1), 1152 (0)
assert {(-9 * nc) % cvm.TILE for nc in TILE_SHAPES} == {0, 1, 2, 57, 63}


def _handle(prob, dtype, absp=None, pair=None, mask=None, **so_kw):
    import rootba_b200 as rb
    bp = rb.BalProblem.from_arrays(prob, dtype)
    if absp is not None:
        bp.camera_prior = absp
    if pair is not None:
        bp.camera_pair_prior = pair
    if mask is not None:
        bp.camera_fixed = mask
    return rb.LinearizorQR.create(bp, rb.SolverOptions(use_double=dtype == np.float64, **so_kw))


def _state(lin):
    """a float64 copy of the handle's current state as BalArrays"""
    from rootba_b200.synthetic import BalArrays
    lin.download_state()
    bp = lin.bal_problem
    return BalArrays(np.array(bp.cams, np.float64), np.array(bp.lms, np.float64), bp.lm_off, bp.obs_cam, bp.obs_xy)


@pytest.mark.parametrize("dtype, nc", [(np.float64, nc) for nc in TILE_SHAPES] + [(np.float32, 64), (np.float32, 128)],
                         ids=[f"f64-nc{nc}" for nc in TILE_SHAPES] + ["f32-nc64", "f32-nc128"])
def test_every_tile_of_the_inverse(nc, dtype):
    prob, absp = cvm.tile_case(nc, nc)
    assert cvm.tile_pairs_read(prob.obs_cam, prob.lm_off) == cvm.all_tile_pairs(nc)  # every tile pair is read
    assert cvm.straddling_cameras(nc)  # some camera block crosses a tile boundary
    lin = _handle(prob, dtype, absp=absp)
    cam, lm = lin.covariance()
    lin.close()
    cvm.check(cam, lm, cvm.reference(prob, dtype, absp=absp), what=f"nc {nc}")


LONG = [2, 3, 31, 32, 33, 63, 64, 65, 150, 300]


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
def test_long_tracks(dtype):
    """N = 2880 (45 tiles, no padding); landmarks on n = 2 .. 300 named cameras: the warp loops over a track's slots make
    up to 10 passes and the marginal up to 90 000 camera pairs per landmark"""
    from rootba_b200.synthetic import synth_bal
    nc = 320
    rng = np.random.default_rng(17)
    tracks = [rng.choice(nc, n, replace=False) for n in LONG]
    tracks += [rng.choice(nc, int(rng.integers(2, 7)), replace=False) for _ in range(3000)]
    prob = synth_bal(nc, len(tracks), 0.0, seed=18, tracks=tracks, lm_spread=0.5)
    assert np.array_equal(np.diff(prob.lm_off)[:len(LONG)], LONG)
    absp = cvm.centre_priors(prob, 19)
    lin = _handle(prob, dtype, absp=absp)
    cam, lm = lin.covariance()
    lin.close()
    cvm.check(cam, lm, cvm.reference(prob, dtype, absp=absp), what="long tracks")


def _bench_priors():
    spec = importlib.util.spec_from_file_location("bench_camera_priors", os.path.join(ROOT, "scripts", "bench_camera_priors.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.camera_centre_priors


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_benchmark_size(dtype):
    """the set-up of scripts/bench_covariance.py (ladybug-1723 stand-in, seed 38401, centre priors, 10 LM steps): all 1723
    camera blocks and all 151 500 landmark blocks against the reference at the state the LM run reached"""
    from rootba_b200.synthetic import synth_config
    arrays = synth_config("ladybug-1723", seed=38401)
    absp = _bench_priors()(arrays)
    lin = _handle(arrays, dtype, absp=absp)
    lin.lm_run(10)
    cam, lm = lin.covariance()
    state = _state(lin)
    lin.close()
    ref = cvm.reference(state, dtype, absp=absp)
    cvm.check(cam, lm, ref, what=f"ladybug-1723 {np.dtype(dtype).name}")


def _rotation_case(seed=61):
    """7 observed cameras with centre priors, then for every angle of ROTATION_ANGLES and both signs of the mean: one
    camera held by a dense absolute prior only, whose rotation is that angle from the mean's, and one with a dense pair prior
    to an observed camera (the pair mean that angle from their relative rotation) and a dense absolute prior at angle 0"""
    from scipy.spatial.transform import Rotation
    from rootba_b200.synthetic import BalArrays, synth_bal
    base = synth_bal(7, 90, 3.6, seed=seed)
    rng = np.random.default_rng(seed)
    cases = [(th, neg) for th in pm.ROTATION_ANGLES for neg in (False, True)]
    extra = []
    for _ in range(2 * len(cases)):
        c = np.asarray(base.cams[0], np.float64).copy()
        c[:4] = Rotation.from_rotvec(rng.uniform(-2, 2, 3)).as_quat()
        c[4:7] += rng.normal(0, 0.5, 3)
        extra.append(c)
    cams = np.vstack([np.asarray(base.cams, np.float64), extra])
    prob = BalArrays(cams, base.lms, base.lm_off, base.obs_cam, base.obs_xy)
    mean, L = cvm.centre_priors(prob, seed)
    pairs, qmean, qL = [], [], []
    for k, (th, neg) in enumerate(cases):
        a = 7 + k  # absolute prior only
        mean[a, :4] = pm.mean_at_angle(cams[a], th, 1000 + k, neg)
        L[a] = pm.sqrt_info_kind("dense", rng)
        b, o = 7 + len(cases) + k, k % 7  # + a pair prior to observed camera o
        L[b] = pm.sqrt_info_kind("dense", rng)  # its own rotation residual is 0: the pair carries the angle
        m = qm.mean_at(cams, np.array([[b, o]]))[0]
        m[:4] = pm.mean_at_angle(m, th, 2000 + k, neg)
        pairs.append((b, o))
        qmean.append(m)
        qL.append(qm.sqrt_info_kind("dense", rng))
    return prob, (mean, L), (np.asarray(pairs, np.int32), np.stack(qmean), np.stack(qL))


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
def test_large_prior_rotations(dtype):
    prob, absp, pair = _rotation_case()
    angles = np.repeat(pm.ROTATION_ANGLES, 2)
    n = len(angles)
    for k in range(n):
        assert abs(np.linalg.norm(pm.residual(prob.cams[7 + k], absp[0][7 + k])[3:6]) - angles[k]) <= 1e-9
        (b, o), m = pair[0][k], pair[1][k]
        assert abs(np.linalg.norm(qm.residual(prob.cams[b], prob.cams[o], m)[3:6]) - angles[k]) <= 1e-9
    lin = _handle(prob, dtype, absp=absp, pair=pair)
    cam, lm = lin.covariance()
    lin.close()
    cvm.check(cam, lm, cvm.reference(prob, dtype, absp=absp, pair=pair), what="large prior rotations")


@pytest.mark.parametrize("cfg", [{}, dict(solver_type="POWER_SCHUR_COMPLEMENT")], ids=["default", "power-sc"])
@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
def test_large_prior_rotations_through_the_solve(cfg, dtype):
    """scaling, b, the preconditioner blocks, the operator, the increment, l_diff and the cost of one LM step with the same
    priors, by objective_checks.check_against_dense as test_gpu_camera_priors / test_gpu_pair_priors call it"""
    from objective_checks import check_against_dense
    prob, absp, pair = _rotation_case()
    check_against_dense(cfg, prob, camera=absp, dtype=dtype)
    check_against_dense(cfg, prob, camera=absp, pairs=pair, dtype=dtype, inc_eta_kappa=True)


def test_moved_state():
    """one handle: after lm_run, after new absolute and pair priors and held flags on the live handle, and after
    backup / lm_run / restore, the covariance is that of the state and priors of that moment"""
    import rootba_b200 as rb
    prob, absp = cvm.tile_case(15, 77)
    rng = np.random.default_rng(78)
    pairs = np.array([[1, 0], [5, 9], [14, 3]], np.int32)
    pair = (pairs, qm.mean_at(prob.cams, pairs), np.stack([qm.sqrt_info_kind("dense", rng) for _ in pairs]))
    lin = _handle(prob, np.float64, absp=absp, pair=pair)
    cam0, lm0 = lin.covariance()
    cvm.check(cam0, lm0, cvm.reference(prob, absp=absp, pair=pair), what="initial")
    lin.lm_run(5)
    state = _state(lin)
    assert not np.array_equal(state.cams, prob.cams)
    cam1, lm1 = lin.covariance()
    cvm.check(cam1, lm1, cvm.reference(state, absp=absp, pair=pair), what="after lm_run")
    absp2 = cvm.centre_priors(state, 79)
    absp2[1][2] = pm.sqrt_info_kind("dense", rng)
    pair2 = (pairs[:2], qm.mean_at(state.cams, pairs[:2]), np.stack([qm.sqrt_info_kind("rotation", rng) for _ in range(2)]))
    mask = np.zeros(15, np.uint8)
    mask[4] = rb.FIX_POSE
    lin.set_camera_prior(absp2)
    lin.set_camera_pair_prior(pair2)
    lin.set_camera_fixed(mask)
    cam2, lm2 = lin.covariance()
    ref2 = cvm.reference(state, absp=absp2, pair=pair2, mask=mask)
    cvm.check(cam2, lm2, ref2, what="new priors and held flags")
    assert (cam2[4][:6, :] == 0).all() and (cam2[4][:, :6] == 0).all()
    lin.bal_problem.backup()
    lin.linearize()
    lin.solve(1e-3, to_host=False)
    lin.apply(None)
    assert not np.array_equal(_state(lin).cams, state.cams)
    lin.bal_problem.restore()
    assert np.array_equal(_state(lin).cams, state.cams)
    cam3, lm3 = lin.covariance()
    assert np.array_equal(cam3, cam2) and np.array_equal(lm3, lm2)
    lin.close()


def test_matrix_larger_than_the_device():
    """13 682 cameras: the dense float64 matrix alone (N = 123 138) is 121 GB, above an 80 GB card: RBA_ERR_UNSUPPORTED with
    the byte count, the output arrays untouched, and the handle's solve afterwards bit-identical to a fresh handle's"""
    from rootba_b200 import _lib
    from rootba_b200.synthetic import synth_bal
    nc = 13682
    prob = synth_bal(nc, 4000, 3.6, seed=5)
    rng = np.random.default_rng(6)
    mean = pm.mean_at(np.asarray(prob.cams, np.float64))
    L = np.broadcast_to(pm.sqrt_info_kind("dense", rng), (nc, 9, 9)).copy()
    a = _handle(prob, np.float64, absp=(mean, L))
    cam = np.full((nc, 9, 9), 7.25)
    lm = np.full((a.nl, 3, 3), -3.5)
    rc = _lib.lib().rba_compute_covariance(a.h, cam.ctypes.data, lm.ctypes.data)
    msg = (_lib.lib().rba_last_error() or b"").decode()
    assert rc == -4, (rc, msg)
    got = re.search(r"needs (\d+) bytes", msg)
    assert got and int(got.group(1)) >= (9 * nc) ** 2 * 8 and "123138 x 123138" in msg, msg
    assert (cam == 7.25).all() and (lm == -3.5).all()
    b = _handle(prob, np.float64, absp=(mean, L))
    out = []
    for lin in (a, b):
        lin.linearize()
        inc = lin.solve(1e-3)
        out.append((inc, lin.get_rhs(), lin.apply(None)))
        lin.close()
    assert np.array_equal(out[0][0], out[1][0]) and np.array_equal(out[0][1], out[1][1]) and out[0][2] == out[1][2]
