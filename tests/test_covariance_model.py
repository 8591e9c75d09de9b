"""CPU checks of the covariance model (tests/covariance_model.py): the eigen-form elimination the device evaluates equals the
blocks of the full inverse of J^T J, and with a rank-deficient landmark it equals the reduced matrix built with pinv."""
import numpy as np
import pytest

import covariance_model as cvm
import camera_model as cm
import camera_prior_model as pm
from scipy.spatial.transform import Rotation


def _random_instance(rng, nc, nl, deficient=()):
    """random per-observation blocks: every landmark on 2..4 cameras (ascending), landmarks in `deficient` with one
    observation zeroed (rank 2); plus an identity prior on every camera parameter so that H is regular"""
    obs_cam, lm_off = [], [0]
    for l in range(nl):
        n = int(rng.integers(2, min(nc, 4) + 1))
        obs_cam += sorted(rng.choice(nc, n, replace=False).tolist())
        lm_off.append(len(obs_cam))
    obs_cam, lm_off = np.asarray(obs_cam), np.asarray(lm_off)
    jp = rng.normal(size=(len(obs_cam), 2, 9))
    jl = rng.normal(size=(len(obs_cam), 2, 3))
    for l in deficient:
        jp[lm_off[l]] = 0.0
        jl[lm_off[l]] = 0.0
    return jp, jl, obs_cam, lm_off


def _dense(jp, jl, obs_cam, lm_off, nc, prior):
    nl, nobs = len(lm_off) - 1, len(obs_cam)
    lm_of_obs = np.repeat(np.arange(nl), np.diff(lm_off))
    Jp = np.zeros((2 * nobs + 9 * nc, 9 * nc))
    Jl = np.zeros((2 * nobs + 9 * nc, 3 * nl))
    for k in range(nobs):
        Jp[2 * k:2 * k + 2, 9 * obs_cam[k]:9 * obs_cam[k] + 9] = jp[k]
        Jl[2 * k:2 * k + 2, 3 * lm_of_obs[k]:3 * lm_of_obs[k] + 3] = jl[k]
    Jp[2 * nobs:] = prior
    return Jp, Jl


@pytest.mark.parametrize("seed", range(6))
def test_eigen_form_equals_full_inverse(seed):
    rng = np.random.default_rng(seed)
    nc, nl = int(rng.integers(2, 6)), int(rng.integers(3, 12))
    jp, jl, obs_cam, lm_off = _random_instance(rng, nc, nl)
    A = rng.normal(size=(9 * nc, 9 * nc)) * 0.3 + np.eye(9 * nc)
    Jp, Jl = _dense(jp, jl, obs_cam, lm_off, nc, A)
    cam_ref, lm_ref, kappa = cvm.dense_inverse(Jp, Jl, nc, nl)
    cam, lm = cvm.eigen_form(jp, jl, obs_cam, lm_off, nc, A.T @ A)
    bar = 64 * (9 * nc + 3 * nl) * kappa * 2.0 ** -53
    assert np.abs(cam - cam_ref).max() <= bar * np.abs(cam_ref).max()
    assert np.abs(lm - lm_ref).max() <= bar * np.abs(lm_ref).max()


@pytest.mark.parametrize("seed", range(4))
def test_pseudo_inverse_form_with_rank_deficient_landmark(seed):
    rng = np.random.default_rng(100 + seed)
    nc, nl = 4, 8
    jp, jl, obs_cam, lm_off = _random_instance(rng, nc, nl, deficient=(0, 3))
    A = rng.normal(size=(9 * nc, 9 * nc)) * 0.3 + np.eye(9 * nc)
    S = cvm.schur_reduced(jp, jl, obs_cam, lm_off, nc) + A.T @ A
    ref = np.linalg.inv(S)
    cam, lm = cvm.eigen_form(jp, jl, obs_cam, lm_off, nc, A.T @ A)
    bar = 64 * 9 * nc * np.linalg.cond(S) * 2.0 ** -53
    for c in range(nc):
        blk = ref[9 * c:9 * c + 9, 9 * c:9 * c + 9]
        assert np.abs(cam[c] - blk).max() <= bar * np.abs(ref).max()
    n_obs = np.diff(lm_off)
    for l in range(nl):
        # a deficient landmark with 2 observations keeps one: rank 2, NaN; with more it keeps rank 3 (generic)
        if l in (0, 3) and n_obs[l] == 2:
            assert np.isnan(lm[l]).all()
        else:
            assert np.isfinite(lm[l]).all()
    # the pinv elimination is the limit of a vanishing landmark prior: eps I on every Hll
    eps = 1e-7
    Jp, Jl = _dense(jp, jl, obs_cam, lm_off, nc, A)
    J = np.hstack([Jp, Jl])
    H = J.T @ J
    H[9 * nc:, 9 * nc:] += eps * np.eye(3 * nl)
    lim = np.linalg.inv(H)[:9 * nc, :9 * nc]
    assert np.abs(lim - ref).max() <= 1e-4 * np.abs(ref).max()


# ------------------------------------------------------------------------------------------------
# the vectorised reference against the loop versions
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(6))
def test_vectorised_reference_equals_loop_reference(seed):
    """eigen_reduced + landmark_marginal against schur_reduced / eigen_form, with rank-deficient landmarks"""
    rng = np.random.default_rng(200 + seed)
    nc, nl = int(rng.integers(3, 8)), int(rng.integers(10, 30))
    jp, jl, obs_cam, lm_off = _random_instance(rng, nc, nl, deficient=(0, 3))
    jl[lm_off[5] + 1:lm_off[6]] = 0.0  # landmark 5 keeps one observation's Jl: rank 2
    A = rng.normal(size=(9 * nc, 9 * nc)) * 0.3 + np.eye(9 * nc)
    S, K, W, rank, _ = cvm.eigen_reduced(jp, jl, obs_cam, lm_off, nc, A.T @ A)
    S_loop = cvm.schur_reduced(jp, jl, obs_cam, lm_off, nc) + A.T @ A
    assert np.abs(S - S_loop).max() <= 1e-12 * np.abs(S_loop).max()
    assert np.array_equal(S, S.T)
    cam_loop, lm_loop = cvm.eigen_form(jp, jl, obs_cam, lm_off, nc, A.T @ A)
    Sig = np.linalg.inv(S)
    cam = np.stack([Sig[9 * c:9 * c + 9, 9 * c:9 * c + 9] for c in range(nc)])
    lm = cvm.landmark_marginal(Sig, K, W, rank, obs_cam, lm_off, chunk=7)  # small chunks: several per track length
    assert np.abs(cam - cam_loop).max() <= 1e-12 * np.abs(cam_loop).max()
    assert np.array_equal(np.isnan(lm), np.isnan(lm_loop)) and np.isnan(lm).any()
    ok = ~np.isnan(lm_loop)
    assert np.abs(lm[ok] - lm_loop[ok]).max() <= 1e-12 * np.abs(lm_loop[ok]).max()
    # the bar magnitudes dominate the landmark formula's own magnitudes
    sig = cvm.entry_bar_scale(Sig)
    assert np.all(np.abs(Sig) <= np.outer(sig, sig) * (1 + 1e-12))
    Ka = np.abs(K)
    mag = cvm.landmark_bar_scale(sig, K, W, obs_cam, lm_off)
    for l in np.flatnonzero(ok.all(axis=(1, 2))):
        o = np.arange(lm_off[l], lm_off[l + 1])
        X = np.eye(3) + sum(Ka[a] @ np.abs(Sig[9 * obs_cam[a]:9 * obs_cam[a] + 9, 9 * obs_cam[b]:9 * obs_cam[b] + 9]) @ Ka[b].T
                            for a in o for b in o)
        assert np.all(np.abs(W[l]) @ X @ np.abs(W[l]).T <= mag[l] * (1 + 1e-12))


def test_device_rotation_formula():
    """Eigen's toRotationMatrix on the stored quaternion equals rotation() for unit quaternions; for a float32-rounded one it
    differs by O(| |q|^2 - 1 |), which is why the float32 references use it"""
    rng = np.random.default_rng(7)
    q = rng.normal(size=(500, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    assert np.abs(cm.rotation(q, device=True) - cm.rotation(q)).max() <= 4 * 2.0 ** -52
    q32 = q.astype(np.float32).astype(np.float64)
    dev = np.abs((q32 ** 2).sum(1) - 1)
    diff = np.abs(cm.rotation(q32, device=True) - cm.rotation(q32)).max(axis=(1, 2))
    assert diff.max() > 1e-9 and np.all(diff <= 2 * dev + 1e-15)


# ------------------------------------------------------------------------------------------------
# which tiles of the inverse the landmark marginals read, and a planted error in each off-diagonal tile
# ------------------------------------------------------------------------------------------------
def test_tile_coverage_helper():
    # camera 7 spans rows 63..71: tiles 0 and 1; a landmark on cameras 0 and 7 reads (0, 0), (1, 0) and (1, 1)
    assert cvm.tile_pairs_read(np.array([0, 7]), np.array([0, 2])) == {(0, 0), (1, 0), (1, 1)}
    assert cvm.tile_pairs_read(np.array([0, 20]), np.array([0, 2])) == {(0, 0), (2, 0), (2, 2)}
    assert cvm.straddling_cameras(15) == [7, 14] and cvm.all_tile_pairs(15) == {(0, 0), (1, 0), (1, 1), (2, 0), (2, 1), (2, 2)}


@pytest.mark.parametrize("nc", [14, 15])
def test_planted_tile_error_is_caught_by_the_landmark_check_only(nc):
    """a relative 1e-6 error in one off-diagonal tile of the inverse (outside the cameras' own 9 x 9 blocks) passes the
    camera check and fails the landmark check, for every off-diagonal tile: the landmark blocks are what pins those tiles"""
    prob, absp = cvm.tile_case(nc, nc)
    assert cvm.tile_pairs_read(prob.obs_cam, prob.lm_off) == cvm.all_tile_pairs(nc)
    ref = cvm.reference(prob, absp=absp)
    assert cvm.check(ref["cam"], ref["lm"], ref) <= 1e-4
    N, T = 9 * nc, cvm.TILE
    same_cam = (np.arange(N)[:, None] // 9) == (np.arange(N)[None, :] // 9)
    for ti, tj in sorted(cvm.all_tile_pairs(nc)):
        if ti == tj:
            continue
        E = np.zeros((N, N), bool)
        E[ti * T:(ti + 1) * T, tj * T:(tj + 1) * T] = True
        E &= ~same_cam
        E |= E.T
        Sig = ref["Sig"] * np.where(E, 1 + 1e-6, 1.0)
        cam = np.stack([Sig[9 * c:9 * c + 9, 9 * c:9 * c + 9] for c in range(nc)])
        lm = cvm.landmark_marginal(Sig, ref["K"], ref["W"], ref["rank"], ref["obs_cam"], ref["lm_off"])
        ex, bar = cvm.camera_excess(cam, ref)
        assert ex <= bar, (ti, tj)
        lex, _ = cvm.landmark_excess(lm, ref)
        assert lex > 1.0, (ti, tj, lex)


# ------------------------------------------------------------------------------------------------
# the kernels' SO(3) formulas at large angles, and planted faults in them
# ------------------------------------------------------------------------------------------------
def _cam_with_angle(theta, seed, negate):
    rng = np.random.default_rng(seed)
    cam = np.concatenate([Rotation.from_rotvec(rng.uniform(-2, 2, 3)).as_quat(), rng.uniform(-2, 2, 3), [800.0, 0.01, -0.001]])
    mean = np.concatenate([pm.mean_at_angle(cam, theta, seed + 1, negate), rng.uniform(-2, 2, 3), [805.0, 0.0, 0.0]])
    return cam, mean


@pytest.mark.parametrize("negate", [False, True], ids=["q", "-q"])
@pytest.mark.parametrize("theta", pm.ROTATION_ANGLES)
def test_so3_models_agree_with_rotvec(theta, negate):
    cam, mean = _cam_with_angle(theta, 31, negate)
    want = (Rotation.from_quat(cam[:4]) * Rotation.from_quat(mean[:4]).inv()).as_rotvec()
    assert abs(np.linalg.norm(want) - theta) <= 1e-12
    phi = pm.residual(cam, mean)[3:6]
    assert np.abs(phi - want).max() <= 1e-12
    assert np.abs(pm.log_quat_device(cam[:4], mean[:4]) - want).max() <= 1e-12
    assert np.abs(pm.jl_inv_device(want) - np.linalg.inv(pm.left_jacobian(want))).max() <= 1e-12
    assert np.abs(pm.rows_device(cam[None], mean[None], np.eye(9)[None])[0] - pm.jacobian(cam, mean, device_rot=True)).max() <= 1e-12


def _prior_block_excess(cam, mean, L, fault):
    """the covariance block inv(A^T A) of a camera held by a dense absolute prior only, with A by the kernels' formulas (and
    a planted fault) against the model's; (excess, bar) as covariance_model.camera_excess"""
    A_ref = L @ pm.jacobian(cam, mean, device_rot=True)
    ref = dict(cam=np.linalg.inv(A_ref.T @ A_ref)[None], N=9)
    d = 1 / np.sqrt(np.diag(A_ref.T @ A_ref))
    ref["kappa"] = cvm.spd_cond(A_ref.T @ A_ref * d[:, None] * d[None, :])
    ref["sigma"] = cvm.entry_bar_scale(ref["cam"][0])
    with np.errstate(all="ignore"):
        A = pm.rows_device(cam[None], mean[None], L[None], fault=fault)[0]
        got = np.linalg.inv(A.T @ A)[None] if np.isfinite(A).all() else np.full((1, 9, 9), np.nan)
    ex, bar = cvm.camera_excess(got, ref)
    return (np.inf if np.isnan(ex) else ex), bar


@pytest.mark.parametrize("fault", [None, "jl_identity", "no_flip", "series_everywhere"])
def test_planted_so3_faults_are_rejected_at_large_angles(fault):
    """the check of the GPU test of prior-only cameras accepts the kernels' formulas at every angle and rejects each fault
    at every angle >= 0.5 rad (the flip fault where the product has w < 0, i.e. for one of q, -q)"""
    L = pm.sqrt_info_kind("dense", np.random.default_rng(4))
    for theta in pm.ROTATION_ANGLES:
        verdict = []
        for negate in (False, True):
            cam, mean = _cam_with_angle(theta, 31, negate)
            ex, bar = _prior_block_excess(cam, mean, L, fault)
            assert bar <= 1e-4
            verdict.append(ex > bar)
        if fault is None:
            assert not any(verdict), theta
        elif theta >= 0.5:
            assert any(verdict) if fault == "no_flip" else all(verdict), (fault, theta)
