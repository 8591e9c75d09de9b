"""CPU checks of the covariance model (tests/covariance_model.py): the eigen-form elimination the device evaluates equals the
blocks of the full inverse of J^T J, and with a rank-deficient landmark it equals the reduced matrix built with pinv."""
import numpy as np
import pytest

import covariance_model as cvm


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
