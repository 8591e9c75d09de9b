"""Triangulation of landmarks from the current cameras (rba_triangulate_landmarks, DESIGN.md section 25) without a device:
the float64 model of tests/triangulation_model.py against synthetic.project, the truth of noise-free problems,
scipy.optimize.least_squares' per-landmark minimum, the planted faults the GPU tests must be able to see, and the struct and
constants of the header and the Python binding."""
import ctypes
import os
import re

import numpy as np
import pytest
from scipy.optimize import least_squares

import camera_model as cm
import observation_loss_model as olm
import triangulation_model as tm
from rootba_b200 import _lib
from rootba_b200.synthetic import project, synth_bal

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = np.finfo(np.float64).eps


def _cam(k1=0.0, k2=0.0, f=800.0):
    return np.array([0, 0, 0, 1, 0, 0, 0, f, k1, k2], np.float64)


@pytest.mark.parametrize("k1", [-0.5, -0.2, -0.01, 0.0, 0.01, 0.2, 0.5])
@pytest.mark.parametrize("k2", [0.0, 0.02])
def test_undistort_round_trips_through_project(k1, k2):
    """every point whose radius lies below the first zero of the derivative comes back from synthetic.project"""
    cam = _cam(k1, k2)
    rhos = np.linspace(0.0, 1.2, 61)[1:]
    d = 1 + 3 * k1 * rhos ** 2 + 5 * k2 * rhos ** 4
    fold = np.flatnonzero(d <= 0)
    rhos = rhos[: fold[0]] if fold.size else rhos
    rhos = rhos[(1 + 3 * k1 * rhos ** 2 + 5 * k2 * rhos ** 4) > 1e-3]  # away from the fold, where Newton is well conditioned
    phi = np.linspace(0, 2 * np.pi, len(rhos), endpoint=False)
    m = np.stack([rhos * np.cos(phi), rhos * np.sin(phi)], 1)
    xy, _ = project(np.repeat(cam[None], len(m), 0), np.hstack([m, np.ones((len(m), 1))]))
    for i in range(len(m)):
        mr, ok = tm.undistort(xy[i] / cam[7], k1, k2)
        assert ok, (k1, k2, rhos[i])
        assert np.abs(mr - m[i]).max() <= 1e-12 * (1 + rhos[i]), (k1, k2, rhos[i], mr, m[i])


@pytest.mark.parametrize("k1", [-0.5, -0.3, -0.1])
def test_undistort_fails_exactly_past_the_fold(k1):
    """k2 = 0: rho (1 + k1 rho^2) peaks at rho* = 1 / sqrt(-3 k1), where the derivative changes sign; every radius up to the
    peak value inverts, none beyond it does"""
    rs = 1 / np.sqrt(-3 * k1)
    peak = rs * (1 + k1 * rs * rs)
    for f in (1 - 1e-6, 1 - 1e-3, 0.5):
        m, ok = tm.undistort(np.array([peak * f, 0.0]), k1, 0.0)
        assert ok and m[0] < rs, f
        assert abs(m[0] * (1 + k1 * m[0] ** 2) - peak * f) <= 1e-12 * peak
    for f in (1 + 1e-6, 1 + 1e-3, 2.0):
        assert not tm.undistort(np.array([0.0, peak * f]), k1, 0.0)[1], f


@pytest.fixture(scope="module")
def clean():
    """noise-free, unperturbed: the stored landmarks are the truth; distortion as in photo collections"""
    return synth_bal(10, 120, 4.0, seed=5, obs_noise=0.0, perturb_lm=0.0, perturb_rot=0.0, perturb_trans=0.0,
                     k1_sigma=0.05, k2_sigma=0.005)


def _kappa(tr):
    """the conditioning of the linear estimate: the largest over the second smallest eigenvalue of M"""
    d, ok = tr.rays()
    c = tr.centres[ok]
    cbar = c.mean(0)
    s = np.sqrt(((c - cbar) ** 2).sum(1).mean())
    M = np.zeros((4, 4))
    for i in np.flatnonzero(ok):
        R, t = tr.R[i], tr.cams[i, 4:7]
        B = np.hstack([R, ((R @ cbar + t) / s)[:, None]])
        v = R @ d[i]
        v /= np.linalg.norm(v)
        M += B.T @ (np.eye(3) - np.outer(v, v)) @ B
    e = np.linalg.eigvalsh(M)
    return e[3] / e[1], s


def test_linear_recovers_noise_free_truth(clean):
    """|X - X_true| <= 100 kappa u (s + |X - cbar|): the error of an eigenvector is u ||M|| over the eigenvalue gap"""
    worst = 0.0
    for l, tr in enumerate(tm.tracks(clean)):
        X, bits = tr.linear()
        assert bits == 0, l
        kappa, s = _kappa(tr)
        bar = 100 * kappa * U * (s + np.linalg.norm(clean.lms[l] - tr.centres.mean(0)))
        err = np.linalg.norm(X - clean.lms[l])
        worst = max(worst, err / bar)
        assert err <= bar, (l, err, bar)
    assert worst < 1.0


def _noisy(seed=11):
    return synth_bal(9, 60, 5.0, seed=seed, obs_noise=1.0, perturb_lm=0.3, perturb_rot=0.0, perturb_trans=0.0,
                     k1_sigma=0.02, k2_sigma=0.002)


def _scipy_min(tr, X0, loss="linear", a=1.0):
    """scipy's minimum of the landmark's share: one residual |W r| per observation in use (and |L e| of the prior), the
    loss on its square"""
    use = tr.in_use()

    def fun(X):
        n = len(tr.cams)
        r = cm.linearize(tr.cams[use], np.broadcast_to(X, (int(use.sum()), 3)), tr.obs[use], device_rot=True)["res"]
        r = np.einsum("nij,nj->ni", tr.W[use], r)
        out = [np.sqrt((r * r).sum(1))]
        if tr.prior is not None:
            out.append([np.linalg.norm(tr.prior[0] @ (X - tr.prior[1]))])
        del n
        return np.concatenate(out)

    res = least_squares(fun, X0, loss=loss, f_scale=a, x_scale="jac", xtol=1e-15, ftol=1e-15, gtol=1e-15, max_nfev=2000)
    return res.x


def _hessian_bar(tr, X):
    """a position tolerance from the landmark's own conditioning: sqrt(u) over the smallest curvature, relative to |X|"""
    _, H, _ = tr.cost(X, with_normal=True)
    ev = np.linalg.eigvalsh(H)
    return 1e3 * np.sqrt(U) * (1 + np.linalg.norm(X)) * np.sqrt(ev[2] / max(ev[0], 1e-300))


@pytest.mark.parametrize("loss", ["NONE", "HUBER", "CAUCHY", "SOFT_L1"])
def test_refine_reaches_the_least_squares_minimum(loss):
    prob = _noisy()
    a = 1.5
    kind = np.full(prob.nobs, olm.NAMES.index(loss))
    sp = {"NONE": "linear", "HUBER": "huber", "CAUCHY": "cauchy", "SOFT_L1": "soft_l1"}[loss]
    for l, tr in enumerate(tm.tracks(prob, kind=kind, a=np.full(prob.nobs, a))):
        X, st, _, cost = tr.triangulate(prob.lms[l], max_iterations=100)  # IRLS is linear near the minimum
        assert st & tm.WRITTEN and not st & (tm.AT_INFINITY | tm.BEHIND), (l, st)
        Xs = _scipy_min(tr, X, sp, a)
        assert np.linalg.norm(X - Xs) <= _hessian_bar(tr, Xs), (l, X, Xs)
        assert cost <= tr.cost(Xs) * (1 + 1e-8) + 1e-12, l  # IRLS converges linearly near a kink


def test_refine_with_information_and_switched_off_observations():
    prob = _noisy(12)
    rng = np.random.default_rng(3)
    W = rng.normal(0, 0.3, (prob.nobs, 2, 2)) + np.eye(2)
    off = rng.random(prob.nobs) < 0.15
    W[off] = 0.0
    for l, tr in enumerate(tm.tracks(prob, W=W)):
        X, st, _, _ = tr.triangulate(prob.lms[l])
        if st & (tm.FEW_RAYS | tm.AT_INFINITY | tm.BEHIND):
            continue
        Xs = _scipy_min(tr, X)
        assert np.linalg.norm(X - Xs) <= _hessian_bar(tr, Xs), l


def test_refine_with_a_landmark_prior():
    prob = _noisy(13)
    rng = np.random.default_rng(4)
    idx = np.arange(0, prob.nl, 2)
    mean = prob.lms[idx] + rng.normal(0, 0.05, (len(idx), 3))
    Ls = np.array([np.linalg.cholesky(np.linalg.inv(np.diag(rng.uniform(0.01, 0.1, 3)))).T for _ in idx])
    prior = (idx, mean, Ls, np.zeros(len(idx), int), np.ones(len(idx)))
    for l, tr in enumerate(tm.tracks(prob, prior=prior)):
        X, st, _, _ = tr.triangulate(prob.lms[l])
        Xs = _scipy_min(tr, X)
        assert np.linalg.norm(X - Xs) <= _hessian_bar(tr, Xs), l


def test_planted_faults_are_seen(clean):
    """each fault moves a result well past the bars the GPU tests use"""
    k = synth_bal(10, 60, 4.0, seed=6, obs_noise=0.0, perturb_lm=0.0, perturb_rot=0.0, perturb_trans=0.0, k1_sigma=0.3)
    trs = tm.tracks(k)
    # distortion left uninverted, and the ray without R^T: the linear estimate misses the truth
    for fault in ("no_undistort", "no_rt"):
        errs = []
        for l, tr in enumerate(trs):
            X, _ = tr.linear(fault)
            errs.append(np.inf if X is None else np.linalg.norm(X - k.lms[l]))
        assert np.median(errs) > 1e-4, fault
    # a flipped cheirality sign: a good landmark is reported behind
    assert all(tr.linear("flip_cheirality")[1] == tm.BEHIND for tr in trs[:10])
    # W ignored: an observation switched off still pulls the landmark
    prob = _noisy(14)
    W = np.broadcast_to(np.eye(2), (prob.nobs, 2, 2)).copy()
    bad = prob.lm_off[:-1] + 1
    prob.obs_xy[bad] += 80.0
    W[bad] = 0.0
    moved = 0
    for l, tr in enumerate(tm.tracks(prob, W=W)):
        X, st, _, _ = tr.triangulate(prob.lms[l])
        Xf, _, _, _ = tr.triangulate(prob.lms[l], fault="ignore_w")
        if st & tm.FEW_RAYS:
            continue
        moved += np.linalg.norm(X - Xf) > 100 * _hessian_bar(tr, X)
    assert moved > 0.5 * prob.nl
    # the loss weight ignored: the fixed point is not the minimum of the robust cost
    prob = _noisy(15)
    prob.obs_xy[prob.lm_off[:-1]] += 40.0
    kind, a = np.full(prob.nobs, olm.CAUCHY), np.full(prob.nobs, 1.0)
    worse = 0
    for l, tr in enumerate(tm.tracks(prob, kind=kind, a=a)):
        _, _, _, c = tr.triangulate(prob.lms[l])
        Xf, _, _, _ = tr.triangulate(prob.lms[l], fault="ignore_loss_weight")
        worse += tr.cost(Xf) > c * (1 + 1e-6)
    assert worse > 0.8 * prob.nl
    # acos instead of atan2 below 1e-4 rad
    errs = []
    for ang in np.geomspace(1e-8, 1e-4, 17):
        tr = tm.Track(np.stack([_cam(), _cam()]), np.zeros((2, 2)))
        d = np.array([[0, 0, 1.0], [np.sin(ang), 0, np.cos(ang)]])
        tr.rays = lambda fault=None, d=d: (d, np.ones(2, bool))
        assert abs(tr.angle() - ang) <= 1e-12 * ang
        errs.append(abs(tr.angle("acos") - ang) / ang)
    assert max(errs) > 1e-4


def test_opts_struct_and_constants():
    assert ctypes.sizeof(_lib.TriangulateOpts) == 32
    assert [f for f, _ in _lib.TriangulateOpts._fields_] == ["mode", "max_iterations", "min_angle", "function_tolerance",
                                                             "reserved"]
    hdr = open(os.path.join(ROOT, "include", "rootba_b200.h")).read()
    want = {"RBA_TRIANGULATE_LINEAR": tm.LINEAR, "RBA_TRIANGULATE_REFINE": tm.REFINE, "RBA_TRI_WRITTEN": tm.WRITTEN,
            "RBA_TRI_FEW_RAYS": tm.FEW_RAYS, "RBA_TRI_SMALL_ANGLE": tm.SMALL_ANGLE, "RBA_TRI_AT_INFINITY": tm.AT_INFINITY,
            "RBA_TRI_BEHIND": tm.BEHIND, "RBA_TRI_REFINED": tm.REFINED, "RBA_TRI_CONVERGED": tm.CONVERGED}
    for name, v in want.items():
        m = re.search(rf"#define {name}\s+(\d+)u?", hdr)
        assert m and int(m.group(1)) == v, name
        assert getattr(_lib, name[4:]) == v, name
    src = open(os.path.join(ROOT, "rootba_b200", "csrc", "triangulate.cuh")).read()
    for name, v in (("TRI_UNDISTORT_ITERS", tm.UNDISTORT_ITERS), ("TRI_UNDISTORT_TOL", tm.UNDISTORT_TOL),
                    ("TRI_INFINITY", tm.INFINITY)):
        m = re.search(rf"constexpr \w+ {name} = ([0-9.e+-]+);", src)
        assert m and float(m.group(1)) == v, name
    assert "rba_triangulate_landmarks" in _lib.declared_symbols()
    assert "rba_default_triangulate_opts" in _lib.declared_symbols()
