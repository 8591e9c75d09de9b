"""Resection of cameras from the current landmarks (rba_resect_cameras, DESIGN.md section 26) without a device: the float64
model of tests/resection_model.py against the truth of noise-free problems, scipy.optimize.least_squares' per-unit minimum,
the planted faults the GPU tests must be able to see, and the struct and constants of the header and the Python binding."""
import ctypes
import os
import re

import numpy as np
import pytest
from scipy.optimize import least_squares
from scipy.spatial.transform import Rotation

import camera_prior_model as pm
import observation_loss_model as olm
import resection_model as rm
from rootba_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = np.finfo(np.float64).eps


def _pose(rng, rot_deg=30.0):
    q = Rotation.from_rotvec(np.deg2rad(rot_deg) * rng.normal(size=3) / np.sqrt(3)).as_quat()
    return np.concatenate([q, rng.normal(0, 0.5, 3)])


def _world(nc=1, n=40, seed=0, noise=0.0, k1=0.0, rig=False, outliers=0.0, f=500.0):
    """nc cameras (a rig of nc when rig) looking at n landmarks each, observations projected with noise [px]; returns
    (problem pieces, true cameras)"""
    rng = np.random.default_rng(seed)
    cams, lms, oc, ol, xy = [], [], [], [], []
    base = _pose(rng)
    M = np.tile([0, 0, 0, 1.0, 0, 0, 0], (nc, 1))
    for c in range(nc):
        if rig and c > 0:
            M[c] = np.concatenate([Rotation.from_rotvec(rng.normal(0, 0.3, 3)).as_quat(), rng.normal(0, 0.3, 3)])
            pose = rm.tie(M[c], base)
        else:
            pose = base if rig else _pose(rng)
        cam = np.concatenate([pose, [f, k1, 0.0]])
        R = rm.rot(cam[:4])
        pc = np.column_stack([rng.uniform(-2, 2, n), rng.uniform(-2, 2, n), rng.uniform(4, 9, n)])
        X = (pc - cam[4:7]) @ R  # R^T (pc - t)
        m = pc[:, :2] / pc[:, 2:]
        r2 = (m * m).sum(1)
        obs = f * (1 + k1 * r2)[:, None] * m + rng.normal(0, noise, (n, 2))
        if outliers:
            bad = rng.random(n) < outliers
            obs[bad] += rng.normal(0, 40, (bad.sum(), 2))
        oc += [c] * n
        n0 = sum(len(x) for x in lms)
        ol += list(range(n0, n0 + n))
        lms.append(X)
        xy.append(obs)
        cams.append(cam)
    lead = np.zeros(nc, int) if rig else None
    return dict(cams=np.array(cams), lms=np.vstack(lms), obs_cam=np.array(oc), obs_lm=np.array(ol), obs=np.vstack(xy),
                lead=lead, M=M if rig else None), np.array(cams)


def _perturb(cam, seed, deg=5.0, trans=0.5):
    rng = np.random.default_rng(seed)
    d = np.zeros(9)
    d[:3] = rng.normal(0, trans, 3)
    d[3:6] = np.deg2rad(deg) * rng.normal(size=3) / np.sqrt(3)
    return pm.apply_inc(cam, d)


def _rot_err(a, b):
    return np.linalg.norm(rm.rot(a[:4] / np.linalg.norm(a[:4])) - rm.rot(b[:4] / np.linalg.norm(b[:4])))


@pytest.mark.parametrize("seed", range(4))
def test_linear_recovers_noise_free_truth(seed):
    """noise-free, distorted observations: the DLT returns the true pose to a bar from the 12x12 eigen-gap"""
    pieces, truth = _world(seed=seed, n=30, k1=0.05)
    p = rm.Problem(**pieces)
    p.cams[0, :7] = _perturb(truth[0], seed, 40.0, 3.0)[:7]
    out, st, pts, _ = p.resect(0, rm.LINEAR)
    assert st == rm.WRITTEN and pts == 30
    # the bar: the eigen-gap of M at the truth over u, on the scale of the normalised points
    idx, m = p.usable(0)
    X = p.lms[p.obs_lm[idx]]
    s = np.sqrt(((X - X.mean(0)) ** 2).sum(1).mean())
    Mm = np.zeros((12, 12))
    for i in range(len(idx)):
        G = np.kron(np.eye(3), np.append((X[i] - X.mean(0)) / s, 1.0)[None])
        v = np.append(m[i], 1.0)
        v /= np.linalg.norm(v)
        Mm += G.T @ (np.eye(3) - np.outer(v, v)) @ G
    ev = np.linalg.eigvalsh(Mm)
    bar = 1e3 * U * ev[-1] / ev[1] * (1 + np.linalg.norm(truth[0, 4:7]) + np.linalg.norm(X.mean(0)))
    assert _rot_err(out[0], truth[0]) <= bar and np.linalg.norm(out[0][4:7] - truth[0, 4:7]) <= bar * (1 + s), bar


def _ls_minimum(p, c, x, free):
    """scipy.optimize.least_squares from the model's result, over the free increment entries, of the unit's share written
    as one residual sqrt(2 err) per term; returns its cost and the cost at x"""
    ld, mem = p.unit(c)
    fi = np.flatnonzero(free)

    def fun(d):
        dx = np.zeros(9)
        dx[fi] = d
        return p.residuals(pm.apply_inc(x, dx), ld, mem)

    r0 = fun(np.zeros(len(fi)))
    sol = least_squares(fun, np.zeros(len(fi)), method="trf", xtol=1e-15, ftol=1e-15, gtol=1e-15, x_scale="jac")
    return 0.5 * float(sol.fun @ sol.fun), 0.5 * float(r0 @ r0)


def _case(name, seed=1):
    rng = np.random.default_rng(seed)
    rig = name == "rig"
    pieces, truth = _world(nc=2 if name in ("rig", "pair") else 1, n=40, seed=seed, noise=1.0, rig=rig,
                           outliers=0.15 if name in ("huber", "cauchy", "soft_l1") else 0.0, k1=0.02)
    n = len(pieces["obs"])
    kind = {"huber": olm.HUBER, "cauchy": olm.CAUCHY, "soft_l1": olm.SOFT_L1}.get(name, olm.NONE)
    pieces.update(kind=np.full(n, kind), a=np.full(n, 2.0))
    if name == "W":
        W = rng.normal(0, 0.2, (n, 2, 2)) + np.eye(2)
        W[rng.random(n) < 0.1] = 0.0
        pieces["W"] = W
    nc = len(pieces["cams"])
    if name == "camera_prior":
        mean = truth.copy()
        mean[:, 4:7] = -np.einsum("nji,nj->ni", rm.rot(truth[:, :4]), truth[:, 4:7]) + 0.3  # a biased centre
        L = np.broadcast_to(np.diag([30, 30, 30, 50, 50, 50, 1e-3, 1, 1.0]), (nc, 9, 9)).copy()
        pieces["cprior"] = (mean, L, np.full(nc, olm.CAUCHY), np.full(nc, 2.0))
    if name == "pair":  # camera 1 held at the truth, camera 0 resected: the pair prior ties them
        from pair_prior_model import mean_at
        mean = mean_at(truth, [(0, 1)])
        mean[0, 4:7] += 0.2
        pieces["pprior"] = (np.array([[0, 1]]), mean, np.diag([5, 5, 5, 40, 40, 40.0])[None], np.array([olm.HUBER]),
                            np.array([1.0]))
    p = rm.Problem(**pieces)
    p.cams[0, :7] = _perturb(truth[0], seed, 3.0, 0.3)[:7]
    if rig:
        p.cams[1, :7] = rm.tie(p.M[1], p.cams[0, :7])
    mode = rm.LINEAR | rm.REFINE | (rm.INTRINSICS if name == "intrinsics" else 0)
    return p, mode


CASES = ["none", "huber", "cauchy", "soft_l1", "W", "camera_prior", "pair", "rig", "intrinsics"]


@pytest.mark.parametrize("name", CASES)
def test_refine_reaches_the_least_squares_minimum(name):
    p, mode = _case(name)
    out, st, pts, cost = p.resect(0, mode, max_iterations=100)
    assert st & rm.WRITTEN and st & rm.REFINED and st & rm.CONVERGED, st
    ld, _ = p.unit(0)
    c_ls, c_x = _ls_minimum(p, 0, out[ld], p.free(0, mode))
    assert abs(c_x - cost) <= 1e-12 * cost
    assert c_ls >= cost * (1 - 1e-9), (c_ls, cost)


@pytest.mark.parametrize("fault", rm.FAULTS)
def test_planted_faults_are_caught(fault):
    if fault in ("unnormalised_ray", "ignore_det_sign"):
        hits = 0
        for seed in range(8):
            pieces, truth = _world(seed=seed, n=30)
            p = rm.Problem(**pieces)
            good, _, _, _ = p.resect(0, rm.LINEAR)
            bad, st, _, _ = p.resect(0, rm.LINEAR, fault=fault)
            hits += (not st & rm.WRITTEN) or _rot_err(bad[0], good[0]) > 1e-6 or np.linalg.norm(bad[0][4:7] - good[0][4:7]) > 1e-6
        assert hits > 0
        return
    name = {"prior_no_rt": "camera_prior", "adjoint_transposed": "rig", "ignore_w": "W", "ignore_loss_weight": "cauchy"}[fault]
    p, mode = _case(name)
    out, st, pts, cost = p.resect(0, mode, max_iterations=100, fault=fault)
    ld, _ = p.unit(0)
    c_ls, c_x = _ls_minimum(p, 0, out[ld], p.free(0, mode))
    assert c_ls < c_x * (1 - 1e-6), (c_ls, c_x)


def test_status_rules():
    pieces, truth = _world(seed=3, n=12)
    p = rm.Problem(**pieces)
    p.fixed[0] = rm.FIX_POSE
    _, st, _, _ = p.resect(0)
    assert st == rm.HELD
    _, st, _, _ = p.resect(0, rm.REFINE | rm.INTRINSICS)  # the pose held, f, k1, k2 free
    assert not st & rm.HELD
    p.fixed[0] = 0
    p.W = p.W.copy()
    p.W[2:] = 0.0
    _, st, pts, _ = p.resect(0)
    assert st == rm.FEW_POINTS and pts == 2
    p.W[:] = np.eye(2)
    p.W[5:] = 0.0
    _, st, pts, _ = p.resect(0)
    assert pts == 5 and st & rm.DEGENERATE
    planar = rm.Problem(**pieces)
    planar.lms = planar.lms.copy()
    planar.lms[:, 2] = 0.0
    _, st, _, _ = planar.resect(0, rm.LINEAR)
    assert st == rm.DEGENERATE


def test_header_struct_and_binding_agree():
    h = open(os.path.join(ROOT, "include", "rootba_b200.h")).read()
    for name, val in [("RBA_RESECT_LINEAR", 1), ("RBA_RESECT_REFINE", 2), ("RBA_RESECT_INTRINSICS", 4)]:
        assert re.search(rf"#define {name}\s+{val}\b", h)
        assert getattr(_lib, name[4:]) == val
    for k, v in {"WRITTEN": 1, "FEW_POINTS": 2, "DEGENERATE": 4, "BEHIND": 8, "REFINED": 16, "CONVERGED": 32,
                 "HELD": 64}.items():
        assert re.search(rf"#define RBA_RES_{k}\s+{v}u", h)
        assert getattr(_lib, "RES_" + k) == v == getattr(rm, k)
    assert ctypes.sizeof(_lib.ResectOpts) == 24
    assert [f[0] for f in _lib.ResectOpts._fields_] == ["mode", "max_iterations", "function_tolerance", "reserved"]
