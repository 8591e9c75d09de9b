"""An independent float64 model of the Gaussian landmark prior (rba_set_landmark_prior, DESIGN.md section 17).

  prior p on landmark l_p: residual e = x - x0, cost 1/2 |L e|^2, L a 3x3 square-root information (any rank)
  rows of the total Jacobian: [0 (cameras) | L (columns of landmark l_p) | L e]

The total objective (tests/objective_checks.py: dense_system, total_cost) is reprojection (tests/camera_model.py) plus these
rows, optionally plus the camera priors of tests/camera_prior_model.py and the pair priors of tests/pair_prior_model.py.  The
dense LM step is that of the whole Jacobian with the Jacobi scaling of its columns (prior columns included):
(J_s^T J_s + lambda I) d = -J_s^T r.

The device folds a prior into the landmark's damping rows: the QR of [L~; sqrt(lambda) I] with the residual [g; 0]
(L~ = L diag(jls), g = L e) gives 3 rows [C | 0 | c], and the damping rotations fold them into the landmark's R.  `compress`
and `fold_damping` restate that with numpy's QR and the rotation order of k_stage2, so the CPU tests can check the algebra
and show that the checkers reject planted faults.
"""
import numpy as np


def rows(lms, idx, mean, sqrt_info):
    """per prior: A [m, 3, 3] = L (the Jacobian in the landmark's columns, unscaled) and r [m, 3] = L (x - x0)"""
    lms = np.asarray(lms, np.float64)
    L = np.asarray(sqrt_info, np.float64)
    e = lms[np.asarray(idx)] - np.asarray(mean, np.float64)
    return L.copy(), np.einsum("mij,mj->mi", L, e)


def sqrt_info_kind(kind, rng, scale=1.0):
    """one 3x3 L: 'dense' (well conditioned), 'height' (one non-zero row), 'rank2' (two rows), 'none' (zero)"""
    L = np.zeros((3, 3))
    if kind == "dense":
        L = scale * (np.eye(3) + 0.3 * rng.standard_normal((3, 3)))
    elif kind == "height":
        L[2, 2] = 2.0 * scale
    elif kind == "rank2":
        L[:2] = scale * (np.eye(3)[:2] + 0.3 * rng.standard_normal((2, 3)))
    return L


def prior_case(lms, every=3, seed=7, kinds=("dense", "height", "rank2", "none"), sigma=0.05, scale=1.0):
    """priors on every `every`-th landmark (so prior and prior-free landmarks share tiles), the kinds in turn, means at the
    landmarks moved by N(0, sigma)"""
    rng = np.random.default_rng(seed)
    lms = np.asarray(lms, np.float64)
    idx = np.arange(0, len(lms), every, dtype=np.int32)
    mean = lms[idx] + rng.normal(0, sigma, (len(idx), 3))
    L = np.stack([sqrt_info_kind(kinds[p % len(kinds)], rng, scale) for p in range(len(idx))])
    return idx, mean, L


def cost(lms, idx, mean, sqrt_info):
    _, r = rows(lms, idx, mean, sqrt_info)
    return float(0.5 * np.sum(r * r))


def append_rows(system, nl, lms, idx, mean, sqrt_info):
    """(Jp, Jl, r) with the prior rows appended: zero camera columns, L in the landmark's 3 columns, residual L e"""
    Jp, Jl, r = system
    A, rp = rows(lms, idx, mean, sqrt_info)
    m = len(idx)
    Jl_p = np.zeros((3 * m, 3 * nl))
    for p, l in enumerate(np.asarray(idx)):
        Jl_p[3 * p:3 * p + 3, 3 * l:3 * l + 3] = A[p]
    return np.vstack([Jp, np.zeros((3 * m, Jp.shape[1]))]), np.vstack([Jl, Jl_p]), np.concatenate([r, rp.ravel()])


def scaling(Jp, Jl, eps):
    """the Jacobi scaling of the whole Jacobian (prior columns included)"""
    return 1.0 / (eps + np.linalg.norm(Jp, axis=0)), 1.0 / (eps + np.linalg.norm(Jl, axis=0))


def lm_step(Jp, Jl, r, lam, eps):
    """the dense LM step of the whole scaled Jacobian: d = (dp, dl) with (J_s^T J_s + lam I) d = -J_s^T r, its model cost
    change l_diff = 1/2 |r|^2 - 1/2 |r + J_s d|^2 and the scalings"""
    D, sl = scaling(Jp, Jl, eps)
    J = np.hstack([Jp * D, Jl * sl])
    d = -np.linalg.solve(J.T @ J + lam * np.eye(J.shape[1]), J.T @ r)
    l_diff = 0.5 * r @ r - 0.5 * np.sum((r + J @ d) ** 2)
    n = Jp.shape[1]
    return d[:n], d[n:], float(l_diff), D, sl


# ------------------------------------------------------------------------------------------------
# the device's compression and damping rotations, restated
# ------------------------------------------------------------------------------------------------
def compress(Lt, g, lam, fault=None):
    """[L~; sqrt(lam) I] with the residual [g; 0] -> (C upper triangular, c): Q^T of the 6x3 QR.  fault: "no_lambda" (the
    damping rows left out), "g_sign" (the residual taken as -g)"""
    Lt, g = np.asarray(Lt, np.float64), np.asarray(g, np.float64)
    if fault == "g_sign":
        g = -g
    M = Lt if fault == "no_lambda" else np.vstack([Lt, np.sqrt(lam) * np.eye(3)])
    rhs = g if fault == "no_lambda" else np.concatenate([g, np.zeros(3)])
    Q, R = np.linalg.qr(M, mode="complete")
    return np.triu(R[:3]), (Q.T @ rhs)[:3]


def _givens(p, q):
    """Eigen makeGivens as make_givens of kernels.cuh: (c, s) with c q + s p = 0"""
    if q == 0:
        return (-1.0 if p < 0 else 1.0), 0.0
    if p == 0:
        return 0.0, (1.0 if q < 0 else -1.0)
    if abs(p) > abs(q):
        t = q / p
        u = np.sqrt(1 + t * t) * (-1 if p < 0 else 1)
        c = 1 / u
        return c, -t * c
    t = p / q
    u = np.sqrt(1 + t * t) * (-1 if q < 0 else 1)
    s = -1 / u
    return -t * s, s


def fold_damping(R, rr, Dw, dr):
    """the 6 rotations of k_stage2: fold the 3 rows [Dw | dr] into [R | rr] (R upper triangular), zeroing Dw[d][n] for d <= n;
    returns the damped (R, rr) and the rotated damping rows (Dw, dr)"""
    R, rr, Dw, dr = (np.array(a, np.float64) for a in (R, rr, Dw, dr))
    for n in range(3):
        for m in range(n + 1):
            d = n - m
            c, s = _givens(R[n, n], Dw[d, n])
            x, y = Dw[d].copy(), R[n].copy()
            Dw[d], R[n] = c * x + s * y, -s * x + c * y
            xr, yr = dr[d], rr[n]
            dr[d], rr[n] = c * xr + s * yr, -s * xr + c * yr
    return R, rr, Dw, dr


def sharded_cost(reproj_partials, prior_partials, per_rank_all_priors=False):
    """the cost the device reports for a sharded problem: each rank adds its own landmark priors to its partial before the
    sum over the shards.  per_rank_all_priors plants the fault of every rank adding every prior (counted once per rank)."""
    if per_rank_all_priors:
        return float(sum(reproj_partials) + len(reproj_partials) * sum(prior_partials))
    return float(sum(r + p for r, p in zip(reproj_partials, prior_partials)))
