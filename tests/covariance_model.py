"""Float64 model of the marginal covariances (rba_compute_covariance, DESIGN.md section 16), written from the mathematics.

- dense_inverse: the definition, inv(J^T J) of the whole problem [Jp | Jl] with the held columns deleted, and the
  condition number of the Jacobi-equilibrated matrix (the bars of the tests are c * kappa * u).
- schur_reduced: the reduced camera matrix S = sum_l (Jp_l^T Jp_l - Jp_l^T Jl_l pinv(Hll) Jl_l^T Jp_l), landmark by
  landmark from the per-observation blocks (no dense Jacobian: usable at hundreds of cameras).
- eigen_form: the formula the device evaluates, Hll = V Lambda V^T with eigenvalues <= 1e-10 lambda_max dropped,
  K_i = Lambda+^-1/2 V+^T Jl_i^T Jp_i, S = sum_l (delta_ij Jp_i^T Jp_i - K_i^T K_j), landmark marginal
  W (I + sum_ab K_a Sigma_ab K_b^T) W^T with W = V+ Lambda+^-1/2 (NaN when rank < 3).
"""
import numpy as np

EIG_DROP = 1e-10


def fixed_mask(flags, nc):
    """[9 nc] bool of the held increment entries (RBA_FIX_* bits per camera), all False for None"""
    if flags is None:
        return np.zeros(9 * nc, bool)
    from test_fixed_cameras import fixed_entries
    return fixed_entries(np.asarray(flags))


def spd_cond(H):
    """2-norm condition number of a symmetric positive definite matrix"""
    ev = np.linalg.eigvalsh(H)
    return float(ev[-1] / ev[0])


def dense_inverse(Jp, Jl, nc, nl, fixed=None):
    """(cam [nc, 9, 9], lm [nl, 3, 3], kappa): blocks of inv(J^T J) with J = [Jp | Jl] and the held camera columns deleted
    (their rows and columns of the output are 0); kappa = 2-norm condition of D H D, D = diag(H)^-1/2"""
    fixed = np.zeros(9 * nc, bool) if fixed is None else fixed
    J = np.hstack([Jp[:, ~fixed], Jl])
    H = J.T @ J
    d = 1.0 / np.sqrt(np.diag(H))
    Heq = H * d[:, None] * d[None, :]
    kappa = spd_cond(Heq)
    C = np.linalg.inv(Heq) * d[:, None] * d[None, :]
    nf = int((~fixed).sum())
    Ccam = np.zeros((9 * nc, 9 * nc))
    Ccam[np.ix_(~fixed, ~fixed)] = C[:nf, :nf]
    cam = np.stack([Ccam[9 * c:9 * c + 9, 9 * c:9 * c + 9] for c in range(nc)])
    lm = np.stack([C[nf + 3 * l:nf + 3 * l + 3, nf + 3 * l:nf + 3 * l + 3] for l in range(nl)])
    return cam, lm, kappa


def schur_reduced(jp, jl, obs_cam, lm_off, nc):
    """S [9 nc, 9 nc] from the per-observation blocks jp [nobs, 2, 9], jl [nobs, 2, 3] with pinv of every Hll"""
    S = np.zeros((9 * nc, 9 * nc))
    for l in range(len(lm_off) - 1):
        o = np.arange(lm_off[l], lm_off[l + 1])
        cams = obs_cam[o]
        Jp = np.zeros((2 * len(o), 9 * len(o)))
        for k in range(len(o)):
            Jp[2 * k:2 * k + 2, 9 * k:9 * k + 9] = jp[o[k]]
        Jl = jl[o].reshape(-1, 3)
        B = Jp.T @ Jp - Jp.T @ Jl @ np.linalg.pinv(Jl.T @ Jl, rcond=EIG_DROP, hermitian=True) @ Jl.T @ Jp
        idx = (9 * cams[:, None] + np.arange(9)[None, :]).ravel()
        S[np.ix_(idx, idx)] += B
    return S


def landmark_factors(jl_l):
    """(W [3, 3] = V+ Lambda+^-1/2 with zero columns for dropped eigenvalues, rank) of one landmark's Jl rows [2n, 3]"""
    lam, V = np.linalg.eigh(jl_l.T @ jl_l)
    lmax = lam.max()
    keep = (lam > EIG_DROP * lmax) if lmax > 0 else np.zeros(3, bool)
    W = np.where(keep[None, :], V / np.sqrt(np.where(keep, lam, 1.0))[None, :], 0.0)
    return W, int(keep.sum())


def eigen_form(jp, jl, obs_cam, lm_off, nc, H_extra=None):
    """(cam [nc, 9, 9], lm [nl, 3, 3]) by the device's formula; H_extra [9 nc, 9 nc] (priors) is added to S"""
    nl = len(lm_off) - 1
    S = np.zeros((9 * nc, 9 * nc)) if H_extra is None else np.array(H_extra, np.float64)
    K = np.zeros((len(obs_cam), 3, 9))
    Ws, ranks = [], []
    for l in range(nl):
        o = np.arange(lm_off[l], lm_off[l + 1])
        W, r = landmark_factors(jl[o].reshape(-1, 3))
        Ws.append(W)
        ranks.append(r)
        for k in o:
            K[k] = W.T @ (jl[k].T @ jp[k])
        for a in o:
            ca = obs_cam[a]
            S[9 * ca:9 * ca + 9, 9 * ca:9 * ca + 9] += jp[a].T @ jp[a]
            for b in o:
                cb = obs_cam[b]
                S[9 * ca:9 * ca + 9, 9 * cb:9 * cb + 9] -= K[a].T @ K[b]
    Sig = np.linalg.inv(S)
    cam = np.stack([Sig[9 * c:9 * c + 9, 9 * c:9 * c + 9] for c in range(nc)])
    lm = np.full((nl, 3, 3), np.nan)
    for l in range(nl):
        if ranks[l] < 3:
            continue
        o = np.arange(lm_off[l], lm_off[l + 1])
        X = np.eye(3)
        for a in o:
            for b in o:
                ca, cb = obs_cam[a], obs_cam[b]
                X += K[a] @ Sig[9 * ca:9 * ca + 9, 9 * cb:9 * cb + 9] @ K[b].T
        lm[l] = Ws[l] @ X @ Ws[l].T
    return cam, lm
