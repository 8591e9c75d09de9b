"""The float64 model of intrinsics shared across groups of cameras (rba_set_intrinsics_groups, DESIGN.md section 18), and the
device's recurrence on the 9 nc layout restated.  Not collected by pytest (no test_ prefix).

The tied problem has a pose per camera and one (f, k1, k2) per group; x = P u with P the 0/1 expansion that copies a group's
intrinsics into every member's entries 6..8.  Its LM step is that of the dense model of the merged Jacobian J P: the Jacobi
scaling of the merged columns, lambda once per reduced parameter.  On the device u lives in the 9 nc layout: the lead's
entries 6..8 hold the group's values, the other members' are 0 (embed)."""
import numpy as np

import camera_prior_model as pm
from objective_checks import reduced
from pcg_replay import block_apply, pcg_replay


def leads(group):
    """[nc] the lead (lowest-index member) of each camera's group of >= 2 cameras, -1 for the others"""
    group = np.asarray(group)
    out = np.full(len(group), -1)
    for g in np.unique(group[group >= 0]):
        m = np.flatnonzero(group == g)
        if len(m) >= 2:
            out[m] = m[0]
    return out


def members(lead):
    """[9 nc] bool: the entries 6..8 of every member that is not its group's lead"""
    lead = np.asarray(lead)
    out = np.zeros((len(lead), 9), bool)
    out[:, 6:] = ((lead >= 0) & (lead != np.arange(len(lead))))[:, None]
    return out.ravel()


def expansion(lead):
    """P [9 nc, nu]: the reduced parameters are the entries of the 9 nc layout that are not members' (see members())"""
    keep = np.flatnonzero(~members(lead))
    col = {e: k for k, e in enumerate(keep)}
    nc = len(lead)
    P = np.zeros((9 * nc, len(keep)))
    for c in range(nc):
        for a in range(9):
            src = 9 * lead[c] + a if (a >= 6 and lead[c] >= 0) else 9 * c + a
            P[9 * c + a, col[src]] = 1.0
    return P


def embed(lead):
    """E [9 nc, nu]: u in the 9 nc layout (P with the members' rows 6..8 zeroed)"""
    E = expansion(lead)
    E[members(lead)] = 0.0
    return E


def tied_step(Jp, Jl, r, lam, nl, lead, dtype=np.float64):
    """the dense model of the tied problem: reduced() of J P.  Returns D (the scaling in the 9 nc layout: every member the
    group's), the landmark scaling, Jls, Minv, H_u, b_u, P, E"""
    P, E = expansion(lead), embed(lead)
    Du, sl, _, Jls, Minv, Hu, bu = reduced(Jp @ P, Jl, r, lam, nl, dtype)
    return P @ Du, sl, Jls, Minv, Hu, bu, P, E


def expand(v, lead):
    """P u of u in the 9 nc layout"""
    v = np.asarray(v, np.float64).reshape(-1, 9).copy()
    g = np.flatnonzero(lead >= 0)
    v[g, 6:] = v[lead[g], 6:]
    return v.ravel()


def contract(y, lead):
    """P^T y in the 9 nc layout: the members' entries 6..8 summed into the lead's, the other members' 0"""
    y = np.asarray(y, np.float64).reshape(-1, 9).copy()
    out = y.copy()
    for c in np.flatnonzero(lead >= 0):
        if lead[c] != c:
            out[lead[c], 6:] += y[c, 6:]
            out[c, 6:] = 0.0
    return out.ravel()


def device_blocks(blocks, lam, lead, fixed=None):
    """the inverse preconditioner of the device (k_group_precond + k_precond_invert) from the per-camera 9x9 blocks of the
    full system (no damping): a grouped camera's pose block alone, the lead's intrinsics block the sum of the members',
    lambda once per reduced parameter, the members' entries 6..8 (and `fixed` entries) zero rows and columns"""
    nc = len(lead)
    hold = members(lead) if fixed is None else (members(lead) | fixed)
    inv = np.zeros((nc, 9, 9))
    for c in range(nc):
        A = np.array(blocks[c], np.float64)
        if lead[c] >= 0:
            A[:6, 6:] = A[6:, :6] = 0.0
            A[6:, 6:] = sum(blocks[m][6:, 6:] for m in np.flatnonzero(lead == c)) if lead[c] == c else 0.0
        A += lam * np.eye(9)
        f = ~hold[9 * c:9 * c + 9]
        inv[c][np.ix_(f, f)] = np.linalg.inv(A[np.ix_(f, f)])
    return inv


def reduced_block_jacobi(blocks, lam, lead):
    """M_u^-1 in reduced coordinates, derived from its definition: the block-diagonal of the tied problem over the blocks
    (pose of a grouped camera), (intrinsics of a group), (all 9 of an ungrouped camera), with the diagonal blocks of the full
    system summed over the members, and lambda I"""
    P = expansion(lead)
    nc = len(lead)
    nu = P.shape[1]
    Hd = np.zeros((9 * nc, 9 * nc))
    for c in range(nc):
        Hd[9 * c:9 * c + 9, 9 * c:9 * c + 9] = blocks[c]
    M = P.T @ Hd @ P + lam * np.eye(nu)
    part = np.zeros(nu, int)  # block label of every reduced parameter
    col = np.argmax(P, axis=1)
    for c in range(nc):
        for a in range(9):
            part[col[9 * c + a]] = 2 * c + (1 if (lead[c] >= 0 and a >= 6) else 0)
    Minv = np.zeros((nu, nu))
    for lab in np.unique(part):
        s = np.flatnonzero(part == lab)
        Minv[np.ix_(s, s)] = np.linalg.inv(M[np.ix_(s, s)])
    return Minv


def replay_9nc(Hfull, b_full, blocks, lam, lead, *, eta, max_it, period=10, fault=None):
    """the device's PCG on the 9 nc layout in float64: contracted b, p, x and z; the operator
    q = P^T H_full (P v) + lambda v (lambda on the contracted v); the inverse blocks of device_blocks().  Hfull: the full
    scaled operator without the pose damping, b_full the full gradient (both with the group-summed scaling).
    fault (planted for the checks of the checks): "lambda_per_member", "b_not_contracted", "x_not_expanded"."""
    inv = device_blocks(blocks, lam, lead)
    if fault == "b_not_contracted":
        b = np.where(members(lead), 0.0, b_full)
    else:
        b = contract(b_full, lead)
    good = lambda v: contract(Hfull @ expand(v, lead), lead) + lam * v
    op = good
    if fault == "lambda_per_member":
        op = lambda v: contract(Hfull @ expand(v, lead) + lam * expand(v, lead), lead)
    elif fault == "x_not_expanded":
        st = {"it": 0, "last_p": False}

        def op(v):
            if st["last_p"] and st["it"] % period == 0:  # the residual refresh, applied to x
                st["last_p"] = False
                return contract(Hfull @ v, lead) + lam * v
            st["it"] += 1
            st["last_p"] = True
            return good(v)
    return pcg_replay(op, b, lambda v: block_apply(inv, v), eta=eta, max_it=max_it, period=period)


def apply_tied(cams, x):
    """the cameras after the (already expanded) increment x [9 nc] (unscaled)"""
    return np.stack([pm.apply_inc(c, d) for c, d in zip(np.asarray(cams, np.float64), np.asarray(x).reshape(-1, 9))])


def tied_covariance(Jp, Jl, lead, fixed9=None):
    """the covariance of the tied problem from its definition, inv(J_u^T J_u) with J_u = [Jp P | Jl] and the held reduced
    parameters deleted: (camera blocks [nc, 9, 9] of P Sigma_u P^T, landmark blocks [nl, 3, 3])"""
    P = expansion(lead)
    keep = np.flatnonzero(~members(lead))
    fu = np.ones(len(keep), bool) if fixed9 is None else ~fixed9[keep]
    J = np.hstack([(Jp @ P)[:, fu], Jl])
    Sig = np.linalg.inv(J.T @ J)
    nu = int(fu.sum())
    Su = np.zeros((P.shape[1], P.shape[1]))
    Su[np.ix_(fu, fu)] = Sig[:nu, :nu]
    return _blocks(P @ Su @ P.T, 9), _blocks(Sig[nu:, nu:], 3)


def contracted_covariance(A, lead, fixed9=None, fault=None):
    """camera blocks of the covariance in the device's order: A [9 nc, 9 nc] the full reduced camera matrix (unscaled,
    lambda = 0, priors included) contracted to P^T A P (planted fault "rows_only": P^T A with the members' columns dropped),
    the held entries deleted, inverted and expanded to P S_u^-1 P^T"""
    P = expansion(lead)
    keep = np.flatnonzero(~members(lead))
    C = P.T @ A @ P if fault is None else (P.T @ A)[:, keep]
    fu = np.ones(len(keep), bool) if fixed9 is None else ~fixed9[keep]
    Su = np.zeros_like(C)
    Su[np.ix_(fu, fu)] = np.linalg.inv(C[np.ix_(fu, fu)])
    return _blocks(P @ Su @ P.T, 9)


def _blocks(M, k):
    return np.stack([M[k * i:k * i + k, k * i:k * i + k] for i in range(M.shape[0] // k)])
