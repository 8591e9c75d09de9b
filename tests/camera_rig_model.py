"""The float64 model of rigid camera rigs (rba_set_camera_rigs, DESIGN.md section 23).  Not collected by pytest (no test_
prefix).

Camera c of a rig has the fixed extrinsics E_c (cam_from_rig) and pose T_c = E_c T_rig; with the lead the rig's
lowest-index camera, every member is T_j = M_j T_lead, M_j = E_j E_lead^-1, composed exactly here.  The tied problem has one
pose per rig and every camera's own intrinsics (or its intrinsics group's, rba_set_intrinsics_groups); x = P u with P
mapping the rig's pose increment to member j through the adjoint A_j.  Its LM step is that of the dense model of J P: the
Jacobi scaling D_u of the merged columns, lambda once per reduced parameter."""
import numpy as np
from scipy.spatial.transform import Rotation

import camera_prior_model as pm


def leads(rig):
    """[nc] the lead (lowest-index member) of each camera's rig of >= 2 cameras, -1 for the others"""
    rig = np.asarray(rig)
    out = np.full(len(rig), -1)
    for r in np.unique(rig[rig >= 0]):
        m = np.flatnonzero(rig == r)
        if len(m) >= 2:
            out[m] = m[0]
    return out


def quat_mul(a, b):
    """Hamilton product of xyzw quaternions"""
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by, aw * by + ay * bw + az * bx - ax * bz,
                     aw * bz + az * bw + ax * by - ay * bx, aw * bw - ax * bx - ay * by - az * bz])


def rot(q):
    return Rotation.from_quat(np.asarray(q, np.float64) / np.linalg.norm(q)).as_matrix()


def relative(a, b):
    """T_a T_b^-1 of two poses (qx,qy,qz,qw, tx,ty,tz ...) as (q [4], t [3])"""
    q = quat_mul(np.asarray(a[:4], np.float64), np.asarray(b[:4], np.float64) * [-1, -1, -1, 1])
    q /= np.linalg.norm(q)
    return q, np.asarray(a[4:7], np.float64) - rot(q) @ np.asarray(b[4:7], np.float64)


def maps(cam_from_rig, lead):
    """[nc, 7] M_j = E_j E_lead^-1 of every rigged camera (the identity for the others)"""
    E = np.asarray(cam_from_rig, np.float64).copy()
    M = np.zeros((len(lead), 7))
    M[:, 3] = 1.0
    for c in np.flatnonzero(lead >= 0):
        q, t = relative(E[c], E[lead[c]])
        M[c] = np.r_[q, t]
    return M


def adjoint(m):
    """A = [[R_m, [t_m]x R_m], [0, R_m]] on (v, w) of M = (q, t)"""
    R = rot(m[:4])
    t = m[4:7]
    tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
    A = np.zeros((6, 6))
    A[:3, :3] = A[3:, 3:] = R
    A[:3, 3:] = tx @ R
    return A


def compose(m, lead_cam, own):
    """the member's camera [10]: pose M T_lead, intrinsics its own"""
    q = quat_mul(m[:4], np.asarray(lead_cam[:4], np.float64))
    q /= np.linalg.norm(q)
    t = rot(m[:4]) @ np.asarray(lead_cam[4:7], np.float64) + m[4:7]
    return np.r_[q, t, np.asarray(own[7:10], np.float64)]


def retie(cams, lead, M):
    """every member's pose := M_j T_lead"""
    out = np.array(cams, np.float64)
    for c in np.flatnonzero((lead >= 0) & (lead != np.arange(len(lead)))):
        out[c] = compose(M[c], out[lead[c]], out[c])
    return out


def held(lead, glead=None):
    """[9 nc] bool: the entries of the 9 nc layout that are not reduced parameters: the rig members' pose entries (and the
    intrinsics group members' entries 6..8)"""
    nc = len(lead)
    out = np.zeros((nc, 9), bool)
    out[:, :6] = ((lead >= 0) & (lead != np.arange(nc)))[:, None]
    if glead is not None:
        out[:, 6:] = ((glead >= 0) & (glead != np.arange(nc)))[:, None]
    return out.ravel()


def expansion(lead, M, glead=None, fault=None):
    """P [9 nc, nu]: member j's pose rows are A_j times its lead's pose columns (fault "tx_sign": [t_m]x with the wrong
    sign), an intrinsics group member's rows 6..8 its lead's; the reduced parameters are the entries not held()"""
    nc = len(lead)
    keep = np.flatnonzero(~held(lead, glead))
    col = {e: k for k, e in enumerate(keep)}
    P = np.zeros((9 * nc, len(keep)))
    for c in range(nc):
        if lead[c] >= 0:
            A = adjoint(M[c])
            if fault == "tx_sign":
                A[:3, 3:] *= -1.0
            for k in range(6):
                P[9 * c:9 * c + 6, col[9 * lead[c] + k]] = A[:, k]
        else:
            for a in range(6):
                P[9 * c + a, col[9 * c + a]] = 1.0
        for a in range(6, 9):
            src = 9 * glead[c] + a if (glead is not None and glead[c] >= 0) else 9 * c + a
            P[9 * c + a, col[src]] = 1.0
    return P


def embed(lead, glead=None):
    """E [9 nc, nu]: u in the 9 nc layout (the reduced parameters at their entries, the held ones 0)"""
    keep = np.flatnonzero(~held(lead, glead))
    E = np.zeros((9 * len(lead), len(keep)))
    E[keep, np.arange(len(keep))] = 1.0
    return E


def apply_tied(cams, x, lead, M):
    """the cameras after the (expanded, unscaled) increment x [9 nc], the members then re-tied"""
    moved = np.stack([pm.apply_inc(c, d) for c, d in zip(np.asarray(cams, np.float64), np.asarray(x).reshape(-1, 9))])
    return retie(moved, lead, M)


def scaled_map(P, D, Du):
    """P~ = D^-1 P D_u: the map of the device's u (reduced, scaled by D_u) to its x (9 nc, scaled by the per-camera D)"""
    return (P * Du[None, :]) / D[:, None]


def rig_case(nc, seed=7, spread=0.05):
    """cam_from_rig [nc, 7] of a rig layout: a unit quaternion near identity and a translation of about 0.3 per camera"""
    rng = np.random.default_rng(seed)
    q = np.c_[spread * rng.standard_normal((nc, 3)), np.ones(nc)]
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    return np.c_[q, 0.3 * rng.standard_normal((nc, 3))]


def extrinsics_from_state(cams, rig):
    """cam_from_rig [nc, 7] that makes the current poses rigid: E_c = T_c T_lead^-1 (the identity for a lead and a free
    camera), the rig's frame being its lead's"""
    cams = np.asarray(cams, np.float64)
    lead = leads(rig)
    E = np.zeros((len(cams), 7))
    E[:, 3] = 1.0
    for c in np.flatnonzero(lead >= 0):
        q, t = relative(cams[c], cams[lead[c]])
        E[c] = np.r_[q, t]
    return E


# ---- the device's 9 nc recurrence restated, its preconditioner, and the covariance --------------------------------------
def reduced_cols(lead, glead=None):
    """[nc, 9] the reduced column of every entry of the 9 nc layout that is a reduced parameter (-1 for the held ones)"""
    keep = np.flatnonzero(~held(lead, glead))
    col = np.full(9 * len(lead), -1)
    col[keep] = np.arange(len(keep))
    return col.reshape(-1, 9)


def device_blocks(blocks, lam, lead, Pt, fixed=None, fault=None):
    """the inverse preconditioner of the device (k_rig_precond + k_precond_invert) from the per-camera 9x9 blocks of the
    full x-space system (no damping) and P~ [9 nc, nu]: a rigged camera's intrinsics block alone (pose-intrinsics entries 0),
    the lead's pose block sum_j P~_j^T B_j P~_j over its rig (without the cross terms between members), lambda once per
    reduced parameter, the members' pose entries (and `fixed` entries) zero rows and columns.  fault "no_pt": the lead's
    pose block the members' B_j summed without P~ (the planted fault)"""
    nc = len(lead)
    col = reduced_cols(lead)
    hold = held(lead) if fixed is None else (held(lead) | fixed)
    inv = np.zeros((nc, 9, 9))
    for c in range(nc):
        A = np.array(blocks[c], np.float64)
        if lead[c] >= 0:
            A[:6, 6:] = A[6:, :6] = 0.0
            if lead[c] == c:
                cols = col[c, :6]
                A[:6, :6] = 0.0
                for j in np.flatnonzero(lead == c):
                    Pj = Pt[9 * j:9 * j + 6][:, cols] if fault != "no_pt" else np.eye(6)
                    A[:6, :6] += Pj.T @ blocks[j][:6, :6] @ Pj
        A += lam * np.eye(9)
        f = ~hold[9 * c:9 * c + 9]
        inv[c][np.ix_(f, f)] = np.linalg.inv(A[np.ix_(f, f)])
    return inv


def reduced_block_jacobi(blocks, lam, lead, Pt):
    """M_u^-1 in reduced coordinates, derived from its definition: the block-diagonal of P~^T blkdiag(B) P~ + lambda I over
    the blocks (pose of a rig), (intrinsics of a rigged camera), (all 9 of a free camera)"""
    nc = len(lead)
    Hd = np.zeros((9 * nc, 9 * nc))
    for c in range(nc):
        Hd[9 * c:9 * c + 9, 9 * c:9 * c + 9] = blocks[c]
    M = Pt.T @ Hd @ Pt + lam * np.eye(Pt.shape[1])
    col = reduced_cols(lead)
    part = np.zeros(Pt.shape[1], int)
    for c in range(nc):
        for a in range(9):
            if col[c, a] >= 0:
                part[col[c, a]] = 2 * c + (1 if (lead[c] >= 0 and a >= 6) else 0)
    Minv = np.zeros_like(M)
    for lab in np.unique(part):
        s = np.flatnonzero(part == lab)
        Minv[np.ix_(s, s)] = np.linalg.inv(M[np.ix_(s, s)])
    return Minv


def replay_9nc(Hfull, b_full, blocks, lam, lead, Pt, *, eta, max_it, period=10, fault=None):
    """the device's PCG on the 9 nc layout in float64: b = P~^T b_full in the lead's entries, the operator
    q = P~^T K (P~ v) + lambda v (lambda on the contracted v), the inverse blocks of device_blocks().  Hfull: the full x-space
    operator K without the pose damping, b_full the full gradient (both with the per-camera scaling).
    fault (planted for the checks of the checks): "lambda_per_member", "b_not_contracted", "no_pt" (device_blocks)."""
    from pcg_replay import block_apply, pcg_replay
    E = embed(lead)
    expand = lambda v: Pt @ (E.T @ v)
    contract = lambda y: E @ (Pt.T @ y)
    inv = device_blocks(blocks, lam, lead, Pt, fault=fault if fault == "no_pt" else None)
    b = np.where(held(lead), 0.0, b_full) if fault == "b_not_contracted" else contract(b_full)
    op = lambda v: contract(Hfull @ expand(v)) + lam * v
    if fault == "lambda_per_member":
        op = lambda v: contract(Hfull @ expand(v) + lam * expand(v))
    return pcg_replay(op, b, lambda v: block_apply(inv, v), eta=eta, max_it=max_it, period=period)


def tied_covariance(Jp, Jl, lead, M, fixed9=None):
    """the covariance of the tied problem from its definition, inv(J_u^T J_u) with J_u = [Jp P | Jl] and the held reduced
    parameters deleted: (camera blocks [nc, 9, 9] of P Sigma_u P^T, landmark blocks [nl, 3, 3], P Sigma_u P^T)"""
    P = expansion(lead, M)
    keep = np.flatnonzero(~held(lead))
    fu = np.ones(len(keep), bool) if fixed9 is None else ~fixed9[keep]
    J = np.hstack([(Jp @ P)[:, fu], Jl])
    Sig = np.linalg.inv(J.T @ J)
    nu = int(fu.sum())
    Su = np.zeros((P.shape[1], P.shape[1]))
    Su[np.ix_(fu, fu)] = Sig[:nu, :nu]
    full = P @ Su @ P.T
    return _blocks(full, 9), _blocks(Sig[nu:, nu:], 3), full


def contracted_covariance(A, lead, M, fixed9=None, fault=None):
    """camera blocks of the covariance in the device's order: A [9 nc, 9 nc] the full reduced camera matrix (unscaled,
    lambda = 0, priors included) contracted to P^T A P (planted fault "rows_only": P^T A with the members' columns dropped),
    the held entries deleted, inverted and expanded to P S_u^-1 P^T"""
    P = expansion(lead, M)
    keep = np.flatnonzero(~held(lead))
    C = P.T @ A @ P if fault is None else (P.T @ A)[:, keep]
    fu = np.ones(len(keep), bool) if fixed9 is None else ~fixed9[keep]
    Su = np.zeros_like(C)
    Su[np.ix_(fu, fu)] = np.linalg.inv(C[np.ix_(fu, fu)])
    return _blocks(P @ Su @ P.T, 9)


def _blocks(Mx, k):
    return np.stack([Mx[k * i:k * i + k, k * i:k * i + k] for i in range(Mx.shape[0] // k)])
