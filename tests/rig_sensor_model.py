"""The float64 model of estimated rig extrinsics (rba_set_rig_sensors, DESIGN.md section 24), built on camera_rig_model.
Not collected by pytest (no test_ prefix).

A rig's lead is its lowest-index camera with held extrinsics (sensor -1); a held member is T_j = M_j T_lead with
M_j = E_j E_lead^-1.  Sensor s has a home, its lowest-index camera; the state defines E_s = T_home T_lead(home)^-1 E_lead(home)
and every other camera j of s is T_j = E_s E_lead(j)^-1 T_lead(j).  A sensor camera moves by A_j d_lead + d_s, A_j the
adjoint of its current M_j = E_s E_lead(j)^-1.  The tied problem has one pose per rig (the lead's entries), one per sensor
(the home's entries) and every camera's own intrinsics; its LM step is that of the dense model of J P."""
import numpy as np

import camera_prior_model as pm
import camera_rig_model as rm


def structure(rig, sensor=None):
    """(lead [nc], home [nc]): a rig's lead is its lowest-index camera without a sensor id, a sensor's home its lowest-index
    camera (-1 for the cameras without a rig of >= 2 cameras, and for held extrinsics)"""
    lead0 = rm.leads(rig)
    nc = len(lead0)
    sensor = np.full(nc, -1) if sensor is None else np.asarray(sensor)
    lead, home = lead0.copy(), np.full(nc, -1)
    for l0 in np.unique(lead0[lead0 >= 0]):
        m = np.flatnonzero(lead0 == l0)
        lead[m] = m[sensor[m] < 0][0]
    for s in np.unique(sensor[sensor >= 0]):
        m = np.flatnonzero(sensor == s)
        home[m] = m[0]
    return lead, home


def pose_mul(a, b):
    """a b of two poses (q [4] xyzw, t [3]) as [7]"""
    q = rm.quat_mul(np.asarray(a[:4], np.float64), np.asarray(b[:4], np.float64))
    q /= np.linalg.norm(q)
    return np.r_[q, rm.rot(a[:4]) @ np.asarray(b[4:7], np.float64) + np.asarray(a[4:7], np.float64)]


def pose_inv(a):
    q = np.asarray(a[:4], np.float64) * [-1, -1, -1, 1]
    return np.r_[q, -(rm.rot(q) @ np.asarray(a[4:7], np.float64))]


def sensor_extrinsics(cams, lead, home, E):
    """[nc, 7] the extrinsics the state defines: E_s = T_home T_lead(home)^-1 E_lead(home) for every camera of sensor s, the
    given E_j for held members, the identity for free cameras"""
    cams = np.asarray(cams, np.float64)
    out = np.zeros((len(lead), 7))
    out[:, 3] = 1.0
    for c in np.flatnonzero(lead >= 0):
        h = home[c]
        if h < 0:
            q = np.asarray(E[c, :4], np.float64)
            out[c] = np.r_[q / np.linalg.norm(q), E[c, 4:]]
        else:
            out[c] = pose_mul(pose_mul(cams[h, :7], pose_inv(cams[lead[h], :7])), E[lead[h]])
    return out


def maps(cams, lead, home, E):
    """[nc, 7] M_j of every rigged camera at the state `cams`: E_j E_lead^-1 (held), E_s E_lead(j)^-1 (sensor)"""
    Es = sensor_extrinsics(cams, lead, home, E)
    M = np.zeros((len(lead), 7))
    M[:, 3] = 1.0
    for c in np.flatnonzero(lead >= 0):
        q, t = rm.relative(Es[c], E[lead[c]])
        M[c] = np.r_[q, t]
    return M


def tie_at_call(cams, lead, home, E):
    """the state rba_set_rig_sensors leaves: every member M_j T_lead with held members through E_j and every camera of a
    sensor (the home included) through its home's given E"""
    out = np.array(cams, np.float64)
    for c in np.flatnonzero((lead >= 0) & (lead != np.arange(len(lead)))):
        src = c if home[c] < 0 else home[c]
        q, t = rm.relative(E[src], E[lead[c]])
        out[c] = rm.compose(np.r_[q, t], out[lead[c]], out[c])
    return out


def retie(cams, lead, home, E):
    """after an update: held members M_j T_lead, the cameras of a sensor but its home E_s E_lead(j)^-1 T_lead(j)"""
    out = np.array(cams, np.float64)
    M = maps(out, lead, home, E)
    for c in np.flatnonzero((lead >= 0) & (lead != np.arange(len(lead))) & (home != np.arange(len(lead)))):
        out[c] = rm.compose(M[c], out[lead[c]], out[c])
    return out


def held(lead, home, glead=None):
    """[9 nc] bool: the entries of the 9 nc layout that are not reduced parameters (the pose of every rig member but the
    lead and the homes; fault-free: a home's entries carry its sensor's)"""
    nc = len(lead)
    out = rm.held(lead, glead).reshape(nc, 9)
    out[home == np.arange(nc), :6] = False
    return out.ravel()


def expansion(lead, home, M, glead=None, fault=None):
    """P [9 nc, nu]: member j's pose rows are A_j times its lead's pose columns plus, for a sensor camera, the identity on its
    home's pose columns.  Planted faults: "right" (the sensor increment applied on the right: A_j d_s), "no_sensor" (the
    homes masked: sensor cameras move with their rig alone)"""
    nc = len(lead)
    hold = held(lead, home, glead)
    if fault == "no_sensor":
        hold = rm.held(lead, glead)
    keep = np.flatnonzero(~hold)
    col = {e: k for k, e in enumerate(keep)}
    P = np.zeros((9 * nc, len(keep)))
    for c in range(nc):
        if lead[c] >= 0:
            A = rm.adjoint(M[c])
            for k in range(6):
                P[9 * c:9 * c + 6, col[9 * lead[c] + k]] += A[:, k]
            if home[c] >= 0 and fault != "no_sensor":
                S = A if fault == "right" else np.eye(6)
                for k in range(6):
                    P[9 * c:9 * c + 6, col[9 * home[c] + k]] += S[:, k]
        else:
            for a in range(6):
                P[9 * c + a, col[9 * c + a]] = 1.0
        for a in range(6, 9):
            src = 9 * glead[c] + a if (glead is not None and glead[c] >= 0) else 9 * c + a
            P[9 * c + a, col[src]] = 1.0
    return P


def embed(lead, home, glead=None):
    """[9 nc, nu]: u in the 9 nc layout (the reduced parameters at their entries, the held ones 0)"""
    keep = np.flatnonzero(~held(lead, home, glead))
    out = np.zeros((9 * len(lead), len(keep)))
    out[keep, np.arange(len(keep))] = 1.0
    return out


def apply_tied(cams, x, lead, home, E):
    """the cameras after the expanded, unscaled increment x [9 nc], then re-tied"""
    moved = np.stack([pm.apply_inc(c, d) for c, d in zip(np.asarray(cams, np.float64), np.asarray(x).reshape(-1, 9))])
    return retie(moved, lead, home, E)


def scaled_maps(P, D, Du, lead, home):
    """(P~ [nc, 6, 6], Q~ [nc, 6]) of the device: P~_j = D_j^-1 A_j D_u and Q~_j = D_j^-1 D_s (the rows of P~ = D^-1 P D_u
    at the lead's and the home's columns)"""
    Pt = (P * Du[None, :]) / D[:, None]
    keep = np.flatnonzero(~held(lead, home))
    pos = {e: k for k, e in enumerate(keep)}
    nc = len(lead)
    pt, qt = np.zeros((nc, 6, 6)), np.zeros((nc, 6))
    for c in np.flatnonzero(lead >= 0):
        pt[c] = Pt[9 * c:9 * c + 6, [pos[9 * lead[c] + k] for k in range(6)]]
        if home[c] >= 0:
            qt[c] = np.diag(Pt[9 * c:9 * c + 6, [pos[9 * home[c] + k] for k in range(6)]])
    return pt, qt


def tied_covariance(Jp, Jl, lead, home, M, fixed9=None):
    """inv(J_u^T J_u), J_u = [Jp P | Jl] with the held reduced parameters deleted: (camera blocks [nc, 9, 9] of
    P Sigma_u P^T, landmark blocks, P Sigma_u P^T)"""
    P = expansion(lead, home, M)
    keep = np.flatnonzero(~held(lead, home))
    fu = np.ones(len(keep), bool) if fixed9 is None else ~fixed9[keep]
    J = np.hstack([(Jp @ P)[:, fu], Jl])
    Sig = np.linalg.inv(J.T @ J)
    nu = int(fu.sum())
    Su = np.zeros((P.shape[1], P.shape[1]))
    Su[np.ix_(fu, fu)] = Sig[:nu, :nu]
    full = P @ Su @ P.T
    blocks = lambda X, k: np.stack([X[k * i:k * i + k, k * i:k * i + k] for i in range(X.shape[0] // k)])
    return blocks(full, 9), blocks(Sig[nu:, nu:], 3), full


def contracted_covariance(A, lead, home, M, fixed9=None):
    """the covariance in the device's order: the full reduced camera matrix A contracted to P^T A P, the held entries
    deleted, inverted and expanded to P S_u^-1 P^T (camera blocks)"""
    P = expansion(lead, home, M)
    keep = np.flatnonzero(~held(lead, home))
    C = P.T @ A @ P
    fu = np.ones(len(keep), bool) if fixed9 is None else ~fixed9[keep]
    Su = np.zeros_like(C)
    Su[np.ix_(fu, fu)] = np.linalg.inv(C[np.ix_(fu, fu)])
    full = P @ Su @ P.T
    return np.stack([full[9 * i:9 * i + 9, 9 * i:9 * i + 9] for i in range(len(lead))])


# ---- the device's 9 nc recurrence and preconditioner restated ---------------------------------------------------------
def reduced_cols(lead, home):
    """[nc, 9] the reduced column of every entry of the 9 nc layout that is a reduced parameter (-1 for the held ones)"""
    keep = np.flatnonzero(~held(lead, home))
    col = np.full(9 * len(lead), -1)
    col[keep] = np.arange(len(keep))
    return col.reshape(-1, 9)


def device_blocks(blocks, lam, lead, home, Pt, fixed9=None, fault=None):
    """the inverse preconditioner of the device (k_rig_precond<S, true> + k_precond_invert) from the per-camera 9x9 blocks of
    the full x-space system (no damping) and P~ [9 nc, nu]: a rigged camera's intrinsics block alone, the lead's pose block
    sum_j P~_j^T B_j P~_j over its rig, the home's pose block sum_j Q~_j B_j Q~_j over its sensor (Q~_j the rows of P~ at the
    home's columns), no cross terms, lambda once per reduced parameter, the other members' pose entries (and `fixed9`) zero
    rows and columns.  fault "home_masked": the homes' pose entries held as well"""
    nc = len(lead)
    col = reduced_cols(lead, home)
    hold = held(lead, home) if fixed9 is None else (held(lead, home) | fixed9)
    if fault == "home_masked":
        hold = hold | rm.held(lead)
    inv = np.zeros((nc, 9, 9))
    for c in range(nc):
        A = np.array(blocks[c], np.float64)
        if lead[c] >= 0:
            A[:6, 6:] = A[6:, :6] = 0.0
            A[:6, :6] = 0.0
            for j in (np.flatnonzero(lead == c) if lead[c] == c else np.flatnonzero(home == c) if home[c] == c else []):
                Pj = Pt[9 * j:9 * j + 6][:, col[c, :6]]
                A[:6, :6] += Pj.T @ blocks[j][:6, :6] @ Pj
        A += lam * np.eye(9)
        f = ~hold[9 * c:9 * c + 9]
        inv[c][np.ix_(f, f)] = np.linalg.inv(A[np.ix_(f, f)])
    return inv


def reduced_block_jacobi(blocks, lam, lead, home, Pt):
    """M_u^-1 in reduced coordinates from its definition: the block-diagonal of P~^T blkdiag(B) P~ + lambda I over the
    blocks (pose of a rig), (pose of a sensor), (intrinsics of a rigged camera), (all 9 of a free camera)"""
    nc = len(lead)
    Hd = np.zeros((9 * nc, 9 * nc))
    for c in range(nc):
        Hd[9 * c:9 * c + 9, 9 * c:9 * c + 9] = blocks[c]
    M = Pt.T @ Hd @ Pt + lam * np.eye(Pt.shape[1])
    col = reduced_cols(lead, home)
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


def replay_9nc(Hfull, b_full, blocks, lam, lead, home, Pt, *, eta, max_it, period=10, fault=None):
    """the device's PCG on the 9 nc layout in float64: b = P~^T b_full at the leads' and homes' entries, the operator
    q = P~^T K (P~ v) + lambda v, the inverse blocks of device_blocks().  Planted faults: "lambda_per_member" (lambda on the
    expanded vector), "home_masked" (the homes' pose entries held like the other members')"""
    from pcg_replay import block_apply, pcg_replay
    E = embed(lead, home)
    mask = np.ones(E.shape[0])
    if fault == "home_masked":
        mask[rm.held(lead)] = 0.0
    expand = lambda v: Pt @ (E.T @ (mask * v))
    contract = lambda y: mask * (E @ (Pt.T @ y))
    inv = device_blocks(blocks, lam, lead, home, Pt, fault=fault if fault == "home_masked" else None)
    op = lambda v: contract(Hfull @ expand(v)) + lam * v
    if fault == "lambda_per_member":
        op = lambda v: contract(Hfull @ expand(v) + lam * expand(v))
    return pcg_replay(op, contract(b_full), lambda v: block_apply(inv, v), eta=eta, max_it=max_it, period=period)
