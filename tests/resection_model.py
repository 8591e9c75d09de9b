"""An independent float64 model of rba_resect_cameras (DESIGN.md section 26).

Per unit (a free camera, or a rig of >= 2 cameras moving as T_j = M_j T_lead), with the landmarks held:
  usable point  observation in use (W != 0) by a camera with f != 0 whose distortion inverts (triangulation_model.undistort)
  LINEAR        the DLT of the member with the most usable points: p the eigenvector (numpy.linalg.eigh here, not Jacobi) of
                the smallest eigenvalue of sum G^T (I - v v^T) G with P X~ = G p, X~ = ((X - Xbar) / s, 1), v = (m, 1) / |(m, 1)|;
                R the polar factor of A (numpy's SVD here), sigma the mean singular value, t = s b / sigma - R Xbar;
                the lead's pose M_j^-1 T_j; DEGENERATE / BEHIND as the header states
  cost          the unit's share of rba_compute_error: rho(|W r|^2) / 2 of every observation in use by a member (and valid with
                valid_only), the members' camera priors and the pair priors with an endpoint in the unit (counted once),
                each with its loss (observation_loss_model.loss)
  REFINE        Levenberg-Marquardt on that cost in the lead's left increment (v, w, df, dk1, dk2), a member's pose columns
                through its adjoint A_j = [[R_m, [t_m]x R_m], [0, R_m]], restricted to the free entries (the rules of
                section 25)

Built on tests/camera_model.py (projection, Jacobians, validity), tests/camera_prior_model.py and tests/pair_prior_model.py
(the prior residuals and Jacobians) and tests/observation_loss_model.py (the losses).  `fault` plants the mistakes the tests
must reject.  Not collected by pytest (no test_ prefix).
"""
import numpy as np
from scipy.spatial.transform import Rotation

import camera_model as cm
import camera_prior_model as pm
import observation_loss_model as olm
import pair_prior_model as ppm
import triangulation_model as tm

WRITTEN, FEW_POINTS, DEGENERATE, BEHIND, REFINED, CONVERGED, HELD = 1, 2, 4, 8, 16, 32, 64
LINEAR, REFINE, INTRINSICS = 1, 2, 4
FIX_POSE, FIX_F, FIX_K1, FIX_K2 = 1, 2, 4, 8
FAULTS = ("unnormalised_ray", "prior_no_rt", "adjoint_transposed", "ignore_det_sign", "ignore_w", "ignore_loss_weight")


def qmul(a, b):
    """Hamilton product of quaternions (x, y, z, w)"""
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by, aw * by + ay * bw + az * bx - ax * bz,
                     aw * bz + az * bw + ax * by - ay * bx, aw * bw - ax * bx - ay * by - az * bz])


def rot(q):
    """R of a quaternion as the kernels build it from the stored (not normalised) values"""
    return cm.rotation(np.asarray(q, np.float64), device=True)


def adjoint(m, fault=None):
    """A_j of M_j = (q, t) [7]: the first-order map of a lead increment (v, w) to the member's"""
    R = cm.rotation(np.asarray(m[:4], np.float64) / np.linalg.norm(m[:4]))
    A = np.zeros((6, 6))
    A[:3, :3] = R
    A[:3, 3:] = cm.hat(m[4:7]) @ R
    A[3:, 3:] = R
    return A.T if fault == "adjoint_transposed" else A


def tie(m, lead):
    """M_j T_lead [7] in double, the quaternion normalised"""
    q = qmul(m[:4], lead[:4])
    q = q / np.linalg.norm(q)
    t = cm.rotation(np.asarray(m[:4]) / np.linalg.norm(m[:4])) @ np.asarray(lead[4:7], np.float64) + m[4:7]
    return np.concatenate([q, t])


def pose_inv(m):
    q = np.array([-m[0], -m[1], -m[2], m[3]])
    R = cm.rotation(q / np.linalg.norm(q))
    return np.concatenate([q, -R @ m[4:7]])


class Problem:
    """cams [nc, 10] (stored values), lms [nl, 3], obs_cam / obs_lm [nobs], obs [nobs, 2]; W [nobs, 2, 2], kind / a [nobs]
    (the handle's Huber is HUBER with its parameter); cprior (mean [nc, 10], L [nc, 9, 9], kind [nc], a [nc]) or None;
    pprior (pairs [m, 2], mean [m, 7], L [m, 6, 6], kind [m], a [m]) or None; lead [nc] the rig lead (-1 free) and M
    [nc, 7] the member maps (the identity for a lead); fixed [nc] RBA_FIX_* bits; grouped [nc] in an intrinsics group of
    >= 2 cameras"""

    def __init__(self, cams, lms, obs_cam, obs_lm, obs, W=None, kind=None, a=None, valid_only=False, cprior=None,
                 pprior=None, lead=None, M=None, fixed=None, grouped=None, dtype=np.float64):
        self.cams = np.asarray(cams, np.float64).reshape(-1, 10).copy()
        self.lms = np.asarray(lms, np.float64).reshape(-1, 3)
        self.obs_cam, self.obs_lm = np.asarray(obs_cam), np.asarray(obs_lm)
        self.obs = np.asarray(obs, np.float64).reshape(-1, 2)
        n, nc = len(self.obs), len(self.cams)
        self.W = np.broadcast_to(np.eye(2), (n, 2, 2)) if W is None else np.asarray(W, np.float64).reshape(n, 2, 2)
        self.kind = np.zeros(n, int) if kind is None else np.broadcast_to(np.asarray(kind), (n,))
        self.a = np.ones(n) if a is None else np.broadcast_to(np.asarray(a, np.float64), (n,))
        self.valid_only = valid_only
        self.cprior, self.pprior = cprior, pprior
        self.lead = np.full(nc, -1) if lead is None else np.asarray(lead)
        self.M = np.tile([0, 0, 0, 1.0, 0, 0, 0], (nc, 1)) if M is None else np.asarray(M, np.float64)
        self.fixed = np.zeros(nc, int) if fixed is None else np.asarray(fixed, int)
        self.grouped = np.zeros(nc, bool) if grouped is None else np.asarray(grouped, bool)
        self.dtype = dtype
        self.eps = float(cm.EPS_SQRT[np.dtype(dtype)])
        self.by_cam = [np.flatnonzero(self.obs_cam == c) for c in range(nc)]

    def rnd(self, v):
        return np.asarray(np.asarray(v, np.float64).astype(self.dtype), np.float64)

    # ---- units ----
    def unit(self, c):
        """(lead, members ascending) of camera c's unit"""
        ld = int(self.lead[c]) if self.lead[c] >= 0 else c
        if self.lead[c] < 0:
            return ld, [c]
        return ld, [int(j) for j in np.flatnonzero(self.lead == ld)]

    def free(self, c, mode):
        ld, mem = self.unit(c)
        f = int(self.fixed[ld])
        mask = np.zeros(9, bool)
        mask[:6] = not f & FIX_POSE
        if mode & INTRINSICS and len(mem) == 1 and not self.grouped[ld]:
            mask[6:] = [not f & FIX_F, not f & FIX_K1, not f & FIX_K2]
        return mask

    def members_at(self, lead_cam, ld, mem, cams, stored):
        """every member's camera [10] for the lead camera; stored: rounded to Scalar as it would be written"""
        out = {}
        for j in mem:
            if j == ld:
                out[j] = np.asarray(lead_cam, np.float64).copy()
            else:
                p = tie(self.M[j], lead_cam[:7])
                out[j] = np.concatenate([self.rnd(p) if stored else p, cams[j, 7:10]])
        return out

    # ---- usable points and the DLT ----
    def in_use(self, o, fault=None):
        if fault == "ignore_w":
            return np.ones(len(o), bool)
        return np.abs(self.W[o]).reshape(-1, 4).max(1) != 0

    def usable(self, c, fault=None):
        """(observation indices, normalised points m [k, 2]) of camera c's usable points"""
        o = self.by_cam[c]
        cam = self.cams[c]
        idx, ms = [], []
        if cam[7] == 0:
            return np.array(idx, int), np.zeros((0, 2))
        for k, use in zip(o, self.in_use(o, fault)):
            if not use:
                continue
            m, ok = tm.undistort(self.obs[k] / cam[7], cam[8], cam[9])
            if ok:
                idx.append(k)
                ms.append(m)
        return np.array(idx, int), np.array(ms).reshape(-1, 2)

    def linear_condition(self, ld, mem):
        """(eigenvalues of the DLT's M, s, Xbar) of the estimating member: the conditioning of the linear estimate"""
        counts = [len(self.usable(j)[0]) for j in mem]
        idx, m = self.usable(mem[int(np.argmax(counts))])
        X = self.lms[self.obs_lm[idx]]
        xb = X.mean(0)
        s = float(np.sqrt(((X - xb) ** 2).sum(1).mean()))
        Mm = np.zeros((12, 12))
        for i in range(len(idx)):
            G = np.kron(np.eye(3), np.append((X[i] - xb) / s, 1.0)[None, :])
            v = np.array([m[i, 0], m[i, 1], 1.0])
            v /= np.linalg.norm(v)
            Mm += G.T @ (np.eye(3) - np.outer(v, v)) @ G
        return np.linalg.eigvalsh(Mm), s, xb

    def linear(self, ld, mem, fault=None):
        """(lead camera [10] or None, status bits) of the DLT on the member with the most usable points"""
        counts = [len(self.usable(j, fault)[0]) for j in mem]
        b = mem[int(np.argmax(counts))]
        idx, m = self.usable(b, fault)
        if len(idx) < 6:
            return None, DEGENERATE
        X = self.lms[self.obs_lm[idx]]
        xb = X.mean(0)
        d = X - xb
        ev = np.linalg.eigvalsh(d.T @ d)
        if not np.sqrt(max(ev[0], 0.0)) >= 1e-3 * np.sqrt(ev[2]):
            return None, DEGENERATE
        s = float(np.sqrt((d * d).sum(1).mean()))
        s = s if s > 0 else 1.0
        Mm = np.zeros((12, 12))
        for i in range(len(idx)):
            xt = np.append(d[i] / s, 1.0)
            G = np.kron(np.eye(3), xt[None, :])
            v = np.array([m[i, 0], m[i, 1], 1.0])
            if fault != "unnormalised_ray":
                v /= np.linalg.norm(v)
            Mm += G.T @ (np.eye(3) - np.outer(v, v)) @ G
        _, V = np.linalg.eigh(Mm)
        P = V[:, 0].reshape(3, 4)
        A, bb = P[:, :3], P[:, 3]
        det = np.linalg.det(A)
        if det < 0 and fault != "ignore_det_sign":
            A, bb, det = -A, -bb, -det
        if not abs(det) > 1e-10 * np.linalg.norm(A) ** 3:
            return None, DEGENERATE
        U_, sv, Vt = np.linalg.svd(A)
        R = U_ @ Vt
        t = s * bb / sv.mean() - R @ xb
        z = (X @ R.T + t)[:, 2]
        if 2 * np.count_nonzero(~(z >= self.eps)) > len(idx):
            return None, BEHIND
        Tj = np.concatenate([Rotation.from_matrix(R).as_quat(), t])
        Tl = tie(pose_inv(self.M[b]), Tj) if b != ld else Tj
        return np.concatenate([Tl, self.cams[ld, 7:10]]), 0

    # ---- the unit's share of the cost ----
    def cost(self, lead_cam, ld, mem, stored=True, start=None, fault=None, with_normal=False, member_cams=None, terms=None):
        """the unit's share at the lead camera (members tied to it), and with with_normal (H [9, 9], g [9], valid per
        observation of the members); start: the cameras pair endpoints outside the unit are read from"""
        start = self.cams if start is None else start
        cams = self.members_at(lead_cam, ld, mem, start, stored) if member_cams is None else member_cams
        single = len(mem) == 1
        H, g, c = np.zeros((9, 9)), np.zeros(9), 0.0
        valid_all = {}

        def lead_rows(J, j):
            """[rows, 9] of the lead from a member's [rows, 6 or 9]"""
            out = np.zeros((len(J), 9))
            out[:, :6] = J[:, :6] @ (np.eye(6) if single else adjoint(self.M[j], fault))
            if J.shape[1] == 9 and single:
                out[:, 6:] = J[:, 6:]
            return out

        for j in mem:
            o = self.by_cam[j]
            if len(o):
                cj = cams[j]
                L = cm.linearize(np.broadcast_to(cj, (len(o), 10)), self.lms[self.obs_lm[o]], self.obs[o], device_rot=True)
                use = self.in_use(o)
                R = rot(cj[:4])
                z = (self.lms[self.obs_lm[o]] @ R.T + cj[4:7])[:, 2]
                valid = z >= self.eps
                valid_all.update(zip(o.tolist(), valid.tolist()))
                keep = use & (valid | (not self.valid_only))
                W = np.broadcast_to(np.eye(2), (len(o), 2, 2)) if fault == "ignore_w" else self.W[o]
                r = np.einsum("nij,nj->ni", W, L["res"])
                J = W @ np.concatenate([L["Jp"], L["Ji"]], axis=2)
                err, w = olm.loss(self.kind[o], self.a[o], (r * r).sum(1))
                if fault == "ignore_loss_weight":
                    w = np.ones_like(w)
                c += float(err[keep].sum())
                if terms is not None:
                    terms.extend(err[keep].tolist())
                Jk = J[keep]
                JL = np.zeros_like(Jk)
                JL[..., :6] = Jk[..., :6] @ (np.eye(6) if single else adjoint(self.M[j], fault))
                if single:
                    JL[..., 6:] = Jk[..., 6:]
                H += np.einsum("n,nki,nkj->ij", w[keep], JL, JL)
                g += np.einsum("n,nki,nk->i", w[keep], JL, r[keep])
            if self.cprior is not None and np.any(self.cprior[1][j]):
                mean, Lc, pk, pa = (x[j] for x in self.cprior)
                e = pm.residual(cams[j], mean, device_rot=True)
                Jp = pm.jacobian(cams[j], mean, device_rot=True)
                if fault == "prior_no_rt":
                    Jp[:3, :3] = -np.eye(3)
                r = Lc @ e
                pe, pw = olm.loss(pk, pa, r @ r)
                c += float(pe)
                if terms is not None:
                    terms.append(float(pe))
                Jl = lead_rows(Lc @ Jp, j)
                H += float(pw) * Jl.T @ Jl
                g += float(pw) * Jl.T @ r
        if self.pprior is not None:
            pairs, mean, Lp, pk, pa = self.pprior
            for p, (i, j) in enumerate(pairs):
                ini, inj = int(i) in cams, int(j) in cams
                if not (ini or inj):
                    continue
                ci = cams[i] if ini else start[i]
                cj = cams[j] if inj else start[j]
                e = ppm.residual(ci, cj, mean[p], device_rot=True)
                Ji, Jj = ppm.jacobians(ci, cj, mean[p], device_rot=True)
                r = Lp[p] @ e
                pe, pw = olm.loss(pk[p], pa[p], r @ r)
                c += float(pe)
                if terms is not None:
                    terms.append(float(pe))
                Jl = np.zeros((6, 9))
                if ini:
                    Jl[:, :6] += (Lp[p] @ Ji)[:, :6] @ (np.eye(6) if single else adjoint(self.M[i], fault))
                if inj:
                    Jl[:, :6] += (Lp[p] @ Jj)[:, :6] @ (np.eye(6) if single else adjoint(self.M[j], fault))
                H += float(pw) * Jl.T @ Jl
                g += float(pw) * Jl.T @ r
        return (c, H, g, valid_all) if with_normal else c

    def residuals(self, lead_cam, ld, mem):
        """sqrt(2 err) of every term of the unit's share, members tied in double: 1/2 |.|^2 of it is the share"""
        terms = []
        self.cost(lead_cam, ld, mem, False, terms=terms)
        return np.sqrt(2.0 * np.maximum(np.array(terms), 0.0))

    def has_prior(self, mem):
        cp = self.cprior is not None and any(np.any(self.cprior[1][j]) for j in mem)
        pp = self.pprior is not None and any(int(i) in mem or int(j) in mem for i, j in self.pprior[0])
        return cp or pp

    # ---- the refinement ----
    def refine(self, lead_cam, ld, mem, free, stored, max_iterations=20, ftol=1e-10, fault=None):
        """(lead camera, accepted steps, converged): the LM of sections 25 and 26"""
        x = np.asarray(lead_cam, np.float64).copy()
        c, H, g, valid = self.cost(x, ld, mem, stored, fault=fault, with_normal=True)
        use = {int(o): bool(u) for j in mem for o, u in zip(self.by_cam[j], self.in_use(self.by_cam[j]))}
        lam, acc, conv = 1e-4, 0, False
        fi = np.flatnonzero(free)
        for _ in range(max_iterations):
            if lam > 1e16:
                break
            if not np.any(g[fi]):
                conv = True
                break
            Hf = H[np.ix_(fi, fi)]
            dg = np.diag(Hf)
            D = np.maximum(dg, 1e-12 * dg.max())
            try:
                Lc = np.linalg.cholesky(Hf + lam * np.diag(D))
            except np.linalg.LinAlgError:
                lam *= 10
                continue
            dx = np.zeros(9)
            dx[fi] = -np.linalg.solve(Lc.T, np.linalg.solve(Lc, g[fi]))
            xn = pm.apply_inc(x, dx)
            if not np.any(dx[:6]):  # a held pose stays as stored
                xn[:7] = x[:7]
            cn, Hn, gn, vn = self.cost(xn, ld, mem, False, fault=fault, with_normal=True)
            lost = any(use[o] and valid[o] and not vn[o] for o in vn)
            if cn < c and not lost:
                conv = c - cn <= ftol * c
                x, c, H, g, valid, acc = xn, cn, Hn, gn, vn, acc + 1
                lam = max(lam * 0.1, 1e-12)
                if conv:
                    break
            else:
                if not lost and cn - c <= ftol * c:
                    conv = True
                    break
                lam *= 10
        return x, acc, conv

    def resect(self, c, mode=LINEAR | REFINE, max_iterations=20, ftol=1e-10, fault=None):
        """({camera: stored [10]} of the unit after the call, status, points, cost) for camera c's unit, from self.cams"""
        ld, mem = self.unit(c)
        free = self.free(c, mode)
        pts = sum(len(self.usable(j)[0]) for j in mem)
        x = self.cams[ld].copy()
        status, untouched, changed, stored = 0, False, False, False
        if not free.any():
            status, untouched = HELD, True
        elif pts < 3:
            status, untouched = FEW_POINTS, not self.has_prior(mem)
        if mode & LINEAR and free[:6].all() and not untouched:
            y, bits = self.linear(ld, mem, fault)
            status |= bits
            if y is not None:
                x, changed, stored = self.rnd(y), True, True
        cost = self.cost(x, ld, mem, True, fault=fault) if stored else self.cost_stored(ld, mem, fault)
        if mode & REFINE and not untouched:
            xr, acc, conv = self.refine(x, ld, mem, free, stored, max_iterations, ftol, fault)
            status |= CONVERGED if conv else 0
            if acc:
                xr = self.rnd(xr)
                cr = self.cost(xr, ld, mem, True, fault=fault)
                if cr < cost:
                    x, cost, changed = xr, cr, True
                    status |= REFINED
        out = self.members_at(x, ld, mem, self.cams, True) if changed else {j: self.cams[j].copy() for j in mem}
        return out, status | (WRITTEN if changed else 0), pts, cost

    def cost_stored(self, ld, mem, fault=None):
        """the unit's share at the stored cameras (every member as stored, not re-tied)"""
        return self.cost(self.cams[ld], ld, mem, fault=fault, member_cams={j: self.cams[j] for j in mem})
