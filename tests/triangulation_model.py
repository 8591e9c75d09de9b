"""An independent float64 model of rba_triangulate_landmarks (DESIGN.md section 25).

Per landmark, with the cameras held:
  usable ray   observation in use (W != 0), f != 0, distortion invertible: rho (1 + k1 rho^2 + k2 rho^4) = |obs / f| by Newton
               from rho = |obs / f|, failing where 1 + 3 k1 rho^2 + 5 k2 rho^4 <= 0 at an iterate or without convergence;
               direction d = R^T (m, 1) from the centre c = -R^T t
  angle        max over pairs of atan2(|d_i x d_j|, d_i . d_j)
  LINEAR       the smallest eigenvector (numpy.linalg.eigh here, not Jacobi) of sum_i B_i^T (I - v v^T) B_i,
               B_i = [R | (R cbar + t) / s], v = R d / |R d|, in coordinates centred on the mean centre cbar and scaled by the
               RMS distance s of the centres; AT_INFINITY / BEHIND as the header states
  cost         the landmark's share of rba_compute_error: rho(|W r|^2) / 2 of each observation in use (and valid with
               valid_only) + rho(|L e|^2) / 2 of its prior, rho from tests/observation_loss_model.py
  REFINE       Levenberg-Marquardt on that cost with IRLS-weighted normal equations (the rules of section 25)

Built on tests/camera_model.py (projection, Jacobians, validity) and tests/observation_loss_model.py (the losses).  `fault`
plants the mistakes the tests must reject.  Not collected by pytest (no test_ prefix).
"""
import numpy as np

import camera_model as cm
import observation_loss_model as olm

WRITTEN, FEW_RAYS, SMALL_ANGLE, AT_INFINITY, BEHIND, REFINED, CONVERGED = 1, 2, 4, 8, 16, 32, 64
LINEAR, REFINE = 1, 2
FAULTS = ("no_undistort", "no_rt", "ignore_w", "ignore_loss_weight", "flip_cheirality", "acos")
UNDISTORT_ITERS, UNDISTORT_TOL, INFINITY = 50, 1e-12, 1e-10


def undistort(u, k1, k2, fault=None):
    """u = obs / f [2] -> (m [2], ok): the normalised point with u = m (1 + k1 |m|^2 + k2 |m|^4)"""
    u = np.asarray(u, np.float64)
    if fault == "no_undistort":
        return u.copy(), True
    t = float(np.hypot(u[0], u[1]))
    if t == 0.0:
        return np.zeros(2), True
    rho, conv = t, False
    for it in range(UNDISTORT_ITERS + 1):
        r2 = rho * rho
        g1, d = 1 + k1 * r2 + k2 * r2 * r2, 1 + 3 * k1 * r2 + 5 * k2 * r2 * r2
        if not d > 0:
            return None, False
        if conv:
            return u / g1, True
        if it == UNDISTORT_ITERS:
            return None, False
        step = (rho * g1 - t) / d
        rho -= step
        if not (rho > 0 and np.isfinite(rho)):
            return None, False
        conv = abs(step) <= UNDISTORT_TOL * rho
    return None, False


class Track:
    """one landmark: cams [n, 10], obs [n, 2], W [n, 2, 2] (identity without information), kind / a [n] (the observation
    losses; the handle's Huber is HUBER with its parameter), prior (L [3, 3], x0 [3], kind, a) or None"""

    def __init__(self, cams, obs, W=None, kind=None, a=None, prior=None, valid_only=False, dtype=np.float64):
        self.cams = np.asarray(cams, np.float64).reshape(-1, 10)
        self.obs = np.asarray(obs, np.float64).reshape(-1, 2)
        n = len(self.cams)
        self.W = np.broadcast_to(np.eye(2), (n, 2, 2)) if W is None else np.asarray(W, np.float64).reshape(n, 2, 2)
        self.kind = np.zeros(n, int) if kind is None else np.asarray(kind).reshape(n)
        self.a = np.ones(n) if a is None else np.asarray(a, np.float64).reshape(n)
        self.prior = prior
        self.valid_only = valid_only
        self.eps = float(cm.EPS_SQRT[np.dtype(dtype)])
        self.R = cm.rotation(self.cams[:, :4], device=True)
        self.centres = -np.einsum("nji,nj->ni", self.R, self.cams[:, 4:7])

    def in_use(self, fault=None):
        if fault == "ignore_w":
            return np.ones(len(self.cams), bool)
        return np.abs(self.W).reshape(-1, 4).max(1) != 0

    def rays(self, fault=None):
        """(directions [n, 3], usable [n])"""
        d, ok = np.zeros((len(self.cams), 3)), self.in_use(fault) & (self.cams[:, 7] != 0)
        for i in np.flatnonzero(ok):
            f, k1, k2 = self.cams[i, 7:10]
            m, good = undistort(self.obs[i] / f, k1, k2, fault)
            ok[i] = good
            if good:
                v = np.array([m[0], m[1], 1.0])
                d[i] = v if fault == "no_rt" else self.R[i].T @ v
        return d, ok

    def depth(self, X, fault=None):
        z = (self.R @ np.asarray(X, np.float64) + self.cams[:, 4:7])[:, 2]
        return -z if fault == "flip_cheirality" else z

    def cost(self, X, fault=None, with_normal=False):
        """the landmark's share of the cost at X, and with with_normal (H, g) of the IRLS normal equations"""
        X = np.asarray(X, np.float64)
        n = len(self.cams)
        L = cm.linearize(self.cams, np.broadcast_to(X, (n, 3)), self.obs, device_rot=True)
        use = self.in_use(fault)
        valid = self.depth(X) >= self.eps
        keep = use & (valid | (not self.valid_only))
        W = np.broadcast_to(np.eye(2), (n, 2, 2)) if fault == "ignore_w" else self.W
        r = np.einsum("nij,nj->ni", W, L["res"])
        Jl = W @ L["Jl"]
        err, w = olm.loss(self.kind, self.a, (r * r).sum(1))
        if fault == "ignore_loss_weight":
            w = np.ones_like(w)
        c = float(err[keep].sum())
        H = np.einsum("n,nki,nkj->ij", w[keep], Jl[keep], Jl[keep])
        g = np.einsum("n,nki,nk->i", w[keep], Jl[keep], r[keep])
        if self.prior is not None:
            Lp, x0, pk, pa = self.prior
            rp = Lp @ (X - x0)
            pe, pw = olm.loss(pk, pa, rp @ rp)
            c += float(pe)
            H = H + float(pw) * Lp.T @ Lp
            g = g + float(pw) * Lp.T @ rp
        return (c, H, g) if with_normal else c

    def angle(self, fault=None):
        d, ok = self.rays(fault)
        d = d[ok]
        best = 0.0
        for i in range(len(d)):
            for j in range(i + 1, len(d)):
                if fault == "acos":
                    c = d[i] @ d[j] / (np.linalg.norm(d[i]) * np.linalg.norm(d[j]))
                    a = float(np.arccos(np.clip(c, -1, 1)))
                else:
                    a = float(np.arctan2(np.linalg.norm(np.cross(d[i], d[j])), d[i] @ d[j]))
                best = max(best, a)
        return best

    def linear(self, fault=None):
        """(X or None, status bits of the estimate)"""
        d, ok = self.rays(fault)
        c = self.centres[ok]
        cbar = c.mean(0)
        s = float(np.sqrt(((c - cbar) ** 2).sum(1).mean()))
        s = s if s > 0 else 1.0
        M = np.zeros((4, 4))
        for i in np.flatnonzero(ok):
            R, t = self.R[i], self.cams[i, 4:7]
            B = np.hstack([R, ((R @ cbar + t) / s)[:, None]])
            v = R @ d[i]
            v /= np.linalg.norm(v)
            P = np.eye(3) - np.outer(v, v)
            M += B.T @ P @ B
        _, V = np.linalg.eigh(M)
        xh = V[:, 0]
        if not abs(xh[3]) > INFINITY * np.linalg.norm(xh):
            return None, AT_INFINITY
        X = cbar + s * xh[:3] / xh[3]
        if np.any(~(self.depth(X, fault)[ok] >= self.eps)):
            return None, BEHIND
        return X, 0

    def refine(self, X, max_iterations=20, ftol=1e-10, fault=None):
        """(X, accepted steps, converged): the LM of section 25"""
        X = np.asarray(X, np.float64).copy()
        use = self.in_use()
        c, H, g = self.cost(X, fault, True)
        valid = self.depth(X) >= self.eps
        lam, acc, conv = 1e-4, 0, False
        for _ in range(max_iterations):
            if lam > 1e16:
                break
            if not np.any(g):
                conv = True
                break
            dg = np.diag(H)
            D = np.maximum(dg, 1e-12 * dg.max())
            try:
                Lc = np.linalg.cholesky(H + lam * np.diag(D))
            except np.linalg.LinAlgError:
                lam *= 10
                continue
            dx = -np.linalg.solve(Lc.T, np.linalg.solve(Lc, g))
            Xn = X + dx
            cn, Hn, gn = self.cost(Xn, fault, True)
            vn = self.depth(Xn) >= self.eps
            lost = bool(np.any(use & valid & ~vn))
            if cn < c and not lost:
                conv = c - cn <= ftol * c
                X, c, H, g, valid, acc = Xn, cn, Hn, gn, vn, acc + 1
                lam = max(lam * 0.1, 1e-12)
                if conv:
                    break
            else:
                if not lost and cn - c <= ftol * c:
                    conv = True
                    break
                lam *= 10
        return X, acc, conv

    def triangulate(self, X0, mode=LINEAR | REFINE, max_iterations=20, min_angle=0.0, ftol=1e-10, dtype=np.float64,
                    fault=None):
        """(X, status, angle, cost) as rba_triangulate_landmarks gives them for a landmark stored at X0 in `dtype`"""
        rnd = lambda v: np.asarray(v, dtype).astype(np.float64)  # noqa: E731
        X = rnd(X0)
        _, ok = self.rays(fault)
        nr = int(ok.sum())
        ang = self.angle(fault) if nr >= 2 else 0.0
        status = FEW_RAYS if nr < 2 else SMALL_ANGLE if ang < min_angle else 0
        rays_ok, changed = status == 0, False
        if mode & LINEAR and rays_ok:
            Y, bits = self.linear(fault)
            status |= bits
            if Y is not None:
                X, changed = rnd(Y), True
        cost = self.cost(X, fault)
        if mode & REFINE and (rays_ok or (status & FEW_RAYS and self.prior is not None)):
            Xr, acc, conv = self.refine(X, max_iterations, ftol, fault)
            status |= CONVERGED if conv else 0
            if acc:
                Xr = rnd(Xr)
                cr = self.cost(Xr, fault)
                if cr < cost:
                    X, cost, changed = Xr, cr, True
                    status |= REFINED
        return X, status | (WRITTEN if changed else 0), ang, cost


def tracks(arrays, W=None, kind=None, a=None, prior=None, valid_only=False, dtype=np.float64):
    """one Track per landmark of a BalArrays-like problem; W [Nobs, 2, 2], kind / a [Nobs] in problem order, prior
    (idx, mean [m, 3], L [m, 3, 3], kind [m], a [m]) or None"""
    pri = {}
    if prior is not None:
        idx, mean, Ls, pk, pa = prior
        pri = {int(l): (np.asarray(Ls[p], np.float64), np.asarray(mean[p], np.float64), int(pk[p]), float(pa[p]))
               for p, l in enumerate(idx)}
    out = []
    for l in range(len(arrays.lm_off) - 1):
        o0, o1 = int(arrays.lm_off[l]), int(arrays.lm_off[l + 1])
        out.append(Track(arrays.cams[arrays.obs_cam[o0:o1]], arrays.obs_xy[o0:o1], None if W is None else W[o0:o1],
                         None if kind is None else kind[o0:o1], None if a is None else a[o0:o1], pri.get(l), valid_only,
                         dtype))
    return out
