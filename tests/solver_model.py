"""A float64 model of the Schur-complement (SC) elimination of the landmarks, per landmark and per camera, with the
componentwise bar of every quantity for an implementation in a scalar type of unit round-off u.

Written from the mathematics (DESIGN.md section 12), not from the oracle or the kernels.  Rows: camera_model.weighted() on
the state cast to the solver's type -- per observation the weighted Jp (2 x 9: pose, then intrinsics), Jl (2 x 3) and r (2),
rows of observations that use_valid_projections_only drops set to 0.  Scaled as the solvers scale them: Jp_s = Jp diag(D)
with the solver's OWN Jacobi scaling D (get_jacobian_scaling or the oracle's scl_get_scaling, so D enters exactly) and
Jl_s = Jl diag(jls) with the model's jls = 1 / (eps + |Jl column|), eps = camera_model.EPS_SQRT of the type.  Per landmark,
observations i (camera c_i), in float64:

  Hll     = Jl_s^T Jl_s + lam I            (3 x 3; R its Cholesky factor, Hll = R^T R)
  s       = Hll^-1 Jl_s^T r
  b_c     = sum_{i at c} Jp_i^T (r_i - Jl_i s)                                   (two parts: Jp^T r, and the rr part Jp^T Jl s)
  SJ_c    = sum_{i at c} (Jp_i^T Jp_i - Jp_i^T Jl_i Hll^-1 Jl_i^T Jp_i) + lam I   (SCHUR_JACOBI blocks)
  J_c     = sum_{i at c} Jp_i^T Jp_i + lam I                                     (JACOBI blocks; Power-SC's Hpp + lam I)
  E0 x    = sum_landmarks sum_i Jp_i^T Jl_i Hll^-1 sum_j Jl_j^T Jp_j x_{c_j}
  H x     = sum_i Jp_i^T Jp_i x_{c_i} - E0 x + lam x
  t       = Hll^-1 Jl_s^T (r + Jp_s dp),   landmark update  dl = -jls * t
  l_diff  = -sum_k j_k (j_k / 2 + r_k),    j = Jp_s dp - Jl_s t   (k over the 2 n rows of every landmark)

Bars.  Each quantity Q comes with a magnitude M_Q >= 0, and an implementation is accepted when, entry by entry,
    |Q_got - Q| <= c u M_Q.
M_Q is Q evaluated on magnitudes: every row entry replaced by the magnitude of its linearisation error (below), r by the
rounding scale sqrt(w) (|proj| + |obs|) of a residual computed as proj - obs, products and sums by the products and sums
of magnitudes, and the landmark block by
    W   = |R^-1| |R^-T|  (>= |Hll^-1| entrywise),        M_H = sqrt(d d^T), d = diag(|Jl_s|^T |Jl_s|) + lam
(M_H dominates |Jl_s|^T |Jl_s| and |R^T| |R| by Cauchy-Schwarz).  A solve y = Hll^-1 v enters as W (M_H |y| + M_v): a
backward-stable solve -- Cholesky with substitution (Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed.,
Thm 10.3 and 8.5) or the reference's explicit 3 x 3 inverse -- solves a system perturbed by O(u) M_H, and the first-order
error of the solution is Hll^-1 dH y; so the Skeel condition || |Hll^-1| |Hll| || of the landmark block enters explicitly,
squared relative to the square-root solver's |R^-1| |R| (the Schur complement forms the normal equations).  A product
with Hll^-1 inside a sum (E0, the SCHUR_JACOBI term) enters as W + W M_H W.  The inverse of a 9 x 9 block B has magnitude
W_B M_B' W_B with W_B = |L^-T| |L^-1| (B = L L^T) and M_B' = sqrt(d d^T), d the diagonal of M_B: the first-order
perturbation B^-1 dB B^-1 of a backward-stable Cholesky inversion.

The magnitude of a row entry: the pose part of a row is d proj / d pc [I | -[pc]x], a sum of products, so its error is
relative to the row's largest pose entry; an intrinsic entry (m rp, f m r2, f m r2^2) is a product, so its error is
relative to the larger of the observation's two rows in that column; Jl uses the row's largest entry; each times its
column's scaling.  The constant, for a problem whose longest track has n observations and whose busiest camera m:
    c = 2 n + m + 128 + 2 * 256 kappa
  2 n        the sums over the 2 n rows of a landmark (Hll, Jl^T r, Jl^T Jp x): Higham's gamma_k for any summation order
  m          the per-camera sums over its observations (b, blocks, H x)
  128        work of fixed length: the 3 x 3 Cholesky and its substitutions (gamma_10), the 9-term products Jp x (gamma_9),
             the 9 x 9 Cholesky inverse (gamma_10 + 2 gamma_9), the scaling of the landmark update, a u per factor of
             the longest product (Jp^T Jl Hll^-1 Jl^T Jp), rounded up
  256 kappa  the linearisation of one observation against the model (c_lin of test_gpu_observation_model); it covers the
             solver's jls too, a column norm of the same rows.  Twice: every term is bilinear in the linearised rows
  kappa      the largest camera_model.condition() of the problem's observations
In units of u M the float32 oracle stays below 1.1 on the test problems, so c leaves a margin of several hundred.
The landmark update is held to c u M_dl + u (|dl| + |p_new|): the last term is the rounding of the new position in the
solver's type.  In float64 c u stays below 1e-9 on the problems of the tests (test_solver_model checks it).
"""
import numpy as np

import camera_model as cm

C_FIXED = 128
C_LIN = 256


def unit_roundoff(dtype):
    return float(np.finfo(dtype).eps) / 2


def bar_constant(n, m, kappa):
    return 2 * n + m + C_FIXED + 2 * C_LIN * kappa


def _sqrt_outer(M):
    d = np.sqrt(np.diag(M))
    return np.outer(d, d)


def _chol_weights(B):
    """|L^-T| |L^-1| of B = L L^T (or |R^-1| |R^-T| of B = R^T R, the same matrix)"""
    Li = np.abs(np.linalg.inv(np.linalg.cholesky(B)))
    return Li.T @ Li


def inverse(B, M):
    """B^-1 of a symmetric positive definite block and its magnitude W_B M_B' W_B (see the module docstring)"""
    W = _chol_weights(B)
    return np.linalg.inv(B), W @ _sqrt_outer(M) @ W


class SCModel:
    def __init__(self, arrays, dtype, D, lam, threshold=None, valid_only=False):
        a = arrays.cast(dtype)
        self.arrays, self.dtype = a, dtype
        self.lam = float(dtype(lam))
        self.u = unit_roundoff(dtype)
        nc, nl = a.nc, a.nl
        self.nc, self.nl = nc, nl
        jp, jl, r, keep, rmag = cm.weighted(a, dtype=dtype, threshold=threshold, valid_only=valid_only, magnitude=True)
        self.keep = keep
        D = np.asarray(D, np.float64).reshape(nc, 9)
        lm_of_obs = np.repeat(np.arange(nl), a.track_lengths())
        l2 = np.zeros((nl, 3))
        np.add.at(l2, lm_of_obs, (jl ** 2).sum(1))
        self.jls = 1 / (float(cm.EPS_SQRT[np.dtype(dtype)]) + np.sqrt(l2))
        self.cam = np.asarray(a.obs_cam)
        self.off = np.asarray(a.lm_off)
        Dc, jc = D[self.cam][:, None, :], self.jls[lm_of_obs][:, None, :]
        self.Jp, self.Jl, self.r = jp * Dc, jl * jc, r
        ajp = np.abs(jp)
        ajp[:, :, :6] = ajp[:, :, :6].max(2, keepdims=True)   # pose: the row's largest pose entry
        ajp[:, :, 6:] = ajp[:, :, 6:].max(1, keepdims=True)   # intrinsics: the larger of the observation's two rows
        self.aJp = ajp * Dc
        self.aJl = np.abs(jl).max(2, keepdims=True) * jc
        self.ar = rmag
        n = int(a.track_lengths().max())
        m = int(np.bincount(self.cam, minlength=nc).max())
        self.kappa = float(cm.condition(a, dtype, threshold).max())
        self.c = bar_constant(n, m, self.kappa)
        eye = np.eye(3)
        self.Hll, self.MH = [], []
        for lm in range(nl):
            J, aJ = self._rows(self.Jl, lm).reshape(-1, 3), self._rows(self.aJl, lm).reshape(-1, 3)
            self.Hll.append(J.T @ J + self.lam * eye)
            self.MH.append(_sqrt_outer(aJ.T @ aJ + self.lam * eye))
        self._factor()

    def _rows(self, v, lm):
        return v[self.off[lm]:self.off[lm + 1]]

    def _factor(self):
        self.Hinv = [np.linalg.inv(H) for H in self.Hll]
        self.W = [_chol_weights(H) for H in self.Hll]

    def set_hll(self, lm, H):
        """replace one landmark block (a test plants errors through this)"""
        self.Hll[lm] = H
        self._factor()

    def _solve(self, lm, v, Mv):
        y = self.Hinv[lm] @ v
        return y, self.W[lm] @ (self.MH[lm] @ np.abs(y) + Mv)

    def _per_camera(self, lm, vals, out):
        np.add.at(out, self.cam[self.off[lm]:self.off[lm + 1]], vals)

    # ---- right-hand side ----
    def gradient_parts(self):
        """(sum Jp_i^T r_i, sum Jp_i^T Jl_i s) per camera [nc, 9] and the magnitude of b = first - second"""
        p1, p2, M = (np.zeros((self.nc, 9)) for _ in range(3))
        for lm in range(self.nl):
            Jp, Jl, r = self._rows(self.Jp, lm), self._rows(self.Jl, lm), self._rows(self.r, lm)
            aJp, aJl, ar = self._rows(self.aJp, lm), self._rows(self.aJl, lm), self._rows(self.ar, lm)
            g = np.einsum("kra,kr->a", Jl, r)
            s, Ms = self._solve(lm, g, np.einsum("kra,kr->a", aJl, ar))
            self._per_camera(lm, np.einsum("krc,kr->kc", Jp, r), p1)
            self._per_camera(lm, np.einsum("krc,kra,a->kc", Jp, Jl, s), p2)
            self._per_camera(lm, np.einsum("krc,kr->kc", aJp, ar + aJl @ (np.abs(s) + Ms)), M)
        return p1, p2, M

    def b(self):
        p1, p2, M = self.gradient_parts()
        return p1 - p2, M

    # ---- preconditioner blocks ----
    def jacobi_blocks(self):
        """sum Jp_i^T Jp_i + lam I per camera [nc, 9, 9] and its magnitude"""
        B = np.zeros((self.nc, 9, 9))
        M = np.zeros((self.nc, 9, 9))
        np.add.at(B, self.cam, np.einsum("krc,krd->kcd", self.Jp, self.Jp))
        np.add.at(M, self.cam, np.einsum("krc,krd->kcd", self.aJp, self.aJp))
        return B + self.lam * np.eye(9), M + self.lam * np.eye(9)

    def schur_blocks(self):
        """the SCHUR_JACOBI blocks + lam I per camera [nc, 9, 9] and their magnitude"""
        B, M = self.jacobi_blocks()
        for lm in range(self.nl):
            T = np.einsum("kra,krc->kac", self._rows(self.Jl, lm), self._rows(self.Jp, lm))
            aT = np.einsum("kra,krc->kac", self._rows(self.aJl, lm), self._rows(self.aJp, lm))
            W = self.W[lm]
            self._per_camera(lm, -np.einsum("kac,ab,kbd->kcd", T, self.Hinv[lm], T), B)
            self._per_camera(lm, np.einsum("kac,ab,kbd->kcd", aT, W + W @ self.MH[lm] @ W, aT), M)
        return B, M

    # ---- operator ----
    def e0(self, x, landmarks=None):
        """E0 x per camera [nc, 9] and its magnitude; `landmarks`: the landmarks that contribute (default all)"""
        x = np.asarray(x, np.float64).reshape(self.nc, 9)
        y, M = np.zeros((self.nc, 9)), np.zeros((self.nc, 9))
        for lm in (range(self.nl) if landmarks is None else landmarks):
            cams = self.cam[self.off[lm]:self.off[lm + 1]]
            T = np.einsum("kra,krc->kac", self._rows(self.Jl, lm), self._rows(self.Jp, lm))
            aT = np.einsum("kra,krc->kac", self._rows(self.aJl, lm), self._rows(self.aJp, lm))
            w, Mw = self._solve(lm, np.einsum("kac,kc->a", T, x[cams]), np.einsum("kac,kc->a", aT, np.abs(x[cams])))
            self._per_camera(lm, np.einsum("kac,a->kc", T, w), y)
            self._per_camera(lm, np.einsum("kac,a->kc", aT, np.abs(w) + Mw), M)
        return y, M

    def hx(self, x):
        """H x = sum Jp^T Jp x - E0 x + lam x per camera [nc, 9] and its magnitude"""
        x = np.asarray(x, np.float64).reshape(self.nc, 9)
        e0, M = self.e0(x)
        y = np.zeros((self.nc, 9))
        np.add.at(y, self.cam, np.einsum("krc,krd,kd->kc", self.Jp, self.Jp, x[self.cam]))
        np.add.at(M, self.cam, np.einsum("krc,krd,kd->kc", self.aJp, self.aJp, np.abs(x[self.cam])))
        return y - e0 + self.lam * x, M + self.lam * np.abs(x)

    # ---- back-substitution ----
    def back_substitute(self, dp):
        """(t [nl, 3], its magnitude, dl = -jls t, its magnitude, l_diff, its magnitude) for the pose increment dp"""
        dp = np.asarray(dp, np.float64).reshape(self.nc, 9)
        t, Mt = np.zeros((self.nl, 3)), np.zeros((self.nl, 3))
        l_diff = l_mag = 0.0
        for lm in range(self.nl):
            cams = self.cam[self.off[lm]:self.off[lm + 1]]
            Jp, Jl, r = self._rows(self.Jp, lm), self._rows(self.Jl, lm), self._rows(self.r, lm)
            aJp, aJl, ar = self._rows(self.aJp, lm), self._rows(self.aJl, lm), self._rows(self.ar, lm)
            Jpdp, aJpdp = np.einsum("krc,kc->kr", Jp, dp[cams]), np.einsum("krc,kc->kr", aJp, np.abs(dp[cams]))
            t[lm], Mt[lm] = self._solve(lm, np.einsum("kra,kr->a", Jl, r + Jpdp), np.einsum("kra,kr->a", aJl, ar + aJpdp))
            j = Jpdp - Jl @ t[lm]
            Mj = aJpdp + aJl @ (np.abs(t[lm]) + Mt[lm])
            l_diff -= float(np.sum(j * (0.5 * j + r)))
            l_mag += float(np.sum(Mj * (np.abs(j) + ar) + np.abs(j) * ar))
        dl = -self.jls * t
        return t, Mt, dl, self.jls * (np.abs(t) + Mt), l_diff, l_mag


# ---- checkers ----
def excess(got, want, mag, c, u):
    """the largest |got - want| / (c u mag) and where it is (<= 1: accepted)"""
    got, want, mag = (np.asarray(v, np.float64) for v in (got, want, mag))
    got = got.reshape(want.shape)
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.abs(got - want) / (c * u * mag)
    ratio = np.where(got == want, 0.0, ratio)
    ratio = np.where(np.isnan(ratio), np.inf, ratio)
    k = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
    return float(ratio[k]), k


def check(got, want, mag, model, what):
    e, k = excess(got, want, mag, model.c, model.u)
    assert e <= 1, (what, "entry", k, "error / bar", e)


def check_landmark_update(got, model, dl, Mdl, p_new, what="landmark update"):
    """got [nl, 3]: the change of every landmark; p_new its new position (rounding of the position in the solver's type)"""
    got = np.asarray(got, np.float64).reshape(-1, 3)
    mag = Mdl + (np.abs(dl) + np.abs(np.asarray(p_new, np.float64).reshape(-1, 3))) / model.c
    check(got, dl, mag, model, what)


def check_inverse(got, B, MB, model, what):
    """got [nc, 9, 9] against the inverse of every block of B (magnitudes MB)"""
    for c in range(B.shape[0]):
        want, M = inverse(B[c], MB[c])
        e, k = excess(got[c], want, M, model.c, model.u)
        assert e <= 1, (what, "camera", c, "entry", k, "error / bar", e)
