"""An independent float64 model of per-observation square-root information (rba_set_observation_info, DESIGN.md section 19).

  observation o with the row-major 2x2 W_o:  whitened residual W_o r, cost rho(|W_o r|^2) (rho the Huber norm in units of sigma,
  1/2 s without one), rows of the Jacobian sqrt(hw) W_o [Jp | Jl | r] with hw the robust weight at |W_o r|^2.
  W_o = 0 switches the observation off: zero rows, counted in "all" only.

Built on tests/camera_model.py (linearize, huber).  `fault` plants the mistakes the tests must reject.  Not collected by
pytest (no test_ prefix).
"""
import numpy as np

import camera_model as cm

FAULTS = ("r_only", "transposed", "huber_unwhitened", "off_counted_valid")


def expand(info, nobs):
    """[nobs] (1 / sigma) or [nobs, 2, 2] -> [nobs, 2, 2] float64"""
    a = np.asarray(info, np.float64)
    if a.shape == (nobs,):
        return a[:, None, None] * np.eye(2)
    assert a.shape == (nobs, 2, 2), a.shape
    return a


def random_info(nobs, seed, cond=10.0, lo=0.3, hi=3.0):
    """well-conditioned W: U diag(s, s / k) V^T with s in [lo, hi] (log-uniform), k in [1, cond], U, V random rotations or
    reflections (so W is neither symmetric nor triangular)"""
    rng = np.random.default_rng(seed)

    def orth():
        a = rng.uniform(0, 2 * np.pi, nobs)
        Q = np.stack([np.stack([np.cos(a), -np.sin(a)], -1), np.stack([np.sin(a), np.cos(a)], -1)], -2)
        Q[rng.random(nobs) < 0.5, :, 1] *= -1
        return Q
    s = np.exp(rng.uniform(np.log(lo), np.log(hi), nobs))
    k = rng.uniform(1.0, cond, nobs)
    S = np.zeros((nobs, 2, 2))
    S[:, 0, 0], S[:, 1, 1] = s, np.maximum(s / k, lo / cond)
    return orth() @ S @ np.swapaxes(orth(), 1, 2)


def whitened(arrays, W, dtype=np.float64, threshold=None, valid_only=False, fault=None, device_rot=False):
    """per observation the rows sqrt(hw) W [Jp (2x9) | Jl (2x3) | r], the whitened residual W r, hw, the projection validity
    and the in-use mask (W != 0).  Rows of a switched-off observation, and with valid_only of an invalid projection, are 0.
    device_rot: rotations as the kernels build them (camera_model.linearize)."""
    L = cm.linearize(*cm.observations(arrays), dtype=dtype, device_rot=device_rot)
    W = expand(W, len(L["res"]))
    on = np.any(W.reshape(-1, 4) != 0, axis=1)
    Wj = np.swapaxes(W, 1, 2) if fault == "transposed" else W
    with np.errstate(invalid="ignore"):
        wr = np.einsum("oij,oj->oi", Wj, L["res"])
        Jp = Wj @ np.concatenate([L["Jp"], L["Ji"]], axis=2)
        Jl = Wj @ L["Jl"]
    if fault == "r_only":
        Jp, Jl = np.concatenate([L["Jp"], L["Ji"]], axis=2), L["Jl"].copy()
    wr[~on] = 0.0
    rsq = (wr ** 2).sum(1)
    _, hw = cm.huber((L["res"] ** 2).sum(1) if fault == "huber_unwhitened" else rsq, threshold)
    keep = on & (L["valid"] if valid_only else True)
    sw = np.sqrt(hw)[:, None]
    Jp, Jl, r = Jp * sw[:, :, None], Jl * sw[:, :, None], wr * sw
    Jp[~keep], Jl[~keep], r[~keep] = 0.0, 0.0, 0.0
    return dict(Jp=Jp, Jl=Jl, r=r, wr=wr, hw=hw, valid=L["valid"], on=on, keep=keep)


def dense_system(arrays, W, **kw):
    """the dense (Jp, Jl, r) objective_checks.reduced takes, from the whitened rows"""
    w = whitened(arrays, W, **kw)
    nobs, nc, nl = len(w["r"]), arrays.cams.shape[0], arrays.lms.shape[0]
    Jp, Jl = np.zeros((2 * nobs, 9 * nc)), np.zeros((2 * nobs, 3 * nl))
    lm_of_obs = np.repeat(np.arange(nl), np.diff(arrays.lm_off))
    for k in range(nobs):
        c, l = int(arrays.obs_cam[k]), int(lm_of_obs[k])
        Jp[2 * k:2 * k + 2, 9 * c:9 * c + 9] = w["Jp"][k]
        Jl[2 * k:2 * k + 2, 3 * l:3 * l + 3] = w["Jl"][k]
    return Jp, Jl, w["r"].ravel()


def residual_info(arrays, W, dtype=np.float64, threshold=None, fault=None):
    """the sums rba_compute_error reports: a switched-off observation stays in "all" (adding 0) and is not in "valid" """
    w = whitened(arrays, W, dtype=dtype, threshold=threshold)
    rsq = (w["wr"] ** 2).sum(1)
    err, _ = cm.huber(rsq, threshold)
    valid = w["valid"] if fault == "off_counted_valid" else w["valid"] & w["on"]
    out = {}
    for key, sel in (("all", np.ones(len(rsq), bool)), ("valid", valid)):
        out[key] = {"num_obs": int(sel.sum()), "error": float(err[sel].sum()), "residual_sum": float(np.sqrt(rsq[sel]).sum())}
    return out


def cost(arrays, W, threshold=None):
    return residual_info(arrays, W, threshold=threshold)["all"]["error"]


def without(arrays, off):
    """the problem with the observations `off` (bool [nobs]) removed from the CSR, and the kept observations' indices"""
    from rootba_b200.synthetic import BalArrays
    keep = ~np.asarray(off, bool)
    lm_of_obs = np.repeat(np.arange(arrays.lms.shape[0]), np.diff(arrays.lm_off))
    counts = np.bincount(lm_of_obs[keep], minlength=arrays.lms.shape[0])
    lm_off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    return BalArrays(arrays.cams, arrays.lms, lm_off, arrays.obs_cam[keep], arrays.obs_xy[keep]), np.flatnonzero(keep)
