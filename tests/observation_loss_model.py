"""An independent float64 model of the robust loss per observation (rba_set_observation_loss, DESIGN.md section 21).

  observation o with the loss kind[o], the scale a = scale[o] and the square-root information W_o (identity without one):
  s = |W_o r|^2, cost rho(s) / 2, robust weight w = rho'(s), rows sqrt(w) W_o [Jp | Jl | r].
  NONE rho = s; HUBER s below a^2, else 2 a sqrt(s) - a^2; CAUCHY a^2 log1p(s / a^2); SOFT_L1 2 a^2 (sqrt(1 + s / a^2) - 1);
  TUKEY (a^2 / 3) (1 - (1 - s / a^2)^3) below a^2, else a^2 / 3.  A Tukey observation beyond its scale has w = 0: zero rows,
  still counted as valid, with the cost a^2 / 6.

Built on tests/camera_model.py (linearize, huber) and tests/observation_info_model.py (the whitening).  `fault` plants the
mistakes the tests must reject.  Not collected by pytest (no test_ prefix).
"""
import numpy as np

import camera_model as cm
import observation_info_model as om

NONE, HUBER, CAUCHY, SOFT_L1, TUKEY = range(5)
NAMES = ("NONE", "HUBER", "CAUCHY", "SOFT_L1", "TUKEY")
FAULTS = ("unwhitened", "w_is_rho", "s_over_a", "ceres_tukey", "tukey_zero_not_valid", "slot_order")


def loss(kind, a, s, fault=None):
    """(rho(s) / 2, w) per entry of the arrays kind, a, s (broadcast), in float64"""
    kind, a, s = np.broadcast_arrays(np.asarray(kind), np.asarray(a, np.float64), np.asarray(s, np.float64))
    a2 = a * a if fault != "s_over_a" else a
    u = s / np.where(kind == NONE, 1.0, a2)
    err, w = 0.5 * s, np.ones_like(s)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.sqrt(s)
        inside = r <= a
        e_h, w_h = np.where(inside, 0.5 * s, a * r - 0.5 * a * a), np.where(inside, 1.0, a / r)
        t = np.sqrt(1.0 + u)
        table = {
            HUBER: (e_h, w_h),
            CAUCHY: (0.5 * a2 * np.log1p(u), 1.0 / (1.0 + u)),
            SOFT_L1: (s / (t + 1.0), 1.0 / t),
            TUKEY: (np.where(u < 1, a2 / 6.0 * u * (3.0 - 3.0 * u + u * u), a2 / 6.0), np.where(u < 1, (1.0 - u) ** 2, 0.0)),
        }
    for k, (e, ww) in table.items():
        sel = kind == k
        err = np.where(sel, e, err)
        w = np.where(sel, ww, w)
    if fault == "ceres_tukey":
        sel = kind == TUKEY
        err, w = np.where(sel, 0.5 * err, err), np.where(sel, 0.5 * w, w)
    if fault == "w_is_rho":
        w = 2.0 * err
    return err, w


def in_slot_order(arrays, kind, scale):
    """the arrays permuted as if they were read in slot order (landmarks longest track first) instead of problem order: the
    planted fault slot_order"""
    n = np.diff(arrays.lm_off)
    order = np.argsort(-n, kind="stable")
    perm = np.concatenate([np.arange(arrays.lm_off[l], arrays.lm_off[l + 1]) for l in order])
    return np.asarray(kind)[perm], np.asarray(scale)[perm]


def rows(arrays, kind, scale, W=None, dtype=np.float64, valid_only=False, fault=None):
    """per observation the rows sqrt(w) W [Jp (2x9) | Jl (2x3) | r], W r, s, w, err, the projection validity and the in-use
    mask (W != 0)"""
    nobs = len(arrays.obs_cam)
    if fault == "slot_order":
        kind, scale = in_slot_order(arrays, kind, scale)
    W = np.broadcast_to(np.eye(2), (nobs, 2, 2)) if W is None else om.expand(W, nobs)
    w0 = om.whitened(arrays, W, dtype=dtype)  # unit weights: the whitened rows
    L = cm.linearize(*cm.observations(arrays), dtype=dtype)
    s = (w0["wr"] ** 2).sum(1) if fault != "unwhitened" else (L["res"] ** 2).sum(1)
    err, w = loss(kind, scale, s, fault)
    keep = w0["on"] & (L["valid"] if valid_only else True)
    sw = np.where(keep, np.sqrt(w), 0.0)
    Jp = w0["Jp"] * sw[:, None, None]
    Jl = w0["Jl"] * sw[:, None, None]
    r = w0["wr"] * sw[:, None]
    err = np.where(w0["on"], err, 0.0)
    return dict(Jp=Jp, Jl=Jl, r=r, wr=w0["wr"], s=s, w=w, err=err, valid=L["valid"], on=w0["on"], keep=keep)


def dense_system(arrays, kind, scale, W=None, **kw):
    """the dense (Jp, Jl, r) objective_checks.reduced takes, from the weighted rows"""
    w = rows(arrays, kind, scale, W, **kw)
    nobs, nc, nl = len(w["r"]), arrays.cams.shape[0], arrays.lms.shape[0]
    Jp, Jl = np.zeros((2 * nobs, 9 * nc)), np.zeros((2 * nobs, 3 * nl))
    lm_of_obs = np.repeat(np.arange(nl), np.diff(arrays.lm_off))
    for k in range(nobs):
        c, l = int(arrays.obs_cam[k]), int(lm_of_obs[k])
        Jp[2 * k:2 * k + 2, 9 * c:9 * c + 9] = w["Jp"][k]
        Jl[2 * k:2 * k + 2, 3 * l:3 * l + 3] = w["Jl"][k]
    return Jp, Jl, w["r"].ravel()


def residual_info(arrays, kind, scale, W=None, dtype=np.float64, fault=None):
    """the sums rba_compute_error reports: a switched-off observation is in "all" only (adding 0); a Tukey observation with
    w = 0 stays valid and adds a^2 / 6"""
    w = rows(arrays, kind, scale, W, dtype=dtype, fault=fault)
    valid = w["valid"] & w["on"]
    if fault == "tukey_zero_not_valid":
        valid = valid & (w["w"] > 0)
    out = {}
    for key, sel in (("all", np.ones(len(w["s"]), bool)), ("valid", valid)):
        out[key] = {"num_obs": int(sel.sum()), "error": float(w["err"][sel].sum()), "residual_sum": float(np.sqrt(w["s"][sel]).sum())}
    return out


def cost(arrays, kind, scale, W=None, fault=None):
    return residual_info(arrays, kind, scale, W, fault=fault)["all"]["error"]


def mixed(nobs, seed, kinds=(NONE, HUBER, CAUCHY, SOFT_L1, TUKEY), lo=0.5, hi=3.0):
    """a random kind per observation from `kinds` and a log-uniform scale in [lo, hi] (NaN for NONE: ignored)"""
    rng = np.random.default_rng(seed)
    kind = rng.choice(np.asarray(kinds, np.uint8), nobs)
    scale = np.exp(rng.uniform(np.log(lo), np.log(hi), nobs))
    scale[kind == NONE] = np.nan
    return kind, scale
