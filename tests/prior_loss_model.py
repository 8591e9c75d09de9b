"""An independent float64 model of the robust losses on the priors (rba_set_prior_loss, DESIGN.md section 22).

  prior p of any kind, with the whitened residual L_p e_p of its own model (tests/camera_prior_model.py,
  tests/pair_prior_model.py, tests/landmark_prior_model.py) and s_p = |L_p e_p|^2: cost rho(s_p) / 2, weight w_p = rho'(s_p),
  rows sqrt(w_p) L_p de/d(inc) and sqrt(w_p) L_p e_p.  rho is that of tests/observation_loss_model.py, one weight per prior.

Because every row of a prior is linear in L, the weighted rows are the prior's own rows with L replaced by sqrt(w) L:
`weighted` gives those prior tuples, which tests/objective_checks.py's dense_system takes as they are.  `fault` plants the
mistakes the tests must reject.  Not collected by pytest (no test_ prefix).
"""
import numpy as np

import camera_prior_model as pm
import landmark_prior_model as lp
import observation_loss_model as olm
import pair_prior_model as qm

CAMERA, PAIR, LANDMARK = range(3)
KINDS = ("camera", "pairs", "landmarks")  # the keyword of each prior kind in objective_checks
FAULTS = ("w_not_sqrt_w", "s_not_rho", "tukey_no_constant", "shift_after_drop")


def whitened(kind, state, prior):
    """[m, 9 | 6 | 3] L e of every prior of one kind at state = (cams, lms), in the caller's order"""
    cams, lms = state
    if kind == CAMERA:
        return pm.rows(cams, *prior)[1]
    if kind == PAIR:
        return qm.rows(cams, *prior)[1].reshape(-1, 6)
    return lp.rows(lms, *prior)[1]


def dropped(kind, prior):
    """[m] bool: the priors the handle drops for an all-zero L (pairs and landmark priors; a camera keeps its item)"""
    if kind == CAMERA:
        return np.zeros(len(prior[-1]), bool)
    return ~np.any(np.asarray(prior[-1]).reshape(len(prior[-1]), -1) != 0, axis=1)


def loss_of(kind, prior, loss, fault=None):
    """(kind [m], scale [m]) as the handle applies them; the planted fault shift_after_drop moves every loss after the first
    dropped prior one entry later"""
    k, a = np.asarray(loss[0]), np.asarray(loss[1], np.float64)
    if fault == "shift_after_drop":
        d = np.flatnonzero(dropped(kind, prior))
        if len(d):
            k, a = k.copy(), a.copy()
            k[d[0] + 1:], a[d[0] + 1:] = np.asarray(loss[0])[d[0]:-1], np.asarray(loss[1], np.float64)[d[0]:-1]
    return k, a


def weights(kind, state, prior, loss, fault=None):
    """(s, err = rho(s) / 2, w) per prior of one kind at `state`"""
    r = whitened(kind, state, prior)
    s = np.sum(r * r, axis=1)
    k, a = loss_of(kind, prior, loss, fault)
    err, w = olm.loss(k, a, s)
    if fault == "s_not_rho":
        err = 0.5 * s
    if fault == "tukey_no_constant":
        err = np.where((k == olm.TUKEY) & (w == 0), 0.0, err)
    return s, err, w


def weighted(kind, state, prior, loss, fault=None, at=None):
    """the prior tuple with L_p replaced by sqrt(w_p) L_p, w at `at` (default `state`); w_not_sqrt_w plants w L"""
    _, _, w = weights(kind, state if at is None else at, prior, loss, fault)
    f = w if fault == "w_not_sqrt_w" else np.sqrt(w)
    L = np.asarray(prior[-1], np.float64)
    return tuple(prior[:-1]) + (L * f.reshape((-1,) + (1,) * (L.ndim - 1)),)


def weighted_all(state, priors, losses, fault=None, at=None):
    """objective_checks keywords (camera, pairs, landmarks) of the weighted priors; `losses` maps a kind to (kind, scale) or
    None (NONE)"""
    out = {}
    for k, name in enumerate(KINDS):
        p = priors.get(name)
        if p is None:
            out[name] = None
        elif losses.get(k) is None:
            out[name] = p
        else:
            out[name] = weighted(k, state, p, losses[k], fault, at)
    return out


def prior_cost(state, priors, losses, fault=None):
    """sum over every prior of rho(s)/2 (1/2 s without a loss)"""
    c = 0.0
    for k, name in enumerate(KINDS):
        p = priors.get(name)
        if p is None:
            continue
        if losses.get(k) is None:
            c += 0.5 * float(np.sum(whitened(k, state, p) ** 2))
        else:
            c += float(np.sum(weights(k, state, p, losses[k], fault)[1]))
    return c


def irls_gradient(kind, state, prior, loss):
    """the gradient of sum rho(|L e|^2)/2 over the increment of one prior kind by IRLS: sum_p w_p (L_p J_p)^T (L_p e_p), in the
    increment's layout [9 nc] (cameras) or [3 nl] (landmarks)"""
    cams, lms = state
    _, _, w = weights(kind, state, prior, loss)
    if kind == CAMERA:
        A, r = pm.rows(cams, *prior)
        return np.concatenate([w[c] * A[c].T @ r[c] for c in range(len(cams))])
    if kind == PAIR:
        J, r = qm.rows(cams, *prior)
        return J.T @ (np.repeat(w, 6) * r)
    A, r = lp.rows(lms, *prior)
    g = np.zeros(3 * len(lms))
    for p, l in enumerate(prior[0]):
        g[3 * l:3 * l + 3] += w[p] * A[p].T @ r[p]
    return g


def cost_of(kind, state, prior, loss):
    return float(np.sum(weights(kind, state, prior, loss)[1]))


def robust_case(seed=41):
    """tests/pair_prior_model.pair_case (8 cameras, one unobserved; a zero-L pair) with camera priors of
    camera_prior_model.small_prior (camera 3's L zero) and the landmark priors of landmark_prior_model.prior_case (zero-L
    ones among them): (prob, priors) with priors the objective_checks keywords"""
    prob, pairs = qm.pair_case(seed=seed)
    mean, L = pm.small_prior(prob, seed=seed + 2)
    L[3] = 0
    return prob, dict(camera=(mean, L), pairs=pairs, landmarks=lp.prior_case(prob.lms, seed=seed + 3))


def losses_around(kind, state, prior, seed, kinds=(olm.NONE, olm.HUBER, olm.CAUCHY, olm.SOFT_L1, olm.TUKEY)):
    """(kind, scale) per prior, the kinds in turn, each scale |L e| times a log-uniform factor in [0.5, 2] so that each loss
    holds priors on both sides of its scale (1 where L e = 0; NaN for NONE: ignored)"""
    m = len(prior[-1])
    rng = np.random.default_rng(seed)
    r = np.linalg.norm(whitened(kind, state, prior), axis=1)
    k = np.asarray([kinds[(p + seed) % len(kinds)] for p in range(m)], np.uint8)
    a = np.where(r > 0, r, 1.0) * np.exp(rng.uniform(np.log(0.5), np.log(2.0), m))
    return k, np.where(k == olm.NONE, np.nan, a)
