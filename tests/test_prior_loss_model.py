"""Robust losses on the priors (rba_set_prior_loss, DESIGN.md section 22) without a device: the float64 model of
tests/prior_loss_model.py against central differences, the planted faults the GPU tests must be able to see, the Python
host's validation and clearing, and the entry points and constants in the header and the library."""
import os
import re
import subprocess

import numpy as np
import pytest

import camera_model as cm
import camera_prior_model as pm
import objective_checks as oc
import observation_loss_model as olm
import prior_loss_model as plm
from conftest import rel_err

KINDS = [olm.NONE, olm.HUBER, olm.CAUCHY, olm.SOFT_L1, olm.TUKEY]


@pytest.fixture(scope="module")
def case():
    prob, priors = plm.robust_case()
    state = (np.asarray(prob.cams, np.float64), np.asarray(prob.lms, np.float64))
    return prob, priors, state


def moved(state, kind, prior, k, h):
    """state with increment entry k of the prior kind's parameters moved by h (cameras by k_camera_update's convention)"""
    cams, lms = state[0].copy(), state[1].copy()
    if kind == plm.LANDMARK:
        lms.reshape(-1)[k] += h
    else:
        d = np.zeros(9)
        d[k % 9] = h
        cams[k // 9] = pm.apply_inc(cams[k // 9], d)
    return cams, lms


@pytest.mark.parametrize("loss_kind", KINDS, ids=olm.NAMES)
@pytest.mark.parametrize("kind", [plm.CAMERA, plm.PAIR, plm.LANDMARK], ids=["camera", "pair", "landmark"])
def test_irls_gradient_is_the_gradient_of_the_robust_cost(case, kind, loss_kind):
    """w (L J)^T (L e) summed over the priors of one kind equals the central difference of sum rho(|L e|^2)/2"""
    prob, priors, state = case
    prior = priors[plm.KINDS[kind]]
    k, a = plm.losses_around(kind, state, prior, seed=5, kinds=(loss_kind,))
    s, _, w = plm.weights(kind, state, prior, (k, a))
    if loss_kind == olm.TUKEY:
        assert np.any((w == 0) & (s > 0)) and np.any(w > 0)  # priors on both sides of the scale
    g = plm.irls_gradient(kind, state, prior, (k, a))
    n = len(g)
    cols = np.arange(n) if kind != plm.LANDMARK else np.flatnonzero(np.repeat(np.isin(np.arange(prob.nl), prior[0]), 3))
    h = 1e-6
    c = lambda st: plm.cost_of(kind, st, prior, (k, a))
    fd = np.array([(c(moved(state, kind, prior, j, h)) - c(moved(state, kind, prior, j, -h))) / (2 * h) for j in cols])
    assert np.max(np.abs(g[cols])) > 0
    assert rel_err(fd, g[cols]) < 1e-5  # the bar of test_observation_loss_model


def _system(prob, priors, losses, state, fault=None, at=None):
    wp = plm.weighted_all(state, priors, losses, fault, at)
    Jp, Jl, r = oc.dense_system(prob, **wp)
    return np.hstack([Jp, Jl]), r


def test_the_checks_reject_the_planted_faults(case):
    """each fault moves what the GPU tests compare (the rows, hence b, H and the covariance; or the cost) by more than the
    float64 bars of objective_checks.BARS"""
    prob, priors, state = case
    losses = {kd: plm.losses_around(kd, state, priors[name], seed=kd) for kd, name in enumerate(plm.KINDS)}
    losses[plm.PAIR] = (np.full(len(losses[plm.PAIR][0]), olm.TUKEY, np.uint8), losses[plm.PAIR][1])
    losses[plm.PAIR][1][np.isnan(losses[plm.PAIR][1])] = 0.05
    J, r = _system(prob, priors, losses, state)
    H, b = J.T @ J, J.T @ r
    # the GPU tests bound the error of the total cost (reprojection + priors), so the bar is on that
    reproj = float(cm.compute_error(prob)["all"]["error"])
    c = reproj + plm.prior_cost(state, priors, losses)
    bar = oc.BARS[np.float64]
    for fault in plm.FAULTS:
        Jf, rf = _system(prob, priors, losses, state, fault)
        moved_rows = rel_err(Jf.T @ rf, b) > bar["b"] or rel_err(Jf.T @ Jf, H) > bar["op"]
        moved_cost = abs(reproj + plm.prior_cost(state, priors, losses, fault) - c) > bar["cost"] * c
        assert moved_rows or moved_cost, fault
    # the covariance weights: at the state of the last linearisation, or at the priors' means, instead of the current state
    lin_state = (np.asarray(prob.cams, np.float64).copy(), state[1] + 0.05)
    lin_state[0][:, 4:7] += 0.1
    # (at the means e = 0 and every w = 1: the unweighted priors)
    for Jf in (_system(prob, priors, losses, state, at=lin_state)[0], _system(prob, priors, {}, state)[0]):
        assert rel_err(Jf.T @ Jf, H) > bar["inv"]


def test_tukey_beyond_its_scale_is_zero_rows_and_a2_over_6(case):
    prob, priors, state = case
    prior = priors["pairs"]
    m = len(prior[0])
    a = np.full(m, 1e-3)
    k = np.full(m, olm.TUKEY, np.uint8)
    s, err, w = plm.weights(plm.PAIR, state, prior, (k, a))
    drop = plm.dropped(plm.PAIR, prior)
    assert np.all(w[~drop] == 0) and np.allclose(err[~drop], 1e-6 / 6, rtol=0, atol=1e-18)
    assert np.all(plm.weighted(plm.PAIR, state, prior, (k, a))[-1][~drop] == 0)


def test_python_host_validates_and_clears():
    import rootba_b200 as rb
    prob, priors = plm.robust_case()
    bp = rb.BalProblem.from_arrays(prob, np.float32)
    nc = bp.num_cameras()
    # without a prior of the kind there is nothing to weight, except the cameras (one entry per camera)
    bp.camera_prior_loss = ("cauchy", 2.0)
    assert bp.camera_prior_loss[0].shape == (nc,) and np.all(bp.camera_prior_loss[0] == olm.CAUCHY)
    assert bp.camera_prior_loss[1].dtype == np.float32
    with pytest.raises(ValueError):
        bp.camera_pair_prior_loss = ("CAUCHY", np.ones(3))
    bp.camera_pair_prior = priors["pairs"]
    bp.landmark_prior = priors["landmarks"]
    m, ml = len(priors["pairs"][0]), len(priors["landmarks"][0])
    bp.camera_pair_prior_loss = ("TUKEY", np.linspace(1, 2, m))
    bp.landmark_prior_loss = (np.array(["NONE", "SOFT_L1"] * (ml // 2) + ["HUBER"] * (ml % 2)), 1.5)
    assert list(bp.landmark_prior_loss[0][:2]) == [olm.NONE, olm.SOFT_L1]
    for name, n in (("camera_prior_loss", nc), ("camera_pair_prior_loss", m), ("landmark_prior_loss", ml)):
        before = getattr(bp, name)
        for bad in [("CAUCHY", 0.0), ("TUKEY", np.inf), ("HUBER", np.nan), (5, 1.0), ("WELSCH", 1.0),
                    (np.zeros(n + 1, np.uint8), 1.0), ("CAUCHY", np.ones(n - 1)), "CAUCHY"]:
            with pytest.raises(ValueError, match=name):
                setattr(bp, name, bad)
        assert getattr(bp, name) is before  # the last accepted value stays
    bp.camera_pair_prior_loss = ("NONE", np.nan)  # NONE ignores its scale
    # a setter of the kind clears its losses, and only its own
    bp.camera_pair_prior = priors["pairs"]
    assert bp.camera_pair_prior_loss is None and bp.landmark_prior_loss is not None and bp.camera_prior_loss is not None
    bp.landmark_prior = None
    assert bp.landmark_prior_loss is None
    bp.camera_prior = priors["camera"]
    assert bp.camera_prior_loss is None
    with pytest.raises(ValueError):
        rb.LinearizorQR._prior_kind("rig")
    assert [rb.LinearizorQR._prior_kind(w) for w in ("camera", "PAIR", 2)] == [0, 1, 2]


def test_symbols_constants_and_a_c99_compile_of_the_header(tmp_path):
    from rootba_b200 import _lib
    for sym in ("rba_set_prior_loss", "rba_get_prior_residuals"):
        assert sym in _lib.declared_symbols()
        if os.path.exists(_lib.LIB_PATH):
            assert hasattr(_lib.lib(), sym)
    hdr = open(_lib.HEADER_PATH).read()
    consts = dict((m.group(1).lower(), int(m.group(2))) for m in re.finditer(r"#define RBA_PRIOR_(\w+)\s+(\d+)", hdr))
    assert consts == _lib.PRIOR_KINDS
    assert re.search(r"int32_t rba_set_prior_loss\(rba_handle\* h, int32_t prior_kind, int32_t num, const uint8_t\* kind, "
                     r"const void\* scale\);", hdr)
    assert re.search(r"int32_t rba_get_prior_residuals\(rba_handle\* h, int32_t prior_kind, void\* residual, void\* robust_weight\);", hdr)
    src = tmp_path / "use.c"
    src.write_text('#include "rootba_b200.h"\nint f(rba_handle* h) { const uint8_t k[1] = {RBA_LOSS_CAUCHY}; const float a[1] = {2.8f};\n'
                   '  return rba_set_prior_loss(h, RBA_PRIOR_LANDMARK, 1, k, a) + rba_get_prior_residuals(h, RBA_PRIOR_PAIR, 0, 0); }\n')
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", "-c", "-I", os.path.dirname(_lib.HEADER_PATH), str(src),
                    "-o", str(tmp_path / "use.o")], check=True)
