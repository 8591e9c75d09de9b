"""Robust losses per observation (rba_set_observation_loss, DESIGN.md section 21) without a device: the float64 model of
tests/observation_loss_model.py against central differences, its normalisation and continuity, the float32 forms the kernels
evaluate, Huber bit for bit, scipy's losses, the planted faults the GPU tests must be able to see, the Python host's
validation, and the entry point and constants in the header and the library."""
import re

import numpy as np
import pytest

import camera_model as cm
import observation_info_model as om
import observation_loss_model as lm
from conftest import rel_err

A = 1.7
KINDS = [lm.NONE, lm.HUBER, lm.CAUCHY, lm.SOFT_L1, lm.TUKEY]


@pytest.fixture(scope="module")
def case():
    """7 cameras, 90 landmarks, residuals of a few sigma so that every loss is active on part of them, mixed kinds"""
    from rootba_b200.synthetic import synth_bal
    prob = synth_bal(7, 90, 3.6, seed=21)
    kind, scale = lm.mixed(prob.nobs, seed=4)
    return prob, om.random_info(prob.nobs, seed=3), kind, scale


def device_form(kind, a, s, dtype):
    """w and rho / 2 as observation_loss (kernels.cuh) evaluates them, in `dtype`"""
    f = np.dtype(dtype).type
    a, s = f(a), f(s)
    a2 = a * a
    hub, cau, tuk = kind == lm.HUBER, kind == lm.CAUCHY, kind == lm.TUKEY
    t = np.sqrt(s if hub else a2 + s)
    q = (a2 if cau else a2 - s if tuk else a) / (a2 + s if cau else a2 if tuk else t)
    if hub:
        w = f(1) if s < a2 else q
        return f(0.5) * (f(2) - w) * w * s, w
    if cau:
        return f(0.5) * a2 * np.log1p(s / a2), q
    if kind == lm.SOFT_L1:
        return a * s / (t + a), q
    if tuk:
        u, c = s / a2, a2 * f(1.0 / 6.0)
        return (c * (u * (f(3) - f(3) * u + u * u)) if s < a2 else c), (q * q if s < a2 else f(0))
    return f(0.5) * s, f(1)


@pytest.mark.parametrize("kind", KINDS, ids=lm.NAMES)
def test_weight_is_the_derivative_of_rho(kind):
    s = np.array([0.01, 0.3, 0.8, 2.0, 5.0, 40.0]) * A * A
    if kind == lm.TUKEY:
        s = s[s < 0.95 * A * A]
    h = 1e-6 * s
    rho = lambda x: 2 * lm.loss(kind, A, x)[0]
    assert rel_err((rho(s + h) - rho(s - h)) / (2 * h), lm.loss(kind, A, s)[1]) < 1e-7


@pytest.mark.parametrize("kind", KINDS, ids=lm.NAMES)
def test_normalised_at_zero(kind):
    s = np.array([1e-6, 1e-9, 1e-12]) * A * A
    err, w = lm.loss(kind, A, s)
    assert np.all(np.abs(2 * err / s - 1) < 1e-5) and np.all(np.abs(w - 1) < 1e-5)


def test_tukey_is_continuous_at_its_scale():
    a2 = A * A
    lo, hi = lm.loss(lm.TUKEY, A, a2 * (1 - 1e-9)), lm.loss(lm.TUKEY, A, a2 * (1 + 1e-9))
    assert abs(lo[0] - a2 / 6) < 1e-12 and hi[0] == a2 / 6
    assert lo[1] < 1e-15 and hi[1] == 0.0
    # the other kinds are continuous at a^2 too (Huber's kink is in w', not in w)
    for k in (lm.HUBER, lm.CAUCHY, lm.SOFT_L1):
        lo, hi = lm.loss(k, A, a2 * (1 - 1e-9)), lm.loss(k, A, a2 * (1 + 1e-9))
        assert abs(lo[0] - hi[0]) < 1e-8 and abs(lo[1] - hi[1]) < 1e-8


@pytest.mark.parametrize("kind", KINDS, ids=lm.NAMES)
@pytest.mark.parametrize("u", [1e-8, 0.5, 1e4])
def test_float32_forms_of_the_kernels(kind, u):
    """the cancellation-free forms the kernels evaluate hold float32 accuracy at tiny and large s"""
    if kind == lm.TUKEY and u >= 1:
        u = 0.999
    s = u * A * A
    e32, w32 = device_form(kind, A, s, np.float32)
    e64, w64 = lm.loss(kind, A, s)
    assert abs(float(e32) - e64) <= 4e-6 * abs(e64)
    assert abs(float(w32) - w64) <= 4e-6 * abs(w64) + (1e-4 if kind == lm.TUKEY and u == 0.999 else 0)
    e, w = device_form(kind, A, s, np.float64)
    assert abs(e - e64) <= 1e-14 * abs(e64) and abs(w - w64) <= 1e-14 * abs(w64) + (1e-10 if kind == lm.TUKEY else 0)


def test_huber_is_the_handles_huber_bit_for_bit():
    s = np.random.default_rng(0).exponential(4.0, 1000) * A * A
    err, w = lm.loss(lm.HUBER, A, s)
    e0, w0 = cm.huber(s, A)
    assert np.array_equal(err, e0) and np.array_equal(w, w0)
    assert np.array_equal(lm.loss(lm.NONE, np.nan, s)[0], 0.5 * s)


@pytest.mark.parametrize("kind,name", [(lm.HUBER, "huber"), (lm.CAUCHY, "cauchy"), (lm.SOFT_L1, "soft_l1")])
def test_costs_are_scipys(kind, name):
    """scipy's least_squares cost 1/2 sum a^2 rho_scipy(f^2 / a^2) with f_scale = a, on one residual per observation"""
    from scipy.optimize import least_squares
    f = np.random.default_rng(1).normal(0, 3 * A, 50)
    res = least_squares(lambda x: f + 0 * x[0], [0.0], loss=name, f_scale=A, max_nfev=1)
    err, _ = lm.loss(kind, A, f * f)
    assert abs(res.cost - err.sum()) <= 1e-12 * err.sum()


def test_rows_give_the_gradient_of_the_robust_cost(case):
    """the weighted rows sqrt(w) W [Jp | Jl | r]: J^T r is the gradient of sum rho(|W r|^2) / 2 (the first-order part of
    l_diff), by central differences in the landmark coordinates and the camera intrinsics"""
    prob, W, kind, scale = case
    from rootba_b200.synthetic import BalArrays
    Jp, Jl, r = lm.dense_system(prob, kind, scale, W)
    g_l, g_p = Jl.T @ r, Jp.T @ r
    h = 1e-6
    for k in range(3):
        e = np.zeros(3)
        e[k] = h
        c = lambda d: lm.cost(BalArrays(prob.cams, prob.lms + d, prob.lm_off, prob.obs_cam, prob.obs_xy), kind, scale, W)
        fd = np.array([(c(np.where(np.arange(prob.nl)[:, None] == l, e, 0)) - c(np.where(np.arange(prob.nl)[:, None] == l, -e, 0)))
                       / (2 * h) for l in range(0, prob.nl, 11)])
        assert rel_err(fd, g_l.reshape(-1, 3)[::11, k]) < 1e-5
    for col in (7, 8, 9):  # f, k1, k2: increment entries 6..8 add to them
        e = np.zeros(10)
        e[col] = h
        c = lambda d: lm.cost(BalArrays(prob.cams + d, prob.lms, prob.lm_off, prob.obs_cam, prob.obs_xy), kind, scale, W)
        fd = np.array([(c(np.where(np.arange(prob.nc)[:, None] == i, e, 0)) - c(np.where(np.arange(prob.nc)[:, None] == i, -e, 0)))
                       / (2 * h) for i in range(prob.nc)])
        assert rel_err(fd, g_p.reshape(-1, 9)[:, col - 1]) < 1e-5


def test_the_checks_reject_the_planted_faults(case):
    prob, W, kind, scale = case
    kind = kind.copy()
    kind[::5] = lm.TUKEY  # some beyond their scale
    scale = np.where(kind == lm.NONE, np.nan, scale)
    scale[::5] = 0.8
    true_rows = lm.rows(prob, kind, scale, W)
    true_info = lm.residual_info(prob, kind, scale, W)
    assert (true_rows["w"][::5] == 0).any() and (true_rows["w"] < 1).mean() > 0.2
    for fault in lm.FAULTS:
        if fault == "tukey_zero_not_valid":
            got = lm.residual_info(prob, kind, scale, W, fault=fault)
            assert got["valid"]["num_obs"] < true_info["valid"]["num_obs"], fault
            continue
        got = lm.rows(prob, kind, scale, W, fault=fault)
        assert rel_err(np.concatenate([got["Jp"].ravel(), got["r"].ravel()]),
                       np.concatenate([true_rows["Jp"].ravel(), true_rows["r"].ravel()])) > 1e-3, fault


def test_switched_off_stays_off_and_tukey_rejection_is_zero_rows(case):
    prob, W, kind, scale = case
    W = W.copy()
    W[::7] = 0
    w = lm.rows(prob, kind, scale, W)
    assert np.all(w["Jp"][::7] == 0) and np.all(w["r"][::7] == 0) and np.all(w["err"][::7] == 0)
    info = lm.residual_info(prob, np.full(prob.nobs, lm.TUKEY, np.uint8), np.full(prob.nobs, 1e-3), W)
    assert info["valid"]["num_obs"] == int((cm.linearize(*cm.observations(prob))["valid"] & w["on"]).sum())
    assert abs(info["all"]["error"] - w["on"].sum() * 1e-6 / 6) < 1e-18


def test_python_host_validates_and_broadcasts():
    import rootba_b200 as rb
    from rootba_b200.synthetic import synth_bal
    prob = synth_bal(4, 20, 3.0, seed=2)
    bp = rb.BalProblem.from_arrays(prob, np.float32)
    n = bp.num_observations()
    bp.observation_loss = ("cauchy", 2.0)
    k, a = bp.observation_loss
    assert k.dtype == np.uint8 and k.shape == (n,) and np.all(k == rb._lib.LOSS_CAUCHY)
    assert a.dtype == np.float32 and np.all(a == 2.0)
    kinds = np.array(["NONE", "TUKEY"] * (n // 2) + ["HUBER"] * (n % 2))
    bp.observation_loss = (kinds, np.linspace(1, 2, n))
    assert list(bp.observation_loss[0][:2]) == [0, 4]
    bp.observation_loss = (np.full(n, 3), 1.0)
    bp.observation_loss = ("NONE", np.nan)  # NONE ignores its scale
    for bad in [("CAUCHY", 0.0), ("CAUCHY", -1.0), ("TUKEY", np.inf), ("HUBER", np.nan), (5, 1.0), ("WELSCH", 1.0),
                (np.zeros(n + 1, np.uint8), 1.0), ("CAUCHY", np.ones(n - 1)), "CAUCHY", (1.5, 1.0)]:
        with pytest.raises(ValueError):
            bp.observation_loss = bad
    assert bp.observation_loss[0][0] == 0  # the last accepted value stays
    bp.observation_loss = None
    assert bp.observation_loss is None


def test_symbol_and_constants():
    from rootba_b200 import _lib
    assert "rba_set_observation_loss" in _lib.declared_symbols()
    import os
    if os.path.exists(_lib.LIB_PATH):
        assert hasattr(_lib.lib(), "rba_set_observation_loss")
    hdr = open(_lib.HEADER_PATH).read()
    consts = dict((m.group(1), int(m.group(2))) for m in re.finditer(r"#define RBA_LOSS_(\w+)\s+(\d+)", hdr))
    assert consts == _lib.LOSS_KINDS
    for name, v in consts.items():
        assert getattr(_lib, "LOSS_" + name) == v
    assert re.search(r"int32_t rba_set_observation_loss\(rba_handle\* h, const uint8_t\* kind, const void\* scale\);", hdr)
