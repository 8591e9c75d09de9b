"""Per-observation square-root information (rba_set_observation_info, DESIGN.md section 19) without a device: the float64
model of tests/observation_info_model.py against central differences and against its own invariants (scalar weight =
scaled rows, W and Q W agree, W = 0 = the observation removed), the planted faults the GPU tests must be able to see, the
Python host's validation and the two entry points in the header and the library."""
import numpy as np
import pytest

import camera_model as cm
import observation_info_model as om
from conftest import rel_err
from objective_checks import reduced

LAM = 1e-3


@pytest.fixture(scope="module")
def case():
    """7 cameras, 90 landmarks, residuals of a few sigma so that Huber at 1 is active on part of them"""
    from rootba_b200.synthetic import synth_bal
    prob = synth_bal(7, 90, 3.6, seed=21)
    return prob, om.random_info(prob.nobs, seed=3)


def _step(prob, W, lam=LAM, **kw):
    """the dense LM step of the whitened system: (D, H, b, inc, landmark update, l_diff)"""
    Jp, Jl, r = om.dense_system(prob, W, **kw)
    D, sl, Jps, Jls, Minv, H, b = reduced(Jp, Jl, r, lam, prob.nl)
    inc = -np.linalg.solve(H, b)
    dl = -Minv @ (Jls.T @ r + Jls.T @ (Jps @ inc))
    l_diff = 0.5 * r @ r - 0.5 * np.sum((r + Jps @ inc + Jls @ dl) ** 2)
    return D, H, b, inc, (sl * dl).reshape(-1, 3), float(l_diff)


def _moved(prob, inc_scaled, D, dlm):
    """the state after the increment: cameras by the left-multiplied pose increment (translation first), landmarks by dlm"""
    from rootba_b200.synthetic import BalArrays
    from scipy.spatial.transform import Rotation
    d = (inc_scaled * D).reshape(-1, 9)
    cams = np.asarray(prob.cams, np.float64).copy()
    R = Rotation.from_rotvec(d[:, 3:6])
    cams[:, :4] = (R * Rotation.from_quat(cams[:, :4])).as_quat()
    cams[:, 4:7] = R.apply(cams[:, 4:7]) + d[:, 0:3]
    cams[:, 7:10] += d[:, 6:9]
    return BalArrays(cams, np.asarray(prob.lms, np.float64) + dlm, prob.lm_off, prob.obs_cam, prob.obs_xy)


def test_whitened_jacobian_against_central_differences(case):
    prob, W = case
    w = om.whitened(prob, W)
    cams, p, obs = (np.asarray(a, np.float64) for a in cm.observations(prob))
    f = lambda c, x: np.einsum("oij,oj->oi", W, cm.linearize(c, x, obs)["res"])
    h = 1e-6
    for k in range(3):  # landmark columns
        e = np.zeros(3)
        e[k] = h
        assert rel_err((f(cams, p + e) - f(cams, p - e)) / (2 * h), w["Jl"][:, :, k]) < 1e-7
    for k in range(3):  # translation and intrinsics columns
        e = np.zeros(10)
        e[4 + k] = h
        assert rel_err((f(cams + e, p) - f(cams - e, p)) / (2 * h), w["Jp"][:, :, k]) < 1e-7
        e = np.zeros(10)
        hk = h * (1000.0 if k == 0 else 1e-3)
        e[7 + k] = hk
        assert rel_err((f(cams + e, p) - f(cams - e, p)) / (2 * hk), w["Jp"][:, :, 6 + k]) < 1e-6
    # rotation columns through the finite step of _moved
    for k in range(3):
        d = np.zeros((prob.nc, 9))
        d[:, 3 + k] = h
        plus, minus = _moved(prob, d.ravel(), 1.0, 0.0), _moved(prob, -d.ravel(), 1.0, 0.0)
        fd = (f(plus.cams[prob.obs_cam], p) - f(minus.cams[prob.obs_cam], p)) / (2 * h)
        assert rel_err(fd, w["Jp"][:, :, 3 + k]) < 1e-7


@pytest.mark.parametrize("threshold", [None, 1.0])
def test_l_diff_predicts_the_change_of_the_whitened_cost(case, threshold):
    """a small step (large lambda): the model cost change of the dense LM step equals the true change of the whitened cost to
    second order"""
    prob, W = case
    lam = 1e3
    D, H, b, inc, dlm, l_diff = _step(prob, W, lam=lam, threshold=threshold)
    c0 = om.cost(prob, W, threshold)
    c1 = om.cost(_moved(prob, inc, D, dlm), W, threshold)
    assert l_diff > 0 and abs((c0 - c1) - l_diff) < 2e-2 * l_diff
    if threshold is not None:
        assert 0 < (om.whitened(prob, W, threshold=threshold)["hw"] < 1).mean() < 1


def test_scalar_weight_scales_the_rows(case):
    prob, _ = case
    w = np.random.default_rng(1).uniform(0.2, 4.0, prob.nobs)
    a, one = om.whitened(prob, np.sqrt(w)), om.whitened(prob, np.ones(prob.nobs))
    for k in ("Jp", "Jl"):
        assert np.allclose(a[k], np.sqrt(w)[:, None, None] * one[k], rtol=1e-14, atol=0)
    assert np.allclose(a["r"], np.sqrt(w)[:, None] * one["r"], rtol=1e-14, atol=0)
    assert np.isclose(om.cost(prob, np.sqrt(w)), 0.5 * np.sum(w * (one["wr"] ** 2).sum(1)), rtol=1e-13)


@pytest.mark.parametrize("threshold", [None, 1.0])
def test_any_square_root_gives_the_same_objective(case, threshold):
    """W and Q W (Q orthogonal 2x2 per observation): the same cost, H and b"""
    prob, W = case
    a = np.random.default_rng(2).uniform(0, 2 * np.pi, prob.nobs)
    Q = np.stack([np.stack([np.cos(a), np.sin(a)], -1), np.stack([np.sin(a), -np.cos(a)], -1)], -2)  # reflections
    s1, s2 = _step(prob, W, threshold=threshold), _step(prob, Q @ W, threshold=threshold)
    assert np.isclose(om.cost(prob, W, threshold), om.cost(prob, Q @ W, threshold), rtol=1e-13)
    assert rel_err(s1[1], s2[1]) < 1e-12 and rel_err(s1[2], s2[2]) < 1e-12


@pytest.mark.parametrize("threshold", [None, 1.0])
def test_switched_off_equals_removed(case, threshold):
    prob, W = case
    off = np.random.default_rng(4).random(prob.nobs) < 0.15
    off[prob.lm_off[3]:prob.lm_off[4]] = True           # a landmark with no observation left
    off[prob.lm_off[5] + 1:prob.lm_off[6]] = True       # and one with a single observation left
    W0 = W.copy()
    W0[off] = 0.0
    sub, kept = om.without(prob, off)
    full, ref = _step(prob, W0, threshold=threshold), _step(sub, W[kept], threshold=threshold)
    for a, b in zip(full[:5], ref[:5]):
        assert rel_err(a, b) < 1e-12
    assert abs(full[5] - ref[5]) <= 1e-12 * abs(ref[5])
    assert np.isclose(om.cost(prob, W0, threshold), om.cost(sub, W[kept], threshold), rtol=1e-12, atol=0)
    ri, rr = om.residual_info(prob, W0, threshold=threshold), om.residual_info(sub, W[kept], threshold=threshold)
    assert ri["all"]["num_obs"] == prob.nobs and ri["valid"]["num_obs"] == rr["valid"]["num_obs"] == int((~off).sum())
    assert np.isclose(ri["valid"]["error"], rr["valid"]["error"], rtol=1e-12)


@pytest.mark.parametrize("fault", ["r_only", "transposed", "huber_unwhitened"])
def test_planted_faults_in_the_rows_are_rejected(case, fault):
    """each fault moves b (and H) of the Huber problem by far more than any bar of the GPU tests (1e-3 in float32)"""
    prob, W = case
    good, bad = _step(prob, W, threshold=1.0), _step(prob, W, threshold=1.0, fault=fault)
    assert rel_err(good[2], bad[2]) > 1e-2
    assert rel_err(good[3], bad[3]) > 1e-2


def test_scaling_from_unwhitened_columns_is_rejected(case):
    prob, W = case
    D = _step(prob, W)[0]
    D_raw = _step(prob, np.ones(prob.nobs))[0]
    assert rel_err(D, D_raw) > 1e-2


def test_switched_off_observation_counted_as_valid_is_rejected(case):
    prob, W = case
    W0 = W.copy()
    W0[::7] = 0.0
    good, bad = om.residual_info(prob, W0), om.residual_info(prob, W0, fault="off_counted_valid")
    assert bad["valid"]["num_obs"] - good["valid"]["num_obs"] == len(W0[::7])
    avg = lambda ri: ri["valid"]["error"] / ri["valid"]["num_obs"]
    assert abs(avg(good) - avg(bad)) > 1e-2 * avg(good)  # ERROR_VALID_AVG would be diluted


# ---- the Python host ----------------------------------------------------------------------------------------------------
def test_python_validation_without_a_device(case):
    import rootba_b200 as rb
    prob, W = case
    bp = rb.BalProblem.from_arrays(prob, np.float32)
    assert bp.observation_sqrt_info is None
    bp.observation_sqrt_info = np.full(prob.nobs, 0.5)
    assert bp.observation_sqrt_info.shape == (prob.nobs, 2, 2) and bp.observation_sqrt_info.dtype == np.float32
    assert np.array_equal(bp.observation_sqrt_info[3], 0.5 * np.eye(2, dtype=np.float32))
    bp.observation_sqrt_info = W
    assert np.array_equal(bp.observation_sqrt_info, W.astype(np.float32)) and bp.observation_sqrt_info.flags.c_contiguous
    bad = W.copy()
    bad[5, 1, 0] = np.nan
    for wrong in (W[:-1], np.ones(prob.nobs + 1), W.reshape(-1, 4), bad, np.full(prob.nobs, np.inf)):
        with pytest.raises(ValueError):
            bp.observation_sqrt_info = wrong
    assert np.array_equal(bp.observation_sqrt_info, W.astype(np.float32))  # a rejected value keeps the previous one
    bp.observation_sqrt_info = None
    assert bp.observation_sqrt_info is None


def test_entry_points_are_declared_and_exported():
    from rootba_b200 import _lib
    names = _lib.declared_symbols()
    L = _lib.lib()
    for s in ("rba_set_observation_info", "rba_get_observation_residuals"):
        assert s in names and hasattr(L, s)
