"""The float64 camera model of tests/camera_model.py against central differences at real lens distortion, and the oracle's
per-observation linearisation and compute_error against the model (CPU only).

Bars:
  central differences  each column j of a Jacobian is compared as the first-order change J[:, j] h_j of a step h_j (1e-6
                       relative to the scale of the parameter): |CD - J| h_j <= 1e-6 max_j |J[:, j] h_j| per residual row.
                       The truncation error of a central difference is O((h / scale)^2) ~ 1e-12, its round-off
                       ~ u |proj| / |J h| ~ 1e-10; a wrong distortion term changes J by O(|k1| r^2) ~ 1.
  oracle f64           |oracle - model| <= 256 u kappa max|row| per row of residual / Jp / Jl and per column of Ji (its
                       columns differ by the factor f), u = 2^-53.  kappa = kappa_pc kappa_rp:  kappa_pc =
                       (|R| |p| + |t|) / |pc| (infinity norms) covers the cancellation in pc = R p + t, kappa_rp =
                       (1 + |k1| r2 + |k2| r2^2) / |rp| the cancellation in rp at real distortion; the remaining steps
                       are a few dozen roundings each (measured: up to ~100 u kappa on Ji, ~70 u kappa elsewhere).
  oracle f32           the same bar with u = 2^-24, the model evaluated on the float32 inputs cast exactly to float64.
  compute_error        counts exact; sums at 1e-12 relative in f64.
"""
import os
import re

import numpy as np
import pytest

import camera_model as cm
from conftest import ROOT


def _random_observations(seed, m=400, zlim=(1e-2, 1e3), tan=1.5, k1=0.5, k2=0.3, flim=(200.0, 5000.0)):
    """cameras with random rotations and real distortion, landmarks with |x/z|, |y/z| <= tan and log-uniform depth"""
    from rootba_b200.synthetic import so3_exp
    rng = np.random.default_rng(seed)
    q = so3_exp(rng.normal(0, 1.5, (m, 3)))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    z = np.exp(rng.uniform(np.log(zlim[0]), np.log(zlim[1]), m))
    pc = np.concatenate([rng.uniform(-tan, tan, (m, 2)) * z[:, None], z[:, None]], axis=1)
    p = rng.normal(0, 50, (m, 3))
    t = pc - np.einsum("mij,mj->mi", cm.rotation(q), p)
    cams = np.concatenate([q, t, rng.uniform(*flim, (m, 1)), rng.uniform(-k1, k1, (m, 1)), rng.uniform(-k2, k2, (m, 1))], axis=1)
    obs = cm.project_pc(pc, cams[:, 7:10]) + rng.normal(0, 2.0, (m, 2))
    return cams, p, obs


def test_thresholds_match_the_sources():
    """the model's validity thresholds are the values kernels.cuh and the oracle state"""
    src = open(os.path.join(ROOT, "rootba_b200", "csrc", "kernels.cuh")).read()
    f = re.search(r"struct ST<float>.*?eps_sqrt\(\) \{ return ([0-9.e+-]+)f; \}.*?eps\(\) \{ return ([0-9.e+-]+)f; \}", src, re.S)
    d = re.search(r"struct ST<double>.*?eps_sqrt\(\) \{ return ([0-9.e+-]+); \}.*?eps\(\) \{ return ([0-9.e+-]+); \}", src, re.S)
    assert np.float32(f.group(1)) == cm.EPS_SQRT[np.dtype(np.float32)] and np.float32(f.group(2)) == cm.EPS[np.dtype(np.float32)]
    assert np.float64(d.group(1)) == cm.EPS_SQRT[np.dtype(np.float64)] and np.float64(d.group(2)) == cm.EPS[np.dtype(np.float64)]
    orc_src = open(os.path.join(ROOT, "oracle", "rootba_oracle.hpp")).read()
    assert re.search(r"sophus_epsilon<double>\(\) \{ return 1e-10; \}", orc_src)
    assert re.search(r"sophus_epsilon<float>\(\) \{ return 1e-5f; \}", orc_src)
    # the oracle takes std::sqrt of epsilon in the scalar type: the same numbers
    assert np.sqrt(np.float32(1e-5)) == cm.EPS_SQRT[np.dtype(np.float32)]
    assert np.sqrt(np.float64(1e-10)) == cm.EPS_SQRT[np.dtype(np.float64)]


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_model_against_central_differences(seed):
    from scipy.spatial.transform import Rotation
    cams, p, obs = _random_observations(seed)
    L = cm.linearize(cams, p, obs)
    pc = L["pc"]
    s = np.linalg.norm(pc, axis=1)
    R = cm.rotation(cams[:, :4])

    def proj(pc_, intr_):
        return cm.project_pc(pc_, intr_)

    def check(J, fwd, steps, what):
        for j, h in enumerate(steps):
            cd = (fwd(j, h) - fwd(j, -h)) / (2 * h[:, None])
            scale = np.max(np.abs(J) * np.stack(steps, axis=1)[:, None, :], axis=2)  # [m, 2]
            err = np.abs(cd - J[:, :, j]) * h[:, None]
            assert np.all(err <= 1e-6 * scale), (what, j, float(np.max(err / scale)))

    intr = cams[:, 7:10]
    one = np.ones(len(s))

    def pose(j, h):
        if j < 3:
            d = np.zeros_like(pc); d[:, j] = h
            return proj(pc + d, intr)
        w = np.zeros_like(pc); w[:, j - 3] = h
        return proj(np.einsum("mij,mj->mi", Rotation.from_rotvec(w).as_matrix(), pc), intr)
    check(L["Jp"], pose, [1e-6 * s] * 3 + [1e-6 * one] * 3, "Jp")

    def intrinsics(j, h):
        d = np.zeros_like(intr); d[:, j] = h
        return proj(pc, intr + d)
    check(L["Ji"], intrinsics, [1e-6 * intr[:, 0], 1e-6 * one, 1e-6 * one], "Ji")

    def landmark(j, h):  # R (p + d) + t = pc + R d, without the cancellation of R p + t when |p| >> |pc|
        d = np.zeros_like(p); d[:, j] = h
        return proj(pc + np.einsum("mij,mj->mi", R, d), intr)
    check(L["Jl"], landmark, [1e-6 * s] * 3, "Jl")
    # the residual itself
    assert np.allclose(L["res"], proj(pc, intr) - obs, rtol=1e-14, atol=0)


def _kappa(cams, p):
    R = cm.rotation(cams[:, :4])
    pc = np.einsum("mij,mj->mi", R, p) + cams[:, 4:7]
    mag = np.einsum("mij,mj->mi", np.abs(R), np.abs(p)).max(1) + np.abs(cams[:, 4:7]).max(1)
    return mag / np.abs(pc).max(1)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("seed", [4, 5])
def test_oracle_linearize_point_against_the_model(dtype, seed):
    from oracle import oracle_py as orc
    cams, p, obs = _random_observations(seed, m=300)
    cams, p, obs = (a.astype(dtype) for a in (cams, p, obs))
    L = cm.linearize(cams, p, obs, dtype=dtype)
    u = float(np.finfo(dtype).eps) / 2
    c64 = cams.astype(np.float64)
    kappa = _kappa(c64, p.astype(np.float64))
    m = L["pc"][:, :2] / L["pc"][:, 2:3]
    r2 = (m * m).sum(1)
    kappa *= (1 + np.abs(c64[:, 8]) * r2 + np.abs(c64[:, 9]) * r2 * r2) / np.abs(1 + c64[:, 8] * r2 + c64[:, 9] * r2 * r2)
    for k in range(len(obs)):
        res, Jp, Ji, Jl, valid = orc.linearize_point(obs[k], p[k], cams[k], dtype=dtype)
        assert valid == bool(L["valid"][k])
        # the residual's scale is the projection, not the (small) residual
        err = np.abs(res.astype(np.float64) - L["res"][k])
        assert np.all(err <= 256 * u * kappa[k] * np.abs(L["res"][k] + obs[k]).max()), ("res", k, err)
        for got, want, axis, what in ((Jp, L["Jp"][k], 1, "Jp"), (Ji, L["Ji"][k], 0, "Ji"), (Jl, L["Jl"][k], 1, "Jl")):
            bar = 256 * u * kappa[k] * np.abs(want).max(axis=axis, keepdims=True)
            err = np.abs(got.astype(np.float64) - want)
            assert np.all(err <= bar), (what, k, err.max(), np.max(bar))


@pytest.mark.parametrize("robust", [None, "median"])
@pytest.mark.parametrize("optimized_cost", [0, 1])
def test_oracle_compute_error_against_the_model(robust, optimized_cost):
    """counts exact and sums at 1e-12 on a problem with real distortion, turned-around cameras (invalid projections) and,
    optionally, the Huber threshold at the median residual"""
    from oracle import oracle_py as orc
    from rootba_b200.synthetic import synth_bal, turn_cameras_around
    a = turn_cameras_around(synth_bal(16, 300, 4.0, seed=9, k1_sigma=0.1, k2_sigma=0.02, max_tan=1.3), [2, 11])
    L = cm.linearize(*cm.observations(a))
    rsq = (L["res"] ** 2).sum(1)
    th = None if robust is None else float(np.sqrt(np.median(rsq)))
    want = cm.compute_error(a, threshold=th)
    assert 0 < want["valid"]["num_obs"] < want["all"]["num_obs"]
    kw = {} if th is None else {"robust_norm": 1, "huber_parameter": th}
    got = orc.Oracle(a, np.float64, orc.default_options(num_threads=1, use_valid_projections_only=optimized_cost, **kw)).compute_error()
    for key in ("all", "valid"):
        assert got[key]["num_obs"] == want[key]["num_obs"]
        for q in ("error", "residual_sum"):
            assert abs(got[key][q] - want[key][q]) <= 1e-12 * want[key][q], (key, q)
    assert got["is_numerically_valid"]
