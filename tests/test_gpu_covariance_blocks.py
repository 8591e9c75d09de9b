"""Covariance blocks of chosen pairs (rba_compute_covariance_blocks, DESIGN.md section 20) on the GPU: every kind against the
full float64 inverse of the dense total system in every solver configuration and both precisions (bit-identical within one),
the bit identities with rba_compute_covariance, every feature against its float64 model (covariance_blocks_model), every tile
pair of the inverse, the benchmark size, the halving identity, many requests, errors and the absence of side effects.

Bars are c kappa u as in test_gpu_covariance.py: against the dense inverse 8 N kappa u relative to the largest entry of each
kind, against the model componentwise (covariance_blocks_model.check: 8 (N kappa + n_l kappa_l) u of the entrywise bound)."""
import ctypes as C

import numpy as np
import pytest

import camera_model as cm
import covariance_blocks_model as cbm
import covariance_model as cvm
import pair_prior_model as qm
from objective_checks import CONFIGS, MASK, dense_system, fixed_entries
from rootba_b200._lib import RBA_NUMERICAL_FAILURE
from test_gpu_covariance import _case, _dense, _handle

pytestmark = pytest.mark.gpu

U = 2.0 ** -53


def _requests(prob, seed, m=60):
    """m random requests of each kind on the problem, the first two of the pair kinds marginals"""
    req = cbm.random_requests(np.random.default_rng(seed), len(prob.cams), len(prob.lm_off) - 1, m)
    req["cameras"][:2] = [[0, 0], [1, 1]]
    req["landmarks"][:2] = [[0, 0], [1, 1]]
    return req


def _model_check(got, prob, dtype, req, what="", **kw):
    """the handle's blocks against covariance_model.reference's Sigma, K, W through the four formulas"""
    ref = cvm.reference(prob, dtype, **kw)
    ref["cams"] = np.asarray(cvm.as_stored(prob, dtype)[0].cams, np.float64)
    cbm.check(got, cbm.blocks(ref, **req), ref, req, what=what)
    return ref


def _dense_check(got, F, kappa, N, nc, cams, req, c=8):
    want = cbm.dense_blocks(F, nc, cams, **req)
    for key in want:
        scale = np.abs(want[key]).max()
        err = np.abs(got[key] - want[key]).max()
        assert err <= c * N * kappa * U * scale, (key, err / scale, c * N * kappa * U)


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("size", [(7, 90, 21), (120, 500, 5)], ids=["nc7", "nc120"])
def test_every_kind_against_the_dense_inverse(size, dtype):
    prob, absp = _case(*size)
    nc = size[0]
    req = _requests(prob, size[2])
    first = None
    for cfg in CONFIGS:
        lin = _handle(prob, dtype, cfg, absp=absp)
        got = lin.covariance_blocks(**req, marginals=True)
        lin.close()
        if first is None:
            first = got
        else:
            for key in got:
                assert np.array_equal(got[key], first[key]), (cfg, key)
    sprob, sabsp, _ = cvm.as_stored(prob, dtype, absp)
    Jp, Jl = _dense(sprob, sabsp, dtype=dtype)
    F, kappa, N = cbm.full_covariance(Jp, Jl)
    _dense_check(first, F, kappa, N, nc, np.asarray(sprob.cams, np.float64), req)


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
def test_bit_identities_with_the_marginals(dtype):
    prob, absp = _case(49, 1800, 38401)
    lin = _handle(prob, dtype, absp=absp)
    cam, lm = lin.covariance()
    nc, nl = lin.nc, lin.nl
    rng = np.random.default_rng(1)
    a, b = rng.integers(0, nc, 300), rng.integers(0, nc, 300)
    l = rng.integers(0, nl, 300)
    got = lin.covariance_blocks(cameras=np.r_[np.c_[np.arange(nc), np.arange(nc)], np.c_[a, b], np.c_[b, a]],
                                landmarks=np.c_[l, l], marginals=True)
    lin.close()
    assert np.array_equal(got["cam"], cam) and np.array_equal(got["lm"], lm)
    assert np.array_equal(got["cameras"][:nc], cam)
    assert np.array_equal(got["landmarks"], lm[l])
    ab, ba = got["cameras"][nc:nc + 300], got["cameras"][nc + 300:].transpose(0, 2, 1)
    assert (np.abs(ab - ba) <= 4 * U * np.abs(ab)).all()


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
def test_absolute_and_pair_priors(dtype):
    prob, pair = qm.pair_case(7, 90)
    import camera_prior_model as pm
    absp = cvm.centre_priors(prob, 9)
    absp[1][-1] = pm.sqrt_info_kind("dense", np.random.default_rng(9))
    lin = _handle(prob, dtype, absp=absp, pair=pair)
    req = _requests(prob, 3)
    got = lin.covariance_blocks(**req)
    lin.close()
    _model_check(got, prob, dtype, req, "priors", absp=absp, pair=pair)


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
def test_held_parameters(dtype):
    prob, absp = _case(7, 90, 21)
    lin = _handle(prob, dtype, absp=absp, mask=MASK)
    req = _requests(prob, 4)
    req["relative"][:2] = [[0, 3], [3, 0]]  # cameras 0 (pose held) and 3 (all held)
    got = lin.covariance_blocks(**req)
    lin.close()
    _model_check(got, prob, dtype, req, "held", absp=absp, mask=MASK)
    assert (got["relative"][:2] == 0).all()
    fixed = fixed_entries(MASK).reshape(7, 9)
    for k, (a, b) in enumerate(req["cameras"]):
        assert (got["cameras"][k][fixed[a], :] == 0).all() and (got["cameras"][k][:, fixed[b]] == 0).all()
    for k, (c, _) in enumerate(req["camera_landmark"]):
        assert (got["camera_landmark"][k][fixed[c], :] == 0).all()


def test_landmark_priors():
    import landmark_prior_model as lp
    import rootba_b200 as rb
    from rootba_b200.synthetic import synth_bal
    prob = synth_bal(7, 90, 3.6, seed=21)
    prior = lp.prior_case(prob.lms, every=3, seed=6, kinds=("dense",), scale=5.0)
    bp = rb.BalProblem.from_arrays(prob, np.float64)
    bp.landmark_prior = prior
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions())
    req = _requests(prob, 5)
    got = lin.covariance_blocks(**req)
    lin.close()
    Jp, Jl, _ = dense_system(prob, landmarks=prior)
    F, kappa, N = cbm.full_covariance(Jp, Jl)
    _dense_check(got, F, kappa, N, 7, np.asarray(prob.cams, np.float64), req)


def test_intrinsics_groups():
    """the reference is the full P Sigma_u P^T of the tied system (shared_intrinsics_model.tied_covariance's definition)"""
    import rootba_b200 as rb
    import shared_intrinsics_model as sim
    from rootba_b200.synthetic import BalArrays
    prob, absp = _case(7, 90, 21)
    group = np.array([0, 0, 1, -1, 1, 0, 2], np.int32)
    lead = sim.leads(group)
    cams = np.array(prob.cams, np.float64)  # the members start at their lead's intrinsics, as the handle ties them
    cams[lead >= 0, 7:] = cams[lead[lead >= 0], 7:]
    prob = BalArrays(cams, prob.lms, prob.lm_off, prob.obs_cam, prob.obs_xy)
    bp = rb.BalProblem.from_arrays(prob, np.float64)
    bp.camera_prior = absp
    bp.intrinsics_group = group
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions())
    req = _requests(prob, 6)
    req["cameras"][2:4] = [[0, 1], [2, 4]]
    got = lin.covariance_blocks(**req, marginals=True)
    lin.close()
    Jp, Jl, _ = dense_system(prob, camera=absp)
    F, kappa, N = cbm.full_covariance(Jp, Jl, lead=lead)
    _dense_check(got, F, kappa, N, 7, np.asarray(prob.cams, np.float64), req)
    want_cam, _ = sim.tied_covariance(Jp, Jl, lead)
    assert np.abs(np.stack([F[9 * c:9 * c + 9, 9 * c:9 * c + 9] for c in range(7)]) - want_cam).max() <= 1e-9 * np.abs(want_cam).max()
    for k in (2, 3):  # two members share the group's intrinsics covariance
        assert np.array_equal(got["cameras"][k][6:, 6:], got["cam"][req["cameras"][k][0]][6:, 6:])


def test_observation_info_with_switched_off_observations():
    import observation_info_model as om
    import rootba_b200 as rb
    prob, absp = _case(7, 90, 21)
    W = om.random_info(len(prob.obs_cam), 3)
    long_tracks = np.repeat(np.diff(prob.lm_off) >= 4, np.diff(prob.lm_off))
    W[np.flatnonzero(long_tracks)[::7]] = 0.0
    bp = rb.BalProblem.from_arrays(prob, np.float64)
    bp.camera_prior = absp
    bp.observation_sqrt_info = W
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions())
    req = _requests(prob, 7)
    got = lin.covariance_blocks(**req)
    lin.close()
    Jp, Jl, _ = om.dense_system(prob, W)
    Jc, _ = _dense(prob, absp)
    Jp = np.vstack([Jp, Jc[len(Jc) - 9 * 7:]])
    Jl = np.vstack([Jl, np.zeros((9 * 7, Jl.shape[1]))])
    F, kappa, N = cbm.full_covariance(Jp, Jl)
    _dense_check(got, F, kappa, N, 7, np.asarray(prob.cams, np.float64), req)


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
def test_huber_with_active_weights(dtype):
    from rootba_b200.linearizor import ResidualOptions
    prob, absp = _case(7, 90, 21)
    L = cm.linearize(*cm.observations(prob))
    th = float(np.median(np.sqrt((L["res"] ** 2).sum(1))))
    lin = _handle(prob, dtype, absp=absp, residual=ResidualOptions("HUBER", th))
    req = _requests(prob, 8)
    got = lin.covariance_blocks(**req)
    lin.close()
    _model_check(got, prob, dtype, req, "huber", absp=absp, threshold=th)


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
def test_rank2_landmark_is_nan_and_the_rest_match(dtype):
    from test_gpu_covariance import _turned
    import camera_prior_model as pm
    prob = _turned()
    absp = cvm.centre_priors(prob, 4)
    absp[1][0] = pm.sqrt_info_kind("dense", np.random.default_rng(1))
    nc, nl = len(prob.cams), len(prob.lm_off) - 1
    req = _requests(prob, 9)
    req["camera_landmark"][:2] = [[3, 0], [5, 0]]
    req["landmarks"][2:4] = [[0, 7], [7, 0]]
    lin = _handle(prob, dtype, absp=absp, optimized_cost="ERROR_VALID")
    got = lin.covariance_blocks(**req)
    lin.close()
    assert np.isnan(got["camera_landmark"][:2]).all() and np.isnan(got["landmarks"][2:4]).all()
    ref = _model_check(got, prob, dtype, req, "rank2", absp=absp, valid_only=True)
    assert ref["rank"][0] == 2 and (ref["rank"][1:] == 3).all()


@pytest.mark.parametrize("nc", [64, 71, 128])
def test_every_tile_pair(nc):
    prob, absp = cvm.tile_case(nc, seed=nc)
    nl = len(prob.lm_off) - 1
    T = cvm.TILE
    # one camera in every tile, and every camera whose rows straddle a tile boundary: all pairs of them
    pick = sorted(set(cvm.straddling_cameras(nc)) | {(T * t + 8) // 9 for t in range(-(-9 * nc // T)) if (T * t + 8) // 9 < nc})
    pa, pb = np.meshgrid(pick, pick, indexing="ij")
    cams = np.c_[pa.ravel(), pb.ravel()]
    tiles = {(max(9 * a // T, 9 * b // T), min(9 * a // T, 9 * b // T)) for a, b in cams} | \
            {(max((9 * a + 8) // T, (9 * b + 8) // T), min((9 * a + 8) // T, (9 * b + 8) // T)) for a, b in cams}
    assert tiles >= cvm.all_tile_pairs(nc)
    req = _requests(prob, nc, m=400)
    req["cameras"] = cams
    req["relative"] = cams[cams[:, 0] != cams[:, 1]]
    req["camera_landmark"] = np.c_[np.repeat(pick, 4)[:len(pick) * 4], np.random.default_rng(0).integers(0, nl, len(pick) * 4)]
    lin = _handle(prob, np.float64, absp=absp)
    got = lin.covariance_blocks(**req)
    lin.close()
    _model_check(got, prob, np.float64, req, f"tiles nc {nc}", absp=absp)


def test_benchmark_size():
    """the Ladybug-1723 stand-in in float32 with centre priors: 10^4 random requests of each kind, componentwise"""
    import rootba_b200 as rb
    from rootba_b200.synthetic import synth_config
    arrays = synth_config("ladybug-1723", seed=38401)
    absp = cvm.centre_priors(arrays, 5)
    bp = rb.BalProblem.from_arrays(arrays, np.float32)
    bp.camera_prior = absp
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(use_double=False))
    req = _requests(arrays, 10, m=10 ** 4)
    got = lin.covariance_blocks(**req)
    lin.close()
    _model_check(got, arrays, np.float32, req, "benchmark size", absp=absp)


def test_halving_identity_on_the_device():
    prob, absp = _case(7, 90, 21)
    lin = _handle(prob, np.float64, absp=absp)
    pairs = np.array([[1, 4]])
    before = lin.covariance_blocks(relative=pairs)["relative"][0]
    assert np.array_equal(before, before.T)
    L = np.linalg.cholesky(np.linalg.inv(before)).T
    cams = np.asarray(prob.cams, np.float64)
    lin.set_camera_pair_prior((pairs.astype(np.int32), qm.mean_at(cams, pairs), L[None]))
    after = lin.covariance_blocks(relative=pairs)["relative"][0]
    lin.close()
    Jp, Jl = _dense(prob, absp)
    _, kappa, N = cbm.full_covariance(Jp, Jl)
    assert np.abs(after - before / 2).max() <= 8 * N * kappa * U * np.abs(before).max()


def test_many_requests():
    """2 10^5 requests of each kind (several sweeps of every grid-stride loop), the first 1000 repeated at the end: the
    repeats equal the first bit for bit, a call with a part of the requests gives that part bit for bit, and a sample matches
    the model"""
    prob, absp = _case(120, 500, 5)
    m = 2 * 10 ** 5
    req = _requests(prob, 11, m=m - 1000)
    req = {k: np.r_[v, v[:1000]] for k, v in req.items()}
    lin = _handle(prob, np.float64, absp=absp)
    got = lin.covariance_blocks(**req)
    part = lin.covariance_blocks(**{k: v[5000:5100] for k, v in req.items()})
    lin.close()
    for key in got:
        assert got[key].shape[0] == m
        assert np.array_equal(got[key][-1000:], got[key][:1000]), key
        assert np.array_equal(part[key], got[key][5000:5100]), key
    sample = {k: v[::97] for k, v in req.items()}
    _model_check({k: v[::97] for k, v in got.items()}, prob, np.float64, sample, "many", absp=absp)


def _raw_query(lin, req, marginals=False, sentinel=-7.25):
    """a CovarianceQuery of the requests with outputs pre-filled with `sentinel`: (query, outputs, request arrays)"""
    from rootba_b200 import _lib
    q = _lib.CovarianceQuery()
    outs, keep = [], []
    names = [("cameras", "num_camera_pairs", "camera_pairs", "camera_cross", 81),
             ("camera_landmark", "num_camera_landmark", "camera_landmark", "camera_landmark_cross", 27),
             ("landmarks", "num_landmark_pairs", "landmark_pairs", "landmark_cross", 9),
             ("relative", "num_relative_poses", "relative_pairs", "relative_cov", 36)]
    for key, count, src, dst, w in names:
        r = np.ascontiguousarray(req[key], np.int32)
        o = np.full(len(r) * w + 1, sentinel)
        keep.append(r)
        outs.append(o)
        setattr(q, count, len(r))
        setattr(q, src, r.ctypes.data)
        setattr(q, dst, o.ctypes.data)
    if marginals:
        for name, size in (("cam_cov", 81 * lin.nc), ("lm_cov", 9 * lin.nl)):
            o = np.full(size, sentinel)
            outs.append(o)
            setattr(q, name, o.ctypes.data)
    return q, outs, keep


def test_errors_leave_the_outputs_untouched():
    import rootba_b200 as rb
    from rootba_b200 import _lib
    from rootba_b200.synthetic import synth_bal
    lib = _lib.lib()
    prob, absp = _case(7, 90, 21)
    lin = _handle(prob, np.float64, absp=absp)
    good = _requests(prob, 12, m=5)
    assert lib.rba_compute_covariance_blocks(lin.h, None) == -1

    def bad(mutate, marginals=True):
        req = {k: v.copy() for k, v in good.items()}
        q, outs, keep = _raw_query(lin, req, marginals)
        mutate(q, req, keep)
        rc = lib.rba_compute_covariance_blocks(lin.h, C.byref(q))
        assert all((o == -7.25).all() for o in outs)
        return rc

    def setf(name, v):
        return lambda q, req, keep: setattr(q, name, v)

    def index(k, i, v):
        return lambda q, req, keep: keep[k].__setitem__((0, i), v)

    cases = [setf("num_camera_pairs", -1), setf("num_relative_poses", -3), setf("camera_pairs", None),
             setf("landmark_cross", None), index(0, 0, 7), index(0, 1, -1), index(1, 0, 7), index(1, 1, prob.nl),
             index(2, 0, prob.nl), index(2, 1, -2), index(3, 0, 7)]
    for mutate in cases:
        assert bad(mutate) == -1
    assert bad(lambda q, req, keep: keep[3].__setitem__((0, 1), keep[3][0, 0])) == -1  # i == j

    def nothing(q, req, keep):
        for name in ("num_camera_pairs", "num_camera_landmark", "num_landmark_pairs", "num_relative_poses"):
            setattr(q, name, 0)
    assert bad(nothing, marginals=False) == -1
    lin.close()
    # a singular gauge
    free = _handle(synth_bal(7, 90, 3.6, seed=21), np.float64)
    q, outs, keep = _raw_query(free, good, True)
    assert lib.rba_compute_covariance_blocks(free.h, C.byref(q)) == RBA_NUMERICAL_FAILURE
    assert all((o == -7.25).all() for o in outs)
    assert "rba_compute_covariance_blocks" in lib.rba_last_error().decode()
    with pytest.raises(rb.RbaError) as e:
        free.covariance_blocks(**good)
    assert e.value.code == RBA_NUMERICAL_FAILURE
    free.close()
    # a sharded handle
    sh = _handle(prob, np.float64, absp=absp, nranks=2, rank=0)
    q, outs, keep = _raw_query(sh, good, True)
    assert lib.rba_compute_covariance_blocks(sh.h, C.byref(q)) == -4
    assert all((o == -7.25).all() for o in outs) and "nranks" in lib.rba_last_error().decode()
    sh.close()


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
def test_no_side_effects(dtype):
    prob, absp = _case(49, 1800, 38401)
    req = _requests(prob, 13)
    a = _handle(prob, dtype, absp=absp)
    b = _handle(prob, dtype, absp=absp)
    g1 = a.covariance_blocks(**req)
    g2 = a.covariance_blocks(**req)
    for key in g1:
        assert np.array_equal(g1[key], g2[key])
    ia, _, _ = a.lm_run(2)
    a.covariance_blocks(**req, marginals=True)
    ja, _, _ = a.lm_run(2)
    ib, _, _ = b.lm_run(2)
    jb, _, _ = b.lm_run(2)
    strip = lambda its: [{k: v for k, v in it.items() if k != "device_seconds"} for it in its]
    assert strip(ia + ja) == strip(ib + jb)
    for lin in (a, b):
        lin.linearize()
        lin.solve(1e-3, to_host=False)
    a.covariance_blocks(**req)
    la, lb = a.apply(None), b.apply(None)
    assert la == lb
    for lin in (a, b):
        lin.download_state()
    assert np.array_equal(a.bal_problem.cams, b.bal_problem.cams) and np.array_equal(a.bal_problem.lms, b.bal_problem.lms)
    assert a.timings()["kernel_launches"] == b.timings()["kernel_launches"]
    a.close()
    b.close()


def test_example_writes_relative_covariances(tmp_path):
    import os
    import subprocess
    import sys
    from conftest import ROOT
    from rootba_b200.synthetic import synth_bal, write_bal
    prob = synth_bal(7, 90, 3.6, seed=21)
    path = tmp_path / "problem.txt"
    write_bal(prob, str(path))
    pairs = np.array([[2, 3], [4, 2], [6, 5]], np.int64)
    np.save(tmp_path / "pairs.npy", pairs)
    cmd = [sys.executable, os.path.join(ROOT, "examples", "solve_bal.py"), str(path), "--max-num-iterations", "3",
           "--log-path", str(tmp_path / "log.json"), "--fix-cameras", "0,1", "--relative-covariance", str(tmp_path / "pairs.npy")]
    r = subprocess.run(cmd + ["--covariance", str(tmp_path / "cov.npz")], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    with np.load(tmp_path / "cov.npz") as f:
        assert f["cam"].shape == (7, 9, 9) and f["lm"].shape == (len(prob.lm_off) - 1, 3, 3)
        assert f["relative"].shape == (3, 6, 6) and np.array_equal(f["relative_pairs"], pairs)
        rel = f["relative"]
        assert np.isfinite(rel).all() and np.array_equal(rel, rel.transpose(0, 2, 1))
        assert (np.linalg.eigvalsh(rel) > 0).all()
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300)
    assert r.returncode != 0 and "requires --covariance" in r.stderr
