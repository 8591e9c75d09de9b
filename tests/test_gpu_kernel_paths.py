"""Run-time alternatives of the CUDA path (environment variables read by Solver::init) and the PCG hand-over above 1808
cameras, each against the default path or the oracle.

  bit-identical to the default   RBA_PCG_PARTIALS=0, RBA_PDL=0, RBA_TILE_DEAL=rr, RBA_MATVEC_DEAL=rr (DESIGN.md section 11):
                                 inc, H x, the state after apply, and a native LM run
  oracle bars (test_gpu_parity)  RBA_PCG_CLUSTER in {1, 2, 4, 8} (one CTA: the vector step leaves the register-resident
                                 layout at 114 cameras), RBA_MATVEC=ldg with the dense and the implicit operator, and more
                                 than 1808 cameras on one GPU, where a 16-CTA cluster takes the arrival-counter reduction
                                 into D.y and the non-register-resident vector step
"""
import numpy as np
import pytest

from conftest import rel_err
from test_gpu_parity import TOL1, TOLS, make_pair

pytestmark = pytest.mark.gpu

VEC_THREADS, VEC_EPT = 512, 2  # kernels.cuh: k_pcg_vec keeps 9 ceil(nc / cluster) <= VEC_THREADS * VEC_EPT in registers


def vec_cached(nc, cluster):
    return 9 * -(-nc // cluster) <= VEC_THREADS * VEC_EPT


@pytest.fixture(scope="module")
def dealt_problem():
    """a scaled Ladybug-1723 stand-in with more small matvec items than the TMA operator has resident warps, so that the
    longest-first dealing with its empty padding items is active (and more tiles than the tile kernels have warps)"""
    from rootba_b200.synthetic import synth_config
    return synth_config("ladybug-1723", scale=0.5)


@pytest.fixture(scope="module")
def mid_problem():
    from rootba_b200.synthetic import synth_bal
    return synth_bal(150, 1500, 4.1, seed=12)


@pytest.fixture(scope="module")
def many_cameras():
    from rootba_b200.synthetic import synth_bal
    a = synth_bal(2200, 16000, 4.5, seed=13)
    assert np.unique(a.obs_cam).size == a.nc and not vec_cached(a.nc, 16)
    return a


def _run(arrays, dtype, env, monkeypatch, **opt):
    """inc, H x, l_diff and state after apply, then a native LM run of 4 iterations from the original state"""
    import rootba_b200 as rb
    with monkeypatch.context() as m:
        for k, v in env.items():
            m.setenv(k, v)
        bp = rb.BalProblem.from_arrays(arrays, dtype)
        lin = rb.LinearizorQR.create(bp, rb.SolverOptions(max_num_iterations=4, **opt))
    out = {"stats": lin.stats()}
    lin.linearize()
    out["inc"] = lin.solve(1e-3)
    out["cg"] = lin.last_cg.num_iterations
    out["Hx"] = lin.right_multiply(np.random.default_rng(1).uniform(-1, 1, 9 * lin.nc).astype(dtype))
    out["l_diff"] = lin.apply(out["inc"])
    lin.download_state()
    out["cams"], out["lms"] = bp.cams.copy(), bp.lms.copy()
    bp2 = rb.BalProblem.from_arrays(arrays, dtype)
    bp.cams[:], bp.lms[:] = bp2.cams, bp2.lms
    lin.upload_state()
    its, _, _ = lin.lm_run(4)
    lin.download_state()
    out["lm"] = [(i["cost"], i["cg_iterations"], i["accepted"], i["lambda"]) for i in its]
    out["lm_state"] = (bp.cams.copy(), bp.lms.copy())
    lin.close()
    return out


def _assert_identical(a, b):
    assert np.array_equal(a["inc"], b["inc"]) and a["cg"] == b["cg"]
    assert np.array_equal(a["Hx"], b["Hx"])
    assert a["l_diff"] == b["l_diff"]
    assert np.array_equal(a["cams"], b["cams"]) and np.array_equal(a["lms"], b["lms"])
    assert a["lm"] == b["lm"]
    assert np.array_equal(a["lm_state"][0], b["lm_state"][0]) and np.array_equal(a["lm_state"][1], b["lm_state"][1])


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("env", [{"RBA_PCG_PARTIALS": "0"}, {"RBA_PDL": "0"}, {"RBA_TILE_DEAL": "rr"}, {"RBA_MATVEC_DEAL": "rr"}],
                         ids=lambda e: "-".join(f"{k}={v}" for k, v in e.items()))
def test_alternative_is_bit_identical(dealt_problem, dtype, env, monkeypatch):
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ref = _run(dealt_problem, dtype, {}, monkeypatch)
    # more small items than warps of the TMA operator (at most 5 CTAs of 4 warps per SM), and more tiles than warps of
    # k_linearize_qr: both dealt layouts are active in the default run
    assert ref["stats"]["num_matvec_items"] > sms * 5 * 4 and ref["stats"]["num_tiles"] > sms * 8 * 4
    _assert_identical(_run(dealt_problem, dtype, env, monkeypatch), ref)


def _against_oracle(arrays, dtype, env, monkeypatch, solver_type="SQUARE_ROOT", **kw):
    """one linearize + solve + H x + apply against the oracle (SQUARE_ROOT: QR restatement, SCHUR_COMPLEMENT: LinearizorSC)"""
    import rootba_b200 as rb
    from oracle import oracle_py as orc
    with monkeypatch.context() as m:
        for k, v in env.items():
            m.setenv(k, v)
        bp = rb.BalProblem.from_arrays(arrays, dtype)
        lin = rb.LinearizorQR.create(bp, rb.SolverOptions(solver_type=solver_type, **kw))
    o = orc.Oracle(arrays, dtype, orc.default_options(num_threads=0))
    lam = 1e-3
    x = np.random.default_rng(2).uniform(-1, 1, 9 * lin.nc).astype(dtype)
    lin.linearize()
    inc_g = lin.solve(lam)
    if solver_type == "SQUARE_ROOT":
        tol, tols = TOL1[dtype] * (10 if kw.get("operator_form") == "IMPLICIT" and dtype == np.float32 else 1), TOLS[dtype]
        assert o.linearize()
        inc_c, dbg = o.solve(lam, want_debug=True)
        y_c = o.right_multiply(x)
    else:  # test_gpu_sc's bars: the Schur complement squares the landmark block's condition number
        tol, tols = {np.float32: 1e-3, np.float64: 1e-9}[dtype] / 4, {np.float32: 1e-2, np.float64: 1e-8}[dtype]
        o.scl_linearize()
        inc_c, dbg = o.scl_solve(lam)
        o.sc_linearize(); o.sc_scale_Jp(o.scl_get_scaling())
        y_c = o.sc_get_Hb(lam, lam, x)[2]
    assert rel_err(lin.get_rhs(), dbg["b"]) < 4 * tol
    assert abs(lin.last_cg.num_iterations - dbg["cg_iterations"]) <= 2
    assert lin.last_cg.termination_type == dbg["cg_termination"]
    assert rel_err(inc_g, inc_c) < tols
    assert rel_err(lin.right_multiply(x), y_c) < 4 * tol
    lin.close()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("cluster", [1, 2, 4, 8])
def test_pcg_cluster_sizes(mid_problem, dtype, cluster, monkeypatch):
    assert vec_cached(mid_problem.nc, cluster) == (cluster > 1)  # one CTA: the non-register-resident vector step
    _against_oracle(mid_problem, dtype, {"RBA_PCG_CLUSTER": str(cluster)}, monkeypatch)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("form", ["DENSE", "IMPLICIT"])
def test_matvec_without_tma(mid_problem, dtype, form, monkeypatch):
    """RBA_MATVEC=ldg: k_matvec_small instead of the TMA kernel (dense), k_matvec_implicit for every tile (implicit)"""
    _against_oracle(mid_problem, dtype, {"RBA_MATVEC": "ldg"}, monkeypatch, operator_form=form)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("solver_type", ["SQUARE_ROOT", "SCHUR_COMPLEMENT"])
def test_more_than_1808_cameras(many_cameras, dtype, solver_type, monkeypatch):
    _against_oracle(many_cameras, dtype, {}, monkeypatch, solver_type=solver_type)
    # the native LM loop equals the Python mirror of the same loop, bit for bit
    import rootba_b200 as rb
    so = rb.SolverOptions(solver_type=solver_type, max_num_iterations=4)
    bpa, bpb = rb.BalProblem.from_arrays(many_cameras, dtype), rb.BalProblem.from_arrays(many_cameras, dtype)
    summ = rb.bundle_adjust_manual(bpa, so)
    lin = rb.LinearizorQR.create(bpb, so)
    its, _, _ = lin.lm_run(64)
    py = summ["iterations"][1:]
    assert len(its) == len(py)
    for a, b in zip(py, its):
        assert bool(a["step_is_successful"]) == b["accepted"] and a["linear_solver_iterations"] == b["cg_iterations"]
        assert a["cost"]["all"]["error"] == b["cost"] and a["lam"] == b["lambda"]
    lin.download_state()
    assert np.array_equal(bpa.cams, bpb.cams) and np.array_equal(bpa.lms, bpb.lms)
    lin.close()
