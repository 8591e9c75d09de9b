"""The assembled reduced camera matrix S = sum_l P_l^T P_l (DESIGN.md section 4, "Assembled operator"): with one GPU and the
dense operator the PCG operator is S x instead of P^T (P x).  Checked against the panel product of the same handle type
(RBA_ASSEMBLED_RCS=0) and against a float64 P^T (P x) of the same panels (rba_debug_get_block), with S built from the
first PCG iteration on (RBA_ASSEMBLED_AT=1; by default a solve builds it once it has run the break-even number of
iterations, RBA_ASSEMBLED_AT=5 covers that switch inside a solve), at every track-length
class, with cameras without observations, held cameras, camera / pair / landmark priors, Huber, Givens QR and
stage2_form IDENTITY; two lambdas on one linearisation, a rejected step, and a bit-identical native LM run on two handles.
"""
import numpy as np
import pytest

from conftest import rel_err

pytestmark = pytest.mark.gpu

TOL = {np.float32: 1e-5, np.float64: 1e-12}
ASM, PANEL = {"RBA_ASSEMBLED_AT": "1"}, {"RBA_ASSEMBLED_RCS": "0"}


def _problem(name):
    from rootba_b200.synthetic import synth_bal
    # enough landmarks per camera that S is at most a quarter of the panels (the assembled operator is taken)
    if name == "mixed":  # every group-size class incl. row-chunked tracks
        return synth_bal(150, 6000, 9.0, seed=11, max_track=150)
    a = synth_bal(30, 3000, 4.1, seed=5)
    if name == "unobserved":  # three cameras at the end that no landmark sees
        from rootba_b200.synthetic import BalArrays
        return BalArrays(np.concatenate([a.cams, a.cams[:3]]), a.lms, a.lm_off, a.obs_cam, a.obs_xy)
    return a


def _priors(lin, arrays, dtype, which):
    rng = np.random.default_rng(3)
    nc = lin.nc
    if which == "camera":
        mean = arrays.cams.astype(np.float64).copy()
        mean[:, :4] /= np.linalg.norm(mean[:, :4], axis=1, keepdims=True)
        L = np.zeros((nc, 9, 9))
        L[:, range(9), range(9)] = rng.uniform(0.5, 2.0, (nc, 9))
        lin.set_camera_prior((mean.astype(dtype), L.astype(dtype)))
    elif which == "pair":
        pairs = np.array([[0, 1], [2, 5], [7, 3]], np.int32)
        mean = np.zeros((3, 7)); mean[:, 0] = 1.0
        L = np.tile(np.eye(6), (3, 1, 1)) * 0.7
        lin.set_camera_pair_prior((pairs, mean.astype(dtype), L.astype(dtype)))
    elif which == "landmark":
        idx = np.arange(0, arrays.nl, 7, dtype=np.int32)
        L = np.tile(np.eye(3), (idx.size, 1, 1)) * 1.5
        lin.set_landmark_prior((idx, arrays.lms[idx].astype(dtype), L.astype(dtype)))
    elif which == "fixed":
        flags = np.zeros(nc, np.uint8); flags[0] = 15; flags[4] = 2
        lin.set_camera_fixed(flags)


def _make(arrays, dtype, env, monkeypatch, prior=None, **opt):
    import rootba_b200 as rb
    with monkeypatch.context() as m:
        for k, v in env.items():
            m.setenv(k, v)
        bp = rb.BalProblem.from_arrays(arrays, dtype)
        if "huber" in opt:
            opt = dict(opt)
            opt["residual"] = rb.ResidualOptions(robust_norm="HUBER", huber_parameter=opt.pop("huber"))
        lin = rb.LinearizorQR.create(bp, rb.SolverOptions(use_double=dtype == np.float64, **opt))
    if prior:
        _priors(lin, arrays, dtype, prior)
    return lin


def _panel_product(lin, arrays, x):
    """float64 sum_l P_l^T (P_l x) over the Q2 panels and damping rows of the handle (rba_debug_get_block)"""
    y = np.zeros(9 * lin.nc)
    for lm in range(arrays.nl):
        k0, k1 = int(arrays.lm_off[lm]), int(arrays.lm_off[lm + 1])
        n = k1 - k0
        blk, _, _, _ = lin.debug_get_block(lm)
        P = blk[3:3 + 2 * n, :9 * n].astype(np.float64)
        cams = arrays.obs_cam[k0:k1]
        xl = x.reshape(-1, 9)[cams].ravel()
        y.reshape(-1, 9)[cams] += (P.T @ (P @ xl)).reshape(n, 9)
    return y


CASES = {
    "mixed": ("mixed", None, {}),
    "unobserved": ("unobserved", None, {}),
    "fixed": ("small", "fixed", {}),
    "camera-prior": ("small", "camera", {}),
    "pair-prior": ("small", "pair", {}),
    "landmark-prior": ("small", "landmark", {}),
    "huber": ("small", None, {"huber": 0.5}),
    "givens": ("small", None, {"use_householder_marginalization": False}),
    "identity": ("mixed", None, {"stage2_form": "IDENTITY"}),
}


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("case", list(CASES))
def test_against_panel_product(case, dtype, monkeypatch):
    name, prior, opt = CASES[case]
    arrays = _problem(name)
    x = np.random.default_rng(1).uniform(-1, 1, 9 * arrays.nc)
    out = {}
    for tag, env in (("asm", ASM), ("panel", PANEL)):
        lin = _make(arrays, dtype, env, monkeypatch, prior, **opt)
        lin.linearize()
        out[tag + "_inc"] = lin.solve(1e-3)
        out[tag + "_cg"] = lin.last_cg.num_iterations
        out[tag + "_bytes"] = lin.stats()["matvec_algorithmic_bytes"]
        out[tag + "_y"] = lin.right_multiply(x.astype(dtype)).astype(np.float64)
        if tag == "asm" and prior is None:
            # without priors right_multiply is the operator plus lambda x
            ref = _panel_product(lin, arrays, x.astype(dtype).astype(np.float64)) + 1e-3 * x.astype(dtype)
            assert rel_err(out["asm_y"], ref) < TOL[dtype]
        lin.close()
    assert out["asm_bytes"] < out["panel_bytes"]  # the assembled operator was taken, and the hook forced the panels
    assert rel_err(out["asm_y"], out["panel_y"]) < TOL[dtype]
    assert abs(out["asm_cg"] - out["panel_cg"]) <= 2
    assert rel_err(out["asm_inc"], out["panel_inc"]) < {np.float32: 1e-3, np.float64: 1e-9}[dtype]
    if name == "unobserved":
        assert np.all(out["asm_y"][-27:] == (1e-3 * x.astype(dtype)[-27:]).astype(dtype))


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_new_lambda_and_rejected_step(dtype, monkeypatch):
    """S is rebuilt for every lambda: two lambdas on one linearisation, then a step undone and a solve at a new lambda"""
    arrays = _problem("mixed")
    x = np.random.default_rng(4).uniform(-1, 1, 9 * arrays.nc).astype(dtype)
    a = _make(arrays, dtype, ASM, monkeypatch)
    b = _make(arrays, dtype, PANEL, monkeypatch)
    for lin in (a, b):
        lin.linearize()
    for lam in (1e-4, 1e2):
        ia, ib = a.solve(lam), b.solve(lam)
        assert rel_err(a.right_multiply(x), b.right_multiply(x)) < TOL[dtype]
        assert rel_err(ia, ib) < {np.float32: 1e-3, np.float64: 1e-9}[dtype]
    for lin in (a, b):  # apply, undo, solve again at a third lambda on the same linearisation
        lin._backup()
        lin.apply(lin.solve(1e-2))
        lin._restore()
    ia, ib = a.solve(3.0), b.solve(3.0)
    assert rel_err(a.right_multiply(x), b.right_multiply(x)) < TOL[dtype]
    assert rel_err(ia, ib) < {np.float32: 1e-3, np.float64: 1e-9}[dtype]
    a.close(); b.close()


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_lm_run_bit_identical_on_two_handles(dtype, monkeypatch):
    """S built inside every solve that reaches iteration 5"""
    arrays = _problem("mixed")
    runs = []
    for _ in range(2):
        lin = _make(arrays, dtype, {"RBA_ASSEMBLED_AT": "5"}, monkeypatch, max_num_iterations=6)
        its, _, _ = lin.lm_run(6)
        lin.download_state()
        runs.append(([(i["cost"], i["cg_iterations"], i["accepted"], i["lambda"]) for i in its],
                     lin.bal_problem.cams.copy(), lin.bal_problem.lms.copy()))
        lin.close()
    assert runs[0][0] == runs[1][0]
    assert np.array_equal(runs[0][1], runs[1][1]) and np.array_equal(runs[0][2], runs[1][2])


def test_ladybug_full_size(monkeypatch):
    """Ladybug-1723 stand-in at full size, float32: H x against the panel product, PCG count within 2"""
    from rootba_b200.synthetic import synth_config
    arrays = synth_config("ladybug-1723")
    x = np.random.default_rng(5).uniform(-1, 1, 9 * arrays.nc).astype(np.float32)
    out = {}
    for tag, env in (("asm", ASM), ("panel", PANEL)):
        lin = _make(arrays, np.float32, env, monkeypatch)
        lin.linearize()
        lin.solve(1e-4)
        out[tag] = (lin.right_multiply(x), lin.last_cg.num_iterations, lin.stats())
        lin.close()
    assert out["asm"][2]["matvec_algorithmic_bytes"] * 4 < out["panel"][2]["matvec_algorithmic_bytes"]
    assert rel_err(out["asm"][0], out["panel"][0]) < 1e-5
    assert abs(out["asm"][1] - out["panel"][1]) <= 2
