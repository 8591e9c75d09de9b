"""The camera dimension of the solve's hot path, camera by camera, against float64 -- the counterpart of
test_gpu_kernel_classes / test_gpu_solver_classes, which sweep the landmark dimension.

The per-camera kernels branch on the number of slots a camera owns (rootba_b200/csrc/layout.hpp, kernels.cuh, solver.cu):
  SEG_LEN = 96          a camera's slot list is cut into segments, one warp each (k_cam_reduce, k_cam_final9,
                        k_cam_reduce_final, and the segment sums inside k_pcg_vec); one segment takes the i1 - i0 == 1
                        shortcut of k_cam_reduce_final, several the arrival counter and its fixed-order sum
  3 x DEPTH = 48        slots per round of cam_sum_staged
  row chunks            tracks with 2n > 48 rows write one y slot per chunk: a camera's csr_y list is then a multiple of its
                        csr_obs list and crosses 96 at another degree
  PB_SEG_LEN = 16       observations per thread of k_precond_partial (modes 0..3), summed per camera by k_precond_final
  grid_for(n, 8, 8)     at most 8 blocks of 8 warps per SM: more reduce items than warps re-stage in the grid-stride loop
  cluster c             k_pcg_vec / k_power_vec give each CTA ceil(nc / c) cameras: empty CTAs when nc < c, a ragged last
                        CTA, register-resident while 9 ceil(nc / c) <= 1024 (up to 113 c cameras), a camera's 9 entries
                        straddling thread element 512 from 57 cameras per CTA; Solver::handover switches the hand-over at
                        the same threshold
A degree case is a problem whose landmarks all have ONE track length n (2, a G = 4 length, two chunked lengths) and whose
"hub" cameras have exactly the degrees of HUB_DEGREES; filler cameras complete the tracks.  Every camera is checked on its
own, with Higham's gamma_k and k counted from the kernel's summation structure with the camera's OWN slot count:
  SCHUR_JACOBI blocks   sum_l P_c^T P_c + lam I from the kernel's own panels (debug_get_block incl. the damping rows):
                          |B - B^| <= (2 n_c + m_c + 4) u (sum |P_c|^T |P_c| + lam)
                        n_c the longest track at camera c, m_c its observations (2 n_c products per entry and slot, m_c
                        slots in PB_SEG_LEN runs and their sum, + lam, the addend of the damping rows, rounding)
  inverse               of those blocks at the bar of solver_model.inverse with c = 2 n_c + m_c + 4 + 128
  H x (dense)           sum_l P_c^T (P x) + lam x:  |y - y^| <= (11 n_c + my_c + 4) u (sum |P_c|^T (|P| |x|) + lam |x|),
                        my_c the camera's y slots (m_c times the row chunks of its tracks)
  b                     rba_debug_get_block does not return the Q2^T r column, so b is held to the float64 model of
                        tests/solver_model.py (QR == SC) at its bar with the camera's own n_c and m_c
  H x (implicit)        per camera against the float64 product of the dense handle's panels at the bars of DESIGN.md
                        section 9 (test_implicit_operator_class)
  SCHUR_COMPLEMENT,     the quantities of tests/solver_model.py at its bars, with the camera's own n_c, m_c
  JACOBI, IDENTITY
The vector step runs at camera counts on both sides of every edge of the cluster partition (VEC_CASES), iterate by
iterate against pcg_replay / power_replay at the bars of test_gpu_pcg_iterates.  Where arrival counters decide the order
of a sum, two fresh handles, two calls and the two hand-overs must agree bit for bit.
"""
import contextlib
import functools
import os
import re

import numpy as np
import pytest

import solver_model as sm
from conftest import ROOT, rel_err
from pcg_replay import NO_CONVERGENCE, lanczos_condition, pcg_replay, power_replay
from test_gpu_kernel_classes import group_size_for, row_chunks

pytestmark = pytest.mark.gpu

# ---- mirror of the camera-side layout (layout.hpp, kernels.cuh, solver.cu) ----
SEG_LEN = 96             # layout.hpp: slots per camera segment (one warp)
PB_SEG_LEN = 16          # layout.hpp: observations per preconditioner-block item
ROUND = 3 * 16           # kernels.cuh cam_sum_staged: 3 slots x DEPTH 16 per round
VEC_THREADS, VEC_EPT = 512, 2  # kernels.cuh: k_pcg_vec register-resident while 9 cameras-per-CTA <= 1024
WARPS_PER_SM = 8 * 8     # solver.cu: grid_for(items, 8, 8) -- 8 warps per block, at most 8 blocks per SM
CLUSTERS = (1, 2, 4, 8, 16)


def _source_constant(path, name):
    with open(os.path.join(ROOT, "rootba_b200", "csrc", path)) as f:
        return int(re.search(rf"constexpr int {name} = (\d+);", f.read()).group(1))


# the mirror fails loudly when a constant of the kernels changes
assert _source_constant("layout.hpp", "SEG_LEN") == SEG_LEN
assert _source_constant("layout.hpp", "PB_SEG_LEN") == PB_SEG_LEN
assert _source_constant("kernels.cuh", "DEPTH") * 3 == ROUND
assert _source_constant("kernels.cuh", "VEC_THREADS") == VEC_THREADS
assert _source_constant("kernels.cuh", "VEC_EPT") == VEC_EPT


def _ceil(a, b):
    return -(-np.asarray(a) // b)


def segments(count):
    """lengths of the segments of a slot list of `count` entries"""
    return [min(SEG_LEN, count - b) for b in range(0, count, SEG_LEN)]


def rounds(count):
    """cam_sum_staged rounds of the longest segment of the list"""
    return max((int(_ceil(s, ROUND)) for s in segments(count)), default=0)


def camera_layout(arrays):
    """per camera: observations m, y slots my, longest track nmax, csr_obs / csr_y segments, pb_items, rounds"""
    nc, n = arrays.nc, arrays.track_lengths()
    per_obs_n = np.repeat(n, n)
    m = np.bincount(arrays.obs_cam, minlength=nc)
    my = np.bincount(arrays.obs_cam, weights=np.array([row_chunks(k) for k in per_obs_n]), minlength=nc).astype(np.int64)
    nmax = np.zeros(nc, np.int64)
    np.maximum.at(nmax, arrays.obs_cam, per_obs_n)
    return {"m": m, "my": my, "nmax": nmax, "obs_segments": _ceil(m, SEG_LEN), "y_segments": _ceil(my, SEG_LEN),
            "pb_items": _ceil(m, PB_SEG_LEN), "rounds": np.array([rounds(k) for k in m]),
            "y_rounds": np.array([rounds(k) for k in my])}


def vec_partition(nc, cluster):
    """k_pcg_vec's split of nc cameras over a cluster of CTAs"""
    per = -(-nc // cluster)
    sizes = [max(0, min(nc, b * per + per) - min(nc, b * per)) for b in range(cluster)]
    last = max(b for b in range(cluster) if sizes[b] > 0)
    cached = 9 * per <= VEC_THREADS * VEC_EPT
    return {"per_cta": per, "empty": sum(s == 0 for s in sizes), "ragged": sizes[last] < per, "cached": cached,
            "straddle": cached and 9 * per > VEC_THREADS,  # a camera's 9 entries cross thread element 512
            "partials": cached,                            # the Partials hand-over (Solver::handover) on one GPU
            "last_range": (last * per, last * per + sizes[last])}


# ---- degree cases ----
BUSY = 2500
HUB_DEGREES = (0, 1, 2, 3, 15, 16, 17, 31, 32, 33, 47, 48, 49, 95, 96, 97, 191, 192, 193, BUSY)
TRACK_NS = (2, 6, 25, 40)  # G = 1, G = 4, chunked with G = 16 and with G = 32
LAM = 0.1


def hub_tracks(n, nfill, seed):
    """tracks giving camera h < len(HUB_DEGREES) exactly HUB_DEGREES[h] observations; the other n - 1 cameras of every
    track are fillers; the landmarks are shuffled so that a hub's landmarks lie in many tiles and matvec items"""
    rng = np.random.default_rng(seed)
    nh = len(HUB_DEGREES)
    tracks = [np.sort(np.concatenate([[h], nh + rng.choice(nfill, n - 1, replace=False)]))
              for h, d in enumerate(HUB_DEGREES) for _ in range(d)]
    return [tracks[i] for i in rng.permutation(len(tracks))]


@functools.lru_cache(maxsize=None)
def degree_problem(n):
    from rootba_b200.synthetic import synth_bal
    nfill = 4 * n + 24
    tracks = hub_tracks(n, nfill, 500 + n)
    return synth_bal(len(HUB_DEGREES) + nfill, len(tracks), 0.0, seed=500 + n, tracks=tracks, lm_spread=0.5)


@functools.lru_cache(maxsize=None)
def restage_problem(sm_count):
    """one observation per camera (pairs of cameras share a landmark of n = 2): more csr_obs and csr_y items than the
    sm_count * 64 warps of grid_for, and, at 16 CTAs, more than 113 cameras per CTA (the arrival-counter hand-over)"""
    from rootba_b200.synthetic import synth_bal
    nc = 2 * ((sm_count * WARPS_PER_SM) // 2 + 64)
    perm = np.random.default_rng(7).permutation(nc)
    tracks = [np.sort(perm[2 * i:2 * i + 2]) for i in range(nc // 2)]
    return synth_bal(nc, len(tracks), 0.0, seed=7, tracks=tracks, lm_spread=0.5)


def _vec_cases():
    out = []
    for c in CLUSTERS:
        for nc in sorted({113 * c, 113 * c + 1, c - 1, c, c + 1, 64, 65}):
            if nc >= 2:
                out.append((c, nc))
    return out


VEC_CASES = _vec_cases()
# an unobserved camera in the last CTA: the last camera of every problem with nc = c + 1 or 113 c + 1 (>= 4) sees nothing
UNOBSERVED_LAST = {(c, nc) for c, nc in VEC_CASES if nc in (c + 1, 113 * c + 1) and nc >= 4}


@functools.lru_cache(maxsize=None)
def vec_problem(nc, unobserved_last):
    """nc cameras, tracks of up to 4 cameras, every camera observed (but the last, if asked)"""
    from rootba_b200.synthetic import synth_bal
    rng = np.random.default_rng(nc)
    seen = nc - 1 if unobserved_last else nc
    nl = max(12, 3 * seen)
    k = min(4, seen)
    tracks = [np.sort(np.concatenate([[i % seen], rng.choice(np.delete(np.arange(seen), i % seen), k - 1, replace=False)]))
              for i in range(nl)]
    return synth_bal(nc, nl, 0.0, seed=nc, tracks=tracks, lm_spread=0.5)


# ---- the boundaries of the module docstring are reached on both sides ----
def _reached():
    seg, rnd, ysplit, pb = set(), set(), set(), set()
    for n in TRACK_NS:
        lay = camera_layout(degree_problem(n))
        hubs = slice(0, len(HUB_DEGREES))
        seg |= set(lay["obs_segments"][hubs]) | set(lay["y_segments"][hubs])
        rnd |= set(lay["rounds"][hubs]) | set(lay["y_rounds"][hubs])
        pb |= set(lay["pb_items"][hubs])
        ysplit.add(bool(np.any(lay["y_segments"] != lay["obs_segments"])))
    return seg, rnd, ysplit, pb


_SEG, _RND, _YSPLIT, _PB = _reached()
assert {0, 1, 2, 3} <= _SEG and max(_SEG) >= 20, _SEG           # none, one, several, tens of segments
assert {0, 1, 2} <= _RND, _RND                                  # one and two 48-slot rounds
assert _YSPLIT == {False, True}                                 # csr_y == csr_obs and csr_y != csr_obs
assert {1, 2, 3, 4} <= _PB and max(_PB) > 100, _PB              # pb_items
assert all(degree_problem(n).track_lengths().max() == n for n in TRACK_NS)
assert {row_chunks(n) > 1 for n in TRACK_NS} == {False, True} and group_size_for(6) == 4
# a degree-48 camera of n = 25 has 96 y slots (one segment), degree 49 has 98 (two)
assert [int(v) for v in _ceil(2 * np.array([48, 49]), SEG_LEN)] == [1, 2] and row_chunks(25) == 2
_PARTS = [vec_partition(nc, c) for c, nc in VEC_CASES]
assert {p["cached"] for p in _PARTS} == {True, False} and {p["partials"] for p in _PARTS} == {True, False}
assert any(p["empty"] > 0 for p in _PARTS) and any(p["empty"] == 0 for p in _PARTS)
assert {p["ragged"] for p in _PARTS} == {True, False} and {p["straddle"] for p in _PARTS} == {True, False}
assert all(vec_partition(113 * c, c)["cached"] and not vec_partition(113 * c + 1, c)["cached"] for c in CLUSTERS)
assert any(vec_partition(nc, c)["last_range"][1] == nc and (c, nc) in UNOBSERVED_LAST for c, nc in VEC_CASES)


# ---- float64 references from the kernel's own panels ----
def chunk_rows(n):
    """row ranges of the matvec items of a track of length n (layout.hpp: rows * c / nchunks)"""
    rows, k = 2 * n, row_chunks(n)
    return [(rows * c // k, rows * (c + 1) // k) for c in range(k)]


class PanelSums:
    """per camera, float64, accumulated batch by batch: b = sum P_c^T t, B = sum P_c^T P_c + lam I, y = sum P_c^T P x + lam x
    and their magnitudes; for the cameras in `record`, every observation's (landmark, contribution to B) and every y slot's
    (landmark, chunk, contribution to y)"""

    def __init__(self, arrays, lam, x, record=()):
        self.arrays, self.nc, self.lam = arrays, arrays.nc, lam
        self.x = np.asarray(x, np.float64).reshape(self.nc, 9)
        self.s = {k: np.zeros((self.nc, 9)) for k in ("b", "Mb", "y", "My")}
        self.s["B"], self.s["MB"] = np.zeros((self.nc, 9, 9)), np.zeros((self.nc, 9, 9))
        self.record = set(int(c) for c in record)
        self.obs = {c: [] for c in self.record}
        self.yslots = {c: [] for c in self.record}

    def add(self, lms, P, t):
        """P [k, 2n, 9n] panels incl. the damping rows and t [k, 2n] Q2^T r columns of the landmarks lms"""
        a, nl = self.arrays, len(lms)
        n = P.shape[2] // 9
        cams = np.stack([a.obs_cam[a.lm_off[lm]:a.lm_off[lm + 1]] for lm in lms])
        P4 = P.reshape(nl, 2 * n, n, 9)
        A4 = np.abs(P4)
        xc = self.x[cams]
        px, apx = np.einsum("lrkc,lkc->lr", P4, xc), np.einsum("lrkc,lkc->lr", A4, np.abs(xc))
        s = self.s
        np.add.at(s["b"], cams, np.einsum("lrkc,lr->lkc", P4, t))
        np.add.at(s["Mb"], cams, np.einsum("lrkc,lr->lkc", A4, np.abs(t)))
        np.add.at(s["B"], cams, np.einsum("lrkc,lrkd->lkcd", P4, P4))
        np.add.at(s["MB"], cams, np.einsum("lrkc,lrkd->lkcd", A4, A4))
        np.add.at(s["y"], cams, np.einsum("lrkc,lr->lkc", P4, px))
        np.add.at(s["My"], cams, np.einsum("lrkc,lr->lkc", A4, apx))
        for i, lm in enumerate(lms):
            for k, c in enumerate(cams[i]):
                if int(c) in self.record:
                    Pk = P4[i, :, k]
                    self.obs[int(c)].append((lm, Pk.T @ Pk))
                    for ch, (r0, r1) in enumerate(chunk_rows(n)):
                        self.yslots[int(c)].append((lm, ch, Pk[r0:r1].T @ px[i, r0:r1]))

    def result(self):
        out = {k: v.copy() for k, v in self.s.items()}
        eye = self.lam * np.eye(9)
        out["B"] += eye
        out["MB"] += eye
        out["y"] += self.lam * self.x
        out["My"] += self.lam * np.abs(self.x)
        return out


def panel_sums(arrays, get_block, lam, x, record=(), batch=128):
    """PanelSums over every landmark; get_block(lm) -> (block, lm_idx, res_idx, ...) in the reference storage layout"""
    ps = PanelSums(arrays, lam, x, record)
    n = int(arrays.track_lengths()[0])
    assert np.all(arrays.track_lengths() == n)
    for b0 in range(0, arrays.nl, batch):
        lms = list(range(b0, min(arrays.nl, b0 + batch)))
        blks = [get_block(lm) for lm in lms]
        P = np.stack([bg[3:, :9 * n] for bg, *_ in blks]).astype(np.float64)
        t = np.stack([bg[3:, ri] for bg, _, ri, *_ in blks]).astype(np.float64)
        ps.add(lms, P, t)
    return ps


def y_segments_of(ps, cam, n):
    """the camera's csr_y list cut into SEG_LEN segments, each a list of (landmark, chunk, contribution): observation slots
    in landmark order, then the slots of the extra row chunks by (tile, chunk, landmark) (one track length: tile = lm // W)"""
    w = 32 // group_size_for(n)
    first = sorted((e for e in ps.yslots[cam] if e[1] == 0), key=lambda e: e[0])
    extra = sorted((e for e in ps.yslots[cam] if e[1] > 0), key=lambda e: (e[0] // w, e[1], e[0]))
    ys = first + extra
    return [ys[b:b + SEG_LEN] for b in range(0, len(ys), SEG_LEN)]


def pb_items_of(ps, cam):
    """the camera's observations (landmark order) cut into PB_SEG_LEN items, each a list of (landmark, P_c^T P_c)"""
    ob = sorted(ps.obs[cam], key=lambda e: e[0])
    return [ob[b:b + PB_SEG_LEN] for b in range(0, len(ob), PB_SEG_LEN)]


def bar_constants(arrays):
    """per-camera c of the blocks / b (2 n_c + m_c + 4) and of H x (11 n_c + my_c + 4)"""
    lay = camera_layout(arrays)
    return 2 * lay["nmax"] + lay["m"] + 4, 11 * lay["nmax"] + lay["my"] + 4


def excess_per_camera(got, want, mag, c, u):
    """the largest |got - want| / (c_cam u mag) of every camera (<= 1: accepted)"""
    nc = want.shape[0]
    got = np.asarray(got, np.float64).reshape(want.shape)
    cc = np.asarray(c, np.float64).reshape((nc,) + (1,) * (want.ndim - 1))
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.abs(got - want) / (cc * u * mag)
    ratio = np.where(got == want, 0.0, ratio)
    ratio = np.where(np.isnan(ratio), np.inf, ratio)
    return ratio.reshape(nc, -1).max(axis=1)


def check_per_camera(got, want, mag, c, u, what):
    e = excess_per_camera(got, want, mag, c, u)
    worst = int(np.argmax(e))
    assert e[worst] <= 1, (what, "camera", worst, "error / bar", e[worst])


def check_inverse_per_camera(got, B, MB, c, u, what):
    for cam in range(B.shape[0]):
        want, M = sm.inverse(B[cam], MB[cam])
        e, k = sm.excess(got[cam], want, M, c[cam] + sm.C_FIXED, u)
        assert e <= 1, (what, "camera", cam, "entry", k, "error / bar", e)


def model_constants(arrays, model):
    """solver_model's c with the camera's own longest track and degree instead of the problem's"""
    lay = camera_layout(arrays)
    return np.array([sm.bar_constant(int(n), int(m), model.kappa) for n, m in zip(lay["nmax"], lay["m"])], np.float64)


def check_model(got, want, mag, c_cam, model, what):
    check_per_camera(got, want, mag, c_cam, model.u, what)


def check_model_inverse(got, B, MB, c_cam, model, what):
    for cam in range(B.shape[0]):
        want, M = sm.inverse(B[cam], MB[cam])
        e, k = sm.excess(got[cam], want, M, c_cam[cam], model.u)
        assert e <= 1, (what, "camera", cam, "entry", k, "error / bar", e)


# ---- GPU helpers ----
@contextlib.contextmanager
def _env(env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _handle(arrays, dtype, env=None, **opt):
    import rootba_b200 as rb
    with _env(env or {}):
        bp = rb.BalProblem.from_arrays(arrays, dtype)
        lin = rb.LinearizorQR.create(bp, rb.SolverOptions(**opt))
    lin.linearize()
    return lin


def _u(dtype):
    return sm.unit_roundoff(dtype)


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _case(name):
    if name == "restage":
        return restage_problem(_sm_count())
    return degree_problem(int(name))


CASES = [str(n) for n in TRACK_NS] + ["restage"]


def _case_dtypes():
    return [(c, d) for c in CASES for d in ((np.float32, np.float64) if c != "restage" else (np.float64,))]


def _ids(v):
    return v if isinstance(v, str) else np.dtype(v).name


def _x(nc, dtype, seed=3):
    return np.random.default_rng(seed).uniform(-1, 1, 9 * nc).astype(dtype)


@pytest.mark.parametrize("case,dtype", _case_dtypes(), ids=lambda v: _ids(v))
def test_dense_camera_class(case, dtype):
    """SCHUR_JACOBI blocks, their inverse and H x from the kernel's own panels, b against the float64 model"""
    arrays = _case(case)
    nc, u = arrays.nc, _u(dtype)
    if case == "restage":
        lay = camera_layout(arrays)
        assert lay["obs_segments"].sum() > _sm_count() * WARPS_PER_SM and not vec_partition(nc, 16)["cached"]
    lin = _handle(arrays, dtype)
    lin.solve(LAM)
    x = _x(nc, dtype)
    ref = panel_sums(arrays, lin.debug_get_block, float(dtype(LAM)), x).result()
    cb, cy = bar_constants(arrays)
    inv, blk = lin.get_preconditioner()
    check_per_camera(blk, ref["B"], ref["MB"], cb, u, "SCHUR_JACOBI blocks")
    check_inverse_per_camera(inv, ref["B"], ref["MB"], cb, u, "inverse")
    check_per_camera(lin.right_multiply(x), ref["y"], ref["My"], cy, u, "H x")
    model = sm.SCModel(arrays, dtype, lin.get_jacobian_scaling()[0], LAM)
    b, Mb = model.b()
    check_model(lin.get_rhs(), b, Mb, model_constants(arrays, model), model, "b")
    lin.close()


@pytest.mark.parametrize("case,dtype", _case_dtypes(), ids=lambda v: _ids(v))
def test_implicit_camera_class(case, dtype):
    """operator_form = IMPLICIT: H x per camera against the float64 product of the dense handle's panels (section 9 bars)"""
    from test_gpu_parity import TOL1
    arrays = _case(case)
    nc = arrays.nc
    dense = _handle(arrays, dtype)
    dense.solve(LAM)
    x = _x(nc, dtype)
    y_hat = panel_sums(arrays, dense.debug_get_block, float(dtype(LAM)), x).result()["y"]
    dense.close()
    lin = _handle(arrays, dtype, operator_form="IMPLICIT")
    lin.solve(LAM)
    y = lin.right_multiply(x).astype(np.float64).reshape(nc, 9)
    lin.close()
    tol = 4 * TOL1[dtype] * (10 if dtype == np.float32 else 1)
    worst = max(range(nc), key=lambda c: rel_err(y[c], y_hat[c]))
    assert rel_err(y[worst], y_hat[worst]) < tol, ("H x", worst, rel_err(y[worst], y_hat[worst]))


MODEL_SOLVERS = {"schur_complement": {"solver_type": "SCHUR_COMPLEMENT"}, "jacobi": {"preconditioner_type": "JACOBI"},
                 "identity": {"stage2_form": "IDENTITY"}}


@pytest.mark.parametrize("solver", list(MODEL_SOLVERS))
@pytest.mark.parametrize("case,dtype", _case_dtypes(), ids=lambda v: _ids(v))
def test_model_camera_class(case, dtype, solver):
    """the quantities of tests/solver_model.py at its bars, with the camera's own n_c and m_c"""
    arrays = _case(case)
    nc = arrays.nc
    lin = _handle(arrays, dtype, **MODEL_SOLVERS[solver])
    lin.solve(LAM)
    model = sm.SCModel(arrays, dtype, lin.get_jacobian_scaling()[0], LAM)
    cc = model_constants(arrays, model)
    inv, blk = lin.get_preconditioner()
    if solver == "jacobi":
        J, MJ = model.jacobi_blocks()
        check_model_inverse(inv, J, MJ, cc, model, "inverse of the JACOBI blocks")
    else:
        B, MB = model.schur_blocks()
        check_model(blk, B, MB, cc, model, "SCHUR_JACOBI blocks")
        check_model_inverse(inv, B, MB, cc, model, "inverse")
    b, Mb = model.b()
    check_model(lin.get_rhs(), b, Mb, cc, model, "b")
    x = _x(nc, dtype)
    y, My = model.hx(x)
    check_model(lin.right_multiply(x), y, My, cc, model, "H x")
    lin.close()


@pytest.mark.parametrize("case,dtype", _case_dtypes(), ids=lambda v: _ids(v))
def test_camera_sums_are_bit_reproducible(case, dtype):
    """b, the blocks, H x and inc of two fresh handles, two consecutive right_multiply calls, and RBA_PCG_PARTIALS=0 (inc,
    the iteration count, H x) agree bit for bit"""
    arrays = _case(case)
    x = _x(arrays.nc, dtype)

    def run(env):
        lin = _handle(arrays, dtype, env)
        inc = lin.solve(LAM)
        inv, blk = lin.get_preconditioner()
        y1, y2 = lin.right_multiply(x), lin.right_multiply(x)
        out = {"b": lin.get_rhs(), "inv": inv, "blk": blk, "inc": inc, "it": lin.last_cg.num_iterations, "y": y1}
        lin.close()
        assert np.array_equal(y1, y2), "two right_multiply calls differ"
        return out

    a, b, c = run({}), run({}), run({"RBA_PCG_PARTIALS": "0"})
    for k in a:
        assert np.array_equal(a[k], b[k]), k
    for k in ("inc", "it", "y"):
        assert np.array_equal(a[k], c[k]), ("RBA_PCG_PARTIALS=0", k)


# ---- the vector step at camera-count edges ----
LAM_PCG = 0.1            # the vector step does not depend on lam; 0.1 keeps kappa of the random-track problems small
LAM_POWER = 0.1
C_BAR = 10
NEVER = -1e30
BAR_MAX = {np.float32: 1e-2, np.float64: 1e-8}
BAR_MAX_CONVERGED = {np.float32: 3e-2, np.float64: 1e-8}
F32_MAX_CAMERAS = 278        # 9 nc <= 2500: H assembled from the unit vectors stays cheap
CONVERGED_POWER = 40


def _vec_params():
    out = []
    for c, nc in VEC_CASES:
        for dtype in (np.float32, np.float64) if nc <= F32_MAX_CAMERAS else (np.float64,):
            out.append(pytest.param(c, nc, dtype, id=f"c{c}-nc{nc}-{np.dtype(dtype).name}"))
    return out


def _vec_setup(c, nc, dtype, **opt):
    arrays = vec_problem(nc, (c, nc) in UNOBSERVED_LAST)
    return arrays, {"RBA_PCG_CLUSTER": str(c)}


def _plain_operator(lin, dtype):
    from test_gpu_pcg_iterates import operator_of
    return operator_of(lin, dtype), (lambda v: v)


def _truncated(arrays, dtype, env, lam, handle=_handle, **opt):
    lin = handle(arrays, dtype, env, **opt)
    inc = lin.solve(lam)
    out = (inc, lin.last_cg.termination_type, lin.last_cg.num_iterations, lin.get_rhs(), lin.get_preconditioner()[0])
    lin.close()
    return out


SENSITIVITY_TRIALS = 8


def replay_sensitivity(op, b, inv, n_it, u, n):
    """S_k: the largest relative deviation of iterate k over SENSITIVITY_TRIALS float64 replays whose every operator
    application is perturbed entry by entry by a uniform C_BAR u (|H| |v|), H assembled from the n unit vectors"""
    H = np.stack([np.asarray(op(np.eye(n)[j]), np.float64) for j in range(n)], axis=1)
    ref = pcg_replay(lambda v: H @ v, b, inv, eta=NEVER, max_it=n_it)["xs"]
    rng = np.random.default_rng(0)
    S = np.zeros(len(ref))
    for _ in range(SENSITIVITY_TRIALS):
        pert = lambda v: H @ v + rng.uniform(-1, 1, n) * C_BAR * u * (np.abs(H) @ np.abs(v))
        xs = pcg_replay(pert, b, inv, eta=NEVER, max_it=n_it)["xs"]
        S[:len(xs)] = np.maximum(S[:len(xs)], [rel_err(x, y) for x, y in zip(xs, ref)])
    return S


def pcg_edge_sweep(arrays, dtype, env, handle=_handle, operator=_plain_operator, sensitivity=False):
    """PCG truncated at 1, 2, 3 iterations and at convergence against pcg_replay on the handle's own b, M^-1 and operator.
    handle(arrays, dtype, env, **opt) makes a linearised handle; operator(lin, dtype) gives the replay's operator and the map
    from the replay's vector to the increment.  sensitivity: the bar of iterate k is at least 4 S_k (replay_sensitivity)"""
    lin = handle(arrays, dtype, env)
    lin.solve(LAM_PCG)
    try:
        b, inv = lin.get_rhs(), lin.get_preconditioner()[0]
        op, expand = operator(lin, dtype)
        full = pcg_replay(op, b, inv, eta=NEVER, max_it=min(600, 9 * arrays.nc))
        xs = full["xs"]
        # converged: the first step that changes the iterate by less than 1e-4; kappa from the Lanczos tridiagonal of the
        # coefficients up to there (beyond it they are rounding noise and the Ritz values lose their meaning)
        k_conv = next((k for k in range(1, len(xs)) if rel_err(xs[k], xs[k - 1]) < 1e-4), len(xs) - 1)
        S = replay_sensitivity(op, b, inv, k_conv, _u(dtype), 9 * arrays.nc) if sensitivity else np.zeros(k_conv + 1)
    finally:
        lin.close()
    lmin, lmax = lanczos_condition(full["alphas"][:k_conv], full["betas"][:k_conv - 1])
    assert lmin > 0, (lmin, lmax)
    kappa = lmax / lmin
    ks = sorted({k for k in (1, 2, 3) if k < len(xs)} | {k_conv})
    for k in ks:
        bar = max(C_BAR * k * _u(dtype) * kappa, 4 * S[k])
        assert bar <= (BAR_MAX_CONVERGED if k == k_conv else BAR_MAX)[dtype], (k, kappa, bar)
        if dtype == np.float64 and k <= 3 and k < k_conv:
            assert rel_err(xs[k], xs[k - 1]) > 100 * bar, k
        inc, term, it, b_k, inv_k = _truncated(arrays, dtype, env, LAM_PCG, handle, eta=NEVER, max_linear_solver_iterations=k)
        assert np.array_equal(b_k, b) and np.array_equal(inv_k, inv), k
        assert (term, it) == (NO_CONVERGENCE, k), (k, term, it)
        assert rel_err(inc, -expand(xs[k])) < bar, (k, rel_err(inc, -expand(xs[k])), bar)
    return b


def power_edge_sweep(arrays, dtype, env, handle=_handle):
    """POWER_SCHUR_COMPLEMENT truncated at 1, 2, 3 and CONVERGED_POWER terms against power_replay"""
    from test_gpu_pcg_iterates import operator_of
    opt = {"solver_type": "POWER_SCHUR_COMPLEMENT"}
    lin = handle(arrays, dtype, env, power_order=CONVERGED_POWER, eta=0.0, **opt)
    lin.solve(LAM_POWER)
    try:
        b, inv = lin.get_rhs(), lin.get_preconditioner()[0]
        full = power_replay(operator_of(lin, dtype), inv, b, order=CONVERGED_POWER, eta=0.0)
    finally:
        lin.close()
    sums = full["sums"]
    d1, d2 = np.linalg.norm(sums[-1] - sums[-2]), np.linalg.norm(sums[-2] - sums[-3])
    rho = d1 / d2 if d2 > 0 else 0.0
    assert rho < 1, rho
    kappa_b = max(np.linalg.cond(blk[np.ix_(nz, nz)]) for blk in inv.astype(np.float64)
                  for nz in [np.any(blk != 0, axis=1)] if nz.any())
    for k in (1, 2, 3, CONVERGED_POWER):
        bar = C_BAR * k * _u(dtype) * kappa_b * min(k, 1 / (1 - rho))
        assert bar <= (BAR_MAX_CONVERGED if k == CONVERGED_POWER else BAR_MAX)[dtype], (k, kappa_b, rho, bar)
        inc, term, it, b_k, inv_k = _truncated(arrays, dtype, env, LAM_POWER, handle, power_order=k, eta=0.0, **opt)
        assert np.array_equal(b_k, b) and np.array_equal(inv_k, inv), k
        assert (term, it) == (NO_CONVERGENCE, k), (k, term, it)
        assert rel_err(inc, sums[k]) < bar, (k, rel_err(inc, sums[k]), bar)


@pytest.mark.parametrize("c,nc,dtype", _vec_params())
def test_pcg_iterates_at_camera_count_edges(c, nc, dtype):
    """PCG truncated at 1, 2, 3 iterations and at convergence against pcg_replay on the handle's own b, M^-1 and operator"""
    arrays, env = _vec_setup(c, nc, dtype)
    b = pcg_edge_sweep(arrays, dtype, env)
    if (c, nc) in UNOBSERVED_LAST:
        assert np.all(b[-9:] == 0)


@pytest.mark.parametrize("c,nc,dtype", _vec_params())
def test_power_series_at_camera_count_edges(c, nc, dtype):
    """POWER_SCHUR_COMPLEMENT truncated at 1, 2, 3 and CONVERGED_POWER terms against power_replay"""
    arrays, env = _vec_setup(c, nc, dtype)
    power_edge_sweep(arrays, dtype, env)
