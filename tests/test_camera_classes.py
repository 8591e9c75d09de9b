"""CPU side of tests/test_gpu_camera_classes.py: the degree-case builder produces exactly the requested camera degrees and
a layout rba_layout_selftest accepts, and the per-camera checkers accept the oracle's own float32 and float64 output and
reject planted faults of the camera reductions, built from that output:
  dropped / doubled     one csr_y segment (SEG_LEN y slots) of H x, one pb item (PB_SEG_LEN observations) of the blocks
  neighbour             one camera's 9-vector (its 9 x 9 block) written to the next camera
  CTA tail              the last camera of a k_pcg_vec CTA range zeroed, for every cluster size
  chunk segment         a csr_y segment made of the extra row-chunk slots of chunked tracks dropped
Every fault is rejected at every degree case where it applies, in float64 and float32, except in float32 a short last
csr_y segment of the busiest camera with chunked tracks (_below_f32_bar).
"""
import ctypes as C

import numpy as np
import pytest

from test_gpu_camera_classes import (BUSY, CLUSTERS, HUB_DEGREES, LAM, SEG_LEN, TRACK_NS, WARPS_PER_SM, bar_constants,
                                     camera_layout, check_per_camera, degree_problem, excess_per_camera, panel_sums,
                                     pb_items_of, restage_problem, vec_partition, vec_problem, y_segments_of, VEC_CASES,
                                     UNOBSERVED_LAST)
from test_gpu_kernel_classes import row_chunks

H100_SMS = 132


def _selftest(a):
    from rootba_b200 import _lib
    L = _lib.lib()
    off = np.ascontiguousarray(a.lm_off, np.int64)
    oc = np.ascontiguousarray(a.obs_cam, np.int32)
    xy = np.ascontiguousarray(a.obs_xy, np.float64)
    pv = _lib.ProblemView(a.nc, a.nl, a.nobs, off.ctypes.data, oc.ctypes.data, xy.ctypes.data)
    for ssz in (4, 8):
        assert L.rba_layout_selftest(C.byref(pv), 0, 1, ssz) == 0, (ssz, L.rba_last_error())


@pytest.mark.parametrize("n", TRACK_NS)
def test_degree_problem(n):
    a = degree_problem(n)
    assert np.all(a.track_lengths() == n)
    lay = camera_layout(a)
    assert list(lay["m"][:len(HUB_DEGREES)]) == list(HUB_DEGREES)
    assert np.all(lay["m"][len(HUB_DEGREES):] > 0)
    assert np.array_equal(lay["my"], lay["m"] * row_chunks(n))
    # a hub's landmarks are spread over the problem, not one run of tiles
    busy = np.nonzero(a.obs_cam == HUB_DEGREES.index(BUSY))[0]
    lms = np.searchsorted(a.lm_off, busy, side="right") - 1
    assert lms.min() < a.nl // 10 and lms.max() > a.nl - a.nl // 10
    _selftest(a)


def test_vector_and_restage_problems():
    for c, nc in VEC_CASES:
        a = vec_problem(nc, (c, nc) in UNOBSERVED_LAST)
        m = np.bincount(a.obs_cam, minlength=nc)
        assert a.nc == nc and np.all(m[:-1] > 0) and (m[-1] == 0) == ((c, nc) in UNOBSERVED_LAST)
        if (c, nc) in UNOBSERVED_LAST:
            lo, hi = vec_partition(nc, c)["last_range"]
            assert lo <= nc - 1 < hi
        _selftest(a)
    a = restage_problem(H100_SMS)
    lay = camera_layout(a)
    assert np.all(lay["m"] == 1) and lay["obs_segments"].sum() > H100_SMS * WARPS_PER_SM
    assert not vec_partition(a.nc, 16)["cached"]
    _selftest(a)


# ---- planted faults on the oracle's output ----
FAULT_NS = (2, 25, 40)


def _oracle_case(n, dtype):
    from oracle import oracle_py as orc
    a = degree_problem(n)
    o = orc.Oracle(a, dtype, orc.default_options(num_threads=0))
    assert o.linearize()
    lam = float(dtype(LAM))
    b, B = o.stage2(LAM)
    o.set_pose_damping(LAM)
    x = np.random.default_rng(3).uniform(-1, 1, 9 * a.nc).astype(dtype)
    y = o.right_multiply(x).astype(np.float64).reshape(a.nc, 9)
    ps = panel_sums(a, o.get_block, lam, x, record=range(len(HUB_DEGREES)))
    ref = ps.result()
    got = {"b": b.astype(np.float64).reshape(a.nc, 9), "B": B.astype(np.float64) + lam * np.eye(9), "y": y}
    return a, ps, ref, got


@pytest.fixture(scope="module", params=[(n, d) for n in FAULT_NS for d in (np.float32, np.float64)],
                ids=lambda p: f"n{p[0]}-{np.dtype(p[1]).name}")
def oracle_case(request):
    n, dtype = request.param
    return (n, dtype) + _oracle_case(n, dtype)


def _u(dtype):
    return float(np.finfo(dtype).eps) / 2


def _rejected(got, want, mag, c, u, cam):
    return excess_per_camera(got, want, mag, c, u)[cam] > 1


def _below_f32_bar(dtype, seg_len, y_slots):
    """float32 H x of a camera with thousands of y slots: the bar grows with the y slots (gamma_k of a sum of Σ |terms|),
    while a short last segment of random-sign terms (8 and 12 of the BUSY camera's 5000 and 7500 y slots at n = 25, 40)
    changes the sum by less (0.3 and 0.4 of the bar; a full segment of 96 is 1.5 .. 2.7 bars)"""
    return dtype == np.float32 and seg_len < SEG_LEN // 4 and y_slots >= 40 * SEG_LEN


def ps_y_slots(ps, cam):
    return len(ps.yslots[cam])


def test_checkers_accept_the_oracle(oracle_case):
    n, dtype, a, ps, ref, got = oracle_case
    cb, cy = bar_constants(a)
    u = _u(dtype)
    check_per_camera(got["b"], ref["b"], ref["Mb"], cb, u, "b")
    check_per_camera(got["B"], ref["B"], ref["MB"], cb, u, "blocks")
    check_per_camera(got["y"], ref["y"], ref["My"], cy, u, "H x")


def test_dropped_or_doubled_segment_is_rejected(oracle_case):
    n, dtype, a, ps, ref, got = oracle_case
    cb, cy = bar_constants(a)
    u = _u(dtype)
    tried = 0
    for h, d in enumerate(HUB_DEGREES):
        segs = y_segments_of(ps, h, n)
        items = pb_items_of(ps, h)
        if len(segs) > 1:
            for s in (segs[0], segs[-1]):
                if _below_f32_bar(dtype, len(s), ps_y_slots(ps, h)):
                    continue
                dy = sum(e[2] for e in s)
                for sign in (-1, 1):
                    y = got["y"].copy()
                    y[h] += sign * dy
                    assert _rejected(y, ref["y"], ref["My"], cy, u, h), ("H x segment", d, len(s), sign)
                    tried += 1
        if len(items) > 1:
            for it in (items[0], items[-1]):
                dB = sum(e[1] for e in it)
                for sign in (-1, 1):
                    B = got["B"].copy()
                    B[h] += sign * dB
                    assert _rejected(B, ref["B"], ref["MB"], cb, u, h), ("blocks item", d, len(it), sign)
                    tried += 1
    assert tried >= 4 * 10


def test_neighbour_write_is_rejected(oracle_case):
    n, dtype, a, ps, ref, got = oracle_case
    cb, cy = bar_constants(a)
    u = _u(dtype)
    for h, d in enumerate(HUB_DEGREES):
        y, B = got["y"].copy(), got["B"].copy()
        y[h + 1], B[h + 1] = y[h], B[h]
        assert _rejected(y, ref["y"], ref["My"], cy, u, h + 1), ("H x", d)
        assert _rejected(B, ref["B"], ref["MB"], cb, u, h + 1), ("blocks", d)


def test_zeroed_cta_tail_is_rejected(oracle_case):
    n, dtype, a, ps, ref, got = oracle_case
    _, cy = bar_constants(a)
    u = _u(dtype)
    for c in CLUSTERS:
        p = vec_partition(a.nc, c)
        for b in range(c):
            last = min(a.nc, (b + 1) * p["per_cta"]) - 1
            if last < b * p["per_cta"]:
                continue
            y = got["y"].copy()
            y[last] = 0
            assert _rejected(y, ref["y"], ref["My"], cy, u, last), (c, b, last)


def test_dropped_chunk_segment_is_rejected(oracle_case):
    n, dtype, a, ps, ref, got = oracle_case
    if row_chunks(n) == 1:
        pytest.skip("no row chunks at this track length")
    _, cy = bar_constants(a)
    u = _u(dtype)
    tried = 0
    for h, d in enumerate(HUB_DEGREES):
        for s in y_segments_of(ps, h, n):
            if all(e[1] > 0 for e in s) and not _below_f32_bar(dtype, len(s), ps_y_slots(ps, h)):
                y = got["y"].copy()
                y[h] -= sum(e[2] for e in s)
                assert _rejected(y, ref["y"], ref["My"], cy, u, h), (d, len(s))
                tried += 1
    assert tried >= 5
