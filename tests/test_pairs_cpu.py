"""The camera-pair structure behind the assembled operator and rba_compute_covariance on the CPU (rba::build_pair_list,
rba::plan_assembled and rba::pack_asm_term in rootba_b200/csrc/layout.hpp, driven by tests/cpp/pairs_cpu.cpp), against
numpy restatements:
  * the pair list is the landmark-major term enumeration sorted stably by ca * nc + cb, and wpos maps it back;
  * the block-row CSR of S holds every pair's lower and upper block exactly once, columns ascending;
  * every packed AsmTerm decodes (the bit layout k_rcs_terms reads) to its landmark's tile, and to the panel address of
    every column in every row that rba_debug_get_block uses;
  * the size rules (all terms staged in one pass of at most 2 GB, S at most a quarter of the panels) accept exactly what
    the earlier landmark-range staging accepted;
  * the break-even switch iteration on the bench.py stand-ins of Ladybug-1723 (float32) and Trafalgar-257 (float64).
The fixed summation orders of S and of the covariance's reduced camera matrix rest on the first point."""
import math
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from rootba_b200.synthetic import synth_bal, synth_config

STAGE_BYTES = 2 << 30  # staging bound of the assembled operator (layout.hpp ASM_STAGE_BYTES)


@pytest.fixture(scope="module")
def pairs():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "cpp"), "-s", "_build/pairs_cpu"])
    exe = os.path.join(ROOT, "tests", "cpp", "_build", "pairs_cpu")

    def run(mode, arrays, rank=0, nranks=1, s=4):
        inp = "\n".join([mode, f"{arrays.nc} {arrays.nl} {rank} {nranks} {s}", " ".join(map(str, arrays.lm_off)),
                         " ".join(map(str, arrays.obs_cam)), ""])
        out = subprocess.run([exe], input=inp, capture_output=True, text=True, check=True).stdout
        return {ln.split()[0]: np.array(ln.split()[1:], dtype=np.int64) for ln in out.splitlines()}

    def pack(rows):
        inp = f"pack\n{len(rows)}\n" + "".join(" ".join(map(str, r)) + "\n" for r in rows)
        out = subprocess.run([exe], input=inp, capture_output=True, text=True, check=True).stdout
        return np.array(out.split(), dtype=np.int64).reshape(-1, 3)
    run.pack = pack
    return run


# ---- restatements ----
def group_size(n):
    return 1 if n <= 2 else 2 if n <= 4 else 4 if n <= 8 else 8 if n <= 16 else 16 if n <= 32 else 32


def kp_for(n, G):
    kp = (9 * n + 2 * G - 1) // (2 * G)
    return (kp + 1) & ~1 if kp > 9 else kp


def lm_major(arrays, lo, hi):
    """landmark-major terms of landmarks lo..hi-1 (landmarks in problem order, then a = 0..n-1, b = 0..a): the local
    landmark and the two observation indices of every term"""
    n = np.diff(arrays.lm_off)[lo:hi]
    cnt = n * (n + 1) // 2
    lm = np.repeat(np.arange(hi - lo), cnt)
    k = np.arange(int(cnt.sum())) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    a = ((np.sqrt(8.0 * k + 1) - 1) // 2).astype(np.int64)
    a += (a + 1) * (a + 2) // 2 <= k
    a -= a * (a + 1) // 2 > k
    b = k - a * (a + 1) // 2
    first = arrays.lm_off[lo + lm]
    return lm, first + a, first + b, a, b


def sorted_key(arrays, oa, ob):
    return arrays.obs_cam[oa].astype(np.int64) * arrays.nc + arrays.obs_cam[ob]


def panel_scalars(arrays, lo, hi):
    n, c = np.unique(np.diff(arrays.lm_off)[lo:hi], return_counts=True)
    total = 0
    for ni, ci in zip(n.tolist(), c.tolist()):
        G = group_size(ni)
        total += -(-ci // (32 // G)) * 2 * ni * kp_for(ni, G) * 64
    return total


def old_fits(arrays, lo, hi, s, nnzb):
    """the earlier rule: landmark ranges of at most 2 GB of staged terms (one landmark's terms if more), taken only when
    there is a single range, and S at most a quarter of the panels"""
    cap = max(1, STAGE_BYTES // (81 * s))
    ranges, w = [0], 0
    for n in np.diff(arrays.lm_off)[lo:hi].tolist():
        k = n * (n + 1) // 2
        if w + k - ranges[-1] > cap and w > ranges[-1]:
            ranges.append(w)
        w += k
    ranges.append(w)
    return len(ranges) <= 2 and 4 * nnzb * 81 * s <= panel_scalars(arrays, lo, hi) * s, len(ranges) - 1


def switch_iteration(nt, panel, s_bytes, s):
    staged, saved = 4.0 * nt * 81 * s, panel * s - s_bytes
    return 1 + math.ceil(2.0 * staged / max(saved, 1.0))


def nnzb_of(arrays, oa, ob):
    keys = np.unique(sorted_key(arrays, oa, ob))
    return 2 * keys.size - int(np.count_nonzero(keys // arrays.nc == keys % arrays.nc))


# ---- problems ----
CLASS_N = [2, 3, 4, 5, 8, 9, 16, 17, 24, 25, 32, 33, 40, 64]  # every group size, row-chunked tracks from n = 25


def classes():
    """every track-length class, some tiles full and some ragged, landmarks of different classes interleaved"""
    rng = np.random.default_rng(4)
    n = np.repeat(CLASS_N, 5 * np.array([37, 20, 9, 11, 5, 3, 6, 2, 2, 3, 1, 2, 1, 2]))  # enough that S is < 1/4 of the panels
    return synth_bal(66, n.size, 4.0, seed=8, track_lengths=rng.permutation(n), lm_spread=0.5)


def unobserved():
    """cameras 3, 7 and 11..13 have no observations"""
    rng = np.random.default_rng(5)
    cams = np.setdiff1d(np.arange(11), [3, 7])
    tracks = [rng.choice(cams, size=int(k), replace=False) for k in rng.integers(2, 9, 60)]
    return synth_bal(14, 60, 4.0, seed=6, tracks=tracks, lm_spread=0.5)


def lone_first(n0, nc, nsmall=40, nsmall_n=3):
    """landmark 0 with a track of n0, then short tracks: with two ranks, rank 0's shard is landmark 0 alone"""
    return synth_bal(nc, 1 + nsmall, 4.0, seed=9, track_lengths=[n0] + [nsmall_n] * nsmall, lm_spread=0.2)


PROBLEMS = {"classes": classes, "unobserved": unobserved, "lone": lambda: lone_first(30, 40)}
_cache = {}


def problem(name):
    if name not in _cache:
        _cache[name] = PROBLEMS[name]()
    return _cache[name]


SHARDS = [("classes", 0, 1), ("classes", 0, 2), ("classes", 1, 2), ("classes", 0, 3), ("classes", 1, 3), ("classes", 2, 3),
          ("unobserved", 0, 1), ("unobserved", 1, 2), ("lone", 0, 2), ("lone", 1, 2)]


@pytest.mark.parametrize("name,rank,nranks", SHARDS)
@pytest.mark.parametrize("s", [4, 8])
def test_pair_list_csr_and_terms(pairs, name, rank, nranks, s):
    arrays = problem(name)
    out = pairs("full", arrays, rank, nranks, s)
    lo, hi = out["lm_range"].tolist()
    if name == "lone" and rank == 0:
        assert (lo, hi) == (0, 1)
    nc = arrays.nc
    lm, oa, ob, a, b = lm_major(arrays, lo, hi)
    nt = lm.size
    assert out["nt"][0] == nt
    slot_obs = out["slot_obs"]
    # order: the landmark-major enumeration sorted stably by ca * nc + cb
    terms = out["terms"].reshape(-1, 2)
    order = np.argsort(sorted_key(arrays, oa, ob), kind="stable")
    assert np.array_equal(slot_obs[terms[:, 0]], oa[order]) and np.array_equal(slot_obs[terms[:, 1]], ob[order])
    # wpos: a permutation, and terms[t] is landmark-major term wpos[t]
    wpos = out["wpos"]
    assert np.array_equal(np.sort(wpos), np.arange(nt))
    assert np.array_equal(slot_obs[terms[:, 0]], oa[wpos]) and np.array_equal(slot_obs[terms[:, 1]], ob[wpos])
    # per landmark its first slot and track length
    n_local = np.diff(arrays.lm_off)[lo:hi]
    assert np.array_equal(out["nn"], n_local)
    assert np.array_equal(slot_obs[out["slot0"]], arrays.lm_off[lo:hi])
    # pairs: the distinct (ca, cb) in order, blk_ptr their term ranges
    ca, cb = arrays.obs_cam[oa[order]], arrays.obs_cam[ob[order]]
    assert np.all(ca >= cb)
    blk_cam, blk_ptr = out["blk_cam"].reshape(-1, 2), out["blk_ptr"]
    nblk = blk_cam.shape[0]
    assert out["nblk"][0] == nblk and blk_ptr[0] == 0 and blk_ptr[-1] == nt and np.all(np.diff(blk_ptr) > 0)
    key = blk_cam[:, 0] * nc + blk_cam[:, 1]
    assert np.all(np.diff(key) > 0)
    assert np.array_equal(np.repeat(blk_cam[:, 0], np.diff(blk_ptr)), ca)
    assert np.array_equal(np.repeat(blk_cam[:, 1], np.diff(blk_ptr)), cb)
    # CSR of the full S
    nnzb = out["nnzb"][0]
    ndiag = int(np.count_nonzero(blk_cam[:, 0] == blk_cam[:, 1]))
    assert nnzb == 2 * nblk - ndiag == nnzb_of(arrays, oa, ob)
    assert out["s_bytes"][0] == nnzb * 81 * s
    assert out["panel_scalars"][0] == panel_scalars(arrays, lo, hi)
    assert out["switch"][0] == switch_iteration(nt, panel_scalars(arrays, lo, hi), nnzb * 81 * s, s)
    # the CSR and the AsmTerms exist when the size rules pass; they do for every one-rank problem here (the assembled
    # operator runs on one GPU), and never for a shard of one landmark (S is ~4.5 times its panel)
    if nranks == 1:
        assert out["fits"][0] == 1
    if name == "lone" and rank == 0:
        assert out["fits"][0] == 0
    if not out["fits"][0]:
        assert all(out[k].size == 0 for k in ("row_ptr", "col", "pos", "asm_base", "asm_ij", "asm_meta"))
        return
    row_ptr, col, pos = out["row_ptr"], out["col"], out["pos"].reshape(-1, 2)
    assert row_ptr.size == nc + 1 and row_ptr[0] == 0 and row_ptr[-1] == nnzb and col.size == nnzb
    for r in range(nc):
        assert np.all(np.diff(col[row_ptr[r]:row_ptr[r + 1]]) > 0)
    row_of = np.repeat(np.arange(nc), np.diff(row_ptr))
    assert np.array_equal(row_of[pos[:, 0]], blk_cam[:, 0]) and np.array_equal(col[pos[:, 0]], blk_cam[:, 1])
    diag = blk_cam[:, 0] == blk_cam[:, 1]
    assert np.all(pos[diag, 1] == -1) and np.all(pos[~diag, 1] >= 0)
    up = pos[~diag, 1]
    assert np.array_equal(row_of[up], blk_cam[~diag, 1]) and np.array_equal(col[up], blk_cam[~diag, 0])
    assert np.array_equal(np.sort(np.concatenate([pos[:, 0], up])), np.arange(nnzb))  # every block exactly once
    # AsmTerm, landmark-major: decoded as k_rcs_terms decodes it
    base, ij, meta = out["asm_base"], out["asm_ij"], out["asm_meta"]
    assert base.size == nt
    n_dec, lg, KP = meta & 0x7FFF, (meta >> 15) & 7, meta >> 18
    G = 1 << lg
    ia, ib = ij & 0xFFFF, ij >> 16
    n_of = n_local[lm]
    G_ref = np.array([group_size(int(v)) for v in n_local])[lm]
    KP_ref = np.array([kp_for(int(v), group_size(int(v))) for v in n_local])[lm]
    assert np.array_equal(n_dec, n_of) and np.array_equal(G, G_ref) and np.array_equal(KP, KP_ref)
    assert np.array_equal(G, out["lm_G"][lm]) and np.array_equal(KP, out["lm_KP"][lm]) and np.array_equal(n_dec, out["lm_n"][lm])
    assert np.array_equal(ia, a) and np.array_equal(ib, b)
    # every column of both slots in every panel row: the address k_rcs_terms reads against rba_debug_get_block's
    tile_off, g = out["lm_panel_off"][lm], out["lm_g"][lm]
    G_t, KP_t = out["lm_G"][lm], out["lm_KP"][lm]

    def debug_addr(r, c):  # rba_debug_get_block: panel[T.panel_off + (((r KP + k) 32 + lane) 2 + v)]
        pr, v = c // 2, c % 2
        lane = g[:, None] * G_t[:, None] + pr % G_t[:, None]
        return tile_off[:, None] + ((r * KP_t[:, None] + pr // G_t[:, None]) * 32 + lane) * 2 + v

    p = np.arange(9)
    col_a = 9 * ia[:, None] + p  # slot a: one scalar per lane
    pa = col_a >> 1
    off_a = 2 * ((pa >> lg[:, None]) * 32 + (pa & (G[:, None] - 1))) + (col_a & 1)
    cb0 = 9 * ib
    odd = (cb0 & 1)[:, None]
    kk, v = (p + odd) // 2, (p + odd) % 2  # slot b: element q of five two-scalar loads
    pb = (cb0 >> 1)[:, None] + kk
    off_b = 2 * ((pb >> lg[:, None]) * 32 + (pb & (G[:, None] - 1))) + v
    for r in range(int(n_local.max()) * 2):
        live = 2 * n_of > r
        rr = base + r * KP * 64
        assert np.array_equal((rr[:, None] + off_a)[live], debug_addr(r, col_a)[live])
        assert np.array_equal((rr[:, None] + off_b)[live], debug_addr(r, 9 * ib[:, None] + p)[live])


def test_asm_term_packing_limits(pairs):
    """the widest fields a problem can have (track length 20000, G = 32) survive the packing"""
    n = 20000
    KP = kp_for(n, 32)
    rows = [(1 << 40, 19999, 19999, n, 32, KP), (0, 0, 19999, n, 32, KP), (123456789012, 19999, 0, n, 32, KP),
            (7, 1, 0, 2, 1, kp_for(2, 1)), (9, 12, 5, 16, 8, kp_for(16, 8))]
    got = pairs.pack(rows)
    for (base, ia, ib, nn, G, kp), (b2, ij, meta) in zip(rows, got.tolist()):
        assert 0 <= ij < 2**31 and 0 <= meta < 2**31
        assert b2 == base and ij & 0xFFFF == ia and ij >> 16 == ib
        assert meta & 0x7FFF == nn and 1 << ((meta >> 15) & 7) == G and meta >> 18 == kp


def _tracks_of_90(nl, s):
    return lambda: synth_bal(100, nl, 4.0, seed=12 if s == 8 else 13, track_lengths=[90] * nl, lm_spread=0.5)


CAP64 = STAGE_BYTES // (81 * 8) // (90 * 91 // 2)  # landmarks of track length 90 whose float64 terms fit in one pass
# (id, problem, rank, nranks, scalar size, terms over 2 GB, shard of one landmark)
QUALIFICATION = [("f64-just-fits", _tracks_of_90(CAP64, 8), 0, 1, 8, False, False),
                 ("f64-over-2GB", _tracks_of_90(CAP64 + 1, 8), 0, 1, 8, True, False),
                 ("f32-over-2GB", _tracks_of_90(1700, 4), 0, 1, 4, True, False),
                 ("f64-lone-landmark-over-2GB", lambda: lone_first(2600, 2600, 10, 2), 0, 2, 8, True, True),
                 ("f32-lone-landmark-over-2GB", lambda: lone_first(3700, 3700, 10, 2), 0, 2, 4, True, True)]


@pytest.mark.parametrize("case", QUALIFICATION, ids=lambda c: c[0])
def test_one_pass_staging_rule_matches_range_rule(pairs, case):
    _, make, rank, nranks, s, over, lone = case
    arrays = make()
    out = pairs("summary", arrays, rank, nranks, s)
    lo, hi = out["lm_range"].tolist()
    lm, oa, ob, _, _ = lm_major(arrays, lo, hi)
    nnzb = nnzb_of(arrays, oa, ob)
    assert out["nt"][0] == lm.size and out["nnzb"][0] == nnzb
    assert (81 * lm.size * s > STAGE_BYTES) == over
    want, nranges = old_fits(arrays, lo, hi, s, nnzb)
    assert out["fits"][0] == want
    if lone:
        assert hi - lo == 1 and nranges == 1 and not want  # one range, refused by the quarter rule
    else:
        assert nranges == (2 if over else 1) and want == (not over)


# bench.py's stand-ins (make_problem: synth_config(workload, seed=38401, scale=1.0)) and the switch iteration the solver
# uses on them
@pytest.mark.parametrize("workload,s,switch", [("ladybug-1723", 4, 24), ("trafalgar-257", 8, 26)])
def test_switch_iteration_on_bench_workloads(pairs, workload, s, switch):
    arrays = synth_config(workload, seed=38401, scale=1.0)
    out = pairs("summary", arrays, 0, 1, s)
    lm, oa, ob, _, _ = lm_major(arrays, 0, arrays.nl)
    nnzb = nnzb_of(arrays, oa, ob)
    assert out["nt"][0] == lm.size and out["nnzb"][0] == nnzb and out["fits"][0] == 1
    assert out["switch"][0] == switch_iteration(lm.size, panel_scalars(arrays, 0, arrays.nl), nnzb * 81 * s, s) == switch
