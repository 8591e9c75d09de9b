"""CPU tests of the float64 model of the covariance blocks (covariance_blocks_model, DESIGN.md section 20): the four formulas
against the blocks of inv(J^T J) of the dense total system (with camera and landmark priors, and with a rank-deficient landmark
eliminated by the pseudo-inverse), the relative-pose Jacobian against central differences of the pair-prior residual, the
halving identity, the planted faults the device check must reject, and the C ABI of rba_compute_covariance_blocks."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import camera_model as cm
import camera_prior_model as pm
import covariance_blocks_model as cbm
import covariance_model as cvm
import pair_prior_model as qm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _instance(nc, nl, seed, lm_priors=False, rank2=False):
    """a synthetic problem with centre priors on every camera: (prob, jp, jl, prior rows [9 nc, 9 nc], landmark priors
    (L^T L, L) or None, the index of a landmark left with one observation or None).  rank2: the rows of all but the first
    observation of landmark 3 are zero, as the device makes those of dropped observations."""
    from rootba_b200.synthetic import synth_bal
    rng = np.random.default_rng(seed)
    tracks = [rng.choice(nc, int(rng.integers(2, 6)), replace=False) for _ in range(nl)]
    prob = synth_bal(nc, nl, 0.0, seed=seed, tracks=tracks, lm_spread=0.5)
    jp, jl, _, _ = cm.weighted(prob)
    if rank2:
        jp[prob.lm_off[3] + 1:prob.lm_off[4]] = 0.0
        jl[prob.lm_off[3] + 1:prob.lm_off[4]] = 0.0
    mean, L = cvm.centre_priors(prob, seed + 1)
    A, _ = pm.rows(np.asarray(prob.cams, np.float64), mean, L)
    Jc = np.zeros((9 * nc, 9 * nc))
    for c in range(nc):
        Jc[9 * c:9 * c + 9, 9 * c:9 * c + 9] = A[c]
    lm_info = None
    if lm_priors:
        Ll = np.zeros((nl, 3, 3))
        for l in range(0, nl, 3):
            Ll[l] = np.eye(3) + 0.3 * rng.standard_normal((3, 3))
        lm_info = np.einsum("lki,lkj->lij", Ll, Ll)
        lm_info = (lm_info, Ll)
    return prob, jp, jl, Jc, lm_info, (3 if rank2 else None)


def _dense_cov(prob, jp, jl, Jc, lm_info, reduce_lm=None):
    """the full covariance of the dense total system; reduce_lm: that landmark's columns are restricted to the range of its
    Hll (the pseudo-inverse elimination: its null direction is not a parameter)"""
    nc, nl = len(prob.cams), len(prob.lm_off) - 1
    Jp, Jl = cbm.dense_rows(jp, jl, np.asarray(prob.obs_cam), np.asarray(prob.lm_off), nc)
    Jp = np.vstack([Jp, Jc])
    Jl = np.vstack([Jl, np.zeros((len(Jc), 3 * nl))])
    if lm_info is not None:
        R = np.zeros((3 * nl, 3 * nl))
        for l in range(nl):
            R[3 * l:3 * l + 3, 3 * l:3 * l + 3] = lm_info[1][l]
        Jp, Jl = np.vstack([Jp, np.zeros((3 * nl, 9 * nc))]), np.vstack([Jl, R])
    if reduce_lm is None:
        J = np.hstack([Jp, Jl])
        return np.linalg.inv(J.T @ J)
    cols = slice(3 * reduce_lm, 3 * reduce_lm + 3)
    lam, V = np.linalg.eigh(Jl[:, cols].T @ Jl[:, cols])
    keep = lam > cvm.EIG_DROP * lam.max()
    Jr = np.hstack([Jl[:, :3 * reduce_lm], Jl[:, cols] @ V[:, keep], Jl[:, 3 * reduce_lm + 3:]])
    J = np.hstack([Jp, Jr])
    Cr = np.linalg.inv(J.T @ J)
    # back to 3 entries per landmark: the reduced landmark's block is embedded with V+ (its true covariance is unbounded)
    E = np.zeros((J.shape[1], 9 * nc + 3 * nl))
    E[:9 * nc + 3 * reduce_lm, :9 * nc + 3 * reduce_lm] = np.eye(9 * nc + 3 * reduce_lm)
    r0 = 9 * nc + 3 * reduce_lm
    E[r0:r0 + keep.sum(), r0:r0 + 3] = V[:, keep].T
    E[r0 + keep.sum():, r0 + 3:] = np.eye(J.shape[1] - r0 - keep.sum())
    return E.T @ Cr @ E


def _requests(nc, nl, rng, m=40, bad=None):
    req = cbm.random_requests(rng, nc, nl, m)
    req["cameras"][:3] = [[0, 0], [1, 2], [2, 1]]
    req["landmarks"][:3] = [[0, 0], [1, 2], [2, 1]]
    if bad is not None:  # every kind involves the rank-deficient landmark at least once
        req["camera_landmark"][3] = [1, bad]
        req["landmarks"][3] = [bad, 0]
        req["landmarks"][4] = [bad, bad]
    return req


@pytest.mark.parametrize("lm_priors", [False, True], ids=["no_lm_priors", "lm_priors"])
@pytest.mark.parametrize("seed", [1, 2])
def test_formulas_equal_blocks_of_the_dense_inverse(seed, lm_priors):
    nc, nl = 6, 40
    prob, jp, jl, Jc, lm_info, _ = _instance(nc, nl, seed, lm_priors)
    ref = cbm.reference(jp, jl, prob.obs_cam, prob.lm_off, prob.cams, Jc.T @ Jc, None if lm_info is None else lm_info[0])
    req = _requests(nc, nl, np.random.default_rng(seed))
    got = cbm.blocks(ref, **req)
    want = cbm.dense_blocks(_dense_cov(prob, jp, jl, Jc, lm_info), nc, np.asarray(prob.cams, np.float64), **req)
    for key in cbm.KINDS:
        scale = np.abs(want[key]).max()
        assert np.abs(got[key] - want[key]).max() <= 1e-9 * scale, key
    # requests (0, 0) and (1, 2), (2, 1) of each pair kind: the marginal and the transpose
    assert np.array_equal(got["cameras"][0], ref["Sig"][:9, :9])
    for key in ("cameras", "landmarks"):
        assert np.abs(got[key][1] - got[key][2].T).max() <= 1e-9 * np.abs(got[key][1]).max()


def test_rank_deficient_landmark_is_nan_and_the_rest_exact():
    nc, nl = 6, 40
    prob, jp, jl, Jc, _, bad = _instance(nc, nl, 5, rank2=True)
    ref = cbm.reference(jp, jl, prob.obs_cam, prob.lm_off, prob.cams, Jc.T @ Jc)
    assert ref["rank"][bad] == 2 and (np.delete(ref["rank"], bad) == 3).all()
    req = _requests(nc, nl, np.random.default_rng(5), bad=bad)
    assert (np.asarray(req["camera_landmark"])[:, 1] == bad).any() and (np.asarray(req["landmarks"]) == bad).sum() >= 3
    got = cbm.blocks(ref, **req)
    want = cbm.dense_blocks(_dense_cov(prob, jp, jl, Jc, None, reduce_lm=bad), nc, np.asarray(prob.cams, np.float64), **req)
    for key in cbm.KINDS:
        r = np.asarray(req[key])
        involved = (r[:, 1] == bad) if key == "camera_landmark" else \
            ((r[:, 0] == bad) | (r[:, 1] == bad)) if key == "landmarks" else np.zeros(len(r), bool)
        assert np.isnan(got[key][involved]).all() and np.isfinite(got[key][~involved]).all(), key
        scale = np.abs(want[key][~involved]).max()
        assert np.abs(got[key][~involved] - want[key][~involved]).max() <= 1e-9 * scale, key


def test_relative_jacobian_matches_central_differences():
    from rootba_b200.synthetic import synth_bal
    cams = np.asarray(synth_bal(5, 20, 3.6, seed=9).cams, np.float64)
    h = 1e-6
    for i, j in [(0, 1), (3, 2), (4, 0)]:
        mean = qm.mean_at(cams, [(i, j)])[0]
        assert np.abs(qm.residual(cams[i], cams[j], mean)).max() < 1e-12  # the mean is the current relative pose
        num = np.zeros((6, 12))
        for side, c in enumerate((i, j)):
            for k in range(6):
                d = np.zeros(9)
                d[k] = h
                cp, cm_ = cams.copy(), cams.copy()
                cp[c], cm_[c] = pm.apply_inc(cams[c], d), pm.apply_inc(cams[c], -d)
                num[:, 6 * side + k] = (qm.residual(cp[i], cp[j], mean) - qm.residual(cm_[i], cm_[j], mean)) / (2 * h)
        A = cbm.relative_jacobian(cams[i], cams[j], device_rot=False)
        assert np.abs(A - num).max() <= 1e-7 * np.abs(A).max()


def test_halving_identity():
    """a pair prior with its mean at the current relative pose and L^T L = Sigma_rel^-1 halves Sigma_rel (Woodbury:
    Sigma_rel - Sigma_rel (Sigma_rel + Sigma_rel)^-1 Sigma_rel)"""
    nc, nl = 6, 40
    prob, jp, jl, Jc, _, _ = _instance(nc, nl, 7)
    cams = np.asarray(prob.cams, np.float64)
    pairs = np.array([[1, 4]])
    before = cbm.dense_blocks(_dense_cov(prob, jp, jl, Jc, None), nc, cams, relative=pairs)["relative"][0]
    L = np.linalg.cholesky(np.linalg.inv(before)).T
    Jq, r = qm.rows(cams, pairs, qm.mean_at(cams, pairs), L[None])
    assert np.abs(r).max() < 1e-9
    after = cbm.dense_blocks(_dense_cov(prob, jp, jl, np.vstack([Jc, Jq]), None), nc, cams, relative=pairs)["relative"][0]
    assert np.abs(after - before / 2).max() <= 1e-9 * np.abs(before).max()


@pytest.mark.parametrize("fault", cbm.BASE_FAULTS)
def test_planted_faults_are_rejected(fault):
    nc, nl = 6, 40
    prob, jp, jl, Jc, _, _ = _instance(nc, nl, 11)
    ref = cbm.reference(jp, jl, prob.obs_cam, prob.lm_off, prob.cams, Jc.T @ Jc)
    req = _requests(nc, nl, np.random.default_rng(11))
    good = cbm.blocks(ref, **req)
    ex, _ = cbm.excess(good, good, ref, req)
    assert max(ex.values()) == 0.0
    cbm.check(good, good, ref, req)
    bad = cbm.blocks(ref, **req, fault=fault)
    with pytest.raises(AssertionError):
        cbm.check(bad, good, ref, req, what=fault)


def test_query_struct_matches_the_c_header(tmp_path):
    from rootba_b200 import _lib
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "q.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "rootba_b200.h"\n'
                   'int main(void) { printf("%zu %zu %zu %zu\\n", sizeof(rba_covariance_query), '
                   'offsetof(rba_covariance_query, camera_pairs), offsetof(rba_covariance_query, relative_cov), '
                   'offsetof(rba_covariance_query, lm_cov)); return 0; }\n')
    exe = tmp_path / "q"
    subprocess.check_call([cc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    size, o_pairs, o_rel, o_lm = map(int, subprocess.check_output([str(exe)]).split())
    Q = _lib.CovarianceQuery
    assert size == C.sizeof(Q) == 96
    assert (o_pairs, o_rel, o_lm) == (Q.camera_pairs.offset, Q.relative_cov.offset, Q.lm_cov.offset)


def test_entry_point_is_declared_and_exported():
    from rootba_b200 import _lib
    assert "rba_compute_covariance_blocks" in _lib.declared_symbols()
    assert hasattr(_lib.lib(), "rba_compute_covariance_blocks")
