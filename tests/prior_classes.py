"""Shared by tests/test_prior_classes.py (CPU) and tests/test_gpu_prior_classes.py: the launch geometry of the prior and
intrinsics-group kernels read from the sources, the problems and prior sets that sit on both sides of every boundary of it,
the float64 prior terms of every camera from the models (camera_prior_model, pair_prior_model), a float64 restatement of
the kernels' per-camera loops with planted faults, and the per-camera / per-item checkers.  Not collected by pytest.

Boundaries (rootba_b200/csrc/solver.cu, kernels.cuh, groups.cuh):
  PER_THREAD = 128      k_prior_linearize, k_prior_scale, k_pair_diag2, k_pair_accum: thread per camera; k_pair_linearize,
                        k_pair_scale: thread per pair; <<<ceil(n / 128), 128>>>
  SUM_THREADS = 256     k_prior_cost, k_prior_ldiff: one block strided over the items, then prior_block_sum
  incident sides        k_pair_accum, pair_ov_entry: a loop over the camera's sides (pair_ptr, pair_item / pair_nbr, O)
  GROUP_THREADS = 128   k_group_sum_diag2, k_group_precond, k_group_contract: a strided member loop, then a fixed tree; grid
                        ceil(nc / 128) camera blocks + one block per group
  VEC_THREADS, VEC_EPT  k_pcg_vec<S, true, *> / k_power_vec<S, true>: the cluster partition of test_gpu_camera_classes

Magnitudes.  A prior row is linearised by the kernel and by the model with different formulas (a quaternion logarithm against
scipy's matrix logarithm, a closed-form J_l^-1 against the inverse of J_l), so the two agree to a few u of the row's
magnitude, not of its value.  Every entry of A = L J gets the magnitude |L| |J| (|J| with |R|, |M|, |J_l^-1| and |t_i| +
|M| |t_j| in the cross product), every entry of r = L e the magnitude |L| e_mag, where e_mag is the rounding scale of e:
|R^T| |t| + |c0| for a centre, |t_i| + |M| |t_j| + |t0| for a relative translation, 1 for a logarithm (quaternions of norm
1), |f| + |f0| for an intrinsic.  C_LIN = 32 units of these magnitudes are added to every bar that contains prior rows.
"""
import functools
import os
import re

import numpy as np

import camera_model as cm
import camera_prior_model as pm
import pair_prior_model as qm
from conftest import ROOT
from test_gpu_camera_classes import VEC_EPT, VEC_THREADS, _source_constant

C_LIN = 32
U64 = 2.0 ** -53


def _source(path):
    with open(os.path.join(ROOT, "rootba_b200", "csrc", path)) as f:
        return f.read()


def launch_block(kernel):
    """(rounding, divisor, block) of `kernel<S><<<(n + rounding) / divisor, block, ...` in solver.cu"""
    m = re.search(rf"{kernel}<S><<<\(\w+ \+ (\d+)\) / (\d+), (\d+),", _source("solver.cu"))
    return tuple(int(v) for v in m.groups())


def one_block_threads(kernel):
    """the block size of every one-block launch `kernel<<<1, T, ...` in solver.cu (a set)"""
    return {int(t) for t in re.findall(rf"{kernel}<<<1, (\d+),", _source("solver.cu"))}


PER_THREAD = 128
SUM_THREADS = 256
GROUP_THREADS = _source_constant("groups.cuh", "GROUP_THREADS")
for _k in ("k_prior_linearize", "k_prior_scale", "k_pair_linearize", "k_pair_diag2", "k_pair_scale", "k_pair_accum"):
    assert launch_block(_k) == (PER_THREAD - 1, PER_THREAD, PER_THREAD), _k
assert one_block_threads("k_prior_cost") == {SUM_THREADS} and one_block_threads("k_prior_ldiff") == {SUM_THREADS}
assert "prior_block_sum" in _source("kernels.cuh") and GROUP_THREADS == 128
assert re.search(r"k_group_sum_diag2<S><<<n_groups, GROUP_THREADS,", _source("solver.cu"))
assert re.search(r"k_group_precond<S><<<ncb \+ n_groups, GROUP_THREADS,", _source("solver.cu"))


def blocks_of(n, per=PER_THREAD):
    return -(-n // per)


# ---- prior sets -------------------------------------------------------------------------------------------------------
CAMERA_KINDS = ("dense", "none", "centre", "intrinsics")  # camera c gets CAMERA_KINDS[c % 4]: 127, 255 -> intrinsics, 128,
PAIR_KINDS = ("dense", "translation", "rotation", "none")  # 256 -> dense: the 128-block edges carry a prior on both sides


def camera_prior(cams, seed, scale=1.0, last_dense=True):
    """mixed kinds (dense, none, centre-only, intrinsics-only) in turn, means near the cameras; the last camera dense (it is
    the unobserved one of the vector cases)"""
    rng = np.random.default_rng(seed)
    cams = np.asarray(cams, np.float64)
    nc = len(cams)
    mean = pm.mean_at(cams)
    mean[:, 4:7] += rng.normal(0, 0.05, (nc, 3))
    mean[:, 7] += rng.normal(0, 2.0, nc)
    L = np.stack([pm.sqrt_info_kind(CAMERA_KINDS[c % 4], rng, scale) for c in range(nc)])
    if last_dense:
        L[-1] = pm.sqrt_info_kind("dense", rng, scale)
    return mean, L


def pair_prior(cams, pairs, seed, scale=1.0, kinds=PAIR_KINDS):
    rng = np.random.default_rng(seed)
    pairs = np.asarray(pairs, np.int32).reshape(-1, 2)
    mean = qm.mean_at(cams, pairs)
    mean[:, 4:7] += rng.normal(0, 0.05, (len(pairs), 3))
    L = np.stack([qm.sqrt_info_kind(kinds[p % len(kinds)], rng, scale) for p in range(len(pairs))])
    return pairs, mean, L


def chain_pairs(nc, m=None):
    """(i, i + 1) along the cameras, then (nc - 1, 0), which ties the last camera (unobserved in the vector cases), and
    further (i, i + 2) to make m pairs"""
    pairs = [(i, i + 1) for i in range(nc - 2)] + [(nc - 1, 0)]
    i = 0
    while m is not None and len(pairs) < m:
        pairs.append((i % nc, (i + 2) % nc))
        i += 1
    return np.asarray(pairs[:m] if m is not None else pairs, np.int32)


# the hub case: incident sides per camera 0, 1, 2, 33 and >= 300
HUB_NC = 1900
HUB, HUB_33, HUB_SIDES = 130, 600, 320
HUB_ISOLATED = tuple(range(1000, 1100))


def hub_pairs(nc=HUB_NC, m=3000, seed=9):
    """camera HUB with HUB_SIDES sides, among them a repeated pair, a reversed pair and a pair to the (unobserved) last camera;
    camera HUB_33 with 33; the cameras HUB_ISOLATED with none; the others on a chain (1 or 2 sides) and on random pairs
    until there are m"""
    rng = np.random.default_rng(seed)
    others = np.setdiff1d(np.arange(nc - 1), (HUB, HUB_33) + HUB_ISOLATED)
    pairs = [(HUB, 5), (HUB, 5), (5, HUB), (nc - 1, HUB), (HUB, HUB + 1)]
    nbr = rng.choice(others, HUB_SIDES - len(pairs), replace=False)
    pairs += [(HUB, int(j)) if k % 2 else (int(j), HUB) for k, j in enumerate(nbr)]
    pairs += [(HUB_33, int(j)) for j in rng.choice(others, 33, replace=False)]
    chain = others[:len(others) // 2]
    pairs += [(int(a), int(b)) for a, b in zip(chain[:-1], chain[1:])]
    rest = others[len(others) // 2:]
    while len(pairs) < m:
        a, b = rng.choice(rest, 2, replace=False)
        pairs.append((int(a), int(b)))
    return np.asarray(pairs, np.int32)


def sides(nc, pairs):
    """incident pair sides per camera, the CSR of k_pair_accum: ptr [nc + 1], item (2 p + side) camera-major, ascending p"""
    pairs = np.asarray(pairs).reshape(-1, 2)
    cam = pairs.ravel()
    order = np.argsort(cam, kind="stable")  # item 2 p + s ascending within a camera
    ptr = np.concatenate([[0], np.cumsum(np.bincount(cam, minlength=nc))])
    return ptr, order


def side_counts(nc, pairs):
    return np.bincount(np.asarray(pairs).ravel(), minlength=nc)


# ---- intrinsics groups ------------------------------------------------------------------------------------------------
GROUP_SIZES = (2, 127, 128, 129, 256, 257, 400)


def group_layout(nc=HUB_NC):
    """groups of GROUP_SIZES consecutive cameras, the first of 2 led by camera 127 (the last of the first 128-camera block);
    in the last camera block two groups of 2 interleaved with ungrouped cameras; every other camera ungrouped"""
    g = np.full(nc, -1, np.int32)
    start = 127
    for k, s in enumerate(GROUP_SIZES):
        g[start:start + s] = k
        start += s
    assert start < nc - 16
    g[[nc - 8, nc - 6]] = len(GROUP_SIZES)
    g[[nc - 5, nc - 3]] = len(GROUP_SIZES) + 1
    return g


def vec_groups(nc):
    """the groups of the vector cases: pairs of consecutive cameras in three groups, every fifth camera ungrouped"""
    c = np.arange(nc)
    return np.where(c % 5 == 4, -1, (c // 2) % 3).astype(np.int32)


# ---- the float64 prior terms of every camera ---------------------------------------------------------------------------
class PriorTerms:
    """the unscaled rows of the priors at the cameras `cams`, with magnitudes:
      camera prior c:  A [nc, 9, 9], r [nc, 9], MA, Mr
      pair p = (i, j): Ai, Aj [m, 6, 9], r [m, 6], MAi, MAj, Mr"""

    def __init__(self, cams, camera=None, pairs=None):
        cams = np.asarray(cams, np.float64)
        self.nc = nc = len(cams)
        self.has_camera, self.has_pairs = camera is not None, pairs is not None
        self.cA, self.cr = np.zeros((nc, 9, 9)), np.zeros((nc, 9))
        self.cMA, self.cMr = np.zeros((nc, 9, 9)), np.zeros((nc, 9))
        if camera is not None:
            mean, L = (np.asarray(a, np.float64) for a in camera)
            self.cA, self.cr = pm.rows(cams, mean, L, device_rot=True)
            aL = np.abs(L)
            for c in range(nc):
                J = np.abs(pm.jacobian(cams[c], mean[c], device_rot=True))
                R = np.abs(cm.rotation(cams[c, :4], device=True))
                emag = np.concatenate([R.T @ np.abs(cams[c, 4:7]) + np.abs(mean[c, 4:7]), np.ones(3),
                                       np.abs(cams[c, 7:10]) + np.abs(mean[c, 7:10])])
                self.cMA[c], self.cMr[c] = aL[c] @ J, aL[c] @ emag
        self.pairs = np.zeros((0, 2), np.int32)
        m = 0
        if pairs is not None:
            self.pairs = np.asarray(pairs[0], np.int32).reshape(-1, 2)
            m = len(self.pairs)
        self.m = m
        self.pAi, self.pAj, self.pr = np.zeros((m, 6, 9)), np.zeros((m, 6, 9)), np.zeros((m, 6))
        self.pMAi, self.pMAj, self.pMr = np.zeros((m, 6, 9)), np.zeros((m, 6, 9)), np.zeros((m, 6))
        if pairs is not None:
            mean, L = (np.asarray(a, np.float64) for a in pairs[1:])
            for p, (i, j) in enumerate(self.pairs):
                Ji, Jj = qm.jacobians(cams[i], cams[j], mean[p], device_rot=True)
                e = qm.residual(cams[i], cams[j], mean[p], device_rot=True)
                Lp, aL = L[p], np.abs(L[p])
                self.pAi[p], self.pAj[p], self.pr[p] = Lp @ Ji, Lp @ Jj, Lp @ e
                M = np.abs(qm._rot(cams[i], True) @ qm._rot(cams[j], True).T)
                tmag = np.abs(cams[i, 4:7]) + M @ np.abs(cams[j, 4:7])
                aJi, aJj = np.abs(Ji), np.abs(Jj)
                aJi[0:3, 3:6] = np.abs(cm.hat(tmag))
                self.pMAi[p], self.pMAj[p] = aL @ aJi, aL @ aJj
                self.pMr[p] = aL @ np.concatenate([tmag + np.abs(mean[p, 4:7]), np.ones(3)])

    # -- per-camera quantities, scaled by D [9 nc] (the handle's own scaling) --
    def diag2(self):
        """the squared column norms of the unscaled prior rows per camera [nc, 9] and their magnitude"""
        d = np.einsum("cij,cij->cj", self.cA, self.cA)
        M = np.einsum("cij,cij->cj", self.cMA, self.cMA)
        for p, (i, j) in enumerate(self.pairs):
            d[i] += np.sum(self.pAi[p] ** 2, axis=0)
            d[j] += np.sum(self.pAj[p] ** 2, axis=0)
            M[i] += np.sum(self.pMAi[p] ** 2, axis=0)
            M[j] += np.sum(self.pMAj[p] ** 2, axis=0)
        return d, M

    def _scaled(self, D):
        D = np.asarray(D, np.float64).reshape(self.nc, 9)
        cA, cMA = self.cA * D[:, None, :], self.cMA * D[:, None, :]
        i, j = self.pairs[:, 0], self.pairs[:, 1]
        return D, cA, cMA, self.pAi * D[i][:, None, :], self.pAj * D[j][:, None, :], self.pMAi * D[i][:, None, :], self.pMAj * D[j][:, None, :]

    def hx(self, D, x):
        """sum over the prior rows of A^T (A x) per camera [nc, 9] (A scaled by D) and its magnitude"""
        D, cA, cMA, Ai, Aj, MAi, MAj = self._scaled(D)
        x = np.asarray(x, np.float64).reshape(self.nc, 9)
        ax = np.abs(x)
        y = np.einsum("cij,cik,ck->cj", cA, cA, x)
        My = np.einsum("cij,cik,ck->cj", cMA, cMA, ax)
        for p, (i, j) in enumerate(self.pairs):
            ap = Ai[p] @ x[i] + Aj[p] @ x[j]
            mp = MAi[p] @ ax[i] + MAj[p] @ ax[j]
            y[i] += Ai[p].T @ ap
            y[j] += Aj[p].T @ ap
            My[i] += MAi[p].T @ mp
            My[j] += MAj[p].T @ mp
        return y, My

    def g(self, D):
        """sum of A^T r per camera [nc, 9] and its magnitude"""
        D, cA, cMA, Ai, Aj, MAi, MAj = self._scaled(D)
        y = np.einsum("cij,ci->cj", cA, self.cr)
        My = np.einsum("cij,ci->cj", cMA, self.cMr)
        for p, (i, j) in enumerate(self.pairs):
            y[i] += Ai[p].T @ self.pr[p]
            y[j] += Aj[p].T @ self.pr[p]
            My[i] += MAi[p].T @ self.pMr[p]
            My[j] += MAj[p].T @ self.pMr[p]
        return y, My

    def blocks(self, D):
        """the diagonal block sum A^T A per camera [nc, 9, 9] and its magnitude"""
        D, cA, cMA, Ai, Aj, MAi, MAj = self._scaled(D)
        B = np.einsum("cij,cik->cjk", cA, cA)
        MB = np.einsum("cij,cik->cjk", cMA, cMA)
        for p, (i, j) in enumerate(self.pairs):
            B[i] += Ai[p].T @ Ai[p]
            B[j] += Aj[p].T @ Aj[p]
            MB[i] += MAi[p].T @ MAi[p]
            MB[j] += MAj[p].T @ MAj[p]
        return B, MB

    def k(self):
        """the gamma_k of the prior terms per camera: 9 for the absolute prior, 12 per incident pair side"""
        return 9 * self.has_camera + 12 * side_counts(self.nc, self.pairs)

    # -- per-item quantities --
    def cost_items(self, kind):
        """1/2 |L e|^2 per item and its magnitude (the rounding of e and of the sum of squares)"""
        r, Mr = (self.cr, self.cMr) if kind == "camera" else (self.pr, self.pMr)
        return 0.5 * np.sum(r * r, axis=1), np.sum(np.abs(r) * Mr, axis=1) + 0.5 * np.sum(r * r, axis=1)

    def ldiff_items(self, kind, d):
        """(A d)^T (1/2 A d + r) per item for the unscaled increment d [9 nc], and its magnitude"""
        d = np.asarray(d, np.float64).reshape(self.nc, 9)
        ad = np.abs(d)
        if kind == "camera":
            u = np.einsum("cij,cj->ci", self.cA, d)
            Mu = np.einsum("cij,cj->ci", self.cMA, ad)
            r, Mr = self.cr, self.cMr
        else:
            i, j = self.pairs[:, 0], self.pairs[:, 1]
            u = np.einsum("pij,pj->pi", self.pAi, d[i]) + np.einsum("pij,pj->pi", self.pAj, d[j])
            Mu = np.einsum("pij,pj->pi", self.pMAi, ad[i]) + np.einsum("pij,pj->pi", self.pMAj, ad[j])
            r, Mr = self.pr, self.pMr
        return np.sum(u * (0.5 * u + r), axis=1), np.sum(Mu * (0.5 * Mu + np.abs(r)) + np.abs(u) * Mr, axis=1)


def gamma(k, u):
    return k * u / (1 - k * u)


# ---- a restatement of the kernels' per-camera loops, with planted faults -------------------------------------------------
def kernel_hx(terms, D, x, fault=None, at=None, dtype=np.float64):
    """the prior part of the operator as the kernels form it, in `dtype`: per camera (thread) A_c^T A_c x_c (k_prior_scale's
    H, then k_pcg_q's row products) plus, over the camera's incident sides in list order, A_s^T A_s x_c (k_pair_accum's H)
    and O_ij x_j (pair_ov_entry).  Planted faults, at camera `at` (a list of cameras for "drop_block_last"):
      "neighbour"        the camera's prior terms written to the next camera (its own lost)
      "drop_block_last"  the cameras at the end of a 128-thread block get no prior terms
      "side_dropped" / "side_doubled"   the first of the camera's sides left out / counted twice
      "O_on_vi"          O_ij applied to x_i instead of x_j"""
    f = lambda a: np.asarray(np.asarray(a, np.float64), dtype)
    Dr, cA, _, Ai, Aj, _, _ = terms._scaled(D)
    cA = f(cA)
    As = f(np.stack([Ai, Aj], axis=1)) if terms.m else np.zeros((0, 2, 6, 9), dtype)  # [m][side] = A_s of item 2 p + side
    x = f(np.asarray(x, np.float64).reshape(terms.nc, 9))
    ptr, item = sides(terms.nc, terms.pairs)
    y = np.zeros((terms.nc, 9), dtype)
    for c in range(terms.nc):
        H = cA[c].T @ cA[c]
        O = []
        sl = list(item[ptr[c]:ptr[c + 1]])
        if fault == "side_dropped" and c == at and sl:
            sl = sl[1:]
        if fault == "side_doubled" and c == at and sl:
            sl = sl[:1] + sl
        for it in sl:
            p, s = divmod(int(it), 2)
            H = H + As[p, s].T @ As[p, s]
            O.append((As[p, s].T @ As[p, 1 - s], int(terms.pairs[p, 1 - s])))
        v = H @ x[c]
        for Oij, j in O:
            v = v + Oij @ (x[c] if (fault == "O_on_vi" and c == at) else x[j])
        if fault == "drop_block_last" and c in at:
            continue
        if fault == "neighbour" and c == at:
            y[(c + 1) % terms.nc] += v
            continue
        y[c] += v
    return y.astype(np.float64)


def kernel_item_sum(items, fault=None, threads=SUM_THREADS, dtype=np.float64):
    """k_prior_cost / k_prior_ldiff: thread t sums items t, t + threads, ... in double, then the fixed block sum; items are
    the Scalar terms.  Fault "item_257_dropped": item 256 (the 257th) left out."""
    items = np.asarray(np.asarray(items, np.float64), dtype).astype(np.float64)
    acc = np.zeros(threads)
    for p in range(len(items)):
        if fault == "item_257_dropped" and p == SUM_THREADS:
            continue
        acc[p % threads] += items[p]
    return float(np.sum(acc))


def kernel_group_sum(d2, group, fault=None, dtype=np.float64):
    """k_group_sum_diag2 on the intrinsics entries of diag2 [nc, 9], in `dtype` (group_block_sum<S> accumulates in S):
    members strided over GROUP_THREADS threads, then a tree, the sum written to every member.  Fault "member_129_dropped":
    the 129th member of every group left out."""
    d2 = np.asarray(np.asarray(d2, np.float64), dtype)
    out = np.array(d2, dtype)
    for g in np.unique(group[group >= 0]):
        mem = np.flatnonzero(group == g)
        if len(mem) < 2:
            continue
        acc = np.zeros((GROUP_THREADS, 3), dtype)
        for q, c in enumerate(mem):
            if fault == "member_129_dropped" and q == GROUP_THREADS:
                continue
            acc[q % GROUP_THREADS] += d2[c, 6:]
        h = GROUP_THREADS // 2
        while h:
            acc[:h] += acc[h:2 * h]
            h //= 2
        out[mem, 6:] = acc[0]
    return out.astype(np.float64)


def group_sum_model(d2, group):
    """the model: every member's intrinsics column norms are the sum over its group (groups of >= 2)"""
    out = np.array(d2, np.float64)
    for g in np.unique(group[group >= 0]):
        mem = np.flatnonzero(group == g)
        if len(mem) >= 2:
            out[mem, 6:] = d2[mem, 6:].sum(axis=0)
    return out


def group_k(group, nc):
    """the gamma_k of the group sum for every camera: its group's size (0 ungrouped)"""
    k = np.zeros(nc)
    for g in np.unique(group[group >= 0]):
        mem = np.flatnonzero(group == g)
        if len(mem) >= 2:
            k[mem] = len(mem)
    return k


# ---- checkers -------------------------------------------------------------------------------------------------------------
def check_item_sum(got, items, mag, u, what, extra=0.0):
    """a sum over n items, accumulated in double (k_prior_cost, k_prior_ldiff): |got - sum items| <= gamma_(n + 2) (in
    double) sum |items| + C_LIN u sum mag_p (each item's own rounding in the handle's Scalar of unit round-off u) + extra
    (the rounding of the part of `got` that is not the items)"""
    items, mag = np.asarray(items, np.float64), np.asarray(mag, np.float64)
    want = float(np.sum(items))
    bar = gamma(len(items) + 2, U64) * float(np.sum(np.abs(items))) + C_LIN * u * float(np.sum(mag)) + extra
    ratio = abs(got - want) / bar if bar > 0 else (0.0 if got == want else np.inf)
    assert ratio <= 1, (what, "items", len(items), "got", got, "want", want, "error / bar", ratio)
    return bar


def landmark_cost_items(lms, idx, mean, L):
    """1/2 |L (x - x0)|^2 per landmark prior and its magnitude (x - x0 rounds at |x| + |x0|)"""
    lms, mean, L = (np.asarray(a, np.float64) for a in (lms, mean, L))
    e = lms[np.asarray(idx)] - mean
    r = np.einsum("mij,mj->mi", L, e)
    Mr = np.einsum("mij,mj->mi", np.abs(L), np.abs(lms[np.asarray(idx)]) + np.abs(mean))
    return 0.5 * np.sum(r * r, axis=1), np.sum(np.abs(r) * Mr, axis=1) + 0.5 * np.sum(r * r, axis=1)


def check_bar(got, want, bar, what):
    """entry by entry |got - want| <= bar, reported per camera: the camera, the entry and error / bar of the worst"""
    nc = want.shape[0]
    got = np.asarray(got, np.float64).reshape(want.shape)
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.where(got == want, 0.0, np.abs(got - want) / bar)
    ratio = np.where(np.isnan(ratio), np.inf, ratio).reshape(nc, -1)
    cam = int(np.argmax(ratio.max(axis=1)))
    assert ratio[cam].max() <= 1, (what, "camera", cam, "entry", int(np.argmax(ratio[cam])), "error / bar", ratio[cam].max())


@functools.lru_cache(maxsize=None)
def item_problem(n_cams, n_lms=12):
    """a problem of n_cams cameras (>= 2) and at least n_lms landmarks, tracks of up to 4 cameras, every camera observed"""
    from rootba_b200.synthetic import synth_bal
    rng = np.random.default_rng(n_cams + 77)
    nl = max(n_lms, 3 * n_cams)
    k = min(4, n_cams)
    tracks = [np.sort(np.concatenate([[i % n_cams], rng.choice(np.delete(np.arange(n_cams), i % n_cams), k - 1, replace=False)]))
              for i in range(nl)]
    return synth_bal(n_cams, nl, 0.0, seed=n_cams + 77, tracks=tracks, lm_spread=0.5)


ITEM_COUNTS = (1, 255, 256, 257, 511, 512, 513, 4100)
# the camera prior has one item per camera and a problem at least two cameras (a track has two): its single-item launch is
# that of the other kinds (the same kernel, another K)
CAMERA_ITEM_COUNTS = (2,) + ITEM_COUNTS[1:]
PAIR_ITEM_CAMERAS = 600
LM_ITEM_CAMERAS = 1400  # 4200 landmarks


def random_pairs(nc, m, seed):
    rng = np.random.default_rng(seed)
    a = rng.integers(0, nc, m)
    b = (a + 1 + rng.integers(0, nc - 1, m)) % nc
    return np.stack([a, b], axis=1).astype(np.int32)


# ---- the per-camera checkers of the scaling, b and the inverse blocks (float64 handles) ------------------------------------
def check_scaling(got_d2, d_rep, s0, s, terms, groups, what="scaling"):
    """diag2 = (1 / s - eps)^2 of the handle against the twin's reprojection column norms d_rep (from its scaling s0) plus
    the prior rows', summed over a group: gamma of the camera's terms + 8 (the two conversions between s and diag2) of the
    magnitudes, + C_LIN units of the prior rows' linearisation"""
    nc = terms.nc
    kp = terms.k()
    gk = group_k(groups, nc) if groups is not None else np.zeros(nc)
    gsum = (lambda v: group_sum_model(v, groups)) if groups is not None else (lambda v: v)
    d_pri, M_pri = terms.diag2()
    s, s0 = np.asarray(s, np.float64).reshape(nc, 9), np.asarray(s0, np.float64).reshape(nc, 9)
    bar = U64 * ((kp + gk + 8)[:, None] * gsum(d_rep + d_pri + 1 / s0 ** 2) + C_LIN * gsum(M_pri)) + 8 * U64 / s ** 2
    check_bar(got_d2, gsum(d_rep + d_pri), bar, what)


def check_b(got, b_rep, Mb, cc, s, terms, groups, what="b"):
    """b against solver_model's b_rep (magnitude Mb, constants cc per camera) + sum A^T r of the priors, contracted over
    the groups (the members' entries 6..8 are 0 exactly)"""
    nc = terms.nc
    kp = terms.k()
    g, Mg = terms.g(s)
    want, bar = b_rep + g, U64 * (cc[:, None] * Mb + (kp + C_LIN)[:, None] * Mg)
    if groups is not None:
        import shared_intrinsics_model as sm
        lead = sm.leads(groups)
        gk = group_k(groups, nc)
        want = sm.contract(want, lead).reshape(nc, 9)
        bar = sm.contract(bar + gk[:, None] * U64 * (np.abs(b_rep) + np.abs(g)), lead).reshape(nc, 9)
        bar = np.where(bar == 0, np.inf, bar)
        assert np.all(np.asarray(got).reshape(nc, 9)[sm.members(lead).reshape(nc, 9)] == 0), (what, "members' entries 6..8")
    check_bar(got, want, bar, what)


def grouped_blocks(B, M, lam, groups):
    """the blocks k_group_precond + k_precond_invert invert (shared_intrinsics_model.device_blocks, with magnitudes) and the
    mask of their free entries"""
    nc = len(B)
    if groups is None:
        return B, M, np.ones((nc, 9), bool)
    import shared_intrinsics_model as sm
    lead = sm.leads(groups)
    Bd, Md = B.copy(), M.copy()
    free = np.ones((nc, 9), bool)
    eye = lam * np.eye(9)
    for c in np.flatnonzero(lead >= 0):
        for X, src in ((Bd, B - eye), (Md, M - eye)):
            X[c][:6, 6:] = X[c][6:, :6] = 0
            X[c][6:, 6:] = (src[lead == c][:, 6:, 6:].sum(axis=0) + eye[6:, 6:]) if lead[c] == c else eye[6:, 6:]
        if lead[c] != c:
            free[c, 6:] = False
    return Bd, Md, free


def check_inverse_blocks(got, B_rep, MB_rep, c_rep, s, lam, terms, groups, what):
    """the inverse blocks against the inverse of the reprojection blocks (incl. lam I) + the prior blocks, in the grouped
    partition, at the bar of solver_model.inverse with c = c_rep + the camera's prior and group terms"""
    import solver_model as smod
    nc = terms.nc
    kp = terms.k()
    gk = group_k(groups, nc) if groups is not None else np.zeros(nc)
    B, MB = terms.blocks(s)
    Bd, Md, free = grouped_blocks(B_rep + B, MB_rep + (1 + C_LIN / np.maximum(kp, 1))[:, None, None] * MB, lam, groups)
    c = c_rep + kp + gk
    for cam in range(nc):
        f = free[cam]
        want, Mw = np.zeros((9, 9)), np.zeros((9, 9))
        want[np.ix_(f, f)], Mw[np.ix_(f, f)] = smod.inverse(Bd[cam][np.ix_(f, f)], Md[cam][np.ix_(f, f)])
        e, k = smod.excess(got[cam], want, Mw, c[cam], U64)
        assert e <= 1, (what, "camera", cam, "entry", k, "error / bar", e)
