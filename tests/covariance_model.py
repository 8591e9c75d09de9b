"""Float64 model of the marginal covariances (rba_compute_covariance, DESIGN.md section 16), written from the mathematics.

- dense_inverse: the definition, inv(J^T J) of the whole problem [Jp | Jl] with the held columns deleted, and the
  condition number of the Jacobi-equilibrated matrix (the bars of the tests are c * kappa * u).
- schur_reduced: the reduced camera matrix S = sum_l (Jp_l^T Jp_l - Jp_l^T Jl_l pinv(Hll) Jl_l^T Jp_l), landmark by
  landmark from the per-observation blocks (no dense Jacobian: usable at hundreds of cameras).
- eigen_form: the formula the device evaluates, Hll = V Lambda V^T with eigenvalues <= 1e-10 lambda_max dropped,
  K_i = Lambda+^-1/2 V+^T Jl_i^T Jp_i, S = sum_l (delta_ij Jp_i^T Jp_i - K_i^T K_j), landmark marginal
  W (I + sum_ab K_a Sigma_ab K_b^T) W^T with W = V+ Lambda+^-1/2 (NaN when rank < 3).
- eigen_reduced / landmark_marginal: the same formula vectorised (batched eigh, the K_a^T K_b blocks of all landmarks of one
  track length at a time, in chunks), for problems of thousands of cameras and hundreds of thousands of landmarks.
- entry_bar_scale / landmark_bar_scale: the magnitudes the componentwise bars of the device tests are multiples of.
- tile_pairs_read: which 64 x 64 tiles of the padded inverse the landmark marginals read.
"""
import numpy as np

EIG_DROP = 1e-10
TILE = 64  # COV_TB of rootba_b200/csrc/covariance.cuh: the tile of the blocked dense inverse


def fixed_mask(flags, nc):
    """[9 nc] bool of the held increment entries (RBA_FIX_* bits per camera), all False for None"""
    if flags is None:
        return np.zeros(9 * nc, bool)
    from objective_checks import fixed_entries
    return fixed_entries(np.asarray(flags))


def spd_cond(H):
    """2-norm condition number of a symmetric positive definite matrix"""
    ev = np.linalg.eigvalsh(H)
    return float(ev[-1] / ev[0])


def dense_inverse(Jp, Jl, nc, nl, fixed=None):
    """(cam [nc, 9, 9], lm [nl, 3, 3], kappa): blocks of inv(J^T J) with J = [Jp | Jl] and the held camera columns deleted
    (their rows and columns of the output are 0); kappa = 2-norm condition of D H D, D = diag(H)^-1/2"""
    fixed = np.zeros(9 * nc, bool) if fixed is None else fixed
    J = np.hstack([Jp[:, ~fixed], Jl])
    H = J.T @ J
    d = 1.0 / np.sqrt(np.diag(H))
    Heq = H * d[:, None] * d[None, :]
    kappa = spd_cond(Heq)
    C = np.linalg.inv(Heq) * d[:, None] * d[None, :]
    nf = int((~fixed).sum())
    Ccam = np.zeros((9 * nc, 9 * nc))
    Ccam[np.ix_(~fixed, ~fixed)] = C[:nf, :nf]
    cam = np.stack([Ccam[9 * c:9 * c + 9, 9 * c:9 * c + 9] for c in range(nc)])
    lm = np.stack([C[nf + 3 * l:nf + 3 * l + 3, nf + 3 * l:nf + 3 * l + 3] for l in range(nl)])
    return cam, lm, kappa


def schur_reduced(jp, jl, obs_cam, lm_off, nc):
    """S [9 nc, 9 nc] from the per-observation blocks jp [nobs, 2, 9], jl [nobs, 2, 3] with pinv of every Hll"""
    S = np.zeros((9 * nc, 9 * nc))
    for l in range(len(lm_off) - 1):
        o = np.arange(lm_off[l], lm_off[l + 1])
        cams = obs_cam[o]
        Jp = np.zeros((2 * len(o), 9 * len(o)))
        for k in range(len(o)):
            Jp[2 * k:2 * k + 2, 9 * k:9 * k + 9] = jp[o[k]]
        Jl = jl[o].reshape(-1, 3)
        B = Jp.T @ Jp - Jp.T @ Jl @ np.linalg.pinv(Jl.T @ Jl, rcond=EIG_DROP, hermitian=True) @ Jl.T @ Jp
        idx = (9 * cams[:, None] + np.arange(9)[None, :]).ravel()
        S[np.ix_(idx, idx)] += B
    return S


def landmark_factors(jl_l):
    """(W [3, 3] = V+ Lambda+^-1/2 with zero columns for dropped eigenvalues, rank) of one landmark's Jl rows [2n, 3]"""
    lam, V = np.linalg.eigh(jl_l.T @ jl_l)
    lmax = lam.max()
    keep = (lam > EIG_DROP * lmax) if lmax > 0 else np.zeros(3, bool)
    W = np.where(keep[None, :], V / np.sqrt(np.where(keep, lam, 1.0))[None, :], 0.0)
    return W, int(keep.sum())


def eigen_form(jp, jl, obs_cam, lm_off, nc, H_extra=None):
    """(cam [nc, 9, 9], lm [nl, 3, 3]) by the device's formula; H_extra [9 nc, 9 nc] (priors) is added to S"""
    nl = len(lm_off) - 1
    S = np.zeros((9 * nc, 9 * nc)) if H_extra is None else np.array(H_extra, np.float64)
    K = np.zeros((len(obs_cam), 3, 9))
    Ws, ranks = [], []
    for l in range(nl):
        o = np.arange(lm_off[l], lm_off[l + 1])
        W, r = landmark_factors(jl[o].reshape(-1, 3))
        Ws.append(W)
        ranks.append(r)
        for k in o:
            K[k] = W.T @ (jl[k].T @ jp[k])
        for a in o:
            ca = obs_cam[a]
            S[9 * ca:9 * ca + 9, 9 * ca:9 * ca + 9] += jp[a].T @ jp[a]
            for b in o:
                cb = obs_cam[b]
                S[9 * ca:9 * ca + 9, 9 * cb:9 * cb + 9] -= K[a].T @ K[b]
    Sig = np.linalg.inv(S)
    cam = np.stack([Sig[9 * c:9 * c + 9, 9 * c:9 * c + 9] for c in range(nc)])
    lm = np.full((nl, 3, 3), np.nan)
    for l in range(nl):
        if ranks[l] < 3:
            continue
        o = np.arange(lm_off[l], lm_off[l + 1])
        X = np.eye(3)
        for a in o:
            for b in o:
                ca, cb = obs_cam[a], obs_cam[b]
                X += K[a] @ Sig[9 * ca:9 * ca + 9, 9 * cb:9 * cb + 9] @ K[b].T
        lm[l] = Ws[l] @ X @ Ws[l].T
    return cam, lm


def _groups(lm_off, chunk):
    """(n, landmark indices) of the landmarks of track length n, in chunks of at most `chunk` camera pairs (m n^2)"""
    n_of = np.diff(lm_off)
    for n in np.unique(n_of):
        idx = np.flatnonzero(n_of == n)
        step = max(1, chunk // int(n * n))
        for s in range(0, len(idx), step):
            yield int(n), idx[s:s + step]


def _slots(lm_off, n, idx):
    return np.asarray(lm_off)[idx][:, None] + np.arange(n)[None, :]


def _add_blocks(Sb, ca, cb, blocks):
    """Sb [nc, nc, 9, 9] += blocks [m, 9, 9] at (ca, cb), duplicates summed (sorted by key, then reduceat)"""
    nc = Sb.shape[0]
    key = ca.ravel().astype(np.int64) * nc + cb.ravel()
    order = np.argsort(key, kind="stable")
    key = key[order]
    starts = np.flatnonzero(np.r_[True, key[1:] != key[:-1]])
    u = key[starts]
    Sb[u // nc, u % nc] += np.add.reduceat(blocks.reshape(-1, 9, 9)[order], starts, axis=0)


def eigen_reduced(jp, jl, obs_cam, lm_off, nc, H_extra=None, chunk=1 << 17):
    """eigen_form's elimination, vectorised: (S [9 nc, 9 nc] full symmetric, K [nobs, 3, 9], W [nl, 3, 3], rank [nl],
    kappa_l [nl] = lambda_max / lambda_min of the kept eigenvalues of every Hll).  H_extra (priors) is added to S."""
    lm_off, obs_cam = np.asarray(lm_off), np.asarray(obs_cam)
    nl = len(lm_off) - 1
    lm_of = np.repeat(np.arange(nl), np.diff(lm_off))
    H = np.add.reduceat(np.einsum("kri,krj->kij", jl, jl), lm_off[:-1], axis=0)
    lam, V = np.linalg.eigh(H)
    lmax = lam[:, -1:]
    keep = (lam > EIG_DROP * lmax) & (lmax > 0)
    W = np.where(keep[:, None, :], V / np.sqrt(np.where(keep, lam, 1.0))[:, None, :], 0.0)
    rank = keep.sum(1)
    with np.errstate(divide="ignore", invalid="ignore"):
        kappa_l = np.where(rank > 0, lmax[:, 0] / np.where(keep, lam, np.inf).min(1), np.inf)
    K = np.einsum("kai,kaj->kij", W[lm_of], np.einsum("kra,krj->kaj", jl, jp))
    Sb = np.zeros((nc, nc, 9, 9))
    _add_blocks(Sb, obs_cam, obs_cam, np.einsum("kri,krj->kij", jp, jp))
    for n, idx in _groups(lm_off, chunk):
        sl = _slots(lm_off, n, idx)
        Kg, C = K[sl], obs_cam[sl]
        blk = -np.einsum("mapi,mbpj->mabij", Kg, Kg)
        _add_blocks(Sb, np.broadcast_to(C[:, :, None], blk.shape[:3]), np.broadcast_to(C[:, None, :], blk.shape[:3]), blk)
    S = Sb.transpose(0, 2, 1, 3).reshape(9 * nc, 9 * nc)
    if H_extra is not None:
        S += H_extra
    return S, K, W, rank, kappa_l


def landmark_marginal(Sig, K, W, rank, obs_cam, lm_off, chunk=1 << 15):
    """lm [nl, 3, 3] = W (I + sum_ab K_a Sigma_ab K_b^T) W^T, the Sigma_ab gathered from the full inverse Sig [9 nc, 9 nc]
    (NaN when rank < 3)"""
    obs_cam = np.asarray(obs_cam)
    nc = Sig.shape[0] // 9
    S4 = Sig.reshape(nc, 9, nc, 9)
    out = np.full((len(lm_off) - 1, 3, 3), np.nan)
    for n, idx in _groups(lm_off, chunk):
        sl = _slots(lm_off, n, idx)
        Kg, C = K[sl], obs_cam[sl]
        Sab = S4[C[:, :, None], :, C[:, None, :], :]  # [m, n, n, 9, 9]
        X = np.eye(3) + np.einsum("mapi,mabij,mbqj->mpq", Kg, Sab, Kg, optimize=True)
        out[idx] = np.einsum("mik,mkl,mjl->mij", W[idx], X, W[idx])
    out[np.asarray(rank) < 3] = np.nan
    return out


def entry_bar_scale(Sig):
    """sigma = sqrt(diag Sig): the scale sigma_i sigma_j >= |Sig_ij| of an entry of an SPD inverse, against which the
    rounding of a Cholesky-based inverse of the Jacobi-equilibrated matrix is measured (it is relative to the equilibrated
    matrix, whose entries are Sig_ij / (d_i d_j) with d_i = Sig_ii^1/2 up to O(kappa))"""
    return np.sqrt(np.diag(Sig))


def landmark_bar_scale(sigma, K, W, obs_cam, lm_off):
    """per landmark [nl, 3, 3] the magnitudes |W| (I + sum_ab |K_a| sigma_a sigma_b^T |K_b|^T) |W|^T, the landmark formula
    with every Sigma_ab replaced by its entrywise bound sigma_a sigma_b^T: it factors as |W| (I + g g^T) |W|^T with
    g = sum_a |K_a| sigma_a"""
    obs_cam = np.asarray(obs_cam)
    s = sigma.reshape(-1, 9)[obs_cam]
    g = np.add.reduceat(np.einsum("kij,kj->ki", np.abs(K), s), np.asarray(lm_off)[:-1], axis=0)
    X = np.eye(3) + g[:, :, None] * g[:, None, :]
    Wa = np.abs(W)
    return np.einsum("mik,mkl,mjl->mij", Wa, X, Wa)


def tile_pairs_read(obs_cam, lm_off, nc=None):
    """the set of tile pairs (ti >= tj) of the TILE-padded 9 nc matrix whose entries some landmark marginal reads: a landmark
    with cameras a, b reads the 9 x 9 block (a, b), which touches the tiles of rows 9a and 9a + 8 and of columns 9b, 9b + 8"""
    obs_cam = np.asarray(obs_cam)
    out = set()
    for n, idx in _groups(lm_off, 1 << 16):
        C = obs_cam[_slots(lm_off, n, idx)]
        tiles = [(9 * C) // TILE, (9 * C + 8) // TILE]
        for ta in tiles:
            for tb in tiles:
                a, b = np.broadcast_arrays(ta[:, :, None], tb[:, None, :])
                hi, lo = np.maximum(a, b).ravel(), np.minimum(a, b).ravel()
                out |= set(zip(*np.unique(np.stack([hi, lo]), axis=1).tolist()))
    return out


def all_tile_pairs(nc):
    nt = -(-9 * nc // TILE)
    return {(i, j) for i in range(nt) for j in range(i + 1)}


def straddling_cameras(nc):
    """cameras whose 9 rows cross a tile boundary"""
    return [c for c in range(nc) if (9 * c) // TILE != (9 * c + 8) // TILE]


def cond_estimate(cho):
    """1-norm condition estimate (LAPACK dpocon) of the SPD matrix whose lower Cholesky factor is cho[0] (scipy
    cho_factor(lower=True)); anorm is the 1-norm of the factored matrix, passed as cho[2]"""
    from scipy.linalg import lapack
    rcond, info = lapack.dpocon(cho[0], cho[2], uplo="L")
    assert info == 0
    return 1.0 / rcond


U = 2.0 ** -53


def centre_priors(prob, seed=3):
    """a centre prior on every camera (they fix the gauge): means near the cameras' centres, 'centre' square roots"""
    import camera_prior_model as pm
    rng = np.random.default_rng(seed)
    mean = pm.mean_at(np.asarray(prob.cams, np.float64))
    mean[:, 4:7] += rng.normal(0, 0.05, (len(mean), 3))
    L = np.stack([pm.sqrt_info_kind("centre", rng) for _ in range(len(mean))])
    return mean, L


def as_stored(prob, dtype, absp=None, pair=None):
    """the problem and prior arrays as a handle of `dtype` holds them, in float64 (float32: rounded; prior quaternions
    normalised, then rounded)"""
    if dtype != np.float32:
        return prob, absp, pair
    from rootba_b200.synthetic import BalArrays
    r = lambda a: np.asarray(a, np.float32).astype(np.float64)
    p32 = BalArrays(r(prob.cams), r(prob.lms), prob.lm_off, prob.obs_cam, r(prob.obs_xy))
    if absp is not None:
        m = np.array(absp[0], np.float64)
        m[:, :4] /= np.linalg.norm(m[:, :4], axis=1, keepdims=True)
        absp = (r(m), r(absp[1]))
    if pair is not None:
        m = np.array(pair[1], np.float64)
        m[:, :4] /= np.linalg.norm(m[:, :4], axis=1, keepdims=True)
        pair = (pair[0], r(m), r(pair[2]))
    return p32, absp, pair


def reference(prob, dtype=np.float64, absp=None, pair=None, threshold=None, valid_only=False, mask=None):
    """the device's covariance formula in float64 at the state of `prob` (as a `dtype` handle stores it), rotations as the
    kernels build them: dict(cam [nc, 9, 9], lm [nl, 3, 3], kappa (dpocon estimate of the equilibrated S), kappa_l [nl],
    sigma [9 nc], lm_scale [nl, 3, 3] (landmark_bar_scale)).  S is factored with LAPACK dpotrf and inverted with dpotri.
    mask: RBA_FIX_* flags per camera; the held entries' rows and columns are deleted (0 in the output)."""
    import camera_model as cm
    import camera_prior_model as pm
    import pair_prior_model as qm
    from scipy.linalg import cho_factor, lapack
    prob, absp, pair = as_stored(prob, dtype, absp, pair)
    nc = len(prob.cams)
    cams = np.asarray(prob.cams, np.float64)
    jp, jl, _, _ = cm.weighted(prob, dtype=dtype, threshold=threshold, valid_only=valid_only, device_rot=True)
    extra = np.zeros((9 * nc, 9 * nc))
    if absp is not None:
        A, _ = pm.rows(cams, *absp, device_rot=True)
        for c in range(nc):
            extra[9 * c:9 * c + 9, 9 * c:9 * c + 9] += A[c].T @ A[c]
    if pair is not None:
        Jq, _ = qm.rows(cams, *pair, device_rot=True)
        extra += Jq.T @ Jq
    S, K, W, rank, kappa_l = eigen_reduced(jp, jl, prob.obs_cam, prob.lm_off, nc, extra)
    del extra
    fixed = fixed_mask(mask, nc)
    S[fixed, :] = 0.0
    S[:, fixed] = 0.0
    S[fixed, fixed] = 1.0
    d = 1.0 / np.sqrt(np.diag(S))
    S *= d[:, None]
    S *= d[None, :]
    anorm = float(np.abs(S).sum(0).max())
    cho = cho_factor(S, lower=True, overwrite_a=True, check_finite=False)
    kappa = cond_estimate((cho[0], cho[1], anorm))
    Sig, info = lapack.dpotri(cho[0], lower=1, overwrite_c=1)
    assert info == 0
    Sig = np.tril(Sig)
    Sig += np.tril(Sig, -1).T
    Sig *= d[:, None]
    Sig *= d[None, :]
    Sig[fixed, :] = 0.0
    Sig[:, fixed] = 0.0
    sigma = np.where(fixed, 1.0, entry_bar_scale(Sig))  # held entries are exactly 0 on both sides
    cam = np.stack([Sig[9 * c:9 * c + 9, 9 * c:9 * c + 9] for c in range(nc)])
    lm = landmark_marginal(Sig, K, W, rank, prob.obs_cam, prob.lm_off)
    scale = landmark_bar_scale(sigma, K, W, prob.obs_cam, prob.lm_off)
    return dict(cam=cam, lm=lm, kappa=kappa, kappa_l=kappa_l, sigma=sigma, lm_scale=scale, N=9 * nc, Sig=Sig, K=K, W=W,
                rank=rank, obs_cam=np.asarray(prob.obs_cam), lm_off=np.asarray(prob.lm_off))


def camera_excess(cam, ref, c=8):
    """(max over the camera blocks of |cam - ref| / (sigma_i sigma_j), bar = c N kappa u): the componentwise camera check
    passes when the first is <= the second"""
    s = ref["sigma"].reshape(-1, 9)
    scale = s[:, :, None] * s[:, None, :]
    return float(np.max(np.abs(cam - ref["cam"]) / scale)), c * ref["N"] * ref["kappa"] * U


def landmark_excess(lm, ref, c=8):
    """(max over the landmarks of |lm - ref| / (bar_l lm_scale), max bar_l) with bar_l = c (N kappa + n_l kappa_l) u per
    landmark: the inverse of the reduced matrix contributes c N kappa u as for the cameras, the landmark's own 3 x 3
    eigen-elimination over its n_l observations c n_l kappa_l u (kappa_l = the condition of its Hll); NaN blocks must be NaN
    in both.  The check passes when the first is <= 1."""
    nan_ref = np.isnan(ref["lm"]).all(axis=(1, 2))
    if not np.array_equal(np.isnan(lm).any(axis=(1, 2)), nan_ref):
        return np.inf, 0.0
    ok = ~nan_ref
    bar = c * (ref["N"] * ref["kappa"] + np.diff(ref["lm_off"])[ok] * ref["kappa_l"][ok]) * U
    ex = np.abs(lm[ok] - ref["lm"][ok]) / (bar[:, None, None] * ref["lm_scale"][ok])
    return (float(ex.max()) if ex.size else 0.0), (float(bar.max()) if bar.size else 0.0)


def check(cam, lm, ref, c=8, what=""):
    """assert the camera blocks and (unless lm is None) the landmark blocks against the reference; every bar <= 1e-4"""
    ex, bar = camera_excess(cam, ref, c)
    assert bar <= 1e-4, f"{what}: camera bar {bar:.3g} above 1e-4 (kappa {ref['kappa']:.3g})"
    assert ex <= bar, f"{what}: camera blocks off by {ex:.3g} sigma_i sigma_j, bar {bar:.3g} (c = {c}, kappa {ref['kappa']:.3g})"
    if lm is not None:
        lex, lbar = landmark_excess(lm, ref, c)
        assert lbar <= 1e-4, f"{what}: landmark bar {lbar:.3g} above 1e-4"
        assert lex <= 1.0, f"{what}: landmark blocks off by {lex:.3g} x their bars (largest bar {lbar:.3g}, c = {c})"
    return bar


def tile_case(nc, seed=0, per_camera=24):
    """nc cameras with uniformly random (non-local) tracks of 2..6 cameras, per_camera landmarks per camera, and a centre
    prior on every camera: every pair of tiles of the inverse is read by some landmark (tile_pairs_read)"""
    from rootba_b200.synthetic import synth_bal
    rng = np.random.default_rng(seed)
    nl = per_camera * nc
    tracks = [rng.choice(nc, int(rng.integers(2, 7)), replace=False) for _ in range(nl)]
    prob = synth_bal(nc, nl, 0.0, seed=seed, tracks=tracks, lm_spread=0.5)
    return prob, centre_priors(prob, seed + 1)
