"""Float64 model of the covariance blocks of chosen pairs (rba_compute_covariance_blocks, DESIGN.md section 20), written from
the block inverse of H = J^T J.  Not collected by pytest (no test_ prefix).

With H = [[Hpp, Hpl], [Hlp, Hll]], S = Hpp - Hpl Hll^-1 Hlp and, per landmark l, Hll^+ = W_l W_l^T (W_l = V+ Lambda+^-1/2,
covariance_model.landmark_factors) and K_i = W_l^T Jl_i^T Jp_i per slot i of l (camera a_i):
  H^-1 = [[S^-1, -S^-1 Hpl Hll^-1], [., Hll^-1 + Hll^-1 Hlp S^-1 Hpl Hll^-1]], so with Sigma = S^-1
  camera pair      Cov(d_a, d_b) = Sigma_ab
  camera-landmark  Cov(d_c, d_l) = -(sum_i Sigma_{c,a_i} K_i^T) W_l^T
  landmark pair    Cov(d_l, d_m) = W_l (delta_lm I + sum_ij K_i Sigma_{a_i b_j} K_j^T) W_m^T
  relative pose    A Sigma_P A^T, Sigma_P the pose entries (v_i, w_i, v_j, w_j) of cameras i, j and
                   A = [[I, -[t_rel]x, -M, 0], [0, I, 0, -M]], M = R_i R_j^T, t_rel = t_i - M t_j (relative_jacobian)

- factors: S, K, W, rank and kappa_l by the device's eigen-elimination, with landmark priors (Hll += L^T L).
- reference: Sigma (held entries deleted, intrinsics groups expanded P S_u^-1 P^T), the condition kappa of the equilibrated S,
  and sigma = sqrt(diag Sigma).
- blocks: the four formulas for the requests, vectorised; `fault` plants one of the errors the check must catch: BASE_FAULTS
  in the formulas themselves, CLASS_FAULTS in the loops and inputs of the kernels (tests/covariance_block_classes.py).
- dense_blocks: the same blocks cut from the full inverse of the dense total system (the definition).
- bar_scales / check: the componentwise check of the device tests, bars c (N kappa + n kappa_l) u as in section 16.
"""
import numpy as np

import camera_model as cm
import covariance_model as cvm

U = 2.0 ** -53
KINDS = ("cameras", "camera_landmark", "landmarks", "relative")
BASE_FAULTS = ("cam_lm_sign", "identity_off_diagonal", "transposed_cameras", "aj_sign", "no_t_rel")
# slot_pair_order: a landmark pair's slot pairs decoded as (t / n_l, t % n_l) instead of (t / n_m, t % n_m) (slots past the
#   landmark's own are its neighbours', as the kernel would read them); first_pass_only: only the first 32 slots (camera-
#   landmark) or slot pairs (landmark pairs) summed, one pass of the warp; w_swapped: W_m on the left of a landmark pair;
#   member_not_expanded: the intrinsics rows and columns of Sigma of the members of an intrinsics group left 0;
#   lm_prior_dropped: the landmark priors' L^T L left out of Hll
CLASS_FAULTS = ("slot_pair_order", "first_pass_only", "w_swapped", "member_not_expanded", "lm_prior_dropped")
FAULTS = BASE_FAULTS + CLASS_FAULTS


def factors(jp, jl, obs_cam, lm_off, nc, H_extra=None, lm_info=None):
    """the device's elimination: (S [9 nc, 9 nc], K [nobs, 3, 9], W [nl, 3, 3], rank [nl], kappa_l [nl]).  H_extra [9 nc, 9 nc]
    (camera and pair priors) is added to S; lm_info [nl, 3, 3] (landmark priors' L^T L, 0 for none) to every Hll."""
    lm_off, obs_cam = np.asarray(lm_off), np.asarray(obs_cam)
    nl = len(lm_off) - 1
    lm_of = np.repeat(np.arange(nl), np.diff(lm_off))
    H = np.add.reduceat(np.einsum("kri,krj->kij", jl, jl), lm_off[:-1], axis=0)
    if lm_info is not None:
        H = H + lm_info
    lam, V = np.linalg.eigh(H)
    lmax = lam[:, -1:]
    keep = (lam > cvm.EIG_DROP * lmax) & (lmax > 0)
    W = np.where(keep[:, None, :], V / np.sqrt(np.where(keep, lam, 1.0))[:, None, :], 0.0)
    rank = keep.sum(1)
    with np.errstate(divide="ignore", invalid="ignore"):
        kappa_l = np.where(rank > 0, lmax[:, 0] / np.where(keep, lam, np.inf).min(1), np.inf)
    K = np.einsum("kai,kaj->kij", W[lm_of], np.einsum("kra,krj->kaj", jl, jp))
    Sb = np.zeros((nc, nc, 9, 9))
    cvm._add_blocks(Sb, obs_cam, obs_cam, np.einsum("kri,krj->kij", jp, jp))
    for n, idx in cvm._groups(lm_off, 1 << 17):
        sl = cvm._slots(lm_off, n, idx)
        Kg, C = K[sl], obs_cam[sl]
        blk = -np.einsum("mapi,mbpj->mabij", Kg, Kg)
        cvm._add_blocks(Sb, np.broadcast_to(C[:, :, None], blk.shape[:3]), np.broadcast_to(C[:, None, :], blk.shape[:3]), blk)
    S = Sb.transpose(0, 2, 1, 3).reshape(9 * nc, 9 * nc)
    if H_extra is not None:
        S = S + H_extra
    return S, K, W, rank, kappa_l


def reference(jp, jl, obs_cam, lm_off, cams, H_extra=None, lm_info=None, fixed=None, lead=None):
    """dict(Sig [9 nc, 9 nc], K, W, rank, kappa_l, kappa, sigma [9 nc], N, obs_cam, lm_off, cams) of the device's formula in
    float64.  fixed [9 nc] bool: held entries (rows and columns of Sig exactly 0); lead: intrinsics groups
    (shared_intrinsics_model.leads), Sig = P S_u^-1 P^T with S_u = P^T S P and the members' entries 6..8 deleted from S_u."""
    import shared_intrinsics_model as sim
    from scipy.linalg import cho_factor, cho_solve
    cams = np.asarray(cams, np.float64)
    nc = len(cams)
    S, K, W, rank, kappa_l = factors(jp, jl, obs_cam, lm_off, nc, H_extra, lm_info)
    fixed = np.zeros(9 * nc, bool) if fixed is None else np.asarray(fixed, bool)
    P = np.eye(9 * nc) if lead is None else sim.expansion(lead)
    keep = np.arange(9 * nc) if lead is None else np.flatnonzero(~sim.members(lead))
    Su = P.T @ S @ P
    fu = ~fixed[keep]
    A = Su[np.ix_(fu, fu)]
    d = 1.0 / np.sqrt(np.diag(A))
    Aeq = A * d[:, None] * d[None, :]
    cho = cho_factor(Aeq, lower=True)
    kappa = cvm.cond_estimate((cho[0], cho[1], float(np.abs(Aeq).sum(0).max())))
    Ginv = np.zeros_like(Su)
    Ginv[np.ix_(fu, fu)] = cho_solve(cho, np.eye(len(A))) * d[:, None] * d[None, :]
    Sig = P @ Ginv @ P.T
    Sig[fixed, :] = 0.0
    Sig[:, fixed] = 0.0
    sigma = np.sqrt(np.diag(Sig))
    return dict(Sig=Sig, K=K, W=W, rank=rank, kappa_l=kappa_l, kappa=kappa, sigma=sigma, N=int(fu.sum()),
                obs_cam=np.asarray(obs_cam), lm_off=np.asarray(lm_off), cams=cams, lead=lead,
                inputs=dict(jp=jp, jl=jl, obs_cam=obs_cam, lm_off=lm_off, cams=cams, H_extra=H_extra, lm_info=lm_info,
                            fixed=fixed, lead=lead))


def relative_jacobian(ci, cj, device_rot=True, fault=None):
    """A [6, 12] on (v_i, w_i, v_j, w_j) of the pair-prior residual at the mean equal to the current relative pose (rotations as
    the kernels build them from the stored quaternions when device_rot)"""
    Ri = cm.rotation(np.asarray(ci[:4], np.float64), device=device_rot)
    Rj = cm.rotation(np.asarray(cj[:4], np.float64), device=device_rot)
    M = Ri @ Rj.T
    t_rel = np.asarray(ci[4:7], np.float64) - M @ np.asarray(cj[4:7], np.float64)
    sj = 1.0 if fault == "aj_sign" else -1.0
    A = np.zeros((6, 12))
    A[0:3, 0:3] = np.eye(3)
    A[0:3, 3:6] = 0.0 if fault == "no_t_rel" else -cm.hat(t_rel)
    A[0:3, 6:9] = sj * M
    A[3:6, 3:6] = np.eye(3)
    A[3:6, 9:12] = sj * M
    return A


def _pose_index(i, j):
    return np.concatenate([9 * i + np.arange(6), 9 * j + np.arange(6)])


def _slot_pairs(lm_off, ls):
    """(request index, slot) of every slot of the landmarks ls [m]"""
    n = np.diff(lm_off)[ls]
    k = np.repeat(np.arange(len(ls)), n)
    s = np.asarray(lm_off)[ls][k] + (np.arange(n.sum()) - np.repeat(np.cumsum(n) - n, n))
    return k, s


def _sum_by(k, v, m):
    out = np.zeros((m,) + v.shape[1:])
    np.add.at(out, k, v)
    return out


def blocks(ref, cameras=None, camera_landmark=None, landmarks=None, relative=None, fault=None, chunk=1 << 16):
    """the four formulas for the requests ([m, 2] int arrays or None) from reference(): dict of [m, 9, 9], [m, 9, 3],
    [m, 3, 3], [m, 6, 6]; blocks of a landmark of rank < 3 are NaN.  fault: one of FAULTS."""
    if fault == "lm_prior_dropped":
        ref, fault = reference(**dict(ref["inputs"], lm_info=None)), None
    Sig, K, W, rank, obs_cam, lm_off = ref["Sig"], ref["K"], ref["W"], ref["rank"], ref["obs_cam"], ref["lm_off"]
    nc = Sig.shape[0] // 9
    if fault == "member_not_expanded" and ref["lead"] is not None:
        import shared_intrinsics_model as sim
        Sig = Sig.copy()
        mem = sim.members(ref["lead"])
        Sig[mem, :] = 0.0
        Sig[:, mem] = 0.0
    S4 = Sig.reshape(nc, 9, nc, 9)
    out = {}
    if cameras is not None:
        a, b = np.asarray(cameras).T
        out["cameras"] = S4[b, :, a, :] if fault == "transposed_cameras" else S4[a, :, b, :]
    if camera_landmark is not None:
        c, l = np.asarray(camera_landmark).T
        k, s = _slot_pairs(lm_off, l)
        if fault == "first_pass_only":
            first = s - lm_off[l[k]] < 32
            k, s = k[first], s[first]
        u = _sum_by(k, np.einsum("kpq,kjq->kpj", S4[c[k], :, obs_cam[s], :], K[s]), len(c))
        o = -np.einsum("kpj,krj->kpr", u, W[l])
        if fault == "cam_lm_sign":
            o = -o
        o[rank[l] < 3] = np.nan
        out["camera_landmark"] = o
    if landmarks is not None:
        lq, mq = np.asarray(landmarks).T
        n = np.diff(lm_off)
        X = np.zeros((len(lq), 3, 3))
        # slot pairs (i of l, j of m) of every request, in chunks
        cnt = n[lq] * n[mq]
        kk = np.repeat(np.arange(len(lq)), cnt)
        t = np.arange(cnt.sum()) - np.repeat(np.cumsum(cnt) - cnt, cnt)
        dec = n[lq][kk] if fault == "slot_pair_order" else n[mq][kk]
        si = np.minimum(lm_off[lq][kk] + t // dec, len(obs_cam) - 1)
        sj = np.minimum(lm_off[mq][kk] + t % dec, len(obs_cam) - 1)
        if fault == "first_pass_only":
            kk, si, sj = kk[t < 32], si[t < 32], sj[t < 32]
        for c0 in range(0, len(kk), chunk):
            sl = slice(c0, c0 + chunk)
            v = np.einsum("kap,kpq,kbq->kab", K[si[sl]], S4[obs_cam[si[sl]], :, obs_cam[sj[sl]], :], K[sj[sl]], optimize=True)
            np.add.at(X, kk[sl], v)
        same = (lq == mq) if fault != "identity_off_diagonal" else np.ones(len(lq), bool)
        X[same] += np.eye(3)
        o = np.einsum("kix,kxy,kjy->kij", W[mq] if fault == "w_swapped" else W[lq], X, W[mq])
        o[(rank[lq] < 3) | (rank[mq] < 3)] = np.nan
        out["landmarks"] = o
    if relative is not None:
        cams = ref["cams"]
        o = np.zeros((len(relative), 6, 6))
        for k, (i, j) in enumerate(np.asarray(relative)):
            A = relative_jacobian(cams[i], cams[j], fault=fault)
            idx = _pose_index(i, j)
            o[k] = A @ Sig[np.ix_(idx, idx)] @ A.T
        out["relative"] = o
    return out


def dense_rows(jp, jl, obs_cam, lm_off, nc):
    """the dense reprojection rows [Jp | Jl] of the per-observation blocks jp [nobs, 2, 9], jl [nobs, 2, 3]"""
    nobs, nl = len(obs_cam), len(lm_off) - 1
    Jp, Jl = np.zeros((2 * nobs, 9 * nc)), np.zeros((2 * nobs, 3 * nl))
    lm_of = np.repeat(np.arange(nl), np.diff(lm_off))
    for k in range(nobs):
        Jp[2 * k:2 * k + 2, 9 * obs_cam[k]:9 * obs_cam[k] + 9] = jp[k]
        Jl[2 * k:2 * k + 2, 3 * lm_of[k]:3 * lm_of[k] + 3] = jl[k]
    return Jp, Jl


def full_covariance(Jp, Jl, fixed=None, lead=None):
    """(F [9 nc + 3 nl, 9 nc + 3 nl], kappa, N): the covariance of the dense total system [Jp | Jl] from its definition, the
    held camera entries deleted (their rows and columns of F are 0) and, with intrinsics groups (lead), the tied parameters
    expanded (F = E inv(J_u^T J_u) E^T with J_u = [Jp P | Jl]); kappa = 2-norm condition of the equilibrated J_u^T J_u"""
    import shared_intrinsics_model as sim
    n9, nl3 = Jp.shape[1], Jl.shape[1]
    P = np.eye(n9) if lead is None else sim.expansion(lead)
    keep = np.arange(n9) if lead is None else np.flatnonzero(~sim.members(lead))
    fu = np.ones(len(keep), bool) if fixed is None else ~np.asarray(fixed, bool)[keep]
    J = np.hstack([(Jp @ P)[:, fu], Jl])
    H = J.T @ J
    d = 1.0 / np.sqrt(np.diag(H))
    Heq = H * d[:, None] * d[None, :]
    kappa = cvm.spd_cond(Heq)
    C = np.linalg.inv(Heq) * d[:, None] * d[None, :]
    E = np.zeros((n9 + nl3, J.shape[1]))
    E[:n9, :int(fu.sum())] = P[:, fu]
    E[n9:, int(fu.sum()):] = np.eye(nl3)
    return E @ C @ E.T, kappa, J.shape[1]


def dense_blocks(F, nc, cams, cameras=None, camera_landmark=None, landmarks=None, relative=None):
    """the requested blocks cut from a full covariance F [9 nc + 3 nl, 9 nc + 3 nl] (cameras first, then landmarks)"""
    cam = lambda a: 9 * a + np.arange(9)
    lmk = lambda l: 9 * nc + 3 * l + np.arange(3)
    out = {}
    if cameras is not None:
        out["cameras"] = np.stack([F[np.ix_(cam(a), cam(b))] for a, b in cameras])
    if camera_landmark is not None:
        out["camera_landmark"] = np.stack([F[np.ix_(cam(c), lmk(l))] for c, l in camera_landmark])
    if landmarks is not None:
        out["landmarks"] = np.stack([F[np.ix_(lmk(l), lmk(m))] for l, m in landmarks])
    if relative is not None:
        out["relative"] = np.stack([relative_jacobian(cams[i], cams[j]) @ F[np.ix_(_pose_index(i, j), _pose_index(i, j))]
                                    @ relative_jacobian(cams[i], cams[j]).T for i, j in relative])
    return out


def bar_scales(ref, requests):
    """per kind the entrywise magnitudes the blocks are bounded by with every Sigma entry replaced by sigma_p sigma_q (as
    covariance_model.landmark_bar_scale): sigma sigma^T (cameras), sigma_c (|W_l| g_l)^T (camera-landmark),
    |W_l| (delta_lm I + g_l g_m^T) |W_m|^T (landmarks), (|A| sigma_P)(|A| sigma_P)^T (relative), g_l = sum_i |K_i| sigma_{a_i}"""
    sig = ref["sigma"].reshape(-1, 9)
    s = sig[ref["obs_cam"]]
    g = np.add.reduceat(np.einsum("kij,kj->ki", np.abs(ref["K"]), s), ref["lm_off"][:-1], axis=0)
    Wa = np.abs(ref["W"])
    out = {}
    if requests.get("cameras") is not None:
        a, b = np.asarray(requests["cameras"]).T
        out["cameras"] = sig[a][:, :, None] * sig[b][:, None, :]
    if requests.get("camera_landmark") is not None:
        c, l = np.asarray(requests["camera_landmark"]).T
        out["camera_landmark"] = sig[c][:, :, None] * np.einsum("kij,kj->ki", Wa[l], g[l])[:, None, :]
    if requests.get("landmarks") is not None:
        l, m = np.asarray(requests["landmarks"]).T
        X = g[l][:, :, None] * g[m][:, None, :] + (l == m)[:, None, None] * np.eye(3)
        out["landmarks"] = np.einsum("kix,kxy,kjy->kij", Wa[l], X, Wa[m])
    if requests.get("relative") is not None:
        v = []
        for i, j in np.asarray(requests["relative"]):
            A = np.abs(relative_jacobian(ref["cams"][i], ref["cams"][j]))
            v.append(A @ ref["sigma"][_pose_index(i, j)])
        v = np.asarray(v)
        out["relative"] = v[:, :, None] * v[:, None, :]
    return out


def bars(ref, requests, c=8):
    """per kind the relative bar per request: c N kappa u, + c n kappa_l u for every landmark involved"""
    base = c * ref["N"] * ref["kappa"] * U
    n, kl = np.diff(ref["lm_off"]), ref["kappa_l"]
    lterm = lambda l: np.where(np.isfinite(kl[l]), n[l] * kl[l], 0.0) * c * U
    out = {}
    for key in KINDS:
        r = requests.get(key)
        if r is None:
            continue
        r = np.asarray(r)
        if key == "camera_landmark":
            out[key] = base + lterm(r[:, 1])
        elif key == "landmarks":
            out[key] = base + lterm(r[:, 0]) + lterm(r[:, 1])
        else:
            out[key] = np.full(len(r), base)
    return out


def excess(got, ref_blocks, ref, requests, c=8):
    """per kind max |got - ref| / (bar scale): <= 1 passes; NaN must be NaN in both (else inf).  Returns (dict, max bar)."""
    sc, br = bar_scales(ref, requests), bars(ref, requests, c)
    out, top = {}, 0.0
    for key in ref_blocks:
        g, r = np.asarray(got[key]), ref_blocks[key]
        nan_r = np.isnan(r).any(axis=(1, 2))
        if not np.array_equal(np.isnan(g).any(axis=(1, 2)), nan_r) or (nan_r & ~np.isnan(g).all(axis=(1, 2))).any():
            out[key] = np.inf
            continue
        ok = ~nan_r
        if not ok.any():
            out[key] = 0.0
            continue
        scale = br[key][ok][:, None, None] * np.maximum(sc[key][ok], np.finfo(float).tiny)
        out[key] = float(np.max(np.abs(g[ok] - r[ok]) / scale))
        top = max(top, float(br[key][ok].max()))
    return out, top


def check(got, ref_blocks, ref, requests, c=8, what=""):
    """assert every kind componentwise against the model (bars <= 1e-4)"""
    ex, top = excess(got, ref_blocks, ref, requests, c)
    assert top <= 1e-4, f"{what}: bar {top:.3g} above 1e-4 (kappa {ref['kappa']:.3g})"
    for key, v in ex.items():
        assert v <= 1.0, f"{what}: {key} off by {v:.3g} x its bar (kappa {ref['kappa']:.3g})"


def random_requests(rng, nc, nl, m, lm_ok=None):
    """m random requests of each kind (relative pairs with i != j)"""
    lm_pool = np.arange(nl) if lm_ok is None else np.flatnonzero(lm_ok)
    i = rng.integers(0, nc, m)
    j = (i + rng.integers(1, nc, m)) % nc
    return dict(cameras=rng.integers(0, nc, (m, 2)),
                camera_landmark=np.stack([rng.integers(0, nc, m), rng.choice(lm_pool, m)], 1),
                landmarks=rng.choice(lm_pool, (m, 2)),
                relative=np.stack([i, j], 1))
