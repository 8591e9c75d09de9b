"""Synthetic BAL problems with the shapes of BASELINE.json's configs.

No BAL file exists in the build container or on the GPU box (no network), so the
bench and the tests run on seeded synthetic stand-ins with matched
(num_cameras, num_landmarks, mean track length).  The generator follows the
spec in SURVEY.md section 8(d):

  cameras on a ring of radius 10 looking at the origin (+N(0, 0.05) rad jitter),
  f ~ U(500, 2000), k1 ~ N(0, 1e-7), k2 ~ N(0, 1e-13); landmarks ~ N(0, 3^2 I);
  track length n = 2 + Geometric(p = 1/(mean_n - 1)) truncated at min(Nc, 400);
  cameras per landmark uniform without replacement, sorted ascending (the
  std::map order of the reference, bal/bal_problem.hpp:137) -- `locality > 0` (used by the BASELINE-config stand-ins,
  synth_config) instead draws them from a window of `locality * n` consecutive camera indices, i.e. sequence-like
  visibility: uniformly random visibility is an expander graph whose reduced camera system is so well conditioned that
  PCG stops after 2-5 iterations, unlike any real BAL problem;
  observation = projection + N(0, 0.5^2) px; only z > 0.1 kept -- and, beyond that spec, only observations inside a
  +-45 degree field of view (|x/z|, |y/z| <= 1): without it a dense camera ring produces grazing observations with
  x/z ~ 1e2 whose r^4 distortion term dominates the whole cost (1e20 for the Final-13682 shape), which no real BAL
  file contains.

Internal conventions are the reference's *after loading* (bal/bal_problem.cpp:189-282):
camera looks along +z, image y points down, no minus sign in the projection;
camera state = (qx, qy, qz, qw, tx, ty, tz, f, k1, k2) (bal/bal_problem.hpp:84-89).
`write_bal` emits the on-disk BAL convention (inverse of the loader's axis flip)
so that the text loaders are exercised as well.
"""
from __future__ import annotations

import dataclasses

import numpy as np

# (num_cameras, num_landmarks, mean track length) -- scripts/num_ops/bal_numbers.csv:1-5
CONFIGS = {
    "ladybug-49": (49, 7776, 31843 / 7776),
    "ladybug-1723": (1723, 156502, 678718 / 156502),
    "trafalgar-257": (257, 65132, 225911 / 65132),
    "venice-1778": (1778, 993923, 5001946 / 993923),
    "final-13682": (13682, 4456117, 28987644 / 4456117),
}


@dataclasses.dataclass
class BalArrays:
    """SoA view of a BalProblem (double precision)."""

    cams: np.ndarray      # [nc, 10] float64
    lms: np.ndarray       # [nl, 3] float64
    lm_off: np.ndarray    # [nl + 1] int64
    obs_cam: np.ndarray   # [nobs] int32, ascending inside each landmark
    obs_xy: np.ndarray    # [nobs, 2] float64

    @property
    def nc(self) -> int:
        return int(self.cams.shape[0])

    @property
    def nl(self) -> int:
        return int(self.lms.shape[0])

    @property
    def nobs(self) -> int:
        return int(self.obs_cam.shape[0])

    def track_lengths(self) -> np.ndarray:
        return np.diff(self.lm_off).astype(np.int64)

    def stats(self) -> dict:
        n = self.track_lengths()
        return {
            "num_cameras": self.nc, "num_landmarks": self.nl, "num_observations": self.nobs,
            "mean_n": float(n.mean()), "max_n": int(n.max()), "sum_n2": int((n * n).sum()),
        }

    def cast(self, dtype) -> "BalArrays":
        return BalArrays(self.cams.astype(dtype), self.lms.astype(dtype), self.lm_off.copy(),
                         self.obs_cam.copy(), self.obs_xy.astype(dtype))


def quat_to_rot(q: np.ndarray) -> np.ndarray:
    """(x, y, z, w) unit quaternions [..., 4] -> rotation matrices [..., 3, 3]."""
    x, y, z, w = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    R = np.empty(q.shape[:-1] + (3, 3), dtype=q.dtype)
    R[..., 0, 0] = 1 - 2 * (y * y + z * z)
    R[..., 0, 1] = 2 * (x * y - z * w)
    R[..., 0, 2] = 2 * (x * z + y * w)
    R[..., 1, 0] = 2 * (x * y + z * w)
    R[..., 1, 1] = 1 - 2 * (x * x + z * z)
    R[..., 1, 2] = 2 * (y * z - x * w)
    R[..., 2, 0] = 2 * (x * z - y * w)
    R[..., 2, 1] = 2 * (y * z + x * w)
    R[..., 2, 2] = 1 - 2 * (x * x + y * y)
    return R


def rot_to_quat(R: np.ndarray) -> np.ndarray:
    from scipy.spatial.transform import Rotation
    q = Rotation.from_matrix(R).as_quat()  # x, y, z, w
    q = np.atleast_2d(q)
    q[q[:, 3] < 0] *= -1
    return q


def so3_exp(w: np.ndarray) -> np.ndarray:
    """Rotation vectors [..., 3] -> quaternions (x, y, z, w)."""
    th = np.linalg.norm(w, axis=-1, keepdims=True)
    half = 0.5 * th
    with np.errstate(invalid="ignore", divide="ignore"):
        k = np.where(th > 1e-12, np.sin(half) / th, 0.5 - th * th / 48.0)
    return np.concatenate([k * w, np.cos(half)], axis=-1)


def project(cams: np.ndarray, p_w: np.ndarray, return_tan: bool = False):
    """Snavely projection in the loaded convention.  cams [m, 10], p_w [m, 3] -> (xy [m, 2], z [m])."""
    R = quat_to_rot(cams[:, :4])
    pc = np.einsum("mij,mj->mi", R, p_w) + cams[:, 4:7]
    z = pc[:, 2]
    with np.errstate(divide="ignore", invalid="ignore"):
        m = pc[:, :2] / z[:, None]
    r2 = (m * m).sum(axis=1)
    rp = 1.0 + cams[:, 8] * r2 + cams[:, 9] * r2 * r2
    xy = cams[:, 7:8] * rp[:, None] * m
    if return_tan:
        return xy, z, np.abs(m).max(axis=1)
    return xy, z


def _sample_tracks_local(rng: np.random.Generator, nc: int, n: np.ndarray, window_factor: float) -> np.ndarray:
    """Sequence-like visibility (what a vehicle-mounted Ladybug rig produces): landmark l is seen by n[l] distinct cameras
    drawn from a window of ~window_factor * n[l] consecutive camera indices around a random centre (wrapping)."""
    total = int(n.sum())
    off = np.concatenate([[0], np.cumsum(n)])
    out = np.empty(total, dtype=np.int32)
    for k in np.unique(n):
        idx = np.nonzero(n == k)[0]
        m = idx.size
        w = int(min(nc, max(k, round(window_factor * k))))
        centre = rng.integers(0, nc, size=m)
        keys = rng.random((m, w))
        rel = np.argsort(keys, axis=1)[:, :k]                      # k distinct offsets inside the window
        sel = ((centre[:, None] + rel - w // 2) % nc).astype(np.int32)
        sel.sort(axis=1)
        pos = (off[idx][:, None] + np.arange(k)[None, :]).ravel()
        out[pos] = sel.ravel()
    return out


def _sample_tracks(rng: np.random.Generator, nc: int, n: np.ndarray) -> np.ndarray:
    """For each landmark l sample n[l] distinct cameras in [0, nc), sorted ascending; flat array."""
    total = int(n.sum())
    off = np.concatenate([[0], np.cumsum(n)])
    out = np.empty(total, dtype=np.int32)
    for k in np.unique(n):
        idx = np.nonzero(n == k)[0]
        m = idx.size
        if k > nc // 4:
            keys = rng.random((m, nc))
            sel = np.argsort(keys, axis=1)[:, :k].astype(np.int32)
        else:
            sel = rng.integers(0, nc, size=(m, k), dtype=np.int32)
            for _ in range(64):
                sel.sort(axis=1)
                dup = np.zeros_like(sel, dtype=bool)
                dup[:, 1:] = sel[:, 1:] == sel[:, :-1]
                nd = int(dup.sum())
                if nd == 0:
                    break
                sel[dup] = rng.integers(0, nc, size=nd, dtype=np.int32)
        sel.sort(axis=1)
        pos = (off[idx][:, None] + np.arange(k)[None, :]).ravel()
        out[pos] = sel.ravel()
    return out


def synth_bal(nc: int, nl: int, mean_n: float, seed: int = 38401, *, max_track: int = 400, max_tan: float = 1.0,
              locality: float = 0.0, track_lengths=None, lm_spread: float = 3.0,
              obs_noise: float = 0.5, perturb_lm: float = 0.05, perturb_rot: float = 0.002,
              perturb_trans: float = 0.01, normalize_scale: float | None = 100.0, k1_sigma: float = 1e-7,
              k2_sigma: float = 1e-13, tracks=None) -> BalArrays:
    """Generate a synthetic BAL problem (already in the loaded convention), optionally normalised
    like the reference's default pipeline (bal/bal_problem.cpp:428-469, scale 100) and with a
    perturbed initial state so that LM has real work to do.

    `track_lengths` (one entry per landmark, each in [2, nc]) replaces the geometric draw of the track lengths: landmark l
    gets exactly track_lengths[l] observations (`nl` must equal its length, `mean_n` and `max_track` are not used).  Pair it
    with a small `lm_spread` (standard deviation of the landmark positions; the cameras stand at distance ~10) so that every
    landmark lies inside every camera's field of view and no observation is filtered; a filtered one raises ValueError.

    `tracks` (one sequence of distinct camera indices per landmark) goes one step further and names the cameras of every
    landmark; it implies the track lengths and the same no-filtering rule.  `k1_sigma` / `k2_sigma` are the standard
    deviations of the radial distortion coefficients (the defaults make distortion negligible, as in the spec above; real
    photo-collection cameras have |k1| up to ~0.5).  With the defaults of every option the output is unchanged."""
    if tracks is not None:
        tracks = [np.unique(np.asarray(t, dtype=np.int64)) for t in tracks]
        track_lengths = [len(t) for t in tracks]
        if any(t.size and (t[0] < 0 or t[-1] >= nc) for t in tracks):
            raise ValueError(f"camera indices of tracks must lie in [0, nc = {nc})")
    if track_lengths is not None:
        want = np.asarray(track_lengths, dtype=np.int64).ravel()
        if want.shape[0] != nl:
            raise ValueError(f"track_lengths has {want.shape[0]} entries for nl = {nl} landmarks")
        if want.size and (want.min() < 2 or want.max() > nc):
            raise ValueError(f"track lengths must lie in [2, nc = {nc}]")
    rng = np.random.default_rng(seed)
    # cameras on a ring of radius 10 looking at the origin
    ang = rng.uniform(0.0, 2 * np.pi, nc)
    if locality > 0:
        ang = np.sort(ang)  # camera index follows the trajectory
    C = np.stack([10 * np.cos(ang), 10 * np.sin(ang), rng.normal(0, 0.5, nc)], axis=1)
    zc = -C / np.linalg.norm(C, axis=1, keepdims=True)
    up = np.array([0.0, 0.0, 1.0])
    xc = np.cross(zc, up)
    xc /= np.linalg.norm(xc, axis=1, keepdims=True)
    yc = np.cross(zc, xc)
    R = np.stack([xc, yc, zc], axis=1)  # rows = camera axes in world => world->cam
    jitter = quat_to_rot(so3_exp(rng.normal(0, 0.05, (nc, 3))))
    R = np.einsum("mij,mjk->mik", jitter, R)
    t = -np.einsum("mij,mj->mi", R, C)
    cams = np.empty((nc, 10))
    cams[:, :4] = rot_to_quat(R)
    cams[:, 4:7] = t
    cams[:, 7] = rng.uniform(500, 2000, nc)
    cams[:, 8] = rng.normal(0, k1_sigma, nc)
    cams[:, 9] = rng.normal(0, k2_sigma, nc)
    # landmarks and track lengths
    lms = rng.normal(0, lm_spread, (nl, 3))
    if track_lengths is None:
        p = 1.0 / (mean_n - 1.0)
        n = 2 + (rng.geometric(p, nl) - 1)
        n = np.minimum(n, min(nc, max_track)).astype(np.int64)
    else:
        n = want
    if tracks is not None:
        obs_cam = np.concatenate(tracks).astype(np.int32) if tracks else np.empty(0, np.int32)
    else:
        obs_cam = _sample_tracks_local(rng, nc, n, locality) if locality > 0 else _sample_tracks(rng, nc, n)
    lm_of_obs = np.repeat(np.arange(nl), n)
    xy, z, tan = project(cams[obs_cam], lms[lm_of_obs], return_tan=True)
    xy = xy + rng.normal(0, obs_noise, xy.shape)
    keep = (z > 0.1) & (tan <= max_tan)
    # drop bad observations, then landmarks with < 2 observations (QR needs n >= 2, ipp:73-76)
    n_keep = np.bincount(lm_of_obs[keep], minlength=nl)
    lm_ok = n_keep >= 2
    keep &= lm_ok[lm_of_obs]
    obs_cam, xy, lm_of_obs = obs_cam[keep], xy[keep], lm_of_obs[keep]
    new_id = np.cumsum(lm_ok) - 1
    lm_of_obs = new_id[lm_of_obs]
    lms = lms[lm_ok]
    nl2 = lms.shape[0]
    counts = np.bincount(lm_of_obs, minlength=nl2)
    lm_off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    prob = BalArrays(cams, lms, lm_off, obs_cam.astype(np.int32), xy)
    if track_lengths is not None and not np.array_equal(prob.track_lengths(), want):
        raise ValueError(f"{int(want.sum()) - prob.nobs} observations fell outside the field of view or behind a camera; "
                         "use a smaller lm_spread")
    if normalize_scale:
        normalize(prob, normalize_scale)
    # perturb the initial state (relative to the normalised scale)
    s = (normalize_scale or 100.0) / 100.0
    if perturb_lm > 0:
        prob.lms += rng.normal(0, perturb_lm * s, prob.lms.shape)
    if perturb_rot > 0 or perturb_trans > 0:
        Rc = quat_to_rot(prob.cams[:, :4])
        dR = quat_to_rot(so3_exp(rng.normal(0, perturb_rot, (nc, 3))))
        Rn = np.einsum("mij,mjk->mik", dR, Rc)
        ctr = -np.einsum("mji,mj->mi", Rc, prob.cams[:, 4:7])
        ctr = ctr + rng.normal(0, perturb_trans * s, ctr.shape)
        prob.cams[:, :4] = rot_to_quat(Rn)
        prob.cams[:, 4:7] = -np.einsum("mij,mj->mi", Rn, ctr)
    return prob


def turn_cameras_around(prob: BalArrays, cams) -> BalArrays:
    """A copy of `prob` in which the chosen cameras are turned by 180 degrees about their own y axis (pc -> (-x, y, -z)):
    every landmark they saw in front of them now lies behind them, at the same distance, so their observations become
    invalid projections while the observed pixel values stay as they were."""
    idx = np.atleast_1d(np.asarray(cams, dtype=np.int64))
    flip = np.diag([-1.0, 1.0, -1.0])
    out = BalArrays(prob.cams.copy(), prob.lms.copy(), prob.lm_off.copy(), prob.obs_cam.copy(), prob.obs_xy.copy())
    R = np.einsum("ij,mjk->mik", flip, quat_to_rot(prob.cams[idx, :4]))
    out.cams[idx, :4] = rot_to_quat(R)
    out.cams[idx, 4:7] = prob.cams[idx, 4:7] @ flip.T
    return out


def synth_config(name: str, seed: int = 38401, scale: float = 1.0, **kw) -> BalArrays:
    """Synthetic stand-in for one of BASELINE.json's configs; `scale` shrinks cameras and landmarks
    proportionally (used by the fast tests)."""
    nc, nl, mean_n = CONFIGS[name]
    nc = max(4, int(round(nc * scale)))
    nl = max(8, int(round(nl * scale)))
    # Ladybug is a vehicle-mounted capture: a track lives in a window of consecutive frames (sequence-like visibility,
    # which is what makes the reduced camera system ill-conditioned and PCG take tens of iterations).  The photo-collection
    # sets (Trafalgar, Venice, Final) are clustered but less strictly sequential.
    kw.setdefault("locality", 2.0 if name.startswith("ladybug") else 6.0)
    return synth_bal(nc, nl, mean_n, seed, **kw)


def normalize(prob: BalArrays, new_scale: float = 100.0) -> None:
    """In-place normalisation, bal/bal_problem.cpp:428-469 (median via nth_element at n/2)."""
    nl = prob.nl
    med = np.array([np.partition(prob.lms[:, j], nl // 2)[nl // 2] for j in range(3)])
    l1 = np.abs(prob.lms - med).sum(axis=1)
    mad = np.partition(l1, nl // 2)[nl // 2]
    scale = new_scale / mad
    prob.lms[:] = scale * (prob.lms - med)
    R = quat_to_rot(prob.cams[:, :4])
    ctr = -np.einsum("mji,mj->mi", R, prob.cams[:, 4:7])
    ctr = scale * (ctr - med)
    prob.cams[:, 4:7] = -np.einsum("mij,mj->mi", R, ctr)


def write_bal(prob: BalArrays, path: str) -> None:
    """Write the on-disk BAL text format (inverse of the loader's conversion,
    bal/bal_problem.cpp:243-258): y of the image and y, z of the camera frame are flipped back."""
    from scipy.spatial.transform import Rotation
    flip = np.diag([1.0, -1.0, -1.0])
    R = quat_to_rot(prob.cams[:, :4])
    Rb = np.einsum("ij,mjk->mik", flip, R)
    rv = Rotation.from_matrix(Rb).as_rotvec()
    tb = prob.cams[:, 4:7] @ flip.T
    lm_of_obs = np.repeat(np.arange(prob.nl), np.diff(prob.lm_off))
    with open(path, "w") as f:
        f.write(f"{prob.nc} {prob.nl} {prob.nobs}\n")
        for c, l, (x, y) in zip(prob.obs_cam, lm_of_obs, prob.obs_xy):
            f.write(f"{c} {l} {x:.17g} {-y:.17g}\n")
        for i in range(prob.nc):
            for v in (*rv[i], *tb[i], *prob.cams[i, 7:10]):
                f.write(f"{v:.17g}\n")
        for i in range(prob.nl):
            for v in prob.lms[i]:
                f.write(f"{v:.17g}\n")


@dataclasses.dataclass
class RigCapture:
    """A synthetic capture of a rigid multi-camera body (synth_rig_capture) and its truth."""

    prob: BalArrays          # the true cameras and landmarks, noise-free observations (nothing perturbed)
    rig: np.ndarray          # [nc] int32 placement (rig id) of each camera: camera f * K + k is sensor k at placement f
    sensor: np.ndarray       # [nc] int32 sensor of each camera
    cam_from_rig: np.ndarray  # [nc, 7] the true extrinsics of each camera's sensor (qx,qy,qz,qw, tx,ty,tz)
    rig_from_world: np.ndarray  # [F, 7] the true pose of every placement


def synth_rig_capture(num_sensors: int, num_placements: int, num_landmarks: int, seed: int = 38401, *,
                      radius: float = 0.15, step: float = 0.6, focal: float = 500.0, max_tan: float = 0.9,
                      max_depth: float = 12.0) -> RigCapture:
    """A seeded rig capture: `num_sensors` cameras on a ring of `radius` around the rig's origin, looking outward and evenly
    spread in yaw (a spherical head), placed `num_placements` times along a gently curving path with `step` between
    placements, and landmarks scattered 3 to 15 units beside the path.  Every landmark keeps the cameras it lies in front of,
    at a depth below max_depth and within |x/z|, |y/z| <= max_tan; landmarks seen fewer than twice are dropped.  Returns the truth; perturb it to test."""
    rng = np.random.default_rng(seed)
    K, F = num_sensors, num_placements
    # sensor k: yaw 2 pi k / K (+ a little tilt), centre on the ring; camera axes as rows (rig -> camera rotation)
    E = np.zeros((K, 7))
    for k in range(K):
        yaw = 2 * np.pi * k / K + rng.normal(0, 0.02)
        zc = np.array([np.cos(yaw), np.sin(yaw), rng.normal(0, 0.05)])
        zc /= np.linalg.norm(zc)
        xc = np.cross(zc, [0.0, 0.0, 1.0])
        xc /= np.linalg.norm(xc)
        yc = np.cross(zc, xc)
        R = np.stack([xc, yc, zc])
        c = radius * np.array([np.cos(yaw), np.sin(yaw), 0.0]) + rng.normal(0, 0.01, 3)
        E[k, :4] = rot_to_quat(R)[0]
        E[k, 4:] = -R @ c
    # placements along the path: rig origin p_f, heading following the path
    s = step * np.arange(F)
    P = np.stack([s, 2.0 * np.sin(s / 15.0), 0.1 * np.sin(s / 4.0)], axis=1)
    head = np.arctan2(np.gradient(P[:, 1]), np.gradient(P[:, 0]))
    T = np.zeros((F, 7))
    for f in range(F):
        ch, sh = np.cos(head[f]), np.sin(head[f])
        R = np.array([[ch, sh, 0.0], [-sh, ch, 0.0], [0.0, 0.0, 1.0]])  # world -> rig
        T[f, :4] = rot_to_quat(R)[0]
        T[f, 4:] = -R @ P[f]
    # cameras T_c = E_k T_f
    nc = K * F
    cams = np.zeros((nc, 10))
    cams[:, 7] = focal
    for f in range(F):
        Rf = quat_to_rot(T[f, :4])
        for k in range(K):
            Rk = quat_to_rot(E[k, :4])
            c = f * K + k
            cams[c, :4] = rot_to_quat(Rk @ Rf)[0]
            cams[c, 4:7] = Rk @ T[f, 4:] + E[k, 4:]
    # landmarks beside the path
    i = rng.integers(0, F, num_landmarks)
    dist = rng.uniform(3.0, 15.0, num_landmarks)
    ang = rng.uniform(0, 2 * np.pi, num_landmarks)
    lms = P[i] + np.stack([dist * np.cos(ang), dist * np.sin(ang), rng.normal(0, 2.0, num_landmarks)], axis=1)
    obs_cam, lm_of, xy = [], [], []
    for lo in range(0, num_landmarks, 4096):  # visibility in chunks of landmarks
        l = np.arange(lo, min(lo + 4096, num_landmarks))
        R = quat_to_rot(cams[:, :4])
        pc = np.einsum("cij,lj->lci", R, lms[l]) + cams[None, :, 4:7]
        z = pc[..., 2]
        with np.errstate(divide="ignore", invalid="ignore"):
            m = pc[..., :2] / z[..., None]
        vis = (z > 0.5) & (z < max_depth) & (np.abs(m).max(axis=-1) <= max_tan)
        ll, cc = np.nonzero(vis)
        obs_cam.append(cc)
        lm_of.append(l[ll])
    obs_cam, lm_of = np.concatenate(obs_cam), np.concatenate(lm_of)
    n = np.bincount(lm_of, minlength=num_landmarks)
    ok = n >= 2
    keep = ok[lm_of]
    obs_cam, lm_of = obs_cam[keep], lm_of[keep]
    new_id = np.cumsum(ok) - 1
    lm_of = new_id[lm_of]
    order = np.lexsort((obs_cam, lm_of))
    obs_cam, lm_of = obs_cam[order].astype(np.int32), lm_of[order]
    lms = lms[ok]
    xy, _ = project(cams[obs_cam], lms[lm_of])
    lm_off = np.concatenate([[0], np.cumsum(np.bincount(lm_of, minlength=lms.shape[0]))]).astype(np.int64)
    rig = np.repeat(np.arange(F), K).astype(np.int32)
    sensor = np.tile(np.arange(K), F).astype(np.int32)
    return RigCapture(BalArrays(cams, lms, lm_off, obs_cam, xy), rig, sensor, E[sensor].copy(), T)
