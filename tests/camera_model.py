"""An independent float64 model of one observation: Snavely projection, its Jacobians, validity and the Huber weight.

Written from the mathematics, not from the oracle or the kernel, so that a mistake both of those share (they state the same
formula line for line) shows up as a disagreement with this model.  Conventions are the loaded ones (DESIGN.md, synthetic.py):

  pc  = R(q) p + t                      camera frame, the camera looks along +z
  m   = pc[:2] / z,  r2 = |m|^2,  rp = 1 + k1 r2 + k2 r2^2
  res = f rp m - obs
  pose increment (translation first), left-multiplied like camera_apply_inc / k_camera_update:
      T <- (Exp(w), v) T,  so  pc <- Exp(w) pc + v,   d pc / d v = I,  d pc / d w = -[pc]x
  Jp  = (d proj / d pc) [I | -[pc]x]      (2 x 6)
  Ji  = (m rp, f m r2, f m r2^2)          (2 x 3, columns f, k1, k2)
  Jl  = (d proj / d pc) R                 (2 x 3)
  d proj / d pc = f (rp I + 2 (k1 + 2 k2 r2) m m^T) (d m / d pc),  d m / d pc = [I | -m] / z

Validity: z >= sqrt(eps_S) (Sophus' epsilon of the scalar type).  Huber with threshold d:  rho(s) = s / 2 for |r| <= d,
d |r| - d^2 / 2 beyond, weight min(1, d / |r|).  Every function takes arrays of observations and computes in float64;
inputs of another type are cast exactly first.
"""
import numpy as np

# Sophus::Constants<S>::epsilon() and its square root: ST<S>::eps_sqrt() (rootba_b200/csrc/kernels.cuh) and
# sophus_epsilon_sqrt<S>() (oracle/rootba_oracle.hpp), the validity threshold of a projection and the default
# Jacobian-scaling epsilon.  tests/test_camera_model.py checks that the sources still state these values.
EPS = {np.dtype(np.float32): np.float32(1e-5), np.dtype(np.float64): np.float64(1e-10)}
EPS_SQRT = {np.dtype(np.float32): np.float32(0.0031622776601683794), np.dtype(np.float64): np.float64(1e-5)}


def rotation(q, device=False):
    """unit quaternions (x, y, z, w) [..., 4] -> rotation matrices: R = (w^2 - |v|^2) I + 2 v v^T + 2 w [v]x.

    device=True evaluates the form the kernels use (Eigen's Quaternion::toRotationMatrix), R = I + 2 w [v]x + 2 [v]x^2, on
    the quaternion as stored: the two agree for a unit quaternion, and for a float32 quaternion whose norm is 1 + O(2^-24)
    only the device form is the matrix the kernels actually apply."""
    q = np.asarray(q, dtype=np.float64)
    v, w = q[..., :3], q[..., 3]
    if device:
        K = hat(v)
        return np.eye(3) + 2 * w[..., None, None] * K + 2 * K @ K
    R = (w * w - (v * v).sum(-1))[..., None, None] * np.eye(3) + 2 * v[..., :, None] * v[..., None, :]
    return R + 2 * w[..., None, None] * hat(v)


def hat(v):
    """[v]x, so that hat(a) @ b = a x b"""
    v = np.asarray(v, dtype=np.float64)
    H = np.zeros(v.shape[:-1] + (3, 3))
    H[..., 0, 1], H[..., 0, 2] = -v[..., 2], v[..., 1]
    H[..., 1, 0], H[..., 1, 2] = v[..., 2], -v[..., 0]
    H[..., 2, 0], H[..., 2, 1] = -v[..., 1], v[..., 0]
    return H


def camera_point(cams, p):
    cams = np.asarray(cams, dtype=np.float64)
    return np.einsum("mij,mj->mi", rotation(cams[:, :4]), np.asarray(p, dtype=np.float64)) + cams[:, 4:7]


def project_pc(pc, intr):
    """pc [m, 3], intr [m, 3] (f, k1, k2) -> pixel [m, 2]"""
    m = pc[:, :2] / pc[:, 2:3]
    r2 = (m * m).sum(1)
    rp = 1 + intr[:, 1] * r2 + intr[:, 2] * r2 * r2
    return (intr[:, 0] * rp)[:, None] * m


def linearize(cams, p, obs, dtype=np.float64, device_rot=False):
    """per observation: residual [m, 2], Jp [m, 2, 6], Ji [m, 2, 3], Jl [m, 2, 3], pc [m, 3], valid [m] (z >= sqrt(eps) of
    `dtype`).  Nothing is filtered: invalid observations get their (finite or not) values too.  device_rot: R as the kernels
    build it (rotation(device=True))."""
    cams = np.asarray(cams, dtype=np.float64).reshape(-1, 10)
    obs = np.asarray(obs, dtype=np.float64).reshape(-1, 2)
    R = rotation(cams[:, :4], device=device_rot)
    pc = np.einsum("mij,mj->mi", R, np.asarray(p, dtype=np.float64).reshape(-1, 3)) + cams[:, 4:7]
    f, k1, k2 = cams[:, 7], cams[:, 8], cams[:, 9]
    z = pc[:, 2]
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        m = pc[:, :2] / z[:, None]
        r2 = (m * m).sum(1)
        rp = 1 + k1 * r2 + k2 * r2 * r2
        res = (f * rp)[:, None] * m - obs
        dm_dpc = np.zeros((len(z), 2, 3))
        dm_dpc[:, 0, 0] = dm_dpc[:, 1, 1] = 1 / z
        dm_dpc[:, :, 2] = -m / z[:, None]
        dproj_dm = f[:, None, None] * (rp[:, None, None] * np.eye(2)
                                       + 2 * (k1 + 2 * k2 * r2)[:, None, None] * m[:, :, None] * m[:, None, :])
        dproj_dpc = dproj_dm @ dm_dpc
        dpc_dpose = np.concatenate([np.broadcast_to(np.eye(3), (len(z), 3, 3)), -hat(pc)], axis=2)
        Jp = dproj_dpc @ dpc_dpose
        Ji = np.stack([rp[:, None] * m, f[:, None] * r2[:, None] * m, f[:, None] * (r2 * r2)[:, None] * m], axis=2)
        Jl = dproj_dpc @ R
    valid = z >= float(EPS_SQRT[np.dtype(dtype)])
    return {"res": res, "Jp": Jp, "Ji": Ji, "Jl": Jl, "pc": pc, "valid": valid}


def huber(rsq, threshold=None):
    """(error, weight) of squared residual norms; threshold None = plain squared loss"""
    rsq = np.asarray(rsq, dtype=np.float64)
    if threshold is None:
        return 0.5 * rsq, np.ones_like(rsq)
    r = np.sqrt(rsq)
    inside = r <= threshold
    with np.errstate(divide="ignore"):
        err = np.where(inside, 0.5 * rsq, threshold * r - 0.5 * threshold * threshold)
        w = np.where(inside, 1.0, threshold / r)
    return err, w


def observations(arrays):
    """(camera rows, landmark rows, observed pixels) of every observation of a BalArrays-like problem, in storage order"""
    lm_of_obs = np.repeat(np.arange(arrays.lms.shape[0]), np.diff(arrays.lm_off))
    return (np.asarray(arrays.cams)[arrays.obs_cam], np.asarray(arrays.lms)[lm_of_obs], np.asarray(arrays.obs_xy))


def compute_error(arrays, dtype=np.float64, threshold=None):
    """the sums of compute_error: {"all"|"valid": {num_obs, error, residual_sum}}, validity of `dtype`"""
    L = linearize(*observations(arrays), dtype=dtype)
    rsq = (L["res"] ** 2).sum(1)
    err, _ = huber(rsq, threshold)
    out = {}
    for key, sel in (("all", np.ones(len(rsq), bool)), ("valid", L["valid"])):
        out[key] = {"num_obs": int(sel.sum()), "error": float(err[sel].sum()), "residual_sum": float(np.sqrt(rsq[sel]).sum())}
    return out


def condition(arrays, dtype=np.float64, threshold=None):
    """per observation, the factor by which rounding in the inputs' type is amplified in the weighted rows:
    kappa_pc = (|R| |p| + |t|) / |pc| (cancellation in R p + t), kappa_rp = (1 + |k1| r2 + |k2| r2^2) / |rp| (cancellation in
    the distortion factor) and, where the Huber weight d / |r| is active, 1 + (|proj| + |obs|) / |r| (a residual is the
    difference of two pixel positions, the weight divides by it)"""
    cams, p, obs = observations(arrays)
    cams, p = np.asarray(cams, np.float64), np.asarray(p, np.float64)
    L = linearize(cams, p, obs, dtype=dtype)
    pc = L["pc"]
    k = (np.einsum("mij,mj->mi", np.abs(rotation(cams[:, :4])), np.abs(p)).max(1) + np.abs(cams[:, 4:7]).max(1)) / np.abs(pc).max(1)
    m = pc[:, :2] / pc[:, 2:3]
    r2 = (m * m).sum(1)
    k *= (1 + np.abs(cams[:, 8]) * r2 + np.abs(cams[:, 9]) * r2 * r2) / np.abs(1 + cams[:, 8] * r2 + cams[:, 9] * r2 * r2)
    if threshold is not None:
        rn = np.sqrt((L["res"] ** 2).sum(1))
        k = np.where(rn > threshold, k * (1 + (np.abs(L["res"] + obs) + np.abs(obs)).max(1) / rn), k)
    return k


def weighted(arrays, dtype=np.float64, threshold=None, valid_only=False, magnitude=False, device_rot=False):
    """per observation sqrt(w) Jp (2 x 9: pose then intrinsics), sqrt(w) Jl, sqrt(w) res and the row mask (0 for an
    observation that use_valid_projections_only drops) -- the unscaled rows of the landmark blocks.  magnitude=True appends
    sqrt(w) (|proj| + |obs|), the scale of the rounding error of a residual computed as proj - obs.  device_rot: see
    linearize."""
    cams, p, obs = observations(arrays)
    L = linearize(cams, p, obs, dtype=dtype, device_rot=device_rot)
    _, w = huber((L["res"] ** 2).sum(1), threshold)
    keep = L["valid"] if valid_only else np.ones(len(w), bool)
    sw = np.where(keep, np.sqrt(w), 0.0)[:, None]
    with np.errstate(invalid="ignore"):
        Jp = np.concatenate([L["Jp"], L["Ji"]], axis=2) * sw[:, :, None]
        Jl = L["Jl"] * sw[:, :, None]
        r = L["res"] * sw
        mag = (np.abs(L["res"] + obs) + np.abs(obs)) * sw
    Jp[~keep], Jl[~keep], r[~keep], mag[~keep] = 0.0, 0.0, 0.0, 0.0
    return (Jp, Jl, r, keep, mag) if magnitude else (Jp, Jl, r, keep)
