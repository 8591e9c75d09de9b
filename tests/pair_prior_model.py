"""An independent float64 model of the relative pose prior between two cameras (rba_set_camera_pair_prior, DESIGN.md
section 15).

Written from the mathematics, not from the kernel: the rotation residual goes through scipy's rotation-vector logarithm of
the rotation matrix R_i R_j^T R0^T (the kernel takes the logarithm of a quaternion product), and J_l^-1 is the numerical
inverse of the closed-form left Jacobian (camera_prior_model.left_jacobian).

  poses world -> camera, T = [R | t];  pair (i, j) with mean Z = (R0, t0) meaning T_i T_j^-1 ~ Z
  e_t = t_i - R_i R_j^T t_j - t0,  e_r = Log(R_i R_j^T R0^T),  cost 1/2 |L (e_t, e_r)|^2
  increment (v, w, ...) as camera_model / k_camera_update:  R' = Exp(w) R,  t' = Exp(w) t + v
  with M = R_i R_j^T, t_rel = t_i - M t_j, phi = e_r:
    de/d(inc_i) = [[I, -[t_rel]x], [0, J_l^-1(phi)]],  de/d(inc_j) = [[-M, 0], [0, -J_l^-1(phi) M]]  (zero intrinsic columns)
"""
import numpy as np
from scipy.spatial.transform import Rotation

import camera_model as cm
import camera_prior_model as pm


def _rot(cam, device_rot=False):
    """R of a camera: of its normalised quaternion, or (device_rot) as the kernels build it from the stored quaternion"""
    cam = np.asarray(cam, np.float64)
    return cm.rotation(cam[:4], device=True) if device_rot else cm.rotation(cam[:4] / np.linalg.norm(cam[:4]))


def residual(ci, cj, mean, device_rot=False):
    """e [6] of one pair: cameras ci, cj [10], mean [7] (qx,qy,qz,qw of R0, t0).  device_rot: M = R_i R_j^T of the kernels'
    rotation matrices in e_t; the logarithm is that of the normalised quaternions either way (camera_prior_model.residual)."""
    ci, cj, mean = (np.asarray(a, np.float64) for a in (ci, cj, mean))
    Ri, Rj, R0 = _rot(ci), _rot(cj), cm.rotation(mean[:4] / np.linalg.norm(mean[:4]))
    Md = _rot(ci, device_rot) @ _rot(cj, device_rot).T
    return np.concatenate([ci[4:7] - Md @ cj[4:7] - mean[4:7], pm.log_so3(Ri @ Rj.T @ R0.T)])


def jacobians(ci, cj, mean, device_rot=False):
    """de/d(inc_i), de/d(inc_j) [6, 9] each at the cameras"""
    ci, cj = np.asarray(ci, np.float64), np.asarray(cj, np.float64)
    M = _rot(ci, device_rot) @ _rot(cj, device_rot).T
    t_rel = ci[4:7] - M @ cj[4:7]
    Jinv = np.linalg.inv(pm.left_jacobian(residual(ci, cj, mean)[3:6]))
    Ji, Jj = np.zeros((6, 9)), np.zeros((6, 9))
    Ji[0:3, 0:3] = np.eye(3)
    Ji[0:3, 3:6] = -cm.hat(t_rel)
    Ji[3:6, 3:6] = Jinv
    Jj[0:3, 0:3] = -M
    Jj[3:6, 3:6] = -Jinv @ M
    return Ji, Jj


def mean_at(cams, pairs):
    """pair means at the cameras' own relative poses [m, 7]"""
    cams = np.asarray(cams, np.float64)
    out = np.zeros((len(pairs), 7))
    for p, (i, j) in enumerate(pairs):
        M = _rot(cams[i]) @ _rot(cams[j]).T
        out[p, :4] = Rotation.from_matrix(M).as_quat()
        out[p, 4:7] = cams[i, 4:7] - M @ cams[j, 4:7]
    return out


def sqrt_info_kind(kind, rng, scale=1.0):
    """one 6x6 L: 'dense' (random, well conditioned), 'translation' (rows 0..2), 'rotation' (rows 3..5), 'none' (zero)"""
    L = np.zeros((6, 6))
    if kind == "dense":
        L = scale * (np.eye(6) + 0.3 * rng.standard_normal((6, 6)))
    elif kind == "translation":
        L[0:3, 0:3] = scale * (np.eye(3) + 0.2 * rng.standard_normal((3, 3)))
    elif kind == "rotation":
        L[3:6, 3:6] = scale * (np.eye(3) + 0.2 * rng.standard_normal((3, 3)))
    return L


def rows(cams, pairs, mean, sqrt_info, device_rot=False):
    """the pair rows of the whole problem, unscaled: Jp [6 m, 9 nc] = L de/d(inc) and r [6 m] = L e"""
    nc, m = len(cams), len(pairs)
    J, r = np.zeros((6 * m, 9 * nc)), np.zeros(6 * m)
    for p, (i, j) in enumerate(pairs):
        L = np.asarray(sqrt_info[p], np.float64)
        Ji, Jj = jacobians(cams[i], cams[j], mean[p], device_rot)
        J[6 * p:6 * p + 6, 9 * i:9 * i + 9] += L @ Ji
        J[6 * p:6 * p + 6, 9 * j:9 * j + 9] += L @ Jj
        r[6 * p:6 * p + 6] = L @ residual(cams[i], cams[j], mean[p], device_rot)
    return J, r


def cost(cams, pairs, mean, sqrt_info):
    """sum over the pairs of 1/2 |L e|^2"""
    return float(sum(0.5 * np.sum((np.asarray(sqrt_info[p], np.float64) @ residual(cams[i], cams[j], mean[p])) ** 2)
                     for p, (i, j) in enumerate(pairs)))


def pair_case(nc=7, nl=90, seed=41, unobserved=True):
    """synth_bal(nc, nl) (+ one camera without observations, tied by a dense pair prior to camera 0): pairs between
    consecutive cameras with dense, translation-only, rotation-only and zero L, a repeated pair, a reversed pair, and means
    near the cameras' relative poses"""
    from rootba_b200.synthetic import BalArrays, synth_bal
    prob = synth_bal(nc, nl, 3.6, seed=seed)
    cams = np.asarray(prob.cams, np.float64)
    if unobserved:
        extra = cams[0].copy()
        extra[4:7] += [0.3, -0.2, 0.1]
        cams = np.vstack([cams, extra])
        prob = BalArrays(cams, prob.lms, prob.lm_off, prob.obs_cam, prob.obs_xy)
    n = len(cams)
    rng = np.random.default_rng(seed + 1)
    pairs = [(i, i + 1) for i in range(nc - 1)] + [(2, 1), (0, 1), (nc - 1, 0)]
    kinds = ["dense", "translation", "rotation", "none"]
    L = [sqrt_info_kind(kinds[p % 4], rng) for p in range(len(pairs))]
    if unobserved:
        pairs.append((n - 1, 0))
        L.append(sqrt_info_kind("dense", rng))
    pairs = np.asarray(pairs, np.int32)
    mean = mean_at(cams, pairs)
    mean[:, 4:7] += rng.normal(0, 0.05, (len(pairs), 3))
    mean[:, :4] = [(Rotation.from_rotvec(rng.normal(0, 0.02, 3)) * Rotation.from_quat(q)).as_quat() for q in mean[:, :4]]
    return prob, (pairs, mean, np.stack(L))


def power_split(Jps, lam):
    """Hpp (the 9x9 diagonal blocks of Jps^T Jps, + lam I: Power-SC's JACOBI blocks, pair diagonals included) and O (the
    off-diagonal camera-camera blocks of Jps^T Jps, which only the pair rows create)"""
    G = Jps.T @ Jps
    n = G.shape[0]
    Hpp = np.zeros_like(G)
    for c in range(n // 9):
        s = slice(9 * c, 9 * c + 9)
        Hpp[s, s] = G[s, s]
    return Hpp + lam * np.eye(n), G - Hpp


def power_series(Hpp, E0mO, b, order, eta):
    """the series of k_power_vec on Hpp^-1 (E_0 - O): accum = -Hpp^-1 b, tmp = Hpp^-1 ((E_0 - O) tmp), stop at i |tmp| / |accum| < eta"""
    Hinv = np.linalg.inv(Hpp)
    tmp = -Hinv @ b
    acc = tmp.copy()
    for i in range(1, order + 1):
        tmp = Hinv @ (E0mO @ tmp)
        acc = acc + tmp
        if i * np.linalg.norm(tmp) / np.linalg.norm(acc) < eta:
            break
    return acc
