"""An independent float64 model of the Gaussian camera prior (rba_set_camera_prior, DESIGN.md section 14).

Written from the mathematics, not from the kernel: the rotation residual goes through scipy's rotation-vector logarithm of
a rotation matrix (the kernel takes the logarithm of a quaternion product), and J_l^-1 is the numerical inverse of the
closed-form left Jacobian J_l (the kernel evaluates a closed form of the inverse).

  camera (q, t, f, k1, k2), R = R(q) world -> camera,  centre c = -R^T t
  e = (c - c0, Log(R R0^T), f - f0, k1 - k1_0, k2 - k2_0),  cost 1/2 |L e|^2
  increment (v, w, df, dk1, dk2) as camera_model / k_camera_update:  R' = Exp(w) R,  t' = Exp(w) t + v
  de/dv = -R^T,  de/dw = [0; J_l^-1(Log(R R0^T))],  identity on the intrinsics
"""
import numpy as np
from scipy.spatial.transform import Rotation

import camera_model as cm


def exp_so3(w):
    return Rotation.from_rotvec(np.asarray(w, np.float64)).as_matrix()


def log_so3(R):
    return Rotation.from_matrix(np.asarray(R, np.float64)).as_rotvec()


def left_jacobian(phi):
    """J_l(phi) = I + (1 - cos th) / th^2 [phi]x + (th - sin th) / th^3 [phi]x^2 (series for small th)"""
    phi = np.asarray(phi, np.float64)
    th = np.linalg.norm(phi)
    K = cm.hat(phi)
    if th < 1e-5:
        return np.eye(3) + K / 2 + K @ K / 6
    return np.eye(3) + (1 - np.cos(th)) / th ** 2 * K + (th - np.sin(th)) / th ** 3 * K @ K


def _cam_rot(cam, device_rot):
    """R of a camera: of its normalised quaternion, or (device_rot) as the kernels build it from the stored quaternion"""
    q = np.asarray(cam[:4], np.float64)
    return cm.rotation(q, device=True) if device_rot else cm.rotation(q / np.linalg.norm(q))


def residual(cam, mean, device_rot=False):
    """e [9] of one camera [10] against one prior mean [10].  device_rot: the centre -R^T t with R as the kernels build it;
    the logarithm depends on the quaternions' directions only (the kernels' Log of a quaternion product is invariant to
    their scale), so it is that of the normalised ones either way."""
    cam, mean = np.asarray(cam, np.float64), np.asarray(mean, np.float64)
    R, R0 = cm.rotation(cam[:4] / np.linalg.norm(cam[:4])), cm.rotation(mean[:4] / np.linalg.norm(mean[:4]))
    Rc = _cam_rot(cam, device_rot)
    return np.concatenate([-Rc.T @ cam[4:7] - mean[4:7], log_so3(R @ R0.T), cam[7:10] - mean[7:10]])


def jacobian(cam, mean, device_rot=False):
    """de/d(increment) [9, 9] at the camera"""
    cam = np.asarray(cam, np.float64)
    R = _cam_rot(cam, device_rot)
    phi = residual(cam, mean)[3:6]
    J = np.zeros((9, 9))
    J[0:3, 0:3] = -R.T
    J[3:6, 3:6] = np.linalg.inv(left_jacobian(phi))
    J[6:9, 6:9] = np.eye(3)
    return J


def apply_inc(cam, d):
    """the camera after the increment d [9] (unscaled): R' = Exp(w) R, t' = Exp(w) t + v, intrinsics + d[6:9]"""
    cam, d = np.asarray(cam, np.float64), np.asarray(d, np.float64)
    E = exp_so3(d[3:6])
    R = E @ cm.rotation(cam[:4] / np.linalg.norm(cam[:4]))
    out = np.empty(10)
    out[:4] = Rotation.from_matrix(R).as_quat()  # x, y, z, w
    out[4:7] = E @ cam[4:7] + d[:3]
    out[7:10] = cam[7:10] + d[6:9]
    return out


def rows(cams, mean, sqrt_info, device_rot=False):
    """the prior rows of the whole problem, unscaled: A [nc, 9, 9] = L de/d(inc) and r [nc, 9] = L e"""
    nc = len(cams)
    A, r = np.zeros((nc, 9, 9)), np.zeros((nc, 9))
    for c in range(nc):
        L = np.asarray(sqrt_info[c], np.float64)
        A[c] = L @ jacobian(cams[c], mean[c], device_rot)
        r[c] = L @ residual(cams[c], mean[c], device_rot)
    return A, r


def cost(cams, mean, sqrt_info):
    """sum over the cameras of 1/2 |L e|^2"""
    return float(sum(0.5 * np.sum((np.asarray(sqrt_info[c], np.float64) @ residual(cams[c], mean[c])) ** 2) for c in range(len(cams))))


def centre(cam):
    cam = np.asarray(cam, np.float64)
    return -cm.rotation(cam[:4] / np.linalg.norm(cam[:4])).T @ cam[4:7]


def mean_at(cams):
    """prior means at the cameras themselves [nc, 10]"""
    cams = np.asarray(cams, np.float64)
    m = np.array(cams, copy=True)
    m[:, :4] /= np.linalg.norm(m[:, :4], axis=1, keepdims=True)
    m[:, 4:7] = [centre(c) for c in cams]
    return m


def sqrt_info_kind(kind, rng, scale=1.0):
    """one 9x9 L: 'dense' (random, well conditioned), 'centre' (rows 0..2), 'intrinsics' (rows 6..8), 'none' (zero)"""
    L = np.zeros((9, 9))
    if kind == "dense":
        L = scale * (np.eye(9) + 0.3 * rng.standard_normal((9, 9)))
    elif kind == "centre":
        L[0:3, 0:3] = scale * (np.eye(3) + 0.2 * rng.standard_normal((3, 3)))
    elif kind == "intrinsics":
        L[6:9, 6:9] = scale * np.diag([0.01, 3.0, 3.0])
    return L


def prior_case(nc=7, nl=90, seed=21, unobserved=True):
    """synth_bal(7, 90) (+ one camera without observations): a mix of dense, centre-only, intrinsics-only and no priors,
    centred near the cameras; the unobserved camera carries a dense prior"""
    from rootba_b200.synthetic import BalArrays, synth_bal
    prob = synth_bal(nc, nl, 3.6, seed=seed)
    cams = np.asarray(prob.cams, np.float64)
    if unobserved:
        extra = cams[0].copy()
        extra[4:7] += [0.3, -0.2, 0.1]
        cams = np.vstack([cams, extra])
        prob = BalArrays(cams, prob.lms, prob.lm_off, prob.obs_cam, prob.obs_xy)
    rng = np.random.default_rng(seed + 1)
    mean = mean_at(cams)
    mean[:, 4:7] += rng.normal(0, 0.05, (len(cams), 3))
    mean[:, :4] = [(Rotation.from_rotvec(rng.normal(0, 0.01, 3)) * Rotation.from_quat(q)).as_quat() for q in mean[:, :4]]
    mean[:, 7] += rng.normal(0, 2.0, len(cams))
    kinds = ["dense", "centre", "intrinsics", "none"]
    L = np.stack([sqrt_info_kind(kinds[c % 4], rng) for c in range(len(cams))])
    if unobserved:
        L[-1] = sqrt_info_kind("dense", rng)
    return prob, mean, L


def small_prior(problem, seed=3):
    """centre, dense and intrinsics priors in turn, centres moved by N(0, 0.05): (mean, L)"""
    rng = np.random.default_rng(seed)
    mean = mean_at(problem.cams)
    mean[:, 4:7] += rng.normal(0, 0.05, (problem.nc, 3))
    L = np.stack([sqrt_info_kind(["centre", "dense", "intrinsics"][c % 3], rng) for c in range(problem.nc)])
    return mean, L


# ------------------------------------------------------------------------------------------------
# The kernels' SO(3) formulas (so3_log_rel, so3_jl_inv of rootba_b200/csrc/kernels.cuh), restated so that the CPU tests can
# show that the device checks would reject a subtly wrong variant of them.  `fault` plants one such variant:
#   "jl_identity"  J_l^-1 replaced by I;  "no_flip"  the product not flipped to w >= 0;  "series_everywhere"  the series of
#   J_l^-1 used at every angle (its range is theta^2 < 1e-4).
# ------------------------------------------------------------------------------------------------
def log_quat_device(a, m, eps_sqrt=1e-5, fault=None):
    """phi = Log(a (x) conj(m)) of two quaternions (x, y, z, w) as the kernels evaluate it: theta / n = 2 atan2(n, w) / n,
    its series 2 / w (1 - n^2 / (3 w^2)) where n < eps_sqrt w, the product first flipped to w >= 0"""
    a, m = np.asarray(a, np.float64), np.asarray(m, np.float64)
    b = np.array([-m[0], -m[1], -m[2], m[3]])
    w = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2]
    v = np.array([a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1],
                  a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2],
                  a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0]])
    if w < 0 and fault != "no_flip":
        w, v = -w, -v
    n2 = float(v @ v)
    n = np.sqrt(n2)
    fac = 2 / w * (1 - n2 / (3 * w * w)) if n < eps_sqrt * w else 2 * np.arctan2(n, w) / n
    return fac * v


def jl_inv_device(phi, fault=None):
    """J_l^-1(phi) = I - 1/2 [phi]x + a [phi]x^2, a = 1/th^2 - cot(th/2) / (2 th) (series 1/12 + th^2/720 + th^4/30240
    below th^2 = 1e-4)"""
    phi = np.asarray(phi, np.float64)
    if fault == "jl_identity":
        return np.eye(3)
    th2 = float(phi @ phi)
    if th2 < 1e-4 or fault == "series_everywhere":
        a = 1 / 12 + th2 * (1 / 720 + th2 / 30240)
    else:
        th = np.sqrt(th2)
        a = 1 / th2 - np.cos(th / 2) / (2 * th * np.sin(th / 2))
    K = cm.hat(phi)
    return np.eye(3) - 0.5 * K + a * K @ K


def rows_device(cams, mean, sqrt_info, fault=None):
    """rows() with the rotation rows by the kernels' formulas (and a planted fault): A [nc, 9, 9]"""
    nc = len(cams)
    A = np.zeros((nc, 9, 9))
    for c in range(nc):
        cam = np.asarray(cams[c], np.float64)
        J = np.zeros((9, 9))
        J[0:3, 0:3] = -cm.rotation(cam[:4], device=True).T
        J[3:6, 3:6] = jl_inv_device(log_quat_device(cam[:4], mean[c][:4], fault=fault), fault=fault)
        J[6:9, 6:9] = np.eye(3)
        A[c] = np.asarray(sqrt_info[c], np.float64) @ J
    return A


# residual angles of the large-rotation tests: 0 exactly, both branches of the log's series and of the J_l^-1 series (its
# switch is at theta = 0.01), and angles up to pi
ROTATION_ANGLES = [0.0, 1e-9, 5e-4, 0.009, 0.011, 0.5, 2.0, 3.0, np.pi - 1e-3]


def mean_at_angle(cam, theta, seed, negate=False):
    """a quaternion R0 with Log(R R0^T) of angle theta about a random axis (R of the camera), or its negative"""
    rng = np.random.default_rng(seed)
    axis = rng.standard_normal(3)
    axis /= np.linalg.norm(axis)
    R = Rotation.from_quat(np.asarray(cam[:4], np.float64))
    q0 = (Rotation.from_rotvec(-theta * axis) * R).as_quat()
    return -q0 if negate else q0
