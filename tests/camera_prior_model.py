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


def residual(cam, mean):
    """e [9] of one camera [10] against one prior mean [10]"""
    cam, mean = np.asarray(cam, np.float64), np.asarray(mean, np.float64)
    R, R0 = cm.rotation(cam[:4] / np.linalg.norm(cam[:4])), cm.rotation(mean[:4] / np.linalg.norm(mean[:4]))
    return np.concatenate([-R.T @ cam[4:7] - mean[4:7], log_so3(R @ R0.T), cam[7:10] - mean[7:10]])


def jacobian(cam, mean):
    """de/d(increment) [9, 9] at the camera"""
    cam = np.asarray(cam, np.float64)
    R = cm.rotation(cam[:4] / np.linalg.norm(cam[:4]))
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


def rows(cams, mean, sqrt_info):
    """the prior rows of the whole problem, unscaled: A [nc, 9, 9] = L de/d(inc) and r [nc, 9] = L e"""
    nc = len(cams)
    A, r = np.zeros((nc, 9, 9)), np.zeros((nc, 9))
    for c in range(nc):
        L = np.asarray(sqrt_info[c], np.float64)
        A[c] = L @ jacobian(cams[c], mean[c])
        r[c] = L @ residual(cams[c], mean[c])
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


def dense_system_with_prior(prob, mean, sqrt_info):
    """the dense system of tests/test_oracle_dense_numpy.py::_dense_system with the prior rows appended: 9 rows per camera,
    pose columns L de/d(inc), zero landmark columns, residual L e.  _reduced() of it is the total (reprojection + prior) LM
    step: the Jacobi scaling over the whole Jacobian, H, b, inc = -H^-1 b, l_diff."""
    from test_oracle_dense_numpy import _dense_system
    Jp, Jl, r = _dense_system(prob)
    A, rp = rows(prob.cams, mean, sqrt_info)
    nc = prob.nc
    Jp_p = np.zeros((9 * nc, Jp.shape[1]))
    for c in range(nc):
        Jp_p[9 * c:9 * c + 9, 9 * c:9 * c + 9] = A[c]
    return np.vstack([Jp, Jp_p]), np.vstack([Jl, np.zeros((9 * nc, Jl.shape[1]))]), np.concatenate([r, rp.ravel()])
