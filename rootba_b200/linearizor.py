"""Host-side mirror of the reference's interface for the QR hot path, on top of the C ABI.

  BalProblem        <-> rootba::BalProblem<Scalar>     (src/rootba/bal/bal_problem.hpp:61-234)
  SolverOptions     <-> rootba::SolverOptions          (src/rootba/bal/solver_options.hpp:46-284)
  LinearizorQR      <-> rootba::LinearizorQR<Scalar>   (src/rootba/solver/linearizor_qr.cpp:52-291)
                        behind rootba::Linearizor      (src/rootba/solver/linearizor.hpp:47-83)

Same names, argument meaning and error behaviour: numerical trouble is reported through return values
(NaN l_diff, non-finite increment), invariant violations raise (the reference CHECK-aborts).
The optimisation state lives on the GPU; `BalProblem.cameras/landmarks` are refreshed on demand.
"""
from __future__ import annotations

import ctypes as C
import os
import dataclasses
import math
import time

import numpy as np

from . import _lib
from ._lib import (FIX_ALL, CgSummary, LmIteration, LmOpts, LmStepResult, ProblemView, RbaError, ResidualInfo, SolverOpts, StageTimings, WorkloadStats,
                   check, struct_to_dict)


@dataclasses.dataclass
class ResidualOptions:  # bal/bal_residual_options.hpp:44-63
    robust_norm: str = "NONE"      # NONE | HUBER
    huber_parameter: float = 1.0


@dataclasses.dataclass
class SolverOptions:  # bal/solver_options.hpp (QR-relevant subset, reference defaults)
    solver_type: str = "SQUARE_ROOT"              # SQUARE_ROOT | SCHUR_COMPLEMENT | POWER_SCHUR_COMPLEMENT (solver_options.hpp:63-76)
    power_order: int = 20                         # :270
    optimized_cost: str = "ERROR"                 # ERROR | ERROR_VALID | ERROR_VALID_AVG
    max_num_iterations: int = 20
    min_relative_decrease: float = 0.0           # solver_options.hpp:146-148
    initial_trust_region_radius: float = 1e4
    min_trust_region_radius: float = 1e-32
    max_trust_region_radius: float = 1e16
    min_linear_solver_iterations: int = 0
    max_linear_solver_iterations: int = 500
    eta: float = 0.1
    residual_reset_period: int = 10              # ConjugateGradientsSolver::Options (cg/conjugate_gradient.hpp:87): r = b - H x every this many iterations
    jacobi_scaling_epsilon: float = 0.0
    preconditioner_type: str = "SCHUR_JACOBI"     # JACOBI | SCHUR_JACOBI | CLUSTER_JACOBI (:73-75; DESIGN.md section 28)
    function_tolerance: float = 1e-6
    use_double: bool = True
    use_householder_marginalization: bool = True
    staged_execution: bool = True
    reduction_alg: int = 1
    initial_vee: float = 2.0
    vee_factor: float = 2.0
    residual: ResidualOptions = dataclasses.field(default_factory=ResidualOptions)
    # placement (not in the reference)
    device: int = -1
    rank: int = 0
    nranks: int = 1
    pcg_check_period: int = 4
    operator_form: str = "DENSE"                  # DENSE (reference: Q2 panels) | IMPLICIT (Jp^T Jp - Q1d^T Q1d from records)
    stage2_form: str = "PANEL"                    # PANEL (reference: b and SCHUR_JACOBI blocks from the Q2 panels) | IDENTITY
    linear_solver_type: str = "ITERATIVE_SCHUR"   # ITERATIVE_SCHUR (PCG / power series) | DENSE_SCHUR (exact, dense Cholesky; :77-80, 225-230)

    def use_projection_validity_check(self) -> bool:  # solver_options.cpp:41-51
        return self.optimized_cost != "ERROR"


def _camera_fixed_array(flags, num_cameras: int):
    """None, or a validated uint8 copy of one FIX_* bit set per camera"""
    if flags is None:
        return None
    a = np.asarray(flags)
    if a.shape != (num_cameras,):
        raise ValueError(f"camera_fixed must have one entry per camera ({num_cameras}), got shape {a.shape}")
    if a.dtype.kind not in "iu" or np.any(a < 0) or np.any(a > FIX_ALL):
        raise ValueError(f"camera_fixed entries must be integers combining FIX_* bits (0..{FIX_ALL})")
    return np.ascontiguousarray(a, dtype=np.uint8).copy()


def _intrinsics_group_array(group, num_cameras: int):
    """None, or a validated int32 copy of one group id per camera (-1 = own intrinsics, else an id in [0, num_cameras))"""
    if group is None:
        return None
    a = np.asarray(group)
    if a.shape != (num_cameras,):
        raise ValueError(f"intrinsics_group must have one entry per camera ({num_cameras}), got shape {a.shape}")
    if a.dtype.kind not in "iu" or np.any(a < -1) or np.any(a >= num_cameras):
        raise ValueError(f"intrinsics_group entries must be integers in [-1, {num_cameras})")
    return np.ascontiguousarray(a, dtype=np.int32).copy()


def _camera_rig_arrays(rig, num_cameras: int, dtype):
    """None, or validated contiguous copies (rig [nc] int32, cam_from_rig [nc,7] in `dtype`) of camera rigs: one rig id per
    camera (-1 = free camera, else an id in [0, num_cameras)) and each camera's extrinsics qx,qy,qz,qw, tx,ty,tz; a rigged
    camera's entries must be finite with a quaternion within 1e-3 of unit norm (the free cameras' are ignored)"""
    if rig is None:
        return None
    rid, e = rig
    a = np.asarray(rid)
    if a.shape != (num_cameras,):
        raise ValueError(f"camera_rig ids must have one entry per camera ({num_cameras}), got shape {a.shape}")
    if a.dtype.kind not in "iu" or np.any(a < -1) or np.any(a >= num_cameras):
        raise ValueError(f"camera_rig ids must be integers in [-1, {num_cameras})")
    e = np.array(e, dtype=dtype, order="C", copy=True)
    if e.shape != (num_cameras, 7):
        raise ValueError(f"camera_rig cam_from_rig must have shape ({num_cameras}, 7), got {e.shape}")
    r = a >= 0
    if not np.all(np.isfinite(e[r])):
        raise ValueError("camera_rig cam_from_rig entries of rigged cameras must be finite")
    qn = np.linalg.norm(e[r, :4].astype(np.float64), axis=1)
    if np.any(np.abs(qn - 1.0) > 1e-3):
        raise ValueError("camera_rig cam_from_rig quaternions must have norm 1 (within 1e-3)")
    return np.ascontiguousarray(a, dtype=np.int32).copy(), e


def _rig_sensor_array(sensor, camera_rig, num_cameras: int):
    """None, or a validated contiguous int32 copy of rig sensor ids (-1 = the camera's extrinsics are held, else an id in
    [0, num_cameras) shared by every capture of one sensor): every camera with an id must be in a rig of >= 2 cameras of
    `camera_rig`, no two cameras of one rig may share an id, and every rig keeps a camera without one"""
    if sensor is None:
        return None
    a = np.asarray(sensor)
    if a.shape != (num_cameras,):
        raise ValueError(f"rig_sensor ids must have one entry per camera ({num_cameras}), got shape {a.shape}")
    if a.dtype.kind not in "iu" or np.any(a < -1) or np.any(a >= num_cameras):
        raise ValueError(f"rig_sensor ids must be integers in [-1, {num_cameras})")
    a = np.ascontiguousarray(a, dtype=np.int32).copy()
    rig = np.full(num_cameras, -1) if camera_rig is None else np.asarray(camera_rig[0])
    rid, count = np.unique(rig[rig >= 0], return_counts=True)
    in_rig = np.isin(rig, rid[count >= 2])
    if np.any((a >= 0) & ~in_rig):
        raise ValueError(f"rig_sensor: camera {int(np.flatnonzero((a >= 0) & ~in_rig)[0])} has a sensor id but is not in a rig of >= 2 cameras")
    for r in rid[count >= 2]:
        s = a[rig == r]
        if np.all(s >= 0):
            raise ValueError(f"rig_sensor: every camera of rig {int(r)} has a sensor id; none is left to carry the rig's pose")
        if len(np.unique(s[s >= 0])) != int(np.sum(s >= 0)):
            raise ValueError(f"rig_sensor: two cameras of rig {int(r)} have the same sensor id")
    return a


def _prior_arrays(name, mean, sqrt_info, dtype, m, mean_len, dim, check_index=None, item=None):
    """validated contiguous copies (mean [m, mean_len], sqrt_info [m, dim, dim]) in `dtype` of the priors `name`.  The checks
    run in this order: the shapes, the kind's own index checks (`check_index`), finiteness and, for a kind whose mean
    starts with a quaternion (`item` names its entries), the quaternion norm."""
    mean = np.array(mean, dtype=dtype, order="C", copy=True)
    sqrt_info = np.array(sqrt_info, dtype=dtype, order="C", copy=True)
    if mean.shape != (m, mean_len):
        raise ValueError(f"{name} mean must have shape ({m}, {mean_len}), got {mean.shape}")
    if sqrt_info.shape != (m, dim, dim):
        raise ValueError(f"{name} sqrt_info must have shape ({m}, {dim}, {dim}), got {sqrt_info.shape}")
    if check_index is not None:
        check_index()
    if not (np.all(np.isfinite(mean)) and np.all(np.isfinite(sqrt_info))):
        raise ValueError(f"{name} entries must be finite")
    if item is not None:
        qn = np.linalg.norm(mean[:, :4].astype(np.float64), axis=1)
        if np.any(np.abs(qn - 1.0) > 1e-3):
            raise ValueError(f"{name} mean quaternions must have norm 1 (within 1e-3); {item} {int(np.argmax(np.abs(qn - 1.0)))} has {qn.max():.6g}")
    return mean, sqrt_info


def _camera_prior_arrays(prior, num_cameras: int, dtype):
    """None, or validated contiguous copies (mean [nc,10], sqrt_info [nc,9,9]) of a camera prior in the problem's dtype"""
    if prior is None:
        return None
    mean, sqrt_info = prior
    return _prior_arrays("camera_prior", mean, sqrt_info, dtype, num_cameras, 10, 9, item="camera")


def _camera_pair_prior_arrays(prior, num_cameras: int, dtype):
    """None, or validated contiguous copies (pairs [m,2] int32, mean [m,7], sqrt_info [m,6,6]) of pair priors in the problem's
    dtype"""
    if prior is None:
        return None
    pairs, mean, sqrt_info = prior
    pairs = np.array(pairs, dtype=np.int32, order="C", copy=True)
    m = pairs.shape[0] if pairs.ndim == 2 else -1
    if pairs.shape != (m, 2):
        raise ValueError(f"camera_pair_prior pairs must have shape (m, 2), got {pairs.shape}")

    def check_index():
        if np.any(pairs < 0) or np.any(pairs >= num_cameras) or np.any(pairs[:, 0] == pairs[:, 1]):
            raise ValueError(f"camera_pair_prior pairs must join two different cameras in [0, {num_cameras})")
    return (pairs, *_prior_arrays("camera_pair_prior", mean, sqrt_info, dtype, m, 7, 6, check_index, item="pair"))


def _landmark_prior_arrays(prior, num_landmarks: int, dtype):
    """None, or validated contiguous copies (idx [m] int32, mean [m,3], sqrt_info [m,3,3]) of landmark priors in the
    problem's dtype"""
    if prior is None:
        return None
    idx, mean, sqrt_info = prior
    idx = np.array(idx, dtype=np.int32, order="C", copy=True)
    m = idx.shape[0] if idx.ndim == 1 else -1
    if idx.shape != (m,):
        raise ValueError(f"landmark_prior idx must have shape (m,), got {idx.shape}")

    def check_index():
        if np.any(idx < 0) or np.any(idx >= num_landmarks):
            raise ValueError(f"landmark_prior idx must be landmark indices in [0, {num_landmarks})")
        if len(np.unique(idx)) != m:
            raise ValueError("landmark_prior idx must not repeat a landmark")
    return (idx, *_prior_arrays("landmark_prior", mean, sqrt_info, dtype, m, 3, 3, check_index))


def _observation_info_array(info, num_observations: int, dtype):
    """None, or a validated contiguous copy [Nobs, 2, 2] in `dtype` of per-observation square-root information given as
    [Nobs] (1 / sigma, expanded to I / sigma) or [Nobs, 2, 2]"""
    if info is None:
        return None
    a = np.array(info, dtype=dtype, order="C", copy=True)
    if a.shape == (num_observations,):
        w = np.zeros((num_observations, 2, 2), dtype)
        w[:, 0, 0] = w[:, 1, 1] = a
        a = w
    if a.shape != (num_observations, 2, 2):
        raise ValueError(f"observation_sqrt_info must have shape ({num_observations},) or ({num_observations}, 2, 2), got {a.shape}")
    if not np.all(np.isfinite(a)):
        raise ValueError("observation_sqrt_info entries must be finite")
    return a


def _loss_arrays(loss, num: int, dtype, name: str = "observation_loss"):
    """None, or validated contiguous (kind [num] uint8, scale [num] in `dtype`) of robust losses given as (kind, scale): kind a
    name of LOSS_KINDS, an RBA_LOSS_* int or a [num] array of either, scale a scalar or [num]; scalars are broadcast.  The
    checks of rba_set_observation_loss and rba_set_prior_loss: a known kind, and a finite scale > 0 for every kind but NONE
    (whose scale is ignored).  `name` names the losses in the messages."""
    if loss is None:
        return None
    try:
        kind, scale = loss
    except (TypeError, ValueError):
        raise ValueError(f"{name} must be None or (kind, scale)") from None
    k = np.asarray(kind)
    if k.dtype.kind in "US":
        names = [str(x).upper() for x in k.ravel()]
        bad = sorted(set(names) - set(_lib.LOSS_KINDS))
        if bad:
            raise ValueError(f"{name} kind must be one of {sorted(_lib.LOSS_KINDS)}, got {bad}")
        k = np.array([_lib.LOSS_KINDS[n] for n in names], np.int64).reshape(k.shape)
    elif k.dtype.kind not in "iu":
        raise ValueError(f"{name} kind must be names or integers, got dtype {k.dtype}")
    if k.ndim == 0:
        k = np.full(num, k)
    if k.shape != (num,):
        raise ValueError(f"{name} kind must be a scalar or have shape ({num},), got {k.shape}")
    if np.any((k < 0) | (k > _lib.LOSS_TUKEY)):
        raise ValueError(f"{name} kinds must be in 0..{_lib.LOSS_TUKEY}")
    a = np.array(scale, dtype=dtype, copy=True)
    if a.ndim == 0:
        a = np.full(num, a, dtype)
    if a.shape != (num,):
        raise ValueError(f"{name} scale must be a scalar or have shape ({num},), got {a.shape}")
    robust = k != _lib.LOSS_NONE
    if not np.all(np.isfinite(a[robust]) & (a[robust] > 0)):
        raise ValueError(f"{name} scales must be finite and > 0 for every kind but NONE")
    return np.ascontiguousarray(k, np.uint8), np.ascontiguousarray(a)


class BalProblem:
    """SoA BalProblem: cameras [nc,10] (quat xyzw, t, f,k1,k2), landmarks [nl,3], observations in
    CSR-by-landmark order with ascending camera index.  `camera_fixed` (not in the reference): None or one uint8 of FIX_*
    bits per camera, held constant by the solver; forwarded to an attached LinearizorQR on assignment.
    `camera_prior` (not in the reference): None or (mean [nc,10], sqrt_info [nc,9,9]), a Gaussian prior per camera with the
    cost 1/2 |L e|^2, e = (centre - c0, Log(R R0^T), f - f0, k1 - k1_0, k2 - k2_0) (rba_set_camera_prior, DESIGN.md section 14);
    mean rows are (qx,qy,qz,qw of R0, camera centre c0, f0, k1_0, k2_0).  Forwarded to an attached LinearizorQR on assignment.
    `camera_pair_prior` (not in the reference): None or (pairs [m,2] int32, mean [m,7], sqrt_info [m,6,6]), relative pose priors
    T_i T_j^-1 ~ (R0, t0) with the cost 1/2 |L e|^2, e = (t_i - R_i R_j^T t_j - t0, Log(R_i R_j^T R0^T))
    (rba_set_camera_pair_prior, DESIGN.md section 15); mean rows are (qx,qy,qz,qw of R0, t0).  Forwarded likewise.
    `landmark_prior` (not in the reference): None or (idx [m] int32, mean [m,3], sqrt_info [m,3,3]), Gaussian priors on
    landmark positions with the cost 1/2 |L (x - x0)|^2 (rba_set_landmark_prior, DESIGN.md section 17).  Forwarded likewise.
    `intrinsics_group` (not in the reference): None or one int32 group id per camera (-1 = own intrinsics); the cameras of a
    group share one f, k1, k2 (rba_set_intrinsics_groups, DESIGN.md section 18).  Forwarded likewise.
    `camera_rig` (not in the reference): None or (rig [nc] int32, cam_from_rig [nc,7]), rigid camera rigs: one rig id per
    camera (-1 = free camera) and each camera's fixed extrinsics (qx,qy,qz,qw, tx,ty,tz of cam_from_rig); the cameras of a rig
    keep the relative poses of their extrinsics and the solve moves one pose per rig (rba_set_camera_rigs, DESIGN.md section
    23).  Forwarded likewise.
    `rig_sensor` (not in the reference): None or one int32 sensor id per camera (-1 = the camera's extrinsics are held, as
    given to camera_rig); the cameras with one id are captures of one physical camera whose extrinsics are estimated and
    shared (rba_set_rig_sensors, DESIGN.md section 24).  Forwarded likewise; setting camera_rig clears it.
    `observation_sqrt_info` (not in the reference): None, [Nobs] (1 / sigma per observation) or [Nobs,2,2] (a square root W of
    the inverse keypoint covariance per observation, in the order of obs_cam / obs_xy); the observation's cost becomes
    rho(|W r|^2) and W = 0 switches it off (rba_set_observation_info, DESIGN.md section 19).  Stored as [Nobs,2,2]; forwarded
    likewise.
    `observation_loss` (not in the reference): None (every observation uses the options' robust_norm) or (kind, scale), a
    robust loss per observation: kind "NONE" | "HUBER" | "CAUCHY" | "SOFT_L1" | "TUKEY" (or RBA_LOSS_* ints), scale the inlier
    threshold in units of sigma, each a scalar (broadcast) or one entry per observation (rba_set_observation_loss, DESIGN.md
    section 21).  Stored as (kind [Nobs] uint8, scale [Nobs]); forwarded likewise.
    `camera_prior_loss`, `camera_pair_prior_loss`, `landmark_prior_loss` (not in the reference): None (NONE on every prior of
    that kind) or (kind, scale) as for observation_loss, one entry per camera / per pair / per landmark prior in the order of
    the kind's prior (rba_set_prior_loss, DESIGN.md section 22): the prior's cost becomes rho(|L e|^2)/2.  Setting the kind's
    prior clears its loss.  Forwarded likewise."""

    def __init__(self, cams, lms, lm_off, obs_cam, obs_xy, dtype=np.float64):
        self.dtype = np.dtype(dtype)
        # the problem owns its optimisation state (it is updated in place by the solver)
        self.cams = np.array(cams, dtype=self.dtype, order="C", copy=True).reshape(-1, 10)
        self.lms = np.array(lms, dtype=self.dtype, order="C", copy=True).reshape(-1, 3)
        self.lm_off = np.ascontiguousarray(lm_off, dtype=np.int64)
        self.obs_cam = np.ascontiguousarray(obs_cam, dtype=np.int32)
        self.obs_xy = np.ascontiguousarray(obs_xy, dtype=self.dtype).reshape(-1, 2)
        self._cams_backup = self.cams.copy()
        self._lms_backup = self.lms.copy()
        self._linearizor = None
        self._camera_fixed = None
        self._camera_prior = None
        self._camera_pair_prior = None
        self._landmark_prior = None
        self._intrinsics_group = None
        self._camera_rig = None
        self._rig_sensor = None
        self._observation_sqrt_info = None
        self._observation_loss = None
        self._prior_loss = {_lib.PRIOR_CAMERA: None, _lib.PRIOR_PAIR: None, _lib.PRIOR_LANDMARK: None}

    def _prior_count(self, which: int) -> int:
        """the entries of one prior kind's losses: the cameras, or the pairs / landmark priors of its prior (0 without one)"""
        if which == _lib.PRIOR_CAMERA:
            return self.num_cameras()
        prior = self._camera_pair_prior if which == _lib.PRIOR_PAIR else self._landmark_prior
        return 0 if prior is None else len(prior[0])

    def _set_prior_loss(self, which: int, loss):
        name = {_lib.PRIOR_CAMERA: "camera_prior_loss", _lib.PRIOR_PAIR: "camera_pair_prior_loss",
                _lib.PRIOR_LANDMARK: "landmark_prior_loss"}[which]
        ls = _loss_arrays(loss, self._prior_count(which), self.dtype, name)
        if self._linearizor is not None:
            self._linearizor._upload_prior_loss(which, ls)  # raises on rejection: the previous losses stay in force
        self._prior_loss[which] = ls

    @property
    def camera_prior_loss(self):
        return self._prior_loss[_lib.PRIOR_CAMERA]

    @camera_prior_loss.setter
    def camera_prior_loss(self, loss):
        self._set_prior_loss(_lib.PRIOR_CAMERA, loss)

    @property
    def camera_pair_prior_loss(self):
        return self._prior_loss[_lib.PRIOR_PAIR]

    @camera_pair_prior_loss.setter
    def camera_pair_prior_loss(self, loss):
        self._set_prior_loss(_lib.PRIOR_PAIR, loss)

    @property
    def landmark_prior_loss(self):
        return self._prior_loss[_lib.PRIOR_LANDMARK]

    @landmark_prior_loss.setter
    def landmark_prior_loss(self, loss):
        self._set_prior_loss(_lib.PRIOR_LANDMARK, loss)

    @property
    def observation_loss(self):
        return self._observation_loss

    @observation_loss.setter
    def observation_loss(self, loss):
        ls = _loss_arrays(loss, self.num_observations(), self.dtype)
        if self._linearizor is not None:
            self._linearizor._upload_observation_loss(ls)  # raises on rejection: the previous losses stay in force
        self._observation_loss = ls

    @property
    def observation_sqrt_info(self):
        return self._observation_sqrt_info

    @observation_sqrt_info.setter
    def observation_sqrt_info(self, info):
        w = _observation_info_array(info, self.num_observations(), self.dtype)
        if self._linearizor is not None:
            self._linearizor._upload_observation_info(w)  # raises on rejection: the previous information stays in force
        self._observation_sqrt_info = w

    @property
    def intrinsics_group(self):
        return self._intrinsics_group

    @intrinsics_group.setter
    def intrinsics_group(self, group):
        g = _intrinsics_group_array(group, self.num_cameras())
        if self._linearizor is not None:
            self._linearizor._upload_intrinsics_group(g)  # raises on rejection: the previous groups stay in force
        self._intrinsics_group = g

    @property
    def camera_rig(self):
        return self._camera_rig

    @camera_rig.setter
    def camera_rig(self, rig):
        r = _camera_rig_arrays(rig, self.num_cameras(), self.dtype)
        if self._linearizor is not None:
            self._linearizor._upload_camera_rig(r)  # raises on rejection: the previous rigs stay in force
        self._camera_rig = r
        self._rig_sensor = None  # the sensors belonged to the previous rigs

    @property
    def rig_sensor(self):
        return self._rig_sensor

    @rig_sensor.setter
    def rig_sensor(self, sensor):
        a = _rig_sensor_array(sensor, self._camera_rig, self.num_cameras())
        if self._linearizor is not None:
            self._linearizor._upload_rig_sensor(a)  # raises on rejection: the previous sensors stay in force
        self._rig_sensor = a

    @property
    def landmark_prior(self):
        return self._landmark_prior

    @landmark_prior.setter
    def landmark_prior(self, prior):
        p = _landmark_prior_arrays(prior, self.num_landmarks(), self.dtype)
        if self._linearizor is not None:
            self._linearizor._upload_landmark_prior(p)  # raises on rejection: the previous landmark priors stay in force
        self._landmark_prior = p
        self._prior_loss[_lib.PRIOR_LANDMARK] = None  # the setter clears the kind's losses (rba_set_prior_loss)

    @property
    def camera_pair_prior(self):
        return self._camera_pair_prior

    @camera_pair_prior.setter
    def camera_pair_prior(self, prior):
        p = _camera_pair_prior_arrays(prior, self.num_cameras(), self.dtype)
        if self._linearizor is not None:
            self._linearizor._upload_camera_pair_prior(p)  # raises on rejection: the previous pair priors stay in force
        self._camera_pair_prior = p
        self._prior_loss[_lib.PRIOR_PAIR] = None  # the setter clears the kind's losses (rba_set_prior_loss)

    @property
    def camera_prior(self):
        return self._camera_prior

    @camera_prior.setter
    def camera_prior(self, prior):
        p = _camera_prior_arrays(prior, self.num_cameras(), self.dtype)
        if self._linearizor is not None:
            self._linearizor._upload_camera_prior(p)  # raises on rejection: the previous priors stay in force
        self._camera_prior = p
        self._prior_loss[_lib.PRIOR_CAMERA] = None  # the setter clears the kind's losses (rba_set_prior_loss)

    @property
    def camera_fixed(self):
        return self._camera_fixed

    @camera_fixed.setter
    def camera_fixed(self, flags):
        self._camera_fixed = _camera_fixed_array(flags, self.num_cameras())
        if self._linearizor is not None:
            self._linearizor._upload_camera_fixed()

    @classmethod
    def from_arrays(cls, arrays, dtype=np.float64) -> "BalProblem":
        return cls(arrays.cams, arrays.lms, arrays.lm_off, arrays.obs_cam, arrays.obs_xy, dtype)

    @classmethod
    def load_bal(cls, path: str, dtype=np.float64, normalize: bool = True, scale: float = 100.0, num_threads: int = 0,
                 init_depth_threshold: float = 0.0, rotation_sigma: float = 0.0, translation_sigma: float = 0.0,
                 point_sigma: float = 0.0, random_seed: int = 38401) -> "BalProblem":
        """load_normalized_bal_problem (bal/bal_problem.cpp:773-852) through the library's multi-threaded BAL parser
        (rba_bal_load): load + normalise in double, then cast to dtype."""
        L = _lib.lib()
        f = C.c_void_p()
        check(L.rba_bal_load(os.fsencode(path), int(normalize), C.c_double(scale), int(num_threads), C.byref(f)))
        try:
            if rotation_sigma > 0 or translation_sigma > 0 or point_sigma > 0:  # BalProblem::perturb (bal_problem.cpp:507-554, :820-822)
                check(L.rba_bal_perturb(f, C.c_double(rotation_sigma), C.c_double(translation_sigma), C.c_double(point_sigma),
                                        C.c_int32(random_seed)))
            if init_depth_threshold > 0:  # BalDatasetOptions::init_depth_threshold -> filter_obs (bal_problem.cpp:471-505, :826)
                check(L.rba_bal_filter_obs(f, C.c_double(init_depth_threshold)))
            nc, nl, nobs = C.c_int32(), C.c_int32(), C.c_int64()
            check(L.rba_bal_dims(f, C.byref(nc), C.byref(nl), C.byref(nobs)))
            cams, lms = np.empty((nc.value, 10)), np.empty((nl.value, 3))
            off, oc, xy = np.empty(nl.value + 1, np.int64), np.empty(nobs.value, np.int32), np.empty((nobs.value, 2))
            check(L.rba_bal_copy(f, _p(cams), _p(lms), _p(off), _p(oc), _p(xy)))
            t = (C.c_double * 5)()
            check(L.rba_bal_load_timings(f, t))
        finally:
            L.rba_bal_free(f)
        bp = cls(cams, lms, off, oc, xy, dtype)
        bp.load_timings = dict(zip(("read", "count", "parse", "csr", "normalize"), t))
        return bp

    def num_cameras(self): return self.cams.shape[0]
    def num_landmarks(self): return self.lms.shape[0]
    def num_observations(self): return self.obs_cam.shape[0]

    # BalProblem::backup / restore (bal/bal_problem.cpp:590-608); forwarded to the device copy when attached
    def backup(self):
        if self._linearizor is not None:
            self._linearizor._backup()
        else:
            self._cams_backup[:] = self.cams
            self._lms_backup[:] = self.lms

    def restore(self):
        if self._linearizor is not None:
            self._linearizor._restore()
        else:
            self.cams[:] = self._cams_backup
            self.lms[:] = self._lms_backup

    def sync_from_device(self):
        if self._linearizor is not None:
            self._linearizor.download_state()


class LinearizorQR:
    """rootba::LinearizorQR on the GPU.  Protocol (linearizor.hpp:56-82):
    create once; per LM iteration start_iteration -> compute_error -> linearize ->
    { solve(lambda) -> [bal_problem.backup()] -> apply -> compute_error -> (restore on reject) }+ ."""

    def __init__(self, bal_problem: BalProblem, options: SolverOptions, summary: dict | None = None):
        if options.solver_type not in ("SQUARE_ROOT", "SCHUR_COMPLEMENT", "POWER_SCHUR_COMPLEMENT"):
            raise ValueError(f"solver_type {options.solver_type} is not provided by rootba_b200")
        self.bal_problem = bal_problem
        self.options = options
        self.summary = summary
        self.it_summary = None
        self.dtype = bal_problem.dtype
        self.sfx = "f32" if self.dtype == np.float32 else "f64"
        self.S = C.c_float if self.dtype == np.float32 else C.c_double
        L = _lib.lib()
        o = SolverOpts()
        L.rba_default_solver_opts(C.byref(o))
        o.use_householder_marginalization = int(options.use_householder_marginalization)
        o.use_valid_projections_only = int(options.use_projection_validity_check())
        o.robust_norm = {"NONE": 0, "HUBER": 1}[options.residual.robust_norm]
        o.huber_parameter = options.residual.huber_parameter
        o.jacobi_scaling_epsilon = options.jacobi_scaling_epsilon
        o.preconditioner_type = {"JACOBI": 0, "SCHUR_JACOBI": 1, "CLUSTER_JACOBI": 2}[options.preconditioner_type]
        o.min_linear_solver_iterations = options.min_linear_solver_iterations
        o.max_linear_solver_iterations = options.max_linear_solver_iterations
        o.eta = options.eta
        o.residual_reset_period = options.residual_reset_period
        o.device, o.rank, o.nranks = options.device, options.rank, options.nranks
        o.pcg_check_period = options.pcg_check_period
        o.operator_form = {"DENSE": 0, "IMPLICIT": 1}[options.operator_form]
        o.stage2_form = {"PANEL": 0, "IDENTITY": 1}[options.stage2_form]
        o.solver_type = {"SQUARE_ROOT": 0, "SCHUR_COMPLEMENT": 1, "POWER_SCHUR_COMPLEMENT": 2}[options.solver_type]  # linearizor.cpp:48-65
        o.power_order = options.power_order
        o.linear_solver_type = {"ITERATIVE_SCHUR": 0, "DENSE_SCHUR": 1}[options.linear_solver_type]
        self._opts = o
        pv = ProblemView(bal_problem.num_cameras(), bal_problem.num_landmarks(), bal_problem.num_observations(),
                         bal_problem.lm_off.ctypes.data, bal_problem.obs_cam.ctypes.data, bal_problem.obs_xy.ctypes.data)
        self.h = C.c_void_p()
        check(getattr(L, f"rba_create_{self.sfx}")(C.byref(pv), C.byref(o), C.byref(self.h)))
        self.nc = bal_problem.num_cameras()
        self.nl = bal_problem.num_landmarks()
        self.upload_state()
        bal_problem._linearizor = self
        self.last_cg = CgSummary()
        if bal_problem.camera_fixed is not None:
            self._upload_camera_fixed()
        if bal_problem.camera_prior is not None:
            self._upload_camera_prior(bal_problem.camera_prior)
        if bal_problem.camera_pair_prior is not None:
            self._upload_camera_pair_prior(bal_problem.camera_pair_prior)
        if bal_problem.landmark_prior is not None:
            self._upload_landmark_prior(bal_problem.landmark_prior)
        if bal_problem.intrinsics_group is not None:
            self._upload_intrinsics_group(bal_problem.intrinsics_group)
        if bal_problem.camera_rig is not None:
            self._upload_camera_rig(bal_problem.camera_rig)
        if bal_problem.rig_sensor is not None:
            self._upload_rig_sensor(bal_problem.rig_sensor)
        if bal_problem.observation_sqrt_info is not None:
            self._upload_observation_info(bal_problem.observation_sqrt_info)
        if bal_problem.observation_loss is not None:
            self._upload_observation_loss(bal_problem.observation_loss)
        for which, loss in bal_problem._prior_loss.items():
            if loss is not None:
                self._upload_prior_loss(which, loss)

    # factory like Linearizor::create (linearizor.cpp:47-65)
    @staticmethod
    def create(bal_problem: BalProblem, options: SolverOptions, summary: dict | None = None) -> "LinearizorQR":
        return LinearizorQR(bal_problem, options, summary)

    def close(self):
        if getattr(self, "h", None):
            _lib.lib().rba_destroy(self.h)
            self.h = None
            if self.bal_problem._linearizor is self:
                self.bal_problem._linearizor = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- state transfer ----
    def upload_state(self):
        check(_lib.lib().rba_set_state(self.h, _p(self.bal_problem.cams), _p(self.bal_problem.lms)))

    def download_state(self):
        check(_lib.lib().rba_get_state(self.h, _p(self.bal_problem.cams), _p(self.bal_problem.lms)))

    def set_camera_fixed(self, flags):
        """hold camera parameters constant (rba_set_camera_fixed): None, or one uint8 of FIX_* bits per camera.  Takes effect
        at the next solve; the flags are stored on the BalProblem."""
        self.bal_problem.camera_fixed = flags  # validates and forwards to _upload_camera_fixed

    def _upload_camera_fixed(self):
        f = self.bal_problem.camera_fixed
        check(_lib.lib().rba_set_camera_fixed(self.h, None if f is None else _p(f)))

    def set_camera_prior(self, prior):
        """Gaussian camera priors (rba_set_camera_prior): None, or (mean [nc,10], sqrt_info [nc,9,9]).  Needs a new linearize
        before the next solve; the priors are stored on the BalProblem."""
        self.bal_problem.camera_prior = prior  # validates and forwards to _upload_camera_prior

    def _upload_camera_prior(self, prior):
        if prior is None:
            check(_lib.lib().rba_set_camera_prior(self.h, None, None))
        else:
            check(_lib.lib().rba_set_camera_prior(self.h, _p(prior[0]), _p(prior[1])))

    def set_camera_pair_prior(self, prior):
        """relative pose priors (rba_set_camera_pair_prior): None, or (pairs [m,2], mean [m,7], sqrt_info [m,6,6]).  Needs a new
        linearize before the next solve; the priors are stored on the BalProblem."""
        self.bal_problem.camera_pair_prior = prior  # validates and forwards to _upload_camera_pair_prior

    def _upload_camera_pair_prior(self, prior):
        if prior is None:
            check(_lib.lib().rba_set_camera_pair_prior(self.h, C.c_int32(0), None, None, None))
        else:
            check(_lib.lib().rba_set_camera_pair_prior(self.h, C.c_int32(len(prior[0])), _p(prior[0]), _p(prior[1]), _p(prior[2])))

    def set_landmark_prior(self, prior):
        """Gaussian landmark priors (rba_set_landmark_prior): None, or (idx [m], mean [m,3], sqrt_info [m,3,3]).  Needs a new
        linearize before the next solve; the priors are stored on the BalProblem."""
        self.bal_problem.landmark_prior = prior  # validates and forwards to _upload_landmark_prior

    def _upload_landmark_prior(self, prior):
        if prior is None:
            check(_lib.lib().rba_set_landmark_prior(self.h, 0, None, None, None))
        else:
            check(_lib.lib().rba_set_landmark_prior(self.h, len(prior[0]), _p(prior[0]), _p(prior[1]), _p(prior[2])))

    def set_intrinsics_groups(self, group):
        """intrinsics shared across groups of cameras (rba_set_intrinsics_groups): None, or one int32 group id per camera
        (-1 = own intrinsics).  The members take their lead's f, k1, k2; needs a new linearize before the next solve.  The
        groups are stored on the BalProblem."""
        self.bal_problem.intrinsics_group = group  # validates and forwards to _upload_intrinsics_group

    def _upload_intrinsics_group(self, group):
        check(_lib.lib().rba_set_intrinsics_groups(self.h, None if group is None else _p(group)))

    def set_camera_rigs(self, rig, cam_from_rig=None):
        """rigid camera rigs (rba_set_camera_rigs): rig None, or one int32 rig id per camera (-1 = free camera) with
        cam_from_rig [nc,7] (qx,qy,qz,qw, tx,ty,tz per camera).  The members take M_j T_lead; needs a new linearize before the
        next solve.  The rigs are stored on the BalProblem."""
        self.bal_problem.camera_rig = None if rig is None else (rig, cam_from_rig)  # validates, forwards to _upload_camera_rig

    def _upload_camera_rig(self, rig):
        if rig is None:
            check(_lib.lib().rba_set_camera_rigs(self.h, None, None))
        else:
            check(_lib.lib().rba_set_camera_rigs(self.h, _p(rig[0]), _p(rig[1])))

    def set_rig_sensors(self, sensor):
        """estimated rig extrinsics (rba_set_rig_sensors): None, or one int32 sensor id per camera (-1 = held extrinsics).
        Every member is re-tied from its lead; needs a new linearize before the next solve.  Stored on the BalProblem."""
        self.bal_problem.rig_sensor = sensor  # validates, forwards to _upload_rig_sensor

    def _upload_rig_sensor(self, sensor):
        check(_lib.lib().rba_set_rig_sensors(self.h, None if sensor is None else _p(sensor)))

    def rig_extrinsics(self):
        """[nc, 7] every camera's current cam_from_rig (qx,qy,qz,qw, tx,ty,tz; rba_get_rig_extrinsics): held ones as given,
        an estimated sensor's from the current state, free cameras the identity"""
        out = np.zeros((self.bal_problem.num_cameras(), 7), self.bal_problem.dtype)
        check(_lib.lib().rba_get_rig_extrinsics(self.h, _p(out)))
        return out

    def set_observation_info(self, info):
        """per-observation square-root information (rba_set_observation_info): None, [Nobs] (1 / sigma) or [Nobs,2,2] in the
        order of the problem's observations; zero switches an observation off.  Needs a new linearize before the next solve;
        the information is stored on the BalProblem."""
        self.bal_problem.observation_sqrt_info = info  # validates and forwards to _upload_observation_info

    def _upload_observation_info(self, info):
        check(_lib.lib().rba_set_observation_info(self.h, None if info is None else _p(info)))

    def set_observation_loss(self, kind, scale=1.0):
        """a robust loss per observation (rba_set_observation_loss): kind None (the options' robust_norm everywhere) or a name /
        RBA_LOSS_* int, scalar or [Nobs]; scale scalar or [Nobs], the inlier threshold in units of sigma.  Needs a new linearize
        before the next solve; the losses are stored on the BalProblem."""
        self.bal_problem.observation_loss = None if kind is None else (kind, scale)  # validates, forwards to _upload_observation_loss

    def _upload_observation_loss(self, loss):
        if loss is None:
            check(_lib.lib().rba_set_observation_loss(self.h, None, None))
        else:
            check(_lib.lib().rba_set_observation_loss(self.h, _p(loss[0]), _p(loss[1])))

    @staticmethod
    def _prior_kind(which) -> int:
        if isinstance(which, str):
            if which.lower() not in _lib.PRIOR_KINDS:
                raise ValueError(f"prior kind must be one of {sorted(_lib.PRIOR_KINDS)}, got {which!r}")
            return _lib.PRIOR_KINDS[which.lower()]
        if which not in _lib.PRIOR_ROWS:
            raise ValueError(f"prior kind must be one of {sorted(_lib.PRIOR_ROWS)} (RBA_PRIOR_*), got {which!r}")
        return int(which)

    def set_prior_loss(self, which, kind, scale=1.0):
        """a robust loss per prior of one kind (rba_set_prior_loss): which "camera" | "pair" | "landmark" (or RBA_PRIOR_*
        ints); kind None (NONE on every prior) or a name / RBA_LOSS_* int, scalar or one per camera / pair / landmark prior in
        the order of the kind's prior; scale likewise, the threshold on |L e|.  Needs a new linearize before the next solve;
        the losses are stored on the BalProblem."""
        self.bal_problem._set_prior_loss(self._prior_kind(which), None if kind is None else (kind, scale))

    def _upload_prior_loss(self, which: int, loss):
        n = self.bal_problem._prior_count(which)
        if loss is None:
            check(_lib.lib().rba_set_prior_loss(self.h, which, n, None, None))
        else:
            check(_lib.lib().rba_set_prior_loss(self.h, which, n, _p(loss[0]), _p(loss[1])))

    def prior_residuals(self, which):
        """per prior of one kind at the current state, in the order of the kind's prior (rba_get_prior_residuals):
        (residual [num, 9 | 6 | 3] = L e, robust_weight [num] = w of its loss).  A camera with an all-zero L or a dropped prior
        gives 0 and 1; a sharded handle fills only the landmark priors of its own shard (the others stay 0)."""
        k = self._prior_kind(which)
        n = self.bal_problem._prior_count(k)
        res, w = np.zeros((n, _lib.PRIOR_ROWS[k]), self.dtype), np.zeros(n, self.dtype)
        check(_lib.lib().rba_get_prior_residuals(self.h, k, _p(res), _p(w)))
        return res, w

    def observation_residuals(self):
        """per observation at the current state, in the order of the problem's observations (rba_get_observation_residuals):
        (residual [Nobs,2] = W r, robust_weight [Nobs] (of each observation's own loss), flags [Nobs] uint8: bit 0 = projection valid, bit 1 = in use).  A
        sharded handle fills only the observations of its own landmark shard (the others stay 0)."""
        nobs = self.bal_problem.num_observations()
        res, hw, flags = np.zeros((nobs, 2), self.dtype), np.zeros(nobs, self.dtype), np.zeros(nobs, np.uint8)
        check(_lib.lib().rba_get_observation_residuals(self.h, _p(res), _p(hw), _p(flags)))
        return res, hw, flags

    def triangulate(self, landmarks=None, mode="linear+refine", max_iterations=20, min_angle_deg=0.0,
                    function_tolerance=1e-10):
        """Re-initialise landmark positions from the current cameras, which are held (rba_triangulate_landmarks, DESIGN.md
        section 25).  landmarks None (every landmark) or problem indices; mode "linear", "refine" or "linear+refine" (or the
        RBA_TRIANGULATE_* bits).  Returns (status uint8 RBA_TRI_* bits, angle [rad] the largest angle between two usable rays,
        cost the landmark's share of compute_error at its final position), in the order of `landmarks`, and copies the new
        positions into the BalProblem.  A sharded handle fills only the entries of its own shard (the others stay 0).  Needs a
        new linearize before the next solve."""
        m = _lib.TRIANGULATE_MODES.get(mode, mode) if isinstance(mode, str) else int(mode)
        if isinstance(mode, str) and mode not in _lib.TRIANGULATE_MODES:
            raise ValueError(f"mode must be one of {sorted(_lib.TRIANGULATE_MODES)}, got {mode!r}")
        o = _lib.TriangulateOpts()
        _lib.lib().rba_default_triangulate_opts(C.byref(o))
        o.mode, o.max_iterations = m, int(max_iterations)
        o.min_angle, o.function_tolerance = float(np.deg2rad(min_angle_deg)), float(function_tolerance)
        idx = None if landmarks is None else np.ascontiguousarray(landmarks, np.int32)
        num = self.nl if idx is None else len(idx)
        status, angle, cost = np.zeros(num, np.uint8), np.zeros(num), np.zeros(num)
        check(_lib.lib().rba_triangulate_landmarks(self.h, C.byref(o), int(num), None if idx is None else _p(idx), _p(status),
                                                   _p(angle), _p(cost)))
        self.download_state()
        return status, angle, cost

    def resect(self, cameras=None, mode="linear+refine", intrinsics=False, max_iterations=20, function_tolerance=1e-10):
        """Re-initialise and refine camera poses from the current landmarks, which are held (rba_resect_cameras, DESIGN.md
        section 26).  cameras None (every camera) or camera indices; a camera of a rig stands for its whole rig.  mode
        "linear", "refine" or "linear+refine" (or the RBA_RESECT_* bits); intrinsics also refines the free f, k1, k2 of
        single cameras.  Returns (status uint8 RBA_RES_* bits, points int32 the unit's usable points, cost the unit's share
        of compute_error at its final pose), in the order of `cameras`, and copies the new cameras into the BalProblem.
        Needs a new linearize before the next solve."""
        if isinstance(mode, str) and mode not in _lib.RESECT_MODES:
            raise ValueError(f"mode must be one of {sorted(_lib.RESECT_MODES)}, got {mode!r}")
        m = _lib.RESECT_MODES[mode] if isinstance(mode, str) else int(mode)
        if intrinsics:
            m |= _lib.RESECT_INTRINSICS
        o = _lib.ResectOpts()
        _lib.lib().rba_default_resect_opts(C.byref(o))
        o.mode, o.max_iterations, o.function_tolerance = m, int(max_iterations), float(function_tolerance)
        idx = None if cameras is None else np.ascontiguousarray(cameras, np.int32)
        num = self.nc if idx is None else len(idx)
        status, points, cost = np.zeros(num, np.uint8), np.zeros(num, np.int32), np.zeros(num)
        check(_lib.lib().rba_resect_cameras(self.h, C.byref(o), int(num), None if idx is None else _p(idx), _p(status),
                                            _p(points), _p(cost)))
        self.download_state()
        return status, points, cost

    def _backup(self):
        check(_lib.lib().rba_backup(self.h))

    def _restore(self):
        check(_lib.lib().rba_restore(self.h))

    def comm_init(self, unique_id: bytes):
        buf = C.create_string_buffer(unique_id, 128)
        check(_lib.lib().rba_comm_init(self.h, buf))

    def ipc_export(self) -> bytes:
        buf = C.create_string_buffer(128)
        check(_lib.lib().rba_ipc_export(self.h, buf))
        return buf.raw

    def ipc_import(self, all_handles: bytes):
        buf = C.create_string_buffer(all_handles, len(all_handles))
        check(_lib.lib().rba_ipc_import(self.h, buf))

    # ---- Linearizor interface ----
    def start_iteration(self, it_summary: dict | None = None):
        self.it_summary = it_summary

    def finish_iteration(self):
        pass

    def compute_error(self) -> dict:
        ri = ResidualInfo()
        check(_lib.lib().rba_compute_error(self.h, C.byref(ri)))
        if self.it_summary is not None:
            self.it_summary["residual_evaluation_time"] = self.it_summary.get("residual_evaluation_time", 0.0) + self.timings()["residual_evaluation_time"]
        return {"all": {"num_obs": ri.all_num_obs, "error": ri.all_error, "residual_sum": ri.all_residual_sum},
                "valid": {"num_obs": ri.valid_num_obs, "error": ri.valid_error, "residual_sum": ri.valid_residual_sum},
                "is_numerically_valid": bool(ri.is_numerically_valid)}

    def linearize(self):
        rc = check(_lib.lib().rba_linearize(self.h), allow_numerical_failure=True)
        if rc != 0:
            raise RbaError(rc, "did not expect numerical failure during linearization")  # linearizor_qr.cpp:121-122
        if self.it_summary is not None:
            self.it_summary["stage1_time"] = self.timings()["stage1_time"]

    def solve(self, lam: float, to_host: bool = True):
        inc = np.empty(9 * self.nc, dtype=self.dtype) if to_host else None
        cg = CgSummary()
        check(getattr(_lib.lib(), f"rba_solve_{self.sfx}")(self.h, self.S(lam), None if inc is None else _p(inc), C.byref(cg)))
        self.last_cg = cg
        if self.it_summary is not None:
            t = self.timings()
            self.it_summary.update(stage2_time=t["stage2_time"], compute_preconditioner_time=t["compute_preconditioner_time"],
                                   solve_reduced_system_time=t["solve_reduced_system_time"],
                                   linear_solver_iterations=cg.num_iterations, linear_solver_termination=cg.termination_type)
        return inc

    def apply(self, inc=None) -> float:
        l = self.S(0)
        arr = None if inc is None else np.ascontiguousarray(inc, dtype=self.dtype)
        p = None if arr is None else _p(arr)
        check(getattr(_lib.lib(), f"rba_apply_{self.sfx}")(self.h, p, C.byref(l)), allow_numerical_failure=True)
        if self.it_summary is not None:
            t = self.timings()
            self.it_summary.update(back_substitution_time=t["back_substitution_time"], update_cameras_time=t["update_cameras_time"])
        return float(l.value)

    def lm_step(self, lam: float, linearize_first: bool) -> dict:
        """one LM inner iteration with a single host synchronisation (rba_lm_step): [linearize] + solve + backup + apply +
        compute_error.  Returns the pieces optimize_lm_ours needs; the caller restores on a rejected / failed step."""
        r = LmStepResult()
        check(getattr(_lib.lib(), f"rba_lm_step_{self.sfx}")(self.h, int(linearize_first), self.S(lam), C.byref(r)),
              allow_numerical_failure=True)
        self.last_cg = r.cg
        ri = r.cost
        return {"solve_failed": bool(r.solve_failed), "l_diff": float(r.l_diff),
                "cost": {"all": {"num_obs": ri.all_num_obs, "error": ri.all_error, "residual_sum": ri.all_residual_sum},
                         "valid": {"num_obs": ri.valid_num_obs, "error": ri.valid_error, "residual_sum": ri.valid_residual_sum},
                         "is_numerically_valid": bool(ri.is_numerically_valid)}}

    def lm_run(self, max_steps: int, options: "SolverOptions | None" = None):
        """optimize_lm_ours natively (rba_lm_run): a NEW solve from the current device state, until the reference's stopping rule
        or `max_steps` iterations.  Returns (list of per-iteration dicts, terminated, phase totals in seconds)."""
        o = options or self.options
        lo = LmOpts()
        _lib.lib().rba_default_lm_opts(C.byref(lo))
        lo.initial_trust_region_radius, lo.min_trust_region_radius = o.initial_trust_region_radius, o.min_trust_region_radius
        lo.max_trust_region_radius, lo.min_relative_decrease = o.max_trust_region_radius, o.min_relative_decrease
        lo.initial_vee, lo.vee_factor, lo.function_tolerance = o.initial_vee, o.vee_factor, o.function_tolerance
        lo.max_num_iterations = o.max_num_iterations
        lo.optimized_cost = {"ERROR": 0, "ERROR_VALID": 1, "ERROR_VALID_AVG": 2}[o.optimized_cost]
        log = (LmIteration * max(max_steps, 1))()
        done, term, tot = C.c_int32(), C.c_int32(), StageTimings()
        check(getattr(_lib.lib(), f"rba_lm_run_{self.sfx}")(self.h, C.byref(lo), int(max_steps), log, C.byref(done), C.byref(term), C.byref(tot)),
              allow_numerical_failure=True)
        its = [{"lambda": log[k].lam, "cost": log[k].cost, "l_diff": log[k].l_diff, "relative_decrease": log[k].relative_decrease,
                "device_seconds": log[k].device_seconds, "cg_iterations": log[k].cg_iterations, "cg_termination": log[k].cg_termination,
                "accepted": bool(log[k].accepted), "terminated": bool(log[k].terminated)} for k in range(done.value)]
        return its, bool(term.value), struct_to_dict(tot)

    # ---- LinearizationQR-level access (tests) ----
    def timings(self) -> dict:
        t = StageTimings()
        check(_lib.lib().rba_get_timings(self.h, C.byref(t)))
        return struct_to_dict(t)

    def stats(self) -> dict:
        s = WorkloadStats()
        check(_lib.lib().rba_get_workload_stats(self.h, C.byref(s)))
        return struct_to_dict(s)

    def get_jacobian_scaling(self):
        s, d = np.empty(9 * self.nc, self.dtype), np.empty(9 * self.nc, self.dtype)
        check(_lib.lib().rba_get_jacobian_scaling(self.h, _p(s), _p(d)))
        return s, d

    def get_rhs(self):
        b = np.empty(9 * self.nc, self.dtype)
        check(_lib.lib().rba_get_rhs(self.h, _p(b)))
        return b

    def set_camera_clusters(self, cluster_of_camera):
        """CLUSTER_JACOBI: the clusters of the preconditioner (rba_set_camera_clusters) from the next solve on: None (the
        default clustering), or one int32 cluster id per camera (dense ids, at most RBA_CLUSTER_MAX_CAMERAS per cluster)."""
        c = None if cluster_of_camera is None else np.ascontiguousarray(cluster_of_camera, dtype=np.int32)
        if c is not None and c.shape != (self.nc,):
            raise ValueError(f"cluster_of_camera must have shape ({self.nc},), not {c.shape}")
        check(_lib.lib().rba_set_camera_clusters(self.h, None if c is None else _p(c)))

    def cluster_preconditioner(self):
        """CLUSTER_JACOBI read-back (rba_get_cluster_preconditioner): (cluster_of_camera [nc], blocks, status [ncl]); blocks
        is a list of the last solve's unfactorised (9k, 9k) float64 cluster blocks in cluster order, cameras ascending."""
        L = _lib.lib()
        c = np.empty(self.nc, np.int32)
        check(L.rba_get_cluster_preconditioner(self.h, _p(c), None, None))
        sizes = np.bincount(c)
        flat = np.empty(int(np.sum((9 * sizes) ** 2)), np.float64)
        status = np.empty(len(sizes), np.int32)
        check(L.rba_get_cluster_preconditioner(self.h, None, _p(flat), _p(status)))
        blocks, off = [], 0
        for k in sizes:
            m = 9 * int(k)
            blocks.append(flat[off:off + m * m].reshape(m, m))
            off += m * m
        return c, blocks, status

    def get_preconditioner(self):
        inv, blk = np.empty(81 * self.nc, self.dtype), np.empty(81 * self.nc, self.dtype)
        check(_lib.lib().rba_get_preconditioner(self.h, _p(inv), _p(blk)))
        return inv.reshape(self.nc, 9, 9), blk.reshape(self.nc, 9, 9)

    def right_multiply(self, x):
        x = np.ascontiguousarray(x, dtype=self.dtype)
        y = np.empty_like(x)
        check(_lib.lib().rba_right_multiply(self.h, _p(x), _p(y)))
        return y

    def back_substitute(self, pose_inc) -> float:
        pose_inc = np.ascontiguousarray(pose_inc, dtype=self.dtype)
        l = self.S(0)
        check(getattr(_lib.lib(), f"rba_back_substitute_{self.sfx}")(self.h, _p(pose_inc), C.byref(l)),
              allow_numerical_failure=True)
        return float(l.value)

    def debug_get_block(self, lm: int):
        n = int(self.bal_problem.lm_off[lm + 1] - self.bal_problem.lm_off[lm])
        pad = (4 - (9 * n) % 4) % 4
        rows, cols = 2 * n + 3, 9 * n + pad + 4
        out = np.zeros((rows, cols), self.dtype)
        jls = np.zeros(3, self.dtype)
        check(_lib.lib().rba_debug_get_block(self.h, C.c_int32(lm), _p(out), rows, cols, _p(jls)))
        return out, 9 * n + pad, 9 * n + pad + 3, jls

    def covariance(self, landmarks: bool = True):
        """marginal covariances at the current state (rba_compute_covariance, DESIGN.md section 16): float64 arrays
        (cam [nc, 9, 9] in the increment order tx,ty,tz, rx,ry,rz, f,k1,k2;  lm [nl, 3, 3], or None without landmarks).
        Raises RbaError (code RBA_NUMERICAL_FAILURE) when the reduced camera matrix is singular (gauge not fixed)."""
        cam = np.empty((self.nc, 9, 9), np.float64)
        lm = np.empty((self.nl, 3, 3), np.float64) if landmarks else None
        check(_lib.lib().rba_compute_covariance(self.h, cam.ctypes.data, None if lm is None else lm.ctypes.data))
        return cam, lm

    def covariance_blocks(self, cameras=None, camera_landmark=None, landmarks=None, relative=None, marginals: bool = False):
        """covariance blocks of chosen pairs at the current state from one factorisation (rba_compute_covariance_blocks,
        DESIGN.md section 20).  Each request argument is an int array [m, 2] or None: cameras (a, b) -> 'cameras' [m, 9, 9]
        Cov(d_a, d_b); camera_landmark (c, l) -> 'camera_landmark' [m, 9, 3]; landmarks (l, m) -> 'landmarks' [m, 3, 3];
        relative (i, j), i != j -> 'relative' [m, 6, 6], the covariance of the pair-prior residual (e_t, e_r) at the current
        relative pose.  marginals=True adds 'cam' [nc, 9, 9] and 'lm' [nl, 3, 3], exactly covariance()'s.  float64 arrays;
        raises RbaError like covariance() (code -1 for an invalid request)."""
        q = _lib.CovarianceQuery()
        out, keep = {}, []
        for key, req, count, src, dst, shape in (("cameras", cameras, "num_camera_pairs", "camera_pairs", "camera_cross", (9, 9)),
                                                 ("camera_landmark", camera_landmark, "num_camera_landmark", "camera_landmark",
                                                  "camera_landmark_cross", (9, 3)),
                                                 ("landmarks", landmarks, "num_landmark_pairs", "landmark_pairs", "landmark_cross", (3, 3)),
                                                 ("relative", relative, "num_relative_poses", "relative_pairs", "relative_cov", (6, 6))):
            if req is None:
                continue
            r = np.ascontiguousarray(np.asarray(req).reshape(-1, 2), dtype=np.int32)
            o = np.empty((len(r),) + shape, np.float64)
            keep.append(r)
            setattr(q, count, len(r))
            setattr(q, src, r.ctypes.data if len(r) else None)
            setattr(q, dst, o.ctypes.data if len(r) else None)
            out[key] = o
        if marginals:
            out["cam"] = np.empty((self.nc, 9, 9), np.float64)
            out["lm"] = np.empty((self.nl, 3, 3), np.float64)
            q.cam_cov, q.lm_cov = out["cam"].ctypes.data, out["lm"].ctypes.data
        check(_lib.lib().rba_compute_covariance_blocks(self.h, C.byref(q)))
        return out

    def timer_start(self):
        check(_lib.lib().rba_timer_start(self.h))

    def timer_stop(self) -> float:
        s = C.c_double()
        check(_lib.lib().rba_timer_stop(self.h, C.byref(s)))
        return s.value

    def time_matvec(self, reps: int = 20) -> float:
        s = C.c_double()
        check(_lib.lib().rba_time_matvec(self.h, reps, C.byref(s)))
        return s.value


def nccl_unique_id() -> bytes:
    buf = C.create_string_buffer(128)
    check(_lib.lib().rba_nccl_unique_id(buf))
    return buf.raw


def cluster_cameras(bal_problem: BalProblem, max_size: int) -> np.ndarray:
    """rba_cluster_cameras: the cameras clustered by single linkage over the co-visibility graph (edge weight = shared
    landmarks), at most max_size cameras per cluster; dense int32 ids numbered by their smallest camera.  Host code only."""
    out = np.empty(bal_problem.num_cameras(), np.int32)
    pv = ProblemView(bal_problem.num_cameras(), bal_problem.num_landmarks(), bal_problem.num_observations(),
                     bal_problem.lm_off.ctypes.data, bal_problem.obs_cam.ctypes.data, bal_problem.obs_xy.ctypes.data)
    check(_lib.lib().rba_cluster_cameras(C.byref(pv), C.c_int32(max_size), _p(out)))
    return out


def partition_landmarks(lm_off: np.ndarray, nranks: int) -> np.ndarray:
    lm_off = np.ascontiguousarray(lm_off, dtype=np.int64)
    bounds = np.zeros(nranks + 1, dtype=np.int32)
    check(_lib.lib().rba_partition_landmarks(C.c_int32(lm_off.shape[0] - 1), _p(lm_off), C.c_int32(nranks), _p(bounds)))
    return bounds


def _p(a):
    return C.c_void_p(a.ctypes.data)


def _cost(ri: dict, optimized_cost: str) -> float:
    if optimized_cost == "ERROR":
        return ri["all"]["error"]
    if optimized_cost == "ERROR_VALID":
        return ri["valid"]["error"]
    n = ri["valid"]["num_obs"]
    return ri["valid"]["error"] / n if n > 0 else 0.0


def bundle_adjust_manual(bal_problem: BalProblem, solver_options: SolverOptions, linearizor=None, verbose=False,
                         comm_setup=None) -> dict:
    """rootba::bundle_adjust_manual -> optimize_lm_ours (solver/bal_bundle_adjustment.cpp:249-544):
    the host-serial LM trust-region loop, unchanged, driving a Linearizor."""
    o = solver_options
    S = np.float32 if bal_problem.dtype == np.float32 else np.float64
    min_lambda = S(1.0 / o.max_trust_region_radius)
    max_lambda = S(1.0 / o.min_trust_region_radius)
    vee_factor, initial_vee = S(o.vee_factor), S(o.initial_vee)
    lam = S(1.0 / o.initial_trust_region_radius)
    lambda_vee = initial_vee
    summary = {"iterations": [], "num_linear_solves": 0, "num_residual_evaluations": 0, "num_jacobian_evaluations": 0,
               "termination_type": "NO_CONVERGENCE", "message": ""}
    t_total = time.perf_counter()
    own = linearizor is None
    if own:
        linearizor = LinearizorQR.create(bal_problem, o, summary)
        if comm_setup is not None:
            comm_setup(linearizor)
    summary["preprocessor_time"] = time.perf_counter() - t_total
    t_iter = [time.perf_counter()]

    def log_iteration(s):  # finish_iteration (bal_bundle_adjustment.cpp:56-88): wall-clock stamps, then push
        now = time.perf_counter()
        s["iteration_time"], s["cumulative_time"] = now - t_iter[0], now - t_total
        t_iter[0] = now
        summary["iterations"].append(s)
    terminated = False
    it = 0
    max_lm_iter = o.max_num_iterations
    try:
        _lm_loop(bal_problem, o, S, linearizor, summary, log_iteration, min_lambda, max_lambda, vee_factor, initial_vee, lam, lambda_vee,
                 max_lm_iter, verbose)
    except BaseException:
        if own:
            linearizor.close()  # do not leak the device handle when the loop raises (numerical failure during linearisation ...)
        raise
    bal_problem.sync_from_device()
    summary["total_time"] = time.perf_counter() - t_total
    summary["minimizer_time"] = summary["total_time"] - summary["preprocessor_time"]
    if own:
        summary["stats"] = linearizor.stats()
        linearizor.close()
    return summary


def _lm_loop(bal_problem, o, S, linearizor, summary, log_iteration, min_lambda, max_lambda, vee_factor, initial_vee, lam, lambda_vee,
             max_lm_iter, verbose):
    """the body of optimize_lm_ours (solver/bal_bundle_adjustment.cpp:291-521)"""
    terminated = False
    it = 0
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        while it <= max_lm_iter and not terminated:
            it_summary = {"iteration": it}
            linearizor.start_iteration(it_summary)
            ri = linearizor.compute_error()
            summary["num_residual_evaluations"] += 1
            if not ri["is_numerically_valid"]:
                raise RbaError(1, "did not expect numerical failure during linearization")  # :307-308
            if it == 0:
                linearizor.finish_iteration()
                it_summary.update(cost=ri, trust_region_radius=1 / float(lam), step_is_successful=True, step_is_valid=True,
                                  lam=float(lam))
                log_iteration(it_summary)
                it += 1
                continue
            linearizor.linearize()
            summary["num_jacobian_evaluations"] += 1
            j = 0
            while it <= max_lm_iter and not terminated:
                if j > 0:
                    it_summary = {"iteration": it}
                    linearizor.start_iteration(it_summary)
                j += 1
                inc = linearizor.solve(float(lam))
                summary["num_linear_solves"] += 1
                it_summary["lam"] = float(lam)
                if not np.all(np.isfinite(inc)):
                    it_summary.update(step_is_valid=False, step_is_successful=False)
                    lam = S(lambda_vee * lam)
                    lambda_vee = S(lambda_vee * vee_factor)
                    linearizor.finish_iteration()
                    it_summary["trust_region_radius"] = 1 / float(lam)
                    log_iteration(it_summary)
                    it += 1
                    if lam > max_lambda:
                        terminated = True
                        summary["message"] = "Solver did not converge and reached maximum damping lambda"
                    continue
                bal_problem.backup()
                l_diff = S(linearizor.apply(inc))
                ri2 = linearizor.compute_error()
                summary["num_residual_evaluations"] += 1
                it_summary["cost"] = ri2
                it_summary["l_diff"] = float(l_diff)
                if not math.isfinite(float(l_diff)) or not ri2["is_numerically_valid"]:
                    it_summary.update(step_is_valid=False, step_is_successful=False)
                else:
                    f_diff = S(_cost(ri, o.optimized_cost) - _cost(ri2, o.optimized_cost))
                    if o.optimized_cost == "ERROR_VALID_AVG":
                        l_diff = S(l_diff / ri["valid"]["num_obs"])
                    step_quality = S(f_diff / l_diff)
                    it_summary["relative_decrease"] = float(step_quality)
                    it_summary["step_is_valid"] = bool(l_diff > 0)
                    it_summary["step_is_successful"] = bool(it_summary["step_is_valid"] and step_quality > o.min_relative_decrease)
                if it_summary["step_is_successful"]:
                    lam = S(lam * S(max(1.0 / 3, 1 - (2 * it_summary["relative_decrease"] - 1) ** 3)))
                    lam = max(min_lambda, lam)
                    lambda_vee = initial_vee
                    linearizor.finish_iteration()
                    it_summary["trust_region_radius"] = 1 / float(lam)
                    zero = {"all": {"num_obs": 0, "error": 0.0}, "valid": {"num_obs": 0, "error": 0.0}}
                    prev = _cost(summary["iterations"][-1].get("cost", zero), "ERROR" if o.optimized_cost == "ERROR" else "ERROR_VALID")
                    cur = _cost(ri2, "ERROR" if o.optimized_cost == "ERROR" else "ERROR_VALID")
                    log_iteration(it_summary)
                    it += 1
                    if abs(prev - cur) <= o.function_tolerance * cur:  # :174-201
                        terminated = True
                        summary["termination_type"] = "CONVERGENCE"
                        summary["message"] = "Function tolerance reached."
                    if verbose:
                        print(f"  it {it - 1}: cost {cur:.6e} lambda {float(lam):.1e} cg {it_summary.get('linear_solver_iterations')}")
                    break
                else:
                    lam = S(lambda_vee * lam)
                    lambda_vee = S(lambda_vee * vee_factor)
                    linearizor.finish_iteration()
                    it_summary["trust_region_radius"] = 1 / float(lam)
                    log_iteration(it_summary)
                    bal_problem.restore()
                    it += 1
                    if lam > max_lambda:
                        terminated = True
                        summary["message"] = "Solver did not converge and reached maximum damping lambda"
    if not terminated:
        summary["message"] = f"Solver did not converge after maximum number of {max_lm_iter} iterations"
