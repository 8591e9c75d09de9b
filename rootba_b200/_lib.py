"""ctypes binding of the C ABI (include/rootba_b200.h) implemented by rootba_b200/librootba_b200.so.

There is no CPU or PyTorch fallback: if the CUDA extension is missing or no CUDA device is visible,
creating a solver raises.  (The library itself loads on a CPU-only box so that its exported symbols can
be checked.)
"""
from __future__ import annotations

import ctypes as C
import os
import re
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("RBA_LIB", os.path.join(_HERE, "librootba_b200.so"))
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "rootba_b200.h")

RBA_OK = 0
RBA_NUMERICAL_FAILURE = 1

# camera parameters held constant, one byte of bits per camera (RBA_FIX_*, rba_set_camera_fixed)
FIX_POSE = 1        # rotation and translation (increment entries 0..5)
FIX_F = 2           # focal length (entry 6)
FIX_K1 = 4          # entry 7
FIX_K2 = 8          # entry 8
FIX_INTRINSICS = FIX_F | FIX_K1 | FIX_K2
FIX_ALL = FIX_POSE | FIX_INTRINSICS

# robust loss kinds per observation (RBA_LOSS_*, rba_set_observation_loss)
LOSS_NONE = 0
LOSS_HUBER = 1
LOSS_CAUCHY = 2
LOSS_SOFT_L1 = 3
LOSS_TUKEY = 4
LOSS_KINDS = {"NONE": LOSS_NONE, "HUBER": LOSS_HUBER, "CAUCHY": LOSS_CAUCHY, "SOFT_L1": LOSS_SOFT_L1, "TUKEY": LOSS_TUKEY}

# prior kinds of rba_set_prior_loss / rba_get_prior_residuals (RBA_PRIOR_*) and the rows of L e of each
PRIOR_CAMERA = 0
PRIOR_PAIR = 1
PRIOR_LANDMARK = 2
PRIOR_KINDS = {"camera": PRIOR_CAMERA, "pair": PRIOR_PAIR, "landmark": PRIOR_LANDMARK}
PRIOR_ROWS = {PRIOR_CAMERA: 9, PRIOR_PAIR: 6, PRIOR_LANDMARK: 3}

# rba_triangulate_landmarks: mode bits (RBA_TRIANGULATE_*) and status bits (RBA_TRI_*)
TRIANGULATE_LINEAR = 1
TRIANGULATE_REFINE = 2
TRIANGULATE_MODES = {"linear": TRIANGULATE_LINEAR, "refine": TRIANGULATE_REFINE,
                     "linear+refine": TRIANGULATE_LINEAR | TRIANGULATE_REFINE}
TRI_WRITTEN = 1
TRI_FEW_RAYS = 2
TRI_SMALL_ANGLE = 4
TRI_AT_INFINITY = 8
TRI_BEHIND = 16
TRI_REFINED = 32
TRI_CONVERGED = 64

# rba_resect_cameras: mode bits (RBA_RESECT_*) and status bits (RBA_RES_*)
RESECT_LINEAR = 1
RESECT_REFINE = 2
RESECT_INTRINSICS = 4
RESECT_MODES = {"linear": RESECT_LINEAR, "refine": RESECT_REFINE, "linear+refine": RESECT_LINEAR | RESECT_REFINE}
RES_WRITTEN = 1
RES_FEW_POINTS = 2
RES_DEGENERATE = 4
RES_BEHIND = 8
RES_REFINED = 16
RES_CONVERGED = 32
RES_HELD = 64


class RbaError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"rootba_b200 error {code}: {msg}")
        self.code = code


class ProblemView(C.Structure):
    _fields_ = [("num_cameras", C.c_int32), ("num_landmarks", C.c_int32), ("num_observations", C.c_int64),
                ("lm_obs_offset", C.c_void_p), ("obs_cam_idx", C.c_void_p), ("obs_xy", C.c_void_p)]


class SolverOpts(C.Structure):
    _fields_ = [("use_householder_marginalization", C.c_int32), ("use_valid_projections_only", C.c_int32),
                ("robust_norm", C.c_int32), ("huber_parameter", C.c_double), ("jacobi_scaling_epsilon", C.c_double),
                ("preconditioner_type", C.c_int32), ("min_linear_solver_iterations", C.c_int32),
                ("max_linear_solver_iterations", C.c_int32), ("eta", C.c_double),
                ("residual_reset_period", C.c_int32), ("device", C.c_int32), ("rank", C.c_int32),
                ("nranks", C.c_int32), ("pcg_check_period", C.c_int32), ("use_cuda_graphs", C.c_int32),
                ("operator_form", C.c_int32), ("stage2_form", C.c_int32), ("solver_type", C.c_int32), ("power_order", C.c_int32),
                ("linear_solver_type", C.c_int32), ("reserved", C.c_int32 * 1)]


class ResidualInfo(C.Structure):
    _fields_ = [("all_num_obs", C.c_int64), ("all_error", C.c_double), ("all_residual_sum", C.c_double),
                ("valid_num_obs", C.c_int64), ("valid_error", C.c_double), ("valid_residual_sum", C.c_double),
                ("is_numerically_valid", C.c_int32), ("pad_", C.c_int32)]


class CgSummary(C.Structure):
    _fields_ = [("termination_type", C.c_int32), ("num_iterations", C.c_int32), ("num_matvecs", C.c_int32),
                ("reason", C.c_int32)]


class LmStepResult(C.Structure):
    _fields_ = [("cg", CgSummary), ("l_diff", C.c_double), ("cost", ResidualInfo), ("solve_failed", C.c_int32), ("pad_", C.c_int32)]


class LmOpts(C.Structure):
    _fields_ = [("initial_trust_region_radius", C.c_double), ("min_trust_region_radius", C.c_double), ("max_trust_region_radius", C.c_double),
                ("min_relative_decrease", C.c_double), ("initial_vee", C.c_double), ("vee_factor", C.c_double),
                ("function_tolerance", C.c_double), ("max_num_iterations", C.c_int32), ("optimized_cost", C.c_int32)]


class LmIteration(C.Structure):
    _fields_ = [("lam", C.c_double), ("cost", C.c_double), ("l_diff", C.c_double), ("relative_decrease", C.c_double),
                ("device_seconds", C.c_double), ("cg_iterations", C.c_int32), ("cg_termination", C.c_int32),
                ("accepted", C.c_int32), ("terminated", C.c_int32)]


class StageTimings(C.Structure):
    _fields_ = [("stage1_time", C.c_double), ("stage2_time", C.c_double),
                ("compute_preconditioner_time", C.c_double), ("solve_reduced_system_time", C.c_double),
                ("back_substitution_time", C.c_double), ("update_cameras_time", C.c_double),
                ("residual_evaluation_time", C.c_double), ("matvec_time", C.c_double),
                ("matvec_launches", C.c_int64), ("kernel_launches", C.c_int64)]


class WorkloadStats(C.Structure):
    _fields_ = [("num_landmarks_local", C.c_int64), ("num_observations_local", C.c_int64), ("sum_n2", C.c_int64),
                ("max_n", C.c_int32), ("num_tiles", C.c_int32), ("panel_scalars", C.c_int64),
                ("panel_scalars_algorithmic", C.c_int64), ("device_bytes", C.c_int64),
                ("matvec_algorithmic_bytes", C.c_int64), ("landmark_begin", C.c_int32),
                ("landmark_end", C.c_int32), ("num_matvec_items", C.c_int32), ("reserved_", C.c_int32)]


class CovarianceQuery(C.Structure):
    _fields_ = [("num_camera_pairs", C.c_int32), ("num_camera_landmark", C.c_int32), ("num_landmark_pairs", C.c_int32),
                ("num_relative_poses", C.c_int32), ("camera_pairs", C.c_void_p), ("camera_landmark", C.c_void_p),
                ("landmark_pairs", C.c_void_p), ("relative_pairs", C.c_void_p), ("camera_cross", C.c_void_p),
                ("camera_landmark_cross", C.c_void_p), ("landmark_cross", C.c_void_p), ("relative_cov", C.c_void_p),
                ("cam_cov", C.c_void_p), ("lm_cov", C.c_void_p)]


class TriangulateOpts(C.Structure):
    _fields_ = [("mode", C.c_int32), ("max_iterations", C.c_int32), ("min_angle", C.c_double),
                ("function_tolerance", C.c_double), ("reserved", C.c_int32 * 2)]


class ResectOpts(C.Structure):
    _fields_ = [("mode", C.c_int32), ("max_iterations", C.c_int32), ("function_tolerance", C.c_double),
                ("reserved", C.c_int32 * 2)]


def struct_to_dict(s: C.Structure) -> dict:
    out = {}
    for name, _ in s._fields_:
        v = getattr(s, name)
        if isinstance(v, (int, float)):
            out[name] = v
    return out


def build(force: bool = False) -> str:
    """Compile the CUDA extension in-tree for sm_90a (nvcc cross-compiles without a GPU)."""
    src_dir = os.path.join(_HERE, "csrc")
    if force and os.path.exists(LIB_PATH):
        os.remove(LIB_PATH)
    subprocess.check_call(["make", "-C", src_dir, "-s"])  # make knows every dependency (kernels, layout, host loaders, header)
    return LIB_PATH


def declared_symbols() -> list[str]:
    """every function the public header declares"""
    txt = open(HEADER_PATH).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(rba_[a-z0-9_]+)\s*\(", txt)))


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RbaError(-100, f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                                 "(there is no CPU fallback)")
        _lib = C.CDLL(LIB_PATH)
        _lib.rba_last_error.restype = C.c_char_p
        _lib.rba_stream.restype = C.c_void_p
        _lib.rba_compute_covariance.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        _lib.rba_compute_covariance_blocks.argtypes = [C.c_void_p, C.POINTER(CovarianceQuery)]
        _lib.rba_set_landmark_prior.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib.rba_set_observation_loss.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        _lib.rba_set_prior_loss.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
        _lib.rba_get_prior_residuals.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
        _lib.rba_set_camera_rigs.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        _lib.rba_set_rig_sensors.argtypes = [C.c_void_p, C.c_void_p]
        _lib.rba_get_rig_extrinsics.argtypes = [C.c_void_p, C.c_void_p]
        _lib.rba_default_triangulate_opts.argtypes = [C.POINTER(TriangulateOpts)]
        _lib.rba_default_triangulate_opts.restype = None
        _lib.rba_triangulate_landmarks.argtypes = [C.c_void_p, C.POINTER(TriangulateOpts), C.c_int32, C.c_void_p, C.c_void_p,
                                                   C.c_void_p, C.c_void_p]
        _lib.rba_default_resect_opts.argtypes = [C.POINTER(ResectOpts)]
        _lib.rba_default_resect_opts.restype = None
        _lib.rba_resect_cameras.argtypes = [C.c_void_p, C.POINTER(ResectOpts), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_void_p]
    return _lib


def check(rc: int, allow_numerical_failure: bool = False) -> int:
    if rc == RBA_OK or (allow_numerical_failure and rc == RBA_NUMERICAL_FAILURE):
        return rc
    raise RbaError(rc, (lib().rba_last_error() or b"").decode())
