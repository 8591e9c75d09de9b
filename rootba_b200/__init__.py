"""rootba_b200 -- H100-native square-root bundle-adjustment inner loop (drop-in for rootba's LinearizorQR path).

The compute path is the CUDA library rootba_b200/librootba_b200.so (C ABI: include/rootba_b200.h).
Python here is only the host-side mirror of the reference interface and the synthetic-data generator.
"""
from .linearizor import (BalProblem, LinearizorQR, ResidualOptions, SolverOptions, bundle_adjust_manual,  # noqa: F401
                         cluster_cameras, nccl_unique_id, partition_landmarks)
from ._lib import FIX_ALL, FIX_F, FIX_INTRINSICS, FIX_K1, FIX_K2, FIX_POSE, RbaError, build  # noqa: F401
from .ba_log import make_ba_log, save_ba_log, summarize_problem  # noqa: F401
