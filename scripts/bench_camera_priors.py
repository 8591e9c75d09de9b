#!/usr/bin/env python
"""bench.py's flagship measurement with a Gaussian prior on every camera centre (rba_set_camera_prior, DESIGN.md section 14).

    python scripts/bench_camera_priors.py --gpus 1 --steps K --warmup W [--pair-priors] [any other bench.py option of the CUDA arm]

Runs bench.py's own protocol and prints its JSON result line.  The only differences: every BalProblem bench.py builds from the
workload carries a centre prior at the camera's initial centre (standard deviation SIGMA scene units per axis, nothing on the
rotation and the intrinsics), and `config.camera_priors` says so.  Run it alternately with bench.py in the same session to
compare the two; the priors change the LM trajectory, so compare microseconds per PCG iteration (`pcg.us_per_iteration`),
not milliseconds per LM iteration.

--pair-priors also puts a relative pose prior (rba_set_camera_pair_prior, DESIGN.md section 15) between consecutive cameras
(i, i + 1) at their initial relative pose: standard deviation PAIR_SIGMA_T scene units on the translation, PAIR_SIGMA_R rad on
the rotation.  Without it the script behaves as before.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench  # noqa: E402
from rootba_b200.linearizor import BalProblem  # noqa: E402

SIGMA = 1.0
PAIR_SIGMA_T, PAIR_SIGMA_R = 1.0, 0.01


def camera_centre_priors(arrays, sigma=SIGMA):
    """(mean [nc, 10], sqrt_info [nc, 9, 9]): a prior on every camera centre c = -R^T t at its initial value, 1 / sigma on
    the centre rows, nothing on the rotation and the intrinsics"""
    cams = np.asarray(arrays.cams, np.float64)
    q = cams[:, :4] / np.linalg.norm(cams[:, :4], axis=1, keepdims=True)
    x, y, z, w = q.T
    R = np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], -1),
                  np.stack([2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)], -1),
                  np.stack([2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], -1)], 1)
    mean = cams.copy()
    mean[:, :4] = q
    mean[:, 4:7] = -np.einsum("cji,cj->ci", R, cams[:, 4:7])
    L = np.zeros((len(cams), 9, 9))
    L[:, [0, 1, 2], [0, 1, 2]] = 1.0 / sigma
    return mean, L


def _rotations(cams):
    q = cams[:, :4] / np.linalg.norm(cams[:, :4], axis=1, keepdims=True)
    x, y, z, w = q.T
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], -1),
                     np.stack([2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)], -1),
                     np.stack([2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], -1)], 1)


def consecutive_pair_priors(arrays):
    """(pairs [nc-1, 2], mean [nc-1, 7], sqrt_info [nc-1, 6, 6]): a pair prior between cameras i and i + 1 at their initial
    relative pose T_i T_{i+1}^-1 = (R_i R_{i+1}^T, t_i - R_i R_{i+1}^T t_{i+1})"""
    from scipy.spatial.transform import Rotation
    cams = np.asarray(arrays.cams, np.float64)
    R = _rotations(cams)
    M = np.einsum("cab,cdb->cad", R[:-1], R[1:])
    pairs = np.stack([np.arange(len(cams) - 1), np.arange(1, len(cams))], 1).astype(np.int32)
    mean = np.zeros((len(pairs), 7))
    mean[:, :4] = Rotation.from_matrix(M).as_quat()
    mean[:, 4:7] = cams[:-1, 4:7] - np.einsum("cab,cb->ca", M, cams[1:, 4:7])
    L = np.tile(np.diag([1 / PAIR_SIGMA_T] * 3 + [1 / PAIR_SIGMA_R] * 3), (len(pairs), 1, 1))
    return pairs, mean, L


def main():
    if "--impl" in sys.argv and "reference" in sys.argv:
        sys.exit("bench_camera_priors.py: the reference has no camera priors; run bench.py --impl reference for that arm")
    pair = "--pair-priors" in sys.argv
    if pair:
        sys.argv.remove("--pair-priors")  # not a bench.py option
    plain_from_arrays = BalProblem.from_arrays.__func__
    plain_config = bench.workload_config

    def from_arrays_with_priors(cls, arrays, dtype=np.float64):
        bp = plain_from_arrays(cls, arrays, dtype)
        bp.camera_prior = camera_centre_priors(arrays)
        if pair:
            bp.camera_pair_prior = consecutive_pair_priors(arrays)
        return bp

    def config_with_priors(args, arrays):
        cfg = plain_config(args, arrays)
        cfg["camera_priors"] = f"centre prior on every camera at its initial centre, sigma {SIGMA} per axis"
        if pair:
            cfg["camera_pair_priors"] = (f"pair prior between consecutive cameras at their initial relative pose, sigma "
                                         f"{PAIR_SIGMA_T} on translation, {PAIR_SIGMA_R} rad on rotation")
        return cfg

    # bench.py builds its problems through BalProblem.from_arrays and its config through workload_config
    BalProblem.from_arrays = classmethod(from_arrays_with_priors)
    bench.workload_config = config_with_priors
    bench.main()


if __name__ == "__main__":
    main()
