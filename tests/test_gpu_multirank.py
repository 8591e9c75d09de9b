"""GPU multi-rank parity (SURVEY 8e): the landmark-sharded CUDA path on 2 GPUs of one box against the single-rank CPU oracle,
through both exchange paths -- the peer-memory exchange over NVLink fused into the PCG kernels (default) and NCCL
all-reduces (RBA_PEER_AR=0).  Skipped on a box with fewer than 2 GPUs."""
import json

import pytest

from objective_checks import run_two_ranks

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("peer", ["1", "0"])
@pytest.mark.parametrize("sfx", ["f32", "f64"])
def test_two_ranks_against_oracle(tmp_path, peer, sfx):
    res = run_two_ranks(tmp_path, "multirank_gpu_worker.py", sfx, peer, 29500, (7 if peer == "1" else 0) + (13 if sfx == "f32" else 0))
    tol1, tols, tolb = (1e-5, 1e-4, 1e-4) if sfx == "f32" else (1e-11, 1e-8, 1e-8)
    print("multirank result", json.dumps(res))
    assert res["cams_without_obs_here"] > 0, res
    assert res["replicas_identical"] and res["Hx_repeat_identical"], res
    assert res["error"][0] == res["error"][1] and res["error"][2] < 20 * tol1, res
    assert res["b"] < 4 * tol1 and res["Hx"] < 4 * tol1 and res["inv"] < tolb, res
    assert abs(res["cg"][0] - res["cg"][1]) <= 2 and res["cg_term"][0] == res["cg_term"][1], res
    assert res["inc"] < tols and res["l_diff"] < 20 * tols, res
    assert res["lms"] < 10 * tols and res["cams"] < tols and res["error_after"] < 100 * tols, res
