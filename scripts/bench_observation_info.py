#!/usr/bin/env python
"""bench.py's flagship measurement with per-observation square-root information (rba_set_observation_info, DESIGN.md
section 19).

    python scripts/bench_observation_info.py [--rounds R] --gpus 1 --steps K --warmup W [any other bench.py option of the CUDA arm]

Runs bench.py's own protocol on its workload (at --gpus 1 the Ladybug-1723 stand-in) in three arms, alternating arm by arm
for R rounds (default 2) in one call, each arm a fresh process:

  none           no observation information: the unmodified kernels
  near_identity  W = (1 + 2^-20) I on every observation.  Not the identity bit for bit, so the flagged kernel instances run
                 and the whole cost of the path is paid, while the LM trajectory stays that of `none` up to rounding: the
                 two arms' milliseconds per LM iteration are comparable
  octaves        W = I / sigma, sigma drawn per observation from {1, 1.2, 1.44, 1.73} (keypoint noise growing with the
                 pyramid level) by a seed.  This changes the LM trajectory, so its milliseconds per LM iteration are
                 reported, not compared with `none`

Prints one JSON line: per arm and round the stage-1 time and the milliseconds per LM iteration, the microseconds per PCG
iteration (no kernel of the PCG iteration reads the information) and the PCG iterations, with the card's name and power
limit read in the same call.
"""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

SIGMAS = (1.0, 1.2, 1.44, 1.73)
SEED = 19
ARMS = {"none": "none", "near_identity": "W = (1 + 2^-20) I on every observation",
        "octaves": f"W = I / sigma, sigma drawn per observation from {SIGMAS} (seed {SEED})"}


def observation_info(arm, nobs):
    """None, or [nobs] (1 / sigma) of the arm"""
    if arm == "none":
        return None
    if arm == "near_identity":
        return np.full(nobs, 1.0 + 2.0 ** -20)
    return 1.0 / np.random.default_rng(SEED).choice(SIGMAS, nobs)


def run_arm(arm):
    """inner process: bench.py's main with every BalProblem it builds carrying the arm's information"""
    import bench
    from rootba_b200.linearizor import BalProblem
    plain_from_arrays = BalProblem.from_arrays.__func__
    plain_config = bench.workload_config

    def from_arrays_with_info(cls, arrays, dtype=np.float64):
        bp = plain_from_arrays(cls, arrays, dtype)
        bp.observation_sqrt_info = observation_info(arm, bp.num_observations())
        return bp

    def config_with_info(args, arrays):
        cfg = plain_config(args, arrays)
        cfg["observation_info"] = ARMS[arm]
        return cfg

    BalProblem.from_arrays = classmethod(from_arrays_with_info)
    bench.workload_config = config_with_info
    bench.main()


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    if q.returncode != 0:
        sys.exit("bench_observation_info.py: nvidia-smi found no GPU; this measurement needs an H100")
    name, power = [s.strip() for s in q.stdout.strip().split("\n")[0].split(",")]
    return name, power


def main():
    if "--arm" in sys.argv:
        i = sys.argv.index("--arm")
        arm = sys.argv[i + 1]
        del sys.argv[i:i + 2]
        return run_arm(arm)
    if "--impl" in sys.argv and "reference" in sys.argv:
        sys.exit("bench_observation_info.py: the reference has no observation information")
    rounds = 2
    args = sys.argv[1:]
    if "--rounds" in args:
        i = args.index("--rounds")
        rounds = int(args[i + 1])
        del args[i:i + 2]
    name, power = card()
    out = {"card": name, "power_limit": power, "rounds": rounds, "arms": {a: [] for a in ARMS}}
    for _ in range(rounds):
        for arm in ARMS:
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--arm", arm, *args], capture_output=True, text=True, cwd=ROOT)
            lines = [ln for ln in p.stdout.splitlines() if ln.startswith("{")]
            if p.returncode != 0 or not lines:
                sys.exit(f"arm {arm} failed:\n{p.stdout[-2000:]}\n{p.stderr[-2000:]}")
            r = json.loads(lines[-1])
            out["arms"][arm].append({"ms_per_lm_iteration": r["ms_per_step"], "stage1_ms_per_lm_iteration": r["phases_ms_per_step"]["stage1_time"],
                                     "pcg_us_per_iteration": r["pcg"]["us_per_iteration"], "pcg_iterations": r["pcg"]["iterations"]})
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
