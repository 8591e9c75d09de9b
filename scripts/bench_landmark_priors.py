#!/usr/bin/env python
"""bench.py's flagship measurement with Gaussian priors on landmark positions (rba_set_landmark_prior, DESIGN.md section 17).

    python scripts/bench_landmark_priors.py [--rounds R] --gpus 1 --steps K --warmup W [any other bench.py option of the CUDA arm]

Runs bench.py's own protocol on its workload (at --gpus 1 the Ladybug-1723 stand-in) in three arms -- no landmark priors,
priors on 1 % of the landmarks (every 100th), priors on every landmark -- alternating arm by arm for R rounds (default 2)
in one call, each arm a fresh process.  A prior sits at the landmark's initial position with standard deviation SIGMA scene
units per axis.  Prints one JSON line: per arm and round the stage-2 time and the milliseconds per LM iteration (the priors
change the LM trajectory, so these differ for that reason too) and the microseconds per PCG iteration (the priors leave
the PCG iteration unchanged), with the card's name and power limit read in the same call.
"""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

SIGMA = 1.0
ARMS = {"none": None, "one_percent": 100, "every_landmark": 1}


def landmark_priors(arrays, every, sigma=SIGMA):
    """(idx, mean, sqrt_info): a prior on every `every`-th landmark at its initial position, 1 / sigma I"""
    lms = np.asarray(arrays.lms, np.float64)
    idx = np.arange(0, len(lms), every, dtype=np.int32)
    return idx, lms[idx].copy(), np.tile(np.eye(3) / sigma, (len(idx), 1, 1))


def run_arm(arm):
    """inner process: bench.py's main with every BalProblem it builds carrying the arm's priors"""
    import bench
    from rootba_b200.linearizor import BalProblem
    every = ARMS[arm]
    plain_from_arrays = BalProblem.from_arrays.__func__
    plain_config = bench.workload_config

    def from_arrays_with_priors(cls, arrays, dtype=np.float64):
        bp = plain_from_arrays(cls, arrays, dtype)
        if every is not None:
            bp.landmark_prior = landmark_priors(arrays, every)
        return bp

    def config_with_priors(args, arrays):
        cfg = plain_config(args, arrays)
        cfg["landmark_priors"] = "none" if every is None else f"every {every}-th landmark at its initial position, sigma {SIGMA} per axis"
        return cfg

    BalProblem.from_arrays = classmethod(from_arrays_with_priors)
    bench.workload_config = config_with_priors
    bench.main()


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    if q.returncode != 0:
        sys.exit("bench_landmark_priors.py: nvidia-smi found no GPU; this measurement needs an H100")
    name, power = [s.strip() for s in q.stdout.strip().split("\n")[0].split(",")]
    return name, power


def main():
    if "--arm" in sys.argv:
        i = sys.argv.index("--arm")
        arm = sys.argv[i + 1]
        del sys.argv[i:i + 2]
        return run_arm(arm)
    if "--impl" in sys.argv and "reference" in sys.argv:
        sys.exit("bench_landmark_priors.py: the reference has no landmark priors")
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
            out["arms"][arm].append({"ms_per_lm_iteration": r["ms_per_step"], "stage2_ms_per_lm_iteration": r["phases_ms_per_step"]["stage2_time"],
                                     "pcg_us_per_iteration": r["pcg"]["us_per_iteration"], "pcg_iterations": r["pcg"]["iterations"]})
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
