#!/usr/bin/env python
"""bench.py's flagship measurement with a robust loss per observation (rba_set_observation_loss, DESIGN.md section 21).

    python scripts/bench_observation_loss.py [--rounds R] --gpus 1 --steps K --warmup W [any other bench.py option of the CUDA arm]

Runs bench.py's own protocol on its workload (at --gpus 1 the Ladybug-1723 stand-in) with the handle's Huber norm at
HUBER_PARAMETER in three arms, alternating arm by arm for R rounds (default 2) in one call, each arm a fresh process:

  handle_huber  no per-observation loss: the unmodified kernels with the handle's Huber norm
  obs_huber     HUBER at HUBER_PARAMETER (1 + 2^-20) on every observation.  Not the handle's own choice, so the OBSL kernel
                instances run and the whole cost of the path is paid, while the LM trajectory stays that of handle_huber up
                to rounding: the two arms' milliseconds per LM iteration are comparable
  mixed         70 % CAUCHY at 1, 20 % TUKEY at 4, 10 % NONE, drawn per observation by a seed.  This changes the LM
                trajectory, so its milliseconds per LM iteration are reported, not compared

Prints one JSON line: per arm and round the stage-1 time and the milliseconds per LM iteration, the microseconds per PCG
iteration (no kernel of the PCG iteration reads the losses) and the PCG iterations, with the card's name and power limit read
in the same call.
"""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

HUBER_PARAMETER = 1.0
SEED = 23
ARMS = {"handle_huber": f"handle Huber at {HUBER_PARAMETER}, no per-observation loss",
        "obs_huber": f"HUBER at {HUBER_PARAMETER} (1 + 2^-20) on every observation",
        "mixed": f"70 % CAUCHY at 1, 20 % TUKEY at 4, 10 % NONE (seed {SEED})"}


def observation_loss(arm, nobs):
    """None, or (kind [nobs], scale [nobs]) of the arm"""
    if arm == "handle_huber":
        return None
    if arm == "obs_huber":
        return "HUBER", HUBER_PARAMETER * (1.0 + 2.0 ** -20)
    kind = np.random.default_rng(SEED).choice(np.array([2, 4, 0], np.uint8), nobs, p=[0.7, 0.2, 0.1])
    return kind, np.where(kind == 4, 4.0, 1.0)


def run_arm(arm):
    """inner process: bench.py's main with the handle's Huber norm and every BalProblem it builds carrying the arm's losses"""
    import bench
    from rootba_b200 import linearizor
    from rootba_b200.linearizor import BalProblem, LinearizorQR, ResidualOptions
    plain_from_arrays = BalProblem.from_arrays.__func__
    plain_config = bench.workload_config
    plain_init = LinearizorQR.__init__

    def from_arrays_with_loss(cls, arrays, dtype=np.float64):
        bp = plain_from_arrays(cls, arrays, dtype)
        bp.observation_loss = observation_loss(arm, bp.num_observations())
        return bp

    def config_with_loss(args, arrays):
        cfg = plain_config(args, arrays)
        cfg["observation_loss"] = ARMS[arm]
        return cfg

    def init_with_huber(self, bal_problem, options, summary=None):
        options.residual = ResidualOptions(robust_norm="HUBER", huber_parameter=HUBER_PARAMETER)
        plain_init(self, bal_problem, options, summary)

    BalProblem.from_arrays = classmethod(from_arrays_with_loss)
    bench.workload_config = config_with_loss
    linearizor.LinearizorQR.__init__ = init_with_huber
    bench.main()


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    if q.returncode != 0:
        sys.exit("bench_observation_loss.py: nvidia-smi found no GPU; this measurement needs an H100")
    name, power = [s.strip() for s in q.stdout.strip().split("\n")[0].split(",")]
    return name, power


def main():
    if "--arm" in sys.argv:
        i = sys.argv.index("--arm")
        arm = sys.argv[i + 1]
        del sys.argv[i:i + 2]
        return run_arm(arm)
    if "--impl" in sys.argv and "reference" in sys.argv:
        sys.exit("bench_observation_loss.py: the reference has no per-observation loss")
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
