#!/usr/bin/env python
"""bench.py's flagship measurement with intrinsics shared across groups of cameras (rba_set_intrinsics_groups, DESIGN.md
section 18).

    python scripts/bench_shared_intrinsics.py [--rounds R] --gpus 1 --steps K --warmup W [any other bench.py option of the CUDA arm]

Runs bench.py's own protocol on its workload (at --gpus 1 the Ladybug-1723 stand-in) in four arms -- no groups, no groups
with the Counter hand-over (RBA_PCG_PARTIALS=0, the hand-over every grouped solve on one GPU uses), every camera in one
group, 8 groups (camera c in group c mod 8) -- each once as bench.py runs it and once with every PCG solve held to exactly
FIXED_PCG iterations (min = max linear solver iterations), alternating arm by arm for R rounds (default 2) in one call,
each arm a fresh process.  Setting the groups ties each member's f, k1, k2 to its lead's, so the grouped arms solve
different problems: their LM trajectories and natural PCG iteration counts differ, and only the fixed-count runs give a
per-PCG-iteration time that compares the paths (no groups + Partials, no groups + Counter, groups: Counter + the two group
kernels).  Prints one JSON line: per arm, variant and round the milliseconds per LM iteration, the microseconds per PCG
iteration and the PCG iterations, with the card's name and power limit read in the same call.
"""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

ARMS = {"none": None, "none_counter": None, "one_group": 1, "eight_groups": 8}
FIXED_PCG = 50


def groups(nc, k):
    """camera c in group c mod k"""
    return (np.arange(nc) % k).astype(np.int32)


def run_arm(arm, fixed):
    """inner process: bench.py's main with every BalProblem it builds carrying the arm's groups (and, fixed > 0, every
    handle's PCG held to `fixed` iterations)"""
    import dataclasses
    import bench
    from rootba_b200.linearizor import BalProblem, LinearizorQR
    k = ARMS[arm]
    if fixed:
        plain_init = LinearizorQR.__init__

        def init_fixed(self, bal_problem, options, summary=None):
            options = dataclasses.replace(options, min_linear_solver_iterations=fixed, max_linear_solver_iterations=fixed)
            plain_init(self, bal_problem, options, summary)
        LinearizorQR.__init__ = init_fixed
    plain_from_arrays = BalProblem.from_arrays.__func__
    plain_config = bench.workload_config

    def from_arrays_with_groups(cls, arrays, dtype=np.float64):
        bp = plain_from_arrays(cls, arrays, dtype)
        if k is not None:
            bp.intrinsics_group = groups(bp.num_cameras(), k)
        return bp

    def config_with_groups(args, arrays):
        cfg = plain_config(args, arrays)
        cfg["intrinsics_groups"] = "none" if k is None else f"camera c in group c mod {k}"
        cfg["pcg_iterations_per_solve"] = fixed if fixed else "as bench.py"
        return cfg

    BalProblem.from_arrays = classmethod(from_arrays_with_groups)
    bench.workload_config = config_with_groups
    bench.main()


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    if q.returncode != 0:
        sys.exit("bench_shared_intrinsics.py: nvidia-smi found no GPU; this measurement needs an H100")
    name, power = [s.strip() for s in q.stdout.strip().split("\n")[0].split(",")]
    return name, power


def main():
    if "--arm" in sys.argv:
        i = sys.argv.index("--arm")
        arm, fixed = sys.argv[i + 1], int(sys.argv[i + 2])
        del sys.argv[i:i + 3]
        return run_arm(arm, fixed)
    if "--impl" in sys.argv and "reference" in sys.argv:
        sys.exit("bench_shared_intrinsics.py: the reference has no shared intrinsics")
    rounds = 2
    args = sys.argv[1:]
    if "--rounds" in args:
        i = args.index("--rounds")
        rounds = int(args[i + 1])
        del args[i:i + 2]
    name, power = card()
    out = {"card": name, "power_limit": power, "rounds": rounds, "fixed_pcg_iterations": FIXED_PCG,
           "arms": {f"{a}/{v}": [] for v in ("natural", "fixed") for a in ARMS}}
    for _ in range(rounds):
        for variant, fixed in (("natural", 0), ("fixed", FIXED_PCG)):
            for arm in ARMS:
                env = dict(os.environ)
                if arm == "none_counter":
                    env["RBA_PCG_PARTIALS"] = "0"
                p = subprocess.run([sys.executable, os.path.abspath(__file__), "--arm", arm, str(fixed), *args], capture_output=True,
                                   text=True, cwd=ROOT, env=env)
                lines = [ln for ln in p.stdout.splitlines() if ln.startswith("{")]
                if p.returncode != 0 or not lines:
                    sys.exit(f"arm {arm} failed:\n{p.stdout[-2000:]}\n{p.stderr[-2000:]}")
                r = json.loads(lines[-1])
                out["arms"][f"{arm}/{variant}"].append({"ms_per_lm_iteration": r["ms_per_step"], "pcg_us_per_iteration": r["pcg"]["us_per_iteration"],
                                         "pcg_iterations": r["pcg"]["iterations"]})
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
