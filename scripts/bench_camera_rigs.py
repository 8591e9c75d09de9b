#!/usr/bin/env python
"""bench.py's flagship measurement with rigid camera rigs (rba_set_camera_rigs, DESIGN.md section 23).

    python scripts/bench_camera_rigs.py [--rounds R] --gpus 1 --steps K --warmup W [any other bench.py option of the CUDA arm]

Runs bench.py's own protocol on its workload (at --gpus 1 the Ladybug-1723 stand-in) in five arms -- no rigs, no rigs with
the Counter hand-over (RBA_PCG_PARTIALS=0, the hand-over every rigged solve on one GPU uses), rigs of 2 consecutive cameras,
rigs of 6 consecutive cameras, and the workaround rigs replace: every pair of consecutive cameras of the rigs of 2 joined by
a stiff relative pose prior (sqrt_info PAIR_STIFFNESS I, mean the initial relative pose) -- each once as bench.py runs it
and once with every PCG solve held to exactly FIXED_PCG iterations (min = max linear solver iterations), alternating arm by
arm for R rounds (default 2) in one call, each arm a fresh process.  cam_from_rig is taken from the stand-in's initial
poses relative to each rig's lead, so the rigged start is the unrigged one.  The arms solve different problems, so only the
fixed-count runs give a per-PCG-iteration time that compares the paths; the natural runs give the PCG iterations per solve.
Prints one JSON line: per arm, variant and round the milliseconds per LM iteration, the microseconds per PCG iteration and
the PCG iterations, with the card's name and power limit read in the same call.
"""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

ARMS = {"none": None, "none_counter": None, "rigs_2": 2, "rigs_6": 6, "pair_priors_2": 2}
FIXED_PCG = 50
PAIR_STIFFNESS = 1e4


def relative(cams, a, b):
    """T_a T_b^-1 of the world->camera poses of cameras a, b (arrays) as (q [m, 4] xyzw, t [m, 3])"""
    from scipy.spatial.transform import Rotation
    ra, rb = Rotation.from_quat(cams[a, :4]), Rotation.from_quat(cams[b, :4])
    r = ra * rb.inv()
    return r.as_quat(), cams[a, 4:7] - r.apply(cams[b, 4:7])


def rig_of(cams, k):
    """rigs of k consecutive cameras, cam_from_rig from the initial poses relative to each rig's lead"""
    nc = len(cams)
    rig = (np.arange(nc) // k).astype(np.int32)
    lead = rig * k
    q, t = relative(np.asarray(cams, np.float64), np.arange(nc), lead)
    return rig, np.c_[q, t]


def pair_priors(cams, k):
    """stiff pair priors between every member and the lead of each rig of k consecutive cameras"""
    nc = len(cams)
    j = np.flatnonzero(np.arange(nc) % k != 0)
    i = j - j % k
    q, t = relative(np.asarray(cams, np.float64), i, j)
    L = np.broadcast_to(PAIR_STIFFNESS * np.eye(6), (len(j), 6, 6))
    return np.c_[i, j].astype(np.int32), np.c_[q, t], L


def run_arm(arm, fixed):
    """inner process: bench.py's main with every BalProblem it builds carrying the arm's rigs or pair priors (and, fixed > 0,
    every handle's PCG held to `fixed` iterations)"""
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

    def from_arrays_with_rigs(cls, arrays, dtype=np.float64):
        bp = plain_from_arrays(cls, arrays, dtype)
        if k is not None and arm.startswith("rigs"):
            bp.camera_rig = rig_of(bp.cams, k)
        elif k is not None:
            bp.camera_pair_prior = pair_priors(bp.cams, k)
        return bp

    def config_with_rigs(args, arrays):
        cfg = plain_config(args, arrays)
        cfg["camera_rigs"] = f"rigs of {k} consecutive cameras" if arm.startswith("rigs") else "none"
        cfg["pair_priors"] = f"sqrt_info {PAIR_STIFFNESS:g} I within rigs of {k}" if arm.startswith("pair") else "none"
        cfg["pcg_iterations_per_solve"] = fixed if fixed else "as bench.py"
        return cfg

    BalProblem.from_arrays = classmethod(from_arrays_with_rigs)
    bench.workload_config = config_with_rigs
    bench.main()


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    if q.returncode != 0:
        sys.exit("bench_camera_rigs.py: nvidia-smi found no GPU; this measurement needs an H100")
    name, power = [s.strip() for s in q.stdout.strip().split("\n")[0].split(",")]
    return name, power


def main():
    if "--arm" in sys.argv:
        i = sys.argv.index("--arm")
        arm, fixed = sys.argv[i + 1], int(sys.argv[i + 2])
        del sys.argv[i:i + 3]
        return run_arm(arm, fixed)
    if "--impl" in sys.argv and "reference" in sys.argv:
        sys.exit("bench_camera_rigs.py: the reference has no camera rigs")
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
                print(f"{arm}/{variant}: {r['ms_per_step']:.3f} ms per LM iteration, {r['pcg']['iterations']} PCG iterations",
                      file=sys.stderr, flush=True)
                out["arms"][f"{arm}/{variant}"].append({"ms_per_lm_iteration": r["ms_per_step"], "pcg_us_per_iteration": r["pcg"]["us_per_iteration"],
                                         "pcg_iterations": r["pcg"]["iterations"]})
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
