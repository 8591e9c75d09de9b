#!/usr/bin/env python
"""Where the assembled PCG product k_rcs_spmv spends its time on the flagship, and whether S comes from L2 or from HBM.
   python scripts/prof_spmv.py [--steps 10] [--warmup 3] [--reps 200]

The flagship stand-in (synth_config("ladybug-1723", seed=38401), float32), with S built at PCG iteration 1
(RBA_ASSEMBLED_AT=1) so that every solve runs on it:
  (a) k_rcs_spmv back to back, as rba_time_matvec (and bench.py's roofline) measures it: CUDA events around --reps
      launches;
  (b) one launch after a write of 128 MB to a scratch buffer (S evicted from L2 unless the cache keeps it), against one
      launch right after another, both through rba_right_multiply, device times from torch.profiler;
  (c) bench.py's LM protocol under torch.profiler: the device time of every k_rcs_spmv inside PCG, the gap from the end of
      the vector step k_pcg_vec before it to its start (negative: it started early, programmatic dependent launch) and
      from that end to its own end (the time the product adds to the PCG iteration).
Bytes per launch are matvec_algorithmic_bytes (S, x, y and the CSR indices).  The profiler slows the host, so (b) and (c)
are the kernels' own times, not those of bench.py's window.  Needs a GPU."""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ["RBA_ASSEMBLED_AT"] = "1"
import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

import rootba_b200 as rb
from rootba_b200.synthetic import synth_config

SPMV, VEC = "k_rcs_spmv", "k_pcg_vec"


def kernels(prof):
    """(name, start us, end us) of every kernel, in stream order"""
    ev = [e for e in prof.events() if str(e.device_type).endswith("CUDA") and not e.name.startswith("Memcpy") and not e.name.startswith("Memset")]
    ev.sort(key=lambda e: e.time_range.start)
    return [(e.name, float(e.time_range.start), float(e.time_range.end)) for e in ev]


def spmv_us(prof):
    return np.array([t1 - t0 for n, t0, t1 in kernels(prof) if SPMV in n])


def stats_line(name, v):
    return f"{name:<44}{v.size:>7}{np.median(v):>10.2f}{np.percentile(v, 10):>10.2f}{np.percentile(v, 90):>10.2f}{v.sum() / 1e3:>11.3f}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prof_spmv.py: no CUDA device (kernel times are measured, not estimated)")
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], capture_output=True, text=True).stdout.strip())
    print("library:", rb._lib.LIB_PATH)
    arrays = synth_config("ladybug-1723", seed=38401)
    init = (arrays.cams.copy(), arrays.lms.copy())
    bp = rb.BalProblem.from_arrays(arrays, np.float32)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(use_double=False))
    lin.linearize()
    lin.solve(1e-4, to_host=False)
    mv_bytes = float(lin.stats()["matvec_algorithmic_bytes"])
    print(f"matvec_algorithmic_bytes {mv_bytes / 1e6:.2f} MB per launch")

    # ---- (a) back to back ----
    t = min(lin.time_matvec(args.reps) for _ in range(3))
    print(f"(a) back to back, rba_time_matvec({args.reps}), best of 3: {1e6 * t:.2f} us per launch, {mv_bytes / t / 1e9:.0f} GB/s")

    # ---- (b) after a 128 MB write, against right after another launch ----
    x = np.random.default_rng(1).uniform(-1, 1, 9 * arrays.nc).astype(np.float32)
    scratch = torch.empty(128 << 20, dtype=torch.uint8, device="cuda")
    for _ in range(5):
        lin.right_multiply(x)
        scratch.fill_(1)
    torch.cuda.synchronize()
    rows = []
    for label, flush in (("(b) after a 128 MB write", True), ("(b) right after another launch", False)):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for i in range(50):
                if flush:
                    scratch.fill_(i & 0xff)
                    torch.cuda.synchronize()
                lin.right_multiply(x)
            torch.cuda.synchronize()
        rows.append((label, spmv_us(prof)))
    print(f"{'k_rcs_spmv device time (us)':<44}{'n':>7}{'median':>10}{'p10':>10}{'p90':>10}{'total ms':>11}")
    for label, v in rows:
        print(stats_line(label, v) + f"   {mv_bytes / np.median(v) / 1e3:.0f} GB/s at the median")
    lin.close()

    # ---- (c) inside PCG, bench.py's protocol ----
    bp = rb.BalProblem.from_arrays(arrays, np.float32)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(use_double=False))

    def run(nsteps):
        left, cg = nsteps, []
        while left > 0:
            its, term, _ = lin.lm_run(left)
            if not its:
                raise RuntimeError("rba_lm_run made no progress")
            left -= len(its)
            cg += [i["cg_iterations"] for i in its]
            if term or left > 0:
                bp.cams[:] = init[0]; bp.lms[:] = init[1]
                lin.upload_state()
        return cg

    run(args.warmup)
    bp.cams[:] = init[0]; bp.lms[:] = init[1]
    lin.upload_state()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        cg = run(args.steps)
        torch.cuda.synchronize()
    lin.close()
    ev = kernels(prof)
    dur, gap, exposed = [], [], []
    for i, (n, t0, t1) in enumerate(ev):
        if SPMV not in n:
            continue
        dur.append(t1 - t0)
        if i > 0 and VEC in ev[i - 1][0]:
            gap.append(t0 - ev[i - 1][2])
            exposed.append(t1 - ev[i - 1][2])
    print(f"(c) {args.steps} LM steps after {args.warmup} warm-up steps, PCG iterations {cg}")
    print(f"{'(us)':<44}{'n':>7}{'median':>10}{'p10':>10}{'p90':>10}{'total ms':>11}")
    print(stats_line("(c) k_rcs_spmv device time", np.array(dur)))
    if gap:
        print(stats_line("(c) end of k_pcg_vec -> start of k_rcs_spmv", np.array(gap)))
        print(stats_line("(c) end of k_pcg_vec -> end of k_rcs_spmv", np.array(exposed)))


if __name__ == "__main__":
    main()
