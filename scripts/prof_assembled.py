#!/usr/bin/env python
"""Where the flagship's device time goes, kernel by kernel, and the assembly of S against the bytes it must move.
   python scripts/prof_assembled.py [--steps 10] [--warmup 3]

Part 1: the flagship stand-in (synth_config("ladybug-1723", seed=38401), float32) through lm_run with bench.py's default
protocol under torch.profiler (CUDA activities): launches and total device time per kernel name.
Part 2: one linearisation with two solves that both pass the switch iteration (eta no residual undercuts), so the first
builds S_u and S (4 launches) and the second S alone (2): every assembly launch in stream order with its time, the bytes
it must move (from T, nblk, nnzb, Nobs and the panel scalars) and bytes / time.
The profiler slows the host, so the times are the kernels' own and not those of bench.py's window.  Needs a GPU."""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import scipy.sparse as sp
import torch
from torch.profiler import ProfilerActivity, profile

import rootba_b200 as rb
from rootba_b200.synthetic import synth_config

NAMED = ("k_rcs_terms", "k_rcs_combine", "k_rcs_damping", "k_rcs_mirror", "k_rcs_spmv", "k_pcg_vec", "k_matvec_small_tma",
         "k_cam_reduce")
ASSEMBLY = NAMED[:4]


def kernel_events(prof):
    """(name, device microseconds) of every kernel, in stream order"""
    ev = [e for e in prof.events() if str(e.device_type).endswith("CUDA") and not e.name.startswith("Memcpy") and not e.name.startswith("Memset")]
    ev.sort(key=lambda e: e.time_range.start)
    return [(e.name, float(e.time_range.elapsed_us())) for e in ev]


def short(name):
    return next((k for k in NAMED if k in name), None)


def structure(arrays, lin, s):
    """T, nblk, nnzb, Nobs, the panel scalars, and the bytes every assembly kernel must move"""
    n = np.diff(arrays.lm_off).astype(np.int64)
    A = sp.csr_matrix((np.ones(arrays.obs_cam.size, np.int32), arrays.obs_cam, arrays.lm_off), shape=(arrays.nl, arrays.nc))
    nnzb = int((A.T @ A).nnz)
    ndiag = int(np.count_nonzero(np.bincount(arrays.obs_cam, minlength=arrays.nc)))
    st = {"T": int(np.sum(n * (n + 1) // 2)), "nblk": (nnzb + ndiag) // 2, "nnzb": nnzb, "Nobs": int(arrays.obs_cam.size),
          "panel": int(lin.stats()["panel_scalars"])}
    T, nblk, nobs = st["T"], st["nblk"], st["Nobs"]
    st["bytes"] = {
        # the panels once, a 16-byte address record per term, every term's block written
        "k_rcs_terms": st["panel"] * s + 16 * T + 81 * T * s,
        # every term's block and its position read, the pair blocks written
        "k_rcs_combine": 81 * T * s + 4 * T + 4 * nblk + 81 * nblk * s,
        # two slots per term, the damping records once (28 Nobs s; the repeats are served by L2), S_u read, the lower blocks
        # of S written
        "k_rcs_damping": 8 * T + 28 * nobs * s + 2 * 81 * nblk * s + 12 * nblk,
        # the lower block of every off-diagonal pair read and written transposed
        "k_rcs_mirror": 2 * 81 * (nnzb - nblk) * s + 8 * nblk,
    }
    return st


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prof_assembled.py: no CUDA device (kernel times are measured, not estimated)")
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], capture_output=True, text=True).stdout.strip())
    print("library:", rb._lib.LIB_PATH)
    arrays = synth_config("ladybug-1723", seed=38401)
    dtype, s = np.float32, 4
    init = (arrays.cams.copy(), arrays.lms.copy())

    # ---- part 1: the flagship protocol ----
    bp = rb.BalProblem.from_arrays(arrays, dtype)
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
    st = structure(arrays, lin, s)
    lin.close()
    print("structure:", {k: v for k, v in st.items() if k != "bytes"})
    print(f"part 1: {args.steps} LM steps after {args.warmup} warm-up steps, PCG iterations {cg}")
    tot = {}
    for name, us in kernel_events(prof):
        k = short(name) or "(the rest)"
        c = tot.setdefault(k, [0, 0.0])
        c[0] += 1; c[1] += us
    all_us = sum(v[1] for v in tot.values())
    print(f"{'kernel':<22}{'launches':>10}{'total ms':>12}{'share':>8}")
    for k in sorted(tot, key=lambda k: -tot[k][1]):
        print(f"{k:<22}{tot[k][0]:>10}{tot[k][1] / 1e3:>12.3f}{tot[k][1] / all_us:>8.1%}")
    print(f"{'all kernels':<22}{sum(v[0] for v in tot.values()):>10}{all_us / 1e3:>12.3f}")

    # ---- part 2: one linearisation, two solves past the switch ----
    bp = rb.BalProblem.from_arrays(arrays, dtype)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(use_double=False, eta=-1e30, max_linear_solver_iterations=40))
    lin.linearize()
    for lam in (1e-4, 1e-2):  # warm-up: the same two solves
        lin.solve(lam, to_host=False)
    lin.linearize()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for lam in (1e-4, 1e-2):
            lin.solve(lam, to_host=False)
        torch.cuda.synchronize()
    lin.close()
    print("part 2: the assembly launches of one linearisation, first solve (S_u and S), then a second lambda (S alone)")
    print(f"{'kernel':<22}{'us':>10}{'MB to move':>12}{'GB/s':>10}")
    asm_us = 0.0
    for name, us in kernel_events(prof):
        k = short(name)
        if k in ASSEMBLY:
            b = st["bytes"][k]
            asm_us += us
            print(f"{k:<22}{us:>10.1f}{b / 1e6:>12.1f}{b / us / 1e3:>10.0f}")
    print(f"assembly, 6 launches: {asm_us / 1e3:.3f} ms")


if __name__ == "__main__":
    main()
