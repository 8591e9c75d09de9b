#!/usr/bin/env python
"""CPU experiment behind DESIGN.md section 9: round-off of the dense Q2-panel product  P^T (P x)  and of the implicit form
Jp^T (Jp x) - Q1d^T (Q1d x)  in float32, both evaluated on the SAME float32 landmark blocks (the float32 oracle's), against
the float64 product of those float32 panels, and of the assembled form  (P^T P) x  with S = sum_l P_l^T P_l accumulated in
float32 block by block (landmarks in problem order) and applied in float32.  Also prints the worst per-landmark cancellation factor |Jp^T Jp x| / |P^T P x|.
   python scripts/implicit_f32_accuracy.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import oracle_py as orc  # noqa: E402
from rootba_b200.synthetic import synth_bal  # noqa: E402


def rel_err(a, b):
    a, b = np.asarray(a, np.float64).ravel(), np.asarray(b, np.float64).ravel()
    return float(np.linalg.norm(a - b) / (np.linalg.norm(a) + np.linalg.norm(b)))


def products(o32, prob, x32):
    yt, yd, yi = np.zeros(9 * prob.nc), np.zeros(9 * prob.nc, np.float32), np.zeros(9 * prob.nc, np.float32)
    S = np.zeros((9 * prob.nc, 9 * prob.nc), np.float32)
    D = o32.get_scaling()
    worst = 0.0
    for lm in range(prob.nl):
        k0, k1 = int(prob.lm_off[lm]), int(prob.lm_off[lm + 1])
        n = k1 - k0
        blk, _, _, _ = o32.get_block(lm)
        P, Q1d = blk[3:, :9 * n], blk[:3, :9 * n]
        cams = [int(prob.obs_cam[k]) for k in range(k0, k1)]
        xr = np.concatenate([x32[9 * c:9 * c + 9] for c in cams])
        t = P.astype(np.float64).T @ (P.astype(np.float64) @ xr.astype(np.float64))
        d = (P.T @ (P @ xr)).astype(np.float32)
        Jp = np.zeros((2 * n, 9 * n), np.float32)
        for i, k in enumerate(range(k0, k1)):
            _, jp, ji, _, _ = orc.linearize_point(prob.obs_xy[k], prob.lms[lm], prob.cams[cams[i]], np.float32)
            Jp[2 * i:2 * i + 2, 9 * i:9 * i + 9] = np.hstack([jp, ji]).astype(np.float32) * D[9 * cams[i]:9 * cams[i] + 9]
        im = (Jp.T @ (Jp @ xr) - Q1d.T @ (Q1d @ xr)).astype(np.float32)
        G = (P.T @ P).astype(np.float32)
        for i, ci in enumerate(cams):
            for j, cj in enumerate(cams):
                S[9 * ci:9 * ci + 9, 9 * cj:9 * cj + 9] += G[9 * i:9 * i + 9, 9 * j:9 * j + 9]
        for i, c in enumerate(cams):
            yt[9 * c:9 * c + 9] += t[9 * i:9 * i + 9]
            yd[9 * c:9 * c + 9] += d[9 * i:9 * i + 9]
            yi[9 * c:9 * c + 9] += im[9 * i:9 * i + 9]
        worst = max(worst, float(np.linalg.norm(Jp.T @ (Jp @ xr)) / max(np.linalg.norm(t), 1e-30)))
    ys = (S @ x32).astype(np.float32)
    return yt, yd, yi, ys, worst


def main():
    cases = (("small (49 cams)", synth_bal(49, 1800, 4.1, seed=38401)),
             ("hard start (20 cams)", synth_bal(20, 500, 4.1, seed=7, perturb_rot=0.3, perturb_trans=3.0, perturb_lm=2.0)),
             ("long tracks (60 cams, n~30)", synth_bal(60, 300, 30.0, seed=3, max_track=60)))
    for name, prob in cases:
        for lam in (1e-6, 1e-2):
            o32 = orc.Oracle(prob, np.float32, orc.default_options(num_threads=1))
            o32.linearize()
            o32.solve(lam)
            x = np.random.default_rng(0).uniform(-1, 1, 9 * prob.nc).astype(np.float32)
            yt, yd, yi, ys, worst = products(o32, prob, x)
            print(f"{name:28s} lambda {lam:g}: dense f32 {rel_err(yd, yt):.2e}  implicit f32 {rel_err(yi, yt):.2e}  "
                  f"assembled S f32 {rel_err(ys, yt):.2e}  "
                  f"max cancellation |JpTJp x|/|PtP x| = {worst:.1f}")


if __name__ == "__main__":
    main()
