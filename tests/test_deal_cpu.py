"""The longest-processing-time-first dealer of the persistent kernels (rba::deal_lpt in rootba_b200/csrc/layout.hpp) on
the CPU: it lays out the small matvec items of the TMA operator and the tiles of k_linearize_qr / k_panel_grad_blocks.
Every job must be taken exactly once, warp w must find its k-th job at position k * nw + w with padding only after its
last job, and the greedy bound must hold: no warp's load exceeds the mean load plus the largest cost."""
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT

FULL_GRID = 132 * 5 * 4  # warps of the float32 TMA matvec on a 132-SM H100: 5 CTAs of 4 warps per SM


@pytest.fixture(scope="module")
def deal():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "cpp"), "-s", "_build/deal_cpu"])
    exe = os.path.join(ROOT, "tests", "cpp", "_build", "deal_cpu")

    def run(cost, nw):
        inp = f"{nw} {len(cost)}\n" + " ".join(str(int(c)) for c in cost) + "\n"
        out = subprocess.run([exe], input=inp, capture_output=True, text=True, check=True).stdout
        return np.array(out.split(), dtype=np.int64)
    return run


def _cases():
    rng = np.random.default_rng(7)
    for nw in (1, 7, FULL_GRID):
        for n in (1, nw, 3 * nw + 5):
            yield nw, rng.integers(1, 2000, n)                       # random costs
            yield nw, rng.integers(1, 4, n)                          # many ties
            yield nw, np.sort(rng.integers(48, 48 + 32 * 9, n))[::-1]  # already sorted, like the matvec items


@pytest.mark.parametrize("nw,cost", list(_cases()), ids=lambda v: str(v) if np.isscalar(v) else f"n{len(v)}")
def test_deal_lpt(deal, nw, cost):
    order = deal(cost, nw)
    n = len(cost)
    assert order.size % nw == 0
    lists = order.reshape(-1, nw).T  # lists[w] = the jobs of warp w, in the order it takes them
    assert np.array_equal(np.sort(order[order >= 0]), np.arange(n))  # every job exactly once
    assert np.any(lists[:, -1] >= 0)  # the order ends with the longest list
    loads = []
    for w in range(nw):
        jobs = lists[w]
        taken = jobs[jobs >= 0]
        assert np.all(jobs[: taken.size] >= 0) and np.all(jobs[taken.size:] == -1)  # padding only at the tail
        assert np.all(np.diff(cost[taken]) <= 0)  # each warp takes its jobs longest first
        loads.append(int(cost[taken].sum()))
    assert max(loads) <= cost.sum() / nw + cost.max()
    if n <= nw:
        assert order.size == nw and np.all(lists[:n, 0] >= 0)  # one job per warp, the first warps
