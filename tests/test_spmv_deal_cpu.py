"""The row deal of the assembled product k_rcs_spmv (rba::deal_spmv in rootba_b200/csrc/layout.hpp, driven by
tests/cpp/spmv_deal_cpu.cpp) on the CPU.  Every block row must be taken by exactly one CTA, as consecutive chunks that
cover its blocks in ascending order, cut at multiples of the stage size from the row's start (so that a block's fma chain
is its position in its chunk mod SPMV_CLASSES), flagged first and last; a row without blocks is one empty chunk flagged
both; every CTA takes its rows longest first, and no CTA's load exceeds the mean load plus the longest row."""
import os
import subprocess

import numpy as np
import pytest
import scipy.sparse as sp

from conftest import ROOT
from rootba_b200.synthetic import synth_config

SPMV_CLASSES = 4           # layout.hpp
CHUNK = {4: 32, 8: 16}     # spmv_chunk_blocks(scalar size)
FIRST, LAST = 1, 2
H100_CTAS = 132 * 5        # co-resident k_rcs_spmv CTAs on a 132-SM H100 (5 per SM, its shared memory)


@pytest.fixture(scope="module")
def deal(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("spmv_deal") / "spmv_deal_cpu")
    src = os.path.join(ROOT, "tests", "cpp", "spmv_deal_cpu.cpp")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-Wall", "-o", exe, src])

    def run(lengths, ctas, chunk):
        row_ptr = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
        inp = f"{ctas} {chunk} {len(lengths)}\n" + " ".join(map(str, row_ptr.tolist())) + "\n"
        out = subprocess.run([exe], input=inp, capture_output=True, text=True, check=True).stdout.splitlines()
        n = int(out[0].split()[1])
        ptr = np.array(out[1].split()[1:], dtype=np.int64)
        chunks = np.array([ln.split() for ln in out[2:]], dtype=np.int64).reshape(-1, 4)
        return row_ptr, n, ptr, chunks
    return run


def flagship_lengths():
    """blocks per row of S on the bench.py stand-in of Ladybug-1723: the co-visible cameras of every camera, itself included"""
    a = synth_config("ladybug-1723", seed=38401)
    A = sp.csr_matrix((np.ones(a.obs_cam.size, np.int32), a.obs_cam, a.lm_off), shape=(a.nl, a.nc))
    return np.diff((A.T @ A).tocsr().indptr)


def _cases():
    rng = np.random.default_rng(11)
    for s, ch in CHUNK.items():
        # every stage edge: one block short of, at and past one, two and three stages, and empty rows
        edges = np.array([0, 1, ch - 1, ch, ch + 1, 2 * ch - 1, 2 * ch, 2 * ch + 1, 3 * ch, 3 * ch + 1, 0, 2])
        for ctas in (1, 3, len(edges), 100):
            yield f"edges-s{s}-c{ctas}", rng.permutation(edges), ctas, ch
        yield f"random-s{s}", rng.integers(0, 420, 500), 37, ch
        yield f"ties-s{s}", rng.integers(0, 3, 300), 64, ch
        yield f"hub-s{s}", np.concatenate([[400], rng.integers(1, 6, 399)]), 50, ch
    yield "no-blocks", np.zeros(5, np.int64), 4, 32
    yield "one-row", np.array([77]), 10, 32
    yield "flagship-f32", flagship_lengths(), H100_CTAS, CHUNK[4]


@pytest.mark.parametrize("name,lengths,ctas,chunk", list(_cases()), ids=lambda v: v if isinstance(v, str) else "")
def test_deal_spmv(deal, name, lengths, ctas, chunk):
    lengths = np.asarray(lengths, np.int64)
    nrows = lengths.size
    row_ptr, n, ptr, chunks = deal(lengths, ctas, chunk)
    assert n == max(1, min(ctas, nrows))
    assert ptr.size == n + 1 and ptr[0] == 0 and ptr[-1] == len(chunks) and np.all(np.diff(ptr) >= 0)
    seen = np.zeros(nrows, np.int64)
    loads = []
    for b in range(n):
        ch = chunks[ptr[b]:ptr[b + 1]]
        rows, i = [], 0
        while i < len(ch):
            r = int(ch[i, 0])
            k0, k1 = int(row_ptr[r]), int(row_ptr[r + 1])
            j = i
            while j < len(ch) and ch[j, 0] == r:
                j += 1
            run = ch[i:j]
            # the row's chunks: consecutive, from its first block to its last, cut every `chunk` blocks from its start
            starts = np.arange(k0, k1, chunk) if k1 > k0 else np.array([k0])
            assert np.array_equal(run[:, 1], starts), (name, r)
            assert np.array_equal(run[:, 2], np.minimum(starts + chunk, k1)), (name, r)
            assert np.all((run[:, 1] - k0) % SPMV_CLASSES == 0)
            flags = np.zeros(len(run), np.int64)
            flags[0] |= FIRST
            flags[-1] |= LAST
            assert np.array_equal(run[:, 3], flags), (name, r)
            seen[r] += 1
            rows.append(r)
            i = j
        assert np.all(np.diff(lengths[rows]) <= 0), (name, b)  # longest first
        loads.append(int(lengths[rows].sum()))
    assert np.all(seen == 1), name  # every row dealt exactly once
    assert max(loads) <= lengths.sum() / n + lengths.max()
    if name == "flagship-f32":
        assert lengths.min() >= 1 and n == H100_CTAS
