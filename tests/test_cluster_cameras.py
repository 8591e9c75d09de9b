"""CPU-side checks of CLUSTER_JACOBI (DESIGN.md section 28): rba_cluster_cameras against a numpy restatement of the
clustering and its properties, the intra-cluster term list of plan_clusters (through tests/cpp_cluster, a small driver
compiled here), and the option's protocol: the struct, the default and the rejected combinations."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

from conftest import ROOT

MAX = 16


def _problem(nc, tracks):
    off = np.zeros(len(tracks) + 1, np.int64)
    off[1:] = np.cumsum([len(t) for t in tracks])
    cam = np.array([c for t in tracks for c in t], np.int32)
    return nc, off, cam


def _cluster(nc, off, cam, k):
    from rootba_b200 import _lib
    xy = np.zeros((max(len(cam), 1), 2))
    pv = _lib.ProblemView(nc, len(off) - 1, len(cam), off.ctypes.data, cam.ctypes.data if len(cam) else xy.ctypes.data, xy.ctypes.data)
    out = np.full(nc, -7, np.int32)
    rc = _lib.lib().rba_cluster_cameras(C.byref(pv), C.c_int32(k), out.ctypes.data_as(C.c_void_p))
    return rc, out


def numpy_clusters(nc, off, cam, k):
    """the algorithm restated: co-visibility weights, edges by (weight desc, i, j), union-find with the size cap, ids by
    smallest camera"""
    w = {}
    for l in range(len(off) - 1):
        cs = cam[off[l]:off[l + 1]]
        for a in range(len(cs)):
            for b in range(a):
                if cs[a] != cs[b]:
                    e = (min(cs[a], cs[b]), max(cs[a], cs[b]))
                    w[e] = w.get(e, 0) + 1
    parent, size = list(range(nc)), [1] * nc

    def find(c):
        while parent[c] != c:
            c = parent[c]
        return c
    for (i, j), _ in sorted(w.items(), key=lambda kv: (-kv[1], kv[0])):
        ri, rj = find(i), find(j)
        if ri != rj and size[ri] + size[rj] <= k:
            lo, hi = min(ri, rj), max(ri, rj)
            parent[hi] = lo
            size[lo] += size[hi]
    ids, out = {}, np.empty(nc, np.int32)
    for c in range(nc):
        out[c] = ids.setdefault(find(c), len(ids))
    return out


problems = st.integers(2, 14).flatmap(lambda nc: st.tuples(
    st.just(nc), st.lists(st.lists(st.integers(0, nc - 1), min_size=2, max_size=min(nc, 6), unique=True).map(sorted), max_size=30),
    st.integers(1, MAX)))


@settings(max_examples=150, deadline=None)
@given(problems)
def test_clustering_properties(case):
    nc, tracks, k = case
    nc, off, cam = _problem(nc, tracks)
    rc, c = _cluster(nc, off, cam, k)
    assert rc == 0
    sizes = np.bincount(c)
    assert c.min() == 0 and len(sizes) == c.max() + 1 and np.all(sizes >= 1)  # every camera in one cluster, dense ids
    assert sizes.max() <= k
    first = [np.flatnonzero(c == i)[0] for i in range(len(sizes))]
    assert first == sorted(first)  # numbered by the smallest camera
    assert np.array_equal(c, _cluster(nc, off, cam, k)[1])  # deterministic
    assert np.array_equal(c, numpy_clusters(nc, off, cam, k))
    # a cluster never joins cameras that no chain of shared landmarks links
    comp = list(range(nc))

    def find(x):
        while comp[x] != x:
            x = comp[x]
        return x
    for t in tracks:
        for a in t[1:]:
            comp[find(a)] = find(t[0])
    for i in range(len(sizes)):
        assert len({find(x) for x in np.flatnonzero(c == i)}) == 1
    if k == 1:
        assert np.array_equal(c, np.arange(nc))


def test_unobserved_cameras_are_singletons_and_bad_input_is_rejected():
    nc, off, cam = _problem(6, [[0, 1], [0, 1, 2], [1, 2]])
    rc, c = _cluster(nc, off, cam, 16)
    assert rc == 0 and c.tolist() == [0, 0, 0, 1, 2, 3]
    for k in (0, 17, -1):
        assert _cluster(nc, off, cam, k)[0] == -1
    assert _cluster(2, *_problem(2, [[0, 5]])[1:], 4)[0] == -1


# ---- the intra-cluster term list --------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.skip("no C++ compiler")
    exe = tmp_path_factory.mktemp("cpd") / "cluster_plan_driver"
    subprocess.check_call([cxx, "-std=c++17", "-O1", "-Wall", "-o", str(exe), os.path.join(ROOT, "tests", "cpp_cluster", "cluster_plan_driver.cpp")])
    return str(exe)


def _plan(driver, nc, off, cam, c):
    txt = " ".join(map(str, [nc, len(off) - 1, *off.tolist(), *cam.tolist(), *c.tolist()]))
    out = subprocess.run([driver], input=txt, capture_output=True, text=True, check=True).stdout.strip().splitlines()
    return [tuple(map(int, l.split())) for l in out[:-1]], out[-1]


@pytest.mark.parametrize("seed", range(6))
def test_term_list_lists_every_in_cluster_pair_once(driver, seed):
    from rootba_b200.synthetic import synth_bal
    prob = synth_bal(12, 80, 4.5, seed=seed, max_track=40)
    for k in (1, 3, 16):
        c = _cluster(prob.nc, prob.lm_off, prob.obs_cam, k)[1]
        terms, tail = _plan(driver, prob.nc, prob.lm_off, prob.obs_cam, c)
        want = sorted((int(c[a]), int(a), int(b), l) for l in range(prob.nl)
                      for a in prob.obs_cam[prob.lm_off[l]:prob.lm_off[l + 1]]
                      for b in prob.obs_cam[prob.lm_off[l]:prob.lm_off[l + 1]] if a > b and c[a] == c[b])
        got = [(k_, ca, cb, lm) for k_, ca, cb, lm, sa, sb in terms]
        assert all(sa == ca and sb == cb and c[ca] == k_ for k_, ca, cb, lm, sa, sb in terms)  # under the right block
        assert sorted(got) == want  # every in-cluster pair of every landmark, exactly once
        keys = [(k_, ca, cb) for k_, ca, cb, _ in got]
        assert keys == sorted(keys)  # grouped by cluster, blocks ascending
        assert tail.startswith("bytes ")


def test_plan_rejects_bad_clusterings(driver):
    nc, off, cam = _problem(4, [[0, 1], [1, 2, 3]])
    for c, why in (([0, 0, 2, 2], "not dense"), ([0, 0, 1, 4], "outside")):
        _, tail = _plan(driver, nc, off, cam, np.array(c))
        assert tail.startswith("error") and why in tail
    nc, off, cam = _problem(17, [list(range(17))])
    _, tail = _plan(driver, nc, off, cam, np.zeros(17, np.int32))
    assert "more than 16" in tail


# ---- the option -------------------------------------------------------------------------------------------------------------
def test_default_and_header_constants():
    from rootba_b200 import _lib
    import rootba_b200 as rb
    o = _lib.SolverOpts()
    _lib.lib().rba_default_solver_opts(C.byref(o))
    assert o.preconditioner_type == 1 and rb.SolverOptions().preconditioner_type == "SCHUR_JACOBI"
    assert _lib.SolverOpts.reserved.size == 4 and _lib.lib().rba_abi_version() == 1  # the struct and the ABI stay as they were
    hdr = open(_lib.HEADER_PATH).read()
    assert "#define RBA_CLUSTER_MAX_CAMERAS 16" in hdr
    for s in ("rba_cluster_cameras", "rba_set_camera_clusters", "rba_get_cluster_preconditioner"):
        assert s in _lib.declared_symbols() and hasattr(_lib.lib(), s)


def _create(**fields):
    from rootba_b200 import _lib
    from rootba_b200.synthetic import synth_bal
    prob = synth_bal(4, 20, 2.5, seed=1)
    L = _lib.lib()
    o = _lib.SolverOpts()
    L.rba_default_solver_opts(C.byref(o))
    for k, v in fields.items():
        setattr(o, k, v)
    off = np.ascontiguousarray(prob.lm_off, np.int64)
    oc_ = np.ascontiguousarray(prob.obs_cam, np.int32)
    xy = np.ascontiguousarray(prob.obs_xy, np.float64)
    pv = _lib.ProblemView(prob.nc, prob.nl, prob.nobs, off.ctypes.data, oc_.ctypes.data, xy.ctypes.data)
    h = C.c_void_p(12345)
    rc = L.rba_create_f64(C.byref(pv), C.byref(o), C.byref(h))
    if rc == 0:
        L.rba_destroy(h)
    return rc, h.value


@pytest.mark.parametrize("fields,code", [(dict(preconditioner_type=3), -1), (dict(preconditioner_type=-1), -1),
                                         (dict(preconditioner_type=2, solver_type=2), -1),
                                         (dict(preconditioner_type=2, linear_solver_type=1), -1),
                                         (dict(preconditioner_type=2, nranks=2, rank=0), -4)],
                         ids=["value_3", "value_-1", "power_series", "dense_schur", "two_ranks"])
def test_rejected_options(fields, code):
    """checked before any device work, so also on a machine without a GPU"""
    assert _create(**fields) == (code, 12345)


def test_python_option_mapping(monkeypatch):
    import rootba_b200 as rb
    from rootba_b200 import _lib
    from rootba_b200.synthetic import synth_bal
    seen = []
    real_lib = _lib.lib()

    class Stub:
        def __getattr__(self, name):
            real = getattr(real_lib, name)
            if not name.startswith("rba_create_"):
                return real

            def create(pv, opts, h):
                seen.append(opts._obj.preconditioner_type)
                raise RuntimeError("stop")
            return create

    monkeypatch.setattr(_lib, "lib", lambda: Stub())
    bp = rb.BalProblem.from_arrays(synth_bal(4, 20, 2.5, seed=1))
    for name, want in (("JACOBI", 0), ("SCHUR_JACOBI", 1), ("CLUSTER_JACOBI", 2)):
        with pytest.raises(RuntimeError, match="stop"):
            rb.LinearizorQR(bp, rb.SolverOptions(preconditioner_type=name))
        assert seen[-1] == want


def test_bal_qr_and_example_parse_the_names():
    from rootba_b200 import _lib
    _lib.build()
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "rootba_b200", "host"), "-s"])
    exe = os.path.join(ROOT, "rootba_b200", "host", "bal_qr")
    assert "CLUSTER_JACOBI" in subprocess.run([exe, "--help"], capture_output=True, text=True, check=True).stdout
    bad = subprocess.run([exe, "--preconditioner-type", "BLOCK"], capture_output=True, text=True)
    assert bad.returncode == 2 and "--preconditioner-type" in bad.stderr
    import sys
    out = subprocess.run([sys.executable, os.path.join(ROOT, "examples", "solve_bal.py"), "--help"], capture_output=True, text=True,
                         check=True).stdout
    assert "CLUSTER_JACOBI" in out and "--cluster-size" in out and "--clusters" in out
