"""CPU-side checks of linear_solver_type (DENSE_SCHUR, DESIGN.md section 27): the field's place in rba_solver_opts agrees
between the C header and the ctypes mirror, the default is ITERATIVE_SCHUR, the Python option maps to the C values, and
bal_qr and examples/solve_bal.py offer the flag."""
import ctypes as C
import os
import shutil
import subprocess
import sys

import pytest

from conftest import ROOT


def test_field_matches_the_c_header(tmp_path):
    from rootba_b200 import _lib
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "o.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "rootba_b200.h"\n'
                   'int main(void) { printf("%zu %zu %zu %zu %zu\\n", sizeof(rba_solver_opts), '
                   'offsetof(rba_solver_opts, linear_solver_type), sizeof(((rba_solver_opts*)0)->linear_solver_type), '
                   'offsetof(rba_solver_opts, reserved), sizeof(((rba_solver_opts*)0)->reserved)); return 0; }\n')
    exe = tmp_path / "o"
    subprocess.check_call([cc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    size, off, fsize, r_off, r_size = map(int, subprocess.check_output([str(exe)]).split())
    O = _lib.SolverOpts
    assert size == C.sizeof(O)
    assert (off, fsize) == (O.linear_solver_type.offset, O.linear_solver_type.size) == (off, 4)
    assert (r_off, r_size) == (O.reserved.offset, O.reserved.size) == (off + 4, 4)
    assert O.power_order.offset + 4 == off  # the field took reserved[0]: the struct keeps its size and every other offset


def test_default_is_iterative_schur():
    from rootba_b200 import _lib
    o = _lib.SolverOpts()
    o.linear_solver_type = 7
    _lib.lib().rba_default_solver_opts(C.byref(o))
    assert o.linear_solver_type == 0 and o.reserved[0] == 0
    assert _lib.lib().rba_abi_version() == 1


def test_python_option_mapping(monkeypatch):
    """SolverOptions.linear_solver_type takes the reference's names and LinearizorQR.__init__ passes 0 / 1 to rba_create_*
    (the create call is stubbed: this machine may have no GPU)"""
    import rootba_b200 as rb
    from rootba_b200 import _lib
    from rootba_b200.synthetic import synth_bal
    assert rb.SolverOptions().linear_solver_type == "ITERATIVE_SCHUR"
    seen = []
    real_lib = _lib.lib()

    class Stub:
        def __getattr__(self, name):
            real = getattr(real_lib, name)
            if not name.startswith("rba_create_"):
                return real

            def create(pv, opts, h):
                seen.append(opts._obj.linear_solver_type)
                raise RuntimeError("stop")
            return create

    monkeypatch.setattr(_lib, "lib", lambda: Stub())
    bp = rb.BalProblem.from_arrays(synth_bal(4, 20, 2.5, seed=1))
    for name, want in (("ITERATIVE_SCHUR", 0), ("DENSE_SCHUR", 1)):
        with pytest.raises(RuntimeError, match="stop"):
            rb.LinearizorQR(bp, rb.SolverOptions(linear_solver_type=name))
        assert seen[-1] == want
    with pytest.raises(KeyError):
        rb.LinearizorQR(bp, rb.SolverOptions(linear_solver_type="SPARSE_SCHUR"))


def test_bal_qr_lists_the_flag():
    from rootba_b200 import _lib
    _lib.build()
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "rootba_b200", "host"), "-s"])
    out = subprocess.run([os.path.join(ROOT, "rootba_b200", "host", "bal_qr"), "--help"], capture_output=True, text=True, check=True).stdout
    assert "--linear-solver-type ITERATIVE_SCHUR|DENSE_SCHUR" in out
    bad = subprocess.run([os.path.join(ROOT, "rootba_b200", "host", "bal_qr"), "--linear-solver-type", "SPARSE_SCHUR"],
                         capture_output=True, text=True)
    assert bad.returncode == 2 and "--linear-solver-type" in bad.stderr


def test_solve_bal_lists_the_flag():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "examples", "solve_bal.py"), "--help"], capture_output=True, text=True,
                         check=True).stdout
    assert "--linear-solver-type" in out and "DENSE_SCHUR" in out
