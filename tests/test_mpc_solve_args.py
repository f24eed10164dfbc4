"""Argument checks of mpc_solve / mpc_solve_history that happen on the host, before any device call (no GPU needed), and the declarations
of the two entry points in the C header, the ctypes binding, INTEGRATION.md and the Julia shim."""
import ctypes
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

import trajopt_b200 as TO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _NoDevice:
    """stands in for a Problem after mpc_setup: any device call is an error, so a test passes only when the check comes first"""

    def __init__(self, B=4, N=11, model=None, ncon=1, done=3, nsteps=5):
        self.model = model if model is not None else TO.Cartpole()
        self.hybrid = isinstance(self.model, (list, tuple))
        self.B, self.N = B, N
        self.constraints = [object()] * ncon
        self._mpc = {"nsteps": nsteps, "done": done}

    def _call(self, name, *args):
        raise AssertionError(f"device call {name} reached")

    _raw_call = _call

    def _ensure_current(self):
        raise AssertionError("device call reached")


def _recorded(N=11, hybrid=False):
    f = lambda x, u: [x[2], x[3], u[0], u[0]]
    if hybrid:
        return [TO.AutodiffDynamics(4, 1, f), TO.AutodiffDynamics(4, 1, f)] * ((N - 1) // 2)
    return [TO.AutodiffDynamics(4, 1, f)] * (N - 1)


def test_before_setup():
    p = _NoDevice()
    del p._mpc
    with pytest.raises(TO.ArgumentError, match="mpc_solve before mpc_setup"):
        TO.mpc_solve(p, 1)
    with pytest.raises(TO.ArgumentError, match="mpc_solve_history before mpc_setup"):
        TO.mpc_solve_history(p)


@pytest.mark.parametrize("steps", [0, -1, 1.5])
def test_steps_must_be_positive_integers(steps):
    p = _NoDevice()
    with pytest.raises(TO.ArgumentError, match="mpc_solve: steps must be a positive integer"):
        TO.mpc_solve(p, steps)
    assert p._mpc["done"] == 3


def test_beyond_nsteps():
    p = _NoDevice()
    with pytest.raises(TO.DimensionMismatch, match="mpc_solve: 3 steps done \\+ 3 exceed the setup's nsteps = 5"):
        TO.mpc_solve(p, 3)
    assert p._mpc["done"] == 3
    with pytest.raises(AssertionError, match="device call to_mpc_solve reached"):   # 3 + 2 fit: the device call comes next
        TO.mpc_solve(p, 2)


def test_unknown_options():
    p = _NoDevice()
    with pytest.raises(TO.ArgumentError, match="unknown solve option cost_tol"):
        TO.mpc_solve(p, 1, cost_tol=1e-3)
    assert p._mpc["done"] == 3


def test_hybrid_problems_refuse():
    p = _NoDevice(model=_recorded(hybrid=True), ncon=0)
    with pytest.raises(TO.ArgumentError, match="mpc_solve: closed-loop MPC is not supported on hybrid problems"):
        TO.mpc_solve(p, 1)
    jump = TO.AutodiffDynamics(4, 1, lambda x, u: [x[2], x[3], u[0], u[0]], discrete=True)
    p = _NoDevice(model=[jump] * 10, ncon=0)
    with pytest.raises(TO.ArgumentError, match="hybrid"):
        TO.mpc_solve(p, 1)


def test_recorded_model_only_without_constraints():
    """one AutodiffDynamics model stepping every knot: no per-instance penalties, so a constrained problem cannot take its outer steps on
    the device; an unconstrained one passes every host check"""
    p = _NoDevice(model=_recorded(), ncon=2)
    with pytest.raises(TO.ArgumentError, match="recorded-program"):
        TO.mpc_solve(p, 1)
    p = _NoDevice(model=_recorded(), ncon=0)
    with pytest.raises(AssertionError, match="device call to_mpc_solve reached"):
        TO.mpc_solve(p, 1, iterations=4)
    assert p._mpc["done"] == 3


def test_built_in_model_with_constraints_reaches_the_device():
    p = _NoDevice(ncon=2)
    with pytest.raises(AssertionError, match="device call to_mpc_solve reached"):
        TO.mpc_solve(p, 2, iterations=7, constraint_tolerance=1e-4)


def test_entry_points_declared():
    from trajopt_b200 import capi
    for name in ("to_mpc_solve", "to_mpc_solve_history"):
        assert name in capi.EXPORTED_SYMBOLS
    lib = capi.load_library()
    assert lib.to_mpc_solve.argtypes[1:] == [ctypes.c_int32, ctypes.POINTER(capi.to_solve_options)]
    assert lib.to_mpc_solve_history.argtypes[1:] == [capi.c_int32_p] * 3 + [capi.c_double_p]
    hdr = open(os.path.join(ROOT, "include", "trajopt_b200.h")).read()
    assert "int to_mpc_solve(to_handle* h, int32_t steps, const struct to_solve_options* o);" in hdr
    assert "int to_mpc_solve_history(to_handle* h, int32_t* status, int32_t* iterations, int32_t* iterations_outer, double* c_max);" in hdr
    mpc_block = hdr[hdr.index("---- closed-loop MPC on the device"):hdr.index("---- kernel 1:")]
    assert "int to_mpc_solve(" in mpc_block and "int to_mpc_solve_history(" in mpc_block
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    assert "`to_mpc_solve(h, steps, const to_solve_options*)`" in doc and "`to_mpc_solve_history(h, status, iterations, iterations_outer, c_max)`" in doc
    jl = open(os.path.join(ROOT, "trajectoryoptimization.jl_b200", "julia", "B200TrajOpt.jl")).read()
    for fn in ("function mpc_solve!(p::BatchedProblem, steps::Integer; kw...)", "function mpc_solve_history(p::BatchedProblem)"):
        assert fn in jl
    assert re.search(r"ccall\(\(:to_mpc_solve, libb200\), Cint, \(Ptr\{Cvoid\}, Int32, Ref\{ToSolveOptions\}\), p\.h, steps, o\)", jl)
    assert re.search(r"ccall\(\(:to_mpc_solve_history, libb200\), Cint, \(Ptr\{Cvoid\}, Ptr\{Int32\}, Ptr\{Int32\}, Ptr\{Int32\}, Ptr\{Float64\}\)", jl)
    assert callable(TO.mpc_solve) and callable(TO.mpc_solve_history)


@pytest.mark.parametrize("lang", ["c", "c++"])
def test_header_declares_to_mpc_solve_on_the_options_typedef(lang):
    """to_mpc_solve is declared in the MPC block, ahead of to_solve_options' definition, through the struct tag: the two must name one type"""
    src = ("#include \"trajopt_b200.h\"\n"
           "int (*fn)(to_handle*, int32_t, const to_solve_options*) = to_mpc_solve;\n"
           "int (*hist)(to_handle*, int32_t*, int32_t*, int32_t*, double*) = to_mpc_solve_history;\n"
           "int main(void) { return fn == 0 || hist == 0; }\n")
    with tempfile.TemporaryDirectory() as d:
        f = os.path.join(d, "l.c" if lang == "c" else "l.cpp")
        open(f, "w").write(src)
        cc = "gcc" if lang == "c" else "g++"
        subprocess.check_call([cc, "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-fsyntax-only", f])


def test_history_object_shapes():
    h = TO.MpcSolveHistory(4, 3)
    assert [getattr(h, f).shape for f in h.FIELDS] == [(4, 3)] * 4
    assert [getattr(h, f).dtype for f in h.FIELDS] == [np.int32] * 3 + [np.float64]
