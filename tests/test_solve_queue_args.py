"""Argument checks of solve_queue that happen on the host, before any device call (no GPU needed), and the declarations of to_solve_queue and
to_queue_spec in the C header, the ctypes binding, INTEGRATION.md and the Julia shim."""
import ctypes
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

import trajopt_b200 as TO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIELDS = ["M", "U0_shared", "x0", "U0", "xf", "goal_objective", "goal_constraint", "params", "nparams", "pad"]


class _NoDevice:
    """stands in for a Problem: any device call is an error, so a test passes only when the check comes first"""

    def __init__(self, model=None, ncon=1, N=11):
        self.model = model if model is not None else TO.Cartpole()
        self.hybrid = isinstance(self.model, (list, tuple))
        m0 = self.model[0] if self.hybrid else self.model
        self.n, self.m = m0.n, m0.m
        self.B, self.N = 4, N
        self.constraints = [object()] * ncon

    def _call(self, name, *args):
        raise AssertionError(f"device call {name} reached")

    _raw_call = _call


def _args(p, M=3):
    return np.zeros((M, p.n)), np.zeros((M, p.N - 1, p.m))


def _recorded(N=11, hybrid=False):
    f = lambda x, u: [x[2], x[3], u[0], u[0]]
    if hybrid:
        return [TO.AutodiffDynamics(4, 1, f), TO.AutodiffDynamics(4, 1, f)] * ((N - 1) // 2)
    return [TO.AutodiffDynamics(4, 1, f)] * (N - 1)


def test_valid_arguments_reach_the_device():
    p = _NoDevice()
    x0, U0 = _args(p)
    with pytest.raises(AssertionError, match="device call to_solve_queue reached"):
        TO.solve_queue(p, x0, U0, xf=np.zeros((3, 4)), params=np.ones((3, 4)), iterations=5)
    with pytest.raises(AssertionError, match="device call to_solve_queue reached"):   # one U0 for every problem
        TO.solve_queue(p, x0, U0[0])


def test_empty_queue():
    p = _NoDevice()
    with pytest.raises(TO.ArgumentError, match="M >= 1"):
        TO.solve_queue(p, np.zeros((0, 4)), np.zeros((10, 1)))


@pytest.mark.parametrize("what", ["x0", "U0", "xf", "params"])
def test_non_finite_entries(what):
    p = _NoDevice()
    x0, U0 = _args(p)
    kw = dict(xf=np.zeros((3, 4)), params=np.ones((3, 4)))
    a = {"x0": x0, "U0": U0, **kw}[what]
    a[(1,) + (0,) * (a.ndim - 1)] = np.nan
    with pytest.raises(TO.ArgumentError, match=f"problem 1: {what} is not finite"):
        TO.solve_queue(p, x0, U0, **kw)


def test_shapes():
    p = _NoDevice()
    x0, U0 = _args(p)
    with pytest.raises(TO.DimensionMismatch, match="x0 must be"):
        TO.solve_queue(p, np.zeros(4), U0)
    with pytest.raises(TO.DimensionMismatch, match="U0 must be"):
        TO.solve_queue(p, x0, np.zeros((2, p.N - 1, p.m)))
    with pytest.raises(TO.DimensionMismatch, match="xf must be"):
        TO.solve_queue(p, x0, U0, xf=np.zeros((2, 4)))
    with pytest.raises(TO.DimensionMismatch, match="params must be"):
        TO.solve_queue(p, x0, U0, params=np.ones((3, 3)))


def test_parameter_rows_the_setter_refuses():
    p = _NoDevice()
    x0, U0 = _args(p)
    params = np.ones((3, 4)); params[2, 1] = 0.0     # mp
    with pytest.raises(TO.ArgumentError, match=r"problem 2, parameter 1 \(mp\) must be positive"):
        TO.solve_queue(p, x0, U0, params=params)


def test_unknown_options():
    p = _NoDevice()
    with pytest.raises(TO.ArgumentError, match="unknown solve option cost_tol"):
        TO.solve_queue(p, *_args(p), cost_tol=1e-3)


def test_hybrid_problems_refuse():
    p = _NoDevice(model=_recorded(hybrid=True), ncon=0)
    with pytest.raises(TO.ArgumentError, match="solve_queue: not supported on hybrid problems"):
        TO.solve_queue(p, *_args(p))


def test_recorded_model():
    """one AutodiffDynamics model stepping every knot: no constraints, no xf, no params; x0 and U0 alone pass every host check"""
    for kw, ncon in ((dict(), 1), (dict(xf=np.zeros((3, 4))), 0), (dict(params=np.ones((3, 4))), 0)):
        p = _NoDevice(model=_recorded(), ncon=ncon)
        with pytest.raises(TO.ArgumentError, match="recorded-program"):
            TO.solve_queue(p, *_args(p), **kw)
    p = _NoDevice(model=_recorded(), ncon=0)
    with pytest.raises(AssertionError, match="device call to_solve_queue reached"):
        TO.solve_queue(p, *_args(p))


def test_entry_point_declared():
    from trajopt_b200 import capi
    assert "to_solve_queue" in capi.EXPORTED_SYMBOLS
    lib = capi.load_library()
    assert lib.to_solve_queue.argtypes[1:] == ([ctypes.POINTER(capi.to_queue_spec), ctypes.POINTER(capi.to_solve_options)] + [capi.c_int32_p] * 3
                                               + [capi.c_double_p] * 6)
    hdr = open(os.path.join(ROOT, "include", "trajopt_b200.h")).read()
    assert ("int to_solve_queue(to_handle* h, const to_queue_spec* q, const to_solve_options* o, int32_t* status, int32_t* iterations, "
            "int32_t* iterations_outer,\n                   double* cost, double* dJ, double* gradient, double* c_max, double* X, double* U);") in hdr
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    assert "`to_solve_queue(h, const to_queue_spec*, const to_solve_options*, status, iterations, iterations_outer, cost, dJ, gradient, c_max, X, U)`" in doc
    jl = open(os.path.join(ROOT, "trajectoryoptimization.jl_b200", "julia", "B200TrajOpt.jl")).read()
    assert "function solve_queue!(p::BatchedProblem, x0s, U0s; xf = nothing, params = nothing" in jl
    assert re.search(r"ccall\(\(:to_solve_queue, libb200\), Cint,\s*\(Ptr\{Cvoid\}, Ref\{ToQueueSpec\}, Ref\{ToSolveOptions\}, Ptr\{Int32\}, Ptr\{Int32\}, "
                     r"Ptr\{Int32\}, Ptr\{Float64\}, Ptr\{Float64\}, Ptr\{Float64\},\s*Ptr\{Float64\}, Ptr\{Float64\}, Ptr\{Float64\}\)", jl)
    assert callable(TO.solve_queue)


@pytest.mark.parametrize("lang", ["c", "c++"])
def test_header_compiles(lang):
    src = ("#include \"trajopt_b200.h\"\n"
           "int (*fn)(to_handle*, const to_queue_spec*, const to_solve_options*, int32_t*, int32_t*, int32_t*, double*, double*, double*, double*,"
           " double*, double*) = to_solve_queue;\n"
           "int main(void) { return fn == 0; }\n")
    with tempfile.TemporaryDirectory() as d:
        f = os.path.join(d, "l.c" if lang == "c" else "l.cpp")
        open(f, "w").write(src)
        subprocess.check_call(["gcc" if lang == "c" else "g++", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-fsyntax-only", f])


def test_queue_spec_layout_matches_the_binding_tables():
    """to_queue_spec's offsets: offsetof / sizeof printed by a C program compiled from include/trajopt_b200.h, against INTEGRATION.md's
    to_queue_spec table, the ctypes structure and the Julia struct's field order"""
    src = "#include <stdio.h>\n#include <stddef.h>\n#include \"trajopt_b200.h\"\nint main() {\n"
    for f in FIELDS:
        src += f'  printf("{f} %zu\\n", offsetof(to_queue_spec, {f}));\n'
    src += '  printf("sizeof %zu\\n", sizeof(to_queue_spec));\n  return 0;\n}\n'
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "l.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "l.c"), "-o", os.path.join(d, "l")])
        out = subprocess.check_output([os.path.join(d, "l")], text=True)
    c_layout = {l.split()[0]: int(l.split()[1]) for l in out.splitlines()}
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    section = doc[doc.index("### `to_queue_spec`"):]
    section = section[:section.index("\n### ", 1)]
    table = {m.group(1): int(m.group(2)) for m in re.finditer(r"^\| (\w+) \| (\d+) \|", section, flags=re.M)}
    table["sizeof"] = int(re.search(r"`sizeof\(to_queue_spec\)` = (\d+)", section).group(1))
    assert table == c_layout
    cls = TO.capi.to_queue_spec
    assert [f for f, _ in cls._fields_] == FIELDS
    assert ctypes.sizeof(cls) == c_layout["sizeof"]
    for f in FIELDS:
        assert getattr(cls, f).offset == c_layout[f], f
    jl = open(os.path.join(ROOT, "trajectoryoptimization.jl_b200", "julia", "B200TrajOpt.jl")).read()
    jbody = re.search(r"struct ToQueueSpec\n(.*?)\nend", jl, flags=re.S).group(1)
    assert re.findall(r"(\w+)::", jbody) == FIELDS
