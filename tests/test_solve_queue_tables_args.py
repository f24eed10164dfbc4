"""Argument checks of solve_queue's per-problem tables that happen on the host, before any device call (no GPU needed), and the declarations
of to_solve_queue_tables and to_queue_table in the C header, the ctypes binding, INTEGRATION.md and the Julia shim."""
import ctypes
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

import trajopt_b200 as TO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIELDS = ["kind", "index", "len", "pad", "rows", "rows2"]
M = 3


class _NoDevice:
    """stands in for a Problem: any device call is an error, so a test passes only when the check comes first"""

    def __init__(self, hybrid=False):
        self.model = TO.Cartpole()
        self.hybrid = hybrid
        self.n, self.m = 4, 1
        self.B, self.N = 4, 11
        self.obj = TO.LQRObjective(np.eye(4), np.eye(1), np.eye(4), np.zeros(4), self.N)
        self._cost_objs = [self.obj[0], self.obj[self.N - 1]]
        self.constraints = TO.ConstraintList(4, 1, self.N)
        self.bound = TO.BoundConstraint(4, 1, u_min=-3.0, u_max=3.0)
        self.goal = TO.GoalConstraint(np.zeros(4))
        TO.add_constraint(self.constraints, self.bound, range(1, self.N))
        TO.add_constraint(self.constraints, self.goal, self.N)

    def _call(self, name, *args):
        raise AssertionError(f"device call {name} reached")

    _raw_call = _call


def _args(p):
    return np.zeros((M, p.n)), np.zeros((M, p.N - 1, p.m))


def _queue(p, **kw):
    return TO.solve_queue(p, *_args(p), **kw)


def _bound_rows(p):
    return np.tile(np.r_[np.full(4, np.inf), 3.0, np.full(4, -np.inf), -3.0], (M, 1))     # z_max | z_min of (x, u)


def test_valid_tables_reach_the_device():
    p = _NoDevice()
    ok = dict(dt=np.full(M, 0.1), cost_weights={0: np.ones((M, 6))}, constraint_data={0: _bound_rows(p)})
    with pytest.raises(AssertionError, match="device call to_solve_queue_tables reached"):
        _queue(p, **ok)
    with pytest.raises(AssertionError, match="device call to_solve_queue_tables reached"):
        _queue(p, Xref=np.zeros((M, 12, 4)), Uref=np.zeros((M, 12, 1)), start=2, xf=np.zeros((M, 4)), objective=False)
    with pytest.raises(AssertionError, match="device call to_solve_queue_tables reached"):
        _queue(p, penalties={1: 10.0}, **ok)
    # cost objects: the problem's linear terms, which their q and r must equal, are read once every other check has passed
    with pytest.raises(AssertionError, match="device call to_get_cost_terms reached"):
        _queue(p, cost_weights={0: [p._cost_objs[0]] * M}, dt=np.full(M, 0.1))
    with pytest.raises(AssertionError, match="device call to_solve_queue_tables reached"):      # a reference replaces every q | r
        _queue(p, cost_weights={0: [p._cost_objs[0]] * M}, Xref=np.zeros((M, 11, 4)), Uref=np.zeros((M, 11, 1)))


def test_no_tables_keep_the_plain_entry_point():
    p = _NoDevice()
    with pytest.raises(AssertionError, match="device call to_solve_queue reached"):
        _queue(p, cost_weights={}, constraint_data={}, penalties={})


def test_time_steps():
    p = _NoDevice()
    with pytest.raises(TO.DimensionMismatch, match=r"solve_queue: expected \[3, 10\] or \[3\] time steps"):
        _queue(p, dt=np.full((4, 10), 0.1))
    dt = np.full((M, 10), 0.1); dt[2, 4] = 0.0
    with pytest.raises(TO.ArgumentError, match="solve_queue: problem 2, knot 4: a time step must be finite and positive"):
        _queue(p, dt=dt)


def test_cost_weights():
    p = _NoDevice()
    w = np.ones((M, 6)); w[1, 3] = np.inf
    with pytest.raises(TO.ArgumentError, match="solve_queue: problem 1, entry 3 is not finite"):
        _queue(p, cost_weights={0: w})
    with pytest.raises(TO.DimensionMismatch, match=r"solve_queue: expected \[3, 6\] rows"):
        _queue(p, cost_weights={0: np.ones((M, 5))})
    with pytest.raises(TO.DimensionMismatch, match="solve_queue: 2 costs for 3 problems"):
        _queue(p, cost_weights={0: [p._cost_objs[0]] * 2})
    with pytest.raises(TO.ArgumentError, match="the same table is given twice"):
        _queue(p, cost_weights={0: np.ones((M, 6)), p._cost_objs[0]: np.ones((M, 6))})


def test_quadratic_cost_h_stays_zero():
    p = _NoDevice()
    cost = TO.QuadraticCost(np.eye(4), np.eye(1))
    p._cost_objs = [cost]
    w = np.tile(TO.api._cost_weight_row(cost), (M, 1)); w[2, 17] = 0.5       # H sits at [16 + 1, 16 + 1 + 4)
    with pytest.raises(TO.ArgumentError, match="solve_queue: problem 2, entry 17: H must stay zero"):
        _queue(p, cost_weights={0: w})


def test_constraint_data():
    p = _NoDevice()
    rows = _bound_rows(p); rows[1, 0] = 5.0
    with pytest.raises(TO.ArgumentError, match="solve_queue: problem 1, entry 0: BoundConstraint entries must be finite exactly where"):
        _queue(p, constraint_data={0: rows})
    rows = _bound_rows(p); rows[2, 9] = 4.0
    with pytest.raises(TO.ArgumentError, match="solve_queue: problem 2, entry 4: Upper bounds must be greater"):
        _queue(p, constraint_data={0: rows})
    with pytest.raises(TO.ArgumentError, match="a Goal constraint's values come from xf"):
        _queue(p, constraint_data={1: np.zeros((M, 4))})
    with pytest.raises(TO.ArgumentError, match="the same table is given twice"):
        _queue(p, constraint_data={0: _bound_rows(p), p.bound: _bound_rows(p)})


def test_norm_value_non_negative():
    p = _NoDevice()
    norm = TO.NormConstraint(4, 1, 2.0, TO.Inequality(), inds="control")
    TO.add_constraint(p.constraints, norm, range(1, p.N))
    rows = np.ones((M, 1)); rows[1, 0] = -1.0
    with pytest.raises(TO.ArgumentError, match="solve_queue: problem 1: NormConstraint value must be non-negative"):
        _queue(p, constraint_data={2: rows})


def test_penalties():
    p = _NoDevice()
    with pytest.raises(TO.ArgumentError, match="solve_queue: problem 2: a penalty must be finite and positive"):
        _queue(p, penalties={0: np.array([1.0, 2.0, 0.0])})
    with pytest.raises(TO.DimensionMismatch, match=r"solve_queue: expected \[3\] penalties"):
        _queue(p, penalties={0: np.ones(4)})
    with pytest.raises(TO.ArgumentError, match="solve_queue: no constraint 5"):
        _queue(p, penalties={5: 1.0})


def test_reference():
    p = _NoDevice()
    X, U = np.zeros((M, 12, 4)), np.zeros((M, 12, 1))
    with pytest.raises(TO.ArgumentError, match="Xref and Uref come together"):
        _queue(p, Xref=X)
    with pytest.raises(TO.DimensionMismatch, match="the reference is shorter than start \\+ N - 1"):
        _queue(p, Xref=X, Uref=U, start=3)
    with pytest.raises(TO.DimensionMismatch, match=r"Xref must be \[3, nref, 4\]"):
        _queue(p, Xref=X[:2], Uref=U[:2])
    X2 = X.copy(); X2[1, 5, 2] = np.nan
    with pytest.raises(TO.ArgumentError, match="solve_queue: problem 1, row 5, entry 2: Xref is not finite"):
        _queue(p, Xref=X2, Uref=U)
    with pytest.raises(TO.ArgumentError, match="a reference and xf with objective=True"):
        _queue(p, Xref=X, Uref=U, xf=np.zeros((M, 4)))


def test_hybrid_problems_refuse_the_tables():
    p = _NoDevice(hybrid=True)
    for kw, msg in ((dict(dt=np.full(M, 0.1)), "time steps"), (dict(cost_weights={0: np.ones((M, 6))}), "cost weights"),
                    (dict(constraint_data={0: _bound_rows(p)}), "constraint data"), (dict(penalties={0: 1.0}), "penalties"),
                    (dict(Xref=np.zeros((M, 11, 4)), Uref=np.zeros((M, 11, 1))), "goals")):
        with pytest.raises(TO.ArgumentError, match=f"per-instance {msg} are not supported on hybrid problems|per-instance {msg} is not supported"):
            TO.api._queue_tables(p, M, None, True, **{**dict(dt=None, cost_weights=None, constraint_data=None, penalties=None, Xref=None,
                                                             Uref=None, start=1), **kw})


def test_entry_point_declared():
    from trajopt_b200 import capi
    assert "to_solve_queue_tables" in capi.EXPORTED_SYMBOLS
    lib = capi.load_library()
    assert lib.to_solve_queue_tables.argtypes[1:] == ([ctypes.POINTER(capi.to_queue_spec), ctypes.POINTER(capi.to_queue_table), ctypes.c_int32,
                                                       ctypes.POINTER(capi.to_solve_options)] + [capi.c_int32_p] * 3 + [capi.c_double_p] * 6)
    hdr = open(os.path.join(ROOT, "include", "trajopt_b200.h")).read()
    assert ("enum to_queue_table_kind { TO_QT_TIME_STEPS = 0, TO_QT_COST_WEIGHTS = 1, TO_QT_CONSTRAINT_DATA = 2, TO_QT_PENALTIES = 3, "
            "TO_QT_REFERENCE = 4 };") in hdr
    assert (capi.QT_TIME_STEPS, capi.QT_COST_WEIGHTS, capi.QT_CONSTRAINT_DATA, capi.QT_PENALTIES, capi.QT_REFERENCE) == (0, 1, 2, 3, 4)
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    assert ("`to_solve_queue_tables(h, const to_queue_spec*, const to_queue_table*, ntables, const to_solve_options*, status, iterations, "
            "iterations_outer, cost, dJ, gradient, c_max, X, U)`") in doc
    jl = open(os.path.join(ROOT, "trajectoryoptimization.jl_b200", "julia", "B200TrajOpt.jl")).read()
    assert re.search(r"function solve_queue!\(p::BatchedProblem, x0s, U0s; xf = nothing, params = nothing, objective::Bool = true, "
                     r"constraint::Bool = true,\s*dt = nothing, cost_weights = Dict\(\), constraint_data = Dict\(\), penalties = Dict\(\), "
                     r"Xref = nothing, Uref = nothing,\s*start::Integer = 1, kw\.\.\.\)", jl)
    assert re.search(r"ccall\(\(:to_solve_queue_tables, libb200\), Cint,\s*\(Ptr\{Cvoid\}, Ref\{ToQueueSpec\}, Ptr\{ToQueueTable\}, Int32, "
                     r"Ref\{ToSolveOptions\}, Ptr\{Int32\}, Ptr\{Int32\}, Ptr\{Int32\},\s*Ptr\{Float64\}, Ptr\{Float64\}, Ptr\{Float64\}, "
                     r"Ptr\{Float64\}, Ptr\{Float64\}, Ptr\{Float64\}\)", jl)


@pytest.mark.parametrize("lang", ["c", "c++"])
def test_header_compiles(lang):
    src = ("#include \"trajopt_b200.h\"\n"
           "int (*fn)(to_handle*, const to_queue_spec*, const to_queue_table*, int32_t, const to_solve_options*, int32_t*, int32_t*, int32_t*,"
           " double*, double*, double*, double*, double*, double*) = to_solve_queue_tables;\n"
           "int main(void) { to_queue_table t = {TO_QT_REFERENCE, 1, 2, 0, 0, 0}; return fn == 0 || t.kind != 4; }\n")
    with tempfile.TemporaryDirectory() as d:
        f = os.path.join(d, "l.c" if lang == "c" else "l.cpp")
        open(f, "w").write(src)
        subprocess.check_call(["gcc" if lang == "c" else "g++", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-fsyntax-only", f])


def test_queue_table_layout_matches_the_binding_tables():
    """to_queue_table's offsets: offsetof / sizeof printed by a C program compiled from include/trajopt_b200.h, against INTEGRATION.md's
    to_queue_table table, the ctypes structure and the Julia struct's field order"""
    src = "#include <stdio.h>\n#include <stddef.h>\n#include \"trajopt_b200.h\"\nint main() {\n"
    for f in FIELDS:
        src += f'  printf("{f} %zu\\n", offsetof(to_queue_table, {f}));\n'
    src += '  printf("sizeof %zu\\n", sizeof(to_queue_table));\n  return 0;\n}\n'
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "l.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "l.c"), "-o", os.path.join(d, "l")])
        out = subprocess.check_output([os.path.join(d, "l")], text=True)
    c_layout = {l.split()[0]: int(l.split()[1]) for l in out.splitlines()}
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    section = doc[doc.index("### `to_queue_table`"):]
    section = section[:section.index("\n### ", 1)]
    table = {m.group(1): int(m.group(2)) for m in re.finditer(r"^\| (\w+) \| (\d+) \|", section, flags=re.M)}
    table["sizeof"] = int(re.search(r"`sizeof\(to_queue_table\)` = (\d+)", section).group(1))
    assert table == c_layout
    cls = TO.capi.to_queue_table
    assert [f for f, _ in cls._fields_] == FIELDS
    assert ctypes.sizeof(cls) == c_layout["sizeof"]
    for f in FIELDS:
        assert getattr(cls, f).offset == c_layout[f], f
    jl = open(os.path.join(ROOT, "trajectoryoptimization.jl_b200", "julia", "B200TrajOpt.jl")).read()
    jbody = re.search(r"struct ToQueueTable\n(.*?)\nend", jl, flags=re.S).group(1)
    assert re.findall(r"(\w+)::", jbody) == FIELDS
