"""Argument checks of the per-instance penalty calls that happen on the host, before any device call (no GPU needed), and the declarations of
the new entry points in the ctypes binding, the C header and the Julia shim."""
import os
import re

import numpy as np
import pytest

import trajopt_b200 as TO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _NoDevice:
    """stands in for a Problem: any device call is an error, so a test passes only when the check comes first"""

    def __init__(self, B=4, hybrid=False):
        n, m, N = 4, 2, 11
        self.n, self.m, self.N, self.B, self.hybrid = n, m, N, B, hybrid
        self.constraints = TO.ConstraintList(n, m, N)
        self.goal = TO.GoalConstraint(np.zeros(n))
        self.bound = TO.BoundConstraint(n, m, u_min=-1.0, u_max=1.0)
        TO.add_constraint(self.constraints, self.goal, N)
        TO.add_constraint(self.constraints, self.bound, (1, N - 1))

    def _call(self, name, *args):
        raise AssertionError(f"device call {name} reached")

    def _raw_call(self, name, *args):
        raise AssertionError(f"device call {name} reached")

    def _ensure_current(self):
        raise AssertionError("device call reached")


def test_shapes_and_scalar_broadcast():
    p = _NoDevice()
    i, mu = TO.api._penalty_rows(p, 1, 3.0)
    assert i == 1 and mu.shape == (4,) and mu.dtype == np.float64 and np.array_equal(mu, [3.0] * 4)
    i, mu = TO.api._penalty_rows(p, p.goal, [1, 2, 3, 4])                # the constraint object, integer entries
    assert i == 0 and np.array_equal(mu, [1.0, 2.0, 3.0, 4.0]) and mu.flags.c_contiguous
    i, mu = TO.api._penalty_rows(p, 0, np.arange(8.0)[::2] + 1)           # a strided view is copied contiguous
    assert mu.flags.c_contiguous and np.array_equal(mu, [1.0, 3.0, 5.0, 7.0])
    for bad in [np.ones(3), np.ones(5), np.ones((4, 1)), np.ones((1, 4))]:
        with pytest.raises(TO.DimensionMismatch):
            TO.set_penalties(p, 0, bad)


@pytest.mark.parametrize("val", [0.0, -1.0, np.nan, np.inf, -np.inf])
def test_entries_must_be_finite_and_positive(val):
    p = _NoDevice()
    mu = np.ones(4); mu[2] = val
    with pytest.raises(TO.ArgumentError, match="instance 2"):
        TO.set_penalties(p, 0, mu)
    with pytest.raises(TO.ArgumentError, match="instance 0"):
        TO.set_penalties(p, 1, val)                                       # a scalar: every instance, the first one named


def test_index_and_problem_errors():
    p = _NoDevice()
    for con in (2, -1, 7):
        with pytest.raises(TO.ArgumentError):
            TO.set_penalties(p, con, 1.0)
    with pytest.raises(TO.ArgumentError):                                 # not one of the problem's constraints
        TO.set_penalties(p, TO.GoalConstraint(np.zeros(4)), 1.0)
    with pytest.raises(TO.ArgumentError, match="hybrid"):
        TO.set_penalties(_NoDevice(hybrid=True), 0, 1.0)


def test_entry_points_declared():
    from trajopt_b200 import capi
    for name in ("to_set_penalties", "to_get_penalties"):
        assert name in capi.EXPORTED_SYMBOLS
    src = open(os.path.join(ROOT, "trajectoryoptimization.jl_b200", "_capi.py")).read()
    assert re.search(r'"to_set_penalties": \[H, C\.c_int32, c_double_p\]', src)
    assert re.search(r'"to_get_penalties": \[H, C\.c_int32, c_double_p\]', src)
    hdr = open(os.path.join(ROOT, "include", "trajopt_b200.h")).read()
    assert re.search(r"int to_set_penalties\(to_handle\* h, int32_t con, const double\* mu /\*\[B\]\*/\);", hdr)
    assert re.search(r"int to_get_penalties\(to_handle\* h, int32_t con, double\* mu /\*\[B\]\*/\);", hdr)
    jl = open(os.path.join(ROOT, "trajectoryoptimization.jl_b200", "julia", "B200TrajOpt.jl")).read()
    assert "function set_penalties!(p::BatchedProblem, con::Integer, mu::AbstractVector)" in jl
    assert "function penalties(p::BatchedProblem, con::Integer)" in jl
    assert re.search(r"ccall\(\(:to_set_penalties, libb200\), Cint, \(Ptr\{Cvoid\}, Int32, Ptr\{Float64\}\), p\.h, con - 1,", jl)
    assert re.search(r"ccall\(\(:to_get_penalties, libb200\), Cint, \(Ptr\{Cvoid\}, Int32, Ptr\{Float64\}\), p\.h, con - 1, mu\)", jl)
    assert callable(TO.set_penalties) and callable(TO.penalties)
    assert "to_set_penalties" in open(os.path.join(ROOT, "INTEGRATION.md")).read()
