"""Argument checks of the per-instance time-step calls that happen on the host, before any device call (no GPU needed), the [B] form against
the [B, N-1] form, and the declarations of the new entry points in the ctypes binding, the C header and the Julia shim."""
import os
import re

import numpy as np
import pytest

import trajopt_b200 as TO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _NoDevice:
    """stands in for a Problem: any device call is an error, so a test passes only when the check comes first"""

    def __init__(self, B=4, N=11, hybrid=False):
        self.n, self.m, self.N, self.B, self.hybrid = 4, 2, N, B, hybrid

    def _call(self, name, *args):
        raise AssertionError(f"device call {name} reached")

    def _raw_call(self, name, *args):
        raise AssertionError(f"device call {name} reached")

    def _ensure_current(self):
        raise AssertionError("device call reached")


def test_shapes():
    p = _NoDevice()
    rows = np.arange(1.0, 41.0).reshape(4, 10) / 40
    dt, t0 = TO.api._time_step_rows(p, rows)
    assert dt.shape == (4, 10) and dt.dtype == np.float64 and dt.flags.c_contiguous and np.array_equal(dt, rows) and t0 is None
    dt, _ = TO.api._time_step_rows(p, np.asfortranarray(rows))          # a Fortran-ordered copy comes back C-contiguous
    assert dt.flags.c_contiguous and np.array_equal(dt, rows)
    _, t0 = TO.api._time_step_rows(p, rows, [0, 1, 2, 3])              # integer initial times
    assert t0.dtype == np.float64 and np.array_equal(t0, [0.0, 1.0, 2.0, 3.0])
    _, t0 = TO.api._time_step_rows(p, rows, 2.5)                       # a scalar initial time: every instance
    assert np.array_equal(t0, [2.5] * 4)
    for bad in [np.ones((4, 9)), np.ones((3, 10)), np.ones((4, 10, 1)), np.ones(3), np.ones(10), np.ones((10, 4)), 0.1]:
        with pytest.raises(TO.DimensionMismatch):
            TO.set_time_steps(p, bad)
    for bad in [np.zeros(3), np.zeros((4, 1)), np.zeros(5)]:
        with pytest.raises(TO.DimensionMismatch):
            TO.set_time_steps(p, np.full((4, 10), 0.1), bad)


def test_uniform_form_is_the_reference_scalar_dt():
    """dt[B]: one uniform step per instance, the bits Problem(..., tf_b) builds (np.full(N - 1, (tf_b - t0) / (N - 1)))"""
    N = 101
    p = _NoDevice(B=5, N=N)
    tf = np.array([4.0, 4.5, 5.0, 5.3, 6.0])
    dt, _ = TO.api._time_step_rows(p, (tf - 0.0) / (N - 1))
    full, _ = TO.api._time_step_rows(p, np.stack([np.full(N - 1, (t - 0.0) / (N - 1)) for t in tf]))
    assert np.array_equal(dt, full)
    for b, t in enumerate(tf):
        assert np.array_equal(dt[b], np.full(N - 1, float(t - 0.0) / (N - 1)))   # api.Problem's dtv for dt=None


@pytest.mark.parametrize("val", [0.0, -0.1, np.nan, np.inf, -np.inf])
def test_steps_must_be_finite_and_positive(val):
    p = _NoDevice()
    rows = np.full((4, 10), 0.1); rows[2, 7] = val
    with pytest.raises(TO.ArgumentError, match="instance 2, knot 7"):
        TO.set_time_steps(p, rows)
    uni = np.full(4, 0.1); uni[3] = val
    with pytest.raises(TO.ArgumentError, match="instance 3, knot 0"):
        TO.set_time_steps(p, uni)


@pytest.mark.parametrize("val", [np.nan, np.inf, -np.inf])
def test_initial_times_must_be_finite(val):
    p = _NoDevice()
    t0 = np.zeros(4); t0[1] = val
    with pytest.raises(TO.ArgumentError, match="instance 1"):
        TO.set_time_steps(p, np.full((4, 10), 0.1), t0)


def test_hybrid_problem_refuses():
    with pytest.raises(TO.ArgumentError, match="hybrid"):
        TO.set_time_steps(_NoDevice(hybrid=True), np.full((4, 10), 0.1))


def test_entry_points_declared():
    from trajopt_b200 import capi
    for name in ("to_set_time_steps", "to_get_time_steps"):
        assert name in capi.EXPORTED_SYMBOLS
    src = open(os.path.join(ROOT, "trajectoryoptimization.jl_b200", "_capi.py")).read()
    assert re.search(r'"to_set_time_steps": \[H, c_double_p, c_double_p\]', src)
    assert re.search(r'"to_get_time_steps": \[H, c_double_p, c_double_p\]', src)
    hdr = open(os.path.join(ROOT, "include", "trajopt_b200.h")).read()
    assert re.search(r"int to_set_time_steps\(to_handle\* h, const double\* dt /\*\[B\]\[N-1\]\*/, const double\* t0 /\*\[B\] or NULL: keep the clocks\*/\);", hdr)
    assert re.search(r"int to_get_time_steps\(to_handle\* h, double\* dt /\*\[B\]\[N-1\]\*/, double\* t0 /\*\[B\] or NULL\*/\);", hdr)
    jl = open(os.path.join(ROOT, "trajectoryoptimization.jl_b200", "julia", "B200TrajOpt.jl")).read()
    assert "function set_time_steps!(p::BatchedProblem, dt::AbstractMatrix, t0::Union{Nothing,AbstractVector}=nothing)" in jl
    assert "function time_steps(p::BatchedProblem)" in jl
    assert re.search(r"ccall\(\(:to_set_time_steps, libb200\), Cint, \(Ptr\{Cvoid\}, Ptr\{Float64\}, Ptr\{Float64\}\), p\.h, Matrix\{Float64\}\(dt\),", jl)
    assert re.search(r"ccall\(\(:to_get_time_steps, libb200\), Cint, \(Ptr\{Cvoid\}, Ptr\{Float64\}, Ptr\{Float64\}\), p\.h, dt, t0\)", jl)
    assert callable(TO.set_time_steps) and callable(TO.time_steps) and callable(TO.instance_times)
    assert "to_set_time_steps" in open(os.path.join(ROOT, "INTEGRATION.md")).read()
