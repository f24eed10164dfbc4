"""Argument checks of the per-instance constraint-data calls that happen on the host, before any device call (no GPU needed)."""

import numpy as np
import pytest

import trajopt_b200 as TO


class _NoDevice:
    """stands in for a Problem: any device call is an error, so a test passes only when the check comes first"""

    def __init__(self, B=4, hybrid=False):
        n, m, N = 4, 2, 11
        self.n, self.m, self.N, self.B, self.hybrid = n, m, N, B, hybrid
        cons = TO.ConstraintList(n, m, N)
        TO.add_constraint(cons, TO.GoalConstraint(np.array([0, 2.0, 0, 0])), N)
        TO.add_constraint(cons, TO.CircleConstraint(n, [0.0, 1.0], [1.0, 0.5], [0.5, 0.2]), (2, N - 1))
        TO.add_constraint(cons, TO.NormConstraint(n, m, 5.0, TO.SecondOrderCone(), "control"), (1, N - 1))
        TO.add_constraint(cons, TO.BoundConstraint(n, m, x_max=[5.0, np.inf, np.inf, np.inf], u_min=-10, u_max=10), (1, N - 1))
        TO.add_constraint(cons, TO.QuatVecEq(n, m, [1.0, 0, 0, 0], (1, 2, 3, 4)), N)
        self.constraints = cons

    def _call(self, name, *args):
        raise AssertionError(f"device call {name} reached")

    def _raw_call(self, name, *args):
        raise AssertionError(f"device call {name} reached")

    def _ensure_current(self):
        raise AssertionError("device call reached")


GOAL, CIRCLE, NORM, BOUND, QUAT = range(5)


def _shared(p, j):
    return np.tile(TO.api._con_row(p.constraints[j])[1], (p.B, 1))


def test_row_lengths():
    p = _NoDevice()
    assert _shared(p, CIRCLE).shape == (4, 6)           # xc | yc | r
    assert _shared(p, NORM).shape == (4, 1)             # val
    assert _shared(p, BOUND).shape == (4, 12)           # z_max[n+m] | z_min[n+m]
    s = TO.api._con_row(TO.SphereConstraint(4, [0.0], [1.0], [2.0], [0.5]))[1]
    assert np.array_equal(s, [0.0, 1.0, 2.0, 0.5])
    assert np.array_equal(TO.api._con_row(TO.CollisionConstraint(4, [1], [2], 0.3))[1], [0.3])
    assert np.array_equal(TO.api._con_row(TO.LinearConstraint(4, 2, np.ones((2, 2)), [1.0, 2.0], TO.Inequality(), "control"))[1], [1.0, 2.0])


def test_wrong_shape_or_count():
    p = _NoDevice()
    for j in (CIRCLE, NORM, BOUND):
        good = _shared(p, j)
        for shape in [(4, good.shape[1] + 1), (3, good.shape[1]), (5, good.shape[1]), (good.shape[1],), (4, good.shape[1], 1)]:
            with pytest.raises(TO.DimensionMismatch):
                TO.set_constraint_data(p, j, np.ones(shape))
    with pytest.raises(TO.DimensionMismatch):
        TO.set_constraint_data(p, GOAL, np.zeros((4, 3)))
    with pytest.raises(TO.DimensionMismatch):       # a sequence of constraints one short
        TO.set_constraint_data(p, CIRCLE, [p.constraints[CIRCLE]] * 3)
    with pytest.raises(TO.DimensionMismatch):       # a Circle with another obstacle count is another shape
        TO.set_constraint_data(p, CIRCLE, [TO.CircleConstraint(4, [0.0], [1.0], [0.5])] * 4)


def test_kind_errors():
    p = _NoDevice()
    with pytest.raises(TO.ArgumentError):
        TO.set_constraint_data(p, QUAT, np.zeros((4, 4)))
    with pytest.raises(TO.ArgumentError):
        TO.set_constraint_data(p, CIRCLE, [TO.SphereConstraint(4, [0.0], [1.0], [2.0], [0.5])] * 4)
    with pytest.raises(TO.ArgumentError):
        TO.set_constraint_data(p, TO.CircleConstraint(4, [0.0], [1.0], [0.5]), _shared(p, CIRCLE))   # not one of the problem's
    with pytest.raises(TO.ArgumentError):
        TO.set_constraint_data(p, 7, np.zeros((4, 1)))
    with pytest.raises(TO.ArgumentError):
        TO.set_constraint_data(_NoDevice(hybrid=True), BOUND, _shared(p, BOUND))
    with pytest.raises(TO.ArgumentError):          # an IndexedConstraint keeps its data shared
        TO.api._con_row(TO.IndexedConstraint(6, 3, TO.BoundConstraint(4, 2, u_min=-1.0, u_max=1.0)))


def test_bound_pattern_and_order_errors():
    p = _NoDevice()
    good = _shared(p, BOUND)
    r = good.copy(); r[1, 1] = 3.0                   # x_max[1] is +Inf in the shared bound
    with pytest.raises(TO.ArgumentError, match="instance 1, entry 1"):
        TO.set_constraint_data(p, BOUND, r)
    r = good.copy(); r[2, 0] = np.inf                # x_max[0] is finite
    with pytest.raises(TO.ArgumentError, match="instance 2, entry 0"):
        TO.set_constraint_data(p, BOUND, r)
    r = good.copy(); r[3, 6] = -np.inf               # x_min[0] is -Inf: -Inf stays, +Inf would not
    r[3, 6] = np.inf
    with pytest.raises(TO.ArgumentError, match="instance 3, entry 6"):
        TO.set_constraint_data(p, BOUND, r)
    r = good.copy(); r[0, 4] = -11.0                 # u_max[0] < u_min[0]
    with pytest.raises(TO.ArgumentError, match="greater than or equal"):
        TO.set_constraint_data(p, BOUND, r)


def test_value_errors():
    p = _NoDevice()
    r = _shared(p, CIRCLE); r[2, 4] = np.nan
    with pytest.raises(TO.ArgumentError, match="instance 2, entry 4"):
        TO.set_constraint_data(p, CIRCLE, r)
    r = _shared(p, NORM); r[1, 0] = -0.5
    with pytest.raises(TO.ArgumentError, match="non-negative"):
        TO.set_constraint_data(p, NORM, r)


def test_constraints_become_rows():
    """a sequence of constraints is the matrix of their data: the rows the device call would take"""
    p = _NoDevice()
    circles = [TO.CircleConstraint(4, [0.1 * b, 1.0], [1.0, 0.5 + 0.1 * b], [0.5, 0.2 + 0.01 * b]) for b in range(4)]
    j, con, rows = TO.api._constraint_data_rows(p, p.constraints[CIRCLE], circles)
    assert j == CIRCLE and con is p.constraints[CIRCLE]
    assert rows.shape == (4, 6) and rows.flags["C_CONTIGUOUS"] and rows.dtype == np.float64
    assert np.array_equal(rows, np.array([np.concatenate([c.x, c.y, c.radius]) for c in circles]))
    goals = [TO.GoalConstraint(np.array([0, 2.0 + b, 0, 0])) for b in range(4)]
    j, con, rows = TO.api._constraint_data_rows(p, GOAL, goals)
    assert j == GOAL and np.array_equal(rows, np.array([g.xf for g in goals]))


def test_new_entry_points_are_declared():
    for name in ("to_constraint_data_len", "to_set_constraint_data", "to_get_constraint_data"):
        assert name in TO._capi.EXPORTED_SYMBOLS
    assert callable(TO.set_constraint_data) and callable(TO.constraint_data)
