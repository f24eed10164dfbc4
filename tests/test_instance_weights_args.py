"""Argument checks of the per-instance cost-weight calls that happen on the host, before any device call (no GPU needed)."""
import os
import re

import numpy as np
import pytest

import trajopt_b200 as TO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _NoDevice:
    """stands in for a Problem: any device call is an error, so a test passes only when the check comes first"""

    def __init__(self, B=4, hybrid=False):
        n, m = 4, 2
        self.n, self.m, self.B, self.hybrid = n, m, B, hybrid
        H = 0.1 * np.ones((m, n))
        self._cost_objs = [
            TO.DiagonalCost(np.arange(1.0, 5.0), [0.1, 0.2], q=np.ones(n), c=0.5),
            TO.QuadraticCost(np.eye(n) + 0.1, np.eye(m), H=H, c=1.0),
            TO.QuadraticCost(2 * np.eye(n), np.eye(m), terminal=True),
            TO.DiagonalQuatCost(np.ones(n), np.ones(m), w=3.0, q_ind=(1, 2, 3, 4)),
            TO.AutodiffCost(n, m, lambda x, u: x[0] * x[0] + u[0] * u[0]),
        ]

    def _call(self, name, *args):
        raise AssertionError(f"device call {name} reached")

    def _raw_call(self, name, *args):
        raise AssertionError(f"device call {name} reached")

    def _ensure_current(self):
        raise AssertionError("device call reached")


DIAG, DENSE, DENSE0, QUAT, EXPR = range(5)


def _shared(p, j):
    return np.tile(TO.api._cost_weight_row(p._cost_objs[j]), (p.B, 1))


def test_row_lengths_and_layout():
    p = _NoDevice()
    n, m = 4, 2
    assert _shared(p, DIAG).shape == (4, n + m + 1)
    assert np.array_equal(_shared(p, DIAG)[0], [1, 2, 3, 4, 0.1, 0.2, 0.5])           # Qd | Rd | c
    assert _shared(p, DENSE).shape == (4, n * n + m * m + m * n + 1)
    row = _shared(p, DENSE)[0]
    c = p._cost_objs[DENSE]
    assert np.array_equal(row[:16], c.Q.ravel(order="F")) and np.array_equal(row[20:28], c.H.ravel(order="F")) and row[-1] == 1.0
    assert _shared(p, QUAT).shape == (4, n + m + 2) and _shared(p, QUAT)[0, -1] == 3.0   # ... | c | w
    with pytest.raises(TO.ArgumentError):
        TO.api._cost_weight_row(p._cost_objs[EXPR])


def test_wrong_shape_or_count():
    p = _NoDevice()
    for j in (DIAG, DENSE, QUAT):
        good = _shared(p, j)
        for shape in [(4, good.shape[1] + 1), (3, good.shape[1]), (5, good.shape[1]), (good.shape[1],), (4, good.shape[1], 1)]:
            with pytest.raises(TO.DimensionMismatch):
                TO.set_cost_weights(p, j, np.ones(shape))
    with pytest.raises(TO.DimensionMismatch):       # a sequence of costs one short
        TO.set_cost_weights(p, DIAG, [p._cost_objs[DIAG]] * 3)
    with pytest.raises(TO.DimensionMismatch):       # a cost of other dimensions
        TO.set_cost_weights(p, DIAG, [TO.DiagonalCost(np.ones(3), np.ones(2))] * 4)


def test_kind_and_index_errors():
    p = _NoDevice()
    with pytest.raises(TO.ArgumentError):           # program costs keep their constants shared
        TO.set_cost_weights(p, EXPR, np.zeros((4, 0)))
    with pytest.raises(TO.ArgumentError):
        TO.set_cost_weights(p, 9, _shared(p, DIAG))
    with pytest.raises(TO.ArgumentError):
        TO.set_cost_weights(p, TO.DiagonalCost(np.ones(4), np.ones(2)), _shared(p, DIAG))   # not one of the problem's
    with pytest.raises(TO.ArgumentError):
        TO.set_cost_weights(_NoDevice(hybrid=True), DIAG, _shared(p, DIAG))
    with pytest.raises(TO.ArgumentError):           # another type
        TO.set_cost_weights(p, DIAG, [TO.QuadraticCost(np.eye(4), np.eye(2))] * 4)
    with pytest.raises(TO.ArgumentError):           # another terminal flag
        TO.set_cost_weights(p, DENSE0, [TO.QuadraticCost(np.eye(4), np.eye(2))] * 4)
    with pytest.raises(TO.ArgumentError):           # another q_ind
        TO.set_cost_weights(p, QUAT, [TO.DiagonalQuatCost(np.ones(4), np.ones(2), w=3.0, q_ind=(4, 3, 2, 1))] * 4)


def test_h_zero_rule():
    p = _NoDevice()
    r = _shared(p, DENSE0); r[2, 16 + 4 + 3] = 0.5   # H[3] of a cost whose shared H is zero
    with pytest.raises(TO.ArgumentError, match="instance 2, entry 23"):
        TO.set_cost_weights(p, DENSE0, r)
    with pytest.raises(TO.ArgumentError, match="H-zero"):
        TO.set_cost_weights(p, DENSE0, [TO.QuadraticCost(np.eye(4), np.eye(2), H=np.ones((2, 4)), terminal=True)] * 4)
    with pytest.raises(TO.ArgumentError, match="H-zero"):
        TO.set_cost_weights(p, DENSE, [TO.QuadraticCost(np.eye(4), np.eye(2))] * 4)


def test_non_finite_entries():
    p = _NoDevice()
    for j, e in ((DIAG, 5), (DENSE, 17), (QUAT, 7)):
        r = _shared(p, j); r[1, e] = np.inf if e % 2 else np.nan
        with pytest.raises(TO.ArgumentError, match=f"instance 1, entry {e}"):
            TO.set_cost_weights(p, j, r)


def test_indefinite_weights_are_accepted():
    """the reference only warns about indefinite Q or R: such rows pass every host check"""
    p = _NoDevice()
    r = _shared(p, DIAG); r[:, 0] = -1.0; r[:, 4] = 0.0
    j, cost, out, lin = TO.api._cost_weight_rows(p, DIAG, r)
    assert j == DIAG and lin is None and np.array_equal(out, r)


def test_cost_objects_become_rows_and_linear_terms():
    p = _NoDevice()
    costs = [TO.DiagonalCost(np.arange(1.0, 5.0) * (1 + b), [0.1, 0.2 * (1 + b)], q=np.full(4, b), r=[b, -b], c=0.1 * b) for b in range(4)]
    j, cost, rows, (q, r) = TO.api._cost_weight_rows(p, p._cost_objs[DIAG], costs)
    assert j == DIAG and cost is p._cost_objs[DIAG]
    assert rows.shape == (4, 7) and rows.flags["C_CONTIGUOUS"] and rows.dtype == np.float64
    assert np.array_equal(rows, np.array([np.concatenate([np.diagonal(c.Q), np.diagonal(c.R), [c.c]]) for c in costs]))
    assert np.array_equal(q, np.array([c.q for c in costs])) and np.array_equal(r, np.array([c.r for c in costs]))
    quats = [TO.DiagonalQuatCost(np.ones(4), np.ones(2), w=1.0 + b, q_ind=(1, 2, 3, 4)) for b in range(4)]
    _, _, rows, _ = TO.api._cost_weight_rows(p, QUAT, quats)
    assert np.array_equal(rows[:, -1], [1.0, 2.0, 3.0, 4.0])


def test_new_entry_points_are_declared():
    names = ("to_cost_weights_len", "to_set_cost_weights", "to_get_cost_weights")
    header = open(os.path.join(ROOT, "include", "trajopt_b200.h")).read()
    shim = open(os.path.join(ROOT, "trajectoryoptimization.jl_b200", "julia", "B200TrajOpt.jl")).read()
    for name in names:
        assert name in TO._capi.EXPORTED_SYMBOLS
        assert re.search(rf"\bint {name}\(", header), name
        assert f"(:{name}, libb200)" in shim, name
    assert callable(TO.set_cost_weights) and callable(TO.cost_weights)
