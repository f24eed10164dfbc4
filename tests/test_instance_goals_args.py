"""Argument checks of the per-instance goal calls that happen on the host, before any device call (no GPU needed)."""

import numpy as np
import pytest

import trajopt_b200 as TO


class _NoDevice:
    """stands in for a Problem: any device call is an error, so a test passes only when the check comes first"""

    def __init__(self, B=4, n=4, m=1, N=21, ncost=2):
        self.B, self.n, self.m, self.N = B, n, m, N
        self._cost_objs = [object()] * ncost
        self.obj = [TO.LQRCost(np.eye(n), np.eye(m), np.zeros(n))] * N
        self.constraints = []

    def _call(self, name, *args):
        raise AssertionError(f"device call {name} reached")

    def _ensure_current(self):
        raise AssertionError("device call reached")


def test_set_goal_state_per_instance_shape():
    with pytest.raises(TO.DimensionMismatch):
        TO.set_goal_state(_NoDevice(), np.zeros((3, 4)))
    with pytest.raises(TO.DimensionMismatch):
        TO.set_goal_state(_NoDevice(), np.zeros((4, 5)))


def test_update_trajectory_per_instance_shapes():
    p = _NoDevice()
    with pytest.raises(TO.DimensionMismatch):
        TO.update_trajectory(p, np.zeros((4, 30, 4)), np.zeros((4, 30, 2)))          # m
    with pytest.raises(TO.DimensionMismatch):
        TO.update_trajectory(p, np.zeros((3, 30, 4)), np.zeros((3, 30, 1)))          # B
    with pytest.raises(TO.DimensionMismatch):
        TO.update_trajectory(p, np.zeros((4, 30, 4)), np.zeros((4, 29, 1)))          # nref
    with pytest.raises(TO.DimensionMismatch):
        TO.update_trajectory(p, np.zeros((4, 10, 4)), np.zeros((4, 10, 1)), 1)       # shorter than start + N - 1
    with pytest.raises(TO.DimensionMismatch):
        TO.update_trajectory(p, np.zeros((4, 30, 4)), np.zeros((4, 30, 1)), 11)


def test_set_cost_terms_shapes():
    p = _NoDevice()
    with pytest.raises(TO.DimensionMismatch):
        TO.set_cost_terms(p, np.zeros((4, 1, 4)), np.zeros((4, 2, 1)))
    with pytest.raises(TO.DimensionMismatch):
        TO.set_cost_terms(p, np.zeros((4, 2, 4)), np.zeros((4, 2, 2)))


def test_new_entry_points_are_declared():
    for name in ("to_set_goal_states", "to_update_trajectories", "to_get_cost_terms", "to_set_cost_terms", "to_get_goal_values",
                 "to_set_goal_values"):
        assert name in TO._capi.EXPORTED_SYMBOLS
