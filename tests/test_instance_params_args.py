"""Argument checks of the per-instance model-parameter calls that happen on the host, before any device call (no GPU needed)."""

import numpy as np
import pytest

import trajopt_b200 as TO


class _NoDevice:
    """stands in for a Problem: any device call is an error, so a test passes only when the check comes first"""

    def __init__(self, model, B=4, hybrid=False):
        self.model, self.B, self.hybrid = model, B, hybrid
        self.n, self.m = model.dims() if not hybrid else (4, 2)

    def _call(self, name, *args):
        raise AssertionError(f"device call {name} reached")

    def _raw_call(self, name, *args):
        raise AssertionError(f"device call {name} reached")

    def _ensure_current(self):
        raise AssertionError("device call reached")


@pytest.mark.parametrize("model, count", [(TO.DoubleIntegrator(), 1), (TO.DoubleIntegrator(2), 1), (TO.Cartpole(), 4),
                                          (TO.Quadrotor(), 10), (TO.Acrobot(), 8)])
def test_wrong_shape_or_count(model, count):
    p = _NoDevice(model)
    for shape in [(4, count + 1), (4, count - 1), (3, count), (5, count), (count,), (4, count, 1)]:
        if shape[-1] < 1:
            continue
        with pytest.raises(TO.DimensionMismatch):
            TO.set_model_params(p, np.ones(shape))


def test_wrong_number_of_models():
    p = _NoDevice(TO.Quadrotor())
    with pytest.raises(TO.DimensionMismatch):
        TO.set_model_params(p, [TO.Quadrotor(mass=0.5 + 0.1 * b) for b in range(3)])
    with pytest.raises(TO.DimensionMismatch):
        TO.set_model_params(p, [TO.Quadrotor() for _ in range(5)])


def test_wrong_model_class():
    p = _NoDevice(TO.Quadrotor())
    with pytest.raises(TO.ArgumentError):
        TO.set_model_params(p, [TO.Quadrotor(), TO.Quadrotor(), TO.Cartpole(), TO.Quadrotor()])
    # a DoubleIntegrator of another dimension is another model
    p = _NoDevice(TO.DoubleIntegrator(2))
    with pytest.raises(TO.ArgumentError):
        TO.set_model_params(p, [TO.DoubleIntegrator(2), TO.DoubleIntegrator(1), TO.DoubleIntegrator(2), TO.DoubleIntegrator(2)])


def test_hybrid_problem_refused_before_device():
    p = _NoDevice(TO.Cartpole(), hybrid=True)
    with pytest.raises(TO.ArgumentError):
        TO.set_model_params(p, np.ones((4, 4)))
    with pytest.raises(TO.ArgumentError):
        TO.model_params(p)


def test_models_become_rows():
    """a sequence of models is the matrix of their .params: the rows the device call would take"""
    models = [TO.Quadrotor(mass=0.5 + 0.05 * b, J=(0.002 + 1e-4 * b, 0.0023, 0.004), km=0.02 + 0.001 * b) for b in range(4)]
    rows = TO.api._model_param_rows(_NoDevice(TO.Quadrotor()), models)
    assert rows.shape == (4, 10) and rows.flags["C_CONTIGUOUS"] and rows.dtype == np.float64
    assert np.array_equal(rows, np.array([m.params for m in models]))


def test_new_entry_points_are_declared():
    for name in ("to_set_model_params", "to_get_model_params"):
        assert name in TO._capi.EXPORTED_SYMBOLS
    assert callable(TO.set_model_params) and callable(TO.model_params)
