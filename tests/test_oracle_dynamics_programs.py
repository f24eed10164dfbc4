"""CPU tests of user dynamics models (AutodiffDynamics, recorded programs) on the oracle: its interpreter (oracle/models.hpp expr_dynamics)
against a NumPy evaluation and central differences for every op code, recorded copies of the built-in models against the built-in
models, Problem(model, ...) against the model vector [model] * (N - 1), the recording limits, and the instruction checks of orc_create."""
import ctypes as C

import numpy as np
import pytest

import trajopt_b200 as TO
from dynamics_programs import (BUILTINS, OP_PROGRAMS, builtin_problem, limit_function, malformed_specs, model_ops, numpy_jacobian,
                               numpy_step, one_step_problem, op_model, pad, padded_closed_form, recorded_builtin)
from oracle_binding import OracleProblem, load_oracle

K = TO.capi
H = 0.1


def rel_err(a, b):
    a, b = np.asarray(a, dtype=float), np.asarray(b, dtype=float)
    return float(np.max(np.abs(a - b) / np.maximum(1.0, np.abs(b)), initial=0.0))


def test_the_programs_record_every_op_code():
    ops = set().union(*(model_ops(op_model(name)) for name in OP_PROGRAMS))
    assert ops == set(range(20)), f"op codes not recorded: {sorted(set(range(20)) - ops)}"
    powc = op_model("powers")
    exps = {float(powc.consts[b]) for op, a, b in np.asarray(powc.prog).reshape(-1, 3) if op == K.OP_POWC}
    assert exps == {1.5, 0.5, 3.0, -1.0, -2.5}
    lim = op_model("limit")
    assert len(lim.prog) == K.EXPR_MAXLEN and len(lim.consts) == K.EXPR_MAXCONST


def draw(model, B, seed):
    r = np.random.default_rng(seed)
    x = r.uniform(-1.0, 1.0, (B, model.n))
    u = r.uniform(-1.0, 1.0, (B, model.m))
    if model.fun is OP_PROGRAMS["transcendental"][2]:
        x[:, 0] = np.linspace(-1.0, 1.0, B)      # tanh(4 x0) over [-4, 4]: 1 - tanh^2 from ~1e-3 to 1
    return x, u


def oracle_step(model, x, u):
    """(x+ [B, n_out], padded [A B] [B, 4, 6]) of the oracle for the states x and controls u of B instances"""
    B = x.shape[0]
    p = one_step_problem(OracleProblem, model, B, h=H)
    TO.set_initial_state(p, pad(x, 4))
    TO.initial_controls(p, pad(u, 2)[:, None, :])
    TO.rollout(p); TO.expand(p)
    X, AB = TO.states(p), TO.dynamics_jacobians(p)
    return X[:, 1], AB[:, 0]


@pytest.mark.parametrize("discrete", [False, True], ids=["rk4", "jump_map"])
@pytest.mark.parametrize("name", sorted(OP_PROGRAMS) + ["limit"])
def test_oracle_interpreter_against_numpy_and_central_differences(name, discrete):
    model = op_model(name, discrete)
    B = 24
    x, u = draw(model, B, seed=3)
    Xn, AB = oracle_step(model, x, u)
    n, m = model.n, model.m
    ref = np.stack([numpy_step(model, x[b], u[b], H) for b in range(B)])
    assert rel_err(Xn[:, :n], ref) < 1e-13
    assert np.all(Xn[:, n:] == 0.0)                       # padded state slots: x+ = x + 0 (RK4) or 0 (jump map), and x = 0
    fd = np.stack([numpy_jacobian(model, x[b], u[b], H) for b in range(B)])
    got = np.concatenate([AB[:, :n, :n], AB[:, :n, 4:4 + m]], axis=-1)
    assert np.allclose(got, fd, rtol=1e-6, atol=1e-7), f"max |[A B] - central differences| {np.abs(got - fd).max():.2e}"
    closed, mask = padded_closed_form(model)
    assert np.array_equal(AB[:, mask], np.broadcast_to(closed[mask], (B, int(mask.sum()))))


@pytest.mark.parametrize("name", BUILTINS)
def test_recorded_copies_of_the_builtin_models(name):
    """a program written from a built-in model's formulas: rollout, [A B] and AL-iLQR iterates equal the built-in model's"""
    rec_model, builtin = recorded_builtin(name)
    n, m = builtin.dims()
    ref = builtin_problem(name, OracleProblem, 3, recorded=False)
    rec = builtin_problem(name, OracleProblem, 3, recorded=True)
    r = np.random.default_rng(2)
    U = TO.controls(ref) + 0.3 * r.standard_normal(TO.controls(ref).shape)
    TO.initial_controls(ref, U); TO.initial_controls(rec, pad(U, 2))
    for p in (ref, rec):
        TO.rollout(p); TO.expand(p)
    Xr, Xp = TO.states(ref), TO.states(rec)
    assert rel_err(Xp[..., :n], Xr) < 1e-13 and np.all(Xp[..., n:] == 0.0)
    ABr, ABp = TO.dynamics_jacobians(ref), TO.dynamics_jacobians(rec)
    assert rel_err(np.concatenate([ABp[..., :n, :n], ABp[..., :n, 4:4 + m]], axis=-1), ABr) < 1e-12
    closed, mask = padded_closed_form(rec_model)
    assert np.array_equal(ABp[..., mask], np.broadcast_to(closed[mask], ABp.shape[:2] + (int(mask.sum()),)))
    assert abs(TO.cost(rec) - TO.cost(ref)).max() <= 1e-12 * np.abs(TO.cost(ref)).max()
    for p in (ref, rec):
        TO.ilqr_step(p, 4); TO.al_update(p); TO.ilqr_step(p, 2)
    assert np.allclose(TO.merit(rec), TO.merit(ref), rtol=1e-7)
    assert rel_err(TO.controls(rec)[..., :m], TO.controls(ref)) < 1e-7 and np.all(TO.controls(rec)[..., m:] == 0.0)
    assert rel_err(TO.states(rec)[..., :n], TO.states(ref)) < 1e-7


def test_single_model_is_the_model_vector():
    """Problem(model, ...) is Problem([model] * (N - 1), ...): padded (4, 2) layout, bit-identical results"""
    N, B = 21, 3
    rec, _ = recorded_builtin("cartpole")
    ref = builtin_problem("cartpole", OracleProblem, B, recorded=False, N=N)

    def build(model):
        p = OracleProblem(model, ref.obj, ref.x0, 5.0, xf=ref.xf, constraints=ref.constraints)
        TO.initial_controls(p, pad(TO.controls(ref), 2))
        return p
    a, b = build(rec), build([rec] * (N - 1))
    assert a.hybrid and (a.n, a.m) == (4, 2) and a.nx == b.nx == [4] * N and a.nu == b.nu == [1] * N
    for p in (a, b):
        TO.rollout(p); TO.expand(p); TO.backward(p)
    for f in (TO.states, TO.controls, TO.dynamics_jacobians):
        assert np.array_equal(f(a), f(b))
    for ga, gb in zip(TO.gains(a), TO.gains(b)):
        assert np.array_equal(ga, gb)
    for p in (a, b):
        TO.ilqr_step(p, 3); TO.al_update(p); TO.ilqr_step(p, 2)
    assert np.array_equal(TO.states(a), TO.states(b)) and np.array_equal(TO.controls(a), TO.controls(b))


def test_single_model_of_fewer_states_and_controls():
    """a 2-state pendulum on its own: the padded state slots and the padded control stay exactly zero through the solver"""
    pend = TO.AutodiffDynamics(2, 1, lambda x, u: [x[1], -9.81 * TO.sin(x[0]) - 0.1 * x[1] + u[0]])
    N = 31
    obj = TO.LQRObjective(np.full(2, 0.1), np.full(1, 0.01), np.full(2, 100.0), np.array([np.pi, 0.0]), N)
    cons = TO.ConstraintList(2, 1, N)
    TO.add_constraint(cons, TO.BoundConstraint(2, 1, u_min=-6.0, u_max=6.0), (1, N - 1))
    p = OracleProblem(pend, obj, np.zeros((2, 2)), 3.0, xf=np.array([np.pi, 0.0]), constraints=cons)
    assert TO.dims(p)[:2] == ([2] * N, [1] * N)
    TO.initial_controls(p, pad(np.full((2, N - 1, 1), 0.5), 2)); TO.rollout(p)
    J0 = TO.merit(p)
    for _ in range(3):
        TO.ilqr_step(p, 5); TO.al_update(p)
    assert np.all(TO.merit(p) < J0)
    assert np.all(TO.states(p)[..., 2:] == 0.0) and np.all(TO.controls(p)[..., 1:] == 0.0)
    with pytest.raises(TO.ArgumentError, match="at most 4 states and 2 controls"):
        OracleProblem(TO.AutodiffDynamics(5, 1, lambda x, u: [x[1], x[2], x[3], x[4], u[0]]),
                      TO.LQRObjective(np.ones(5), np.ones(1), np.ones(5), np.zeros(5), 3), np.zeros(5), 1.0)
    with pytest.raises(TO.ArgumentError, match="at most 4 states and 2 controls"):
        OracleProblem(TO.AutodiffDynamics(2, 3, lambda x, u: [x[1], u[0] + u[1] + u[2]]),
                      TO.LQRObjective(np.ones(2), np.ones(3), np.ones(2), np.zeros(2), 3), np.zeros(2), 1.0)


def test_recording_limits():
    TO.AutodiffDynamics(4, 2, limit_function(128, 64))
    with pytest.raises(TO.ArgumentError, match="recorded dynamics model exceeds 128 instructions"):
        TO.AutodiffDynamics(4, 2, limit_function(129, 64))         # one more: the last output copy does not fit
    TO.AutodiffDynamics(4, 2, limit_function(128, 63))
    with pytest.raises(TO.ArgumentError, match="recorded dynamics model exceeds 64 constants"):
        TO.AutodiffDynamics(4, 2, limit_function(128, 65))
    with pytest.raises(TO.ArgumentError, match="Expr"):
        TO.AutodiffDynamics(2, 1, lambda x, u: [x[1], x[0] ** u[0]])
    with pytest.raises(TO.ArgumentError, match="recorded dynamics model cannot branch"):
        TO.AutodiffDynamics(2, 1, lambda x, u: [x[1], u[0] if x[0] else -u[0]])
    with pytest.raises(TO.ArgumentError, match="recorded cost exceeds 128 instructions"):
        TO.AutodiffCost(2, 1, lambda x, u: sum(x[0] * (1.0 + 0.0 * i) for i in range(100)))
    with pytest.raises(TO.ArgumentError, match="recorded constraint exceeds 128 instructions"):
        TO.AutodiffConstraint(2, 1, lambda x: [sum(x[0] * x[1] for i in range(100))], TO.Inequality(), "state")


@pytest.mark.parametrize("case", range(len(malformed_specs())))
def test_oracle_rejects_malformed_programs_like_the_library(case):
    """orc_create runs to_create's program checks: the same error code and message for every malformed spec"""
    name, spec, code, msg = malformed_specs()[case]
    lib = load_oracle()
    h = C.c_void_p()
    rc = lib.orc_create(C.byref(spec.c), C.byref(h))
    assert rc == code and not h, f"{name}: rc {rc}"
    assert msg in lib.orc_last_error(None).decode(), f"{name}: {lib.orc_last_error(None).decode()}"


def test_oracle_accepts_the_valid_spec_behind_the_malformed_ones():
    name, spec, _, _ = malformed_specs()[0]
    good = K.Spec(K.MODEL_EXPR, 4, 2, spec.N, spec.B, spec.dt, spec.costs, spec.cost_index, spec.cons, dyn=[op_model("transcendental")._spec()],
                  dyn_index=[0] * (spec.N - 1), nx=[4] * spec.N, nu=[2] * spec.N)
    lib = load_oracle()
    h = C.c_void_p()
    assert lib.orc_create(C.byref(good.c), C.byref(h)) == K.TO_OK and h
    lib.orc_destroy(h)
