"""Closed-loop MPC on the device (to_mpc_setup / to_mpc_run / to_mpc_history).

Central property: a device run computes, bit for bit, what the host-scripted loop of existing entry points computes -- per step
update_trajectory (per instance), rollout, ilqr_step, controls / merit, the plant step taken by a second Problem with N = 2 holding the
plant's parameters and knot-0 time steps (through rollout), then shift_trajectory(1) and set_initial_state.  Two identical problems are
built for each case: one runs the device loop, the other the scripted loop."""
import numpy as np
import pytest

import trajopt_b200 as TO
from trajopt_b200 import problems
from dynamics_programs import recorded_builtin

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(TO.Problem.__name__ == "OracleProblem", reason="closed-loop MPC has no oracle counterpart")]


def _cartpole(B=64, N=21):
    return problems.cartpole(B=B, N=N, u_bound=4.0, goal=True)


def _double_integrator(B=64, N=21):
    return problems.double_integrator(B=B, N=N, dim=2)


def _quadrotor(B=64, N=31):
    return problems.quadrotor(B=B, N=N, error_state=True, u_noise=0.01)


def _autodiff(B=32, N=21):
    rec, _ = recorded_builtin("cartpole")
    obj = TO.LQRObjective(1e-2 * np.eye(4), 1e-1 * np.eye(1), 100.0 * np.eye(4), np.array([0, np.pi, 0, 0.0]), N)
    x0 = np.zeros((B, 4)); x0[:, :2] += 0.1 * np.random.default_rng(2).standard_normal((B, 2))
    p = TO.Problem(rec, obj, x0, 2.0)
    TO.initial_controls(p, np.full((B, N - 1, 2), 0.01) * np.array([1.0, 0.0]))
    return p


def _reference(p, nref, seed=5):
    """a smooth per-instance reference Xref[B, nref, n], Uref[B, nref, m] around each instance's start (identity attitude kept unit)"""
    r = np.random.default_rng(seed)
    t = np.arange(nref)[None, :, None]
    Xref = p.x0[:, None, :] + 0.05 * np.sin(0.2 * t + r.uniform(0, 6, (p.B, 1, p.n)))
    if p.n == 13:
        Xref[:, :, 3:7] = np.array([1.0, 0, 0, 0])
        Xref[:, :, 7:] *= 0.0
    Uref = 0.1 * np.cos(0.3 * t + r.uniform(0, 6, (p.B, 1, p.m)))
    if p.n == 13:
        Uref = Uref + TO.Quadrotor().hover_control()
    return Xref, Uref


def _plant(p, params=None, dt=None):
    """the scripted loop's plant: a Problem with N = 2 stepping the model once over knot 0's step, with the plant's parameters"""
    model = p.model[0] if p.hybrid else p.model        # one recorded model: the plant problem pads it as the planner does
    n, m = model.n, model.m
    obj = TO.LQRObjective(np.eye(n), np.eye(m), np.eye(n), np.zeros(n), 2)
    q = TO.Problem(model, obj, p.x0[:, :n], float(p.spec.dt[0]), integration=TO.integration(p), error_state=p.error_state)
    if params is not None:
        TO.set_model_params(q, params)
    if dt is not None:
        TO.set_time_steps(q, dt[:, :1])
    return q


def _scripted(p, plant, steps, iters, ref=None, start=1, W=None, j0=0):
    X, U, J = [p.x0.copy()], [], []
    for s in range(steps):
        j = j0 + s
        if ref is not None:
            TO.update_trajectory(p, ref[0], ref[1], start + j)
        TO.rollout(p)
        TO.ilqr_step(p, iters)
        u = TO.controls(p)[:, 0].copy()
        J.append(TO.merit(p).copy())
        TO.set_initial_state(plant, p.x0)
        TO.initial_controls(plant, u[:, None, :])
        TO.rollout(plant)
        xn = TO.states(plant)[:, 1].copy()
        if W is not None:
            xn = xn + W[:, j]
        TO.shift_trajectory(p, 1)
        TO.set_initial_state(p, xn)
        X.append(xn); U.append(u)
    return np.stack(X, 1), np.stack(U, 1), np.stack(J, 1)


def _state(p):
    """everything a step leaves behind that the tests compare"""
    out = {"X": TO.states(p), "U": TO.controls(p), "t": TO.instance_times(p), "x0": TO.states(p)[:, 0]}
    if not p.hybrid:
        out["q"], out["r"] = TO.cost_terms(p)
    for i in range(len(p.constraints)):
        out[f"lambda{i}"] = TO.multipliers(p, i)
    return out


def _equal(a, b, what):
    for k in a:
        assert np.array_equal(a[k], b[k]), f"{what}: {k} differs (max |d| = {np.nanmax(np.abs(a[k] - b[k])):.3e})"


CASES = {
    # name: (factory, reference, per-instance plant params / dt / weights, iterations)
    "cartpole_ref": (_cartpole, True, False, 2),
    "cartpole_noref": (_cartpole, False, False, 1),
    "double_integrator_ref": (_double_integrator, True, False, 2),
    "quadrotor_record_inst": (_quadrotor, True, True, 2),
    "autodiff_dynamics": (_autodiff, False, False, 1),
}


def _setup_case(name):
    factory, ref, inst, iters = CASES[name]
    dev, scr = factory(), factory()
    steps = 5
    B = dev.B
    r = np.random.default_rng(11)
    kw, plant_rows, dtb = {}, None, None
    if ref:
        nref = dev.N + steps + 3
        kw["Xref"], kw["Uref"] = _reference(dev, nref)
        kw["start"] = 2
    if inst:
        base = np.asarray(dev.model.params, dtype=float)
        plant_rows = base[None, :] * (1.0 + 0.05 * r.uniform(-1, 1, (B, base.size)))
        kw["plant_params"] = plant_rows
        dtb = np.tile(dev.spec.dt, (B, 1)) * (1.0 + 0.1 * (np.arange(B) % 3))[:, None]
        nc = len(dev._cost_objs)
        for p in (dev, scr):
            TO.set_time_steps(p, dtb)
            TO.set_model_params(p, base[None, :] * (1.0 + 0.02 * (np.arange(B) % 4))[:, None])
            for c in range(nc):
                row = TO.cost_weights(p, c)
                TO.set_cost_weights(p, c, row * (1.0 + 0.25 * (np.arange(B) % 5))[:, None])
    return dev, scr, steps, iters, kw, plant_rows, dtb


@pytest.mark.parametrize("name", sorted(CASES))
def test_device_loop_is_the_scripted_loop(name):
    dev, scr, steps, iters, kw, plant_rows, dtb = _setup_case(name)
    TO.mpc_setup(dev, steps, **kw)
    plant = _plant(scr, plant_rows if plant_rows is not None else (TO.model_params(scr) if dtb is not None else None), dtb)
    l0 = dev._lib.to_launch_count(dev._h), scr._lib.to_launch_count(scr._h)
    TO.mpc_run(dev, steps, iters)
    X, U, J = TO.mpc_history(dev)
    ref = (kw["Xref"], kw["Uref"]) if "Xref" in kw else None
    Xs, Us, Js = _scripted(scr, plant, steps, iters, ref, kw.get("start", 1))
    dl, sl = dev._lib.to_launch_count(dev._h) - l0[0], scr._lib.to_launch_count(scr._h) - l0[1]
    assert np.array_equal(X, Xs), f"{name}: Xcl (max |d| = {np.max(np.abs(X - Xs)):.3e})"
    assert np.array_equal(U, Us), f"{name}: Ucl"
    assert np.array_equal(J, Js), f"{name}: J"
    _equal(_state(dev), _state(scr), name)
    # per step the scripted loop's controls (gather) and shift are replaced by the advance kernel, and a reference adds the window kernel
    assert dl == sl - steps + (steps if ref is not None else 0), (dl, sl)
    assert not np.array_equal(X[:, 0], X[:, -1])
    for p in (dev, scr, plant):
        p.close()


PLANT_MODELS = {"cartpole": TO.Cartpole, "acrobot": TO.Acrobot, "double_integrator_1": lambda: TO.DoubleIntegrator(1),
                "double_integrator_2": lambda: TO.DoubleIntegrator(2), "quadrotor": TO.Quadrotor}


@pytest.mark.parametrize("inst", [False, True])
@pytest.mark.parametrize("rule", ["Euler", "RK2", "RK3", "RK4"])
@pytest.mark.parametrize("name", sorted(PLANT_MODELS))
def test_plant_step_is_k_rollout(name, rule, inst):
    """the advance kernel's plant step against k_rollout on a problem with N = 2 holding the plant's parameters, bit for bit: every
    built-in model, every rule, with the shared parameters (the parameter bank) and with per-instance plant rows (staged in shared memory)"""
    model = PLANT_MODELS[name]()
    n, m = model.dims()
    B, N = 8, 6
    r = np.random.default_rng(21)
    x0 = 0.3 * r.standard_normal((B, n))
    U0 = 0.5 * r.standard_normal((B, N - 1, m))
    if name == "quadrotor":
        x0[:, 3:7] = np.array([1.0, 0, 0, 0]) + 0.2 * r.standard_normal((B, 4))
        x0[:, 3:7] /= np.linalg.norm(x0[:, 3:7], axis=1, keepdims=True)
        U0 = model.hover_control() + 0.1 * r.standard_normal((B, N - 1, m))
    obj = TO.LQRObjective(np.eye(n), 0.1 * np.eye(m), np.eye(n), np.zeros(n), N)
    p = TO.Problem(model, obj, x0, 1.0, integration=rule)
    TO.initial_controls(p, U0)
    base = np.asarray(model.params, dtype=float)
    rows = base[None, :] * (1.0 + 0.05 * r.uniform(-1, 1, (B, base.size))) if inst else None
    TO.mpc_setup(p, 2, plant_params=rows)
    TO.mpc_run(p, 2, 1)
    X, U, _ = TO.mpc_history(p)
    plant = TO.Problem(model, TO.LQRObjective(np.eye(n), np.eye(m), np.eye(n), np.zeros(n), 2), x0, float(p.spec.dt[0]), integration=rule)
    if inst:
        TO.set_model_params(plant, rows)
    for j in range(2):
        TO.set_initial_state(plant, X[:, j]); TO.initial_controls(plant, U[:, j][:, None, :]); TO.rollout(plant)
        xk = TO.states(plant)[:, 1]
        assert np.array_equal(xk, X[:, j + 1]), f"step {j}: max |d| = {np.max(np.abs(xk - X[:, j + 1])):.3e}"
    p.close(); plant.close()


def test_vector_disturbances_are_added():
    dev, scr = _double_integrator(), _double_integrator()
    steps = 6
    W = 0.01 * np.random.default_rng(3).standard_normal((dev.B, steps, dev.ne))
    Xref, Uref = _reference(dev, dev.N + steps)
    TO.mpc_setup(dev, steps, disturbances=W, Xref=Xref, Uref=Uref)
    TO.mpc_run(dev, steps, 2)
    X, U, J = TO.mpc_history(dev)
    plant = _plant(scr)
    Xs, Us, Js = _scripted(scr, plant, steps, 2, (Xref, Uref), 1, W=W)
    assert np.array_equal(X, Xs) and np.array_equal(U, Us) and np.array_equal(J, Js)
    _equal(_state(dev), _state(scr), "disturbed double integrator")
    for p in (dev, scr, plant):
        p.close()


def test_quadrotor_disturbance_is_the_inverse_of_state_diff():
    dev = _quadrotor()
    steps = 4
    W = 0.02 * np.random.default_rng(4).standard_normal((dev.B, steps, dev.ne))
    TO.mpc_setup(dev, steps, disturbances=W)
    TO.mpc_run(dev, steps, 1)
    X, U, J = TO.mpc_history(dev)
    plant = _plant(dev)
    for j in range(steps):
        TO.set_initial_state(plant, X[:, j]); TO.initial_controls(plant, U[:, j][:, None, :]); TO.rollout(plant)
        x = TO.states(plant)[:, 1]
        dx = TO.state_diff(plant, np.stack([X[:, j], X[:, j + 1]], 1))[:, 1]
        assert np.max(np.abs(dx - W[:, j])) <= 1e-13 * np.max(np.abs(W[:, j])), f"step {j}: state_diff(x (+) w, x) != w"
        ratio = np.linalg.norm(X[:, j + 1, 3:7], axis=1) / np.linalg.norm(x[:, 3:7], axis=1)
        assert np.max(np.abs(ratio - 1.0)) <= 1e-14, f"step {j}: the Cayley composition changed the quaternion's norm"
    dev.close(); plant.close()


def test_chunked_runs_equal_one_run():
    a, b = _quadrotor(), _quadrotor()
    Xref, Uref = _reference(a, a.N + 8)
    for p in (a, b):
        TO.mpc_setup(p, 7, Xref=Xref, Uref=Uref)
    TO.mpc_run(a, 3, 2); TO.mpc_run(a, 4, 2)
    TO.mpc_run(b, 7, 2)
    for x, y in zip(TO.mpc_history(a), TO.mpc_history(b)):
        assert x.shape == y.shape and np.array_equal(x, y)
    _equal(_state(a), _state(b), "3 + 4 steps against 7")
    with pytest.raises(TO.DimensionMismatch):
        TO.mpc_run(a, 1)
    a.close(); b.close()


def test_run_is_asynchronous():
    import torch
    ref, dev = _double_integrator(), _double_integrator()
    for p in (ref, dev):
        TO.mpc_setup(p, 3)
    TO.mpc_run(ref, 3, 2)
    expected = TO.mpc_history(ref)
    with torch.cuda.stream(torch.cuda.Stream()):
        stream = torch.cuda.current_stream()
        dev._call("to_set_stream", stream.cuda_stream)
        torch.cuda._sleep(1_000_000_000)     # about half a second of GPU time ahead of the run on the same stream
        TO.mpc_run(dev, 3, 2)
        pending = not stream.query()
        stream.synchronize()
    assert pending, "to_mpc_run waited for the device"
    for x, y in zip(TO.mpc_history(dev), expected):
        assert np.array_equal(x, y)
    ref.close(); dev.close()


def test_plant_step_against_the_oracle():
    from oracle_binding import oracle_discrete_dynamics
    dev = _quadrotor(B=16)
    plant_model = TO.Quadrotor(mass=0.55, J=(0.0025, 0.0021, 0.0043), km=0.026)
    rows = np.tile(np.asarray(plant_model.params, dtype=float), (dev.B, 1))
    TO.mpc_setup(dev, 3, plant_params=rows)
    TO.mpc_run(dev, 3, 1)
    X, U, _ = TO.mpc_history(dev)
    h = float(dev.spec.dt[0])
    for j in range(3):
        for b in range(dev.B):
            xo = oracle_discrete_dynamics(plant_model, X[b, j], U[b, j], h)
            assert np.max(np.abs(X[b, j + 1] - xo) / np.maximum(1.0, np.abs(xo))) <= 1e-12, (j, b)
    dev.close()


def test_setup_refusals_leave_the_previous_setup():
    p = _cartpole(B=8)
    TO.mpc_setup(p, 2)
    TO.mpc_run(p, 1)
    with pytest.raises(TO.DimensionMismatch):
        TO.mpc_setup(p, 3, Xref=np.zeros((8, p.N, 4)), Uref=np.zeros((8, p.N, 1)))      # 1 - 1 + 2 + N > N
    bad = np.tile(np.asarray(p.model.params, dtype=float), (8, 1)); bad[3, 0] = -1.0
    with pytest.raises(TO.ArgumentError, match="instance 3"):
        p._call("to_mpc_setup", TO.capi.to_mpc_spec(2, 4, TO.capi._dp(bad), None, None, None, 0, 1))
    TO.mpc_run(p, 1)                          # the earlier setup still holds room for its second step
    X, U, J = TO.mpc_history(p)
    assert X.shape == (8, 3, 4) and U.shape == (8, 2, 1) and J.shape == (8, 2)
    p.close()
