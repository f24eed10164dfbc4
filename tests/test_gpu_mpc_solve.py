"""Closed-loop MPC whose plan is a solve (to_mpc_solve / to_mpc_solve_history).

Central property: a device run computes, bit for bit, what the host-scripted loop of existing entry points computes -- set_penalties with
the shared penalties for every constraint (once), then per step update_trajectory (per instance), solve, controls / merit, the plant step
taken by a second Problem with N = 2 (as in test_gpu_mpc), shift_trajectory(1) and set_initial_state.  Two identical problems are built for
each case: one runs the device loop, the other the scripted loop.  The options of each case give, within one step, instances that stop
early, instances stopped at the iteration cap and (constrained cases) instances that took an outer step, and the test checks that they do."""
import numpy as np
import pytest

import trajopt_b200 as TO
from trajopt_b200 import problems
from test_gpu_mpc import _autodiff, _equal, _plant, _reference, _state

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(TO.Problem.__name__ == "OracleProblem", reason="closed-loop MPC has no oracle counterpart")]

STATS = ("status", "iterations", "iterations_outer", "c_max")


def _cartpole(B=64, N=21):
    return problems.cartpole(B=B, N=N, u_bound=4.0, goal=True)


def _double_integrator(B=64, N=21):
    return problems.double_integrator(B=B, N=N, dim=2, constrained=False)


def _quadrotor(B=64, N=31):
    return problems.quadrotor(B=B, N=N, error_state=True, u_noise=0.01)


CASES = {
    # name: (factory, reference, per-instance plant params / dt / weights, solve options)
    "cartpole_ref": (_cartpole, True, False, dict(iterations=15, iterations_inner=4, cost_tolerance_intermediate=1e-2,
                                                  gradient_tolerance_intermediate=10.0, constraint_tolerance=1e-2)),
    "double_integrator": (_double_integrator, True, False, dict(iterations=3, cost_tolerance=1e-3)),
    "quadrotor_record_inst": (_quadrotor, True, True, dict(iterations=6, cost_tolerance_intermediate=1e-1, gradient_tolerance_intermediate=10.0,
                                                           constraint_tolerance=1e-3)),
    "autodiff_dynamics": (_autodiff, False, False, dict(iterations=4, cost_tolerance=1e-2)),
}


def _setup(name, steps=5):
    """two identical problems (device, scripted), the mpc_setup keywords, and the scripted loop's plant"""
    factory, ref, inst, _ = CASES[name]
    dev, scr = factory(), factory()
    B = dev.B
    r = np.random.default_rng(11)
    kw, plant_rows, dtb = {}, None, None
    if ref:
        kw["Xref"], kw["Uref"] = _reference(dev, dev.N + steps + 3)
        kw["start"] = 2
    if inst:
        base = np.asarray(dev.model.params, dtype=float)
        plant_rows = base[None, :] * (1.0 + 0.05 * r.uniform(-1, 1, (B, base.size)))
        kw["plant_params"] = plant_rows
        dtb = np.tile(dev.spec.dt, (B, 1)) * (1.0 + 0.1 * (np.arange(B) % 3))[:, None]
        for p in (dev, scr):
            TO.set_time_steps(p, dtb)
            TO.set_model_params(p, base[None, :] * (1.0 + 0.02 * (np.arange(B) % 4))[:, None])
            for c in range(len(dev._cost_objs)):
                TO.set_cost_weights(p, c, TO.cost_weights(p, c) * (1.0 + 0.25 * (np.arange(B) % 5))[:, None])
    plant = _plant(scr, plant_rows if plant_rows is not None else (TO.model_params(scr) if dtb is not None else None), dtb)
    return dev, scr, kw, plant


def _table(p):
    """what the first mpc_solve does on a constrained problem: every instance holds the shared penalties"""
    for i in range(len(p.constraints)):
        TO.set_penalties(p, i, TO.penalty(p, i))


def _scripted(p, plant, steps, opts, ref=None, start=1, j0=0, solve=True):
    """`steps` MPC steps from step j0: a solve with `opts` per step (solve=False: rollout + ilqr_step(opts["iterations"]), mpc_run's plan)"""
    X, U, J, S = [p.x0.copy()], [], [], {f: [] for f in STATS}
    for s in range(steps):
        j = j0 + s
        if ref is not None:
            TO.update_trajectory(p, ref[0], ref[1], start + j)
        if solve:
            st = TO.solve(p, **opts)
            for f in STATS:
                S[f].append(getattr(st, f).copy())
        else:
            TO.rollout(p)
            TO.ilqr_step(p, opts["iterations"])
            for f, v in zip(STATS, (-1, 0, 0, np.nan)):
                S[f].append(np.full(p.B, v, dtype=np.float64 if f == "c_max" else np.int32))
        u = TO.controls(p)[:, 0].copy()
        J.append(TO.merit(p).copy())
        TO.set_initial_state(plant, p.x0)
        TO.initial_controls(plant, u[:, None, :])
        TO.rollout(plant)
        xn = TO.states(plant)[:, 1].copy()
        TO.shift_trajectory(p, 1)
        TO.set_initial_state(p, xn)
        X.append(xn); U.append(u)
    return (np.stack(X, 1), np.stack(U, 1), np.stack(J, 1)), {f: np.stack(v, 1) for f, v in S.items()}


def _stats(p):
    h = TO.mpc_solve_history(p)
    return {f: getattr(h, f) for f in STATS}


def _full_state(p):
    out = _state(p)
    for i in range(len(p.constraints)):
        out[f"penalties{i}"] = TO.penalties(p, i)
    s = TO.solver_state(p)
    for k in ("rho", "alpha", "ls_iters", "bp_status"):
        out[k] = s[k]
    return out


def _assert_history(dev, hist, stats, what):
    for name, x, y in zip(("Xcl", "Ucl", "J"), TO.mpc_history(dev), hist):
        assert x.shape == y.shape and np.array_equal(x, y), f"{what}: {name} (max |d| = {np.nanmax(np.abs(x - y)):.3e})"
    got = _stats(dev)
    for f in STATS:
        assert got[f].dtype == stats[f].dtype and np.array_equal(got[f], stats[f], equal_nan=True), f"{what}: {f}"


def _assert_mix(stats, budget, constrained, what):
    """some step had instances that stopped early, instances stopped at the cap and (constrained) an outer step"""
    it, st, outer = stats["iterations"], stats["status"], stats["iterations_outer"]
    early = (it < budget).any(axis=0)
    capped = ((it == budget) & (st == TO.capi.SOLVE_MAX_ITERATIONS)).any(axis=0)
    stepped = (outer > 1).any(axis=0) if constrained else np.ones_like(early)
    assert (early & capped & stepped).any(), (f"{what}: no step mixes early stops, the cap{' and outer steps' if constrained else ''}: "
                                              f"iterations {it.min(0)}..{it.max(0)}, outer max {outer.max(0)}")


@pytest.mark.parametrize("name", sorted(CASES))
def test_device_loop_is_the_scripted_solve_loop(name):
    steps = 5
    opts = CASES[name][3]
    dev, scr, kw, plant = _setup(name, steps)
    constrained = len(dev.constraints) > 0
    TO.mpc_setup(dev, steps, **kw)
    TO.mpc_solve(dev, steps, **opts)
    if constrained:
        _table(scr)
    hist, stats = _scripted(scr, plant, steps, opts, (kw["Xref"], kw["Uref"]) if "Xref" in kw else None, kw.get("start", 1))
    _assert_history(dev, hist, stats, name)
    _equal(_full_state(dev), _full_state(scr), name)
    _assert_mix(stats, opts["iterations"], constrained, name)
    assert not np.array_equal(hist[0][:, 0], hist[0][:, -1])
    for p in (dev, scr, plant):
        p.close()


def test_mixed_runs_equal_the_scripted_mix():
    """mpc_run steps, then mpc_solve steps, then mpc_run steps; the mpc_run rows keep the marker"""
    name = "cartpole_ref"
    opts = CASES[name][3]
    dev, scr, kw, plant = _setup(name, 7)
    ref = (kw["Xref"], kw["Uref"])
    TO.mpc_setup(dev, 7, **kw)
    TO.mpc_run(dev, 2, 2)
    TO.mpc_solve(dev, 3, **opts)
    TO.mpc_run(dev, 2, 2)
    parts = [_scripted(scr, plant, 2, dict(iterations=2), ref, 2, 0, solve=False)]
    _table(scr)
    parts.append(_scripted(scr, plant, 3, opts, ref, 2, 2))
    parts.append(_scripted(scr, plant, 2, dict(iterations=2), ref, 2, 5, solve=False))
    X = np.concatenate([parts[0][0][0]] + [q[0][0][:, 1:] for q in parts[1:]], 1)
    U, J = (np.concatenate([q[0][i] for q in parts], 1) for i in (1, 2))
    stats = {f: np.concatenate([q[1][f] for q in parts], 1) for f in STATS}
    _assert_history(dev, (X, U, J), stats, "run 2, solve 3, run 2")
    _equal(_full_state(dev), _full_state(scr), "run 2, solve 3, run 2")
    got = _stats(dev)
    assert (got["status"][:, [0, 1, 5, 6]] == -1).all() and np.isnan(got["c_max"][:, [0, 1, 5, 6]]).all()
    assert (got["status"][:, 2:5] >= 0).all()
    for p in (dev, scr, plant):
        p.close()


def test_chunked_solves_equal_one_run():
    opts = CASES["quadrotor_record_inst"][3]
    a, b = _quadrotor(), _quadrotor()
    Xref, Uref = _reference(a, a.N + 8)
    for p in (a, b):
        TO.mpc_setup(p, 7, Xref=Xref, Uref=Uref)
    TO.mpc_solve(a, 3, **opts); TO.mpc_solve(a, 4, **opts)
    TO.mpc_solve(b, 7, **opts)
    for x, y in zip(TO.mpc_history(a), TO.mpc_history(b)):
        assert x.shape == y.shape and np.array_equal(x, y)
    sa, sb = _stats(a), _stats(b)
    for f in STATS:
        assert np.array_equal(sa[f], sb[f]), f
    _equal(_full_state(a), _full_state(b), "3 + 4 steps against 7")
    with pytest.raises(TO.DimensionMismatch):
        TO.mpc_solve(a, 1, **opts)
    a.close(); b.close()


def test_sub_batch_gives_the_batch_rows():
    from test_gpu_solve import subset
    opts = CASES["cartpole_ref"][3]
    g = problems.cartpole(B=48, N=21, u_bound=4.0, goal=True)
    idx = np.array([1, 7, 30, 47])
    q = subset(problems.cartpole(B=48, N=21, u_bound=4.0, goal=True), idx)
    for p in (g, q):
        TO.set_options(p, backward_kernel=1)      # the kernel a batch of 4 takes (test_gpu_instance_penalties COMPOSE)
    assert TO.kernel_choice(g)["backward"] == TO.kernel_choice(q)["backward"]
    Xref, Uref = _reference(g, g.N + 6)
    TO.mpc_setup(g, 5, Xref=Xref, Uref=Uref)
    TO.mpc_setup(q, 5, Xref=Xref[idx], Uref=Uref[idx])
    TO.mpc_solve(g, 5, **opts)
    TO.mpc_solve(q, 5, **opts)
    for x, y in zip(TO.mpc_history(g), TO.mpc_history(q)):
        assert np.array_equal(x[idx], y)
    sg, sq = _stats(g), _stats(q)
    assert len(np.unique(sg["iterations"])) > 1
    for f in STATS:
        assert np.array_equal(sg[f][idx], sq[f]), f
    g.close(); q.close()


def test_solve_run_is_asynchronous():
    import torch
    opts = CASES["cartpole_ref"][3]
    ref, dev = _cartpole(), _cartpole()
    for p in (ref, dev):
        TO.mpc_setup(p, 3)
        _table(p)      # the table exists: the first mpc_solve has nothing to create
    TO.mpc_solve(ref, 3, **opts)
    expected = TO.mpc_history(ref), _stats(ref)
    with torch.cuda.stream(torch.cuda.Stream()):
        stream = torch.cuda.current_stream()
        dev._call("to_set_stream", stream.cuda_stream)
        torch.cuda._sleep(1_000_000_000)     # about half a second of GPU time ahead of the run on the same stream
        TO.mpc_solve(dev, 3, **opts)
        pending = not stream.query()
        stream.synchronize()
    assert pending, "to_mpc_solve waited for the device"
    for x, y in zip(TO.mpc_history(dev), expected[0]):
        assert np.array_equal(x, y)
    got = _stats(dev)
    for f in STATS:
        assert np.array_equal(got[f], expected[1][f]), f
    ref.close(); dev.close()


def test_constrained_recorded_model_is_refused_with_nothing_changed():
    """per-instance penalties are not supported on recorded-program models, so the device cannot take their outer steps"""
    import ctypes
    from dynamics_programs import recorded_builtin
    rec, _ = recorded_builtin("cartpole")
    N, B = 21, 8
    obj = TO.LQRObjective(1e-2 * np.eye(4), 1e-1 * np.eye(1), 100.0 * np.eye(4), np.array([0, np.pi, 0, 0.0]), N)
    cons = TO.ConstraintList([rec] * (N - 1))
    TO.add_constraint(cons, TO.BoundConstraint(4, 1, u_min=-4.0, u_max=4.0), (1, N - 1))
    x0 = np.zeros((B, 4)); x0[:, :2] += 0.1 * np.random.default_rng(2).standard_normal((B, 2))
    p = TO.Problem(rec, obj, x0, 2.0, constraints=cons)
    TO.initial_controls(p, np.full((B, N - 1, 2), 0.01) * np.array([1.0, 0.0]))
    TO.mpc_setup(p, 3)
    TO.mpc_run(p, 1)
    before = _state(p), TO.mpc_history(p), _stats(p), TO.penalties(p, 0)
    l0 = p._lib.to_launch_count(p._h)
    with pytest.raises(TO.ArgumentError, match="recorded-program"):
        TO.mpc_solve(p, 1)
    assert p._mpc["done"] == 1
    o = TO.solve_options()
    assert p._lib.to_mpc_solve(p._h, 1, ctypes.byref(o)) == -1                 # TO_EINVAL, from the C check itself
    assert "recorded-program" in p._lib.to_last_error(p._h).decode()
    assert p._lib.to_launch_count(p._h) == l0
    _equal(_state(p), before[0], "refused mpc_solve")
    for x, y in zip(TO.mpc_history(p), before[1]):
        assert np.array_equal(x, y)
    after = _stats(p)
    for f in STATS:
        assert np.array_equal(after[f], before[2][f], equal_nan=True), f
    assert np.array_equal(TO.penalties(p, 0), before[3])
    TO.mpc_run(p, 2)                    # the setup still holds room for two steps
    assert TO.mpc_history(p)[1].shape == (B, 3, 2)
    p.close()
