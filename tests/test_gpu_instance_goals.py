"""Per-instance goal states and tracking references (to_set_goal_states / to_update_trajectories / to_set_cost_terms).

Central property: a batch whose instance b is sent to goal g[b % 3] through the per-instance call computes, bit for bit, what instance b of
a batch of the same size, x0 and U0 computes with the shared goal g[b % 3].  Same B on both sides, so that the same kernels are selected."""
import numpy as np
import pytest

import trajopt_b200 as TO
from trajopt_b200 import problems

pytestmark = pytest.mark.gpu

G = 3


def _goals(xf, rng_seed=7, scale=0.3):
    rng = np.random.default_rng(rng_seed)
    out = []
    for _ in range(G):
        g = np.array(xf, dtype=float)
        g[:3] += rng.uniform(-scale, scale, 3)
        out.append(g)
    return out


def _snapshot(p):
    s = dict(cost=TO.cost(p), cost_knots=TO.cost_knots(p), cost_gradient=TO.cost_gradient(p), merit=TO.merit(p),
             max_violation=TO.max_violation(p), X=TO.states(p), U=TO.controls(p))
    for i in range(len(p.constraints)):
        s[f"eval_constraints{i}"] = TO.evaluate_constraints(p, i)
        s[f"multipliers{i}"] = TO.multipliers(p, i)
    return s


def _assert_rows_equal(per, shared, what):
    """per: snapshot of the per-instance batch; shared[j]: snapshot of the batch with the shared goal j"""
    for key, v in per.items():
        for b in range(v.shape[0]):
            ref = shared[b % G][key][b]
            assert np.array_equal(v[b], ref, equal_nan=True), f"{what}: {key} of instance {b} differs from the shared-goal batch"


PATHS = {
    # full-state Quadrotor: k_riccati (tensor-MMA kernel), line search fast path, goal + control bounds
    "quadrotor_full": (lambda: problems.quadrotor(B=48, N=31, dt=0.05), {}),
    # Cartpole, goal + bounds, warp-per-instance and thread-per-instance Riccati kernels
    "cartpole_warp": (lambda: problems.cartpole(B=48, N=51, u_bound=3.0, goal=True), dict(backward_kernel=1)),
    "cartpole_thread": (lambda: problems.cartpole(B=48, N=51, u_bound=3.0, goal=True), dict(backward_kernel=2)),
    # Acrobot with the dense QuadraticCost (dense q = -Q xf): the generic line search
    "acrobot_dense": (lambda: problems.acrobot(B=48, N=41), {}),
    # error-state Quadrotor (the flagship problem class): record path (k_expansion_rec16b + k_riccati_frag), the shared-memory kernel on the
    # compact expansion (k_expansion_compact) and the generic kernel on the materialised expansion (al_expansion + error expansion)
    "quadrotor_rec": (lambda: problems.quadrotor(B=48, N=31, error_state=True), {}),
    "quadrotor_compact": (lambda: problems.quadrotor(B=48, N=31, error_state=True), dict(backward_kernel=5)),
    "quadrotor_dense_lie": (lambda: problems.quadrotor(B=48, N=31, error_state=True), dict(backward_kernel=3)),
    # quaternion costs + QuatVecEq: q_ref / w / QuatVecEq stay shared, the Goal on position and velocities is per instance
    "quadrotor_lie": (lambda: problems.quadrotor_lie(B=48, N=31), {}),
}


def _make(factory, opts):
    p = factory()
    if opts:
        TO.set_options(p, **opts)
    return p


@pytest.mark.parametrize("path", sorted(PATHS))
def test_instance_goals_equal_shared_batches(path):
    factory, opts = PATHS[path]
    per = _make(factory, opts)
    goals = _goals(per.xf)
    B = per.B
    TO.set_goal_state(per, np.stack([goals[b % G] for b in range(B)]))
    assert per.xf.shape == (B, per.n)
    shared = []
    for j in range(G):
        s = _make(factory, opts)
        TO.set_goal_state(s, goals[j])
        shared.append(s)
    probs = [per] + shared
    for p in probs:
        TO.rollout(p)
    _assert_rows_equal(_snapshot(per), [_snapshot(s) for s in shared], f"{path} after rollout")
    for p in probs:
        TO.expand(p)
        TO.backward(p)
    if TO.backward_algebra(per) == 1:   # record path: the cost + AL expansion the Riccati kernel read
        _assert_rows_equal({"records": TO.expansion_records(per)}, [{"records": TO.expansion_records(s)} for s in shared], f"{path} records")
    K = TO.gains(per)
    Ks = [TO.gains(s) for s in shared]
    for b in range(B):
        for a, ref in zip(K, Ks[b % G]):
            assert np.array_equal(a[b], ref[b]), f"{path}: gains of instance {b}"
    for p in probs:
        TO.ilqr_step(p, 3)
    _assert_rows_equal(_snapshot(per), [_snapshot(s) for s in shared], f"{path} after ilqr_step(3)")
    stats = [TO.solve(p, iterations=40) for p in probs]
    for f in TO.SolveStats.FIELDS:
        v = getattr(stats[0], f)
        for b in range(B):
            assert np.array_equal(v[b], getattr(stats[1 + b % G], f)[b]), f"{path}: solve {f} of instance {b}"
    # after to_solve the penalties are those of the batch's last outer iteration, which depends on every instance of the batch: the
    # merit (cost + AL penalty at the current penalties) is a batch-level quantity there, everything else is per instance
    snap = lambda p: {k: v for k, v in _snapshot(p).items() if k != "merit"}
    _assert_rows_equal(snap(per), [snap(s) for s in shared], f"{path} after solve")
    for p in probs:
        p.close()


def _tracking_problem(B, N, Xref, Uref):
    n, m = 4, 1
    obj = TO.TrackingObjective(1e-1 * np.eye(n), 1e-2 * np.eye(m), Xref[:N], Uref[:N - 1], Qf=10 * np.eye(n))
    cons = TO.ConstraintList(n, m, N)
    TO.add_constraint(cons, TO.BoundConstraint(n, m, u_min=-5.0, u_max=5.0), (1, N - 1))
    rng = np.random.default_rng(3)
    x0 = np.zeros((B, n)); x0[:, :2] += 0.05 * rng.standard_normal((B, 2))
    p = TO.Problem(TO.Cartpole(), obj, x0, 0.05 * (N - 1), constraints=cons)
    TO.initial_controls(p, np.full((B, N - 1, m), 0.01) + 0.01 * rng.standard_normal((B, N - 1, m)))
    return p


def test_tracking_mpc_loop_equals_shared_references():
    B, N, nref, steps = 48, 21, 40, 4
    t = np.linspace(0, 2, nref)
    refs = []
    for j in range(G):
        X = np.zeros((nref, 4)); X[:, 0] = (0.2 + 0.1 * j) * np.sin(t + j); X[:, 1] = 0.3 * j * t / 2
        U = np.zeros((nref, 1)); U[:, 0] = 0.1 * j
        refs.append((X, U))
    per = _tracking_problem(B, N, *refs[0])
    # every batch is built from the same reference (the constant terms c of the costs come from it and update_trajectory! leaves c as
    # it is), then each follows its own
    shared = [_tracking_problem(B, N, *refs[0]) for j in range(G)]
    Xb = np.stack([refs[b % G][0] for b in range(B)]); Ub = np.stack([refs[b % G][1] for b in range(B)])
    for step in range(1, steps + 1):
        TO.update_trajectory(per, Xb, Ub, step)
        for j, s in enumerate(shared):
            # the shared C entry point directly: the Python wrapper also mutates the host cost objects, which makes the next call
            # rebuild the handle and restart its multipliers -- the per-instance batch would then be compared against another solve
            Xj, Uj = np.ascontiguousarray(refs[j][0]), np.ascontiguousarray(refs[j][1])
            s._call("to_update_trajectory", TO._capi._dp(Xj), TO._capi._dp(Uj), nref, step)
        for p in [per] + shared:
            TO.rollout(p)
            TO.ilqr_step(p, 2)
        _assert_rows_equal(_snapshot(per), [_snapshot(s) for s in shared], f"MPC step {step}")
        for p in [per] + shared:
            TO.shift_trajectory(p, 1)
    for p in [per] + shared:
        p.close()


def test_shared_goal_after_instance_goals_equals_fresh_batch():
    mk = lambda: problems.cartpole(B=32, N=41, u_bound=3.0, goal=True)
    p, fresh = mk(), mk()
    goals = _goals(p.xf)
    TO.set_goal_state(p, np.stack([goals[b % G] for b in range(p.B)]))
    TO.set_goal_state(p, goals[1])
    TO.set_goal_state(fresh, goals[1])
    for q in (p, fresh):
        TO.rollout(q); TO.ilqr_step(q, 3)
    a, b = _snapshot(p), _snapshot(fresh)
    for k in a:
        assert np.array_equal(a[k], b[k], equal_nan=True), k


def test_objective_and_constraint_flags():
    p = problems.cartpole(B=8, N=21, u_bound=3.0, goal=True)
    q0, r0 = TO.cost_terms(p)
    xf = np.stack([np.array([0.1 * b, np.pi, 0, 0]) for b in range(p.B)])
    TO.set_goal_state(p, xf, objective=False, constraint=True)
    q1, r1 = TO.cost_terms(p)
    assert np.array_equal(q0, q1) and np.array_equal(r0, r1)
    TO.rollout(p)
    c = TO.evaluate_constraints(p, 1)                 # the Goal constraint at N: x_N - xf_b
    X = TO.states(p)
    assert np.array_equal(c[:, 0, :], X[:, -1, :] - xf)
    TO.set_goal_state(p, xf * 0.5, objective=True, constraint=False)
    assert np.array_equal(TO.evaluate_constraints(p, 1), c)
    q2, _ = TO.cost_terms(p)
    assert not np.array_equal(q2, q1)


def test_instance_q_equals_shared_setter_bitwise():
    mk = lambda: problems.acrobot(B=6, N=21)
    p = mk()
    goals = _goals(p.xf)
    TO.set_goal_state(p, np.stack([goals[b % G] for b in range(p.B)]))
    q, r = TO.cost_terms(p)
    for j in range(G):
        s = mk()
        TO.set_goal_state(s, goals[j])
        qs, rs = TO.cost_terms(s)
        for b in range(j, p.B, G):
            assert np.array_equal(q[b], qs[b]) and np.array_equal(r[b], rs[b])
        # the cost gradient at X = 0, U = 0 is q (and r) exactly
        for pp in (p, s):
            TO.initial_states(pp, np.zeros((pp.B, pp.N, pp.n))); TO.initial_controls(pp, np.zeros((pp.B, pp.N - 1, pp.m)))
        g, gs = TO.cost_gradient(p), TO.cost_gradient(s)
        for b in range(j, p.B, G):
            assert np.array_equal(g[b], gs[b])
        s.close()


def test_aliased_cost_tracks_last_knot_per_instance():
    B, N, n, m = 4, 6, 4, 1
    c1 = TO.LQRCost(np.eye(n), np.eye(m), np.zeros(n))
    c2 = TO.LQRCost(10 * np.eye(n), np.eye(m), np.zeros(n), terminal=True)
    obj = TO.Objective([c1] * (N - 1) + [c2])
    p = TO.Problem(TO.Cartpole(), obj, np.zeros((B, n)), 1.0)
    Xref = np.arange(B * 10 * n, dtype=float).reshape(B, 10, n) / 7.0
    Uref = np.arange(B * 10 * m, dtype=float).reshape(B, 10, m) / 3.0
    TO.update_trajectory(p, Xref, Uref, 2)
    q, r = TO.cost_terms(p)
    for b in range(B):
        assert np.array_equal(q[b, 0], -(np.eye(n) @ Xref[b, 2 - 1 + N - 2]))     # the shared stage cost follows its last knot N-1
        assert np.array_equal(r[b, 0], -(np.eye(m) @ Uref[b, 2 - 1 + N - 2]))
        assert np.array_equal(q[b, 1], -(10 * np.eye(n) @ Xref[b, 2 - 1 + N - 1]))
    p.close()


def test_bad_shapes_and_codes():
    p = problems.cartpole(B=4, N=21, u_bound=3.0, goal=True)
    with pytest.raises(TO.DimensionMismatch):
        TO.set_goal_state(p, np.zeros((3, 4)))
    with pytest.raises(TO.DimensionMismatch):
        TO.update_trajectory(p, np.zeros((4, 30, 4)), np.zeros((4, 30, 2)))
    with pytest.raises(TO.DimensionMismatch):
        TO.update_trajectory(p, np.zeros((4, 10, 4)), np.zeros((4, 10, 1)), 1)    # shorter than start + N - 1
    with pytest.raises(TO.DimensionMismatch):
        TO.set_cost_terms(p, np.zeros((4, 1, 4)), np.zeros((4, 2, 1)))
    # the C entry points themselves
    lib, h = p._lib, p._h
    X = np.zeros((4, 10, 4)); U = np.zeros((4, 10, 1))
    assert lib.to_update_trajectories(h, TO._capi._dp(X), TO._capi._dp(U), 10, 1) == TO._capi.TO_EDIM
    assert lib.to_set_goal_states(h, None, 1, 1) == TO._capi.TO_EINVAL
    assert lib.to_get_cost_terms(h, None, None) == TO._capi.TO_EINVAL
    assert lib.to_set_cost_terms(h, None, None) == TO._capi.TO_EINVAL
    vals = np.zeros((4, 4))
    assert lib.to_get_goal_values(h, 0, TO._capi._dp(vals)) == TO._capi.TO_EINVAL      # constraint 0 is the Bound constraint
    assert lib.to_get_goal_values(h, 1, TO._capi._dp(vals)) == TO._capi.TO_OK
    assert np.array_equal(vals, np.tile(p.xf, (4, 1)))                                     # the shared values broadcast
    p.close()


def test_rebuild_keeps_instance_goals():
    mk = lambda: problems.cartpole(B=12, N=31, u_bound=3.0)
    p = mk()
    goals = _goals(p.xf)
    xf = np.stack([goals[b % G] for b in range(p.B)])
    TO.set_goal_state(p, xf)
    q_before, r_before = TO.cost_terms(p)
    TO.add_constraint(p.constraints, TO.GoalConstraint(p.xf[0]), p.N)       # live add_constraint!: the handle is rebuilt
    q_after, r_after = TO.cost_terms(p)
    assert np.array_equal(q_before, q_after) and np.array_equal(r_before, r_after)
    TO.rollout(p)
    c = TO.evaluate_constraints(p, len(p.constraints) - 1)
    # the Goal constraint added after the per-instance call holds the value it was built with, in every instance
    assert np.array_equal(c[:, 0, :], TO.states(p)[:, -1, :] - xf[0])
    # a cost mutated in place after the per-instance call takes its new value in every instance
    c0 = p.obj[0]
    TO.set_LQR_goal(c0, np.zeros(p.n))
    q_new, _ = TO.cost_terms(p)
    j = [id(c) for c in p._cost_objs].index(id(c0))
    assert np.all(q_new[:, j] == q_new[0, j])
    others = [k for k in range(q_new.shape[1]) if k != j]
    assert np.array_equal(q_new[:, others], q_before[:, others])
    p.close()


def test_rebuild_carries_goal_rows_of_unchanged_constraints():
    p = problems.cartpole(B=12, N=31, u_bound=3.0, goal=True)
    goals = _goals(p.xf)
    xf = np.stack([goals[b % G] for b in range(p.B)])
    TO.set_goal_state(p, xf)
    goal_idx = 1
    TO.add_constraint(p.constraints, TO.BoundConstraint(4, 1, u_min=-10.0, u_max=10.0), (1, p.N - 1))    # rebuild
    TO.rollout(p)
    assert np.array_equal(TO.evaluate_constraints(p, goal_idx)[:, 0, :], TO.states(p)[:, -1, :] - xf)
    # a Goal constraint whose xf is changed on the host takes the new value in every instance
    p.constraints[goal_idx].xf = np.array([0.5, np.pi, 0, 0])
    p.constraints._version = getattr(p.constraints, "_version", 0) + 1
    TO.add_constraint(p.constraints, TO.BoundConstraint(4, 1, u_min=-20.0, u_max=20.0), (1, p.N - 1))
    TO.rollout(p)
    assert np.array_equal(TO.evaluate_constraints(p, goal_idx)[:, 0, :], TO.states(p)[:, -1, :] - np.array([0.5, np.pi, 0, 0]))
    p.close()


def test_instance_goals_flagship_size():
    """BASELINE size: error-state Quadrotor 4096 x 101 on the record path"""
    mk = lambda: problems.quadrotor(B=4096, N=101, error_state=True)
    per = mk()
    goals = _goals(per.xf)
    TO.set_goal_state(per, np.stack([goals[b % G] for b in range(per.B)]))
    shared = []
    for j in range(G):
        s = mk(); TO.set_goal_state(s, goals[j]); shared.append(s)
    for p in [per] + shared:
        TO.rollout(p); TO.ilqr_step(p, 2)
    snap = lambda p: dict(merit=TO.merit(p), X=TO.states(p), U=TO.controls(p))
    _assert_rows_equal(snap(per), [snap(s) for s in shared], "4096 x 101")
    for p in [per] + shared:
        p.close()
