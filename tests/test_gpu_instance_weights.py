"""Per-instance cost weights (to_set_cost_weights).

Central property: a batch whose instance b holds the weights w[b % 3] computes, bit for bit, what instance b of a batch of the same size,
x0 and U0 built with w[b % 3] as its shared cost weights computes.  Same B on both sides, so that the same kernels are selected."""
import copy

import numpy as np
import pytest

import trajopt_b200 as TO
from trajopt_b200 import problems
from test_gpu_instance_params import PATHS, G, _compare_pipeline, _assert_rows_equal, _snapshot

pytestmark = pytest.mark.gpu


def _scaled(cost, j, ci):
    """cost with weight set j: Q, R (and H) scaled by factors in [0.5, 2], c shifted, the quaternion weight w scaled; q and r kept"""
    rng = np.random.default_rng(100 * j + ci)
    c = copy.copy(cost)
    n, m = c.state_dim, c.control_dim
    if c.is_diag:
        c.Q = np.diag(np.diagonal(c.Q) * rng.uniform(0.5, 2.0, n))
        c.R = np.diag(np.diagonal(c.R) * rng.uniform(0.5, 2.0, m))
    else:
        c.Q = c.Q * rng.uniform(0.5, 2.0)
        c.R = c.R * rng.uniform(0.5, 2.0)
        c.H = c.H * rng.uniform(0.5, 2.0)
    c.c = c.c + 0.25 * j
    if isinstance(c, TO.DiagonalQuatCost):
        c.w = c.w * rng.uniform(0.5, 2.0)
    return c


def _weighted(j):
    """a `cls` for the problem builders: the problem is built with weight set j on each of its distinct costs"""
    def cls(model, obj, *a, **k):
        uniq, _ = obj._tables()
        for ci, c in enumerate(uniq):
            s = _scaled(c, j, ci)
            c.Q, c.R, c.H, c.c = s.Q, s.R, s.H, s.c
            if isinstance(c, TO.DiagonalQuatCost):
                c.w = s.w
        return TO.Problem(model, obj, *a, **k)
    return cls


def _set_rows(p, sets=G):
    """instance b of p takes weight set b % sets on every distinct cost, as raw rows"""
    for ci, c in enumerate(p._cost_objs):
        rows = np.stack([TO.api._cost_weight_row(_scaled(c, b % sets, ci)) for b in range(p.B)])
        TO.set_cost_weights(p, ci, rows)
        assert np.array_equal(TO.cost_weights(p, ci), rows)


def _make(factory, opts, cls=None):
    p = factory(cls)
    if opts:
        TO.set_options(p, **opts)
    return p


def _dense_h_quadrotor(cls):
    """full-state Quadrotor with a QuadraticCost with a non-zero H: the dense DFMA k_riccati path"""
    return problems.quadrotor(B=48, N=31, dt=0.05, dense_cost=True, cls=cls)


def _tracking(cls, B=48, N=21):
    """Cartpole tracking objective: one distinct cost per knot, more than the line search caches (FWD_MAX_COST)"""
    n, m = 4, 1
    t = np.linspace(0, 2, N)
    X = np.zeros((N, n)); X[:, 0] = 0.2 * np.sin(t); U = np.zeros((N - 1, m))
    obj = TO.TrackingObjective(1e-1 * np.eye(n), 1e-2 * np.eye(m), X, U, Qf=10 * np.eye(n))
    cons = TO.ConstraintList(n, m, N)
    TO.add_constraint(cons, TO.BoundConstraint(n, m, u_min=-5.0, u_max=5.0), (1, N - 1))
    rng = np.random.default_rng(3)
    x0 = np.zeros((B, n)); x0[:, :2] += 0.05 * rng.standard_normal((B, 2))
    p = (cls or TO.Problem)(TO.Cartpole(), obj, x0, 0.05 * (N - 1), constraints=cons)
    TO.initial_controls(p, np.full((B, N - 1, m), 0.01) + 0.01 * rng.standard_normal((B, N - 1, m)))
    return p


WPATHS = dict(PATHS)
WPATHS["quadrotor_dense_h"] = (_dense_h_quadrotor, {})
WPATHS["cartpole_tracking"] = (_tracking, {})


@pytest.mark.parametrize("path", sorted(WPATHS))
def test_instance_weights_equal_shared_batches(path):
    factory, opts = WPATHS[path]
    per = _make(factory, opts)
    _set_rows(per)
    shared = [_make(factory, opts, _weighted(j)) for j in range(G)]
    _compare_pipeline(per, shared, path)
    for p in [per] + shared:
        p.close()


def test_setup_covers_both_sides_of_the_cost_cache():
    assert len(_tracking(None)._cost_objs) > 4                           # forward.cu FWD_MAX_COST
    assert len(problems.cartpole(B=4, N=11, u_bound=3.0, goal=True)._cost_objs) <= 4
    p = _dense_h_quadrotor(None)
    assert any(not c.is_blockdiag() for c in p._cost_objs)


@pytest.mark.parametrize("path", ["quadrotor_rec", "double_integrator_quickstart", "acrobot_dense"])
def test_equal_rows_equal_untouched_batch(path):
    """every row equal to the shared weights: the outputs of a batch that never called the setter; only the inst_* choices differ"""
    factory, opts = PATHS[path]
    per, plain = _make(factory, opts), _make(factory, opts)
    for ci, c in enumerate(per._cost_objs):
        TO.set_cost_weights(per, ci, np.tile(TO.api._cost_weight_row(c), (per.B, 1)))
    a, b = TO.kernel_choice(per), TO.kernel_choice(plain)
    for k in a:
        if not k.startswith("inst"):
            assert a[k] == b[k], k
    assert a["inst_forward"] and a["inst_backward"] and not b["inst_forward"]
    _compare_pipeline(per, [plain], path, sets=1)
    per.close(); plain.close()


def test_weights_with_goals_params_and_constraint_data():
    """weights, goals, model parameters and constraint data per instance together, on the record path"""
    factory = lambda cls: problems.quadrotor(B=48, N=31, error_state=True, cls=cls)
    per = factory(None)
    xf = per.xf
    goals = [xf + 0.1 * j for j in range(G)]
    mass = [0.5 * (1 + 0.1 * j) for j in range(G)]
    _set_rows(per)
    TO.set_goal_state(per, np.stack([goals[b % G] for b in range(per.B)]))
    base = np.array(per.model.params, dtype=float)
    params = []
    for j in range(G):
        q = base.copy(); q[0] = mass[j]; params.append(q)
    TO.set_model_params(per, np.stack([params[b % G] for b in range(per.B)]))
    bi = next(i for i, c in enumerate(per.constraints) if isinstance(c, TO.BoundConstraint))
    rows0 = TO.constraint_data(per, bi)
    nm = per.n + per.m
    data = [rows0[0].copy() for _ in range(G)]
    for j in range(G):
        data[j][per.n:nm] *= 1 + 0.1 * j; data[j][nm + per.n:] *= 1 + 0.1 * j
    TO.set_constraint_data(per, bi, np.stack([data[b % G] for b in range(per.B)]))
    shared = []
    for j in range(G):
        mdl = TO.Quadrotor(); mdl.params = [float(v) for v in params[j]]
        s = factory(lambda model, obj, *a, _j=j, _m=mdl, **k: _weighted(_j)(_m, obj, *a, **k))
        TO.set_goal_state(s, goals[j])
        TO.set_constraint_data(s, bi, np.tile(data[j], (s.B, 1)))
        shared.append(s)
    _compare_pipeline(per, shared, "weights + goals + params + data")
    for p in [per] + shared:
        p.close()


def _lqr_problem(Qs, Rs, xf, B=48, N=41, cls=None):
    n, m = 4, 1
    obj = TO.LQRObjective(Qs[0], Rs[0], Qs[1], xf, N)
    cons = TO.ConstraintList(n, m, N)
    TO.add_constraint(cons, TO.BoundConstraint(n, m, u_min=-3.0, u_max=3.0), (1, N - 1))
    rng = np.random.default_rng(5)
    x0 = np.zeros((B, n)); x0[:, :2] += 0.05 * rng.standard_normal((B, 2))
    p = TO.Problem(TO.Cartpole(), obj, x0, 2.0, constraints=cons)
    TO.initial_controls(p, 0.01 * rng.standard_normal((B, N - 1, m)))
    return p


def _lqr_sets():
    rng = np.random.default_rng(7)
    return [((np.diag(rng.uniform(0.5, 2, 4)), np.diag(100 * rng.uniform(0.5, 2, 4))), (np.diag(0.1 * rng.uniform(0.5, 2, 1)),))
            for _ in range(G)]


def _set_rows_of(per, shared):
    """instance b of per takes the weights (c included) of the costs of shared[b % len(shared)] as raw rows"""
    for ci in range(len(per._cost_objs)):
        TO.set_cost_weights(per, ci, np.stack([TO.api._cost_weight_row(shared[b % len(shared)]._cost_objs[ci]) for b in range(per.B)]))


@pytest.mark.parametrize("how", ["goal_states", "goal_state_shared", "update_trajectories"])
def test_linear_terms_follow_instance_weights(how):
    """after per-instance weights the goal setters use each instance's Q and R: the batches built with LQRObjective(Q_j, R_j, Qf_j, xf)"""
    sets = _lqr_sets()
    xf0 = np.array([0.0, np.pi, 0.0, 0.0]); xf = np.array([0.1, np.pi, 0.0, 0.0])
    per = _lqr_problem((np.eye(4), np.eye(4)), (np.eye(1),), xf0)
    shared = [_lqr_problem((sets[j][0][0], sets[j][0][1]), (sets[j][1][0],), xf) for j in range(G)]
    _set_rows_of(per, shared)
    N = per.N
    if how != "update_trajectories":   # the shared batches' q through the same C setter (LQRObjective computed it in NumPy)
        for s in shared:
            s._call("to_set_goal_state", TO._capi._dp(np.ascontiguousarray(xf)), 1, 0)
    if how == "goal_states":
        TO.set_goal_state(per, np.tile(xf, (per.B, 1)), constraint=False)
    elif how == "goal_state_shared":
        TO.set_goal_state(per, xf, constraint=False)
    else:
        Xr = np.tile(xf, (per.B, N, 1)); Ur = np.zeros((per.B, N, 1))
        TO.update_trajectory(per, Xr, Ur, 1)
        for s in shared:
            Xj, Uj = np.ascontiguousarray(np.tile(xf, (N, 1))), np.zeros((N, 1))
            s._call("to_update_trajectory", TO._capi._dp(Xj), TO._capi._dp(Uj), N, 1)
    q, r = TO.cost_terms(per)
    for b in range(per.B):
        qs, rs = TO.cost_terms(shared[b % G])
        assert np.array_equal(q[b], qs[b]) and np.array_equal(r[b], rs[b]), f"{how}: linear terms of instance {b}"
    for ci, c in enumerate(per._cost_objs):
        W = TO.cost_weights(per, ci)
        for b in range(per.B):
            assert np.array_equal(W[b], TO.cost_weights(shared[b % G], ci)[b])
    _compare_pipeline(per, shared, how)
    for p in [per] + shared:
        p.close()


def test_weights_after_goals_keep_cost_terms():
    p = problems.cartpole(B=32, N=41, u_bound=3.0, goal=True)
    TO.set_goal_state(p, np.stack([p.xf + 0.01 * b for b in range(p.B)]))
    q0, r0 = TO.cost_terms(p)
    _set_rows(p)
    q1, r1 = TO.cost_terms(p)
    assert np.array_equal(q0, q1) and np.array_equal(r0, r1)
    p.close()


def test_cost_objects_give_the_batch_built_with_them():
    """[cost_b] * B: weights and linear terms of the cost objects, the batch built with them"""
    factory = lambda cls: problems.cartpole(B=48, N=51, u_bound=3.0, goal=True, cls=cls)
    per = factory(None)
    shared = [factory(_weighted(j)) for j in range(G)]
    for ci, c in enumerate(per._cost_objs):
        TO.set_cost_weights(per, ci, [shared[b % G]._cost_objs[ci] for b in range(per.B)])
    _compare_pipeline(per, shared, "cost objects")
    for p in [per] + shared:
        p.close()


def test_solve_composition_independence():
    """the solve of a batch with weight set b % 3 against the shared batches, and the instances holding set 0 against a batch where every
    instance holds it: statuses, counts, X, U, multipliers, K, d"""
    sets = _lqr_sets()
    xf = np.array([0.0, np.pi, 0.0, 0.0])
    shared = [_lqr_problem((sets[j][0][0], sets[j][0][1]), (sets[j][1][0],), xf) for j in range(G)]
    mixed = _lqr_problem((np.eye(4), np.eye(4)), (np.eye(1),), xf)
    alone = _lqr_problem((np.eye(4), np.eye(4)), (np.eye(1),), xf)
    _set_rows_of(mixed, shared)
    _set_rows_of(alone, shared[:1])
    for p in [mixed, alone] + shared:
        p._call("to_set_goal_state", TO._capi._dp(np.ascontiguousarray(xf)), 1, 0)
    st = [TO.solve(p, iterations=30) for p in [mixed, alone] + shared]
    X = [TO.states(p) for p in [mixed, alone] + shared]
    U = [TO.controls(p) for p in [mixed, alone] + shared]
    L = [[TO.multipliers(p, i) for i in range(len(mixed.constraints))] for p in [mixed, alone] + shared]
    K = [TO.gains(p) for p in [mixed, alone] + shared]
    for b in range(mixed.B):
        refs = [1] if b % G == 0 else []
        refs.append(2 + b % G)
        for r in refs:
            assert np.array_equal(X[0][b], X[r][b]), f"X of instance {b}"
            assert np.array_equal(U[0][b], U[r][b]), f"U of instance {b}"
            for i, (a, ref) in enumerate(zip(L[0], L[r])):
                assert np.array_equal(a[b], ref[b]), f"multipliers of constraint {i}, instance {b}"
            for f in TO.SolveStats.FIELDS:
                assert np.array_equal(getattr(st[0], f)[b], getattr(st[r], f)[b]), f"{f} of instance {b}"
            for a, ref in zip(K[0], K[r]):
                assert np.array_equal(a[b], ref[b]), f"gains of instance {b}"
    for p in [mixed, alone] + shared:
        p.close()


def test_refusals_leave_the_table_and_rebuild_carries_rows():
    p = problems.acrobot(B=8, N=21)
    ci = 0
    shared = TO.cost_weights(p, ci)
    bad = shared.copy(); bad[3, 2] = np.nan
    with pytest.raises(TO.ArgumentError, match="instance 3, entry 2"):
        TO.set_cost_weights(p, ci, bad)
    assert np.array_equal(TO.cost_weights(p, ci), shared)
    # the C entry point refuses the same rows and names them, and the table stays absent
    with pytest.raises(TO.ArgumentError, match="instance 3, entry 2"):
        p._call("to_set_cost_weights", ci, TO._capi._dp(np.ascontiguousarray(bad)))
    assert not TO.kernel_choice(p)["inst_forward"]
    good = shared * 1.5
    TO.set_cost_weights(p, ci, good)
    with pytest.raises(TO.ArgumentError, match="instance 3, entry 2"):
        p._call("to_set_cost_weights", ci, TO._capi._dp(np.ascontiguousarray(bad)))
    assert np.array_equal(TO.cost_weights(p, ci), good)
    # a rebuild (a constraint added) carries the rows of unchanged costs; a cost whose weights change in place wins in every instance
    TO.add_constraint(p.constraints, TO.BoundConstraint(4, 1, x_max=[10.0, 10, 10, 10]), (1, p.N - 1))
    assert np.array_equal(TO.cost_weights(p, ci), good)
    c = p._cost_objs[ci]
    c.Q = c.Q * 2.0
    c._version = getattr(c, "_version", 0) + 1
    assert np.array_equal(TO.cost_weights(p, ci), np.tile(TO.api._cost_weight_row(c), (p.B, 1)))
    p.close()


def test_mpc_loop_with_instance_weights():
    """per-instance weights, then an MPC loop: update_trajectory with each instance's reference, a solve, shift_trajectory; every step
    against the shared batches built with each weight set and following that set's reference"""
    B, N, nref, steps = 48, 21, 40, 4
    shared = [_tracking(_weighted(j), B, N) for j in range(G)]
    per = _tracking(None, B, N)
    _set_rows_of(per, shared)
    t = np.linspace(0, 2, nref)
    refs = []
    for j in range(G):
        X = np.zeros((nref, 4)); X[:, 0] = (0.2 + 0.1 * j) * np.sin(t + j); X[:, 1] = 0.3 * j * t / 2
        U = np.zeros((nref, 1)); U[:, 0] = 0.1 * j
        refs.append((X, U))
    Xb = np.stack([refs[b % G][0] for b in range(B)]); Ub = np.stack([refs[b % G][1] for b in range(B)])
    probs = [per] + shared
    for step in range(1, steps + 1):
        TO.update_trajectory(per, Xb, Ub, step)
        for j, s in enumerate(shared):
            # the shared C entry point: the Python wrapper also mutates the host cost objects, which rebuilds the handle
            Xj, Uj = np.ascontiguousarray(refs[j][0]), np.ascontiguousarray(refs[j][1])
            s._call("to_update_trajectory", TO._capi._dp(Xj), TO._capi._dp(Uj), nref, step)
        q, r = TO.cost_terms(per)
        for b in range(B):
            qs, rs = TO.cost_terms(shared[b % G])
            assert np.array_equal(q[b], qs[b]) and np.array_equal(r[b], rs[b]), f"MPC step {step}: linear terms of instance {b}"
        for p in probs:
            TO.rollout(p)
        stats = [TO.solve(p, iterations=15) for p in probs]
        for f in TO.SolveStats.FIELDS:
            for b in range(B):
                assert np.array_equal(getattr(stats[0], f)[b], getattr(stats[1 + b % G], f)[b]), f"MPC step {step}: solve {f} of instance {b}"
        snap = lambda p: {k: v for k, v in _snapshot(p).items() if k != "merit"}
        _assert_rows_equal(snap(per), [snap(s) for s in shared], f"MPC step {step}")
        Kp = TO.gains(per)
        Ks = [TO.gains(s) for s in shared]
        for b in range(B):
            for a, ref in zip(Kp, Ks[b % G]):
                assert np.array_equal(a[b], ref[b]), f"MPC step {step}: gains of instance {b}"
        for p in probs:
            TO.shift_trajectory(p, 1)
    for p in probs:
        p.close()


def _mild(cost, j, ci):
    """cost with weight set j of the BASELINE-size test: Qd and Rd scaled entry by entry by factors in [0.8, 1.25], c shifted"""
    rng = np.random.default_rng(1000 + 100 * j + ci)
    c = copy.copy(cost)
    c.Q = np.diag(np.diagonal(c.Q) * rng.uniform(0.8, 1.25, c.state_dim))
    c.R = np.diag(np.diagonal(c.R) * rng.uniform(0.8, 1.25, c.control_dim))
    c.c = c.c + 0.25 * j
    return c


def test_flagship_size_against_the_oracle():
    """BASELINE size, error-state Quadrotor 4096 x 101, 8 weight sets (b % 8, Qd and Rd within [0.8, 1.25], as the parameter sets of
    test_gpu_instance_params.py stay within +-20 %: GAIN_TOL was measured on the BASELINE weights, and a kernel's rounding error in the
    gains grows with the conditioning the weights give Quu).  Per set: the rows of the per-instance batch are bit for bit those of a
    4096-instance batch built with the set; rollout and [A_e B_e] are within the one-kernel tolerance of the oracle built with the set, and
    the gains of one expansion + backward pass within GAIN_TOL of it; the shared weights give other gains on those instances."""
    from oracle_binding import OracleProblem, match_algebra
    from parity_util import GAIN_TOL
    KERNEL_RTOL = 1e-10      # test_gpu_parity.py: one kernel against the oracle

    def close(a, b, rtol, what):
        scale = max(1.0, float(np.max(np.abs(b))))
        err = float(np.max(np.abs(a - b)))
        assert np.all(np.isfinite(a)) and err <= rtol * scale, f"{what}: max abs err {err:.3e} > {rtol:.0e} * {scale:.3e}"

    def with_set(j):
        def cls(model, obj, *a, **k):
            for ci, c in enumerate(obj._tables()[0]):
                s = _mild(c, j, ci)
                c.Q, c.R, c.c = s.Q, s.R, s.c
            return TO.Problem(model, obj, *a, **k)
        return cls

    def run(p):
        TO.rollout(p); TO.expand(p)
        X, ABe = TO.states(p), TO.error_dynamics(p)
        TO.backward(p)
        return X, ABe, TO.gains(p)

    S = 8
    g = problems.quadrotor(B=4096, N=101, error_state=True)
    assert TO.backward_algebra(g) == 1
    for ci, c in enumerate(g._cost_objs):
        TO.set_cost_weights(g, ci, np.stack([TO.api._cost_weight_row(_mild(c, b % S, ci)) for b in range(g.B)]))
    X, ABe, (Kg, dg) = run(g)
    U = TO.controls(g)
    t = TO.gettimes(g)
    for j in range(S):
        idx = np.arange(j, g.B, S)
        s = problems.quadrotor(B=4096, N=101, error_state=True, cls=with_set(j))
        Xs, ABes, (Ks, ds) = run(s)
        for name, a, ref in (("X", X, Xs), ("ABe", ABe, ABes), ("K", Kg, Ks), ("d", dg, ds)):
            assert np.array_equal(a[idx], ref[idx]), f"set {j}: {name} differs from the batch built with the set"
        s.close()
        obj = g.obj.copy()
        for ci, c in enumerate(obj._tables()[0]):
            m = _mild(c, j, ci)
            c.Q, c.R, c.c = m.Q, m.R, m.c
        o = OracleProblem(g.model, obj, g.x0[idx].copy(), float(t[-1]), xf=g.xf.copy(), constraints=g.constraints.copy(),
                          t0=float(t[0]), dt=g.spec.dt.copy(), error_state=True)
        match_algebra(g, o)
        TO.initial_controls(o, U[idx])
        TO.rollout(o)
        close(X[idx], TO.states(o), KERNEL_RTOL, f"set {j}: rollout X")
        TO.expand(o)
        close(ABe[idx], TO.error_dynamics(o), KERNEL_RTOL, f"set {j}: [A_e B_e]")
        TO.backward(o)
        Ko, do = TO.gains(o)
        close(Kg[idx], Ko, GAIN_TOL, f"set {j}: K"); close(dg[idx], do, GAIN_TOL, f"set {j}: d")
        o.close()
        if j == 1:   # the weights reach the gains: the oracle with the shared weights gives other gains on these instances
            o = OracleProblem(g.model, g.obj.copy(), g.x0[idx].copy(), float(t[-1]), xf=g.xf.copy(), constraints=g.constraints.copy(),
                              t0=float(t[0]), dt=g.spec.dt.copy(), error_state=True)
            match_algebra(g, o)
            TO.initial_controls(o, U[idx])
            TO.rollout(o); TO.expand(o); TO.backward(o)
            Ksh = TO.gains(o)[0]
            assert float(np.max(np.abs(Ksh - Kg[idx]))) > 1e3 * GAIN_TOL * max(1.0, float(np.max(np.abs(Ksh))))
            o.close()
    g.close()
