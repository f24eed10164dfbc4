"""Per-instance model parameters (to_set_model_params).

Central property: a batch whose instance b integrates with the parameters p[b % 3] computes, bit for bit, what instance b of a batch of the
same size, x0 and U0 built with the model of p[b % 3] computes.  Same B on both sides, so that the same kernels are selected."""
import numpy as np
import pytest

import trajopt_b200 as TO
from trajopt_b200 import problems

pytestmark = pytest.mark.gpu

G = 3


def _param_sets(model, count=G, seed=11, spread=0.2):
    """parameter vectors that really change the dynamics: Quadrotor mass, J and km; Cartpole mp and l; Acrobot masses; DoubleIntegrator mass"""
    rng = np.random.default_rng(seed)
    base = np.array(model.params, dtype=float)
    idx = {TO.Quadrotor: [0, 1, 2, 3, 9], TO.Cartpole: [1, 2], TO.Acrobot: [2, 3], TO.DoubleIntegrator: [0]}[type(model)]
    out = []
    for _ in range(count):
        p = base.copy()
        p[idx] *= 1.0 + rng.uniform(-spread, spread, len(idx))
        out.append(p)
    return out


def _model_of(model, p):
    """a model of type(model) with the parameter vector p"""
    m = type(model)(model.m) if isinstance(model, TO.DoubleIntegrator) else type(model)()
    m.params = [float(v) for v in p]
    return m


def _with_model(mdl):
    """a `cls` for the problem builders: the problem is built with the model `mdl` instead of the builder's own"""
    return lambda model, *a, **k: TO.Problem(mdl, *a, **k)


def _snapshot(p):
    s = dict(cost=TO.cost(p), cost_knots=TO.cost_knots(p), cost_gradient=TO.cost_gradient(p), merit=TO.merit(p),
             max_violation=TO.max_violation(p), X=TO.states(p), U=TO.controls(p))
    for i in range(len(p.constraints)):
        s[f"eval_constraints{i}"] = TO.evaluate_constraints(p, i)
        s[f"multipliers{i}"] = TO.multipliers(p, i)
    return s


def _assert_rows_equal(per, shared, what, sets=G):
    for key, v in per.items():
        for b in range(v.shape[0]):
            ref = shared[b % sets][key][b]
            assert np.array_equal(v[b], ref, equal_nan=True), f"{what}: {key} of instance {b} differs from the shared-parameter batch"


def _quickstart(B=48, cls=None):
    """examples/quickstart.jl, batched: DoubleIntegrator(2), Goal + Circle + SOC norm + bounds (the generic line search)"""
    cls = cls or TO.Problem
    model = TO.DoubleIntegrator(2)
    n, m, N = 4, 2, 21
    xf = np.array([0, 2.0, 0, 0])
    obj = TO.LQRObjective(np.eye(n), np.eye(m), np.eye(n) * (N - 1), xf, N)
    cons = TO.ConstraintList(n, m, N)
    TO.add_constraint(cons, TO.GoalConstraint(xf), N)
    TO.add_constraint(cons, TO.CircleConstraint(n, [0.0], [1.0], [0.5]), (2, N - 1))
    TO.add_constraint(cons, TO.NormConstraint(n, m, 5.0, TO.SecondOrderCone(), "control"), (1, N - 1))
    TO.add_constraint(cons, TO.BoundConstraint(n, m, u_min=-10, u_max=10), (1, N - 1))
    r = np.random.default_rng(1)
    p = cls(model, obj, np.zeros((B, n)), 3.0, xf=xf, constraints=cons)
    TO.initial_controls(p, r.standard_normal((B, N - 1, m)))
    return p


PATHS = {
    # the paths of test_gpu_instance_goals.py
    "quadrotor_full": (lambda cls: problems.quadrotor(B=48, N=31, dt=0.05, cls=cls), {}),
    "cartpole_warp": (lambda cls: problems.cartpole(B=48, N=51, u_bound=3.0, goal=True, cls=cls), dict(backward_kernel=1)),
    "cartpole_thread": (lambda cls: problems.cartpole(B=48, N=51, u_bound=3.0, goal=True, cls=cls), dict(backward_kernel=2)),
    "acrobot_dense": (lambda cls: problems.acrobot(B=48, N=41, cls=cls), {}),
    "quadrotor_rec": (lambda cls: problems.quadrotor(B=48, N=31, error_state=True, cls=cls), {}),
    "quadrotor_compact": (lambda cls: problems.quadrotor(B=48, N=31, error_state=True, cls=cls), dict(backward_kernel=5)),
    "quadrotor_dense_lie": (lambda cls: problems.quadrotor(B=48, N=31, error_state=True, cls=cls), dict(backward_kernel=3)),
    "quadrotor_lie": (lambda cls: problems.quadrotor_lie(B=48, N=31, cls=cls), {}),
    # the quickstart problem: generic line search, general constraints
    "double_integrator_quickstart": (lambda cls: _quickstart(48, cls), {}),
}


def _make(factory, opts, mdl=None):
    p = factory(_with_model(mdl) if mdl is not None else None)
    if opts:
        TO.set_options(p, **opts)
    return p


def _compare_pipeline(per, shared, what, sets=G):
    """rollout, Jacobians, records, gains, 3 iLQR iterations and a solve of `per` against the shared batches, row by row"""
    probs = [per] + shared
    for p in probs:
        TO.rollout(p)
    _assert_rows_equal(_snapshot(per), [_snapshot(s) for s in shared], f"{what} after rollout", sets)
    for p in probs:
        TO.expand(p)
    jac = lambda p: dict(AB=TO.dynamics_jacobians(p), **({"ABe": TO.error_dynamics(p)} if p.error_state else {}))
    _assert_rows_equal(jac(per), [jac(s) for s in shared], f"{what} Jacobians", sets)
    for p in probs:
        TO.backward(p)
    if TO.backward_algebra(per) == 1:   # record path: the records the Riccati kernel read
        _assert_rows_equal({"records": TO.expansion_records(per)}, [{"records": TO.expansion_records(s)} for s in shared], f"{what} records", sets)
    K, Ks = TO.gains(per), [TO.gains(s) for s in shared]
    for b in range(per.B):
        for a, ref in zip(K, Ks[b % sets]):
            assert np.array_equal(a[b], ref[b]), f"{what}: gains of instance {b}"
    for p in probs:
        TO.ilqr_step(p, 3)
    _assert_rows_equal(_snapshot(per), [_snapshot(s) for s in shared], f"{what} after ilqr_step(3)", sets)
    stats = [TO.solve(p, iterations=40) for p in probs]
    for f in TO.SolveStats.FIELDS:
        v = getattr(stats[0], f)
        for b in range(per.B):
            assert np.array_equal(v[b], getattr(stats[1 + b % sets], f)[b]), f"{what}: solve {f} of instance {b}"
    # the merit after to_solve is taken at the batch's last penalties (a batch-level quantity, test_gpu_instance_goals.py)
    snap = lambda p: {k: v for k, v in _snapshot(p).items() if k != "merit"}
    _assert_rows_equal(snap(per), [snap(s) for s in shared], f"{what} after solve", sets)


@pytest.mark.parametrize("path", sorted(PATHS))
def test_instance_params_equal_shared_batches(path):
    factory, opts = PATHS[path]
    per = _make(factory, opts)
    sets = _param_sets(per.model)
    TO.set_model_params(per, np.stack([sets[b % G] for b in range(per.B)]))
    shared = [_make(factory, opts, _model_of(per.model, sets[j])) for j in range(G)]
    assert np.array_equal(TO.model_params(per), np.stack([sets[b % G] for b in range(per.B)]))
    _compare_pipeline(per, shared, path)
    for p in [per] + shared:
        p.close()


@pytest.mark.parametrize("path", sorted(PATHS))
def test_equal_rows_are_the_shared_path(path):
    """every row set to the shared parameters: the outputs of a batch that never called the setter"""
    factory, opts = PATHS[path]
    per, plain = _make(factory, opts), _make(factory, opts)
    TO.set_model_params(per, [per.model] * per.B)
    _compare_pipeline(per, [plain], path, sets=1)
    per.close(); plain.close()


def test_with_instance_goals_on_the_record_path():
    factory, opts = PATHS["quadrotor_rec"]
    per = _make(factory, opts)
    sets = _param_sets(per.model)
    rng = np.random.default_rng(5)
    goals = []
    for _ in range(G):
        g = np.array(per.xf, dtype=float); g[:3] += rng.uniform(-0.3, 0.3, 3); goals.append(g)
    TO.set_model_params(per, np.stack([sets[b % G] for b in range(per.B)]))
    TO.set_goal_state(per, np.stack([goals[b % G] for b in range(per.B)]))
    shared = []
    for j in range(G):
        s = _make(factory, opts, _model_of(per.model, sets[j]))
        TO.set_goal_state(s, goals[j])
        shared.append(s)
    assert TO.backward_algebra(per) == 1
    _compare_pipeline(per, shared, "params + goals")
    for p in [per] + shared:
        p.close()


def test_flagship_size_against_the_oracle():
    """BASELINE size, error-state Quadrotor 4096 x 101, 8 parameter sets (b % 8, mass and J within +-20 %): rollout and [A_e B_e] within the
    one-kernel tolerance of the oracle built with each set, the gains of one expansion + backward pass within GAIN_TOL"""
    from oracle_binding import OracleProblem, match_algebra
    from parity_util import GAIN_TOL
    KERNEL_RTOL = 1e-10      # test_gpu_parity.py: one kernel against the oracle

    def close(a, b, rtol, what):
        scale = max(1.0, float(np.max(np.abs(b))))
        err = float(np.max(np.abs(a - b)))
        assert np.all(np.isfinite(a)) and err <= rtol * scale, f"{what}: max abs err {err:.3e} > {rtol:.0e} * {scale:.3e}"

    S = 8
    g = problems.quadrotor(B=4096, N=101, error_state=True)
    assert TO.backward_algebra(g) == 1
    rng = np.random.default_rng(2)
    sets = []
    for _ in range(S):
        p = np.array(g.model.params, dtype=float); p[:4] *= 1.0 + rng.uniform(-0.2, 0.2, 4); sets.append(p)
    TO.set_model_params(g, np.stack([sets[b % S] for b in range(g.B)]))
    TO.rollout(g); TO.expand(g)
    X, ABe = TO.states(g), TO.error_dynamics(g)
    TO.backward(g)
    Kg, dg = TO.gains(g)
    U = TO.controls(g)
    t = TO.gettimes(g)
    for j in range(S):
        idx = np.arange(j, g.B, S)
        mdl = _model_of(g.model, sets[j])
        o = OracleProblem(mdl, g.obj.copy(), g.x0[idx].copy(), float(t[-1]), xf=g.xf.copy(), constraints=g.constraints.copy(),
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
    g.close()


def test_solve_is_independent_of_the_batch_composition():
    from test_gpu_solve import subset
    build = lambda: problems.quadrotor(B=48, N=51, error_state=True)
    g = build()
    sets = _param_sets(g.model)
    rows = np.stack([sets[b % G] for b in range(g.B)])
    TO.set_model_params(g, rows)
    st = TO.solve(g)
    assert len(np.unique(st.iterations)) > 1
    idx = np.array([1, 7, 30, 47])
    q = subset(build(), idx)
    TO.set_model_params(q, rows[idx])
    sq = TO.solve(q)
    for f in TO.SolveStats.FIELDS:
        assert np.array_equal(getattr(st, f)[idx], getattr(sq, f)), f
    assert np.array_equal(TO.states(g)[idx], TO.states(q))
    assert np.array_equal(TO.controls(g)[idx], TO.controls(q))
    Kg, dg = TO.gains(g); Kq, dq = TO.gains(q)
    assert np.array_equal(Kg[idx], Kq) and np.array_equal(dg[idx], dq)
    g.close(); q.close()


def test_rebuild_keeps_the_rows():
    mk = lambda: problems.cartpole(B=12, N=31, u_bound=3.0)
    p = mk()
    sets = _param_sets(p.model)
    rows = np.stack([sets[b % G] for b in range(p.B)])
    TO.set_model_params(p, rows)
    TO.add_constraint(p.constraints, TO.GoalConstraint(p.xf), p.N)       # live add_constraint!: the handle is rebuilt
    assert np.array_equal(TO.model_params(p), rows)
    TO.rollout(p)
    X = TO.states(p)
    ref = [mk() for _ in range(G)]
    for j, s in enumerate(ref):
        TO.set_model_params(s, np.tile(sets[j], (s.B, 1)))
        TO.initial_controls(s, TO.controls(p))
        TO.rollout(s)
        Xs = TO.states(s)
        for b in range(j, p.B, G):
            assert np.array_equal(X[b], Xs[b]), f"instance {b} after the rebuild"
        s.close()
    p.close()


def test_refusals_leave_the_rows_as_they_were():
    p = problems.quadrotor(B=4, N=11, dt=0.05)
    lib, h, C = p._lib, p._h, TO._capi
    base = TO.model_params(p)
    assert np.array_equal(base, np.tile(p.model.params, (4, 1)))          # the shared values broadcast
    rows = base.copy(); rows[:, 0] *= 1.1
    TO.set_model_params(p, rows)
    for bad, code, words in [(("nan", 2, 5), C.TO_EINVAL, "instance 2, parameter 5"), (("inf", 1, 9), C.TO_EINVAL, "instance 1, parameter 9"),
                             ((0.0, 3, 0), C.TO_EINVAL, "mass"), ((-1e-3, 0, 2), C.TO_EINVAL, "J2")]:
        val, b, i = bad
        r = rows.copy(); r[b, i] = float(val)
        assert lib.to_set_model_params(h, C._dp(np.ascontiguousarray(r)), 10) == code
        msg = lib.to_last_error(h).decode()
        assert words in msg and f"instance {b}" in msg, msg
        assert np.array_equal(TO.model_params(p), rows)
    assert lib.to_set_model_params(h, C._dp(np.ascontiguousarray(rows)), 9) == C.TO_EDIM
    assert lib.to_set_model_params(h, None, 10) == C.TO_EINVAL
    assert np.array_equal(TO.model_params(p), rows)
    p.close()
    # a refused first call creates no rows: the shared values still broadcast
    c = problems.cartpole(B=3, N=11)
    r = np.tile(c.model.params, (3, 1)); r[1, 2] = 0.0                      # l
    assert c._lib.to_set_model_params(c._h, C._dp(r), 4) == C.TO_EINVAL
    assert np.array_equal(TO.model_params(c), np.tile(c.model.params, (3, 1)))
    a = problems.acrobot(B=2, N=11)
    r = np.tile(a.model.params, (2, 1)); r[0, 3] = -1.0                     # m2
    assert a._lib.to_set_model_params(a._h, C._dp(r), 8) == C.TO_EINVAL
    d = problems.double_integrator(B=2, N=11)
    assert d._lib.to_set_model_params(d._h, C._dp(np.array([[1.0], [0.0]])), 1) == C.TO_EINVAL
    for q in (c, a, d):
        q.close()


def test_hybrid_problem_refuses():
    from dynamics_programs import builtin_problem
    p = builtin_problem("cartpole", TO.Problem, 4, recorded=True)
    with pytest.raises(TO.ArgumentError):
        TO.set_model_params(p, np.ones((4, 4)))
    assert p._lib.to_set_model_params(p._h, TO._capi._dp(np.ones((4, 4))), 4) == TO._capi.TO_EINVAL
    p.close()
