"""Per-instance constraint data (to_set_constraint_data): bounds, obstacles, collision radii, norm values, linear right-hand sides.

Central property: a batch whose instance b holds the data d[b % 3] computes, bit for bit, what instance b of a batch of the same size, x0 and
U0 built with d[b % 3] as its shared constraint data computes.  Same B on both sides, so that the same kernels are selected."""
import copy

import numpy as np
import pytest

import trajopt_b200 as TO
from trajopt_b200 import problems
from test_gpu_instance_params import PATHS as _PARAM_PATHS, _compare_pipeline, _assert_rows_equal, _snapshot, _param_sets

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(TO.Problem.__name__ == "OracleProblem", reason="per-instance constraint data has no oracle counterpart")]

G = 3


def _generic_spheres(B=48, cls=None, goal=False):
    """DoubleIntegrator(2) with a Sphere field on (x, y, vx), a Collision and a Linear constraint: the generic line search and general
    constraint rows (goal: and a Goal on the last knot)"""
    cls = cls or TO.Problem
    model = TO.DoubleIntegrator(2)
    n, m, N = 4, 2, 21
    xf = np.array([1.0, 2.0, 0, 0])
    obj = TO.LQRObjective(np.eye(n), 0.1 * np.eye(m), np.eye(n) * (N - 1), xf, N)
    cons = TO.ConstraintList(n, m, N)
    TO.add_constraint(cons, TO.SphereConstraint(n, [0.5, 1.2], [1.0, 1.4], [0.2, 0.3], [0.3, 0.25]), (2, N - 1))
    TO.add_constraint(cons, TO.CollisionConstraint(n, [1], [2], 0.1), (2, N - 1))
    TO.add_constraint(cons, TO.LinearConstraint(n, m, np.array([[1.0, 1.0]]), [6.0], TO.Inequality(), "control"), (1, N - 1))
    TO.add_constraint(cons, TO.BoundConstraint(n, m, u_min=-8, u_max=8), (1, N - 1))
    if goal:
        TO.add_constraint(cons, TO.GoalConstraint(xf), N)
    r = np.random.default_rng(3)
    p = cls(model, obj, np.zeros((B, n)), 3.0, xf=xf, constraints=cons)
    TO.initial_controls(p, 0.3 * r.standard_normal((B, N - 1, m)))
    return p


PATHS = dict(_PARAM_PATHS)
PATHS["double_integrator_spheres_generic"] = (lambda cls: _generic_spheres(48, cls), {})


def _data_indices(p):
    """the constraints whose data may differ per instance"""
    out = []
    for j, c in enumerate(p.constraints.constraints):
        try:
            TO.api._con_row(c)
        except TO.ArgumentError:
            continue
        out.append(j)
    return out


def _vary(con, rng):
    """data of a constraint of type(con) that really changes the problem, with the shape (and Bound's infinities) of con's"""
    _, row = TO.api._con_row(con)
    kind = con._spec(1, 1)["kind"]
    r = row.copy()
    fin = np.isfinite(r)
    if kind == TO._capi.CON_BOUND:   # additive, so that a zero bound (the Quadrotor's thrust floor) moves as well
        nm = r.size // 2
        while True:
            r = row.copy()
            r[fin] += rng.uniform(-0.2, 0.2, fin.sum()) * np.maximum(1.0, np.abs(row[fin]))
            if np.all(r[:nm] >= r[nm:]):
                return r
    if kind in (TO._capi.CON_CIRCLE, TO._capi.CON_SPHERE):
        p = con.p
        nc = 2 if kind == TO._capi.CON_CIRCLE else 3
        r[:nc * p] += rng.uniform(-0.2, 0.2, nc * p)
        r[nc * p:] *= 1.0 + rng.uniform(-0.2, 0.2, p)
        return r
    if kind == TO._capi.CON_LINEAR:
        return r + rng.uniform(-0.5, 0.5, r.size)
    return r * (1.0 + rng.uniform(-0.2, 0.2, r.size))      # NORM val, COLLISION radius


def _con_with(con, row):
    """a copy of con holding the data row (the layout of to_set_constraint_data)"""
    c = copy.copy(con)
    kind = con._spec(1, 1)["kind"]
    p = getattr(con, "p", 1)
    if kind == TO._capi.CON_BOUND:
        nm = row.size // 2
        c.z_max, c.z_min = row[:nm].copy(), row[nm:].copy()
    elif kind == TO._capi.CON_LINEAR:
        c.b = row.copy()
    elif kind == TO._capi.CON_CIRCLE:
        c.x, c.y, c.radius = row[:p].copy(), row[p:2 * p].copy(), row[2 * p:].copy()
    elif kind == TO._capi.CON_SPHERE:
        c.x, c.y, c.z, c.radius = row[:p].copy(), row[p:2 * p].copy(), row[2 * p:3 * p].copy(), row[3 * p:].copy()
    elif kind == TO._capi.CON_NORM:
        c.val = float(row[0])
    else:
        c.radius = float(row[0])
    return c


def _rebuilt(p, repl, opts):
    """the batch p with the constraints repl {index: constraint} in place of its own: same B, x0, controls, time grid and options"""
    cons = p.constraints.copy()
    for j, c in repl.items():
        cons.constraints[j] = c
    t = TO.gettimes(p)
    q = type(p)(p.model, p.obj.copy(), p.x0.copy(), float(t[-1]), xf=p.xf.copy(), constraints=cons, t0=float(t[0]), dt=p.spec.dt.copy(),
                error_state=p.error_state)
    if opts:
        TO.set_options(q, **opts)
    TO.initial_controls(q, TO.controls(p))
    return q


def _data_sets(p, seed=7, count=G):
    """count data sets {index: row} over every data-carrying constraint of p"""
    rng = np.random.default_rng(seed)
    return [{j: _vary(p.constraints.constraints[j], rng) for j in _data_indices(p)} for _ in range(count)]


def _per_and_shared(path, sets=None, seed=7):
    factory, opts = PATHS[path]
    per = factory(None)
    if opts:
        TO.set_options(per, **opts)
    sets = sets or _data_sets(per, seed)
    S = len(sets)
    cons = per.constraints.constraints
    shared = [_rebuilt(per, {j: _con_with(cons[j], row) for j, row in s.items()}, opts) for s in sets]
    for j in sets[0]:
        TO.set_constraint_data(per, j, np.stack([sets[b % S][j] for b in range(per.B)]))
    return per, shared, sets


@pytest.mark.parametrize("path", sorted(PATHS))
def test_instance_constraint_data_equal_shared_batches(path):
    per, shared, sets = _per_and_shared(path)
    assert sets[0], "the path has data-carrying constraints"
    for j in sets[0]:
        assert np.array_equal(TO.constraint_data(per, j), np.stack([sets[b % G][j] for b in range(per.B)]))
    # every constraint's Jacobians and second-order terms, as well
    TO.rollout(per)
    for s in shared:
        TO.rollout(s)
    for i in range(len(per.constraints)):
        for f in (TO.constraint_jacobians, TO.constraint_hessians):
            _assert_rows_equal({f.__name__: f(per, i)}, [{f.__name__: f(s, i)} for s in shared], f"{path} constraint {i}")
    _compare_pipeline(per, shared, path)
    for p in [per] + shared:
        p.close()


@pytest.mark.parametrize("path", sorted(PATHS))
def test_equal_rows_are_the_shared_path(path):
    """every row set to the shared data: the outputs of a batch that never called the setter; the same kernels but for the INST flags"""
    factory, opts = PATHS[path]
    per, plain = factory(None), factory(None)
    for p in (per, plain):
        if opts:
            TO.set_options(p, **opts)
    for j in _data_indices(per):
        TO.set_constraint_data(per, j, [per.constraints.constraints[j]] * per.B)
    kp, kq = TO.kernel_choice(per), TO.kernel_choice(plain)
    assert kp["inst_forward"] == 1 and kp["inst_backward"] == 1 and kq["inst_forward"] == 0 and kq["inst_backward"] == 0
    assert {k: v for k, v in kp.items() if not k.startswith("inst_")} == {k: v for k, v in kq.items() if not k.startswith("inst_")}
    _compare_pipeline(per, [plain], path, sets=1)
    per.close(); plain.close()


def test_with_instance_goals_and_params_on_the_record_path():
    path = "quadrotor_rec"
    factory, opts = PATHS[path]
    per = factory(None)
    dsets = _data_sets(per, seed=9)
    psets = _param_sets(per.model)
    rng = np.random.default_rng(5)
    goals = []
    for _ in range(G):
        g = np.array(per.xf, dtype=float); g[:3] += rng.uniform(-0.3, 0.3, 3); goals.append(g)
    cons = per.constraints.constraints
    shared = []
    for j in range(G):
        s = _rebuilt(per, {i: _con_with(cons[i], row) for i, row in dsets[j].items()}, opts)
        TO.set_model_params(s, np.tile(psets[j], (s.B, 1)))   # p[j] in every row: the shared parameters of that batch
        TO.set_goal_state(s, goals[j])
        shared.append(s)
    for i in dsets[0]:
        TO.set_constraint_data(per, i, np.stack([dsets[b % G][i] for b in range(per.B)]))
    TO.set_model_params(per, np.stack([psets[b % G] for b in range(per.B)]))
    TO.set_goal_state(per, np.stack([goals[b % G] for b in range(per.B)]))
    assert TO.backward_algebra(per) == 1
    _compare_pipeline(per, shared, "constraint data + params + goals")
    for p in [per] + shared:
        p.close()


def test_flagship_size_against_the_oracle():
    """BASELINE size, error-state Quadrotor 4096 x 101, 8 control boxes (b % 8, u_max in [8, 12], u_min in [-0.5, 0.5]): rollout and [A_e B_e]
    within the one-kernel tolerance of the oracle built with each box, the gains of one expansion + backward pass within GAIN_TOL.

    The box enters the gains only through its AL rows, and a row counts where lambda - mu c <= 0 (inequality multipliers are <= 0).  From the
    initial hover controls every row is inactive (c < 0), so the multipliers are drawn <= 0 and large enough that lambda - mu c straddles 0:
    which rows count, and their gradient lambda - mu c, then depend on each instance's box.  The oracle built with the shared box gives other
    gains: the test would see a kernel that read the shared box."""
    from oracle_binding import OracleProblem, match_algebra
    from parity_util import GAIN_TOL
    KERNEL_RTOL = 1e-10

    def err(a, b):
        return float(np.max(np.abs(a - b))), max(1.0, float(np.max(np.abs(b))))

    def close(a, b, rtol, what):
        e, scale = err(a, b)
        assert np.all(np.isfinite(a)) and e <= rtol * scale, f"{what}: max abs err {e:.3e} > {rtol:.0e} * {scale:.3e}"

    S = 8
    g = problems.quadrotor(B=4096, N=101, error_state=True)
    assert TO.backward_algebra(g) == 1
    n, m = g.n, g.m
    ci = next(j for j, c in enumerate(g.constraints.constraints) if isinstance(c, TO.BoundConstraint))
    box = g.constraints.constraints[ci]
    shared_row = TO.api._con_row(box)[1]
    nm = shared_row.size // 2
    assert np.all(np.isfinite(shared_row[n:nm])) and np.all(np.isfinite(shared_row[nm + n:])) and box.p == 2 * m   # rows: u_max | u_min
    rng = np.random.default_rng(2)
    rows = []
    for _ in range(S):
        r = shared_row.copy()
        r[n:nm] = rng.uniform(8.0, 12.0, m)
        r[nm + n:] = rng.uniform(-0.5, 0.5, m)
        rows.append(r)
    R = np.stack([rows[b % S] for b in range(g.B)])
    TO.set_constraint_data(g, ci, R)
    TO.rollout(g)
    U = TO.controls(g)
    mu = TO.penalty(g, ci)
    lam = TO.multipliers(g, ci)                                  # [B, N-1, 2m]: knot k+1 of the box acts on u_k
    lr = np.random.default_rng(4)
    lam[:, :, :m] = -mu * lr.uniform(6.0, 12.0, lam[:, :, :m].shape)       # upper rows: -mu c = mu (u_max - u) in about [6.5, 11]
    lam[:, :, m:] = -mu * lr.uniform(0.5, 2.0, lam[:, :, m:].shape)        # lower rows: -mu c = mu (u - u_min) in about [0.6, 1.8]
    lbar_u = lam[:, :, :m] - mu * (U - R[:, None, n:nm])
    lbar_l = lam[:, :, m:] - mu * (R[:, None, nm + n:] - U)
    for lb in (lbar_u, lbar_l):
        share = float(np.mean(lb <= 0.0))
        assert 0.1 < share < 0.9, f"{share:.2f} of the box rows active: the box data would not decide the active set"
    TO.set_multipliers(g, box, lam)
    TO.expand(g)
    X, ABe = TO.states(g), TO.error_dynamics(g)
    TO.backward(g)
    Kg, dg = TO.gains(g)
    t = TO.gettimes(g)

    def oracle(idx, row):
        cons = g.constraints.copy()
        cons.constraints[ci] = _con_with(box, row)
        o = OracleProblem(g.model, g.obj.copy(), g.x0[idx].copy(), float(t[-1]), xf=g.xf.copy(), constraints=cons,
                          t0=float(t[0]), dt=g.spec.dt.copy(), error_state=True)
        match_algebra(g, o)
        TO.initial_controls(o, U[idx])
        TO.set_multipliers(o, cons.constraints[ci], lam[idx])
        TO.rollout(o)
        return o

    for j in range(S):
        idx = np.arange(j, g.B, S)
        o = oracle(idx, rows[j])
        close(X[idx], TO.states(o), KERNEL_RTOL, f"set {j}: rollout X")
        TO.expand(o)
        close(ABe[idx], TO.error_dynamics(o), KERNEL_RTOL, f"set {j}: [A_e B_e]")
        TO.backward(o)
        Ko, do = TO.gains(o)
        close(Kg[idx], Ko, GAIN_TOL, f"set {j}: K"); close(dg[idx], do, GAIN_TOL, f"set {j}: d")
        o.close()
        if j == 0:   # sensitivity: the shared box gives other gains than the instance's
            o = oracle(idx, shared_row)
            TO.expand(o); TO.backward(o)
            Ks, ds = TO.gains(o)
            e, scale = err(dg[idx], ds)
            assert e > 1e3 * GAIN_TOL * scale, f"the gains do not depend on the box ({e:.3e})"
            o.close()
    g.close()


def test_solve_is_independent_of_the_batch_composition():
    from test_gpu_solve import subset
    build = lambda: _generic_spheres(48)
    g = build()
    sets = _data_sets(g, seed=13)
    rows = {j: np.stack([sets[b % G][j] for b in range(g.B)]) for j in sets[0]}
    for j, r in rows.items():
        TO.set_constraint_data(g, j, r)
    st = TO.solve(g)
    assert len(np.unique(st.iterations)) > 1
    idx = np.array([1, 7, 30, 47])
    q = subset(build(), idx)
    for j, r in rows.items():
        TO.set_constraint_data(q, j, r[idx])
    sq = TO.solve(q)
    for f in TO.SolveStats.FIELDS:
        assert np.array_equal(getattr(st, f)[idx], getattr(sq, f)), f
    assert np.array_equal(TO.states(g)[idx], TO.states(q))
    assert np.array_equal(TO.controls(g)[idx], TO.controls(q))
    g.close(); q.close()


def test_mpc_loop_with_moving_obstacles():
    """obstacles moved every step with set_constraint_data, next to shift_trajectory, against shared batches moved the same way"""
    path = "double_integrator_quickstart"
    per, shared, sets = _per_and_shared(path, seed=21)
    ci = next(j for j, c in enumerate(per.constraints.constraints) if isinstance(c, TO.CircleConstraint))
    for p in [per] + shared:
        TO.rollout(p); TO.ilqr_step(p, 2)
    for step in range(4):
        moved = [s[ci].copy() for s in sets]
        for s in moved:
            s[0] += 0.05 * (step + 1); s[1] -= 0.03 * (step + 1)
        for p in [per] + shared:
            TO.shift_trajectory(p, 1)
        TO.set_constraint_data(per, ci, np.stack([moved[b % G] for b in range(per.B)]))
        for j, s in enumerate(shared):
            TO.set_constraint_data(s, ci, np.tile(moved[j], (s.B, 1)))
        for p in [per] + shared:
            TO.rollout(p); TO.ilqr_step(p, 2)
        _assert_rows_equal(_snapshot(per), [_snapshot(s) for s in shared], f"MPC step {step}")
    for p in [per] + shared:
        p.close()


def test_rebuild_keeps_the_rows_and_an_in_place_change_wins():
    mk = lambda: problems.cartpole(B=12, N=31, u_bound=3.0)
    p = mk()
    ci = next(j for j, c in enumerate(p.constraints.constraints) if isinstance(c, TO.BoundConstraint))
    box = p.constraints.constraints[ci]
    sets = _data_sets(p, seed=3)
    rows = np.stack([sets[b % G][ci] for b in range(p.B)])
    TO.set_constraint_data(p, ci, rows)
    TO.add_constraint(p.constraints, TO.GoalConstraint(p.xf), p.N)       # live add_constraint!: the handle is rebuilt
    assert np.array_equal(TO.constraint_data(p, ci), rows)
    TO.rollout(p)
    X = TO.states(p)
    for j in range(G):
        s = mk()
        TO.add_constraint(s.constraints, TO.GoalConstraint(s.xf), s.N)
        TO.set_constraint_data(s, ci, np.tile(sets[j][ci], (s.B, 1)))
        TO.initial_controls(s, TO.controls(p))
        TO.rollout(s)
        Xs = TO.states(s)
        for b in range(j, p.B, G):
            assert np.array_equal(X[b], Xs[b]), f"instance {b} after the rebuild"
        s.close()
    # an in-place change to the constraint, picked up by the next rebuild, takes its new value in every instance
    box.z_max = box.z_max * 1.5; box.z_min = box.z_min * 1.5
    TO.add_constraint(p.constraints, TO.BoundConstraint(p.n, p.m, u_min=-100.0, u_max=100.0), (1, p.N - 1))
    assert np.array_equal(TO.constraint_data(p, ci), np.tile(TO.api._con_row(box)[1], (p.B, 1)))
    p.close()


def test_refusals_leave_the_table_as_it_was():
    p = _generic_spheres(4)
    lib, h, C = p._lib, p._h, TO._capi
    cons = p.constraints.constraints
    isph, icol, ilin, ibox = 0, 1, 2, 3
    import ctypes
    for j, want in [(isph, 8), (icol, 1), (ilin, 1), (ibox, 12)]:
        v = ctypes.c_int32(-1)
        assert lib.to_constraint_data_len(h, j, ctypes.byref(v)) == 0 and v.value == want
    before = {j: TO.constraint_data(p, j) for j in (isph, icol, ilin, ibox)}
    for j in before:
        assert np.array_equal(before[j], np.tile(TO.api._con_row(cons[j])[1], (4, 1)))     # the shared data broadcast
    rows = before[isph].copy(); rows[:, 6:] *= 1.2
    TO.set_constraint_data(p, isph, rows)
    before[isph] = rows

    def refused(j, r, words):
        assert lib.to_set_constraint_data(h, j, C._dp(np.ascontiguousarray(r))) == C.TO_EINVAL
        msg = lib.to_last_error(h).decode()
        assert all(w in msg for w in words), msg
        for k, v in before.items():
            assert np.array_equal(TO.constraint_data(p, k), v)

    r = before[ibox].copy(); r[2, 0] = 1.0                      # x_max[0] is +Inf in the shared bound
    refused(ibox, r, ["instance 2", "entry 0"])
    r = before[ibox].copy(); r[1, 4] = np.inf                   # u_max[0] is finite in the shared bound
    refused(ibox, r, ["instance 1", "entry 4"])
    r = before[ibox].copy(); r[3, 5] = -9.0                     # u_max[1] < u_min[1]
    refused(ibox, r, ["instance 3", "entry 5", "greater than or equal"])
    r = before[isph].copy(); r[0, 3] = np.nan
    refused(isph, r, ["instance 0", "entry 3", "not finite"])
    r = before[icol].copy(); r[2, 0] = np.inf
    refused(icol, r, ["instance 2", "not finite"])
    assert lib.to_set_constraint_data(h, 99, C._dp(before[icol])) == C.TO_EINVAL
    assert lib.to_set_constraint_data(h, ilin, None) == C.TO_EINVAL
    with pytest.raises(TO.ArgumentError):
        TO.set_constraint_data(p, ibox, np.where(np.isinf(before[ibox]), 0.0, before[ibox]))
    with pytest.raises(TO.DimensionMismatch):
        TO.set_constraint_data(p, isph, before[isph][:, :-1])
    for k, v in before.items():
        assert np.array_equal(TO.constraint_data(p, k), v)
    p.close()
    # NormConstraint val < 0, Goal, QuatVecEq and a refused first call (no table afterwards)
    q = _PARAM_PATHS["double_integrator_quickstart"][0](None)
    inorm = next(j for j, c in enumerate(q.constraints.constraints) if isinstance(c, TO.NormConstraint))
    igoal = next(j for j, c in enumerate(q.constraints.constraints) if isinstance(c, TO.GoalConstraint))
    r = TO.constraint_data(q, inorm); r[5, 0] = -1.0
    assert q._lib.to_set_constraint_data(q._h, inorm, C._dp(r)) == C.TO_EINVAL
    assert "non-negative" in q._lib.to_last_error(q._h).decode()
    assert q._lib.to_set_constraint_data(q._h, igoal, C._dp(np.zeros((q.B, 4)))) == C.TO_EINVAL
    assert TO.kernel_choice(q)["inst_forward"] == 0 and TO.kernel_choice(q)["inst_backward"] == 0
    q.close()
    lie = problems.quadrotor_lie(B=4, N=11)
    iq = next((j for j, c in enumerate(lie.constraints.constraints) if isinstance(c, TO.QuatVecEq)), None)
    if iq is not None:
        assert lie._lib.to_set_constraint_data(lie._h, iq, C._dp(np.zeros((4, 4)))) == C.TO_EINVAL
    lie.close()


# a Goal next to data-carrying constraints, on the record path (ExpTab) and on the generic path
GOAL_PATHS = {"quadrotor_rec": PATHS["quadrotor_rec"],
              "double_integrator_spheres_generic": (lambda cls: _generic_spheres(48, cls, goal=True), {})}


def _goals(p, seed):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(G):
        g = np.array(p.xf, dtype=float); g[:2] += rng.uniform(-0.3, 0.3, 2); out.append(g)
    return out


@pytest.mark.parametrize("path", sorted(GOAL_PATHS))
def test_shared_goal_after_instance_data(path):
    """per-instance data on every data-carrying constraint, then a shared set_goal_state: every instance goes to the new goal, and keeps its data.
    objective=False: a new goal for the cost objects would rebuild the handle from them (set_LQR_goal!), this one reaches the handle as it is"""
    factory, opts = GOAL_PATHS[path]
    per = factory(None)
    if opts:
        TO.set_options(per, **opts)
    sets = _data_sets(per, seed=17)
    cons = per.constraints.constraints
    igoal = next(j for j, c in enumerate(cons) if isinstance(c, TO.GoalConstraint))
    g = _goals(per, 19)[0]
    shared = []
    for s in sets:   # each with a Goal object of its own: set_goal_state assigns its xf
        q = _rebuilt(per, {igoal: copy.copy(cons[igoal]), **{j: _con_with(cons[j], row) for j, row in s.items()}}, opts)
        TO.set_goal_state(q, g, objective=False)
        shared.append(q)
    for j in sets[0]:
        TO.set_constraint_data(per, j, np.stack([sets[b % G][j] for b in range(per.B)]))
    TO.set_goal_state(per, g, objective=False)
    assert np.array_equal(TO.constraint_data(per, igoal), np.tile(cons[igoal].xf, (per.B, 1)))
    _compare_pipeline(per, shared, f"{path}: instance data, then a shared goal")
    for p in [per] + shared:
        p.close()


@pytest.mark.parametrize("path", sorted(GOAL_PATHS))
def test_instance_goal_values_then_bound_data(path):
    """per-instance Goal values, then per-instance Bound data: the Bound call keeps the Goal rows"""
    factory, opts = GOAL_PATHS[path]
    per = factory(None)
    if opts:
        TO.set_options(per, **opts)
    cons = per.constraints.constraints
    igoal = next(j for j, c in enumerate(cons) if isinstance(c, TO.GoalConstraint))
    ibox = next(j for j, c in enumerate(cons) if isinstance(c, TO.BoundConstraint))
    goal = cons[igoal]
    vals = [g[goal.inds - 1] for g in _goals(per, 23)]
    boxes = [s[ibox] for s in _data_sets(per, seed=29)]
    shared = []
    for j in range(G):
        gc = copy.copy(goal); gc.xf = vals[j].copy()
        shared.append(_rebuilt(per, {igoal: gc, ibox: _con_with(cons[ibox], boxes[j])}, opts))
    TO.set_constraint_data(per, igoal, np.stack([vals[b % G] for b in range(per.B)]))
    TO.set_constraint_data(per, ibox, np.stack([boxes[b % G] for b in range(per.B)]))
    assert np.array_equal(TO.constraint_data(per, igoal), np.stack([vals[b % G] for b in range(per.B)]))
    _compare_pipeline(per, shared, f"{path}: instance Goal values, then instance Bound data")
    for p in [per] + shared:
        p.close()


def test_goal_routes_to_the_goal_values():
    p = _PARAM_PATHS["double_integrator_quickstart"][0](None)
    igoal = next(j for j, c in enumerate(p.constraints.constraints) if isinstance(c, TO.GoalConstraint))
    goal = p.constraints.constraints[igoal]
    rows = np.tile(goal.xf, (p.B, 1)); rows[:, 1] += np.linspace(-0.5, 0.5, p.B)
    TO.set_constraint_data(p, goal, rows)
    assert np.array_equal(TO.constraint_data(p, goal), rows)
    vals = np.empty((p.B, goal.p))
    p._call("to_get_goal_values", igoal, TO._capi._dp(vals))
    assert np.array_equal(vals, rows)
    p.close()


def test_hybrid_problem_refuses():
    from dynamics_programs import builtin_problem
    p = builtin_problem("cartpole", TO.Problem, 4, recorded=True)
    with pytest.raises(TO.ArgumentError):
        TO.set_constraint_data(p, 0, np.ones((4, 1)))
    for j in range(len(p.constraints)):
        assert p._lib.to_set_constraint_data(p._h, j, TO._capi._dp(np.ones((4, 64)))) == TO._capi.TO_EINVAL
    p.close()
