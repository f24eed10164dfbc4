"""A queue of problems that each bring their own rows of the per-instance tables (to_solve_queue_tables): time steps, cost weights,
constraint data, AL penalties and tracking references.

Central property: problem p's results are, bit for bit, what to_solve gives an instance that starts from the rows the setters write, in the
order to_set_time_steps, to_set_cost_weights, to_set_constraint_data, to_update_trajectories, to_set_goal_states, to_set_model_params,
to_set_penalties.  The reference is to_solve itself on fresh handles of the same B, loaded chunk by chunk with those setters in that order,
the last chunk padded with copies of its last problem.  Every comparison is np.array_equal."""
import ctypes as C

import numpy as np
import pytest

import trajopt_b200 as TO
from trajopt_b200 import _capi as K
from trajopt_b200 import problems
from test_gpu_solve_queue import _getters, _loaded

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(TO.Problem.__name__ == "OracleProblem", reason="the queue has no oracle counterpart")]

FIELDS = TO.SolveStats.FIELDS
CONSTRAINED = dict(iterations=80, cost_tolerance_intermediate=1e-2, constraint_tolerance=1e-3)


def _cartpole(B):
    p = problems.cartpole(B=B, N=51, u_bound=3.0, goal=True)
    TO.set_options(p, backward_kernel=1)
    return p


def _quadrotor_rec(B):
    return problems.quadrotor(B=B, N=51, error_state=True, u_noise=0.01)


def _quadrotor_full(B):
    return problems.quadrotor(B=B, N=51, u_noise=0.01)


def _quadrotor_quat(B):
    return problems.quadrotor_lie(B=B, N=51)


def _double_integrator(B):
    return problems.double_integrator(B=B, N=21, dim=2, constrained=False)


def _starts(make, M):
    """x0 and U0 of M problems: those of a batch of M built by the factory (its own random starts)"""
    src = make(M)
    x0, U0 = src.x0.copy(), TO.controls(src)
    src.close()
    return x0, U0


def _chunked(make, B, x0, U0, xf=None, objective=True, constraint=True, params=None, dt=None, cost_weights=None, constraint_data=None,
             penalties=None, Xref=None, Uref=None, start=1, **opts):
    """to_solve on fresh handles of B instances, chunk by chunk, each loaded with the setters in the order of the header: (stats [M], X, U)"""
    M = x0.shape[0]
    out = {f: [] for f in FIELDS}
    Xs, Us = [], []
    for c in range(0, M, B):
        idx = np.arange(c, c + B).clip(max=M - 1)        # the last chunk padded with its last problem
        p = make(B)
        if dt is not None:
            TO.set_time_steps(p, dt[idx])
        for j, rows in (cost_weights or {}).items():
            TO.set_cost_weights(p, j, [rows[i] for i in idx] if isinstance(rows, list) else rows[idx])
        for j, rows in (constraint_data or {}).items():
            TO.set_constraint_data(p, j, rows[idx])
        if Xref is not None:
            TO.update_trajectory(p, Xref[idx], Uref[idx], start)
        TO.set_initial_state(p, x0[idx])
        TO.initial_controls(p, U0[idx])
        if xf is not None:
            TO.set_goal_state(p, xf[idx], objective=objective, constraint=constraint)
        if params is not None:
            TO.set_model_params(p, params[idx])
        for i, mu in (penalties or {}).items():
            TO.set_penalties(p, i, mu[idx])
        st = TO.solve(p, **opts)
        k = min(B, M - c)
        for f in FIELDS:
            out[f].append(getattr(st, f)[:k])
        Xs.append(TO.states(p)[:k]); Us.append(TO.controls(p)[:k])
        p.close()
    return {f: np.concatenate(v) for f, v in out.items()}, np.concatenate(Xs), np.concatenate(Us)


def _check(make, B, x0, U0, **kw):
    """the queue on a handle of B slots against the chunked reference; returns the queue's result"""
    g = make(B)
    r = TO.solve_queue(g, x0, U0, **kw)
    g.close()
    ref, X, U = _chunked(make, B, x0, U0, **kw)
    for f in FIELDS:
        assert np.array_equal(getattr(r, f), ref[f]), f
    assert np.array_equal(r.X, X), "X"
    assert np.array_equal(r.U, U), "U"
    assert x0.shape[0] > B and len(np.unique(r.iterations)) > 1      # the slots were refilled mid-solve
    return r


def _scaled(row, M, k=4, step=0.1):
    return np.asarray(row)[None, :] * (1.0 + step * (np.arange(M) % k))[:, None]


def _bound_index(p):
    return next(i for i, c in enumerate(p.constraints) if isinstance(c, TO.BoundConstraint))


def _cartpole_tables(M):
    """per-problem tf (dt rows), control limits and penalties of the Cartpole with |u| <= 3 + Goal"""
    p = _cartpole(1)
    bi = _bound_index(p)
    d = np.tile(TO.constraint_data(p, bi)[0], (M, 1))
    lim = 3.0 - 0.25 * (np.arange(M) % 4)
    d[:, 4], d[:, 9] = lim, -lim                         # z_max | z_min of (x, u), the control at index n = 4
    mu = {i: 1.0 + (np.arange(M) % 3) * (1.0 + 9.0 * i) for i in range(len(p.constraints))}
    p.close()
    return dict(dt=(4.5 + 0.25 * (np.arange(M) % 4)) / 50, constraint_data={bi: d}, penalties=mu)


def test_cartpole_time_steps_limits_and_penalties():
    B, M = 16, 53
    x0, U0 = _starts(_cartpole, M)
    r = _check(_cartpole, B, x0, U0, **_cartpole_tables(M), **CONSTRAINED)
    assert r.iterations_outer.max() > 1


def test_quadrotor_record_path_weights_goals_bounds_and_time_steps():
    """per-problem weights with xf: each problem's q comes from its own weights"""
    B, M = 48, 149
    g = _quadrotor_rec(B)
    assert TO.kernel_choice(g)["backward"] == "fragment"
    w = TO.cost_weights(g, 0)[0]
    bi = _bound_index(g)
    d = np.tile(TO.constraint_data(g, bi)[0], (M, 1))
    d[:, 13:17] -= (np.arange(M) % 3)[:, None]          # the upper control bounds 10 -> 10, 9, 8
    g.close()
    x0, U0 = _starts(_quadrotor_rec, M)
    xf = np.tile([0, 0, 2, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0.0], (M, 1))
    xf[:, :3] += 0.2 * np.random.default_rng(3).uniform(-1, 1, (M, 3))
    _check(_quadrotor_rec, B, x0, U0, xf=xf, cost_weights={0: _scaled(w, M)}, constraint_data={bi: d}, dt=(4.0 + 0.5 * (np.arange(M) % 4)) / 50,
           iterations=60, cost_tolerance_intermediate=1e-2, constraint_tolerance=1e-3)


@pytest.mark.parametrize("make", [_quadrotor_full, _quadrotor_quat], ids=["full_state", "error_state_quat_cost"])
def test_closed_form_columns_follow_each_slots_time_steps(make):
    """B = 4 slots through M = 28 problems of 7 different time steps: each slot takes several, so stale closed-form Jacobian columns of a
    previous problem would show"""
    B, M = 4, 28
    g = make(B)
    assert TO.kernel_choice(g)["backward"] != "fragment"   # the closed-form columns live in [A B] / the materialised [A_e B_e]
    g.close()
    x0, U0 = _starts(make, M)
    _check(make, B, x0, U0, dt=(1.8 + 0.15 * (np.arange(M) % 7)) / 50, iterations=60, cost_tolerance_intermediate=1e-2, constraint_tolerance=1e-3)


def _reference(M, N, n, m, nref, seed=5):
    r = np.random.default_rng(seed)
    t = np.linspace(0.0, 1.0, nref)[None, :, None]
    Xref = t * r.uniform(-2, 2, (M, 1, n))
    Uref = 0.1 * r.standard_normal((M, nref, m))
    return Xref, Uref


def test_double_integrator_tracking_references():
    B, M = 16, 53
    x0, U0 = _starts(_double_integrator, M)
    Xref, Uref = _reference(M, 21, 4, 2, 24)
    _check(_double_integrator, B, x0, U0, Xref=Xref, Uref=Uref, start=3, iterations=40)


def _all_kinds(M):
    p = _cartpole(1)
    w0, w1 = TO.cost_weights(p, 0)[0], TO.cost_weights(p, 1)[0]
    p.close()
    Xref, Uref = _reference(M, 51, 4, 1, 51, seed=9)
    Xref[:, :, 1] += np.pi * np.linspace(0, 1, 51)[None, :]
    xf = np.tile([0, np.pi, 0, 0.0], (M, 1)); xf[:, 0] += 0.1 * (np.arange(M) % 5)
    return dict(**_cartpole_tables(M), cost_weights={0: _scaled(w0, M), 1: _scaled(w1, M, 3, 0.2)}, Xref=Xref, Uref=Uref, xf=xf,
                objective=False, **CONSTRAINED)


def test_all_kinds_at_once():
    B, M = 16, 53
    x0, U0 = _starts(_cartpole, M)
    _check(_cartpole, B, x0, U0, **_all_kinds(M))


def test_order_and_slot_count():
    """a permuted order gives permuted results, and B = 16 and B = 24 slots give the same results"""
    M = 60
    x0, U0 = _starts(_cartpole, M)
    kw = _all_kinds(M)
    g16, g24 = _cartpole(16), _cartpole(24)
    assert TO.kernel_choice(g16)["backward"] == TO.kernel_choice(g24)["backward"]
    a = TO.solve_queue(g16, x0, U0, **kw)
    perm = np.random.default_rng(7).permutation(M)
    pk = dict(kw, dt=kw["dt"][perm], xf=kw["xf"][perm], Xref=kw["Xref"][perm], Uref=kw["Uref"][perm],
              cost_weights={j: v[perm] for j, v in kw["cost_weights"].items()},
              constraint_data={j: v[perm] for j, v in kw["constraint_data"].items()}, penalties={j: v[perm] for j, v in kw["penalties"].items()})
    b = TO.solve_queue(g16, x0[perm], U0[perm], **pk)
    c = TO.solve_queue(g24, x0, U0, **kw)
    for f in FIELDS + ("X", "U"):
        assert np.array_equal(getattr(b, f), getattr(a, f)[perm]), f"permuted {f}"
        assert np.array_equal(getattr(c, f), getattr(a, f)), f"B = 24 {f}"
    g16.close(); g24.close()


def _tables_for(p, M):
    bi = _bound_index(p)
    d = np.tile(TO.constraint_data(p, bi)[0], (M, 1)); d[:, 13:17] -= (np.arange(M) % 3)[:, None]
    return dict(dt=(4.0 + 0.5 * (np.arange(M) % 4)) / 50, cost_weights={0: _scaled(TO.cost_weights(p, 0)[0], M)}, constraint_data={bi: d},
                penalties={i: 1.0 + np.arange(M) % (3 + i) for i in range(len(p.constraints))})


def test_handle_is_left_as_it_was():
    """every getter, and a later solve against an untouched twin; on the full-state Quadrotor the closed-form columns of [A B] too"""
    B, M = 16, 40
    g, twin = _loaded(B), _loaded(B)
    before = _getters(g)
    x0, U0 = _starts(_quadrotor_rec, M)
    opts = dict(iterations=60, cost_tolerance_intermediate=1e-2, constraint_tolerance=1e-3)
    params = np.asarray(g.model.params, dtype=float)[None, :] * (1.0 + 0.03 * (np.arange(M) % 5))[:, None]   # the handle's rows differ
    TO.solve_queue(g, x0, U0, params=params, **_tables_for(g, M), **opts)
    after = _getters(g)
    for k, v in before.items():
        assert np.array_equal(after[k], v), k
    sg, st = TO.solve(g, **opts), TO.solve(twin, **opts)
    for f in FIELDS:
        assert np.array_equal(getattr(sg, f), getattr(st, f)), f"solve after the queue: {f}"
    assert np.array_equal(TO.states(g), TO.states(twin)) and np.array_equal(TO.controls(g), TO.controls(twin))
    g.close(); twin.close()
    g, twin = _quadrotor_full(4), _quadrotor_full(4)
    x0, U0 = _starts(_quadrotor_full, 12)
    TO.solve_queue(g, x0, U0, dt=(1.8 + 0.15 * (np.arange(12) % 7)) / 50, iterations=20)
    for p in (g, twin):
        TO.rollout(p); TO.expand(p)
    assert np.array_equal(TO.dynamics_jacobians(g), TO.dynamics_jacobians(twin))
    sg, st = TO.solve(g, iterations=20), TO.solve(twin, iterations=20)
    for f in FIELDS:
        assert np.array_equal(getattr(sg, f), getattr(st, f)), f"full state, solve after the queue: {f}"
    g.close(); twin.close()


def test_handle_weights_that_differ_are_replaced():
    """a handle whose weights differ between instances queues weight rows for every weighted cost: accepted, and the results ignore the
    handle's rows"""
    B, M = 16, 40
    g = _cartpole(B)
    w = [TO.cost_weights(g, j) for j in range(2)]
    for j in range(2):
        TO.set_cost_weights(g, j, w[j] * (1.0 + 0.5 * (np.arange(B) % 2))[:, None])
    x0, U0 = _starts(_cartpole, M)
    cw = {j: _scaled(w[j][0], M) for j in range(2)}
    r = TO.solve_queue(g, x0, U0, cost_weights=cw, **CONSTRAINED)
    with pytest.raises(TO.ArgumentError, match="cost weights differ"):      # one cost's rows alone do not cover the other's
        TO.solve_queue(g, x0, U0, cost_weights={0: cw[0]}, **CONSTRAINED)
    g.close()
    ref, X, U = _chunked(_cartpole, B, x0, U0, cost_weights=cw, **CONSTRAINED)
    for f in FIELDS:
        assert np.array_equal(getattr(r, f), ref[f]), f
    assert np.array_equal(r.X, X) and np.array_equal(r.U, U)


def _raw(p, tables, M=4, xf=None, objective=1):
    """to_solve_queue_tables straight through the C ABI (past the Python checks): the return code and the handle's message"""
    x0 = np.ascontiguousarray(np.tile(p.x0[0], (M, 1)))
    U0 = np.ascontiguousarray(TO.controls(p)[0])
    xf = None if xf is None else np.ascontiguousarray(xf)
    spec = K.to_queue_spec(M, 1, K._dp(x0), K._dp(U0), K._dp(xf), objective, 1, None, 0, 0)
    keep = [(np.ascontiguousarray(a, dtype=np.float64), None if a2 is None else np.ascontiguousarray(a2, dtype=np.float64))
            for _, _, _, a, a2 in tables]
    arr = (K.to_queue_table * max(len(tables), 1))(*(K.to_queue_table(kind, index, ln, 0, K._dp(a), K._dp(a2))
                                                     for (kind, index, ln, _, _), (a, a2) in zip(tables, keep)))
    o = TO.solve_options(iterations=20)
    st = np.zeros(M, dtype=np.int32)
    rc = p._lib.to_solve_queue_tables(p._h, C.byref(spec), arr, len(tables), C.byref(o), K._ip(st), None, None, None, None, None, None, None,
                                      None)
    return rc, p._lib.to_last_error(p._h).decode()


def test_c_side_refusals_change_nothing():
    p = _cartpole(8)
    TO.rollout(p)
    M, K1, bi = 4, 50, _bound_index(p)
    gi = next(i for i, c in enumerate(p.constraints) if isinstance(c, TO.GoalConstraint))
    before = _getters(p)
    dt = np.full((M, K1), 0.1)
    w = np.tile(TO.cost_weights(p, 0)[0], (M, 1))
    d = np.tile(TO.constraint_data(p, bi)[0], (M, 1))
    mu = np.ones(M)
    X, U = np.zeros((M, 51, 4)), np.zeros((M, 51, 1))
    bad = lambda a, i, v: (lambda b: (b.__setitem__(i, v), b)[1])(a.copy())
    cases = [
        ([(K.QT_TIME_STEPS, 0, K1, bad(dt, (2, 7), 0.0), None)], K.TO_EINVAL, "problem 2, knot 7: a time step must be finite and positive"),
        ([(K.QT_TIME_STEPS, 0, K1 - 1, dt, None)], K.TO_EDIM, "len is 49"),
        ([(K.QT_COST_WEIGHTS, 0, w.shape[1], bad(w, (1, 2), np.nan), None)], K.TO_EINVAL, "problem 1, entry 2 is not finite"),
        ([(K.QT_CONSTRAINT_DATA, bi, d.shape[1], bad(d, (3, 4), -5.0), None)], K.TO_EINVAL, "problem 3, entry 4: Upper bounds"),
        ([(K.QT_CONSTRAINT_DATA, bi, d.shape[1], bad(d, (0, 0), 1.0), None)], K.TO_EINVAL, "problem 0, entry 0: BoundConstraint entries"),
        ([(K.QT_CONSTRAINT_DATA, gi, 4, np.zeros((M, 4)), None)], K.TO_EINVAL, "Goal constraint"),
        ([(K.QT_PENALTIES, 1, 1, bad(mu, 1, 0.0), None)], K.TO_EINVAL, "constraint 1: problem 1: a penalty must be finite and positive"),
        ([(K.QT_PENALTIES, 2, 1, mu, None)], K.TO_EINVAL, "no constraint 2"),
        ([(K.QT_PENALTIES, 0, 2, mu, None)], K.TO_EDIM, "len is 2"),
        ([(K.QT_REFERENCE, 1, 51, bad(X, (2, 7, 3), np.inf), U)], K.TO_EINVAL, "problem 2, row 7, entry 3: Xref is not finite"),
        ([(K.QT_REFERENCE, 3, 51, X, U)], K.TO_EDIM, "shorter than start + N - 1"),
        ([(K.QT_TIME_STEPS, 0, K1, dt, None), (K.QT_TIME_STEPS, 0, K1, dt, None)], K.TO_EINVAL, "the same table is given twice"),
        ([(K.QT_COST_WEIGHTS, 0, w.shape[1], w, None), (K.QT_COST_WEIGHTS, 0, w.shape[1], w, None)], K.TO_EINVAL, "given twice"),
        ([(7, 0, 1, dt, None)], K.TO_EINVAL, "unknown kind 7"),
    ]
    for tables, code, msg in cases:
        rc, err = _raw(p, tables)
        assert rc == code and msg in err, (msg, rc, err)
    rc, err = _raw(p, [(K.QT_REFERENCE, 1, 51, X, U)], xf=np.zeros((M, 4)))
    assert rc == K.TO_EINVAL and "a reference and xf with goal_objective = 1" in err
    after = _getters(p)
    for k, v in before.items():
        assert np.array_equal(after[k], v), k
    p.close()
    # penalties on an unconstrained problem
    q = _double_integrator(4)
    rc, err = _raw(q, [(K.QT_PENALTIES, 0, 1, np.ones(M), None)])
    assert rc == K.TO_EINVAL and "no constraint 0" in err
    q.close()


def test_cost_objects():
    """cost objects give their weights; set_cost_weights also writes their q and r, so the queue takes them only where xf or a reference
    replaces those terms, and refuses objects whose q or r would otherwise differ from the problem's"""
    B, M = 16, 40
    x0, U0 = _starts(_cartpole, M)
    xf0 = np.array([0, np.pi, 0, 0.0])
    objs = [TO.LQRCost(1e-2 * (1.0 + 0.25 * (p % 4)) * np.eye(4), 1e-1 * np.eye(1), xf0) for p in range(M)]
    xf = np.tile(xf0, (M, 1)); xf[:, 0] += 0.1 * (np.arange(M) % 5)
    _check(_cartpole, B, x0, U0, cost_weights={0: objs}, xf=xf, **CONSTRAINED)
    g = _cartpole(B)
    with pytest.raises(TO.ArgumentError, match="problem [01]: cost 0.s q differs from the problem.s linear terms"):
        TO.solve_queue(g, x0, U0, cost_weights={0: objs}, **CONSTRAINED)
    g.close()


def test_handle_rows_the_tables_replace_need_not_agree():
    """a handle whose Bound data, linear terms or penalties differ between instances: a table that replaces them is accepted, and the results
    ignore the handle's rows (the constraints a penalty table does not name keep the shared penalty, not the handle's rows)"""
    B, M = 16, 40
    g = _cartpole(B)
    bi = _bound_index(g)
    d = TO.constraint_data(g, bi); d[:, 4] -= 0.1 * (np.arange(B) % 3)
    TO.set_constraint_data(g, bi, d)
    TO.set_penalties(g, 1 - bi, 1.0 + np.arange(B) % 2)
    x0, U0 = _starts(_cartpole, M)
    kw = _cartpole_tables(M)
    kw["penalties"] = {bi: kw["penalties"][bi]}
    with pytest.raises(TO.ArgumentError, match="constraint data differ"):
        TO.solve_queue(g, x0, U0, penalties=kw["penalties"], **CONSTRAINED)
    r = TO.solve_queue(g, x0, U0, **kw, **CONSTRAINED)
    g.close()
    ref, X, U = _chunked(_cartpole, B, x0, U0, **kw, **CONSTRAINED)
    for f in FIELDS:
        assert np.array_equal(getattr(r, f), ref[f]), f"constraint data: {f}"
    assert np.array_equal(r.X, X) and np.array_equal(r.U, U)
    # linear terms that differ, replaced by a reference
    g = _double_integrator(B)
    Xh, Uh = _reference(B, 21, 4, 2, 24, seed=11)
    TO.update_trajectory(g, Xh, Uh, 2)
    x0, U0 = _starts(_double_integrator, M)
    Xref, Uref = _reference(M, 21, 4, 2, 24)
    with pytest.raises(TO.ArgumentError, match="linear cost terms differ"):
        TO.solve_queue(g, x0, U0, iterations=40)
    r = TO.solve_queue(g, x0, U0, Xref=Xref, Uref=Uref, start=3, iterations=40)
    g.close()
    ref, X, U = _chunked(_double_integrator, B, x0, U0, Xref=Xref, Uref=Uref, start=3, iterations=40)
    for f in FIELDS:
        assert np.array_equal(getattr(r, f), ref[f]), f"reference: {f}"
    assert np.array_equal(r.X, X) and np.array_equal(r.U, U)
