"""Per-instance time steps and initial times (to_set_time_steps).

Central property: a batch whose instance b holds the grid GRIDS[b % 3] = (t0_j, dt_j) computes, bit for bit, what instance b of a batch of
the same size, x0 and U0 built with Problem(..., tf_j; t0 = t0_j, dt = dt_j) computes.  Same B on both sides, so that the same kernels are
selected."""
import numpy as np
import pytest

import trajopt_b200 as TO
from trajopt_b200 import problems
from test_gpu_instance_params import PATHS, G, _assert_rows_equal, _compare_pipeline, _model_of, _param_sets, _snapshot
from test_gpu_solve import subset

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(TO.Problem.__name__ == "OracleProblem", reason="per-instance time steps have no oracle counterpart")]


def _grids(p, seed=3):
    """three grids (t0_j, dt_j) around the problem's own horizon tf: uniform with 0.9 tf; the reference's uneven steps
    (test/problems_tests.jl:79-81: N/2 steps of 1 then steps of 0.5, scaled to the horizon) over tf; steps drawn in [0.5, 1.5] over 1.1 tf"""
    N, tf = p.N, float(TO.gettimes(p)[-1] - TO.gettimes(p)[0])
    uneven = np.concatenate([np.full(N // 2, 1.0), np.full(N - N // 2 - 1, 0.5)])
    drawn = np.random.default_rng(seed).uniform(0.5, 1.5, N - 1)
    return [(0.0, np.full(N - 1, 0.9 * tf / (N - 1))),
            (1.5, uneven * (tf / uneven.sum())),
            (-0.25, drawn * (1.1 * tf / drawn.sum()))]


def _with_grid(grid, mdl=None):
    """a `cls` for the problem builders: the problem is built with the grid (t0, dt) instead of the builder's horizon (and with `mdl`)"""
    t0, dt = grid
    return lambda model, obj, x0, tf, **k: TO.Problem(mdl if mdl is not None else model, obj, x0, t0 + float(np.sum(dt)),
                                                      **{**k, "t0": t0, "dt": dt.copy()})


def _make(factory, opts, grid=None, mdl=None):
    p = factory(_with_grid(grid, mdl) if grid is not None else None)
    if opts:
        TO.set_options(p, **opts)
    return p


def _rows(grids, B, sets=G):
    return np.stack([grids[b % sets][1] for b in range(B)]), np.array([grids[b % sets][0] for b in range(B)])


@pytest.mark.parametrize("path", sorted(PATHS))
def test_instance_grids_equal_shared_batches(path):
    factory, opts = PATHS[path]
    per = _make(factory, opts)
    grids = _grids(per)
    dt, t0 = _rows(grids, per.B)
    TO.set_time_steps(per, dt, t0)
    got_dt, got_t0 = TO.time_steps(per)
    assert np.array_equal(got_dt, dt) and np.array_equal(got_t0, t0)
    shared = [_make(factory, opts, grids[j]) for j in range(G)]
    for b in range(per.B):
        assert np.array_equal(TO.instance_times(per)[b], TO.gettimes(shared[b % G]))
    # a table the kernels ignored would give every instance the untouched batch's trajectory: the drawn grid does not
    plain = _make(factory, opts)
    TO.rollout(plain); TO.rollout(shared[2])
    assert not np.array_equal(TO.states(plain)[2::G], TO.states(shared[2])[2::G]), f"{path}: the drawn grid changes no instance"
    assert np.array_equal(TO.gettimes(per), TO.gettimes(plain))          # the shared grid stays what the spec holds
    plain.close()
    _compare_pipeline(per, shared, path)
    for p in [per] + shared:
        p.close()


@pytest.mark.parametrize("path", sorted(PATHS))
def test_equal_rows_are_the_shared_path(path):
    """every row set to the shared grid: the outputs of a batch that never called the setter"""
    factory, opts = PATHS[path]
    per, plain = _make(factory, opts), _make(factory, opts)
    t = TO.gettimes(per)
    TO.set_time_steps(per, np.tile(per.spec.dt, (per.B, 1)), np.full(per.B, t[0]))
    assert TO.kernel_choice(per)["inst_forward"] == 1
    _compare_pipeline(per, [plain], path, sets=1)
    per.close(); plain.close()


def test_uniform_form_is_a_batch_built_with_tf():
    """dt[B] with dt_b = tf_b / (N - 1): the batch built with Problem(..., tf_b) and no dt"""
    factory, opts = PATHS["quadrotor_rec"]
    per = _make(factory, opts)
    N = per.N
    tfs = [4.5, 5.0, 5.5]
    TO.set_time_steps(per, np.array([tfs[b % G] / (N - 1) for b in range(per.B)]))
    shared = [factory(lambda model, obj, x0, tf, _t=tfs[j], **k: TO.Problem(model, obj, x0, _t, **k)) for j in range(G)]
    _compare_pipeline(per, shared, "uniform steps")
    for p in [per] + shared:
        p.close()


def test_with_instance_goals_and_params_on_the_record_path():
    factory, opts = PATHS["quadrotor_rec"]
    per = _make(factory, opts)
    grids, sets = _grids(per), _param_sets(per.model)
    rng = np.random.default_rng(5)
    goals = []
    for _ in range(G):
        g = np.array(per.xf, dtype=float); g[:3] += rng.uniform(-0.3, 0.3, 3); goals.append(g)
    TO.set_time_steps(per, *_rows(grids, per.B))
    TO.set_model_params(per, np.stack([sets[b % G] for b in range(per.B)]))
    TO.set_goal_state(per, np.stack([goals[b % G] for b in range(per.B)]))
    shared = []
    for j in range(G):
        s = _make(factory, opts, grids[j], _model_of(per.model, sets[j]))
        TO.set_goal_state(s, goals[j])
        shared.append(s)
    assert TO.backward_algebra(per) == 1
    _compare_pipeline(per, shared, "time steps + params + goals")
    for p in [per] + shared:
        p.close()


def test_mpc_shift_moves_each_clock():
    """shift_trajectory advances each instance's clock by its own skipped steps (the rows stay): instance_times = each shared batch's
    gettimes after the same shift, and the warm-started rollout after a new initial state is the shared batch's, bit for bit"""
    factory, opts = PATHS["quadrotor_rec"]
    per = _make(factory, opts)
    grids = _grids(per)
    TO.set_time_steps(per, *_rows(grids, per.B))
    shared = [_make(factory, opts, grids[j]) for j in range(G)]
    for p in [per] + shared:
        TO.rollout(p); TO.ilqr_step(p, 2)
    for steps in (3, 1):
        for p in [per] + shared:
            TO.shift_trajectory(p, steps)
        t = TO.instance_times(per)
        for b in range(per.B):
            assert np.array_equal(t[b], TO.gettimes(shared[b % G])), f"instance {b} after shift_trajectory({steps})"
        assert np.array_equal(TO.time_steps(per)[0], _rows(grids, per.B)[0])       # the rows are not shifted
        x0 = TO.states(per)[:, 0] + 1e-3
        TO.set_initial_state(per, x0)
        for j, s in enumerate(shared):
            TO.set_initial_state(s, x0)
        for p in [per] + shared:
            TO.rollout(p); TO.ilqr_step(p, 1)
        _assert_rows_equal(_snapshot(per), [_snapshot(s) for s in shared], f"MPC step after shift_trajectory({steps})")
    tf = TO.setinitialtime(per, 2.0)
    assert np.array_equal(TO.time_steps(per)[1], np.full(per.B, 2.0))            # every clock; tf stays the shared grid's
    assert tf == TO.gettimes(per)[-1] and TO.gettimes(per)[0] == 2.0
    for p in [per] + shared:
        p.close()


def test_solve_is_independent_of_the_batch_composition():
    build = lambda: problems.quadrotor(B=48, N=51, error_state=True)
    g = build()
    dt, t0 = _rows(_grids(g), g.B)
    TO.set_time_steps(g, dt, t0)
    st = TO.solve(g)
    assert len(np.unique(st.iterations)) > 1
    idx = np.array([1, 7, 30, 47])
    q = subset(build(), idx)
    TO.set_time_steps(q, dt[idx], t0[idx])
    sq = TO.solve(q)
    for f in TO.SolveStats.FIELDS:
        assert np.array_equal(getattr(st, f)[idx], getattr(sq, f)), f
    assert np.array_equal(TO.states(g)[idx], TO.states(q))
    assert np.array_equal(TO.controls(g)[idx], TO.controls(q))
    Kg, dg = TO.gains(g); Kq, dq = TO.gains(q)
    assert np.array_equal(Kg[idx], Kq) and np.array_equal(dg[idx], dq)
    g.close(); q.close()


def test_rebuild_keeps_the_rows_and_clocks():
    mk = lambda cls=None: problems.cartpole(B=12, N=31, u_bound=3.0, cls=cls)
    p = mk()
    grids = _grids(p)
    dt, t0 = _rows(grids, p.B)
    TO.set_time_steps(p, dt, t0)
    TO.shift_trajectory(p, 2)
    times = TO.instance_times(p)
    TO.add_constraint(p.constraints, TO.GoalConstraint(p.xf), p.N)       # live add_constraint!: the handle is rebuilt
    assert np.array_equal(TO.time_steps(p)[0], dt)
    assert np.array_equal(TO.instance_times(p), times)
    TO.rollout(p)
    X = TO.states(p)
    for j in range(G):
        s = mk(_with_grid(grids[j]))
        TO.initial_controls(s, TO.controls(p))
        TO.set_initial_state(s, p.x0)
        TO.rollout(s)
        Xs = TO.states(s)
        for b in range(j, p.B, G):
            assert np.array_equal(X[b], Xs[b]), f"instance {b} after the rebuild"
        s.close()
    p.close()


def test_refusals_leave_the_table_as_it_was():
    p = problems.quadrotor(B=4, N=11, dt=0.05)
    lib, h, C = p._lib, p._h, TO._capi
    base_dt, base_t0 = TO.time_steps(p)
    assert np.array_equal(base_dt, np.tile(p.spec.dt, (4, 1))) and np.array_equal(base_t0, np.zeros(4))   # the shared grid broadcast
    # a refused first call creates no table
    bad = base_dt.copy(); bad[1, 3] = 0.0
    assert lib.to_set_time_steps(h, C._dp(bad), None) == C.TO_EINVAL
    msg = lib.to_last_error(h).decode()
    assert "instance 1" in msg and "knot 3" in msg, msg
    assert TO.kernel_choice(p)["inst_forward"] == 0
    assert np.array_equal(TO.time_steps(p)[0], base_dt)
    rows = base_dt * np.array([[1.0], [1.1], [0.9], [1.2]])
    t0 = np.array([0.0, 1.0, 2.0, 3.0])
    TO.set_time_steps(p, rows, t0)
    for (b, k, val) in [(2, 5, np.nan), (0, 9, np.inf), (3, 0, -0.05), (1, 1, 0.0)]:
        r = rows.copy(); r[b, k] = val
        assert lib.to_set_time_steps(h, C._dp(r), C._dp(t0 + 5.0)) == C.TO_EINVAL
        msg = lib.to_last_error(h).decode()
        assert f"instance {b}" in msg and f"knot {k}" in msg, msg
        got_dt, got_t0 = TO.time_steps(p)
        assert np.array_equal(got_dt, rows) and np.array_equal(got_t0, t0)
    for val in (np.nan, np.inf):
        bt = t0.copy(); bt[2] = val
        assert lib.to_set_time_steps(h, C._dp(rows * 2), C._dp(bt)) == C.TO_EINVAL
        assert "instance 2" in lib.to_last_error(h).decode()
        got_dt, got_t0 = TO.time_steps(p)
        assert np.array_equal(got_dt, rows) and np.array_equal(got_t0, t0)
    assert lib.to_set_time_steps(h, None, None) == C.TO_EINVAL
    TO.set_time_steps(p, rows * 2)                                         # t0 = None keeps the clocks
    assert np.array_equal(TO.time_steps(p)[1], t0)
    p.close()


def test_hybrid_problem_refuses():
    from dynamics_programs import builtin_problem
    p = builtin_problem("cartpole", TO.Problem, 4, recorded=True)
    with pytest.raises(TO.ArgumentError):
        TO.set_time_steps(p, np.full((4, p.N - 1), 0.1))
    assert p._lib.to_set_time_steps(p._h, TO._capi._dp(np.full((4, p.N - 1), 0.1)), None) == TO._capi.TO_EINVAL
    p.close()


def test_flagship_size_against_the_oracle():
    """BASELINE size, error-state Quadrotor 4096 x 101, 8 horizons tf in [4.5, 5.5] s (b % 8, uniform steps): rollout and [A_e B_e] within the
    one-kernel tolerance of the oracle built with each grid, the gains of one expansion + backward pass within GAIN_TOL, and every result
    bit-identical to the batch built with that grid"""
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
    N = g.N
    tfs = np.random.default_rng(2).uniform(4.5, 5.5, S)
    grids = [(0.0, np.full(N - 1, tf / (N - 1))) for tf in tfs]
    TO.set_time_steps(g, np.array([tfs[b % S] / (N - 1) for b in range(g.B)]))
    U = TO.controls(g)
    TO.rollout(g); TO.expand(g)
    X, ABe = TO.states(g), TO.error_dynamics(g)
    TO.backward(g)
    Kg, dg = TO.gains(g)
    TO.ilqr_step(g, 1)
    after = _snapshot(g)
    for j in range(S):
        idx = np.arange(j, g.B, S)
        o = OracleProblem(g.model, g.obj.copy(), g.x0[idx].copy(), float(tfs[j]), xf=g.xf.copy(), constraints=g.constraints.copy(),
                          t0=0.0, dt=grids[j][1].copy(), error_state=True)
        match_algebra(g, o)
        TO.initial_controls(o, U[idx])
        TO.rollout(o)
        close(X[idx], TO.states(o), KERNEL_RTOL, f"grid {j}: rollout X")
        TO.expand(o)
        close(ABe[idx], TO.error_dynamics(o), KERNEL_RTOL, f"grid {j}: [A_e B_e]")
        TO.backward(o)
        Ko, do = TO.gains(o)
        close(Kg[idx], Ko, GAIN_TOL, f"grid {j}: K"); close(dg[idx], do, GAIN_TOL, f"grid {j}: d")
        o.close()
        s = problems.quadrotor(B=4096, N=101, error_state=True, cls=_with_grid(grids[j]))
        TO.initial_controls(s, U)
        TO.rollout(s); TO.expand(s)
        assert np.array_equal(TO.states(s)[idx], X[idx]) and np.array_equal(TO.error_dynamics(s)[idx], ABe[idx]), f"grid {j}: X / [A_e B_e]"
        TO.backward(s)
        Ks, ds = TO.gains(s)
        assert np.array_equal(Ks[idx], Kg[idx]) and np.array_equal(ds[idx], dg[idx]), f"grid {j}: gains"
        TO.ilqr_step(s, 1)
        ref = _snapshot(s)
        for key, v in after.items():
            assert np.array_equal(v[idx], ref[key][idx], equal_nan=True), f"grid {j}: {key} after ilqr_step"
        s.close()
    g.close()
