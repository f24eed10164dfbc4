"""Per-instance AL penalties (to_set_penalties) and the per-instance outer step of to_solve.

Central property: a batch whose instance b holds the penalties MU[b % 3] computes, bit for bit, what instance b of a batch of the same size,
x0 and U0 built with to_set_penalty(MU[b % 3]) computes -- through the expansion, the backward pass, the line search and the dual update.
to_solve with the table takes each instance's outer step on the device when its inner loop ends; its statistics and trajectories are
those of the shared (batch-synchronous) solve, and each instance ends at its own penalties."""
import ctypes

import numpy as np
import pytest

import trajopt_b200 as TO
from trajopt_b200 import problems
from test_gpu_instance_params import PATHS, G, _assert_rows_equal, _snapshot
from test_gpu_solve import subset

pytestmark = pytest.mark.gpu

SCALE = (1.0, 4.0, 0.25)       # instance b: every penalty = the shared one x SCALE[b % 3]


def _make(factory, opts):
    p = factory(None)
    if opts:
        TO.set_options(p, **opts)
    return p


def _ncon(p):
    return len(p.constraints)


def _mu0(p):
    return [TO.penalty(p, i) for i in range(_ncon(p))]


def _set_rows(p, sets=G):
    mu0 = _mu0(p)
    for i in range(_ncon(p)):
        rows = np.array([mu0[i] * SCALE[b % sets] for b in range(p.B)])
        TO.set_penalties(p, i, rows)
        assert np.array_equal(TO.penalties(p, i), rows)


def _shared_batches(factory, opts, mu0):
    out = []
    for j in range(G):
        s = _make(factory, opts)
        for i, m in enumerate(mu0):
            TO.set_penalty(s, i, m * SCALE[j])
        out.append(s)
    return out


def _opts(p):
    """the handle's solver options (the defaults until set_options)"""
    o = getattr(p, "_options", None)
    if o is None:
        o = TO._capi.to_options()
        p._default_options(o)
    return o


def _penalty_rows(p):
    """{penalties i: [B]}; a shared batch broadcasts its shared value"""
    return {f"penalties{i}": TO.penalties(p, i) for i in range(_ncon(p))}


def _compare_pipeline(per, shared, what, sets=G, solve=True):
    """merit, AL expansion, records, gains, 3 iLQR iterations, the dual + penalty update and a solve of `per` against the shared batches"""
    probs = [per] + shared
    for p in probs:
        TO.rollout(p)
    _assert_rows_equal(_snapshot(per), [_snapshot(s) for s in shared], f"{what} after rollout", sets)
    alx = lambda p: dict(zip(("al_grad", "al_hess"), TO.al_expansion(p)))
    _assert_rows_equal(alx(per), [alx(s) for s in shared], f"{what} AL expansion", sets)
    for p in probs:
        TO.expand(p)
        TO.backward(p)
    if TO.backward_algebra(per) == 1:   # record path: the records (FASTAL / fused term table) the Riccati kernel read
        _assert_rows_equal({"records": TO.expansion_records(per)}, [{"records": TO.expansion_records(s)} for s in shared], f"{what} records", sets)
    gk = lambda p: dict(zip(("K", "d"), TO.gains(p)))
    _assert_rows_equal(gk(per), [gk(s) for s in shared], f"{what} gains", sets)
    for p in probs:
        TO.ilqr_step(p, 3)
    _assert_rows_equal(_snapshot(per), [_snapshot(s) for s in shared], f"{what} after ilqr_step(3)", sets)
    _assert_rows_equal(gk(per), [gk(s) for s in shared], f"{what} gains after ilqr_step(3)", sets)
    for p in probs:
        TO.al_update(p)
    _assert_rows_equal(_penalty_rows(per), [_penalty_rows(s) for s in shared], f"{what} penalties after al_update", sets)
    _assert_rows_equal(_snapshot(per), [_snapshot(s) for s in shared], f"{what} after al_update", sets)
    if not solve:
        return
    stats = [TO.solve(p, iterations=40) for p in probs]
    for f in TO.SolveStats.FIELDS:
        v = getattr(stats[0], f)
        for b in range(per.B):
            assert np.array_equal(v[b], getattr(stats[1 + b % sets], f)[b]), f"{what}: solve {f} of instance {b}"
    # after the solve a shared batch holds its last outer iteration's penalties, so its merit is not instance b's (see test_solve_equal_rows)
    snap = lambda p: {k: v for k, v in _snapshot(p).items() if k != "merit"}
    _assert_rows_equal(snap(per), [snap(s) for s in shared], f"{what} after solve", sets)
    _assert_rows_equal(gk(per), [gk(s) for s in shared], f"{what} gains after solve", sets)


@pytest.mark.parametrize("path", sorted(PATHS))
def test_equal_rows_equal_untouched_batch(path):
    """every row equal to the shared penalties: the outputs of a batch that never called the setter, bit for bit"""
    factory, opts = PATHS[path]
    per, plain = _make(factory, opts), _make(factory, opts)
    for i, m in enumerate(_mu0(per)):
        TO.set_penalties(per, i, m)
    a, b = TO.kernel_choice(per), TO.kernel_choice(plain)
    for k in a:
        if not k.startswith("inst"):
            assert a[k] == b[k], k
    assert a["inst_forward"] and a["inst_backward"] and not b["inst_forward"]
    _compare_pipeline(per, [plain], path, sets=1)
    per.close(); plain.close()


@pytest.mark.parametrize("path", sorted(PATHS))
def test_instance_penalties_equal_shared_batches(path):
    factory, opts = PATHS[path]
    per = _make(factory, opts)
    shared = _shared_batches(factory, opts, _mu0(per))
    _set_rows(per)
    _compare_pipeline(per, shared, path)
    for p in [per] + shared:
        p.close()


def _schedule(mu0, outer, opts):
    """min(mu0 phi^(outer - 1), mu_max), one multiplication at a time as the device takes it"""
    mu = mu0
    for _ in range(outer - 1):
        mu = min(mu * opts.penalty_scaling, opts.penalty_max)
    return mu


@pytest.mark.parametrize("path", ["cartpole_warp", "quadrotor_rec", "double_integrator_quickstart"])
def test_solve_equal_rows(path):
    """to_solve with rows equal to the shared penalties gives the shared solve bit for bit; each instance then holds its own schedule's
    penalty and its merit at that penalty"""
    factory, opts = PATHS[path]
    per, plain = _make(factory, opts), _make(factory, opts)
    mu0 = _mu0(per)
    for i, m in enumerate(mu0):
        TO.set_penalties(per, i, m)
    sp, sq = TO.solve(per), TO.solve(plain)
    for f in TO.SolveStats.FIELDS:
        assert np.array_equal(getattr(sp, f), getattr(sq, f)), f
    assert np.array_equal(TO.states(per), TO.states(plain)) and np.array_equal(TO.controls(per), TO.controls(plain))
    for i in range(_ncon(per)):
        assert np.array_equal(TO.multipliers(per, i), TO.multipliers(plain, i))
    assert all(np.array_equal(a, b) for a, b in zip(TO.gains(per), TO.gains(plain)))
    o = _opts(per)
    for i in range(_ncon(per)):
        want = np.array([_schedule(mu0[i], int(k), o) for k in sp.iterations_outer])
        assert np.array_equal(TO.penalties(per, i), want)
    # the merit of each instance, at its own penalties: the untouched batch's merit with its shared penalties set to that schedule
    Jp = TO.merit(per)
    for k in np.unique(sp.iterations_outer):
        for i in range(_ncon(plain)):
            TO.set_penalty(plain, i, _schedule(mu0[i], int(k), o))
        sel = sp.iterations_outer == k
        assert np.array_equal(Jp[sel], TO.merit(plain)[sel]), f"merit of the instances that ended in outer iteration {k}"
    per.close(); plain.close()


def _distinct(build, opts):
    g = build()
    if opts:
        TO.set_options(g, **opts)
    mu0 = _mu0(g)
    rows = [np.array([mu0[i] * SCALE[b % G] for b in range(g.B)]) for i in range(_ncon(g))]
    return g, rows


COMPOSE = {
    "cartpole": (lambda: problems.cartpole(B=48, N=51, u_bound=3.0, goal=True), dict(backward_kernel=1)),
    "quadrotor_rec": (lambda: problems.quadrotor(B=48, N=51, error_state=True), {}),
}


@pytest.mark.parametrize("case", sorted(COMPOSE))
def test_solve_is_independent_of_the_batch_composition(case):
    build, opts = COMPOSE[case]
    g, rows = _distinct(build, opts)
    idx = np.array([1, 7, 30, 47])
    q = subset(build(), idx)
    if opts:
        TO.set_options(q, **opts)
    for i, r in enumerate(rows):
        TO.set_penalties(g, i, r)
        TO.set_penalties(q, i, r[idx])
    assert TO.kernel_choice(g)["backward"] == TO.kernel_choice(q)["backward"]
    st, sq = TO.solve(g), TO.solve(q)
    assert len(np.unique(st.iterations)) > 1
    for f in TO.SolveStats.FIELDS:
        assert np.array_equal(getattr(st, f)[idx], getattr(sq, f)), f
    assert np.array_equal(TO.states(g)[idx], TO.states(q)) and np.array_equal(TO.controls(g)[idx], TO.controls(q))
    Kg, dg = TO.gains(g); Kq, dq = TO.gains(q)
    assert np.array_equal(Kg[idx], Kq) and np.array_equal(dg[idx], dq)
    for i in range(_ncon(g)):
        assert np.array_equal(TO.multipliers(g, i)[idx], TO.multipliers(q, i))
        assert np.array_equal(TO.penalties(g, i)[idx], TO.penalties(q, i))
    assert np.array_equal(TO.merit(g)[idx], TO.merit(q))
    g.close(); q.close()


def _mpc(p, x1):
    """solve, shift by one knot, a new measured state, solve"""
    s1 = TO.solve(p, iterations=60)
    TO.shift_trajectory(p, 1)
    TO.set_initial_state(p, x1)
    s2 = TO.solve(p, iterations=60)
    return s1, s2


def test_warm_started_sequence_equals_each_instance_alone():
    """MPC: with the table the batch equals each instance run alone through the same sequence; with shared penalties it does not (the
    second solve of an instance starts from the batch's last penalty)"""
    build, opts = COMPOSE["cartpole"]
    idx = [0, 5, 13, 22, 40]
    rng = np.random.default_rng(9)
    g0 = build()
    x1 = g0.x0 + 0.01 * rng.standard_normal(g0.x0.shape)
    g0.close()

    def run(table):
        g, rows = _distinct(build, opts)
        solo = [subset(build(), np.array([b])) for b in idx]
        for q in solo:
            TO.set_options(q, **opts)
        if table:
            for i, r in enumerate(rows):
                TO.set_penalties(g, i, r)
                for q, b in zip(solo, idx):
                    TO.set_penalties(q, i, r[b:b + 1])
        else:
            for i, r in enumerate(rows):
                TO.set_penalty(g, i, r[0])
                for q in solo:
                    TO.set_penalty(q, i, r[0])
        sg = _mpc(g, x1)
        same = []
        for q, b in zip(solo, idx):
            sq = _mpc(q, x1[b:b + 1])
            eq = all(np.array_equal(getattr(s, f)[b], getattr(t, f)[0]) for s, t in zip(sg, sq) for f in TO.SolveStats.FIELDS)
            eq = eq and np.array_equal(TO.states(g)[b], TO.states(q)[0]) and np.array_equal(TO.controls(g)[b], TO.controls(q)[0])
            for i in range(_ncon(g)):
                eq = eq and np.array_equal(TO.multipliers(g, i)[b], TO.multipliers(q, i)[0])
            if table:
                for i in range(_ncon(g)):
                    eq = eq and np.array_equal(TO.penalties(g, i)[b], TO.penalties(q, i)[0])
            same.append(eq)
            q.close()
        g.close()
        return same

    same = run(True)
    assert all(same), same
    same = run(False)
    assert not all(same), "with shared penalties every sampled instance matched its solo sequence: the test shows nothing"


def test_refusals_leave_the_table_as_it_was():
    p = problems.cartpole(B=4, N=11, u_bound=3.0, goal=True)
    lib, h, C = p._lib, p._h, TO._capi
    mu0 = _mu0(p)
    # a refused first call creates no table
    assert lib.to_set_penalties(h, 0, C._dp(np.array([1.0, 0.0, 1.0, 1.0]))) == C.TO_EINVAL
    assert "instance 1" in lib.to_last_error(h).decode()
    assert not TO.kernel_choice(p)["inst_backward"]
    rows = np.array([1.0, 2.0, 3.0, 4.0])
    TO.set_penalties(p, 1, rows)
    table = lambda: [TO.penalties(p, i) for i in range(2)]
    before = table()
    assert np.array_equal(before[0], np.full(4, mu0[0])) and np.array_equal(before[1], rows)
    for bad, b in [((np.nan,), 2), ((-1.0,), 0), ((0.0,), 3), ((np.inf,), 1)]:
        r = rows.copy(); r[b] = bad[0]
        assert lib.to_set_penalties(h, 1, C._dp(r)) == C.TO_EINVAL
        assert f"instance {b}" in lib.to_last_error(h).decode()
        assert all(np.array_equal(x, y) for x, y in zip(table(), before))
    for con in (-1, 2):
        assert lib.to_set_penalties(h, con, C._dp(rows)) == C.TO_EINVAL
    assert lib.to_set_penalties(h, 1, None) == C.TO_EINVAL
    assert all(np.array_equal(x, y) for x, y in zip(table(), before))
    # the shared getter: the common value while the rows agree, TO_ESTATE once they differ
    assert TO.penalty(p, 0) == mu0[0]
    v = ctypes.c_double()
    assert lib.to_get_penalty(h, 1, ctypes.byref(v)) == C.TO_ESTATE
    assert "to_get_penalties" in lib.to_last_error(h).decode()
    # the shared setter writes through
    TO.set_penalty(p, 1, 7.0)
    assert np.array_equal(TO.penalties(p, 1), np.full(4, 7.0)) and TO.penalty(p, 1) == 7.0
    # al_update scales every row as the host scales the shared value
    TO.set_penalties(p, 1, rows)
    TO.al_update(p)
    o = _opts(p)
    assert np.array_equal(TO.penalties(p, 1), [min(r * o.penalty_scaling, o.penalty_max) for r in rows])
    # a new penalty_initial resets every row
    TO.set_options(p, penalty_initial=3.5)
    for i in range(2):
        assert np.array_equal(TO.penalties(p, i), np.full(4, 3.5))
    p.close()
    from dynamics_programs import builtin_problem
    q = builtin_problem("cartpole", TO.Problem, 4, recorded=True)
    if len(q.constraints):
        with pytest.raises(TO.ArgumentError):
            TO.set_penalties(q, 0, 1.0)
        assert q._lib.to_set_penalties(q._h, 0, C._dp(np.ones(4))) == C.TO_EINVAL
    q.close()


def test_flagship_size():
    """BASELINE size (4096 x 101, error-state Quadrotor): three penalty values by b % 3 give one expansion + backward pass + line search
    bit-identical to the three shared batches, and a full solve leaves no device error"""
    factory = lambda cls: problems.quadrotor(B=4096, N=101, error_state=True, cls=cls)
    per = factory(None)
    shared = _shared_batches(factory, {}, _mu0(per))
    _set_rows(per)
    probs = [per] + shared
    for p in probs:
        TO.rollout(p)
        TO.ilqr_step(p, 1)
    keys = lambda p: dict(X=TO.states(p), U=TO.controls(p), merit=TO.merit(p), **dict(zip(("K", "d"), TO.gains(p))))
    _assert_rows_equal(keys(per), [keys(s) for s in shared], "BASELINE iteration")
    for s in shared:
        s.close()
    st = TO.solve(per)
    assert per._lib.to_synchronize(per._h) == 0
    assert np.all(st.iterations >= 1)
    per.close()
