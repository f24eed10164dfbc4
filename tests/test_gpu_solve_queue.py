"""A queue of problems through the batch's slots (to_solve_queue).

Central property: problem p's results are, bit for bit, what to_solve gives an instance that starts from x0[p], U0[p], zero multipliers,
the shared penalties and the goal / parameter rows of the per-instance setters.  The reference is to_solve itself on fresh handles of the
same B, the problems loaded chunk by chunk with set_initial_state, initial_controls, set_goal_state (per instance) and set_model_params, the
last chunk padded with copies of its last problem.  Every comparison is np.array_equal."""
import ctypes as C

import numpy as np
import pytest

import trajopt_b200 as TO
from trajopt_b200 import _capi as K
from trajopt_b200 import problems
from test_gpu_mpc import _autodiff, recorded_builtin

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(TO.Problem.__name__ == "OracleProblem", reason="the queue has no oracle counterpart")]

FIELDS = TO.SolveStats.FIELDS


def _cartpole(B):
    return problems.cartpole(B=B, N=51, u_bound=3.0, goal=True)


def _quadrotor(B):
    return problems.quadrotor(B=B, N=51, error_state=True, u_noise=0.01)


def _double_integrator(B):
    return problems.double_integrator(B=B, N=21, dim=2, constrained=False)


CASES = {
    # name: (factory, set_options, per-problem xf, per-problem params, solve options)
    "cartpole": (_cartpole, dict(backward_kernel=1), True, False, dict(iterations=80, cost_tolerance_intermediate=1e-2, constraint_tolerance=1e-3)),
    "quadrotor_rec": (_quadrotor, {}, True, True, dict(iterations=60, cost_tolerance_intermediate=1e-2, constraint_tolerance=1e-3)),
    "double_integrator": (_double_integrator, {}, False, False, dict(iterations=40)),
    "autodiff_dynamics": (lambda B: _autodiff(B=B), {}, False, False, dict(iterations=40, cost_tolerance=1e-3)),
}


def _make(name, B):
    factory, opts, *_ = CASES[name]
    p = factory(B)
    if opts:
        TO.set_options(p, **opts)
    return p


def _inputs(name, M, seed=3):
    """M problems: x0 and U0 from a batch of M built by the case's factory (its own random starts), goals and parameters perturbed"""
    factory, _, with_xf, with_params, _ = CASES[name]
    src = factory(M)
    x0, U0 = src.x0.copy(), TO.controls(src)
    r = np.random.default_rng(seed)
    xf = params = None
    if with_xf:
        xf = np.tile(np.asarray(src.xf, dtype=float), (M, 1))
        k = 3 if src.n == 13 else 2                      # positions (Quadrotor) / cart and angle (Cartpole): the attitude stays unit
        xf[:, :k] += 0.2 * r.uniform(-1, 1, (M, k))
    if with_params:
        base = np.asarray(src.model.params, dtype=float)
        params = base[None, :] * (1.0 + 0.03 * (np.arange(M) % 5))[:, None]
    src.close()
    return x0, U0, xf, params


def _chunked(name, B, x0, U0, xf, params, **opts):
    """to_solve on fresh handles of B instances, chunk by chunk: (stats dict [M], X [M], U [M])"""
    M = x0.shape[0]
    out = {f: [] for f in FIELDS}
    Xs, Us = [], []
    for c in range(0, M, B):
        idx = np.arange(c, c + B).clip(max=M - 1)        # the last chunk padded with its last problem
        p = _make(name, B)
        TO.set_initial_state(p, x0[idx])
        TO.initial_controls(p, U0[idx])
        if xf is not None:
            TO.set_goal_state(p, xf[idx])
        if params is not None:
            TO.set_model_params(p, params[idx])
        st = TO.solve(p, **opts)
        k = min(B, M - c)
        for f in FIELDS:
            out[f].append(getattr(st, f)[:k])
        Xs.append(TO.states(p)[:k]); Us.append(TO.controls(p)[:k])
        p.close()
    return {f: np.concatenate(v) for f, v in out.items()}, np.concatenate(Xs), np.concatenate(Us)


def _assert_equal(r, ref, X, U, what):
    for f in FIELDS:
        assert np.array_equal(getattr(r, f), ref[f]), f"{what}: {f}"
    assert np.array_equal(r.X, X), f"{what}: X"
    assert np.array_equal(r.U, U), f"{what}: U"


@pytest.mark.parametrize("name", sorted(CASES))
def test_queue_equals_chunked_solve(name):
    B = {"cartpole": 16, "quadrotor_rec": 48}.get(name, 16)
    M = 3 * B + 5
    x0, U0, xf, params = _inputs(name, M)
    opts = CASES[name][4]
    g = _make(name, B)
    if name == "quadrotor_rec":
        assert TO.kernel_choice(g)["backward"] == "fragment"
    r = TO.solve_queue(g, x0, U0, xf=xf, params=params, **opts)
    ref, X, U = _chunked(name, B, x0, U0, xf, params, **opts)
    _assert_equal(r, ref, X, U, name)
    assert M > B and len(np.unique(r.iterations)) > 1     # the slots were refilled mid-solve
    if len(g.constraints):
        assert r.iterations_outer.max() > 1               # outer steps happened on the device
    g.close()


@pytest.mark.parametrize("M", [1, 5])
def test_small_queues(M):
    """M = 1 and M < B: idle slots"""
    x0, U0, xf, _ = _inputs("cartpole", M)
    opts = CASES["cartpole"][4]
    g = _make("cartpole", 16)
    r = TO.solve_queue(g, x0, U0, xf=xf, **opts)
    ref, X, U = _chunked("cartpole", 16, x0, U0, xf, None, **opts)
    _assert_equal(r, ref, X, U, f"M={M}")
    g.close()


def test_order_and_slot_count():
    """a permuted order gives permuted results, and B = 16 and B = 24 slots give the same results"""
    M = 60
    x0, U0, xf, _ = _inputs("cartpole", M)
    opts = CASES["cartpole"][4]
    g16, g24 = _make("cartpole", 16), _make("cartpole", 24)
    assert TO.kernel_choice(g16)["backward"] == TO.kernel_choice(g24)["backward"]
    a = TO.solve_queue(g16, x0, U0, xf=xf, **opts)
    perm = np.random.default_rng(7).permutation(M)
    b = TO.solve_queue(g16, x0[perm], U0[perm], xf=xf[perm], **opts)
    c = TO.solve_queue(g24, x0, U0, xf=xf, **opts)
    for f in FIELDS + ("X", "U"):
        assert np.array_equal(getattr(b, f), getattr(a, f)[perm]), f"permuted {f}"
        assert np.array_equal(getattr(c, f), getattr(a, f)), f"B = 24 {f}"
    shared = TO.solve_queue(g16, x0, U0[0], xf=xf, trajectories=False, **opts)   # one U0 for every problem
    ref, _, _ = _chunked("cartpole", 16, x0, np.broadcast_to(U0[0], U0.shape), xf, None, **opts)
    for f in FIELDS:
        assert np.array_equal(getattr(shared, f), ref[f]), f"shared U0 {f}"
    assert shared.X is None and shared.U is None
    g16.close(); g24.close()


def _getters(p):
    out = {"states": TO.states(p), "controls": TO.controls(p), "model_params": TO.model_params(p)}
    out["cost_terms_q"], out["cost_terms_r"] = TO.cost_terms(p)
    out["dt"], out["t0"] = TO.time_steps(p)
    for i in range(len(p.constraints)):
        out[f"multipliers{i}"] = TO.multipliers(p, i)
        out[f"penalties{i}"] = TO.penalties(p, i)
        out[f"constraint_data{i}"] = TO.constraint_data(p, i)
    for j in range(len(p._cost_objs)):
        out[f"cost_weights{j}"] = TO.cost_weights(p, j)
    return out


def _loaded(B):
    """a Quadrotor handle with per-instance tables: penalties and parameters that differ, equal weights and time steps, multipliers set"""
    p = _make("quadrotor_rec", B)
    base = np.asarray(p.model.params, dtype=float)
    TO.set_model_params(p, base[None, :] * (1.0 + 0.02 * (np.arange(B) % 3))[:, None])
    for i in range(len(p.constraints)):
        TO.set_penalties(p, i, TO.penalty(p, i) * (1.0 + np.arange(B) % 2))
        lam = TO.multipliers(p, i)
        TO.set_multipliers(p, i, 0.01 * np.arange(lam.size).reshape(lam.shape))
    TO.set_cost_weights(p, 0, np.tile(TO.cost_weights(p, 0)[0], (B, 1)))
    TO.set_time_steps(p, np.tile(p.spec.dt, (B, 1)))
    TO.rollout(p)
    return p


def test_handle_is_left_as_it_was():
    B, M = 16, 40
    g, twin = _loaded(B), _loaded(B)
    before = _getters(g)
    x0, U0, xf, params = _inputs("quadrotor_rec", M)
    opts = CASES["quadrotor_rec"][4]
    TO.solve_queue(g, x0, U0, xf=xf, params=params, **opts)
    after = _getters(g)
    for k, v in before.items():
        assert np.array_equal(after[k], v), k
    sg, st = TO.solve(g, **opts), TO.solve(twin, **opts)
    for f in FIELDS:
        assert np.array_equal(getattr(sg, f), getattr(st, f)), f"solve after the queue: {f}"
    assert np.array_equal(TO.states(g), TO.states(twin)) and np.array_equal(TO.controls(g), TO.controls(twin))
    g.close(); twin.close()


def _raw(p, M, x0=None, U0=None, **opts):
    """to_solve_queue straight through the C ABI (past the Python checks): the return code and the handle's message"""
    x0 = np.zeros((max(M, 1), p.n)) if x0 is None else x0
    U0 = np.zeros((p.N - 1, p.m)) if U0 is None else U0
    spec = K.to_queue_spec(M, 1, K._dp(np.ascontiguousarray(x0)), K._dp(np.ascontiguousarray(U0)), None, 1, 1, None, 0, 0)
    o = TO.solve_options(**opts)
    st = np.zeros(max(M, 1), dtype=np.int32)
    rc = p._lib.to_solve_queue(p._h, C.byref(spec), C.byref(o), K._ip(st), None, None, None, None, None, None, None, None)
    return rc, p._lib.to_last_error(p._h).decode()


def test_c_side_refusals():
    p = _make("quadrotor_rec", 8)
    B = p.B
    rc, msg = _raw(p, 0)
    assert rc == K.TO_EINVAL and "M must be >= 1" in msg
    rc, msg = _raw(p, 4, iterations=0)
    assert rc == K.TO_EINVAL and "iterations" in msg
    w = np.tile(TO.cost_weights(p, 0)[0], (B, 1)); w[3, 0] *= 2
    TO.set_cost_weights(p, 0, w)
    rc, msg = _raw(p, 4)
    assert rc == K.TO_EINVAL and "cost weights differ" in msg
    p.close()
    p = _make("quadrotor_rec", 8)
    TO.set_time_steps(p, np.tile(p.spec.dt, (B, 1)) * (1.0 + (np.arange(B) % 2))[:, None])
    rc, msg = _raw(p, 4)
    assert rc == K.TO_EINVAL and "time steps differ" in msg
    p.close()
    p = _make("quadrotor_rec", 8)
    bound = next(i for i, c in enumerate(p.constraints) if isinstance(c, TO.BoundConstraint))
    d = TO.constraint_data(p, bound); d[2, p.n:p.n + p.m] *= 0.5      # the upper control bounds of instance 2 (the state is unbounded)
    TO.set_constraint_data(p, bound, d)
    rc, msg = _raw(p, 4)
    assert rc == K.TO_EINVAL and "constraint data differ" in msg
    with pytest.raises(TO.ArgumentError, match="constraint data differ"):
        x0, U0, xf, _ = _inputs("quadrotor_rec", 4)
        TO.solve_queue(p, x0, U0, xf=xf)
    p.close()
    # a constrained recorded-program model: no per-instance penalties for its outer steps
    m0, _ = recorded_builtin("cartpole")
    N = 21
    obj = TO.LQRObjective(1e-2 * np.eye(4), 1e-1 * np.eye(1), 100.0 * np.eye(4), np.array([0, np.pi, 0, 0.0]), N)
    cons = TO.ConstraintList(4, 1, N)
    TO.add_constraint(cons, TO.BoundConstraint(4, 1, u_min=-5.0, u_max=5.0), (1, N - 1))
    a = TO.Problem(m0, obj, np.zeros((4, 4)), 2.0, constraints=cons)
    rc, msg = _raw(a, 4)
    assert rc == K.TO_EINVAL and "recorded-program" in msg
    a.close()
    # a hybrid problem: two recorded models with different programs
    m1 = TO.AutodiffDynamics(4, 1, lambda x, u: [x[2], x[3], u[0], -u[0]])
    h = TO.Problem([m0 if k % 2 == 0 else m1 for k in range(N - 1)], obj.copy(), np.zeros((4, 4)), 2.0)
    assert h.hybrid
    rc, msg = _raw(h, 4)
    assert rc == K.TO_EINVAL and "hybrid" in msg
    h.close()
