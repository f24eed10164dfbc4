"""CPU tests of the costs of user dynamics models on the padded size classes (4, 2), (8, 4) and (16, 8): Problem's padding of a
QuadraticCost, a DiagonalCost and an AutodiffCost onto the class, the padded user cost run by the size-class oracle's interpreter against
NumPy and central differences, the refusals, and set_goal_state's padding of xf."""
import numpy as np
import pytest

import trajopt_b200 as TO
from dynamics_programs import pad
from recorded_classes import ClassesOracleProblem, planar_quadrotor_model
from recorded_costs import CLASS_MODELS, dense_blocks, dense_cost, user_cost

K = TO.capi
CLASSES = sorted(CLASS_MODELS)


def problem_with(model, stage, term, N=4, B=2, cls=ClassesOracleProblem):
    return cls(model, TO.Objective([stage] * (N - 1) + [term]), np.zeros(model.n), 1.0, batch=B)


# ---- QuadraticCost -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cls", CLASSES)
def test_quadratic_cost_padded_entry_by_entry(cls):
    model = CLASS_MODELS[cls]()
    nk, mk, (n, m) = model.n, model.m, cls
    stage, term = dense_cost(nk, mk, 1), dense_cost(nk, mk, 2, terminal=True)
    p = problem_with(model, stage, term)
    assert (p.n, p.m) == cls and p.spec.cost_index == [0] * (p.N - 1) + [1]
    for spec, c in zip(p.spec.costs, (stage, term)):
        assert spec["kind"] == K.COST_QUADRATIC and spec["terminal"] == c.terminal and spec["c"] == c.c
        Q, R, H, q, r = spec["Q"], spec["R"], spec["H"], spec["q"], spec["r"]
        assert Q.shape == (n, n) and R.shape == (m, m) and H.shape == (m, n) and q.shape == (n,) and r.shape == (m,)
        for i in range(n):
            for j in range(n):
                assert Q[i, j] == (c.Q[i, j] if i < nk and j < nk else 0.0), ("Q", i, j)
        for i in range(m):
            for j in range(m):
                assert R[i, j] == (c.R[i, j] if i < mk and j < mk else float(i == j)), ("R", i, j)
        for i in range(m):
            for j in range(n):
                assert H[i, j] == (c.H[i, j] if i < mk and j < nk else 0.0), ("H", i, j)
        assert np.array_equal(q, pad(c.q, n)) and np.array_equal(r, pad(c.r, m))
    # the padded cost's structure: dense with a cross term, and block diagonal when H is zero
    k = TO.QuadraticCost(stage.Q, stage.R, q=stage.q, r=stage.r)
    p2 = problem_with(model, k, term)
    assert not np.any(p2.spec.costs[0]["H"]) and np.any(p.spec.costs[0]["H"])
    p.close(); p2.close()


@pytest.mark.parametrize("cls", CLASSES)
def test_quadratic_cost_padded_through_the_oracle(cls):
    """the oracle's cost, gradient and Hessian of the padded cost, at pad entries that are zero as the solver keeps them, are the user's"""
    model = CLASS_MODELS[cls]()
    nk, mk, (n, m) = model.n, model.m, cls
    stage, term = dense_cost(nk, mk, 3), dense_cost(nk, mk, 4, terminal=True)
    B, N = 3, 4
    p = problem_with(model, stage, term, N=N, B=B)
    r = np.random.default_rng(0)
    X, U = r.uniform(-1, 1, (B, N, nk)), r.uniform(-1, 1, (B, N - 1, mk))
    TO.initial_states(p, pad(X, n)); TO.initial_controls(p, pad(U, m))
    J, g, Hs = TO.cost_knots(p), TO.cost_gradient(p), TO.cost_hessian(p)
    for b in range(B):
        for k in range(N):
            c = stage if k < N - 1 else term
            x, u = X[b, k], (U[b, k] if k < N - 1 else np.zeros(mk))
            want = 0.5 * x @ c.Q @ x + c.q @ x + c.c + (0.0 if k == N - 1 else 0.5 * u @ c.R @ u + c.r @ u + u @ c.H @ x)
            assert abs(J[b, k] - want) <= 1e-12 * max(1.0, abs(want))
            assert np.allclose(g[b, k, :nk], c.Q @ x + c.q + (c.H.T @ u if k < N - 1 else 0.0), rtol=1e-12, atol=1e-12)
            assert np.all(g[b, k, nk:n] == 0.0)
            if k < N - 1:
                assert np.allclose(g[b, k, n:n + mk], c.R @ u + c.r + c.H @ x, rtol=1e-12, atol=1e-12) and np.all(g[b, k, n + mk:] == 0.0)
                assert np.array_equal(Hs[b, k][n + mk:, n + mk:], np.eye(m - mk))
    p.close()


# ---- DiagonalCost: the spec of every existing problem stays as it was ------------------------------------------------------------------
def test_diagonal_cost_spec_is_unchanged():
    """a hybrid 6 -> 3 problem of LQRCosts on class (8, 4): the padded spec, frozen as the padding of DiagonalCosts has always written it"""
    a = planar_quadrotor_model()
    jump = TO.AutodiffDynamics(6, 2, lambda x, u: [x[0] + 0.1 * TO.sin(x[2]), x[1], x[3] * TO.cos(x[2]) + 0.1 * u[0]], output_dim=3, discrete=True)
    b = TO.AutodiffDynamics(3, 1, lambda x, u: [x[2], -0.2 * x[1], u[0] - 0.3 * x[2]])
    models = [a] * 2 + [jump] + [b] * 2
    nx, nu = TO.dims(models)
    N = len(nx)
    costs = [TO.LQRCost(np.full(nx[k], 0.5), np.full(nu[k], 0.25), np.arange(1.0, nx[k] + 1.0), uf=np.full(nu[k], 2.0), terminal=(k == N - 1))
             for k in range(N)]
    p = ClassesOracleProblem(models, TO.Objective(costs), np.zeros(6), 1.0)
    assert (p.n, p.m) == (8, 4) and nx == [6, 6, 6, 3, 3, 3] and nu == [2, 2, 2, 1, 1, 1]
    assert p.spec.cost_index == [0, 1, 2, 3, 4, 5]
    six = dict(Q=[0.5] * 6 + [0.0] * 2, R=[0.25, 0.25, 1.0, 1.0], q=[-0.5, -1.0, -1.5, -2.0, -2.5, -3.0, 0.0, 0.0], r=[-0.5, -0.5, 0.0, 0.0],
               c=0.5 * 0.5 * 91.0 + 0.5 * 0.25 * 8.0)
    three = dict(Q=[0.5] * 3 + [0.0] * 5, R=[0.25, 1.0, 1.0, 1.0], q=[-0.5, -1.0, -1.5, 0.0, 0.0, 0.0, 0.0, 0.0], r=[-0.5, 0.0, 0.0, 0.0],
                 c=0.5 * 0.5 * 14.0 + 0.5 * 0.25 * 4.0)
    for k, spec in enumerate(p.spec.costs):
        want = six if k < 3 else three
        assert spec["kind"] == K.COST_DIAGONAL and spec["terminal"] == (k == N - 1)
        assert set(spec) == {"kind", "terminal", "Q", "R", "q", "r", "c"}
        for f in ("Q", "R", "q", "r"):
            assert spec[f].dtype == np.float64 and np.array_equal(spec[f], np.asarray(want[f])), (k, f, spec[f])
        assert spec["c"] == want["c"]
    p.close()


# ---- AutodiffCost ------------------------------------------------------------------------------------------------------------------------
def central_gradient(f, z, eps=1e-6):
    g = np.zeros_like(z)
    for i in range(z.size):
        e = np.zeros_like(z); e[i] = eps
        g[i] = (f(z + e) - f(z - e)) / (2 * eps)
    return g


def central_hessian(f, z, eps=1e-4):
    H = np.zeros((z.size, z.size))
    for i in range(z.size):
        e = np.zeros_like(z); e[i] = eps
        H[:, i] = (central_gradient(f, z + e) - central_gradient(f, z - e)) / (2 * eps)
    return 0.5 * (H + H.T)


@pytest.mark.parametrize("cls", CLASSES)
def test_user_cost_padded_program(cls):
    """the padded program, run by the oracle's interpreter at nonzero pad controls, is the user cost + 1/2 |u_pad|^2 on non-terminal
    knots and the user cost at the terminal knot; its gradient and Hessian agree with central differences, with a unit pad diagonal"""
    model = CLASS_MODELS[cls]()
    nk, mk, (n, m) = model.n, model.m, cls
    (stage, fs), (term, ft) = user_cost(nk, mk), user_cost(nk, mk, terminal=True)
    B, N = 3, 3
    p = problem_with(model, stage, term, N=N, B=B)
    s0, s1 = p.spec.costs
    npad = m - mk
    # the user's program comes first, unchanged; a terminal cost is not padded
    assert np.array_equal(s0["prog"][:len(stage.prog)], stage.prog) and len(s0["prog"]) == len(stage.prog) + (3 * npad + 1 if npad else 0)
    assert np.array_equal(s1["prog"], term.prog) and np.array_equal(s1["consts"], term.consts)
    r = np.random.default_rng(1)
    X, U = r.uniform(-1, 1, (B, N, n)), r.uniform(-1, 1, (B, N - 1, m))
    X[..., nk:] = 0.0
    TO.initial_states(p, X); TO.initial_controls(p, U)
    J, g, Hs = TO.cost_knots(p), TO.cost_gradient(p), TO.cost_hessian(p)

    def padded(z, f, last):
        x, u = z[:n], z[n:]
        return f(x[:nk], u[:mk]) + (0.0 if last else 0.5 * float(u[mk:] @ u[mk:]))
    for b in range(B):
        for k in range(N):
            last = k == N - 1
            f = ft if last else fs
            z = np.concatenate([X[b, k], U[b, k] if not last else np.zeros(m)])
            fz = lambda v: padded(v, f, last)
            want = fz(z)
            assert abs(J[b, k] - want) <= 1e-13 * max(1.0, abs(want)), (b, k)
            lim = n if last else n + m
            gd = central_gradient(fz, z)[:lim]
            assert np.allclose(g[b, k, :lim], gd, rtol=1e-7, atol=1e-8), (b, k, np.abs(g[b, k, :lim] - gd).max())
            Hd = central_hessian(fz, z)[:lim, :lim]
            assert np.allclose(Hs[b, k][:lim, :lim], Hd, rtol=1e-5, atol=1e-5), (b, k, np.abs(Hs[b, k][:lim, :lim] - Hd).max())
            if not last and npad:
                assert np.array_equal(Hs[b, k][n + mk:, n + mk:], np.eye(npad))
                assert np.all(Hs[b, k][n + mk:, :n + mk] == 0.0)
    p.close()


def test_user_cost_keeps_its_program_on_its_own_class():
    """a knot whose dimensions equal the class takes the user's program as it is"""
    model = TO.AutodiffDynamics(8, 4, lambda x, u: [x[(i + 1) % 8] + u[i % 4] for i in range(8)])
    (stage, _), (term, _) = user_cost(8, 4), user_cost(8, 4, terminal=True)
    p = problem_with(model, stage, term)
    assert (p.n, p.m) == (8, 4)
    assert np.array_equal(p.spec.costs[0]["prog"], stage.prog) and np.array_equal(p.spec.costs[0]["consts"], stage.consts)
    p.close()


def test_user_cost_and_dense_cost_on_a_hybrid_problem():
    """knot by knot: the 6-state knots' costs are padded from (6, 2), the 3-state knots' from (3, 1), to (8, 4)"""
    a = planar_quadrotor_model()
    jump = TO.AutodiffDynamics(6, 2, lambda x, u: [x[0], x[1], x[3] + 0.1 * u[0]], output_dim=3, discrete=True)
    b = TO.AutodiffDynamics(3, 1, lambda x, u: [x[2], -0.2 * x[1], u[0]])
    models = [a, a, jump, b, b]
    nx, nu = TO.dims(models)
    costs = [user_cost(6, 2)[0], dense_cost(6, 2, 5), user_cost(6, 2)[0], dense_cost(3, 1, 6), user_cost(3, 1)[0], dense_cost(3, 1, 7, terminal=True)]
    p = ClassesOracleProblem(models, TO.Objective(costs), np.zeros(6), 1.0)
    kinds = [s["kind"] for s in p.spec.costs]
    assert kinds == [K.COST_EXPR, K.COST_QUADRATIC, K.COST_EXPR, K.COST_QUADRATIC, K.COST_EXPR, K.COST_QUADRATIC]
    for k, (s, c) in enumerate(zip(p.spec.costs, costs)):
        if s["kind"] == K.COST_EXPR:
            assert len(s["prog"]) == len(c.prog) + 3 * (4 - nu[k]) + 1
        else:
            assert np.array_equal(s["Q"][:nx[k], :nx[k]], c.Q) and np.array_equal(s["H"][:nu[k], :nx[k]], c.H)
    p.close()


# ---- refusals ----------------------------------------------------------------------------------------------------------------------------
def test_quaternion_cost_is_refused_on_a_user_model():
    model = TO.AutodiffDynamics(13, 4, lambda x, u: [x[i] for i in range(13)])
    xf = np.zeros(13); xf[3] = 1.0
    qc = TO.QuatLQRCost(np.ones(13), np.ones(4), xf)
    for stage in (qc, TO.DiagonalQuatCost(np.ones(13), np.ones(4))):
        with pytest.raises(TO.ArgumentError, match=r"knot 1: quaternion costs \(DiagonalQuatCost / QuatLQRCost\) need a built-in rigid body"):
            problem_with(model, stage, TO.LQRCost(np.ones(13), np.ones(4), xf, terminal=True))


def test_too_long_padded_program_is_refused():
    """(6, 2) on (8, 4): padding appends 3 * 2 + 1 instructions and, without one already, the constant 0.5"""
    model = planar_quadrotor_model()

    def long_fun(extra):
        def f(x, u):
            s = x[0]
            for i in range(extra):
                s = s + x[i % 6]
            return s
        return f
    term = TO.LQRCost(np.ones(6), np.ones(2), np.zeros(6), terminal=True)
    fits = TO.AutodiffCost(6, 2, long_fun(K.EXPR_MAXLEN - 8 - 7))           # 8 loads + the additions + 7 = the limit
    assert len(fits.prog) == K.EXPR_MAXLEN - 7
    problem_with(model, fits, term).close()
    over = TO.AutodiffCost(6, 2, long_fun(K.EXPR_MAXLEN - 8 - 6))
    with pytest.raises(TO.ArgumentError, match=rf"knot 1: .* needs {K.EXPR_MAXLEN + 1} instructions, past the limit of {K.EXPR_MAXLEN}"):
        problem_with(model, over, term)

    def many_constants(x, u):
        s = x[0]
        for i in range(K.EXPR_MAXCONST):
            s = s + float(i + 1)
        return s
    c = TO.AutodiffCost(6, 2, many_constants)
    assert len(c.consts) == K.EXPR_MAXCONST and 0.5 not in c.consts
    with pytest.raises(TO.ArgumentError, match=rf"knot 1: .* needs {K.EXPR_MAXCONST + 1} constants, past the limit of {K.EXPR_MAXCONST}"):
        problem_with(model, c, term)
    # a terminal user cost takes no padding
    problem_with(model, fits, TO.AutodiffCost(6, 2, long_fun(K.EXPR_MAXLEN - 8), terminal=True)).close()


# ---- set_goal_state on a padded problem --------------------------------------------------------------------------------------------------
def test_set_goal_state_pads_xf():
    """the caller's xf has the terminal knot's 6 entries; what lies after them in memory must not reach the cost terms"""
    model = planar_quadrotor_model()
    N = 5
    obj = TO.LQRObjective(np.full(6, 2.0), np.ones(2), np.full(6, 4.0), np.zeros(6), N)
    cons = TO.ConstraintList(6, 2, N)
    TO.add_constraint(cons, TO.GoalConstraint(np.zeros(6)), N)
    p = ClassesOracleProblem(model, obj, np.zeros(6), 1.0, constraints=cons, batch=2)
    buf = np.full(8, np.nan)
    buf[:6] = np.arange(1.0, 7.0)
    xf = buf[:6]
    TO.set_goal_state(p, xf)
    TO.initial_states(p, np.zeros((2, N, 8)))
    g = TO.cost_gradient(p)                     # at x = 0, u = 0: the linear terms q | r
    assert np.all(np.isfinite(g))
    assert np.array_equal(g[:, :N - 1, :8], np.broadcast_to(pad(-2.0 * xf, 8), (2, N - 1, 8)))
    assert np.array_equal(g[:, N - 1, :8], np.broadcast_to(pad(-4.0 * xf, 8), (2, 8)))
    assert np.array_equal(p.xf, xf)
    p.close()
