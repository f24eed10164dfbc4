"""The integration rule on the device (``Problem(..., integration)``, include/trajopt_b200.h to_set_integration): every solver path with Euler,
RK2 and RK3 against the oracle with the same rule (tests/oracle_rules.cpp) and against NumPy restatements of the rules; the double integrator,
which every rule but Euler integrates exactly; RK4 set explicitly against a handle that never called the setter; each rule with per-instance
time steps and model parameters and in the hybrid example with its jump map; a handle rebuild; and the reference's recorded Cartpole outputs
(examples/Cartpole.ipynb, RK3) pinned on the device."""
import numpy as np
import pytest

import trajopt_b200 as TO
from integration_rules import RulesOracleProblem, double_integrator_step_errors, jacobian_fd, model_step
from oracle_binding import match_algebra
from parity_util import FACTOR, GAIN_TOL, check, decisions_agree, inst_err
from test_gpu_instance_params import G, PATHS, _compare_pipeline, _make, _model_of, _param_sets
from test_hybrid_models import hybrid_problem

pytestmark = pytest.mark.gpu
P = TO.problems

KERNEL_RTOL = 1e-10     # tests/test_gpu_parity.py: one kernel against the oracle on the same inputs


def _close(a, b, rtol, what):
    a, b = np.asarray(a), np.asarray(b)
    err = float(np.max(np.abs(a - b) / np.maximum(1.0, np.abs(b)))) if a.size else 0.0
    assert np.all(np.isfinite(a)) and err <= rtol, f"{what}: max rel err {err:.3e}"


def _jacobians(p):
    return TO.error_dynamics(p) if p.error_state else TO.dynamics_jacobians(p)


# The first gains of the register-resident kernel (quadrotor_rec) against the oracle, in units of the disagreement of the oracle's two algebraic
# forms of the backward pass on the same inputs: a problem that amplifies rounding more moves both.  Only one instance goes beyond GAIN_TOL,
# RK3's instance 27 (RK4 stays within it): 8.3e-9, which is 124 times the forms' disagreement on the device's trajectory (6.7e-11) and 65 times
# it on the oracle's own rollout (1.3e-10).  The yardstick is one rounding sample and moves by 2x with inputs 1e-10 apart; the bound is 200.
ALG_FACTOR = 200.0


@pytest.mark.parametrize("rule", ["Euler", "RK2", "RK3"])
@pytest.mark.parametrize("path", sorted(PATHS))
def test_rules_against_the_oracle(path, rule):
    """Every solver path with each rule, device vs oracle with the same rule (tests/test_gpu_parity.py's method): the rollout at kernel tolerance
    (an unstable open loop: within FACTOR times its sensitivity to x0), then, on the device's trajectory, [A B] / [A_e B_e] (on the record path
    exported from the records) at kernel tolerance; the gains of the first backward pass at GAIN_TOL or within ALG_FACTOR
    times the disagreement of the oracle's two algebraic forms; after 3 iLQR iterations, within the budget of the twin, the oracle whose gains
    carry GAIN_TOL noise.  Instances whose open-loop rollout runs away (|x| > 100 on the oracle: the Euler Acrobot) are left out; at least 4
    of every batch are compared.  Euler and RK2 do not keep the quaternion's norm (it reaches 16 on quadrotor_rec's rollout under RK2), and at
    such norms the error-state expansions and line search of the compact and record paths, which do not depend on the rule, part from the
    oracle's (DESIGN.md 5k).  On those paths Euler and RK2 are compared up to their own kernels: the rollout and [A_e B_e]."""
    factory, opts = PATHS[path]
    g = _make(factory, opts)
    oracle = lambda: match_algebra(g, _make(lambda cls: factory(RulesOracleProblem), opts))
    o, t, a = oracle(), oracle().set_gain_noise(GAIN_TOL), oracle()
    a.set_backward_variant(1 - TO.backward_algebra(g))        # the other algebraic form
    for p in (g, o, t, a):
        TO.set_integration(p, rule)
        TO.rollout(p)
    assert isinstance(TO.integration(g), getattr(TO, rule)) and isinstance(TO.integration(o), getattr(TO, rule))
    Xo = TO.states(o)
    sel = np.abs(Xo).reshape(g.B, -1).max(axis=1) < 100.0
    assert sel.sum() >= 4, f"{path} {rule}: {int(sel.sum())} of {g.B} rollouts stay bounded"

    def close(x, y, tol, what):
        e = inst_err(x, y)[sel]
        assert np.all(e <= tol), f"{path} {rule} {what}: max rel err {e.max():.3e}"

    # the rollout at KERNEL_RTOL, or within FACTOR times what the oracle's own rollout moves when x0 moves by one part in 1e15: an unstable
    # open loop (the Euler Acrobot) amplifies a one-ulp difference of sin / cos along the horizon
    Xg, x0 = TO.states(g), g.x0.copy()
    TO.set_initial_state(a, x0 * (1.0 + 1e-15))
    TO.rollout(a)
    e, amp = inst_err(Xg, Xo), inst_err(TO.states(a), Xo)
    bad = np.nonzero(sel & ~(e <= np.maximum(KERNEL_RTOL, FACTOR * amp)))[0]
    assert bad.size == 0, f"{path} {rule} rollout: instances {bad[:5]} differ by {e[bad].max():.3e} (x0 moved by 1e-15: {amp[bad].max():.3e})"
    # every later kernel reads the same inputs on both sides: the device's trajectory (parity_util: one kernel application on identical inputs)
    Xin = np.nan_to_num(np.where(sel[:, None, None], Xg, Xo))
    for p in (o, t, a):
        TO.set_initial_state(p, x0)
        TO.initial_states(p, Xin)
    TO.initial_states(g, Xin)
    for p in (g, o, t, a):
        TO.expand(p)
    close(_jacobians(g), _jacobians(o), KERNEL_RTOL, "Jacobians")
    if g.error_state and isinstance(g.model, TO.Quadrotor) and rule in ("Euler", "RK2") and path != "quadrotor_lie":
        for p in (g, o, t, a):
            p.close()
        return
    for p in (g, o, t, a):
        TO.backward(p)
    for what, (xg, xo, xa) in zip("Kd", zip(TO.gains(g), TO.gains(o), TO.gains(a))):
        e, s = inst_err(xg, xo), inst_err(xa, xo)
        bad = np.nonzero(sel & ~(e <= np.maximum(GAIN_TOL, ALG_FACTOR * s)))[0]
        assert bad.size == 0, f"{path} {rule} {what}: instances {bad[:5]} differ by {e[bad].max():.3e} (the algebraic forms by {s[bad].max():.3e})"
    a.close()
    for p in (g, o, t):
        TO.ilqr_step(p, 3)
    sg, so, st_ = TO.solver_state(g), TO.solver_state(o), TO.solver_state(t)
    live = sel & (np.abs(so["dV"][:, 0]) > 1e-9 * np.maximum(1.0, np.abs(TO.merit(o))))
    dec = live & (so["alpha"] == st_["alpha"]) & (so["bp_status"] == st_["bp_status"]) & (sg["alpha"] == so["alpha"]) & (sg["bp_status"] == so["bp_status"])
    check(f"{path} {rule} merit after 3 iterations", TO.merit(g), TO.merit(o), TO.merit(t), 1e-8, dec)
    check(f"{path} {rule} X after 3 iterations", TO.states(g), TO.states(o), TO.states(t), 1e-8, dec)
    check(f"{path} {rule} U after 3 iterations", TO.controls(g), TO.controls(o), TO.controls(t), 1e-8, dec)
    for k in ("alpha", "ls_iters", "bp_status"):
        decisions_agree(f"{path} {rule} {k}", sg[k], so[k], st_[k], live, allow=0.05)
    for p in (g, o, t):
        p.close()


@pytest.mark.parametrize("rule", ["Euler", "RK2", "RK3", "RK4"])
def test_double_integrator_exactness(rule):
    """the device's rollout of the double integrator (1-D and 2-D): every step of RK2, RK3 and RK4 is the exact solution under constant u;
    Euler's is off by h^2 a / 2 in position and exact in velocity"""
    for dim, N in ((1, 51), (2, 21)):
        p = P.double_integrator(B=64, N=N, dim=dim, integration=rule)
        TO.initial_controls(p, np.random.default_rng(3).standard_normal((64, N - 1, dim)))
        TO.rollout(p)
        X, U, h = TO.states(p), TO.controls(p), np.diff(TO.gettimes(p))
        for b in range(p.B):
            dr, dv = double_integrator_step_errors(X[b], U[b], h, p.model.params[0])
            scale = max(1.0, np.abs(X[b]).max())
            if rule == "Euler":
                dr = dr + 0.5 * (h * h)[:, None] * U[b] / p.model.params[0]
            assert np.abs(dr).max() < 1e-13 * scale and np.abs(dv).max() < 1e-13 * scale, (rule, dim, b)
        p.close()


def _G(q):
    """the attitude columns of the error state at q (csrc/rollout.cu expand_lie_column): L(q) H, 4 x 3"""
    w, x, y, z = q
    return np.array([[-x, -y, -z], [w, -z, y], [z, w, -x], [-y, x, w]])


def _E(xk, n, m):
    """(n + m) x (n - 1 + m): the full-state directions of the error-state coordinates of knot state xk (and the controls)"""
    E = np.zeros((n + m, n - 1 + m))
    E[0:3, 0:3] = np.eye(3)
    E[3:7, 3:6] = _G(xk[3:7])
    E[7:n, 6:n - 1] = np.eye(n - 7)
    E[n:, n - 1:] = np.eye(m)
    return E


@pytest.mark.parametrize("rule", ["Euler", "RK2", "RK3", "RK4"])
@pytest.mark.parametrize("path", sorted(PATHS))
def test_rules_against_numpy(path, rule):
    """The device's rollout, Jacobians and line-search trajectories with each rule against the NumPy restatement of the rule on the oracle's
    continuous dynamics: the rollout to 1e-12, [A B] (or E(x_k+1)' [A B] E(x_k) for [A_e B_e]) to central differences of the restated step,
    and after 3 iLQR iterations every accepted knot x_k+1 = step(x_k, u_k) and a merit no larger than the first."""
    factory, opts = PATHS[path]
    g = _make(factory, opts)
    TO.set_integration(g, rule)
    stp = model_step(g.model, rule)
    n, m = g.n, g.m
    TO.rollout(g)
    X, U, t = TO.states(g), TO.controls(g), TO.gettimes(g)
    h = np.diff(t)
    picks = (0, g.B // 2, g.B - 1)
    for b in picks:
        for k in range(g.N - 1):
            _close(X[b, k + 1], stp(X[b, k], U[b, k], h[k]), 1e-12, f"{path} {rule} rollout b={b} k={k}")
    TO.expand(g)
    J = _jacobians(g)
    for b in picks:
        # central differences lose digits in proportion to the state: knots where an open-loop Euler rollout has grown large are left out
        for k in [k for k in (0, g.N // 2, g.N - 2) if np.abs(X[b, k:k + 2]).max() < 100.0]:
            fd = jacobian_fd(stp, X[b, k], U[b, k], h[k])
            if g.error_state:
                fd = _E(X[b, k + 1], n, 0)[:n, :n - 1].T @ fd @ _E(X[b, k], n, m)
            _close(J[b, k], fd, 2e-6, f"{path} {rule} Jacobian b={b} k={k}")
    J0 = TO.merit(g)
    TO.ilqr_step(g, 3)
    X, U = TO.states(g), TO.controls(g)
    for b in picks:
        for k in range(g.N - 1):
            _close(X[b, k + 1], stp(X[b, k], U[b, k], h[k]), 1e-12, f"{path} {rule} line-search trajectory b={b} k={k}")
    ok = np.isfinite(J0)                        # (an open-loop Euler rollout of the Acrobot overflows on some instances)
    assert np.all(TO.merit(g)[ok] <= J0[ok] * (1 + 1e-12))
    g.close()


@pytest.mark.parametrize("path", sorted(PATHS))
def test_rk4_set_explicitly_is_the_default(path):
    """to_set_integration(TO_RK4) computes, bit for bit, what a handle that never called the setter computes"""
    factory, opts = PATHS[path]
    a, b = _make(factory, opts), _make(factory, opts)
    TO.set_integration(b, TO.RK4)
    for p in (a, b):
        TO.rollout(p); TO.expand(p); TO.backward(p)
    assert np.array_equal(TO.states(a), TO.states(b)) and np.array_equal(_jacobians(a), _jacobians(b))
    for x, y in zip(TO.gains(a), TO.gains(b)):
        assert np.array_equal(x, y)
    for p in (a, b):
        TO.ilqr_step(p, 3)
    for f in (TO.states, TO.controls, TO.merit):
        assert np.array_equal(f(a), f(b)), f.__name__
    a.close(); b.close()


@pytest.mark.parametrize("rule", ["Euler", "RK2", "RK3"])
def test_rules_with_instance_parameters_and_time_steps_on_the_record_path(rule):
    """each rule with per-instance model parameters and time steps (the INST kernels of every dynamics-stepping family) on the record path:
    each instance computes, bit for bit, what a batch built with its parameters and the rule computes"""
    factory, opts = PATHS["quadrotor_rec"]
    base = _make(factory, opts)
    sets = _param_sets(base.model)
    B = base.B
    per = _make(factory, opts)
    TO.set_integration(per, rule)
    TO.set_model_params(per, np.array([sets[b % G] for b in range(B)]))
    dt, _ = TO.time_steps(per)
    TO.set_time_steps(per, dt)                 # rows equal to the shared grid: the INST kernels on the shared steps
    shared = []
    for s in sets:
        q = _make(factory, opts, _model_of(base.model, s))
        TO.set_integration(q, rule)
        shared.append(q)
    _compare_pipeline(per, shared, f"{rule} + instance parameters and time steps")
    for p in [base, per] + shared:
        p.close()


@pytest.mark.parametrize("rule", ["Euler", "RK2", "RK3"])
def test_hybrid_problem(rule):
    """the hybrid example (test/hybrid_dynamics_model.jl) with each rule on its continuous models, against the oracle with the same rule; the
    jump map is applied as it is"""
    B = 64
    rng = np.random.default_rng(5)
    gp, _ = hybrid_problem(TO.Problem, batch=B, integration=rule)
    op, _ = hybrid_problem(RulesOracleProblem, batch=B, integration=rule)
    x0 = 0.3 * rng.standard_normal((B, 4))
    U = rng.standard_normal((B, 10, 2)); U[:, 6:, 1] = 0.0
    for p in (gp, op):
        TO.set_initial_state(p, x0); TO.initial_controls(p, U); TO.rollout(p); TO.expand(p)
    X = TO.states(gp)
    assert np.allclose(X, TO.states(op), atol=1e-13)
    assert np.allclose(TO.dynamics_jacobians(gp), TO.dynamics_jacobians(op), atol=1e-13)
    # knot 6 is the jump map of knot 5: ((x3 + x4) / 2, (u1 + u2) / 2), exactly
    assert np.array_equal(X[:, 6, 0], (X[:, 5, 2] + X[:, 5, 3]) / 2) and np.array_equal(X[:, 6, 1], (U[:, 5, 0] + U[:, 5, 1]) / 2)
    for outer in range(4):
        for p in (gp, op):
            TO.ilqr_step(p, 6); TO.al_update(p)
    assert np.allclose(TO.states(gp), TO.states(op), atol=1e-7)
    assert np.allclose(TO.controls(gp), TO.controls(op), atol=1e-7)
    gp.close(); op.close()


def test_rebuild_keeps_the_rule():
    """a change of the objective rebuilds the handle (Problem._ensure_current): the new handle steps with the same rule"""
    p = P.cartpole(B=8, N=31, integration="Euler")
    TO.rollout(p)
    X = TO.states(p)
    sig = p._sig
    TO.set_LQR_goal(p.obj[0], np.array([0.1, np.pi, 0.0, 0.0]))
    assert isinstance(TO.integration(p), TO.Euler) and p._sig != sig
    TO.rollout(p)
    assert np.array_equal(TO.states(p), X)
    q = TO.copy_problem(p)
    assert isinstance(TO.integration(q), TO.Euler)
    p.close(); q.close()


def test_refusal_leaves_the_rule():
    p = P.cartpole(B=2, N=11, integration=TO.RK2)
    lib = p._lib
    assert lib.to_set_integration(p._h, 5) == TO.capi.TO_EINVAL and b"5" in lib.to_last_error(p._h)
    assert lib.to_set_integration(p._h, 0) == TO.capi.TO_EINVAL
    assert isinstance(TO.integration(p), TO.RK2)
    p.close()


# ---- the reference's recorded outputs (examples/Cartpole.ipynb, RK3, dt-scaled stage costs; tests/test_oracle_solve.py holds the oracle) ----
def _notebook_cartpole(**kw):
    return P.cartpole(B=1, N=101, dt_scaled_cost=True, integration=TO.RK3, **kw)


def test_cartpole_rollout_matches_the_notebooks_ipopt_log():
    """Ipopt's iteration-0 objective (cell 29, 2.4696994e-01): the dt-integrated stage costs of the RK3 rollout of U0 = 0.01"""
    p = _notebook_cartpole(u_bound=3.0, goal=True)
    TO.rollout(p)
    assert abs(TO.cost_knots(p)[0][:-1].sum() - 0.24696994) < 5e-9
    p.close()


def test_cartpole_ilqr_solve_reproduces_altros_recorded_summary():
    """HARD PIN: Altro's iLQRSolver (examples/Cartpole.ipynb:378-382, cost_tolerance 1e-4): 84 iterations, cost 1.4497436179031664,
    dJ 6.889787558717053e-5, gradient 0.038402688096996665"""
    p = _notebook_cartpole()
    st = TO.solve(p, cost_tolerance=1e-4)
    assert st.status_names() == ["SOLVE_SUCCEEDED"]
    assert st.iterations[0] == 84 and st.iterations_outer[0] == 1
    assert abs(st.cost[0] - 1.4497436179031664) < 1e-9
    assert abs(st.dJ[0] - 6.889787558717053e-5) < 1e-11
    assert abs(st.gradient[0] - 0.038402688096996665) < 1e-9
    p.close()


def test_cartpole_altro_solve_against_the_notebook():
    """the notebook's ALTRO run (examples/Cartpole.ipynb:216-223) to the oracle's soft pin (tests/test_oracle_solve.py)"""
    p = _notebook_cartpole(u_bound=3.0, goal=True)
    TO.set_options(p, penalty_initial=1.0, penalty_scaling=10.0)
    st = TO.solve(p, cost_tolerance_intermediate=1e-2, constraint_tolerance=1e-3)
    assert st.status_names() == ["SOLVE_SUCCEEDED"]
    assert st.c_max[0] < 1e-3
    assert abs(st.cost[0] - 1.552558743680986) < 2e-2
    assert 20 <= st.iterations[0] <= 80
    assert np.abs(TO.controls(p)).max() <= 3.0 + 1e-3
    p.close()
