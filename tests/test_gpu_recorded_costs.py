"""Costs of user dynamics models on the padded size classes (4, 2), (8, 4) and (16, 8) on the GPU (`-m gpu`), against the size-class
oracle (recorded_classes.ClassesOracleProblem) with the tolerances of test_gpu_recorded_classes.py.  A user cost (AutodiffCost) runs the
materialised expansion and k_riccati_dense (lie.cu); a dense QuadraticCost without one runs k_riccati (riccati.cu) and k_riccati_small.

  a. cost, gradient, Hessian and AL expansion of a dense QuadraticCost and a user cost at random states and controls, on each class;
  b. one iLQR step: K, d and the merit;
  c. solves to convergence: the planar quadrotor with a DARE terminal cost, and the 7-joint arm reaching with its end effector;
  d. a user cost restating a DiagonalCost solves to the DiagonalCost problem's result;
  e. the hybrid 6 -> 3 problem with QuadraticCosts on both sides;
  f. kernel_choice for each cost on each class;
  g. unconstrained solve_queue and mpc_solve with a user cost at (8, 4) equal chunked solve and the scripted loop, bit for bit."""
import numpy as np
import pytest

import trajopt_b200 as TO
from dynamics_programs import pad
from parity_util import GAIN_TOL, check, inst_err, triple
from recorded_classes import ClassesOracleProblem, on_class_oracle, planar_quadrotor_model
from recorded_costs import (CLASS_MODELS, HOVER, PLANAR_XF, arm_reach_problem, dense_cost, diagonal_as_user_cost, planar_dare_problem,
                            user_cost)
from test_gpu_dynamics_programs import report
from test_gpu_fullsize import ROLLOUT_TOL
from test_gpu_parity import KERNEL_RTOL
from test_gpu_solve import compare, sm_count

pytestmark = pytest.mark.gpu
K = TO.capi
CLASSES = sorted(CLASS_MODELS)
KINDS = ["dense", "user"]


def class_problem(cls_, size_class, kind, B=33, N=21, seed=0):
    """the class's model with a dense QuadraticCost or a user cost on every knot, a Bound and a Goal constraint, at random controls"""
    model = CLASS_MODELS[size_class]()
    nk, mk = model.n, model.m
    if kind == "dense":
        stage, term = dense_cost(nk, mk, 11), dense_cost(nk, mk, 12, terminal=True)
    else:
        stage, term = user_cost(nk, mk)[0], user_cost(nk, mk, terminal=True)[0]
    cons = TO.ConstraintList(nk, mk, N)
    TO.add_constraint(cons, TO.BoundConstraint(nk, mk, u_min=-3.0, u_max=3.0), (1, N - 1))
    TO.add_constraint(cons, TO.GoalConstraint(np.full(nk, 0.1)), N)
    r = np.random.default_rng(seed)
    p = cls_(model, TO.Objective([stage] * (N - 1) + [term]), 0.2 * r.standard_normal((B, nk)), 1.0, constraints=cons)
    U = 0.5 * r.standard_normal((B, N - 1, mk))
    if size_class == (8, 4):
        U += HOVER
    TO.initial_controls(p, pad(U, p.m))
    return p


# ---- a: cost, gradient, Hessian, AL expansion ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("size_class", CLASSES, ids=lambda c: f"{c[0]}x{c[1]}")
def test_cost_expansion(size_class, kind):
    g, o = (class_problem(c, size_class, kind) for c in (TO.Problem, ClassesOracleProblem))
    r = np.random.default_rng(5)
    nk, mk = CLASS_MODELS[size_class]().n, CLASS_MODELS[size_class]().m
    X, U = pad(r.uniform(-1, 1, (g.B, g.N, nk)), g.n), pad(r.uniform(-1, 1, (g.B, g.N - 1, mk)), g.m)
    for p in (g, o):
        TO.initial_states(p, X); TO.initial_controls(p, U)
        TO.al_update(p)            # nonzero multipliers
    errs = {"J": inst_err(TO.cost_knots(g), TO.cost_knots(o)).max(), "grad": inst_err(TO.cost_gradient(g), TO.cost_gradient(o)).max(),
            "hess": inst_err(TO.cost_hessian(g), TO.cost_hessian(o)).max()}
    (gg, hg), (go, ho) = TO.al_expansion(g), TO.al_expansion(o)
    errs["al grad"], errs["al hess"] = inst_err(gg, go).max(), inst_err(hg, ho).max()
    assert max(errs.values()) <= KERNEL_RTOL, errs
    report("a", f"{size_class} {kind} cost / grad / hess / AL expansion", max(errs.values()))
    g.close(); o.close()


# ---- b: one iLQR step ----------------------------------------------------------------------------------------------------------------------
def ilqr_step(size_class, kind, B=33):
    g, o = (class_problem(c, size_class, kind, B=B) for c in (TO.Problem, ClassesOracleProblem))
    for p in (g, o):
        TO.rollout(p); TO.expand(p); TO.backward(p)
    eX = inst_err(TO.states(g), TO.states(o)).max()
    assert eX <= ROLLOUT_TOL, eX
    (Kg, dg), (Ko, do) = TO.gains(g), TO.gains(o)
    eK = max(inst_err(Kg, Ko).max(), inst_err(dg, do).max())
    assert eK <= GAIN_TOL, eK
    mk = CLASS_MODELS[size_class]().m
    assert np.all(Kg[..., mk:, :] == 0.0) and np.all(dg[..., mk:] == 0.0)
    for p in (g, o):
        TO.ilqr_step(p, 1)
    same = TO.solver_state(g)["alpha"] == TO.solver_state(o)["alpha"]
    assert same.mean() >= 0.95
    eJ = float(np.max(np.abs(TO.merit(g) - TO.merit(o))[same] / np.maximum(1.0, np.abs(TO.merit(o)[same]))))
    assert eJ < 1e-6, eJ
    report("b", f"{size_class} {kind} {TO.kernel_choice(g)['backward']} K / d / merit", max(eK, eJ))
    g.close(); o.close()


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("size_class", CLASSES, ids=lambda c: f"{c[0]}x{c[1]}")
def test_ilqr_step(size_class, kind):
    ilqr_step(size_class, kind)


def test_ilqr_step_thread_kernel_at_4_2():
    """a dense QuadraticCost at (4, 2) past one wave of the warp kernel: k_riccati_small"""
    ilqr_step((4, 2), "dense", B=16 * sm_count() + 5)


# ---- c: solves -----------------------------------------------------------------------------------------------------------------------------
def test_solve_planar_quadrotor_with_a_dare_terminal_cost():
    p = planar_dare_problem(TO.Problem)
    assert (p.n, p.m) == (8, 4) and TO.kernel_choice(p)["backward"] == "warp_dfma"
    p.close()
    sg, ro = compare("planar quadrotor DARE", on_class_oracle(planar_dare_problem), iterations=80, allow=0.0)
    assert np.all(sg.status == ro.status) and np.all(sg.iterations == ro.iterations) and np.all(sg.iterations_outer == ro.iterations_outer)
    assert np.any(sg.status == K.SOLVE_SUCCEEDED)


def test_solve_arm_reaching_with_its_end_effector():
    p = arm_reach_problem(TO.Problem)
    assert (p.n, p.m) == (16, 8) and TO.kernel_choice(p)["backward"] == "dense_dfma"
    p.close()
    sg, ro = compare("7-joint arm end effector", on_class_oracle(arm_reach_problem), iterations=80, allow=0.0)
    assert np.all(sg.status == ro.status) and np.all(sg.iterations == ro.iterations) and np.all(sg.iterations_outer == ro.iterations_outer)
    assert np.any(sg.status == K.SOLVE_SUCCEEDED)


# ---- d: a user cost restating a DiagonalCost -----------------------------------------------------------------------------------------------
def planar_lqr(user, B=16, N=41):
    Qd, Rd, Qf = np.full(6, 0.1), np.full(2, 0.01), np.full(6, 50.0)
    if user:
        obj = TO.Objective([diagonal_as_user_cost(Qd, Rd, PLANAR_XF)] * (N - 1) + [diagonal_as_user_cost(Qf, Rd, PLANAR_XF, terminal=True)])
    else:
        obj = TO.LQRObjective(Qd, Rd, Qf, PLANAR_XF, N)
    cons = TO.ConstraintList(6, 2, N)
    TO.add_constraint(cons, TO.BoundConstraint(6, 2, u_min=0.0, u_max=12.0), (1, N - 1))
    r = np.random.default_rng(3)
    p = TO.Problem(planar_quadrotor_model(), obj, 0.1 * r.standard_normal((B, 6)), 2.0, constraints=cons)
    TO.initial_controls(p, pad(np.full((B, N - 1, 2), HOVER) + 0.3 * r.standard_normal((B, N - 1, 2)), 4))
    return p


def test_user_cost_restating_a_diagonal_cost():
    u, d = planar_lqr(True), planar_lqr(False)
    assert TO.kernel_choice(u)["backward"] == "dense_dfma" and TO.kernel_choice(d)["backward"] != "dense_dfma"
    su, sd = TO.solve(u, iterations=80), TO.solve(d, iterations=80)
    same = (su.iterations == sd.iterations) & (su.status == sd.status)
    assert same.mean() >= 0.9 and np.any(su.status == K.SOLVE_SUCCEEDED)
    eX = inst_err(TO.states(u)[same], TO.states(d)[same]).max()
    eU = inst_err(TO.controls(u)[same], TO.controls(d)[same]).max()
    eJ = float(np.max(np.abs(su.cost - sd.cost)[same] / np.maximum(1.0, np.abs(sd.cost[same]))))
    assert max(eX, eU) <= 1e-6 and eJ <= 1e-8, (eX, eU, eJ)
    report("d", "user cost vs DiagonalCost X / U / cost", max(eX, eU, eJ))
    u.close(); d.close()


# ---- e: the hybrid 6 -> 3 problem with QuadraticCosts ----------------------------------------------------------------------------------
def hybrid_quadratic(cls, B=64):
    a = planar_quadrotor_model()
    jump = TO.AutodiffDynamics(6, 2, lambda x, u: [x[0] + 0.1 * TO.sin(x[2]), x[1], x[3] * TO.cos(x[2]) + 0.1 * u[0]], output_dim=3, discrete=True)
    b = TO.AutodiffDynamics(3, 1, lambda x, u: [x[2], -0.2 * x[1], u[0] - 0.3 * x[2]])
    models = [a] * 6 + [jump] + [b] * 6
    nx, nu = TO.dims(models)
    N = len(nx)
    costs = {(6, 2): dense_cost(6, 2, 21), (3, 1): dense_cost(3, 1, 22)}
    obj = TO.Objective([costs[(nx[k], nu[k])] for k in range(N - 1)] + [dense_cost(3, 1, 23, terminal=True)])
    cons = TO.ConstraintList(models)
    TO.add_constraint(cons, TO.BoundConstraint(6, 2, u_min=0.0, u_max=12.0), (1, 6))
    TO.add_constraint(cons, TO.GoalConstraint(np.array([0.2, 0.0, 0.0])), N)
    r = np.random.default_rng(4)
    p = cls(models, obj, 0.2 * r.standard_normal((B, 6)), 1.2, constraints=cons)
    U = np.zeros((B, N - 1, 4))
    for k in range(N - 1):
        U[:, k, :nu[k]] = (HOVER if nu[k] == 2 else 0.0) + 0.3 * r.standard_normal((B, nu[k]))
    TO.initial_controls(p, U)
    return p


def test_hybrid_problem_with_quadratic_costs():
    g, o, t = triple(on_class_oracle(hybrid_quadratic))
    assert (g.n, g.m) == (8, 4) and TO.kernel_choice(g)["backward"] == "warp_dfma"
    for p in (g, o, t):
        TO.rollout(p); TO.expand(p)
    eX = inst_err(TO.states(g), TO.states(o)).max()
    assert eX <= ROLLOUT_TOL, eX
    for p in (g, o, t):
        TO.ilqr_step(p, 4); TO.al_update(p); TO.ilqr_step(p, 2)
    sgs, sos, sts = TO.solver_state(g), TO.solver_state(o), TO.solver_state(t)
    live = np.abs(sos["dV"][:, 0]) > 1e-9 * np.maximum(1.0, np.abs(TO.merit(o)))
    dec = live & (sos["alpha"] == sts["alpha"]) & (sgs["alpha"] == sos["alpha"])
    e = max(check("X", TO.states(g), TO.states(o), TO.states(t), 1e-8, dec)[0], check("U", TO.controls(g), TO.controls(o), TO.controls(t), 1e-8, dec)[0])
    report("e", "hybrid (8, 4) QuadraticCost iterates", e)
    X, U = TO.states(g), TO.controls(g)
    for k in range(g.N):
        assert np.all(X[:, k, g.nx[k]:] == 0.0)
        if k < g.N - 1:
            assert np.all(U[:, k, g.nu[k]:] == 0.0)


# ---- f: kernel_choice ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("size_class", CLASSES, ids=lambda c: f"{c[0]}x{c[1]}")
def test_kernel_choice(size_class):
    """a user cost takes the materialised expansion and the dense DFMA pass; a dense QuadraticCost keeps the in-kernel expansion"""
    B = 16 * sm_count() + 5           # past one wave of the warp kernel
    user, dense = class_problem(TO.Problem, size_class, "user", B=B), class_problem(TO.Problem, size_class, "dense", B=B)
    assert TO.kernel_choice(user)["backward"] == "dense_dfma"
    assert TO.kernel_choice(dense)["backward"] == ("thread" if size_class == (4, 2) else "warp_dfma")
    user.close(); dense.close()


# ---- g: the queue and MPC with a user cost at (8, 4) ---------------------------------------------------------------------------------------
def unconstrained_user(B=32, N=21):
    xf = np.array([0.5, 0.3, 0.0, 0.0, 0.0, 0.0])
    obj = TO.Objective([diagonal_as_user_cost(np.full(6, 0.1), np.full(2, 0.01), xf)] * (N - 1) +
                       [diagonal_as_user_cost(np.full(6, 50.0), np.full(2, 0.01), xf, terminal=True)])
    x0 = 0.1 * np.random.default_rng(2).standard_normal((B, 6))
    p = TO.Problem(planar_quadrotor_model(), obj, x0, 1.0)
    TO.initial_controls(p, np.full((B, N - 1, 4), HOVER) * np.array([1.0, 1.0, 0.0, 0.0]))
    return p


def test_solve_queue_with_a_user_cost_is_chunked_solve():
    B, M, N = 16, 40, 21
    r = np.random.default_rng(9)
    mask = np.array([1.0, 1.0, 0.0, 0.0])
    x0s = 0.1 * r.standard_normal((M, 6))
    U0s = np.full((M, N - 1, 4), HOVER) * mask + 0.1 * r.standard_normal((M, N - 1, 4)) * mask
    q = unconstrained_user(B, N)
    assert TO.kernel_choice(q)["backward"] == "dense_dfma"
    res = TO.solve_queue(q, pad(x0s, 8), U0s)
    for c0 in range(0, M, B):
        idx = np.arange(c0, min(c0 + B, M))
        p = unconstrained_user(B, N)
        xs, us = np.zeros((B, 8)), np.zeros((B, N - 1, 4))
        xs[:len(idx)], us[:len(idx)] = pad(x0s[idx], 8), U0s[idx]
        TO.set_initial_state(p, xs); TO.initial_controls(p, us)
        st = TO.solve(p)
        for f in TO.SolveStats.FIELDS:
            assert np.array_equal(getattr(res, f)[idx], getattr(st, f)[:len(idx)]), f
        assert np.array_equal(res.X[idx], TO.states(p)[:len(idx)]) and np.array_equal(res.U[idx], TO.controls(p)[:len(idx)])
        p.close()
    q.close()


def test_mpc_solve_with_a_user_cost_is_the_scripted_solve_loop():
    from test_gpu_mpc import _plant
    from test_gpu_mpc_solve import _assert_history, _equal, _full_state, _scripted
    dev, scr = unconstrained_user(), unconstrained_user()
    steps, opts = 4, dict(iterations=6)
    TO.mpc_setup(dev, steps)
    plant = _plant(scr)
    TO.mpc_solve(dev, steps, **opts)
    hist, stats = _scripted(scr, plant, steps, opts)
    _assert_history(dev, hist, stats, "planar quadrotor user cost mpc_solve")
    _equal(_full_state(dev), _full_state(scr), "planar quadrotor user cost mpc_solve")
    for p in (dev, scr, plant):
        p.close()
