"""User dynamics models of the padded size classes (8, 4) and (16, 8) on the GPU (`-m gpu`), against the oracle with the tolerances of
test_gpu_dynamics_programs.py.  The classes are the kernel instances MODEL_EXPR_84 / MODEL_EXPR_168 (csrc/models.cuh) and k_riccati<8, 4>
(tensor-MMA and DFMA micro-block kernels) and <16, 8> (DFMA kernel).  The oracle side is recorded_classes.ClassesOracleProblem, the oracle's
sources with the size classes (tests/oracle_classes.cpp).

  A. every op code in each class, explicit rule and jump map: rollout, [A B] and its padded rows / columns, and the padded control rows of
     K and d;
  B. a recorded copy of the Quadrotor (13, 4), run as class (16, 8), against the built-in CUDA Quadrotor on the full-state path and the
     oracle (controls kept positive, so that the built-in's relu on thrust is the identity);
  C. solve to convergence: a planar quadrotor at (8, 4) on both sides of the MMA / DFMA choice, and a 7-joint arm (14, 7) at (16, 8);
     every explicit rule on (8, 4);
  D. a hybrid problem whose largest knot needs class (8, 4): 6 -> 3 states through a jump map;
  E. mpc_run, unconstrained mpc_solve and unconstrained solve_queue on an (8, 4) model equal the scripted loop and chunked solve, bit for bit;
  F. to_create takes only the class of a spec."""
import ctypes as C

import numpy as np
import pytest

import trajopt_b200 as TO
from dynamics_programs import pad
from parity_util import GAIN_TOL, check, decisions_agree, inst_err, triple
from recorded_classes import (CLASS_PROGRAMS, ClassesOracleProblem, arm7_model, class_model, on_class_oracle, padded_closed_form,
                              planar_quadrotor_model, quadrotor_model)
from test_gpu_dynamics_programs import nonuniform_dt, report
from test_gpu_fullsize import ROLLOUT_TOL
from test_gpu_parity import KERNEL_RTOL
from test_gpu_solve import compare

pytestmark = pytest.mark.gpu
K = TO.capi


def both(build):
    return build(TO.Problem), build(ClassesOracleProblem)


# ---- A: every op code in each class ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("discrete", [False, True], ids=["rk4", "jump_map"])
@pytest.mark.parametrize("name", sorted(CLASS_PROGRAMS))
def test_every_op_in_each_class(name, discrete):
    model = class_model(name, discrete)
    n, m = model.n, model.m
    cn, cm = K.recorded_dims(n, m)
    B, N = 37, 21
    dt = nonuniform_dt(N, 0.4)

    def build(cls):
        obj = TO.LQRObjective(np.ones(n), np.ones(m), np.ones(n), np.zeros(n), N)
        return cls(model, obj, np.zeros(n), 0.4, dt=dt, batch=B)
    g, o = both(build)
    assert (g.n, g.m) == (cn, cm)
    r = np.random.default_rng(7)
    X = pad(r.uniform(-1.0, 1.0, (B, N, n)), cn)
    U = pad(r.uniform(-1.0, 1.0, (B, N - 1, m)), cm)
    X[:, :, 0] = np.linspace(-1.0, 1.0, B)[:, None]             # tanh(4 x0) over [-4, 4]
    for p in (g, o):
        TO.initial_states(p, X); TO.initial_controls(p, U); TO.expand(p)
    ABg, ABo = TO.dynamics_jacobians(g), TO.dynamics_jacobians(o)
    e = inst_err(ABg, ABo).max()
    assert e <= KERNEL_RTOL, f"[A B] {e:.3e}"
    closed, mask = padded_closed_form(model, cn, cm)
    assert np.array_equal(ABg[..., mask], np.broadcast_to(closed[mask], ABg.shape[:2] + (int(mask.sum()),)))
    report("A", f"{name}-{'jump' if discrete else 'rk4'} [A B]", e)
    if not discrete:        # the gains of the padded controls: zero columns of B, unit weights
        for p in (g, o):
            TO.backward(p)
        (Kg, dg), (Ko, do) = TO.gains(g), TO.gains(o)
        assert max(inst_err(Kg, Ko).max(), inst_err(dg, do).max()) <= GAIN_TOL
        assert np.all(Kg[..., m:, :] == 0.0) and np.all(dg[..., m:] == 0.0)
    x0 = pad(r.uniform(-1.0, 1.0, (B, n)), cn)
    for p in (g, o):
        TO.set_initial_state(p, x0); TO.rollout(p)
    Xg, Xo = TO.states(g), TO.states(o)
    steps = 2 if discrete else N
    e = inst_err(Xg[:, :steps], Xo[:, :steps]).max()
    assert np.all(np.isfinite(Xo[:, :steps])) and e <= ROLLOUT_TOL, f"rollout {e:.3e}"
    assert np.all(Xg[:, :, n:] == 0.0)
    report("A", f"{name}-{'jump' if discrete else 'rk4'} rollout", e)


# ---- B: a recorded copy of the Quadrotor at (16, 8) ----------------------------------------------------------------------------------------
def quadrotor_problem(cls, model, B=29, N=51):
    """hover with a small displacement of the goal, so that every iterate keeps every thrust well above zero (the built-in's relu is the
    identity on them)"""
    x0 = np.zeros((B, 13)); x0[:, 3] = 1.0
    x0[:, :3] = 0.05 * np.random.default_rng(8).standard_normal((B, 3))
    xf = np.zeros(13); xf[3] = 1.0; xf[:3] = [0.05, -0.05, 0.05]
    obj = TO.LQRObjective(np.full(13, 1.0), np.full(4, 10.0), np.full(13, 1.0), xf, N)
    cons = TO.ConstraintList(13, 4, N)
    TO.add_constraint(cons, TO.BoundConstraint(13, 4, u_min=0.2, u_max=6.0), (1, N - 1))
    return cls(model, obj, x0, 0.05 * (N - 1), xf=xf, constraints=cons, dt=0.05)


def test_recorded_quadrotor_at_16_8_against_the_builtin():
    B, N = 29, 51
    gb = quadrotor_problem(TO.Problem, TO.Quadrotor(), B, N)
    g, o, t = triple(on_class_oracle(lambda cls: quadrotor_problem(cls, quadrotor_model(), B, N)))
    assert (g.n, g.m) == (16, 8) and TO.kernel_choice(g)["backward"] == "warp_dfma"
    r = np.random.default_rng(3)
    U = TO.Quadrotor().hover_control() * (1.0 + 0.001 * r.uniform(-1.0, 1.0, (B, N - 1, 4)))    # strictly positive thrust
    TO.initial_controls(gb, U)
    for p in (g, o, t):
        TO.initial_controls(p, pad(U, 8))
    for p in (gb, g, o, t):
        TO.rollout(p); TO.expand(p)
    Xb, Xg, Xo = TO.states(gb), TO.states(g), TO.states(o)
    e_rec, e_orc = inst_err(Xg[..., :13], Xb).max(), inst_err(Xg, Xo).max()
    assert e_rec <= ROLLOUT_TOL and e_orc <= ROLLOUT_TOL and np.all(Xg[..., 13:] == 0.0), (e_rec, e_orc)
    report("B", "quadrotor rollout rec-vs-builtin / gpu-vs-oracle", max(e_rec, e_orc))
    ABb, ABg, ABo = TO.dynamics_jacobians(gb), TO.dynamics_jacobians(g), TO.dynamics_jacobians(o)
    lead = np.concatenate([ABg[..., :13, :13], ABg[..., :13, 16:20]], axis=-1)
    e_rec, e_orc = inst_err(lead, ABb).max(), inst_err(ABg, ABo).max()
    assert e_rec <= ROLLOUT_TOL and e_orc <= ROLLOUT_TOL, (e_rec, e_orc)
    closed, mask = padded_closed_form(g.model[0], 16, 8)
    assert np.array_equal(ABg[..., mask], np.broadcast_to(closed[mask], ABg.shape[:2] + (int(mask.sum()),)))
    report("B", "quadrotor [A B] rec-vs-builtin / gpu-vs-oracle", max(e_rec, e_orc))
    sb, sg, so = TO.backward(gb), TO.backward(g), TO.backward(o)
    TO.backward(t)
    assert np.array_equal(sg, so) and np.array_equal(sg, sb)
    (Kb, db), (Kg, dg), (Ko, do) = TO.gains(gb), TO.gains(g), TO.gains(o)
    errs = [inst_err(Kg, Ko).max(), inst_err(dg, do).max(), inst_err(TO.solver_state(g)["dV"], TO.solver_state(o)["dV"]).max(),
            inst_err(Kg[..., :4, :13], Kb).max(), inst_err(dg[..., :4], db).max(), inst_err(TO.solver_state(g)["dV"], TO.solver_state(gb)["dV"]).max()]
    assert max(errs) <= GAIN_TOL, errs
    assert np.all(Kg[..., 4:, :] == 0.0) and np.all(dg[..., 4:] == 0.0)
    report("B", "quadrotor K/d/dV gpu-vs-oracle, rec-vs-builtin", max(errs))
    for p in (gb, g, o, t):
        TO.ilqr_step(p, 3); TO.al_update(p); TO.ilqr_step(p, 2)
    sgs, sos, sts = TO.solver_state(g), TO.solver_state(o), TO.solver_state(t)
    live = np.abs(sos["dV"][:, 0]) > 1e-9 * np.maximum(1.0, np.abs(TO.merit(o)))
    dec = live & (sos["alpha"] == sts["alpha"]) & (sgs["alpha"] == sos["alpha"])
    e1, _ = check("X after AL-iLQR", TO.states(g), TO.states(o), TO.states(t), 1e-8, dec)
    e2, _ = check("U after AL-iLQR", TO.controls(g), TO.controls(o), TO.controls(t), 1e-8, dec)
    e3, _ = check("X recorded vs built-in", pad(TO.states(gb), 16), TO.states(o), TO.states(t), 1e-8, dec)
    assert np.all(TO.controls(g)[..., 4:] == 0.0) and TO.controls(gb).min() > 0.0
    report("B", "quadrotor iterates gpu-vs-oracle / builtin-vs-oracle", max(e1, e2, e3))


# ---- C: solves -----------------------------------------------------------------------------------------------------------------------------
def planar_problem(cls, B=8, N=41, general=False, integration=TO.RK4, seed=0):
    model = planar_quadrotor_model()
    xf = np.array([1.0, 0.5, 0.0, 0.0, 0.0, 0.0])
    obj = TO.LQRObjective(np.full(6, 0.1), np.full(2, 0.01), np.full(6, 50.0), xf, N)
    cons = TO.ConstraintList(6, 2, N)
    TO.add_constraint(cons, TO.BoundConstraint(6, 2, u_min=0.0, u_max=12.0), (1, N - 1))
    TO.add_constraint(cons, TO.GoalConstraint(xf), N)
    if general:     # a state constraint the diagonal kernels do not take: the DFMA micro-block kernel of k_riccati<8, 4>
        TO.add_constraint(cons, TO.CircleConstraint(6, [0.5], [0.2], [0.15]), (2, N - 1))
    r = np.random.default_rng(seed)
    x0 = 0.1 * r.standard_normal((B, 6))
    p = cls(model, obj, x0, 2.0, xf=xf, constraints=cons, integration=integration)
    TO.initial_controls(p, pad(np.full((B, N - 1, 2), 4.905) + 0.3 * r.standard_normal((B, N - 1, 2)), 4))
    return p


def arm7_problem(cls, B=8, N=41, seed=1):
    model = arm7_model()
    xf = np.concatenate([np.full(7, 0.5), np.zeros(7)])
    obj = TO.LQRObjective(np.full(14, 0.1), np.full(7, 0.01), np.full(14, 50.0), xf, N)
    cons = TO.ConstraintList(14, 7, N)
    TO.add_constraint(cons, TO.BoundConstraint(14, 7, u_min=-4.0, u_max=4.0), (1, N - 1))
    TO.add_constraint(cons, TO.GoalConstraint(xf), N)
    r = np.random.default_rng(seed)
    p = cls(model, obj, 0.1 * r.standard_normal((B, 14)), 2.0, xf=xf, constraints=cons)
    TO.initial_controls(p, pad(0.3 * r.standard_normal((B, N - 1, 7)), 8))
    return p


@pytest.mark.parametrize("general,kernel", [(False, "warp_mma"), (True, "warp_dfma")])
def test_solve_planar_quadrotor_at_8_4(general, kernel):
    p = planar_problem(TO.Problem, general=general)
    assert (p.n, p.m) == (8, 4) and TO.kernel_choice(p)["backward"] == kernel
    p.close()
    sg, ro = compare(f"planar quadrotor {kernel}", on_class_oracle(lambda cls: planar_problem(cls, general=general)), iterations=80)
    assert np.any(sg.status == K.SOLVE_SUCCEEDED) and np.any(sg.iterations_outer > 1)


def test_solve_seven_joint_arm_at_16_8():
    p = arm7_problem(TO.Problem)
    assert (p.n, p.m) == (16, 8) and TO.kernel_choice(p)["backward"] == "warp_dfma"
    p.close()
    sg, ro = compare("7-joint arm", on_class_oracle(arm7_problem), iterations=80)
    assert np.any(sg.status == K.SOLVE_SUCCEEDED)


@pytest.mark.parametrize("rule", ["Euler", "RK2", "RK3", "RK4"])
def test_every_rule_at_8_4(rule):
    """the size-class oracle, which has every explicit rule: rollout, [A B], gains and one AL-iLQR iteration"""
    g, o = planar_problem(TO.Problem, B=33, integration=rule), planar_problem(ClassesOracleProblem, B=33, integration=rule)
    assert type(TO.integration(g)) is type(TO.integration(o))
    for p in (g, o):
        TO.rollout(p); TO.expand(p); TO.backward(p)
    eX, eAB = inst_err(TO.states(g), TO.states(o)).max(), inst_err(TO.dynamics_jacobians(g), TO.dynamics_jacobians(o)).max()
    assert eX <= ROLLOUT_TOL and eAB <= ROLLOUT_TOL, (eX, eAB)
    (Kg, dg), (Ko, do) = TO.gains(g), TO.gains(o)
    eK = max(inst_err(Kg, Ko).max(), inst_err(dg, do).max())
    assert eK <= GAIN_TOL, eK
    for p in (g, o):
        TO.ilqr_step(p, 1)
    same = TO.solver_state(g)["alpha"] == TO.solver_state(o)["alpha"]
    assert same.mean() >= 0.95
    eJ = float(np.max(np.abs(TO.merit(g) - TO.merit(o))[same] / np.maximum(1.0, np.abs(TO.merit(o)[same]))))
    assert eJ < 1e-6, eJ
    report("C", f"planar quadrotor {rule} rollout / [A B] / K d / merit", max(eX, eAB, eK, eJ))


# ---- D: hybrid problem on class (8, 4) -----------------------------------------------------------------------------------------------------
def hybrid_problem(cls, B=64):
    a = planar_quadrotor_model()
    jump = TO.AutodiffDynamics(6, 2, lambda x, u: [x[0] + 0.1 * TO.sin(x[2]), x[1], x[3] * TO.cos(x[2]) + 0.1 * u[0]], output_dim=3, discrete=True)
    b = TO.AutodiffDynamics(3, 1, lambda x, u: [x[2], -0.2 * x[1], u[0] - 0.3 * x[2]])
    models = [a] * 6 + [jump] + [b] * 6
    nx, nu = TO.dims(models)
    N = len(nx)
    obj = TO.Objective([TO.LQRCost(np.full(nx[k], 0.5), np.full(nu[k], 0.1), np.zeros(nx[k]), terminal=(k == N - 1)) for k in range(N)])
    cons = TO.ConstraintList(models)
    TO.add_constraint(cons, TO.BoundConstraint(6, 2, u_min=0.0, u_max=12.0), (1, 6))
    TO.add_constraint(cons, TO.GoalConstraint(np.array([0.2, 0.0, 0.0])), N)
    r = np.random.default_rng(4)
    p = cls(models, obj, 0.2 * r.standard_normal((B, 6)), 1.2, constraints=cons)
    U = np.zeros((B, N - 1, 4))
    for k in range(N - 1):
        U[:, k, :nu[k]] = (4.905 if nu[k] == 2 else 0.0) + 0.3 * r.standard_normal((B, nu[k]))
    TO.initial_controls(p, U)
    return p


def test_hybrid_problem_runs_on_its_largest_knots_class():
    g, o, t = triple(on_class_oracle(hybrid_problem))
    assert (g.n, g.m) == (8, 4) and g.nx == [6] * 7 + [3] * 7
    for p in (g, o, t):
        TO.rollout(p); TO.expand(p)
    eX, eAB = inst_err(TO.states(g), TO.states(o)).max(), inst_err(TO.dynamics_jacobians(g), TO.dynamics_jacobians(o)).max()
    assert eX <= ROLLOUT_TOL and eAB <= ROLLOUT_TOL, (eX, eAB)
    for p in (g, o, t):
        TO.ilqr_step(p, 4); TO.al_update(p); TO.ilqr_step(p, 2)
    sgs, sos, sts = TO.solver_state(g), TO.solver_state(o), TO.solver_state(t)
    live = np.abs(sos["dV"][:, 0]) > 1e-9 * np.maximum(1.0, np.abs(TO.merit(o)))
    dec = live & (sos["alpha"] == sts["alpha"]) & (sgs["alpha"] == sos["alpha"])
    e = max(check("X", TO.states(g), TO.states(o), TO.states(t), 1e-8, dec)[0], check("U", TO.controls(g), TO.controls(o), TO.controls(t), 1e-8, dec)[0])
    report("D", "hybrid (8, 4) iterates", e)
    X, U = TO.states(g), TO.controls(g)
    for k in range(g.N):
        assert np.all(X[:, k, g.nx[k]:] == 0.0)
        if k < g.N - 1:
            assert np.all(U[:, k, g.nu[k]:] == 0.0)


# ---- E: MPC and the queue on an (8, 4) model -------------------------------------------------------------------------------------------
def unconstrained_planar(B=32, N=21):
    model = planar_quadrotor_model()
    xf = np.array([0.5, 0.3, 0.0, 0.0, 0.0, 0.0])
    obj = TO.LQRObjective(np.full(6, 0.1), np.full(2, 0.01), np.full(6, 50.0), xf, N)
    x0 = 0.1 * np.random.default_rng(2).standard_normal((B, 6))
    p = TO.Problem(model, obj, x0, 1.0)
    TO.initial_controls(p, np.full((B, N - 1, 4), 4.905) * np.array([1.0, 1.0, 0.0, 0.0]))
    return p


def test_mpc_run_is_the_scripted_loop_at_8_4():
    from test_gpu_mpc import _equal, _plant, _scripted, _state
    dev, scr = unconstrained_planar(), unconstrained_planar()
    assert (dev.n, dev.m) == (8, 4)
    steps, iters = 5, 2
    TO.mpc_setup(dev, steps)
    plant = _plant(scr)
    TO.mpc_run(dev, steps, iters)
    X, U, J = TO.mpc_history(dev)
    Xs, Us, Js = _scripted(scr, plant, steps, iters)
    assert np.array_equal(X, Xs) and np.array_equal(U, Us) and np.array_equal(J, Js)
    _equal(_state(dev), _state(scr), "planar quadrotor mpc_run")
    assert not np.array_equal(X[:, 0], X[:, -1])
    for p in (dev, scr, plant):
        p.close()


def test_mpc_solve_is_the_scripted_solve_loop_at_8_4():
    from test_gpu_mpc import _plant
    from test_gpu_mpc_solve import _assert_history, _equal, _full_state, _scripted
    dev, scr = unconstrained_planar(), unconstrained_planar()
    steps, opts = 4, dict(iterations=6)
    TO.mpc_setup(dev, steps)
    plant = _plant(scr)
    TO.mpc_solve(dev, steps, **opts)
    hist, stats = _scripted(scr, plant, steps, opts)
    _assert_history(dev, hist, stats, "planar quadrotor mpc_solve")
    _equal(_full_state(dev), _full_state(scr), "planar quadrotor mpc_solve")
    for p in (dev, scr, plant):
        p.close()


def test_solve_queue_is_chunked_solve_at_8_4():
    B, M, N = 16, 40, 21
    r = np.random.default_rng(9)
    x0s = 0.1 * r.standard_normal((M, 6))
    U0s = np.full((M, N - 1, 4), 4.905) * np.array([1.0, 1.0, 0.0, 0.0]) + 0.1 * r.standard_normal((M, N - 1, 4)) * np.array([1.0, 1.0, 0.0, 0.0])
    q = unconstrained_planar(B, N)
    res = TO.solve_queue(q, pad(x0s, 8), U0s)
    for c0 in range(0, M, B):
        idx = np.arange(c0, min(c0 + B, M))
        p = unconstrained_planar(B, N)
        xs, us = np.zeros((B, 8)), np.zeros((B, N - 1, 4))
        xs[:len(idx)], us[:len(idx)] = pad(x0s[idx], 8), U0s[idx]
        TO.set_initial_state(p, xs); TO.initial_controls(p, us)
        st = TO.solve(p)
        for f in TO.SolveStats.FIELDS:
            assert np.array_equal(getattr(res, f)[idx], getattr(st, f)[:len(idx)]), f
        assert np.array_equal(res.X[idx], TO.states(p)[:len(idx)]) and np.array_equal(res.U[idx], TO.controls(p)[:len(idx)])
        p.close()
    q.close()


# ---- F: to_create takes only the class ------------------------------------------------------------------------------------------------------
def test_to_create_takes_only_the_class():
    from test_recorded_classes import class_spec
    lib = K.load_library()
    model = planar_quadrotor_model()
    for (n, m), want in (((8, 4), K.TO_OK), ((4, 2), K.TO_EDIM), ((16, 8), K.TO_EDIM), ((6, 2), K.TO_EDIM)):
        h = C.c_void_p()
        rc = lib.to_create(C.byref(class_spec(model, n, m).c), C.byref(h))
        assert rc == want, (n, m, lib.to_last_error(None))
        if want == K.TO_OK:
            assert h
            lib.to_destroy(h)
        else:
            assert not h and "run on the padded size class n = 8, m = 4" in lib.to_last_error(None).decode()
    for field, v in (("n_in", 9), ("m_in", 5), ("n_out", 9)):
        d = dict(model._spec()); d[field] = v
        h = C.c_void_p()
        assert lib.to_create(C.byref(class_spec(model, 8, 4, dyn=d).c), C.byref(h)) == K.TO_EINVAL and not h
