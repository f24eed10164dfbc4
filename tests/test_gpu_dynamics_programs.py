"""User dynamics models (AutodiffDynamics, TO_MODEL_EXPR) on the GPU against the oracle (`-m gpu`).  The device interprets the recorded
program with dual numbers (csrc/models.cuh dynamics<MODEL_EXPR_42>); the oracle's interpreter is pinned to NumPy and central differences
in test_oracle_dynamics_programs.py.

  A. every op code, RK4 and jump map, one random state / control per instance and knot, and the program at the 128-instruction /
     64-constant limit: rollout and [A B];
  B. recorded copies of the built-in models against the built-in CUDA models and the oracle: rollout, [A B] and its padded rows /
     columns, the gains and their padded control row, iterates;
  C. the whole solver on nonlinear user models: every backward kernel choice (the automatic one past 16 x the SM count resolves to the
     thread-per-instance kernel), N = 2, 3, 101, non-uniform time steps, Goal + Bound and a general constraint (the generic AL path);
  D. a hybrid problem 4 -> 2 -> 3 states through two nonlinear jump maps, with 2, 1 and 0 controls;
  E. Problem(model, ...) is Problem([model] * (N - 1), ...);
  F. to_create rejects malformed programs."""
import ctypes as C

import numpy as np
import pytest

import trajopt_b200 as TO
from dynamics_programs import BUILTINS, OP_PROGRAMS, builtin_problem, malformed_specs, op_model, pad, padded_closed_form, recorded_builtin
from oracle_binding import OracleProblem
from parity_util import GAIN_TOL, check, decisions_agree, inst_err, triple, triple_with_options
from test_gpu_fullsize import ROLLOUT_TOL
from test_gpu_parity import KERNEL_RTOL

pytestmark = pytest.mark.gpu
K = TO.capi


def report(group, what, err):
    print(f"\nMAXERR {group} {what} {err:.3e}")


def nonuniform_dt(N, tf, seed=0):
    w = 0.6 + 0.8 * np.random.default_rng(seed).random(N - 1)
    return tf * w / w.sum()


def both(build):
    return build(TO.Problem), build(OracleProblem)


# ---- A: every op code, GPU vs oracle -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("discrete", [False, True], ids=["rk4", "jump_map"])
@pytest.mark.parametrize("name", sorted(OP_PROGRAMS) + ["limit"])
def test_every_op_matches_the_oracle(name, discrete):
    model = op_model(name, discrete)
    B, N = 37, 21
    n, m = model.n, model.m
    dt = nonuniform_dt(N, 0.4)

    def build(cls):
        obj = TO.LQRObjective(np.ones(n), np.ones(m), np.ones(n), np.zeros(n), N)
        return cls(model, obj, np.zeros(n), 0.4, dt=dt, batch=B)
    g, o = both(build)
    r = np.random.default_rng(7)
    X = pad(r.uniform(-1.0, 1.0, (B, N, n)), 4)
    U = pad(r.uniform(-1.0, 1.0, (B, N - 1, m)), 2)
    if name == "transcendental":
        X[:, :, 0] = np.linspace(-1.0, 1.0, B)[:, None]         # tanh(4 x0) over [-4, 4]
    for p in (g, o):
        TO.initial_states(p, X); TO.initial_controls(p, U); TO.expand(p)
    ABg, ABo = TO.dynamics_jacobians(g), TO.dynamics_jacobians(o)
    e = inst_err(ABg, ABo).max()
    assert e <= KERNEL_RTOL, f"[A B] {e:.3e}"
    closed, mask = padded_closed_form(model)
    assert np.array_equal(ABg[..., mask], np.broadcast_to(closed[mask], ABg.shape[:2] + (int(mask.sum()),)))
    report("A", f"{name}-{'jump' if discrete else 'rk4'} [A B]", e)
    # rollout from random initial states (a jump map is iterated, so one step of it is compared: N = 2 semantics on knot 1)
    x0 = pad(r.uniform(-1.0, 1.0, (B, n)), 4)
    for p in (g, o):
        TO.set_initial_state(p, x0); TO.rollout(p)
    Xg, Xo = TO.states(g), TO.states(o)
    steps = 2 if discrete else N
    e = inst_err(Xg[:, :steps], Xo[:, :steps]).max()
    assert np.all(np.isfinite(Xo[:, :steps])) and e <= ROLLOUT_TOL, f"rollout {e:.3e}"
    assert np.all(Xg[:, :, n:] == 0.0)
    report("A", f"{name}-{'jump' if discrete else 'rk4'} rollout", e)


# ---- B: recorded copies of the built-in models --------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", BUILTINS)
def test_recorded_copies_match_the_builtin_cuda_models(name):
    rec_model, builtin = recorded_builtin(name)
    n, m = builtin.dims()
    B = 29
    gb = builtin_problem(name, TO.Problem, B, recorded=False)
    g, o, t = triple(lambda cls: builtin_problem(name, cls, B, recorded=True))
    r = np.random.default_rng(3)
    U = TO.controls(gb) + 0.3 * r.standard_normal(TO.controls(gb).shape)
    TO.initial_controls(gb, U)
    for p in (g, o, t):
        TO.initial_controls(p, pad(U, 2))
    for p in (gb, g, o, t):
        TO.rollout(p); TO.expand(p)
    Xb, Xg, Xo = TO.states(gb), TO.states(g), TO.states(o)
    e_rec, e_orc = inst_err(Xg[..., :n], Xb).max(), inst_err(Xg, Xo).max()
    assert e_rec <= ROLLOUT_TOL and e_orc <= ROLLOUT_TOL and np.all(Xg[..., n:] == 0.0)
    report("B", f"{name} rollout rec-vs-builtin / gpu-vs-oracle", max(e_rec, e_orc))
    ABb, ABg, ABo = TO.dynamics_jacobians(gb), TO.dynamics_jacobians(g), TO.dynamics_jacobians(o)
    lead = np.concatenate([ABg[..., :n, :n], ABg[..., :n, 4:4 + m]], axis=-1)
    e_rec, e_orc = inst_err(lead, ABb).max(), inst_err(ABg, ABo).max()
    assert e_rec <= ROLLOUT_TOL and e_orc <= ROLLOUT_TOL, (e_rec, e_orc)
    closed, mask = padded_closed_form(rec_model)
    assert np.array_equal(ABg[..., mask], np.broadcast_to(closed[mask], ABg.shape[:2] + (int(mask.sum()),)))
    report("B", f"{name} [A B] rec-vs-builtin / gpu-vs-oracle", max(e_rec, e_orc))
    sb, sg, so = TO.backward(gb), TO.backward(g), TO.backward(o)
    TO.backward(t)
    assert np.array_equal(sg, so) and np.array_equal(sg, sb)
    (Kb, db), (Kg, dg), (Ko, do) = TO.gains(gb), TO.gains(g), TO.gains(o)
    errs = [inst_err(Kg, Ko).max(), inst_err(dg, do).max(), inst_err(TO.solver_state(g)["dV"], TO.solver_state(o)["dV"]).max(),
            inst_err(Kg[..., :m, :n], Kb).max(), inst_err(dg[..., :m], db).max(), inst_err(TO.solver_state(g)["dV"], TO.solver_state(gb)["dV"]).max()]
    assert max(errs) <= GAIN_TOL, errs
    assert np.all(Kg[..., m:, :] == 0.0) and np.all(dg[..., m:] == 0.0)      # the padded control: zero column of B, unit weight
    report("B", f"{name} K/d/dV gpu-vs-oracle, rec-vs-builtin", max(errs))
    for p in (gb, g, o, t):
        TO.ilqr_step(p, 3); TO.al_update(p); TO.ilqr_step(p, 2)
    sgs, sos, sts = TO.solver_state(g), TO.solver_state(o), TO.solver_state(t)
    live = np.abs(sos["dV"][:, 0]) > 1e-9 * np.maximum(1.0, np.abs(TO.merit(o)))
    dec = live & (sos["alpha"] == sts["alpha"]) & (sgs["alpha"] == sos["alpha"])
    e1, _ = check("X after AL-iLQR", TO.states(g), TO.states(o), TO.states(t), 1e-8, dec)
    e2, _ = check("U after AL-iLQR", TO.controls(g), TO.controls(o), TO.controls(t), 1e-8, dec)
    e3, _ = check("X recorded vs built-in", pad(TO.states(gb), 4), TO.states(o), TO.states(t), 1e-8, dec)
    assert np.all(TO.controls(g)[..., m:] == 0.0)
    report("B", f"{name} iterates gpu-vs-oracle / builtin-vs-oracle", max(e1, e2, e3))


# ---- C: the whole solver on nonlinear user models -----------------------------------------------------------------------------------
def pendulum():
    return TO.AutodiffDynamics(2, 1, lambda x, u: [x[1], -9.81 * TO.sin(x[0]) - 0.1 * x[1] + u[0]])


def exp_tanh_powc():
    """(4, 2): exp, tanh and POWC in the dynamics the solver differentiates"""
    return TO.AutodiffDynamics(4, 2, lambda x, u: [x[2], x[3],
                                                   TO.tanh(u[0] - 0.2 * x[0]) * 2.0 - 0.1 * TO.exp(0.2 * x[2]),
                                                   u[1] / (1.0 + x[1] * x[1]) ** 1.5 - 0.3 * x[3]])


SOLVER_MODELS = {"pendulum": pendulum, "cartpole": lambda: recorded_builtin("cartpole")[0], "exp_tanh_powc": exp_tanh_powc}


def solver_problem(model_name, B, N, general=False, seed=0):
    def build(cls):
        model = SOLVER_MODELS[model_name]()
        n, m = model.n, model.m
        r = np.random.default_rng(seed)
        xf = np.zeros(n); xf[0] = 1.0
        obj = TO.LQRObjective(np.full(n, 0.1), np.full(m, 0.05), np.full(n, 20.0), xf, N)
        cons = TO.ConstraintList(n, m, N)
        TO.add_constraint(cons, TO.BoundConstraint(n, m, u_min=-2.0, u_max=2.0), (1, N - 1))
        TO.add_constraint(cons, TO.GoalConstraint(xf), N)
        if general:      # a state constraint the diagonal kernels do not take: the generic AL path of k_riccati<4, 2>
            TO.add_constraint(cons, TO.CircleConstraint(n, [0.5], [0.3], [0.2]), (2, N - 1))
        tf = 0.05 * (N - 1)
        x0 = 0.2 * r.standard_normal((B, n))
        p = cls(model, obj, x0, tf, xf=xf, constraints=cons, dt=nonuniform_dt(N, tf, seed))
        TO.initial_controls(p, pad(0.3 * r.standard_normal((B, N - 1, m)), 2))
        return p
    return build


def big_batch():
    import torch
    return 16 * torch.cuda.get_device_properties(0).multi_processor_count + 5


SOLVER_CASES = [   # (model, backward_kernel, B, N, general constraint)
    ("pendulum", 0, 1, 2, False), ("pendulum", 1, 33, 3, False), ("pendulum", 2, 33, 101, False), ("pendulum", 0, "big", 101, False),
    ("cartpole", 0, 33, 101, False), ("cartpole", 1, 1, 101, False), ("cartpole", 2, 33, 3, False), ("cartpole", 0, "big", 101, False),
    ("exp_tanh_powc", 0, 33, 101, False), ("exp_tanh_powc", 1, 33, 2, False), ("exp_tanh_powc", 2, 1, 101, False),
    ("exp_tanh_powc", 0, "big", 101, False), ("exp_tanh_powc", 0, 33, 101, True), ("pendulum", 2, 33, 51, True),
]


@pytest.mark.parametrize("case", SOLVER_CASES, ids=lambda c: f"{c[0]}-k{c[1]}-B{c[2]}-N{c[3]}{'-circle' if c[4] else ''}")
def test_solver_on_user_models(case):
    name, kernel, B, N, general = case
    if B == "big":
        B = big_batch()
        import torch
        assert B > 16 * torch.cuda.get_device_properties(0).multi_processor_count   # the automatic choice is the thread-per-instance kernel
    g, o, t = triple_with_options(solver_problem(name, B, N, general), {"backward_kernel": kernel})
    m = SOLVER_MODELS[name]().m
    n = SOLVER_MODELS[name]().n
    for p in (g, o, t):
        TO.rollout(p); TO.expand(p)
    sg, so = TO.backward(g), TO.backward(o)
    TO.backward(t)
    assert np.array_equal(sg, so), f"restarts cuda {np.unique(sg)} oracle {np.unique(so)}"
    (Kg, dg), (Ko, do) = TO.gains(g), TO.gains(o)
    errs = [inst_err(Kg, Ko).max(), inst_err(dg, do).max(), inst_err(TO.solver_state(g)["dV"], TO.solver_state(o)["dV"]).max()]
    assert max(errs) <= GAIN_TOL, errs
    assert np.all(Kg[..., m:, :] == 0.0) and np.all(dg[..., m:] == 0.0)
    report("C", f"{name}-k{kernel}-B{B}-N{N}{'-circle' if general else ''} K/d/dV", max(errs))
    (Jg, ag), (Jo, ao), (Jt, at) = TO.forward(g), TO.forward(o), TO.forward(t)
    ok = decisions_agree("accepted step sizes", ag, ao, at)
    check("J after forward pass", Jg, Jo, Jt, 1e-10, ok)
    decisions_agree("line-search trials", TO.solver_state(g)["ls_iters"], TO.solver_state(o)["ls_iters"], TO.solver_state(t)["ls_iters"])
    for p in (g, o, t):
        TO.ilqr_step(p, 3); TO.al_update(p); TO.ilqr_step(p, 2)
    sgs, sos, sts = TO.solver_state(g), TO.solver_state(o), TO.solver_state(t)
    live = np.abs(sos["dV"][:, 0]) > 1e-9 * np.maximum(1.0, np.abs(TO.merit(o)))
    dec = live & (sos["alpha"] == sts["alpha"]) & (sgs["alpha"] == sos["alpha"]) & (sgs["bp_status"] == sos["bp_status"])
    for k in ("alpha", "ls_iters", "bp_status"):
        decisions_agree(k, sgs[k], sos[k], sts[k], live, allow=0.05)
    e = max(check("merit", TO.merit(g), TO.merit(o), TO.merit(t), 1e-8, dec)[0],
            check("X", TO.states(g), TO.states(o), TO.states(t), 1e-8, dec)[0],
            check("U", TO.controls(g), TO.controls(o), TO.controls(t), 1e-8, dec)[0])
    for i in range(len(g.constraints)):
        e = max(e, check(f"multipliers {i}", TO.multipliers(g, i), TO.multipliers(o, i), TO.multipliers(t, i), 1e-8, dec)[0])
    assert np.all(TO.controls(g)[..., m:] == 0.0) and np.all(TO.states(g)[..., n:] == 0.0)
    report("C", f"{name}-k{kernel}-B{B}-N{N}{'-circle' if general else ''} iterates", e)


# ---- D: hybrid problem beyond the reference example ---------------------------------------------------------------------------------
def hybrid_models():
    a = TO.AutodiffDynamics(4, 2, lambda x, u: [x[2], x[3], u[0] - 0.3 * TO.sin(x[0]), u[1] + 0.2 * TO.tanh(x[1] - x[0])])
    j1 = TO.AutodiffDynamics(4, 2, lambda x, u: [TO.tanh(x[0] + 0.5 * x[2]) + 0.1 * u[0], TO.sin(x[1]) * (1.0 + 0.2 * x[3]) + 0.1 * u[1]],
                             output_dim=2, discrete=True)
    b = TO.AutodiffDynamics(2, 1, lambda x, u: [x[1], -4.0 * TO.sin(x[0]) - 0.2 * x[1] + u[0]])
    j2 = TO.AutodiffDynamics(2, 1, lambda x, u: [x[0], x[1], TO.exp(0.2 * x[0]) * u[0]], output_dim=3, discrete=True)
    c = TO.AutodiffDynamics(3, 0, lambda x, u: [x[1], -x[0] - 0.1 * x[1] + 0.5 * x[2], -0.3 * x[2] / TO.sqrt(1.0 + x[2] * x[2])])
    return [a] * 5 + [j1] + [b] * 4 + [j2] + [c] * 4


def hybrid_problem(B):
    def build(cls):
        models = hybrid_models()
        nx, nu = TO.dims(models)
        N = len(nx)
        obj = TO.Objective([TO.LQRCost(np.full(nx[k], 0.5), np.full(nu[k], 0.1), np.zeros(nx[k]), terminal=(k == N - 1)) for k in range(N)])
        cons = TO.ConstraintList(models)
        TO.add_constraint(cons, TO.BoundConstraint(4, 2, u_min=-3.0, u_max=3.0, x_max=[2.0, 2.0, np.inf, np.inf]), (1, 5))
        TO.add_constraint(cons, TO.GoalConstraint(np.array([0.5, -0.2, 0.0, 0.0]), inds=[1, 2]), 6)
        TO.add_constraint(cons, TO.BoundConstraint(2, 1, u_min=-2.0, u_max=2.0, x_max=[1.5, np.inf]), (7, 10))
        TO.add_constraint(cons, TO.GoalConstraint(np.array([0.3, 0.0])), 11)
        TO.add_constraint(cons, TO.BoundConstraint(3, 0, x_min=[-np.inf, -np.inf, -1.0], x_max=[np.inf, np.inf, 1.0]), (12, 15))
        TO.add_constraint(cons, TO.GoalConstraint(np.array([0.0, 0.0, 0.2]), inds=[3]), 16)
        r = np.random.default_rng(11)
        p = cls(models, obj, 0.3 * r.standard_normal((B, 4)), 1.5, constraints=cons, dt=nonuniform_dt(N, 1.5, 4))
        U = np.zeros((B, N - 1, 2))
        for k in range(N - 1):
            U[:, k, :nu[k]] = 0.3 * r.standard_normal((B, nu[k]))
        TO.initial_controls(p, U)
        return p
    return build


def test_hybrid_problem_with_nonlinear_jump_maps_and_a_control_free_phase():
    B = 300
    g, o, t = triple(hybrid_problem(B))
    nx, nu = g.nx, g.nu
    assert nx == [4] * 6 + [2] * 5 + [3] * 5 and nu == [2] * 6 + [1] * 5 + [0] * 5
    for p in (g, o, t):
        TO.rollout(p); TO.expand(p)
    eX = inst_err(TO.states(g), TO.states(o)).max()
    eAB = inst_err(TO.dynamics_jacobians(g), TO.dynamics_jacobians(o)).max()
    assert eX <= ROLLOUT_TOL and eAB <= ROLLOUT_TOL, (eX, eAB)
    report("D", "rollout / [A B]", max(eX, eAB))
    sg, so = TO.backward(g), TO.backward(o)
    TO.backward(t)
    assert np.array_equal(sg, so)
    (Kg, dg), (Ko, do) = TO.gains(g), TO.gains(o)
    e = max(inst_err(Kg, Ko).max(), inst_err(dg, do).max())
    assert e <= GAIN_TOL
    report("D", "K/d", e)
    for outer in range(3):
        for p in (g, o, t):
            TO.ilqr_step(p, 4); TO.al_update(p)
    sgs, sos, sts = TO.solver_state(g), TO.solver_state(o), TO.solver_state(t)
    live = np.abs(sos["dV"][:, 0]) > 1e-9 * np.maximum(1.0, np.abs(TO.merit(o)))
    dec = live & (sos["alpha"] == sts["alpha"]) & (sgs["alpha"] == sos["alpha"])
    e = max(check("X", TO.states(g), TO.states(o), TO.states(t), 1e-8, dec)[0],
            check("U", TO.controls(g), TO.controls(o), TO.controls(t), 1e-8, dec)[0],
            check("violation", TO.max_violation(g), TO.max_violation(o), TO.max_violation(t), 1e-8, dec)[0])
    report("D", "iterates", e)
    X, U = TO.states(g), TO.controls(g)
    for k in range(g.N):
        assert np.all(X[:, k, nx[k]:] == 0.0), f"padded states of knot {k + 1}"
        if k < g.N - 1:
            assert np.all(U[:, k, nu[k]:] == 0.0), f"padded controls of knot {k + 1}"
    assert np.all(U[:, 11:, :] == 0.0)                     # the control-free phase


# ---- E: Problem(model, ...) == Problem([model] * (N - 1), ...) ----------------------------------------------------------------------
@pytest.mark.parametrize("name", ["pendulum", "exp_tanh_powc"])
def test_single_model_is_the_model_vector_on_the_gpu(name):
    N, B = 41, 33
    single = solver_problem(name, B, N)(TO.Problem)
    model = single.model[0]
    tf = 0.05 * (N - 1)       # the time steps of solver_problem
    vec = TO.Problem([model] * (N - 1), single.obj, single.x0[:, :model.n], tf, xf=single.xf, constraints=single.constraints, dt=nonuniform_dt(N, tf, 0))
    TO.initial_controls(vec, TO.controls(single))
    assert single.hybrid and single.nx == vec.nx and single.nu == vec.nu
    for p in (single, vec):
        TO.rollout(p); TO.expand(p); TO.backward(p)
    for f in (TO.states, TO.controls, TO.dynamics_jacobians):
        assert np.array_equal(f(single), f(vec))
    for a, b in zip(TO.gains(single), TO.gains(vec)):
        assert np.array_equal(a, b)
    for p in (single, vec):
        TO.ilqr_step(p, 3); TO.al_update(p); TO.ilqr_step(p, 2)
    assert np.array_equal(TO.states(single), TO.states(vec)) and np.array_equal(TO.controls(single), TO.controls(vec))


# ---- F: program validation in the C ABI ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", range(len(malformed_specs())))
def test_to_create_rejects_malformed_programs(case):
    name, spec, code, msg = malformed_specs()[case]
    lib = K.load_library()
    h = C.c_void_p()
    rc = lib.to_create(C.byref(spec.c), C.byref(h))
    err = lib.to_last_error(None).decode()
    assert rc == code and not h, f"{name}: rc {rc} ({err})"
    assert msg in err, f"{name}: {err}"
