"""GPU tests of to_solve (include/trajopt_b200.h; DESIGN.md 5d): whole solves against the per-instance restatement on the oracle
(tests/solve_reference.py) on every solver path, independence of a solve from the composition of its batch (retired and waiting instances
are untouched, the outer loop is synchronised correctly), and the entry points after a solve working on every instance again."""
import numpy as np
import pytest
import torch

import trajopt_b200 as TO
from oracle_binding import OracleProblem, match_algebra
from parity_util import GAIN_TOL, check, decisions_agree, triple_with_options
from solve_reference import reference_solve
import dynamics_programs as DP

pytestmark = pytest.mark.gpu
P = TO.problems
K = TO.capi


def _setups(g):
    v = TO.backward_algebra(g)
    return (lambda p: p.set_backward_variant(v)), (lambda p: p.set_backward_variant(v).set_gain_noise(GAIN_TOL))


def subset(prob, idx, cls=None):
    """the instances `idx` of `prob` as a batch of their own: x0, controls, multipliers, penalties, solver options"""
    t = TO.gettimes(prob)
    q = (cls or type(prob))(prob.model, prob.obj.copy(), prob.x0[idx].copy(), float(t[-1]), xf=prob.xf.copy(), constraints=prob.constraints.copy(),
                            t0=float(t[0]), dt=prob.spec.dt.copy(), error_state=prob.error_state)
    if getattr(prob, "_options", None) is not None:
        TO.set_options(q, **{f: getattr(prob._options, f) for f, _ in K.to_options._fields_})
    TO.initial_controls(q, TO.controls(prob)[idx])
    for i, c in enumerate(prob.constraints.constraints):
        TO.set_multipliers(q, q.constraints.constraints[i], TO.multipliers(prob, c)[idx])
    return q


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def compare(what, build, sample=None, opts=None, allow=0.05, outliers=0.05, **solve_opts):
    """GPU solve of the whole batch vs the oracle restatement (and its gain-noise twin) on the instances `sample`"""
    g, o, t = triple_with_options(build, opts)
    so, st_ = _setups(g)
    idx = np.arange(g.B) if sample is None else np.asarray(sample)
    if sample is not None:
        o, t = subset(o, idx), subset(t, idx)
    sg = TO.solve(g, **solve_opts)
    ro = reference_solve(o, setup=so, **solve_opts)
    rt = reference_solve(t, setup=st_, **solve_opts)
    Xg, Ug = TO.states(g)[idx], TO.controls(g)[idx]
    decisions_agree(f"{what} status", sg.status[idx], ro.status, rt.status, allow=allow)
    decisions_agree(f"{what} iterations", sg.iterations[idx], ro.iterations, rt.iterations, allow=2 * allow)
    decisions_agree(f"{what} outer iterations", sg.iterations_outer[idx], ro.iterations_outer, rt.iterations_outer, allow=allow)
    same = (sg.iterations[idx] == ro.iterations) & (ro.iterations == rt.iterations)
    check(f"{what} X", Xg, ro.X, rt.X, 1e-8, sel=same, outliers=outliers)
    check(f"{what} U", Ug, ro.U, rt.U, 1e-8, sel=same, outliers=outliers)
    check(f"{what} cost", sg.cost[idx][:, None], ro.cost[:, None], rt.cost[:, None], 1e-9, sel=same, outliers=outliers)
    check(f"{what} c_max", sg.c_max[idx][:, None], ro.c_max[:, None], rt.c_max[:, None], 1e-9, sel=same, outliers=outliers)
    check(f"{what} dJ", sg.dJ[idx][:, None], ro.dJ[:, None], rt.dJ[:, None], 1e-9, sel=same, outliers=outliers)
    check(f"{what} gradient", sg.gradient[idx][:, None], ro.gradient[:, None], rt.gradient[:, None], 1e-9, sel=same, outliers=outliers)
    for i, c in enumerate(g.constraints.constraints):
        check(f"{what} multipliers of constraint {i}", TO.multipliers(g, c)[idx], ro.lam[i], rt.lam[i], 1e-8, sel=same, outliers=outliers)
    assert g._lib.to_synchronize(g._h) == 0
    return sg, ro


def test_solve_cartpole_constrained_warp_riccati():
    sg, ro = compare("cartpole AL", lambda cls: P.cartpole(B=16, N=51, cls=cls, u_bound=3.0, goal=True), opts={"backward_kernel": 1})
    assert np.any(sg.status == K.SOLVE_SUCCEEDED) and np.any(sg.iterations_outer > 1)


def test_solve_cartpole_unconstrained():
    sg, ro = compare("cartpole", lambda cls: P.cartpole(B=16, N=51, cls=cls))
    assert np.all(sg.iterations_outer == 1) and np.all(sg.c_max == 0)


def test_solve_acrobot_beyond_one_wave_thread_kernel():
    B = 16 * sm_count() + 5
    sample = np.linspace(0, B - 1, 12).astype(int)
    compare("acrobot", lambda cls: P.acrobot(B=B, N=51, cls=cls, dense_cost=False), sample=sample, opts={"backward_kernel": 2}, iterations=60)


def test_solve_quadrotor_error_state_record_path():
    # (the closed loop of the Quadrotor amplifies rounding by orders of magnitude per iteration, parity_util: over 60-80 iterations one in
    # four decidable instances may take another discrete decision, or land outside the one noise draw of the twin)
    compare("quadrotor error state", lambda cls: P.quadrotor(B=8, N=51, cls=cls, error_state=True), allow=0.25, outliers=0.25, iterations=80)


def test_solve_quadrotor_full_state():
    compare("quadrotor full state", lambda cls: P.quadrotor(B=4, N=31, cls=cls, dt=0.05), allow=0.25, outliers=0.25, iterations=60)


def test_solve_quatvec_materialised_expansion():
    compare("quadrotor QuatVecEq", lambda cls: P.quadrotor_lie(B=4, N=31, cls=cls), allow=0.25, outliers=0.25, iterations=60)


def test_solve_user_dynamics_model():
    """recorded user dynamics (AutodiffDynamics, the padded (4, 2) kernel instance)"""
    compare("user model", lambda cls: DP.builtin_problem("cartpole", cls, 8, recorded=True), iterations=60)


@pytest.mark.parametrize("which", ["cartpole", "quadrotor_error_state"])
def test_solve_is_independent_of_the_batch_composition(which):
    """a solve of a batch and a solve of some of its instances alone give bit-identical per-instance results: instances that stopped early
    (retired, or waiting for the outer update) are untouched by the iterations that follow, and each outer iteration sees the same penalties"""
    def build():
        if which == "cartpole":      # (the backward kernel is chosen explicitly: the automatic choice depends on the batch size)
            p = P.cartpole(B=48, N=51, u_bound=3.0, goal=True)
            TO.set_options(p, backward_kernel=1)
            return p
        return P.quadrotor(B=48, N=51, error_state=True)
    g = build()
    st = TO.solve(g)
    assert len(np.unique(st.iterations)) > 1 and len(np.unique(st.iterations_outer)) > 1     # the instances stop at different iterations
    idx = np.array([1, 7, 30, 47])
    q = subset(build(), idx)
    sq = TO.solve(q)
    for f in TO.SolveStats.FIELDS:
        assert np.array_equal(getattr(st, f)[idx], getattr(sq, f)), f
    assert np.array_equal(TO.states(g)[idx], TO.states(q))
    assert np.array_equal(TO.controls(g)[idx], TO.controls(q))
    for cg, cq in zip(g.constraints.constraints, q.constraints.constraints):
        assert np.array_equal(TO.multipliers(g, cg)[idx], TO.multipliers(q, cq))
    Kg, dg = TO.gains(g); Kq, dq = TO.gains(q)
    assert np.array_equal(Kg[idx], Kq) and np.array_equal(dg[idx], dq)


def test_mixed_status_batch_against_the_restatement():
    """ONE batch whose instances end in different statuses (success and at least two of: iteration cap, outer cap, regularisation failure):
    the restatement on a sample that holds one instance of each status, and the statuses of the sample solved within the whole batch"""
    build = lambda cls: P.cartpole(B=48, N=51, cls=cls, u_bound=3.0, goal=True)
    g = build(TO.Problem)
    TO.set_options(g, backward_kernel=1)
    st = TO.solve(g)
    kinds = set(st.status.tolist())
    assert len(kinds) >= 3 and K.SOLVE_SUCCEEDED in kinds, st
    sample = [int(np.nonzero(st.status == k)[0][0]) for k in sorted(kinds)]
    sg, ro = compare("mixed", build, sample=sample, opts={"backward_kernel": 1})
    assert np.array_equal(sg.status, st.status)
    assert set(ro.status.tolist()) == kinds


def test_an_iteration_without_active_instances_changes_nothing():
    """every instance stops at the same iteration (the cap), so the iteration queued behind the last real one has no ACTIVE instance: the
    problem after the solve -- trajectory, gains, regularisation, line-search state -- equals, bit for bit, the same problem after exactly that
    many to_ilqr_step iterations"""
    cap = 7
    g = P.cartpole(B=8, N=51)
    st = TO.solve(g, iterations=cap, cost_tolerance=1e-30)
    assert np.all(st.iterations == cap) and np.all(st.status == K.SOLVE_MAX_ITERATIONS)
    h = P.cartpole(B=8, N=51)
    TO.rollout(h)
    TO.ilqr_step(h, cap)
    assert np.array_equal(TO.states(g), TO.states(h)) and np.array_equal(TO.controls(g), TO.controls(h))
    Kg, dg = TO.gains(g); Kh, dh = TO.gains(h)
    assert np.array_equal(Kg, Kh) and np.array_equal(dg, dh)
    sg, sh = TO.solver_state(g), TO.solver_state(h)
    for k in sg:
        assert np.array_equal(sg[k], sh[k]), k
    assert np.array_equal(st.cost, TO.cost(h))


def test_every_status_and_caps_on_the_gpu():
    """each cap and the regularisation failure on its own: iteration cap, outer cap, backward pass failing at bp_reg_max"""
    g = P.cartpole(B=8, N=41, u_bound=3.0, goal=True)
    st = TO.solve(g, iterations=6)
    assert np.all(st.status == K.SOLVE_MAX_ITERATIONS) and np.all(st.iterations == 6)
    g = P.cartpole(B=8, N=41, u_bound=3.0, goal=True)
    st = TO.solve(g, iterations_outer=1, constraint_tolerance=1e-12)
    assert np.all(st.status == K.SOLVE_MAX_ITERATIONS_OUTER) and np.all(st.iterations_outer == 1)
    from test_oracle_solve import restart_problem
    r = restart_problem(TO.Problem)
    st = TO.solve(r)
    assert np.all(st.status == K.SOLVE_MAX_REGULARIZATION)
    assert r._lib.to_synchronize(r._h) == 0


def test_entry_points_work_on_every_instance_after_a_solve():
    """after to_solve, to_ilqr_step and to_al_update iterate every instance again (the oracle from the same state agrees), and the
    backward pass's queue never reported an error"""
    g = P.cartpole(B=32, N=51, u_bound=3.0, goal=True)
    TO.solve(g, iterations=40)
    o = match_algebra(g, subset(g, np.arange(g.B), cls=OracleProblem))
    for c_g, c_o in zip(g.constraints.constraints, o.constraints.constraints):
        TO.set_penalty(o, c_o, TO.penalty(g, c_g))
    for p in (g, o):          # the AL update also restarts rho, which the solve left per instance
        TO.rollout(p)
        TO.al_update(p)
    assert np.allclose(TO.multipliers(g, g.constraints.constraints[0]), TO.multipliers(o, o.constraints.constraints[0]), rtol=1e-9, atol=1e-12)
    for p in (g, o):
        TO.ilqr_step(p, 1)
    rel = np.abs(TO.merit(g) - TO.merit(o)) / np.maximum(1.0, np.abs(TO.merit(o)))
    assert rel.max() < 1e-6
    assert g._lib.to_synchronize(g._h) == 0


def test_solve_rejects_bad_options():
    g = P.cartpole(B=2, N=21)
    for kw in ({"cost_tolerance": 0.0}, {"gradient_tolerance": -1.0}, {"constraint_tolerance": 0.0}, {"iterations": 0}, {"iterations_outer": 0}):
        with pytest.raises(TO.ArgumentError, match="to_solve"):
            TO.solve(g, **kw)
    with pytest.raises(TO.ArgumentError, match="unknown solve option"):
        TO.solve(g, cost_tol=1.0)
