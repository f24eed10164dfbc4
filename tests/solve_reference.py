"""Test-side restatement of ``to_solve`` (Altro's AL-iLQR ``solve!``, include/trajopt_b200.h, DESIGN.md 5d) for ONE instance at a time,
sequentially, written as Altro writes it: each instance runs in a B = 1 copy of the problem with its own penalties, on the CPU oracle's
iteration primitives (``ilqr_step``, ``merit``, ``al_update``).  The GPU's batch-synchronous outer loop with retired instances is checked
against this independent orchestration.

``reference_solve(prob, setup, **options)`` returns a ``SolveStats`` with, in addition, the final ``X``, ``U`` and multipliers ``lam`` (one
array per constraint) of every instance.  ``setup(p)`` configures each B = 1 copy the way the batch problem was configured (oracle arithmetic
form, gain noise, integrator); solver options are copied from ``prob``.
"""
import numpy as np

import trajopt_b200 as TO

K = TO.capi


def todorov_gradient(d, U):
    """Altro gradient_todorov: mean_k max_i |d_k,i| / (|u_k,i| + 1)"""
    return float(np.mean(np.max(np.abs(d) / (np.abs(U) + 1.0), axis=1)))


def instance_copy(prob, b, setup=None):
    """a B = 1 problem holding instance b of `prob`: x0, controls, multipliers, penalties and solver options"""
    t = TO.gettimes(prob)
    p = type(prob)(prob.model, prob.obj.copy(), prob.x0[b:b + 1].copy(), float(t[-1]), xf=prob.xf.copy(), constraints=prob.constraints.copy(),
                   t0=float(t[0]), dt=prob.spec.dt.copy(), error_state=prob.error_state)
    if setup is not None:
        setup(p)
    if getattr(prob, "_options", None) is not None:
        TO.set_options(p, **{f: getattr(prob._options, f) for f, _ in K.to_options._fields_})
    TO.initial_controls(p, TO.controls(prob)[b:b + 1])
    for i, con in enumerate(prob.constraints.constraints):
        TO.set_multipliers(p, p.constraints.constraints[i], TO.multipliers(prob, con)[b:b + 1])
        TO.set_penalty(p, p.constraints.constraints[i], TO.penalty(prob, con))
    return p


def solve_one(p, o):
    """the solve of a B = 1 problem `p` with to_solve_options `o`; returns (status, iterations, outer, dJ, gradient, c_max)"""
    ncon = len(p.constraints.constraints)
    TO.rollout(p)
    J_prev = TO.merit(p)[0]
    it, outer = 0, 1
    while True:
        final = ncon == 0 or outer >= o.iterations_outer                              # Altro set_tolerances!
        ctol = o.cost_tolerance if final else o.cost_tolerance_intermediate
        gtol = o.gradient_tolerance if final else o.gradient_tolerance_intermediate
        inner, dj_zero = 0, 0
        while True:                                                                   # the inner (iLQR) loop
            TO.ilqr_step(p, 1)
            it += 1; inner += 1
            st = TO.solver_state(p)
            if st["bp_status"][0] < 0:                                                 # the backward pass failed at bp_reg_max
                c_max = TO.max_violation(p)[0] if ncon else 0.0
                return K.SOLVE_MAX_REGULARIZATION, it, outer, 0.0, grad if it > 1 else 0.0, c_max
            J = TO.merit(p)[0]
            stepped = st["alpha"][0] > 0
            dJ = J_prev - J if stepped else 0.0
            dj_zero += not stepped
            J_prev = J
            grad = todorov_gradient(TO.gains(p)[1][0], TO.controls(p)[0])
            converged = stepped and 0.0 <= dJ < ctol and grad < gtol
            if converged or dj_zero > o.dJ_counter_limit or it >= o.iterations or (ncon and inner >= o.iterations_inner):
                break
        if ncon == 0:
            status = K.SOLVE_SUCCEEDED if converged else K.SOLVE_MAX_ITERATIONS if it >= o.iterations else K.SOLVE_UNSOLVED
            return status, it, outer, dJ, grad, 0.0
        c_max = TO.max_violation(p)[0]                                                # the outer (AL) loop
        if c_max < o.constraint_tolerance:
            return K.SOLVE_SUCCEEDED, it, outer, dJ, grad, c_max
        if it >= o.iterations:
            return K.SOLVE_MAX_ITERATIONS, it, outer, dJ, grad, c_max
        if outer >= o.iterations_outer:
            return K.SOLVE_MAX_ITERATIONS_OUTER, it, outer, dJ, grad, c_max
        TO.al_update(p)                                                               # dual update, penalty update, rho reset
        outer += 1
        J_prev = TO.merit(p)[0]


def reference_solve(prob, setup=None, **options):
    o = TO.solve_options(**options)
    B = prob.B
    st = TO.SolveStats(B)
    st.X, st.U = np.empty((B, prob.N, prob.n)), np.empty((B, prob.N - 1, prob.m))
    st.lam = [np.empty_like(TO.multipliers(prob, c)) for c in prob.constraints.constraints]
    for b in range(B):
        p = instance_copy(prob, b, setup)
        st.status[b], st.iterations[b], st.iterations_outer[b], st.dJ[b], st.gradient[b], st.c_max[b] = solve_one(p, o)
        st.cost[b] = TO.cost(p)[0]
        st.X[b], st.U[b] = TO.states(p)[0], TO.controls(p)[0]
        for i, c in enumerate(p.constraints.constraints):
            st.lam[i][b] = TO.multipliers(p, c)[0]
        p.close()
    return st
