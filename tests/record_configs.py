"""Error-state Quadrotor problems of the record path's compact class (DiagonalCost + Goal / Bound constraints) that reach the corners of
the record cost expansion (rollout.cu k_expansion_rec16b, riccati_frag.cu k_expansion_rec) -- test infrastructure shared by
tests/test_gpu_record_expansion.py (CUDA records against the oracle) and tests/test_costexp_emulator.py (the kernel's algorithm in NumPy).
Every builder takes the Problem class (CUDA or oracle) and returns the same problem for both."""
import numpy as np

import trajopt_b200 as TO

n, m = 13, 4
XF = np.array([0, 0, 2, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0.0])
X0 = np.array([1, 2, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0.0])
HOVER = TO.Quadrotor().hover_control()


def _x0(r, B, attitude):
    x0 = np.tile(X0, (B, 1))
    x0[:, :3] += r.uniform(-1, 1, (B, 3))
    if attitude:                                   # random initial attitudes: the attitude projection G is far from the identity
        q = np.array([1.0, 0, 0, 0]) + 0.3 * r.standard_normal((B, 4))
        x0[:, 3:7] = q / np.linalg.norm(q, axis=1, keepdims=True)
    return x0


def _problem(cls, obj, cons, B, N, seed, attitude=False, error_state=True, dt=0.05):
    r = np.random.default_rng(seed)
    p = cls(TO.Quadrotor(), obj, _x0(r, B, attitude), dt * (N - 1), xf=XF, constraints=cons, error_state=error_state)
    TO.initial_controls(p, HOVER + 0.05 * r.standard_normal((B, N - 1, m)))
    return p


def _lqr(N, Qd=None, Qfd=None):
    Qd = np.full(n, 0.1) if Qd is None else Qd
    Qfd = np.full(n, 100.0) if Qfd is None else Qfd
    return TO.Objective(TO.LQRCost(Qd, np.full(m, 0.01), XF, HOVER), TO.LQRCost(Qfd, np.full(m, 0.01), XF, HOVER, terminal=True), N)


def quat_weights(cls, B=5, N=41):
    """non-uniform quaternion weights + random attitudes: G' diag(h_q) G has off-diagonal entries"""
    Qd = np.full(n, 0.1); Qd[3:7] = (0.3, 0.05, 0.2, 0.1)
    Qfd = np.full(n, 100.0); Qfd[3:7] = (30.0, 5.0, 20.0, 10.0)
    cons = TO.ConstraintList(n, m, N)
    TO.add_constraint(cons, TO.BoundConstraint(n, m, u_min=np.zeros(m), u_max=np.full(m, 10.0)), (1, N - 1))
    TO.add_constraint(cons, TO.GoalConstraint(XF), N)
    return _problem(cls, _lqr(N, Qd, Qfd), cons, B, N, seed=3, attitude=True)


def state_bounds(cls, B=6, N=41, error_state=True):
    """two-sided bounds on position, q_w >= 0.9, q_x..q_z, velocity and angular rate on knots 2..N (terminal knot included: state rows beside
    the goal's), control bounds on 1..N-1, goal at N: inequality rows on every state lane, AL rows on the attitude lanes"""
    x_max, x_min = np.full(n, np.inf), np.full(n, -np.inf)
    x_max[:3], x_min[:3] = (1.8, 2.6, 2.2), (-0.6, -0.3, 0.6)
    x_min[3] = 0.9
    x_max[4:7], x_min[4:7] = 0.15, -0.15
    x_max[7:10], x_min[7:10] = 0.5, -0.5
    x_max[10:13], x_min[10:13] = 1.0, -1.0
    cons = TO.ConstraintList(n, m, N)
    TO.add_constraint(cons, TO.BoundConstraint(n, m, x_min=x_min, x_max=x_max), (2, N))
    TO.add_constraint(cons, TO.BoundConstraint(n, m, u_min=np.full(m, 0.5), u_max=np.full(m, 9.0)), (1, N - 1))
    TO.add_constraint(cons, TO.GoalConstraint(XF), N)
    return _problem(cls, _lqr(N), cons, B, N, seed=4, attitude=True, error_state=error_state)


MIDBLOCK = dict(A=(5, 37), B=(38, 100), G=50)


def midblock_ranges(cls, B=4, N=101):
    """constraint ranges that start and end inside 16-knot blocks: Bound A on 5..37, another Bound on 38..N-1, a goal on the attitude and
    angular rate at knot 50, the full goal at N (<= 3 rows per z entry: the term-table kernel)"""
    a_max, a_min = np.full(n, np.inf), np.full(n, -np.inf)
    a_max[:3], a_min[:3] = (1.8, 2.6, 2.2), (-0.6, -0.3, 0.6)
    a_max[7:10] = 0.15
    b_min = np.full(n, -np.inf); b_min[7:10] = -0.3
    cons = TO.ConstraintList(n, m, N)
    TO.add_constraint(cons, TO.BoundConstraint(n, m, x_min=a_min, x_max=a_max, u_min=np.zeros(m), u_max=np.full(m, 10.0)), MIDBLOCK["A"])
    TO.add_constraint(cons, TO.BoundConstraint(n, m, x_min=b_min, u_max=np.full(m, 9.0)), (MIDBLOCK["B"][0], N - 1))
    TO.add_constraint(cons, TO.GoalConstraint(XF, inds=[4, 5, 6, 7, 11, 12, 13]), MIDBLOCK["G"])
    TO.add_constraint(cons, TO.GoalConstraint(XF), N)
    return _problem(cls, _lqr(N), cons, B, N, seed=5)


def four_terms(cls, B=4, N=33, error_state=True):
    """two overlapping Bound constraints on the position and the controls + the goal: 5 rows on some z entries, more than the term table
    holds -> the descriptor-walking kernels (k_expansion_rec; full state: k_riccati<FASTAL = false>); non-uniform quaternion weights and
    random attitudes"""
    x1_max, x1_min = np.full(n, np.inf), np.full(n, -np.inf)
    x1_max[:3], x1_min[:3] = 2.5, -0.5
    x2_max, x2_min = np.full(n, np.inf), np.full(n, -np.inf)
    x2_max[:3], x2_min[:3] = (1.6, 2.4, 2.1), (-0.3, -0.2, 0.7)
    cons = TO.ConstraintList(n, m, N)
    TO.add_constraint(cons, TO.BoundConstraint(n, m, x_min=x1_min, x_max=x1_max, u_min=np.zeros(m), u_max=np.full(m, 10.0)), (1, N - 1))
    TO.add_constraint(cons, TO.BoundConstraint(n, m, x_min=x2_min, x_max=x2_max, u_min=np.full(m, 0.5), u_max=np.full(m, 9.0)), (3, N - 1))
    TO.add_constraint(cons, TO.GoalConstraint(XF), N)
    Qd = np.full(n, 0.1); Qd[3:7] = (0.3, 0.05, 0.2, 0.1)           # (attitude off-diagonals in the fallback kernel too)
    return _problem(cls, _lqr(N, Qd), cons, B, N, seed=6, attitude=True, error_state=error_state)


def bounded(cls, B=6, N=40):
    """Bound rows on states AND controls (three AL terms on some entries at the last stage knots) + goal"""
    obj = TO.LQRObjective(np.full(n, 0.1), np.full(m, 0.01), np.full(n, 100.0), XF, N)
    cons = TO.ConstraintList(n, m, N)
    x_max = np.full(n, np.inf); x_min = np.full(n, -np.inf)
    x_max[:3] = 2.5; x_min[:3] = -0.5; x_max[7:10] = 1.0; x_min[7:10] = -1.0; x_max[12] = 0.3
    TO.add_constraint(cons, TO.BoundConstraint(n, m, x_min=x_min, x_max=x_max, u_min=np.zeros(4), u_max=np.full(4, 10.0)), (1, N - 1))
    TO.add_constraint(cons, TO.GoalConstraint(XF), N)
    r = np.random.default_rng(5)
    x0 = np.tile(X0, (B, 1)); x0[:, :3] += r.uniform(-1, 1, (B, 3))
    prob = cls(TO.Quadrotor(), obj, x0, 0.05 * (N - 1), xf=XF, constraints=cons, error_state=True)
    TO.initial_controls(prob, HOVER[None, None, :] + 0.01 * r.standard_normal((B, N - 1, m)))
    return prob


def long_horizon(cls, N, B=2, error_state=True):
    """the BASELINE constraints over N knots of a 4 s horizon: N = 4094 is the last horizon the 12-bit knot field of the term table takes"""
    return TO.problems.quadrotor(B=B, N=N, dt=4.0 / (N - 1), cls=cls, error_state=error_state)


def tracking(cls, B=4, N=51):
    """TrackingObjective (one cost per knot) with control bounds, for update_trajectory / shift_trajectory on the error state; -> (problem,
    Xref, Uref)"""
    nref = 80
    t = np.linspace(0, 4, nref)
    Xref = np.zeros((nref, n)); Xref[:, 0] = np.sin(t); Xref[:, 1] = 0.5 * t; Xref[:, 2] = 1.0; Xref[:, 3] = 1.0
    Uref = np.tile(HOVER, (nref, 1))
    r = np.random.default_rng(11)
    x0 = np.tile(Xref[0], (B, 1)); x0[:, :3] += 0.05 * r.standard_normal((B, 3)); x0[:, 7:] += 0.05 * r.standard_normal((B, 6))
    cons = TO.ConstraintList(n, m, N)
    TO.add_constraint(cons, TO.ControlBound(m, u_min=0.0, u_max=8.0), (1, N - 1))
    obj = TO.TrackingObjective(np.full(n, 1.0), np.full(m, 0.1), Xref[:N], Uref[:N - 1], Qf=np.full(n, 10.0))
    p = cls(TO.Quadrotor(), obj, x0, 2.5, constraints=cons, error_state=True)
    TO.initial_controls(p, HOVER)
    return p, Xref, Uref


def max_terms_per_z(prob):
    """Goal / Bound rows acting on one z entry, counted as capi.cu to_create does (P.max_terms_per_z): > 3 leaves the term table"""
    cnt = np.zeros(n + m, dtype=int)
    for c in prob.constraints:
        if isinstance(c, TO.GoalConstraint):
            cnt[np.asarray(c.inds) - 1] += 1
        else:
            cnt += np.isfinite(c.z_max).astype(int) + np.isfinite(c.z_min).astype(int)
    return int(cnt.max())


def term_inputs(prob):
    """what the host-built term table and the cost table of `prob` are made of: (constraints with 1-based knot ranges, per-knot cost index,
    per cost (Qd, q, Rd, r)) -- the inputs of costexp_emulator"""
    cons = [(c, f, l) for (f, l), c in zip(prob.constraints.inds, prob.constraints.constraints)]
    uniq, index = prob.obj._tables()
    costs = [(np.diag(c.Q).copy(), np.asarray(c.q, dtype=float), np.diag(c.R).copy(), np.asarray(c.r, dtype=float)) for c in uniq]
    return cons, index, costs
