"""Costs of user dynamics models on the padded size classes (4, 2), (8, 4) and (16, 8), shared by the CPU and GPU tests of those costs:
one model per class, dense QuadraticCosts with a cross term, a user cost (AutodiffCost) with its NumPy twin, and the two problems the
classes were built for -- a planar quadrotor with a DARE terminal cost and a 7-joint arm reaching with its end effector."""
import numpy as np
import scipy.linalg

import trajopt_b200 as TO
from dynamics_programs import pad
from recorded_classes import arm7_model, planar_quadrotor_model

K = TO.capi
HOVER = 4.905                 # each thrust of the planar quadrotor at hover (mass 1, g = 9.81)


def small_model():
    """(3, 1): a damped pendulum on a cart-like chain, class (4, 2)"""
    return TO.AutodiffDynamics(3, 1, lambda x, u: [x[1], x[2], u[0] - 0.5 * TO.sin(x[0]) - 0.2 * x[2]])


CLASS_MODELS = {(4, 2): small_model, (8, 4): planar_quadrotor_model, (16, 8): arm7_model}


def dense_blocks(n, m, seed):
    """Q, R, H with [Q H'; H R] positive definite and every entry nonzero, and q, r, c"""
    r = np.random.default_rng(seed)
    G = r.uniform(-1.0, 1.0, (n + m, n + m))
    W = G @ G.T / (n + m) + np.eye(n + m)
    return W[:n, :n].copy(), W[n:, n:].copy(), W[n:, :n].copy(), r.uniform(-1.0, 1.0, n), r.uniform(-1.0, 1.0, m), float(r.uniform(0.5, 1.0))


def dense_cost(n, m, seed, terminal=False):
    Q, R, H, q, r, c = dense_blocks(n, m, seed)
    return TO.QuadraticCost(Q, R, H=H, q=q, r=r, c=c, terminal=terminal)


# ---- a user cost and its NumPy twin: weighted squares, a cross term and transcendental terms of every state and control -----------------
def user_cost_function(n, m, w=1.0, terminal=False):
    """``(fun, numpy_fun)``: ``fun`` records a cost of (n, m); ``numpy_fun`` evaluates the same arithmetic on arrays"""
    def make(sin, cos):
        def f(x, u):
            J = 0.5 * w * (x[0] * x[0]) + 0.3 * cos(x[n - 1]) + 0.1 * (x[0] * x[n - 1])
            for i in range(1, n):
                J = J + (0.2 + 0.05 * i) * (x[i] * x[i])
                if i < 4:
                    J = J + 0.05 * sin(x[i] - x[i - 1])
            if not terminal:
                for j in range(m):
                    J = J + (0.1 + 0.02 * j) * (u[j] * u[j])
                    if j < 2:
                        J = J + 0.05 * (u[j] * x[j % n])
            return J
        return f
    return make(TO.sin, TO.cos), make(np.sin, np.cos)


def user_cost(n, m, terminal=False):
    fun, npf = user_cost_function(n, m, terminal=terminal)
    return TO.AutodiffCost(n, m, fun, terminal=terminal), npf


def diagonal_as_user_cost(Qd, Rd, xf, terminal=False):
    """``LQRCost(Qd, Rd, xf)`` (uf = 0) restated as a recorded program: 1/2 sum Qd (x - xf)^2 + 1/2 sum Rd u^2"""
    Qd, Rd, xf = (np.asarray(a, dtype=float) for a in (Qd, Rd, xf))

    def f(x, u):
        J = None
        for i in range(len(Qd)):
            d = x[i] - xf[i]
            t = (0.5 * Qd[i]) * (d * d)
            J = t if J is None else J + t
        if not terminal:
            for j in range(len(Rd)):
                J = J + (0.5 * Rd[j]) * (u[j] * u[j])
        return J
    return TO.AutodiffCost(len(Qd), len(Rd), f, terminal=terminal)


# ---- the planar quadrotor with a DARE terminal cost ------------------------------------------------------------------------------------
PLANAR_XF = np.array([1.0, 0.5, 0.0, 0.0, 0.0, 0.0])


def planar_hover_linearisation(h):
    """[A B] of one explicit-Euler step of the planar quadrotor at hover (x = 0, u = (4.905, 4.905)): the DARE's model"""
    A = np.eye(6); A[0, 3] = A[1, 4] = A[2, 5] = h
    A[3, 2] = -h * 2.0 * HOVER                       # d(-T sin(theta)) / d theta at T = mg
    B = np.zeros((6, 2)); B[4, :] = h; B[5, 0], B[5, 1] = h * 20.0, -h * 20.0     # arm / J = 0.2 / 0.01
    return A, B


def planar_dare_objective(N, h):
    """a stage QuadraticCost tracking (PLANAR_XF, hover) with a cross term, and the DARE cost-to-go of the hover LQR as a dense terminal
    QuadraticCost"""
    Q = np.diag([1.0, 1.0, 0.5, 0.1, 0.1, 0.1]); Q[0, 2] = Q[2, 0] = 0.1
    R = np.array([[0.02, 0.005], [0.005, 0.02]])
    H = np.array([[0.0, 0.01, 0.005, 0.0, 0.002, 0.0], [0.0, 0.01, -0.005, 0.0, 0.002, 0.0]])
    A, B = planar_hover_linearisation(h)
    P = scipy.linalg.solve_discrete_are(A, B, Q, R)
    P = 0.5 * (P + P.T)
    uh, xf = np.full(2, HOVER), PLANAR_XF
    stage = TO.QuadraticCost(Q, R, H=H, q=-Q @ xf - H.T @ uh, r=-R @ uh - H @ xf, c=0.5 * xf @ Q @ xf + 0.5 * uh @ R @ uh + uh @ H @ xf)
    term = TO.QuadraticCost(P, R, q=-P @ xf, c=0.5 * xf @ P @ xf, terminal=True)
    return TO.Objective([stage] * (N - 1) + [term]), P


def planar_dare_problem(cls, B=8, N=41, seed=0, constrained=True):
    h = 2.0 / (N - 1)
    obj, _ = planar_dare_objective(N, h)
    cons = TO.ConstraintList(6, 2, N)
    if constrained:
        TO.add_constraint(cons, TO.BoundConstraint(6, 2, u_min=0.0, u_max=12.0), (1, N - 1))
    r = np.random.default_rng(seed)
    p = cls(planar_quadrotor_model(), obj, 0.1 * r.standard_normal((B, 6)), 2.0, xf=PLANAR_XF, constraints=cons)
    TO.initial_controls(p, pad(np.full((B, N - 1, 2), HOVER) + 0.3 * r.standard_normal((B, N - 1, 2)), 4))
    return p


# ---- the 7-joint arm reaching with its end effector ------------------------------------------------------------------------------------
LINKS = (0.3, 0.28, 0.26, 0.24, 0.22, 0.2, 0.18)
TARGET = np.array([0.9, 1.1])
JOINT_LIMIT = 1.2


def end_effector_function(w=10.0, wv=0.05, wu=0.01, terminal=False):
    """``(fun, numpy_fun)`` of w/2 |p(q) - target|^2 + wv/2 |qdot|^2 (+ wu/2 |u|^2), with p(q) the planar forward kinematics of the arm
    (joint i turns link i by q_0 + ... + q_i)"""
    def make(sin, cos):
        def f(x, u):
            th = x[0]
            px, py = LINKS[0] * cos(th), LINKS[0] * sin(th)
            for i in range(1, 7):
                th = th + x[i]
                px, py = px + LINKS[i] * cos(th), py + LINKS[i] * sin(th)
            dx, dy = px - TARGET[0], py - TARGET[1]
            J = (0.5 * w) * (dx * dx + dy * dy)
            v = x[7] * x[7]
            for i in range(8, 14):
                v = v + x[i] * x[i]
            J = J + (0.5 * wv) * v
            if not terminal:
                e = u[0] * u[0]
                for j in range(1, 7):
                    e = e + u[j] * u[j]
                J = J + (0.5 * wu) * e
            return J
        return f
    return make(TO.sin, TO.cos), make(np.sin, np.cos)


def arm_reach_problem(cls, B=8, N=41, seed=1):
    stage = TO.AutodiffCost(14, 7, end_effector_function()[0])
    term = TO.AutodiffCost(14, 7, end_effector_function(w=100.0, wv=1.0, terminal=True)[0], terminal=True)
    obj = TO.Objective([stage] * (N - 1) + [term])
    cons = TO.ConstraintList(14, 7, N)
    lim = np.concatenate([np.full(7, JOINT_LIMIT), np.full(7, np.inf)])
    TO.add_constraint(cons, TO.BoundConstraint(14, 7, x_min=-lim, x_max=lim, u_min=-4.0, u_max=4.0), (1, N - 1))
    r = np.random.default_rng(seed)
    p = cls(arm7_model(), obj, 0.1 * r.standard_normal((B, 14)), 2.0, constraints=cons)
    TO.initial_controls(p, pad(0.3 * r.standard_normal((B, N - 1, 7)), 8))
    return p
