"""Exact reference (fractions.Fraction) of the branch points of the cost + AL expansion, restated from the reference's formulas:

  * projection and its Jacobian on the NegativeOrthant and the SecondOrderCone, and the SOC's second derivative
    (src/cones.jl:96-127, :129-188, :201-276), with the reference's tie conventions:
      NegativeOrthant  J_ii = 1 when x_i <= 0                          (cones.jl:140-142)
      SecondOrderCone  below when a <= -s, in when a <= s, outside when a >= |s|, tested in that order   (cones.jl:84-90, :151-161)
                       ∇²: zero below and in, the formula only when a > |s|                             (cones.jl:223-228)
  * the Gauss-Newton AL terms of one constraint at one knot: lbar = lambda - mu c, g -= (D c_z)' Pi(lbar), H += mu (D c_z)'(D c_z),
    D = ∇Pi(lbar) on the dual cone; the AL penalty (|Pi(lbar)|^2 - |lambda|^2) / (2 mu) and the violation |c - Pi_K(c)|_inf;
  * the DiagonalCost gradient and Hessian (src/cost_functions.jl:137-233; the terminal knot has no control terms);
  * the error-state expansion of a unit quaternion at z[qs:qs+4]: g_e = G'g, H_e = G'HG - (q'g_q) I3 on the attitude block.

Every quantity is a Fraction, so on inputs whose square roots are rational (Pythagorean triples) the result is exact and a kernel can be
compared with it entry by entry.  Matrices are lists of rows."""
from fractions import Fraction
from math import isqrt

import numpy as np

IDENTITY, ZERO, NEGATIVE, SOC = "identity", "zero", "negative_orthant", "second_order"


def fr(v):
    """a float (or int, or Fraction) as the exact Fraction it stands for"""
    return v if isinstance(v, Fraction) else Fraction(float(v))


def frs(a):
    return [fr(v) for v in np.ravel(np.asarray(a, dtype=object))]


def zeros(r, c):
    return [[Fraction(0)] * c for _ in range(r)]


def exact_sqrt(q):
    q = fr(q)
    if q < 0:
        raise ValueError("negative")
    a, b = isqrt(q.numerator), isqrt(q.denominator)
    if a * a != q.numerator or b * b != q.denominator:
        raise ValueError(f"{q} is not the square of a rational: choose Pythagorean inputs")
    return Fraction(a, b)


def dualcone(cone):   # cones.jl:65-69
    return {IDENTITY: ZERO, ZERO: IDENTITY}.get(cone, cone)


def soc_case(x):
    """'below', 'in' or 'outside' (cones.jl:84-88), the first test that holds"""
    x = frs(x)
    s, a = x[-1], exact_sqrt(sum(v * v for v in x[:-1]))
    if a <= -s:
        return "below"
    if a <= s:
        return "in"
    assert a >= abs(s)
    return "outside"


def projection(cone, x):   # cones.jl:72-127
    x = frs(x)
    if cone == IDENTITY:
        return x
    if cone == ZERO:
        return [Fraction(0)] * len(x)
    if cone == NEGATIVE:
        return [min(Fraction(0), v) for v in x]
    if cone == SOC:
        case, s = soc_case(x), x[-1]
        if case == "below":
            return [Fraction(0)] * len(x)
        if case == "in":
            return x
        a = exact_sqrt(sum(v * v for v in x[:-1]))
        c = (1 + s / a) / 2
        return [c * v for v in x[:-1]] + [c * a]
    raise ValueError(cone)


def grad_projection(cone, x):   # cones.jl:129-188
    x = frs(x)
    p = len(x)
    J = zeros(p, p)
    if cone == IDENTITY:
        for i in range(p):
            J[i][i] = Fraction(1)
    elif cone == NEGATIVE:
        for i in range(p):
            J[i][i] = Fraction(1 if x[i] <= 0 else 0)     # cones.jl:141: the tie x_i == 0 is active
    elif cone == SOC:
        case, s = soc_case(x), x[-1]
        if case == "in":
            for i in range(p):
                J[i][i] = Fraction(1)
        elif case == "outside":
            v, a = x[:-1], exact_sqrt(sum(t * t for t in x[:-1]))
            c = (1 + s / a) / 2
            for i in range(p - 1):
                for j in range(p - 1):
                    J[i][j] = -s / (2 * a ** 3) * v[i] * v[j] + (c if i == j else 0)
                J[i][p - 1] = v[i] / (2 * a)
                J[p - 1][i] = (-s / (2 * a * a) + c / a) * v[i]
            J[p - 1][p - 1] = Fraction(1, 2)
    elif cone != ZERO:
        raise ValueError(cone)
    return J


def hess_projection(cone, x, b):
    """the second derivative of x -> Pi(x)'b (cones.jl:190-276), from the matrix expressions the reference states in its comment
    (cones.jl:228-239) with P = I - v v' / a^2:
        dvdv = -s/a^3 P bv v' + s/a (2 (v'bv) v v' / a^4 - ((v'bv) I + v bv') / a^2) + bs/a P,   dvds = P bv / a,
        H = [dvdv, dvds; dvds', 0] / 2,
    of which the reference's evaluation (cones.jl:241-270) keeps the lower triangle of dvdv and mirrors it.  Zero below and in the cone
    (cones.jl:223-226)."""
    x, b = frs(x), frs(b)
    p = len(x)
    H = zeros(p, p)
    if cone != SOC:
        return H
    n, s, bs = p - 1, x[-1], b[-1]
    v, bv = x[:-1], b[:-1]
    a = exact_sqrt(sum(t * t for t in v))
    if a <= -s or a <= s:
        return H
    assert a > abs(s)
    I = [[Fraction(int(i == j)) for j in range(n)] for i in range(n)]
    P = [[I[i][j] - v[i] * v[j] / a ** 2 for j in range(n)] for i in range(n)]
    Pb = [sum(P[i][j] * bv[j] for j in range(n)) for i in range(n)]
    vb = sum(v[i] * bv[i] for i in range(n))
    dvdv = [[-s / a ** 3 * Pb[i] * v[j] + s / a * (2 * vb * v[i] * v[j] / a ** 4 - (vb * I[i][j] + v[i] * bv[j]) / a ** 2) + bs / a * P[i][j]
             for j in range(n)] for i in range(n)]
    for i in range(n):
        H[i][n] = H[n][i] = Pb[i] / a / 2
        for j in range(i + 1):
            H[i][j] = H[j][i] = dvdv[i][j] / 2
    return H


# ---- one knot ------------------------------------------------------------------------------------------------------------------------
class Row:
    """one constraint at one knot: its value c (p), Jacobian C (p x nz, lists of rows), multipliers and penalty, and its cone"""

    def __init__(self, cone, c, C, lam, mu):
        self.cone, self.c, self.C, self.lam, self.mu = cone, frs(c), [frs(r) for r in C], frs(lam), fr(mu)


def goal_row(xf, x, nz, lam, mu, inds=None):
    """GoalConstraint (src/constraints.jl:55-68): c = x[inds] - xf[inds], equality"""
    x, xf = frs(x), frs(xf)
    inds = list(range(len(x))) if inds is None else list(inds)
    C = zeros(len(inds), nz)
    for r, j in enumerate(inds):
        C[r][j] = Fraction(1)
    return Row(ZERO, [x[j] - xf[j] for j in inds], C, lam, mu)


def quatvec_row(qf, x, nz, lam, mu, qs=3):
    """QuatVecEq (src/constraints.jl:938-965): c = qhat[2:4] - sign(qf'qhat) qf[2:4] with qhat = q / |q|, equality; its Jacobian
    (I - qhat qhat') / |q| (rows 2:4)"""
    x, qf = frs(x), frs(qf)
    q = x[qs:qs + 4]
    nq = exact_sqrt(sum(t * t for t in q))
    qh = [t / nq for t in q]
    sg = -1 if sum(f * t for f, t in zip(qf, qh)) < 0 else 1
    C = zeros(3, nz)
    for i in range(3):
        for j in range(4):
            C[i][qs + j] = (Fraction(int(i + 1 == j)) - qh[i + 1] * qh[j]) / nq
    return Row(ZERO, [qh[i + 1] - sg * qf[i + 1] for i in range(3)], C, lam, mu)


def bound_row(z_max, z_min, z, lam, mu):
    """BoundConstraint (src/constraints.jl:738-765): the finite upper rows z_j - z_max_j, then the finite lower rows z_min_j - z_j"""
    z = frs(z)
    up = [j for j in range(len(z)) if np.isfinite(z_max[j])]
    lo = [j for j in range(len(z)) if np.isfinite(z_min[j])]
    c = [z[j] - fr(z_max[j]) for j in up] + [fr(z_min[j]) - z[j] for j in lo]
    C = zeros(len(c), len(z))
    for r, j in enumerate(up):
        C[r][j] = Fraction(1)
    for r, j in enumerate(lo):
        C[len(up) + r][j] = Fraction(-1)
    return Row(NEGATIVE, c, C, lam, mu)


def circle_row(xc, yc, rad, z, lam, mu, xi=0, yi=1):
    """CircleConstraint (src/constraints.jl:190-213): c_i = r_i^2 - (x - xc_i)^2 - (y - yc_i)^2"""
    z = frs(z)
    c, C = [], zeros(len(xc), len(z))
    for i, (a, b, r) in enumerate(zip(frs(xc), frs(yc), frs(rad))):
        dx, dy = z[xi] - a, z[yi] - b
        c.append(r * r - dx * dx - dy * dy)
        C[i][xi], C[i][yi] = -2 * dx, -2 * dy
    return Row(NEGATIVE, c, C, lam, mu)


def soc_norm_row(val, inds, z, lam, mu):
    """NormConstraint(..., SecondOrderCone()) (src/constraints.jl:462-517): c = [z[inds]; val], a selector Jacobian"""
    z = frs(z)
    C = zeros(len(inds) + 1, len(z))
    for r, j in enumerate(inds):
        C[r][j] = Fraction(1)
    return Row(SOC, [z[j] for j in inds] + [fr(val)], C, lam, mu)


def al_terms(row, g, H, lim):
    """the Gauss-Newton AL terms of `row` added to g, H on the first `lim` entries of z -> (penalty, violation)"""
    lbar = [l - row.mu * c for l, c in zip(row.lam, row.c)]
    dc = dualcone(row.cone)
    P, D = projection(dc, lbar), grad_projection(dc, lbar)
    p, nz = len(lbar), len(g)
    DC = [[sum(D[i][r] * row.C[r][j] for r in range(p)) for j in range(nz)] for i in range(p)]
    for j in range(lim):
        g[j] -= sum(DC[i][j] * P[i] for i in range(p))
        for j2 in range(lim):
            H[j][j2] += row.mu * sum(DC[i][j] * DC[i][j2] for i in range(p))
    pen = (sum(t * t for t in P) - sum(t * t for t in row.lam)) / (2 * row.mu)
    pc = projection(row.cone, row.c)
    return pen, max(abs(c - t) for c, t in zip(row.c, pc))


def diagonal_cost(Qd, Rd, q, r, x, u, terminal, c=0.0):
    """DiagonalCost (src/cost_functions.jl:89-233) -> (J, g, H) over z = [x; u]; the terminal knot has no control terms"""
    x, Qd, q = frs(x), frs(Qd), frs(q)
    n, m = len(x), len(Rd)
    g = [Qd[i] * x[i] + q[i] for i in range(n)] + [Fraction(0)] * m
    H = zeros(n + m, n + m)
    for i in range(n):
        H[i][i] = Qd[i]
    J = sum(Qd[i] * x[i] * x[i] / 2 + q[i] * x[i] for i in range(n)) + fr(c)
    if not terminal:
        u, Rd, r = frs(u), frs(Rd), frs(r)
        for a in range(m):
            g[n + a] = Rd[a] * u[a] + r[a]
            H[n + a][n + a] = Rd[a]
        J += sum(Rd[a] * u[a] * u[a] / 2 + r[a] * u[a] for a in range(m))
    return J, g, H


def knot_expansion(cost, rows, terminal, n):
    """cost = diagonal_cost(...) of the knot, rows = its constraints -> (J + penalty, violation, g, H), the AL terms on x alone at the
    terminal knot"""
    J, g, H = cost
    lim = n if terminal else len(g)
    pen, viol = Fraction(0), Fraction(0)
    for row in rows:
        p_, v_ = al_terms(row, g, H, lim)
        pen, viol = pen + p_, max(viol, v_)
    return J + pen, viol, g, H


def quat_G(q):
    """the 4 x 3 attitude block of RD.errstate_jacobian: columns (-x, w, z, -y), (-y, -z, w, x), (-z, y, -x, w)"""
    w, x, y, z = frs(q)
    cols = ((-x, w, z, -y), (-y, -z, w, x), (-z, y, -x, w))
    return [[cols[c][r] for c in range(3)] for r in range(4)]


def error_expansion(g, H, q, qs=3):
    """(g, H) over z = [x; u] with a unit quaternion at x[qs:qs+4] -> (G'g, G'HG - (q'g_q) I3 on the attitude block) over [dx; u]"""
    nz = len(g)
    Gq = quat_G(q)
    G = zeros(nz, nz - 1)
    for i in range(qs):
        G[i][i] = Fraction(1)
    for r in range(4):
        for c in range(3):
            G[qs + r][qs + c] = Gq[r][c]
    for i in range(qs + 4, nz):
        G[i][i - 1] = Fraction(1)
    ne = nz - 1
    ge = [sum(G[i][e] * g[i] for i in range(nz)) for e in range(ne)]
    HG = [[sum(H[i][k] * G[k][e] for k in range(nz)) for e in range(ne)] for i in range(nz)]
    He = [[sum(G[i][e] * HG[i][f] for i in range(nz)) for f in range(ne)] for e in range(ne)]
    qg = sum(fr(q[r]) * g[qs + r] for r in range(4))
    for c in range(3):
        He[qs + c][qs + c] -= qg
    return ge, He


def assert_entrywise(got, ref, what, ulps=4, floor=0.0):
    """every entry within `ulps` units in the last place of ITS OWN exact value (an exact zero must come out zero); `floor`: the least
    magnitude the ulps are taken of (for values that cancel to zero through inexact operations)"""
    got = np.asarray(got, dtype=float)
    ref_f = np.asarray(ref, dtype=object)
    assert got.shape == ref_f.shape, f"{what}: shape {got.shape} != {ref_f.shape}"
    exact = np.vectorize(lambda v: float(v))(ref_f) if ref_f.size else np.zeros(got.shape)
    tol = ulps * np.spacing(np.maximum(np.abs(exact), floor))
    err = np.abs(got - exact)
    bad = np.argwhere(~(err <= tol))
    assert bad.size == 0, (f"{what}: {len(bad)} entries off; first at {tuple(bad[0])}: got {got[tuple(bad[0])]!r}, exact "
                           f"{exact[tuple(bad[0])]!r}")


# ---- cases: problems whose inputs put rows exactly on their branch points -------------------------------------------------------------
# Every input is dyadic with a moderate exponent, every penalty a power of two, every quaternion (1,0,0,0) or (1/2,1/2,1/2,1/2) and every SOC
# vector a Pythagorean triple, so that lambda - mu c and the SOC norm are computed exactly by any evaluation order.  `inputs(eps)` moves each
# tie by the exact step eps to the side of its branch that the reference does NOT take (eps = 0: on the tie).
EPS = 2.0 ** -20
QW = (np.array([1.0, 0, 0, 0]), np.array([0.5, 0.5, 0.5, 0.5]))


class Con:
    """one constraint of a case: kind in goal / bound / circle / soc, its knot range (1-based, inclusive) and its data"""

    def __init__(self, kind, first, last, mu, **data):
        self.kind, self.first, self.last, self.mu, self.d = kind, first, last, mu, data

    def knots(self):
        return self.last - self.first + 1

    def p(self, n):
        """rows of the constraint at one knot"""
        if self.kind == "goal":
            return len(self.d.get("inds", range(n)))
        if self.kind == "bound":
            return int(np.isfinite(self.d["z_max"]).sum() + np.isfinite(self.d["z_min"]).sum())
        return {"circle": len(self.d.get("xc", ())), "soc": 3, "quatvec": 3}[self.kind]


class Case:
    """model, horizon, diagonal LQR cost (Qd, Rd, Qfd, xf), constraints; inputs(eps) -> X[B,N,n], U[B,N-1,m], [lambda_i[B,K_i,p_i]] and the
    per-instance Bound data {constraint index: (z_max[B,n+m], z_min[B,n+m])}"""

    def __init__(self, name, model, N, B, dt, cost, cons, inputs, error_state=False, inst_bounds=None):
        self.name, self.model, self.N, self.B, self.dt = name, model, N, B, dt
        self.cost, self.cons, self.inputs, self.error_state = cost, cons, inputs, error_state
        self.inst_bounds = inst_bounds or (lambda eps: {})

    def build(self, cls, TO, eps=0.0, instance=None):
        """the problem on `cls` (the CUDA Problem or the oracle) with the inputs of inputs(eps) set through the public setters;
        `instance`: that instance alone, its per-instance Bound data as the constraint's own (the oracle has no per-instance data)"""
        n, m = self.model.dims()
        Qd, Rd, Qfd, xf = self.cost
        obj = TO.LQRObjective(np.asarray(Qd, float), np.asarray(Rd, float), np.asarray(Qfd, float), np.asarray(xf, float), self.N)
        cons = TO.ConstraintList(n, m, self.N)
        for i, c in enumerate(self.cons):
            d = c.d
            if c.kind == "goal":
                con = TO.GoalConstraint(np.asarray(xf, float), inds=None if "inds" not in d else [j + 1 for j in d["inds"]])
            elif c.kind == "quatvec":
                con = TO.QuatVecEq(n, m, np.asarray(xf, float)[3:7])
            elif c.kind == "bound":
                zmax, zmin = (d["z_max"], d["z_min"]) if instance is None else self.bound_data(i, instance, eps)
                con = TO.BoundConstraint(n, m, x_min=zmin[:n], x_max=zmax[:n], u_min=zmin[n:], u_max=zmax[n:])
            elif c.kind == "circle":
                con = TO.CircleConstraint(n, d["xc"], d["yc"], d["r"])
            else:
                con = TO.NormConstraint(n, m, d["val"], TO.SecondOrderCone(), "control")
            TO.add_constraint(cons, con, (c.first, c.last))
        X, U, lams = self.inputs(eps)
        sl = slice(None) if instance is None else slice(instance, instance + 1)
        p = cls(self.model, obj, X[sl, 0].copy(), self.dt * (self.N - 1), xf=np.asarray(xf, float), constraints=cons,
                error_state=self.error_state)
        TO.rollout(p)
        TO.initial_states(p, X[sl])
        TO.initial_controls(p, U[sl])
        for i, c in enumerate(self.cons):
            TO.set_penalty(p, i, c.mu)
            TO.set_multipliers(p, i, lams[i][sl])
        if instance is None:
            for i, (zmax, zmin) in self.inst_bounds(eps).items():
                TO.set_constraint_data(p, i, np.concatenate([zmax, zmin], axis=1))
        return p

    def bound_data(self, i, b, eps):
        ib = self.inst_bounds(eps)
        if i in ib:
            return ib[i][0][b], ib[i][1][b]
        return self.cons[i].d["z_max"], self.cons[i].d["z_min"]

    def reference(self, eps=0.0):
        """exact (merit[B], violation[B], g[B][N], H[B][N]) of the full-state z = [x; u]"""
        X, U, lams = self.inputs(eps)
        n, m = self.model.dims()
        Qd, Rd, Qfd, xf = (np.asarray(a, float) for a in self.cost)
        merit, viol, G, H = [], [], [], []
        for b in range(self.B):
            Jb, vb, Gb, Hb = Fraction(0), Fraction(0), [], []
            for k in range(self.N):
                last = k == self.N - 1
                x = X[b, k]
                u = np.zeros(m) if last else U[b, k]
                z = np.concatenate([x, u])
                Qk = Qfd if last else Qd
                cost = diagonal_cost(Qk, Rd, -Qk * xf, np.zeros(m), x, u, last, c=Fraction(0))
                cost = (cost[0] + sum(fr(Qk[i]) * fr(xf[i]) ** 2 / 2 for i in range(n)), cost[1], cost[2])
                rows = []
                for i, c in enumerate(self.cons):
                    if not c.first <= k + 1 <= c.last:
                        continue
                    lam, d = lams[i][b, k + 1 - c.first], c.d
                    if c.kind == "goal":
                        rows.append(goal_row(xf, x, n + m, lam, c.mu, inds=d.get("inds")))
                    elif c.kind == "quatvec":
                        rows.append(quatvec_row(xf[3:7], x, n + m, lam, c.mu))
                    elif c.kind == "bound":
                        zmax, zmin = self.bound_data(i, b, eps)
                        rows.append(bound_row(zmax, zmin, z, lam, c.mu))
                    elif c.kind == "circle":
                        rows.append(circle_row(d["xc"], d["yc"], d["r"], z, lam, c.mu))
                    else:
                        rows.append(soc_norm_row(d["val"], [n + a for a in range(m)], z, lam, c.mu))
                Jk, vk, g, Hk = knot_expansion(cost, rows, last, n)
                Jb, vb = Jb + Jk, max(vb, vk)
                Gb.append(g); Hb.append(Hk)
            merit.append(Jb); viol.append(vb); G.append(Gb); H.append(Hb)
        return merit, viol, G, H

    def error_reference(self, eps=0.0):
        """exact (g_e[B][N], H_e[B][N]) over [dx; u] (Quadrotor: the attitude at x[3:7])"""
        X = self.inputs(eps)[0]
        _, _, G, H = self.reference(eps)
        out_g, out_H = [], []
        for b in range(self.B):
            ge_b, He_b = [], []
            for k in range(self.N):
                ge, He = error_expansion(G[b][k], H[b][k], X[b, k, 3:7])
                ge_b.append(ge); He_b.append(He)
            out_g.append(ge_b); out_H.append(He_b)
        return out_g, out_H


def _quad_states(B, N):
    """dyadic Quadrotor states: positions, velocities and rates on a coarse grid, the attitude alternating (1,0,0,0) / (1/2,1/2,1/2,1/2)"""
    X = np.zeros((B, N, 13))
    for b in range(B):
        for k in range(N):
            X[b, k, :3] = (k / 4 - b / 8, -k / 8, 1 + k / 16)
            X[b, k, 3:7] = QW[(k + b) % 2]
            X[b, k, 7:10] = (1 / 8, -1 / 4, b / 16)
            X[b, k, 10:13] = (1 / 32, 0, -1 / 16)
    return X


def quadrotor_case(error_state=True, extra_box=False, inst_data=False, quat_goal=False, B=3, N=6):
    """Quadrotor, DiagonalCost, the control box u in [0, 8] with u_4 pinned (u_min == u_max == 1), a position box on every knot and the
    Goal at N.  Ties (instance, entry): b0 u_1 = 0 (lower row; the motor at w = 0), b1 u_2 = 8 (upper row), b2 u_3 = 8 + 1/4 with
    lambda = mu / 4 (a tie with lambda != 0), every instance u_4 = 1 (both rows of one entry), b0 x_1 = 4 at knot 1 (state upper row),
    b1 y = -4 and b2 z = 4 at the terminal knot (state lower and upper rows beside the Goal's equality row).  `extra_box`: a second, inactive control box
    (4 rows on u_4: the descriptor walk).  `inst_data`: instance b's control box from set_constraint_data, the tie on u_2 moved into the data:
    b0 u_max_2 = u_2 (tie), b1 u_max_2 = u_2 + 2^-20 (inactive by one step), b2 u_max_2 = u_2 - 1/4 with lambda = mu / 4.
    `quat_goal`: the Goal on position and rates and a QuatVecEq on the attitude instead (examples' quadrotor_lie: not the compact class)"""
    import trajopt_b200 as TO
    n, m = 13, 4
    xf = np.array([0, 0, 2, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0.0])
    inf = np.inf
    box = Con("bound", 1, N - 1, 4.0, z_max=np.r_[np.full(n, inf), [8, 8, 8, 1.0]], z_min=np.r_[np.full(n, -inf), [0, 0, 0, 1.0]])
    pos = Con("bound", 1, N, 2.0, z_max=np.r_[[4, 4, 4.0], np.full(n - 3 + m, inf)], z_min=np.r_[[-4, -4, -4.0], np.full(n - 3 + m, -inf)])
    cons = [box, pos, Con("goal", N, N, 8.0)]
    if quat_goal:
        cons = [box, pos, Con("goal", N, N, 8.0, inds=[0, 1, 2, 7, 8, 9, 10, 11, 12]), Con("quatvec", N, N, 4.0)]
    if extra_box:
        cons.append(Con("bound", 1, N - 1, 16.0, z_max=np.r_[np.full(n, inf), np.full(m, 16.0)], z_min=np.r_[np.full(n, -inf), np.full(m, -16.0)]))

    def inputs(eps):
        X = _quad_states(B, N)
        U = np.tile(np.array([2, 3, 5 / 2, 1.0]), (B, N - 1, 1))
        lams = [np.zeros((B, c.knots(), c.p(n))) for c in cons]
        lams[2][:, 0, :] = np.arange(cons[2].p(n)) / 8 - 1 / 2      # the Goal's equality rows: always active, any lambda
        if quat_goal:
            lams[3][:, 0, :] = (1 / 4, -1 / 8, 1 / 2)
        U[0, :, 0] = eps                                            # lower row of u_1 (and the motor tie)
        if not inst_data:
            U[1, :, 1] = 8 - eps                                    # upper row of u_2
        U[2, :, 2] = 8 + 1 / 4
        lams[0][2, :, 2] = box.mu / 4 + eps                         # upper row of u_3 at a tie with lambda != 0
        U[:, :, 3] = 1 + eps                                        # both rows of the pinned u_4 (eps > 0: the lower row leaves)
        X[0, 0, 0] = 4 - eps                                        # state upper row at knot 1
        X[1, N - 1, 1] = -4 + eps                                   # state lower row at the terminal knot, beside the Goal
        X[2, N - 1, 2] = 4 - eps                                    # state upper row at the terminal knot
        if inst_data:
            lams[0][2, :, 1] = box.mu / 4 + eps
        return X, U, lams

    def inst_bounds(eps):
        if not inst_data:
            return {}
        zmax = np.tile(box.d["z_max"], (B, 1)); zmin = np.tile(box.d["z_min"], (B, 1))
        zmax[0, n + 1] = 3 + eps; zmax[1, n + 1] = 3 + EPS + eps; zmax[2, n + 1] = 3 - 1 / 4
        return {0: (zmax, zmin)}

    name = "quadrotor_" + ("error_state" if error_state else "full_state") + ("_extra_box" if extra_box else "") + ("_inst_data" if inst_data else "")
    name += "_quat_goal" if quat_goal else ""
    return Case(name, TO.Quadrotor(), N, B, 1 / 16, (np.full(n, 1 / 8), np.full(m, 1 / 64), np.full(n, 64.0), xf), cons, inputs,
                error_state=error_state, inst_bounds=inst_bounds)


def small_case(model_name, B=2, N=6):
    """Cartpole or DoubleIntegrator(2), DiagonalCost, the control box u in [-3, 3] and the Goal.  Ties: b0 u = -3 at even knots (lower row),
    +3 at odd knots (upper row); b1 u_1 = 3 + 1/2 with lambda = mu / 2 (a tie with lambda != 0); the rest strictly inside"""
    import trajopt_b200 as TO
    model = TO.Cartpole() if model_name == "cartpole" else TO.DoubleIntegrator(2)
    n, m = model.dims()
    xf = np.array([0, 3, 0, 0.0])
    box = Con("bound", 1, N - 1, 2.0, z_max=np.r_[np.full(n, np.inf), np.full(m, 3.0)], z_min=np.r_[np.full(n, -np.inf), np.full(m, -3.0)])
    cons = [box, Con("goal", N, N, 4.0)]

    def inputs(eps):
        X = np.zeros((B, N, n))
        for k in range(N):
            X[:, k] = (k / 8, 1 + k / 4, 1 / 16, -k / 32)
        U = np.full((B, N - 1, m), 1 / 2)
        for k in range(N - 1):
            U[0, k, 0] = -3 + eps if k % 2 == 0 else 3 - eps
        U[1, :, 0] = 3 + 1 / 2
        lams = [np.zeros((B, N - 1, 2 * m)), np.zeros((B, 1, n))]
        lams[0][1, :, 0] = box.mu / 2 + eps
        lams[1][:, 0] = (1 / 4, -1 / 2, 1, 0)
        return X, U, lams

    return Case(model_name, model, N, B, 1 / 8, (np.full(n, 1 / 8), np.full(m, 1 / 16), np.full(n, 16.0), xf), cons, inputs)


def soc_case_problem(B=3, N=5):
    """examples/quickstart.jl-like: DoubleIntegrator(2), Goal, a Circle (knots 2..N-1), the SOC NormConstraint |u| <= 5 and the box
    u in [-4, 4].  u = (3, 4) everywhere and mu = 1 on the norm, so lambda = (6, 8, 10) / (3, 4, 5) / 0 puts lambda - mu c on the SOC
    boundary (a = s), at the apex and below the cone (a = -s) in instances 0, 1, 2.  The circle's row ties at knot 2 ((x, y) on the
    circle), is active at knot 3 (the centre) and inactive at knot 4; u_2 = 4 ties the box's upper row"""
    import trajopt_b200 as TO
    n, m = 4, 2
    xf = np.array([0, 2, 0, 0.0])
    cons = [Con("goal", N, N, 2.0), Con("circle", 2, N - 1, 4.0, xc=[0.0], yc=[1.0], r=[5 / 8]), Con("soc", 1, N - 1, 1.0, val=5.0),
            Con("bound", 1, N - 1, 2.0, z_max=np.r_[np.full(n, np.inf), [4, 4.0]], z_min=np.r_[np.full(n, -np.inf), [-4, -4.0]])]

    def inputs(eps):
        X = np.zeros((B, N, n))
        for k in range(N):
            X[:, k] = (1 / 2, k / 2, 1 / 8, -1 / 4)
        X[:, 1, :2] = (3 / 8, 3 / 2 + eps)                    # on the circle (3-4-5 triangle of radius 5/8)
        X[:, 2, :2] = (0, 1)                                  # its centre
        X[:, 3, :2] = (2, 2)                                  # outside
        U = np.tile(np.array([3, 4.0]), (B, N - 1, 1))
        U[:, :, 1] -= eps
        soc = np.zeros((B, N - 1, 3))
        soc[0] = (6, 8, 10 - eps)
        soc[1] = (3 + 3 * eps, 4 + 4 * eps, 5)
        soc[2] = (0, 0, eps)
        lams = [np.zeros((B, 1, n)), np.zeros((B, N - 2, 1)), soc, np.zeros((B, N - 1, 2 * m))]
        lams[0][:, 0] = (1 / 2, -1 / 4, 1 / 8, 1)
        return X, U, lams

    return Case("double_integrator_soc", TO.DoubleIntegrator(2), N, B, 1 / 4, (np.ones(n), np.ones(m), np.full(n, 8.0), xf), cons, inputs)


def soc_points(p):
    """(x, b, case) with x[:-1] of rational norm a and x[-1] = s: on the boundary (a = s), at the apex, below (a = -s), strictly in,
    strictly below and outside (s = 0, s = a / 2, s = -a / 2)"""
    v = {1: [3.0], 2: [3.0, 4.0], 3: [1.0, 2.0, 2.0], 6: [1.0, 1.0, 1.0, 1.0, 4.0, 4.0]}[p - 1]
    v = np.array(v) / 2
    a = float(exact_sqrt(sum(fr(t) ** 2 for t in v)))
    pts = [(a, "in"), (-a, "below"), (2 * a, "in"), (-2 * a, "below"), (0.0, "outside"), (a / 2, "outside"), (-a / 2, "outside")]
    out = [(np.r_[v, s], case) for s, case in pts] + [(np.zeros(p), "below")]
    b = np.arange(1, p + 1) / 4 - 1
    return [(x, b, case) for x, case in out]
