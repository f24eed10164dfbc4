// costcon.cuh -- per-knot cost / constraint / cone device functions (pointer based, runtime n and m).
// Every function is a pure map over ONE knot z = [x;u] (reference docs/src/costfunctions.md:16) so any
// (instance, knot) pair can be evaluated by any thread.
//
// Mirrors (reference file:line):
//   cost_value        RD.evaluate(::QuadraticCostFunction,x,u)   src/cost_functions.jl:89-104
//   cost_gradient     RD.gradient!                               src/cost_functions.jl:137-172
//   cost_hessian      RD.hessian!                                src/cost_functions.jl:212-233
//   con_evaluate      RD.evaluate(con, z)                        src/constraints.jl:55-61 (Goal), :738-755 (Bound),
//                                                                :135-139 (Linear), :190-199 (Circle), :278-290 (Sphere), :462-465 (Norm)
//   con_jacobian      RD.jacobian!(con, jac, c, z)               src/constraints.jl:62-68, :757-765, :140-144, :201-213, :292-306, :493-517
//   cone_projection / cone_grad_projection / cone_hess_projection  src/cones.jl:96-127, :129-188, :201-276
//   dualcone          src/cones.jl:65-69
#pragma once
#include "common.cuh"

__device__ __forceinline__ int dualcone(int cone) {
    return cone == CONE_IDENTITY ? CONE_ZERO : (cone == CONE_ZERO ? CONE_IDENTITY : cone);
}

// ---- user cost as a straight-line program, evaluated with second-order forward-mode duals (value, d/ds, d/dt, d2/dsdt) ----------
struct Hyper { double v, d1, d2, d12; };
__device__ __forceinline__ Hyper hyp_unary(const Hyper& a, double f, double f1, double f2) {
    Hyper r; r.v = f; r.d1 = f1 * a.d1; r.d2 = f1 * a.d2; r.d12 = f1 * a.d12 + f2 * a.d1 * a.d2; return r;
}
__device__ __forceinline__ Hyper hyp_mul(const Hyper& a, const Hyper& b) {
    Hyper r; r.v = a.v * b.v; r.d1 = a.d1 * b.v + a.v * b.d1; r.d2 = a.d2 * b.v + a.v * b.d2;
    r.d12 = a.d12 * b.v + a.d1 * b.d2 + a.d2 * b.d1 + a.v * b.d12; return r;
}
// z_s1 seeded in d1, z_s2 in d2 (index into [x;u], -1 = none); has_u = false: u = 0 (terminal knot).  Mirrors oracle expr_eval.
__device__ inline void expr_run(const int* prog, int L, const double* pconst, int n, const double* x, const double* u, bool has_u, int s1, int s2, Hyper* reg) {
    for (int i = 0; i < L; i++) {
        const int op = prog[3 * i], a = prog[3 * i + 1], b = prog[3 * i + 2];
        Hyper r; r.v = 0; r.d1 = 0; r.d2 = 0; r.d12 = 0;
        switch (op) {
            case 0: r.v = pconst[a]; break;
            case 1: r.v = x[a]; r.d1 = (a == s1) ? 1.0 : 0.0; r.d2 = (a == s2) ? 1.0 : 0.0; break;
            case 2: r.v = has_u ? u[a] : 0.0; r.d1 = (n + a == s1) ? 1.0 : 0.0; r.d2 = (n + a == s2) ? 1.0 : 0.0; break;
            case 3: r.v = reg[a].v + reg[b].v; r.d1 = reg[a].d1 + reg[b].d1; r.d2 = reg[a].d2 + reg[b].d2; r.d12 = reg[a].d12 + reg[b].d12; break;
            case 4: r.v = reg[a].v - reg[b].v; r.d1 = reg[a].d1 - reg[b].d1; r.d2 = reg[a].d2 - reg[b].d2; r.d12 = reg[a].d12 - reg[b].d12; break;
            case 5: r = hyp_mul(reg[a], reg[b]); break;
            case 6: { const double iv = 1.0 / reg[b].v; r = hyp_mul(reg[a], hyp_unary(reg[b], iv, -iv * iv, 2 * iv * iv * iv)); break; }
            case 7: r.v = -reg[a].v; r.d1 = -reg[a].d1; r.d2 = -reg[a].d2; r.d12 = -reg[a].d12; break;
            case 8: { double sv, cv; sincos(reg[a].v, &sv, &cv); r = hyp_unary(reg[a], sv, cv, -sv); break; }
            case 9: { double sv, cv; sincos(reg[a].v, &sv, &cv); r = hyp_unary(reg[a], cv, -sv, -cv); break; }
            case 10: { const double e = exp(reg[a].v); r = hyp_unary(reg[a], e, e, e); break; }
            case 11: { const double iv = 1.0 / reg[a].v; r = hyp_unary(reg[a], log(reg[a].v), iv, -iv * iv); break; }
            case 12: { const double sq = sqrt(reg[a].v); r = hyp_unary(reg[a], sq, 0.5 / sq, -0.25 / (sq * reg[a].v)); break; }
            case 13: { const double e = pconst[b], v = reg[a].v; r = hyp_unary(reg[a], pow(v, e), e * pow(v, e - 1), e * (e - 1) * pow(v, e - 2)); break; }
            case 14: { const double t = tanh(reg[a].v); r = hyp_unary(reg[a], t, 1 - t * t, -2 * t * (1 - t * t)); break; }
            case 15: r = reg[a]; r.v += pconst[b]; break;
            case 16: { const double k = pconst[b]; r.v = reg[a].v * k; r.d1 = reg[a].d1 * k; r.d2 = reg[a].d2 * k; r.d12 = reg[a].d12 * k; break; }
            case 17: { const double k = pconst[b]; r.v = reg[a].v / k; r.d1 = reg[a].d1 / k; r.d2 = reg[a].d2 / k; r.d12 = reg[a].d12 / k; break; }
            case 18: { const double k = pconst[b], iv = 1.0 / reg[a].v; r = hyp_unary(reg[a], k * iv, -k * iv * iv, 2 * k * iv * iv * iv); break; }
            case 19: r.v = pconst[b] - reg[a].v; r.d1 = -reg[a].d1; r.d2 = -reg[a].d2; r.d12 = -reg[a].d12; break;
        }
        reg[i] = r;
    }
}
__device__ inline Hyper expr_eval(const DevCost& c, int n, const double* x, const double* u, bool has_u, int s1, int s2) {
    Hyper reg[TO_EXPR_LEN];
    expr_run(c.prog, c.prog_len, c.pconst, n, x, u, has_u, s1, s2, reg);
    return reg[c.prog_len - 1];
}

// geodesic term of DiagonalQuatCost (src/lie_costs.jl:74-76): w min(1 + dq, 1 - dq), dq = q_ref'x[q_ind]
__device__ __forceinline__ double quat_cost_term(const DevCost& c, const double* x) {
    double dq = 0;
    for (int i = 0; i < 4; i++) dq = fma(c.q_ref[i], x[c.q_ind[i]], dq);
    return c.w * fmin(1 + dq, 1 - dq);
}

// q, r: the linear terms to use (c.q / c.r, or an instance's row of DevProblem::qr, inst_q / inst_r)
__device__ inline double cost_value(const DevCost& c, const double* q, const double* r, int n, int m, const double* x, const double* u, bool has_u) {
    if (c.expr) return expr_eval(c, n, x, u, has_u, -1, -1).v;
    double J = 0;
    if (c.diag) {
        double a = 0, l = 0;
        for (int i = 0; i < n; i++) { a = fma(c.Qd[i] * x[i], x[i], a); l = fma(q[i], x[i], l); }
        J = 0.5 * a + l + c.c;
        if (has_u) {
            double au = 0, lu = 0;
            for (int i = 0; i < m; i++) { au = fma(c.Rd[i] * u[i], u[i], au); lu = fma(r[i], u[i], lu); }
            J += 0.5 * au + lu;
        }
        if (c.quat) J += quat_cost_term(c, x);
        return J;
    }
    for (int j = 0; j < n; j++) {
        double qx = 0;
        for (int i = 0; i < n; i++) qx = fma(c.Q[j * n + i], x[i], qx);
        J = fma(0.5 * qx, x[j], J);
    }
    double lin = 0;
    for (int i = 0; i < n; i++) lin = fma(q[i], x[i], lin);
    J += lin + c.c;
    if (has_u) {
        double Ju = 0, linu = 0;
        for (int j = 0; j < m; j++) {
            double ru = 0;
            for (int i = 0; i < m; i++) ru = fma(c.R[j * m + i], u[i], ru);
            Ju = fma(0.5 * ru, u[j], Ju);
        }
        for (int i = 0; i < m; i++) linu = fma(r[i], u[i], linu);
        J += Ju + linu;
        if (!c.zeroH) {
            double h = 0;
            for (int j = 0; j < n; j++)
                for (int i = 0; i < m; i++) h = fma(u[i] * c.H[j * m + i], x[j], h);
            J += h;
        }
    }
    return J;
}
__device__ inline double cost_value(const DevCost& c, int n, int m, const double* x, const double* u, bool has_u) {
    return cost_value(c, c.q, c.r, n, m, x, u, has_u);
}

// grad[n+m]; the u-part is left untouched at the terminal knot (the reference skips it when is_terminal(z))
template <bool QUAT = true>
__device__ inline void cost_gradient_quadratic(const DevCost& c, const double* q, const double* r, int n, int m, const double* x, const double* u, bool is_terminal, double* grad);
__device__ inline void cost_gradient(const DevCost& c, const double* q, const double* r, int n, int m, const double* x, const double* u, bool is_terminal, double* grad) {
    if (c.expr) {   // RD.gradient!(ForwardAD) of a user cost
        const int lim = is_terminal ? n : n + m;
        for (int i = 0; i < lim; i++) grad[i] = expr_eval(c, n, x, u, !is_terminal, i, -1).d1;
        return;
    }
    cost_gradient_quadratic(c, q, r, n, m, x, u, is_terminal, grad);
}
__device__ inline void cost_gradient(const DevCost& c, int n, int m, const double* x, const double* u, bool is_terminal, double* grad) {
    cost_gradient(c, c.q, c.r, n, m, x, u, is_terminal, grad);
}
// QuadraticCostFunction only (the register-resident kernels call this directly with QUAT = false: no dynamically indexed stores)
template <bool QUAT>
__device__ inline void cost_gradient_quadratic(const DevCost& c, const double* q, const double* r, int n, int m, const double* x, const double* u, bool is_terminal, double* grad) {
    for (int i = 0; i < n; i++) {
        double g = q[i];
        if (c.diag) g = fma(c.Qd[i], x[i], g);
        else for (int j = 0; j < n; j++) g = fma(c.Q[j * n + i], x[j], g);
        grad[i] = g;
    }
    if (QUAT && c.quat) {   // gradient!(::DiagonalQuatCost) src/lie_costs.jl:79-95: -+ w q_ref by the sign of q_ref'p
        double dq = 0;
        for (int i = 0; i < 4; i++) dq = fma(c.q_ref[i], x[c.q_ind[i]], dq);
        const double sw = dq < 0 ? c.w : -c.w;
        for (int i = 0; i < 4; i++) grad[c.q_ind[i]] = fma(sw, c.q_ref[i], grad[c.q_ind[i]]);
    }
    if (!is_terminal) {
        for (int i = 0; i < m; i++) {
            double g = r[i];
            if (c.diag) g = fma(c.Rd[i], u[i], g);
            else for (int j = 0; j < m; j++) g = fma(c.R[j * m + i], u[j], g);
            grad[n + i] = g;
        }
        if (!c.zeroH)
            for (int j = 0; j < n; j++)
                for (int i = 0; i < m; i++) {
                    grad[j] = fma(c.H[j * m + i], u[i], grad[j]);
                    grad[n + i] = fma(c.H[j * m + i], x[j], grad[n + i]);
                }
    }
}

// hess (n+m)x(n+m) col-major, written in full and symmetric (the reference writes only the lower-left H block
// and leaves the rest to the caller's zero initialisation, SURVEY.md 2.4)
__device__ inline void cost_hessian_quadratic(const DevCost& c, int n, int m, bool is_terminal, double* hess);
__device__ inline void cost_hessian(const DevCost& c, int n, int m, const double* x, const double* u, bool is_terminal, double* hess) {
    const int nm = n + m;
    if (c.expr) {   // RD.hessian!(ForwardAD) of a user cost: one second-order pass per entry of the lower triangle
        for (int i = 0; i < nm * nm; i++) hess[i] = 0;
        const int lim = is_terminal ? n : nm;
        for (int j = 0; j < lim; j++)
            for (int i = j; i < lim; i++) { const double h = expr_eval(c, n, x, u, !is_terminal, i, j).d12; hess[j * nm + i] = h; hess[i * nm + j] = h; }
        return;
    }
    cost_hessian_quadratic(c, n, m, is_terminal, hess);
}
__device__ inline void cost_hessian_quadratic(const DevCost& c, int n, int m, bool is_terminal, double* hess) {
    const int nm = n + m;
    for (int i = 0; i < nm * nm; i++) hess[i] = 0;
    for (int j = 0; j < n; j++)
        for (int i = 0; i < n; i++) if (!c.diag || i == j) hess[j * nm + i] = c.Q[j * n + i];
    if (!is_terminal) {
        for (int j = 0; j < m; j++)
            for (int i = 0; i < m; i++) if (!c.diag || i == j) hess[(n + j) * nm + n + i] = c.R[j * m + i];
        if (!c.zeroH)
            for (int j = 0; j < n; j++)
                for (int i = 0; i < m; i++) { hess[j * nm + n + i] = c.H[j * m + i]; hess[(n + i) * nm + j] = c.H[j * m + i]; }
    }
}

__device__ __forceinline__ double zget(int n, const double* x, const double* u, int j) { return j < n ? x[j] : u[j - n]; }

// goal: the Goal values to use (con.a, or an instance's row of DevProblem::cdata, con_data); read for CON_GOAL only
__device__ inline void con_evaluate(const DevCon& con, const double* goal, int n, int m, const double* x, const double* u, double* c) {
    switch (con.kind) {
        case CON_GOAL:
            for (int i = 0; i < con.p; i++) c[i] = x[con.inds[i]] - goal[i];
            break;
        case CON_BOUND: {   // upper block first, then the lower block
            int i = 0;
            for (int r = 0; r < con.n_max; r++, i++) { int j = con.a_max[r]; c[i] = zget(n, x, u, j) - con.a[j]; }
            for (int r = 0; r < con.n_min; r++, i++) { int j = con.a_min[r]; c[i] = con.b[j] - zget(n, x, u, j); }
            break;
        }
        case CON_LINEAR: {
            const double* y = con.flag ? u : x;
            const int w = con.flag ? m : n;
            for (int i = 0; i < con.p; i++) {
                double s = -con.b[i];
                for (int j = 0; j < w; j++) s = fma(con.a[j * con.p + i], y[j], s);
                c[i] = s;
            }
            break;
        }
        case CON_CIRCLE:
            for (int i = 0; i < con.p; i++) {
                double dx = x[con.inds[0]] - con.a[i], dy = x[con.inds[1]] - con.b[i];
                c[i] = -(dx * dx) - (dy * dy) + con.rad[i] * con.rad[i];
            }
            break;
        case CON_SPHERE:
            for (int i = 0; i < con.p; i++) {
                double dx = x[con.inds[0]] - con.a[i], dy = x[con.inds[1]] - con.b[i], dz = x[con.inds[2]] - con.c3[i];
                c[i] = -(dx * dx) - (dy * dy) - (dz * dz) + con.rad[i] * con.rad[i];
            }
            break;
        case CON_NORM:
            if (con.sense == CONE_SECOND_ORDER) {
                for (int i = 0; i < con.ninds; i++) c[i] = zget(n, x, u, con.inds[i]);
                c[con.ninds] = con.val;
            } else {
                double s = 0;
                for (int i = 0; i < con.ninds; i++) { double z = zget(n, x, u, con.inds[i]); s = fma(z, z, s); }
                c[0] = s - con.val * con.val;
            }
            break;
        case CON_COLLISION: {   // src/constraints.jl:367-376: r^2 - sum_i (x[x1_i] - x[x2_i])^2, accumulated in that order
            const int D = con.ninds / 2;
            double s = con.val * con.val;
            for (int i = 0; i < D; i++) { const double d = x[con.inds[i]] - x[con.inds[D + i]]; s -= d * d; }
            c[0] = s;
            break;
        }
        case CON_EXPR: {   // user constraint recorded as a program (docs/src/constraint_interface.md:52-72)
            Hyper reg[TO_EXPR_LEN];
            expr_run(con.prog, con.prog_len, con.pconst, n, x, u, true, -1, -1, reg);
            for (int i = 0; i < con.p; i++) c[i] = reg[con.prog_len - con.p + i].v;
            break;
        }
        case CON_QUATVEC: {   // QuatVecEq src/constraints.jl:947-956
            double q[4], nrm = 0, dq = 0;
            for (int i = 0; i < 4; i++) { q[i] = x[con.inds[i]]; nrm = fma(q[i], q[i], nrm); }
            nrm = sqrt(nrm);
            for (int i = 0; i < 4; i++) { q[i] /= nrm; dq = fma(con.a[i], q[i], dq); }
            const double sg = dq < 0 ? -1.0 : 1.0;
            for (int i = 0; i < 3; i++) c[i] = -(sg * con.a[i + 1] - q[i + 1]);
            break;
        }
    }
}
__device__ inline void con_evaluate(const DevCon& con, int n, int m, const double* x, const double* u, double* c) {
    con_evaluate(con, con.a, n, m, x, u, c);
}

// jac: p x (n+m) col-major, fully written
__device__ inline void con_jacobian(const DevCon& con, int n, int m, const double* x, const double* u, double* jac) {
    const int p = con.p, w = n + m;
    for (int i = 0; i < p * w; i++) jac[i] = 0;
    switch (con.kind) {
        case CON_GOAL: for (int i = 0; i < p; i++) jac[con.inds[i] * p + i] = 1; break;
        case CON_BOUND: {
            int i = 0;
            for (int r = 0; r < con.n_max; r++, i++) jac[con.a_max[r] * p + i] = 1;
            for (int r = 0; r < con.n_min; r++, i++) jac[con.a_min[r] * p + i] = -1;
            break;
        }
        case CON_LINEAR: {
            const int off = con.flag ? n : 0, wd = con.flag ? m : n;
            for (int j = 0; j < wd; j++) for (int i = 0; i < p; i++) jac[(off + j) * p + i] = con.a[j * p + i];
            break;
        }
        case CON_CIRCLE:
            for (int i = 0; i < p; i++) {
                jac[con.inds[0] * p + i] = -2 * (x[con.inds[0]] - con.a[i]);
                jac[con.inds[1] * p + i] = -2 * (x[con.inds[1]] - con.b[i]);
            }
            break;
        case CON_SPHERE:
            for (int i = 0; i < p; i++) {
                jac[con.inds[0] * p + i] = -2 * (x[con.inds[0]] - con.a[i]);
                jac[con.inds[1] * p + i] = -2 * (x[con.inds[1]] - con.b[i]);
                jac[con.inds[2] * p + i] = -2 * (x[con.inds[2]] - con.c3[i]);
            }
            break;
        case CON_NORM:
            if (con.sense == CONE_SECOND_ORDER) for (int i = 0; i < con.ninds; i++) jac[con.inds[i] * p + i] = 1;
            else for (int i = 0; i < con.ninds; i++) jac[con.inds[i] * p + 0] = 2 * zget(n, x, u, con.inds[i]);
            break;
        case CON_COLLISION: {   // :378-389 (assignments, as in the reference)
            const int D = con.ninds / 2;
            for (int i = 0; i < D; i++) {
                const double d = x[con.inds[i]] - x[con.inds[D + i]];
                jac[con.inds[i] * p] = -2 * d;
                jac[con.inds[D + i] * p] = 2 * d;
            }
            break;
        }
        case CON_EXPR: {   // RD.jacobian!(ForwardAD): one first-order pass per input
            Hyper reg[TO_EXPR_LEN];
            for (int j = 0; j < w; j++) {
                expr_run(con.prog, con.prog_len, con.pconst, n, x, u, true, j, -1, reg);
                for (int i = 0; i < p; i++) jac[j * p + i] = reg[con.prog_len - p + i].d1;
            }
            break;
        }
        case CON_QUATVEC: {   // d normalize(q)/dq = (I - qh qh')/|q|, rows 2:4 (what ForwardAD gives, src/constraints.jl:938,962)
            double q[4], nrm = 0;
            for (int i = 0; i < 4; i++) { q[i] = x[con.inds[i]]; nrm = fma(q[i], q[i], nrm); }
            nrm = sqrt(nrm);
            for (int i = 0; i < 4; i++) q[i] /= nrm;
            for (int j = 0; j < 4; j++)
                for (int i = 0; i < 3; i++) jac[con.inds[j] * p + i] = ((i + 1 == j ? 1.0 : 0.0) - q[i + 1] * q[j]) / nrm;
            break;
        }
    }
}

// The INST overloads: d = the data of an instance (con_data).  The kinds whose data may differ per instance are evaluated here with the shared
// overloads' arithmetic, operation for operation; the others go to the shared overloads (a Goal with d.a, its instance's values).
__device__ inline void con_evaluate(const DevCon& con, const ConData& d, int n, int m, const double* x, const double* u, double* c) {
    switch (con.kind) {
        case CON_BOUND: {
            int i = 0;
            for (int r = 0; r < con.n_max; r++, i++) { int j = con.a_max[r]; c[i] = zget(n, x, u, j) - d.a[j]; }
            for (int r = 0; r < con.n_min; r++, i++) { int j = con.a_min[r]; c[i] = d.b[j] - zget(n, x, u, j); }
            break;
        }
        case CON_LINEAR: {
            const double* y = con.flag ? u : x;
            const int w = con.flag ? m : n;
            for (int i = 0; i < con.p; i++) {
                double s = -d.b[i];
                for (int j = 0; j < w; j++) s = fma(con.a[j * con.p + i], y[j], s);
                c[i] = s;
            }
            break;
        }
        case CON_CIRCLE:
            for (int i = 0; i < con.p; i++) {
                double dx = x[con.inds[0]] - d.a[i], dy = x[con.inds[1]] - d.b[i];
                c[i] = -(dx * dx) - (dy * dy) + d.rad[i] * d.rad[i];
            }
            break;
        case CON_SPHERE:
            for (int i = 0; i < con.p; i++) {
                double dx = x[con.inds[0]] - d.a[i], dy = x[con.inds[1]] - d.b[i], dz = x[con.inds[2]] - d.c3[i];
                c[i] = -(dx * dx) - (dy * dy) - (dz * dz) + d.rad[i] * d.rad[i];
            }
            break;
        case CON_NORM:
            if (con.sense == CONE_SECOND_ORDER) {
                for (int i = 0; i < con.ninds; i++) c[i] = zget(n, x, u, con.inds[i]);
                c[con.ninds] = d.val;
            } else {
                double s = 0;
                for (int i = 0; i < con.ninds; i++) { double z = zget(n, x, u, con.inds[i]); s = fma(z, z, s); }
                c[0] = s - d.val * d.val;
            }
            break;
        case CON_COLLISION: {
            const int D = con.ninds / 2;
            double s = d.val * d.val;
            for (int i = 0; i < D; i++) { const double dd = x[con.inds[i]] - x[con.inds[D + i]]; s -= dd * dd; }
            c[0] = s;
            break;
        }
        default: con_evaluate(con, d.a, n, m, x, u, c);
    }
}
__device__ inline void con_jacobian(const DevCon& con, const ConData& d, int n, int m, const double* x, const double* u, double* jac) {
    const int p = con.p, w = n + m;
    switch (con.kind) {
        case CON_CIRCLE:
            for (int i = 0; i < p * w; i++) jac[i] = 0;
            for (int i = 0; i < p; i++) {
                jac[con.inds[0] * p + i] = -2 * (x[con.inds[0]] - d.a[i]);
                jac[con.inds[1] * p + i] = -2 * (x[con.inds[1]] - d.b[i]);
            }
            break;
        case CON_SPHERE:
            for (int i = 0; i < p * w; i++) jac[i] = 0;
            for (int i = 0; i < p; i++) {
                jac[con.inds[0] * p + i] = -2 * (x[con.inds[0]] - d.a[i]);
                jac[con.inds[1] * p + i] = -2 * (x[con.inds[1]] - d.b[i]);
                jac[con.inds[2] * p + i] = -2 * (x[con.inds[2]] - d.c3[i]);
            }
            break;
        default: con_jacobian(con, n, m, x, u, jac);   // independent of the data that may differ per instance
    }
}
// the values / Jacobian of constraint con = P.cons[ci] for instance b: the INST overloads with its data (con_data), or the shared overloads
template <bool INST>
__device__ __forceinline__ void con_evaluate_b(const DevProblem& P, const DevCon& con, int b, int ci, int n, int m, const double* x, const double* u, double* c) {
    if constexpr (INST) con_evaluate(con, con_data<true>(P, b, ci), n, m, x, u, c);
    else con_evaluate(con, P.cons[ci].a, n, m, x, u, c);
}
template <bool INST>
__device__ __forceinline__ void con_jacobian_b(const DevProblem& P, const DevCon& con, int b, int ci, int n, int m, const double* x, const double* u, double* jac) {
    if constexpr (INST) con_jacobian(con, con_data<true>(P, b, ci), n, m, x, u, jac);
    else con_jacobian(con, n, m, x, u, jac);
}

// H[(n+m)^2] col-major = d/dz (cz' lambda) = sum_i lambda_i Hess c_i(z), overwritten: the second-order constraint term the reference hands to
// solvers through grad-constraint_jacobians! (src/abstract_constraint.jl:267-280; `∇jacobian!` is zero for Goal / Bound, src/constraints.jl:70-73,
// :767-770, ForwardDiff for the rest).
__device__ inline void con_hess_vec(const DevCon& con, int n, int m, const double* x, const double* u, const double* lam, double* H) {
    const int w = n + m;
    for (int i = 0; i < w * w; i++) H[i] = 0.0;
    switch (con.kind) {
        case CON_CIRCLE: case CON_SPHERE: {
            const int nd = con.kind == CON_CIRCLE ? 2 : 3;
            for (int i = 0; i < con.p; i++) for (int d = 0; d < nd; d++) H[con.inds[d] * w + con.inds[d]] += -2 * lam[i];
            break;
        }
        case CON_NORM:
            if (con.sense != CONE_SECOND_ORDER) for (int i = 0; i < con.ninds; i++) H[con.inds[i] * w + con.inds[i]] += 2 * lam[0];
            break;
        case CON_COLLISION: {
            const int D = con.ninds / 2;
            for (int i = 0; i < D; i++) {
                const int a = con.inds[i], b = con.inds[D + i];
                H[a * w + a] += -2 * lam[0]; H[b * w + b] += -2 * lam[0]; H[b * w + a] += 2 * lam[0]; H[a * w + b] += 2 * lam[0];
            }
            break;
        }
        case CON_EXPR: {
            Hyper reg[TO_EXPR_LEN];
            for (int j = 0; j < w; j++)
                for (int k = j; k < w; k++) {
                    expr_run(con.prog, con.prog_len, con.pconst, n, x, u, true, j, k, reg);
                    double v = 0;
                    for (int i = 0; i < con.p; i++) v += lam[i] * reg[con.prog_len - con.p + i].d12;
                    H[k * w + j] = v; H[j * w + k] = v;
                }
            break;
        }
        case CON_QUATVEC: {
            double q[4], n2 = 0;
            for (int i = 0; i < 4; i++) { q[i] = x[con.inds[i]]; n2 = fma(q[i], q[i], n2); }
            const double n1 = sqrt(n2), i3 = 1.0 / (n2 * n1), i5 = i3 / n2;
            for (int j = 0; j < 4; j++)
                for (int k = 0; k < 4; k++) {
                    double v = 0;
                    for (int i = 0; i < 3; i++) {
                        const int a = i + 1;
                        v += lam[i] * (-((a == j ? q[k] : 0.0) + (a == k ? q[j] : 0.0) + (j == k ? q[a] : 0.0)) * i3 + 3 * q[a] * q[j] * q[k] * i5);
                    }
                    H[con.inds[k] * w + con.inds[j]] += v;
                }
            break;
        }
        default: break;   // Goal, Bound, Linear: linear in z
    }
}

// returns 0, or 1 for the reference's "Invalid second-order cone projection" error branch
__device__ inline int cone_projection(int cone, const double* x, int p, double* px) {
    switch (cone) {
        case CONE_IDENTITY: for (int i = 0; i < p; i++) px[i] = x[i]; return 0;
        case CONE_ZERO: for (int i = 0; i < p; i++) px[i] = 0; return 0;
        case CONE_NEGATIVE_ORTHANT: for (int i = 0; i < p; i++) px[i] = fmin(0.0, x[i]); return 0;
        case CONE_POSITIVE_ORTHANT: for (int i = 0; i < p; i++) px[i] = fmax(0.0, x[i]); return 0;
        case CONE_SECOND_ORDER: {
            double s = x[p - 1], a = 0;
            for (int i = 0; i < p - 1; i++) a = fma(x[i], x[i], a);
            a = sqrt(a);
            if (a <= -s) { for (int i = 0; i < p; i++) px[i] = 0; }
            else if (a <= s) { for (int i = 0; i < p; i++) px[i] = x[i]; }
            else if (a >= fabs(s)) {
                double sc = 0.5 * (1 + s / a);
                for (int i = 0; i < p - 1; i++) px[i] = sc * x[i];
                px[p - 1] = sc * a;
            } else return 1;
            return 0;
        }
    }
    return 1;
}

// J: p x p col-major, fully written
__device__ inline int cone_grad_projection(int cone, const double* x, int p, double* J) {
    for (int i = 0; i < p * p; i++) J[i] = 0;
    switch (cone) {
        case CONE_IDENTITY: for (int i = 0; i < p; i++) J[i * p + i] = 1; return 0;
        case CONE_ZERO: return 0;
        case CONE_NEGATIVE_ORTHANT: for (int i = 0; i < p; i++) J[i * p + i] = x[i] <= 0 ? 1 : 0; return 0;
        case CONE_POSITIVE_ORTHANT: for (int i = 0; i < p; i++) J[i * p + i] = x[i] >= 0 ? 1 : 0; return 0;
        case CONE_SECOND_ORDER: {
            const int n = p;
            double s = x[n - 1], a = 0;
            for (int i = 0; i < n - 1; i++) a = fma(x[i], x[i], a);
            a = sqrt(a);
            if (a <= -s) return 0;
            if (a <= s) { for (int i = 0; i < n; i++) J[i * n + i] = 1; return 0; }
            if (a >= fabs(s)) {
                double c = 0.5 * (1 + s / a);
                for (int i = 0; i < n - 1; i++)
                    for (int j = 0; j < n - 1; j++) {
                        double v = -0.5 * s / (a * a * a) * x[i] * x[j];
                        if (i == j) v += c;
                        J[j * n + i] = v;
                    }
                for (int i = 0; i < n - 1; i++) J[(n - 1) * n + i] = 0.5 * x[i] / a;
                for (int i = 0; i < n - 1; i++) J[i * n + (n - 1)] = ((-0.5 * s / (a * a)) + c / a) * x[i];
                J[(n - 1) * n + (n - 1)] = 0.5;
                return 0;
            }
            return 1;
        }
    }
    return 1;
}

__device__ inline int cone_hess_projection(int cone, const double* x, const double* b, int p, double* hess) {
    for (int i = 0; i < p * p; i++) hess[i] = 0;
    if (cone != CONE_SECOND_ORDER) return 0;
    const int n = p - 1;
    double s = x[n], bs = b[n], a = 0, vbv = 0;
    for (int i = 0; i < n; i++) { a = fma(x[i], x[i], a); vbv = fma(x[i], b[i], vbv); }
    a = sqrt(a);
    if (a <= -s) return 0;
    if (a <= s) return 0;
    if (a > fabs(s)) {
        for (int i = 0; i < n; i++) {
            double hi = 0;
            for (int j = 0; j < n; j++) {
                double Hij = -x[i] * x[j] / (a * a);
                if (i == j) Hij += 1;
                hi += Hij * b[j];
            }
            hess[n * p + i] = hi / (2 * a);
            hess[i * p + n] = hi / (2 * a);
            for (int j = 0; j <= i; j++) {
                double vij = x[i] * x[j];
                double H1 = hi * x[j] * (-s / (a * a * a));
                double H2 = vij * (2 * vbv) / (a * a * a * a) - x[i] * b[j] / (a * a);
                double H3 = -vij / (a * a);
                if (i == j) { H2 -= vbv / (a * a); H3 += 1; }
                H2 *= s / a;
                H3 *= bs / a;
                hess[j * p + i] = (H1 + H2 + H3) / 2;
                hess[i * p + j] = hess[j * p + i];
            }
        }
        hess[n * p + n] = 0;
        return 0;
    }
    return 1;
}

// AL penalty of one knot (conic form): sum_c (|Pi_{K*}(lambda - mu c)|^2 - |lambda|^2) / (2 mu); also the
// knot's constraint violation |c - Pi_K(c)|_inf.  k1 = 1-based knot, b = instance (its Goal values when INST).  x/u may be registers, local or global.
template <bool INST = false>
__device__ inline double al_knot_penalty(const DevProblem& P, int k1, const double* x, const double* u,
                                         const double* lam_b, double& viol, int b = 0) {
    double pen = 0;
    for (int ci = 0; ci < P.ncon; ci++) {
        const DevCon& con = P.cons[ci];
        if (k1 < con.first || k1 > con.last) continue;
        const double mu = P.mu[ci];
        const double* lam = lam_b + con.offset + (size_t)(k1 - con.first) * con.p;
        double c[TO_MAXPV], lbar[TO_MAXPV], lp[TO_MAXPV];
        con_evaluate_b<INST>(P, con, b, ci, P.n, P.m, x, u, c);
        for (int i = 0; i < con.p; i++) lbar[i] = lam[i] - mu * c[i];
        cone_projection(dualcone(con.sense), lbar, con.p, lp);
        double a = 0, l2 = 0;
        for (int i = 0; i < con.p; i++) { a = fma(lp[i], lp[i], a); l2 = fma(lam[i], lam[i], l2); }
        pen += (a - l2) / (2 * mu);
        cone_projection(con.sense, c, con.p, lp);
        for (int i = 0; i < con.p; i++) viol = fmax(viol, fabs(c[i] - lp[i]));
    }
    return pen;
}

// Cost expansion of one knot with the AL terms (Gauss-Newton):
//   grad += -cz' D' lp ; hess += mu cz' D'D cz,  D = grad Pi_{K*}(lambda - mu c), lp = Pi_{K*}(lambda - mu c)
// k0 = 0-based knot, b = instance (its linear cost terms and Goal values when INST).  grad[n+m], hess[(n+m)^2] col-major symmetric.
template <bool INST = false>
__device__ inline void al_knot_expansion(const DevProblem& P, int k0, const double* x, const double* u, const double* lam_b,
                                         double* grad, double* hess, int b = 0) {
    const int n = P.n, m = P.m, nm = n + m;
    const bool last = (k0 == P.N - 1);
    const int cid = P.cost_index[k0];
    const DevCost& cost = P.costs[cid];
    for (int i = 0; i < nm; i++) grad[i] = 0;
    cost_gradient(cost, inst_q<INST>(P, b, cid), inst_r<INST>(P, b, cid), n, m, x, u, last, grad);
    cost_hessian(cost, n, m, x, u, last, hess);
    const int lim = last ? n : nm;
    for (int ci = 0; ci < P.ncon; ci++) {
        const DevCon& con = P.cons[ci];
        if (k0 + 1 < con.first || k0 + 1 > con.last) continue;
        const int p = con.p;
        const double mu = P.mu[ci];
        const double* lam = lam_b + con.offset + (size_t)(k0 + 1 - con.first) * p;
        double c[TO_MAXPV], lbar[TO_MAXPV], lp[TO_MAXPV];
        con_evaluate_b<INST>(P, con, b, ci, n, m, x, u, c);
        if (con.diagonal) {   // Goal / Bound: +-1 selector rows (src/constraints.jl:62-68, :757-765) -- row by row, no dense products
            const bool eq = (con.kind == CON_GOAL);
            const int nrow = eq ? p : con.n_max + con.n_min;
            for (int r = 0; r < nrow; r++) {
                const int j = eq ? con.inds[r] : (r < con.n_max ? con.a_max[r] : con.a_min[r - con.n_max]);
                const double sgn = (eq || r < con.n_max) ? 1.0 : -1.0;
                const double lb = lam[r] - mu * c[r];
                if ((eq || lb <= 0.0) && j < lim) { grad[j] -= sgn * lb; hess[j * nm + j] += mu; }
            }
            continue;
        }
        double jac[TO_MAXP * TO_MAXNM], Dm[TO_MAXP * TO_MAXP], tmp[TO_MAXP * TO_MAXNM];
        con_jacobian_b<INST>(P, con, b, ci, n, m, x, u, jac);
        for (int i = 0; i < p; i++) lbar[i] = lam[i] - mu * c[i];
        const int dc = dualcone(con.sense);
        cone_projection(dc, lbar, p, lp);
        cone_grad_projection(dc, lbar, p, Dm);
        for (int j = 0; j < nm; j++)
            for (int i = 0; i < p; i++) {
                double s = 0;
                for (int r = 0; r < p; r++) s = fma(Dm[r * p + i], jac[j * p + r], s);
                tmp[j * p + i] = s;
            }
        for (int j = 0; j < lim; j++) {
            double g = 0;
            for (int i = 0; i < p; i++) g = fma(tmp[j * p + i], lp[i], g);
            grad[j] -= g;
            for (int j2 = 0; j2 < lim; j2++) {
                double hsum = 0;
                for (int i = 0; i < p; i++) hsum = fma(tmp[j * p + i], tmp[j2 * p + i], hsum);
                hess[j2 * nm + j] += mu * hsum;
            }
        }
    }
}

// ---- Lie-group error state (RobotDynamics LieState / Rotations.jl / Altro.jl, restated in oracle/oracle.hpp) -------------------
// grad-differential(q) = L(q) H, 4 x 3 col-major: columns (-x,w,z,-y), (-y,-z,w,x), (-z,y,-x,w)
__device__ __forceinline__ void quat_G(const double* q, double* G) {
    const double w = q[0], x = q[1], y = q[2], z = q[3];
    G[0] = -x; G[1] = w;  G[2] = z;   G[3] = -y;
    G[4] = -y; G[5] = -z; G[6] = w;   G[7] = x;
    G[8] = -z; G[9] = y;  G[10] = -x; G[11] = w;
}
// rotation part of RD.state_diff(xbar, x): inverse Cayley map of conj(q) (x) p
__device__ __forceinline__ void quat_diff(const double* q, const double* p, double* phi) {
    const double dw = q[0] * p[0] + q[1] * p[1] + q[2] * p[2] + q[3] * p[3];
    const double d1 = q[0] * p[1] - p[0] * q[1] - (q[2] * p[3] - q[3] * p[2]);
    const double d2 = q[0] * p[2] - p[0] * q[2] - (q[3] * p[1] - q[1] * p[3]);
    const double d3 = q[0] * p[3] - p[0] * q[3] - (q[1] * p[2] - q[2] * p[1]);
    phi[0] = d1 / dw; phi[1] = d2 / dw; phi[2] = d3 / dw;
}
// dx[ne] = state_diff(xbar, x); plain difference when the problem has no Lie-group state
__device__ __forceinline__ void state_diff(bool lie, int n, int qs, const double* xbar, const double* x, double* dx) {
    if (!lie) { for (int i = 0; i < n; i++) dx[i] = xbar[i] - x[i]; return; }
    for (int i = 0; i < qs; i++) dx[i] = xbar[i] - x[i];
    quat_diff(x + qs, xbar + qs, dx + qs);
    for (int i = qs + 4; i < n; i++) dx[i - 1] = xbar[i] - x[i];
}
