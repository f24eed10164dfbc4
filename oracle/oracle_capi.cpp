// oracle/oracle_capi.cpp -- TEST INFRASTRUCTURE ONLY.  Flat C interface (ctypes) over oracle.hpp.
// It accepts the same `to_spec` description as the product's C ABI (include/trajopt_b200.h is the interface
// description, not product code) so parity tests feed both sides identical inputs.  Entry points are
// prefixed `orc_`; nothing here is exported by, linked into, or reachable from libtrajopt_b200.so.
#include <omp.h>

#include <cstdio>
#include <cstring>
#include <string>

#include "../include/trajopt_b200.h"
#include "oracle.hpp"

using namespace oracle;

struct orc_handle {
    Problem P;
    std::string err;
};

static std::string g_err;

static int fail(orc_handle* h, int code, const std::string& msg) {
    if (h) h->err = msg; else g_err = msg;
    return code;
}

extern "C" {

const char* orc_last_error(const orc_handle* h) { return h ? h->err.c_str() : g_err.c_str(); }

int orc_create(const to_spec* s, orc_handle** out) {
    if (!s || !out) return fail(nullptr, TO_EINVAL, "null argument");
    *out = nullptr;
    if (s->model < 0 || s->model > MODEL_EXPR) return fail(nullptr, TO_EINVAL, "unknown model id");
    if (s->N < 2 || s->B < 1) return fail(nullptr, TO_EINVAL, "need N >= 2 and B >= 1");
    ModelParams mp = default_model(s->model, s->model == MODEL_DOUBLE_INTEGRATOR ? s->m : 1);
    if (mp.n != s->n) return fail(nullptr, TO_EDIM, "Objective state dimensions don't match model.");      // src/problem.jl:67
    if (mp.m != s->m) return fail(nullptr, TO_EDIM, "Objective control dimensions don't match model.");    // src/problem.jl:68
    if (s->params) for (int i = 0; i < s->nparams && i < 16; i++) mp.p[i] = s->params[i];
    auto* h = new orc_handle();
    Problem& P = h->P;
    P.model = mp; P.N = s->N; P.B = s->B; P.t0 = s->t0;
    if (s->model == MODEL_EXPR) {   // Problem(models::Vector, ...): RD.dims(models), src/dynamics.jl:15-31
        if (!s->dyn || s->ndyn < 1 || !s->dyn_index || !s->nx || !s->nu) { delete h; return fail(nullptr, TO_EINVAL, "recorded-program models: null dyn / dyn_index / nx / nu"); }
        for (int i = 0; i < s->ndyn; i++) {
            const to_dynamics_spec& d = s->dyn[i];
            DynProg dp; dp.n_in = d.n_in; dp.m_in = d.m_in; dp.n_out = d.n_out; dp.discrete = d.discrete != 0;
            if (!d.prog || d.prog_len < 1 || d.prog_len > TO_EXPR_MAXLEN || d.nconst < 0 || d.nconst > TO_EXPR_MAXCONST || (d.nconst > 0 && !d.consts) ||
                d.n_in < 1 || d.n_in > mp.n || d.m_in < 0 || d.m_in > mp.m || d.n_out < 1 || d.n_out > mp.n || d.n_out > d.prog_len) {
                delete h; return fail(nullptr, TO_EINVAL, "recorded-program model: bad program size or dimensions");
            }
            // the instruction checks of to_create: operands of earlier instructions only, constants and inputs in range
            for (int j = 0; j < d.prog_len; j++) {
                const int op = d.prog[3 * j], a = d.prog[3 * j + 1], b = d.prog[3 * j + 2];
                const bool bin = op >= TO_OP_ADD && op <= TO_OP_DIV;
                bool ok = op >= 0 && op <= TO_OP_RSUBC;
                if (op == TO_OP_CONST) ok = ok && a >= 0 && a < d.nconst;
                else if (op == TO_OP_X) ok = ok && a >= 0 && a < d.n_in;
                else if (op == TO_OP_U) ok = ok && a >= 0 && a < d.m_in;
                else { ok = ok && a >= 0 && a < j; if (bin) ok = ok && b >= 0 && b < j; if (op == TO_OP_POWC || op >= TO_OP_ADDC) ok = ok && b >= 0 && b < d.nconst; }
                if (!ok) { delete h; return fail(nullptr, TO_EINVAL, "recorded-program model: invalid instruction"); }
            }
            dp.prog.assign(d.prog, d.prog + 3 * d.prog_len); dp.consts.assign(d.consts, d.consts + d.nconst);
            P.dyn.push_back(dp);
        }
        for (int k = 0; k < s->N - 1; k++) {
            const int di = s->dyn_index[k];
            if (di < 0 || di >= s->ndyn) { delete h; return fail(nullptr, TO_EINVAL, "dyn_index out of range"); }
            const DynProg& d = P.dyn[di];
            if (d.n_in != s->nx[k] || d.m_in != s->nu[k]) {
                const std::string msg = "Model " + std::to_string(k + 1) + " has state / control dimensions (" + std::to_string(d.n_in) + ", " + std::to_string(d.m_in) +
                                        ") but knot " + std::to_string(k + 1) + " has (" + std::to_string(s->nx[k]) + ", " + std::to_string(s->nu[k]) + ").";
                delete h;
                return fail(nullptr, TO_EDIM, msg);
            }
            if (d.n_out != s->nx[k + 1]) {    // src/dynamics.jl:23-28
                const std::string msg = "Model mismatch at time step " + std::to_string(k + 1) + ". Model " + std::to_string(k + 1) + " has an output dimension of " +
                                        std::to_string(d.n_out) + " but model " + std::to_string(k + 2) + " has a state dimension of " + std::to_string(s->nx[k + 1]) + ".";
                delete h;     // (d lives in h: the message is built first)
                return fail(nullptr, TO_EDIM, msg);
            }
            P.dyn_index.push_back(di);
        }
    }
    P.dt.assign(s->dt, s->dt + (s->N - 1));
    const int n = mp.n, m = mp.m;
    for (int i = 0; i < s->ncost; i++) {
        const to_cost_spec& tc = s->costs[i];
        Cost c; c.n = n; c.m = m; c.diag = (tc.kind == TO_COST_DIAGONAL || tc.kind == TO_COST_DIAGONAL_QUAT); c.terminal = tc.terminal != 0; c.c = tc.c;
        if (tc.kind == TO_COST_EXPR) {
            if (!tc.prog || tc.prog_len < 1 || tc.prog_len > TO_EXPR_MAXLEN || tc.nconst < 0 || tc.nconst > TO_EXPR_MAXCONST || (tc.nconst > 0 && !tc.consts)) {
                delete h; return fail(nullptr, TO_EINVAL, "expression cost: bad program size");
            }
            c.expr = true; c.diag = false; c.zeroH = false;
            c.prog.assign(tc.prog, tc.prog + 3 * tc.prog_len); c.consts.assign(tc.consts, tc.consts + tc.nconst);
            for (int j = 0; j < tc.prog_len; j++) {
                const int op = c.prog[3 * j], a = c.prog[3 * j + 1], b = c.prog[3 * j + 2];
                const bool bin = op >= TO_OP_ADD && op <= TO_OP_DIV;
                bool ok = op >= 0 && op <= TO_OP_RSUBC;
                if (op == TO_OP_CONST) ok = ok && a >= 0 && a < tc.nconst;
                else if (op == TO_OP_X) ok = ok && a >= 0 && a < n;
                else if (op == TO_OP_U) ok = ok && a >= 0 && a < m;
                else { ok = ok && a >= 0 && a < j; if (bin) ok = ok && b >= 0 && b < j; if (op == TO_OP_POWC || op >= TO_OP_ADDC) ok = ok && b >= 0 && b < tc.nconst; }
                if (!ok) { delete h; return fail(nullptr, TO_EINVAL, "expression cost: invalid instruction"); }
            }
            c.Q.assign((size_t)n * n, 0.0); c.R.assign((size_t)m * m, 0.0); c.H.assign((size_t)m * n, 0.0); c.q.assign(n, 0.0); c.r.assign(m, 0.0);
            P.costs.push_back(c);
            continue;
        }
        if (tc.kind == TO_COST_DIAGONAL_QUAT) {
            if (!tc.q_ref) { delete h; return fail(nullptr, TO_EINVAL, "DiagonalQuatCost: null q_ref"); }
            c.quat = true; c.w = tc.w;
            for (int j = 0; j < 4; j++) {
                c.q_ref[j] = tc.q_ref[j]; c.q_ind[j] = tc.q_ind ? tc.q_ind[j] - 1 : 3 + j;
                if (c.q_ind[j] < 0 || c.q_ind[j] >= n) { delete h; return fail(nullptr, TO_EDIM, "DiagonalQuatCost: q_ind outside the state"); }
            }
        }
        c.Q.assign((size_t)n * n, 0.0); c.R.assign((size_t)m * m, 0.0); c.H.assign((size_t)m * n, 0.0);
        c.q.assign(tc.q, tc.q + n); c.r.assign(tc.r, tc.r + m);
        if (c.diag) {
            for (int j = 0; j < n; j++) c.Q[j * n + j] = tc.Q[j];
            for (int j = 0; j < m; j++) c.R[j * m + j] = tc.R[j];
        } else {
            std::memcpy(c.Q.data(), tc.Q, sizeof(double) * n * n);
            std::memcpy(c.R.data(), tc.R, sizeof(double) * m * m);
            if (tc.H) std::memcpy(c.H.data(), tc.H, sizeof(double) * m * n);
        }
        double hn = 0; for (double v : c.H) hn = std::max(hn, std::fabs(v));
        c.zeroH = c.diag || hn == 0.0;                                    // zeroH = norm(H,Inf) ~ 0, src/cost_functions.jl:445
        P.costs.push_back(c);
    }
    P.cost_index.assign(s->cost_index, s->cost_index + s->N);
    for (int k = 0; k < s->N; k++)
        if (P.cost_index[k] < 0 || P.cost_index[k] >= s->ncost) { delete h; return fail(nullptr, TO_EINVAL, "cost_index out of range"); }
    for (int i = 0; i < s->ncon; i++) {
        const to_constraint_spec& tc = s->cons[i];
        Constraint c; c.kind = tc.kind; c.first = tc.first; c.last = tc.last; c.n = n; c.m = m;
        if (tc.first < 1 || tc.last > s->N || tc.last < tc.first) { delete h; return fail(nullptr, TO_EINVAL, "constraint knot range outside 1:N"); }
        switch (tc.kind) {
            case TO_CON_GOAL:
                c.p = tc.ninds; c.sense = CONE_ZERO;
                for (int j = 0; j < tc.ninds; j++) { c.inds.push_back(tc.inds[j] - 1); c.a.push_back(tc.a[j]); }
                break;
            case TO_CON_BOUND:
                c.a.assign(tc.a, tc.a + n + m); c.b.assign(tc.b, tc.b + n + m);
                for (int j = 0; j < n + m; j++)
                    if (!(c.a[j] >= c.b[j])) { delete h; return fail(nullptr, TO_EINVAL, "Upper bounds must be greater than or equal to lower bounds"); }  // :712
                bound_finalize(c);
                if (tc.last == s->N && !c.a_max.empty() && (c.a_max.back() >= n || (!c.a_min.empty() && c.a_min.back() >= n))) { /* control bounds at the terminal knot act on u = 0 */ }
                break;
            case TO_CON_LINEAR: {
                c.p = tc.p; c.sense = tc.sense; c.lin_on_control = tc.flag;
                const int w = tc.flag ? m : n;
                c.a.assign(tc.a, tc.a + (size_t)tc.p * w); c.b.assign(tc.b, tc.b + tc.p);
                break;
            }
            case TO_CON_CIRCLE:
                c.p = tc.p; c.sense = CONE_NEGATIVE_ORTHANT;
                c.a.assign(tc.a, tc.a + tc.p); c.b.assign(tc.b, tc.b + tc.p); c.rad.assign(tc.rad, tc.rad + tc.p);
                c.xi = tc.ninds >= 1 ? tc.inds[0] - 1 : 0; c.yi = tc.ninds >= 2 ? tc.inds[1] - 1 : 1;
                break;
            case TO_CON_SPHERE:
                c.p = tc.p; c.sense = CONE_NEGATIVE_ORTHANT;
                c.a.assign(tc.a, tc.a + tc.p); c.b.assign(tc.b, tc.b + tc.p); c.c3.assign(tc.c, tc.c + tc.p); c.rad.assign(tc.rad, tc.rad + tc.p);
                c.xi = tc.ninds >= 1 ? tc.inds[0] - 1 : 0; c.yi = tc.ninds >= 2 ? tc.inds[1] - 1 : 1; c.zi = tc.ninds >= 3 ? tc.inds[2] - 1 : 2;
                break;
            case TO_CON_NORM:
                c.sense = tc.sense; c.val = tc.val;
                for (int j = 0; j < tc.ninds; j++) c.inds.push_back(tc.inds[j] - 1);
                c.p = (tc.sense == TO_CONE_SECOND_ORDER) ? tc.ninds + 1 : 1;
                break;
            case TO_CON_COLLISION:
                if (tc.ninds < 2 || (tc.ninds & 1)) { delete h; return fail(nullptr, TO_EDIM, "Position dimensions must be of equal length"); }
                c.sense = CONE_NEGATIVE_ORTHANT; c.val = tc.val; c.p = 1;
                for (int j = 0; j < tc.ninds; j++) c.inds.push_back(tc.inds[j] - 1);
                break;
            case TO_CON_EXPR: {
                const int L = tc.ninds / 3;
                if (!tc.inds || tc.ninds % 3 || L < 1 || L > TO_EXPR_MAXLEN || tc.p < 1 || tc.p > L || tc.p > MAXP || tc.flag < 0 || tc.flag > TO_EXPR_MAXCONST || (tc.flag > 0 && !tc.a)) {
                    delete h; return fail(nullptr, TO_EINVAL, "expression constraint: bad program size");
                }
                c.p = tc.p; c.sense = tc.sense;
                c.prog.assign(tc.inds, tc.inds + tc.ninds); c.consts.assign(tc.a, tc.a + tc.flag);
                for (int j = 0; j < L; j++) {
                    const int op = c.prog[3 * j], a = c.prog[3 * j + 1], b = c.prog[3 * j + 2];
                    const bool bin = op >= TO_OP_ADD && op <= TO_OP_DIV;
                    bool ok = op >= 0 && op <= TO_OP_RSUBC;
                    if (op == TO_OP_CONST) ok = ok && a >= 0 && a < tc.flag;
                    else if (op == TO_OP_X) ok = ok && a >= 0 && a < n;
                    else if (op == TO_OP_U) ok = ok && a >= 0 && a < m;
                    else { ok = ok && a >= 0 && a < j; if (bin) ok = ok && b >= 0 && b < j; if (op == TO_OP_POWC || op >= TO_OP_ADDC) ok = ok && b >= 0 && b < tc.flag; }
                    if (!ok) { delete h; return fail(nullptr, TO_EINVAL, "expression constraint: invalid instruction"); }
                }
                break;
            }
            case TO_CON_QUATVEC:
                if (!tc.a || n < 4) { delete h; return fail(nullptr, TO_EINVAL, "QuatVecEq: null qf"); }
                c.sense = CONE_ZERO; c.p = 3; c.a.assign(tc.a, tc.a + 4);
                for (int j = 0; j < 4; j++) {
                    c.inds.push_back((tc.inds && tc.ninds == 4) ? tc.inds[j] - 1 : 3 + j);
                    if (c.inds[j] < 0 || c.inds[j] >= n) { delete h; return fail(nullptr, TO_EDIM, "QuatVecEq: qind outside the state"); }
                }
                break;
            default: delete h; return fail(nullptr, TO_EINVAL, "unknown constraint kind");
        }
        P.cons.push_back(c);
    }
    if (s->error_state) {
        if (s->model != MODEL_QUADROTOR) { delete h; return fail(nullptr, TO_EINVAL, "error_state: the model has no Lie-group state (only the Quadrotor does)"); }
        P.lie = true; P.qs = 3;
    }
    P.finalize();
    *out = h;
    return TO_OK;
}

int orc_destroy(orc_handle* h) { delete h; return TO_OK; }

int orc_set_options(orc_handle* h, const to_options* o) {
    Options& q = h->P.opts;
    const bool reset_mu = q.penalty_initial != o->penalty_initial, reset_rho = q.bp_reg_initial != o->bp_reg_initial;   // as to_set_options
    q.bp_reg_increase_factor = o->bp_reg_increase_factor; q.bp_reg_max = o->bp_reg_max; q.bp_reg_min = o->bp_reg_min;
    q.bp_reg_initial = o->bp_reg_initial; q.bp_reg_fp = o->bp_reg_fp;
    q.line_search_lower_bound = o->line_search_lower_bound; q.line_search_upper_bound = o->line_search_upper_bound;
    q.iterations_linesearch = o->iterations_linesearch; q.max_state_value = o->max_state_value; q.max_control_value = o->max_control_value;
    q.penalty_initial = o->penalty_initial; q.penalty_scaling = o->penalty_scaling; q.penalty_max = o->penalty_max; q.dual_max = o->dual_max;
    if (reset_mu) for (auto& mu : h->P.mu) mu = q.penalty_initial;
    if (reset_rho) for (int b = 0; b < h->P.B; b++) { h->P.rho[b] = q.bp_reg_initial; h->P.drho[b] = 0; }
    h->P.J_valid = false;
    return TO_OK;
}
int orc_default_options(to_options* o) {
    Options q;
    o->bp_reg_increase_factor = q.bp_reg_increase_factor; o->bp_reg_max = q.bp_reg_max; o->bp_reg_min = q.bp_reg_min;
    o->bp_reg_initial = q.bp_reg_initial; o->bp_reg_fp = q.bp_reg_fp;
    o->line_search_lower_bound = q.line_search_lower_bound; o->line_search_upper_bound = q.line_search_upper_bound;
    o->iterations_linesearch = q.iterations_linesearch; o->backward_kernel = 0; o->max_state_value = q.max_state_value; o->max_control_value = q.max_control_value;
    o->penalty_initial = q.penalty_initial; o->penalty_scaling = q.penalty_scaling; o->penalty_max = q.penalty_max; o->dual_max = q.dual_max;
    return TO_OK;
}
// integrator of the discretised dynamics: 4 = RK4 (default), 3 = RK3 (oracle only; pins the oracle to the recorded notebook outputs)
int orc_set_integrator(orc_handle* h, int order) {
    if (order != 3 && order != 4) return TO_EINVAL;
    h->P.model.integrator = order; h->P.J_valid = false;
    return TO_OK;
}
// algebra of the backward pass: 0 = Cholesky solve (default), 1 = the block-inverse form of csrc/riccati_frag.cu (oracle.hpp Options)
int orc_set_backward_variant(orc_handle* h, int v) {
    if (v != 0 && v != 1) return TO_EINVAL;
    h->P.opts.backward_variant = v;
    return TO_OK;
}
// test instrument (oracle.hpp Options::gain_noise): relative perturbation of the gains after every backward pass
int orc_set_gain_noise(orc_handle* h, double rel) { h->P.opts.gain_noise = rel; return TO_OK; }
int orc_get_backward_variant(orc_handle* h) { return h->P.opts.backward_variant; }
int orc_set_threads(int nthreads) { omp_set_num_threads(nthreads > 0 ? nthreads : omp_get_num_procs()); return omp_get_max_threads(); }

int orc_set_initial_state(orc_handle* h, const double* x0) { std::memcpy(h->P.x0.data(), x0, sizeof(double) * h->P.x0.size()); h->P.J_valid = false; return TO_OK; }
int orc_set_controls(orc_handle* h, const double* U) { std::memcpy(h->P.U.data(), U, sizeof(double) * h->P.U.size()); h->P.J_valid = false; return TO_OK; }
int orc_set_states(orc_handle* h, const double* X) { std::memcpy(h->P.X.data(), X, sizeof(double) * h->P.X.size()); h->P.J_valid = false; return TO_OK; }
int orc_get_states(orc_handle* h, double* X) { std::memcpy(X, h->P.X.data(), sizeof(double) * h->P.X.size()); return TO_OK; }
int orc_get_controls(orc_handle* h, double* U) { std::memcpy(U, h->P.U.data(), sizeof(double) * h->P.U.size()); return TO_OK; }

// set_goal_state!  src/problem.jl:294-310 (+ set_LQR_goal! src/cost_functions.jl:245-248: only q changes, not c)
int orc_set_goal_state(orc_handle* h, const double* xf, int objective, int constraint) {
    Problem& P = h->P; const int n = P.n;
    if (objective)
        for (auto& c : P.costs)
            for (int i = 0; i < n; i++) { double t = 0; for (int j = 0; j < n; j++) t += c.Q[j * n + i] * xf[j]; c.q[i] = -t; }
    if (constraint)
        for (auto& c : P.cons)
            if (c.kind == CON_GOAL) for (int i = 0; i < c.p; i++) c.a[i] = xf[c.inds[i]];
    P.J_valid = false;
    return TO_OK;
}


// update_trajectory!(obj, Z, start)  src/objective.jl:207-212 with set_LQR_goal! src/cost_functions.jl:245-254
int orc_update_trajectory(orc_handle* h, const double* Xref, const double* Uref, int32_t nref, int32_t start) {
    Problem& P = h->P; const int n = P.n, m = P.m, N = P.N;
    if (start < 1 || start - 1 + N > nref) return fail(h, TO_EDIM, "update_trajectory!: the reference is shorter than start + N - 1");
    for (int i = 0; i < N; i++) {
        Cost& c = P.costs[P.cost_index[i]];
        const double* xf = Xref + (size_t)(start - 1 + i) * n;
        const double* uf = Uref + (size_t)(start - 1 + i) * m;
        for (int a = 0; a < n; a++) { double t = 0; for (int j = 0; j < n; j++) t += c.Q[j * n + a] * xf[j]; c.q[a] = -t; }
        for (int a = 0; a < m; a++) { double t = 0; for (int j = 0; j < m; j++) t += c.R[j * m + a] * uf[j]; c.r[a] = -t; }
    }
    P.J_valid = false;
    return TO_OK;
}
// receding-horizon warm start (see include/trajopt_b200.h, to_shift_trajectory): plain loops over instances and knots
int orc_shift_trajectory(orc_handle* h, int32_t steps) {
    Problem& P = h->P; const int n = P.n, m = P.m, N = P.N;
    if (steps < 0) return TO_EINVAL;
    if (steps == 0) return TO_OK;
    if (steps > N - 1) steps = N - 1;
    for (int b = 0; b < P.B; b++) {
        double* X = &P.X[(size_t)b * N * n]; double* U = &P.U[(size_t)b * (N - 1) * m];
        for (int i = 0; i < n; i++) P.x0[(size_t)b * n + i] = X[(size_t)steps * n + i];
        for (int k = 0; k < N; k++) { const int s = std::min(k + steps, N - 1); for (int i = 0; i < n; i++) X[(size_t)k * n + i] = X[(size_t)s * n + i]; }
        for (int k = 0; k < N - 1; k++) { const int s = std::min(k + steps, N - 2); for (int i = 0; i < m; i++) U[(size_t)k * m + i] = U[(size_t)s * m + i]; }
        double* lam = &P.lambda[(size_t)b * P.lambda_len];
        for (size_t ci = 0; ci < P.cons.size(); ci++) {
            const Constraint& c = P.cons[ci];
            const int nk = c.last - c.first + 1;
            for (int k = 0; k + steps < nk; k++) for (int r = 0; r < c.p; r++) lam[P.con_offset[ci] + k * c.p + r] = lam[P.con_offset[ci] + (k + steps) * c.p + r];
        }
    }
    for (int k = 0; k < steps; k++) P.t0 += P.dt[k];
    P.J_valid = false;
    return TO_OK;
}

int orc_get_times(orc_handle* h, double* t) {
    t[0] = h->P.t0;
    for (int k = 1; k < h->P.N; k++) t[k] = t[k - 1] + h->P.dt[k - 1];
    return TO_OK;
}
int orc_set_initial_time(orc_handle* h, double t0, double* tf_out) {
    h->P.t0 = t0;
    if (tf_out) { double t = t0; for (double d : h->P.dt) t += d; *tf_out = t; }
    return TO_OK;
}
int orc_synchronize(orc_handle*) { return TO_OK; }

int orc_rollout(orc_handle* h) {
    Problem& P = h->P;
#pragma omp parallel for schedule(static)
    for (int b = 0; b < P.B; b++) rollout(P, b);
    P.J_valid = false;
    return TO_OK;
}
int orc_expand(orc_handle* h) {
    Problem& P = h->P;
#pragma omp parallel for schedule(static)
    for (int b = 0; b < P.B; b++) expand_dynamics(P, b);
    return TO_OK;
}
int orc_get_dynamics_jacobians(orc_handle* h, double* AB) { std::memcpy(AB, h->P.AB.data(), sizeof(double) * h->P.AB.size()); return TO_OK; }

int orc_cost(orc_handle* h, double* J) {
    Problem& P = h->P;
#pragma omp parallel for schedule(static)
    for (int b = 0; b < P.B; b++) J[b] = cost_total(P, P.Xb(b), P.Ub(b));
    return TO_OK;
}
int orc_cost_knots(orc_handle* h, double* Jk) {
    Problem& P = h->P;
#pragma omp parallel for schedule(static)
    for (int b = 0; b < P.B; b++) cost_knots(P, P.Xb(b), P.Ub(b), &Jk[(size_t)b * P.N]);
    return TO_OK;
}
int orc_cost_gradient(orc_handle* h, double* grad) {
    Problem& P = h->P; const int nm = P.n + P.m;
#pragma omp parallel for schedule(static)
    for (int b = 0; b < P.B; b++)
        for (int k = 0; k < P.N; k++) {
            double* g = &grad[((size_t)b * P.N + k) * nm];
            std::fill(g, g + nm, 0.0);
            const bool last = k == P.N - 1;
            cost_gradient(P.costs[P.cost_index[k]], &P.Xb(b)[k * P.n], last ? ZERO_U : &P.Ub(b)[k * P.m], last, g);
        }
    return TO_OK;
}
int orc_cost_hessian(orc_handle* h, double* hess) {
    Problem& P = h->P; const int nm = P.n + P.m;
#pragma omp parallel for schedule(static)
    for (int b = 0; b < P.B; b++)
        for (int k = 0; k < P.N; k++) {
            double* H = &hess[((size_t)b * P.N + k) * nm * nm];
            std::fill(H, H + nm * nm, 0.0);
            const bool last = k == P.N - 1;
            cost_hessian(P.costs[P.cost_index[k]], &P.Xb(b)[k * P.n], last ? ZERO_U : &P.Ub(b)[k * P.m], last, H, true);
        }
    return TO_OK;
}
int orc_eval_constraints(orc_handle* h, int con, double* vals) {
    Problem& P = h->P;
    if (con < 0 || con >= (int)P.cons.size()) return fail(h, TO_EINVAL, "constraint index out of range");
    const size_t len = (size_t)P.cons[con].nknots() * P.cons[con].p;
#pragma omp parallel for schedule(static)
    for (int b = 0; b < P.B; b++) evaluate_constraints(P, con, P.Xb(b), P.Ub(b), &vals[b * len]);
    return TO_OK;
}
int orc_constraint_jacobians(orc_handle* h, int con, double* jac) {
    Problem& P = h->P;
    if (con < 0 || con >= (int)P.cons.size()) return fail(h, TO_EINVAL, "constraint index out of range");
    const size_t len = (size_t)P.cons[con].nknots() * P.cons[con].p * (P.n + P.m);
#pragma omp parallel for schedule(static)
    for (int b = 0; b < P.B; b++) constraint_jacobians(P, con, P.Xb(b), P.Ub(b), &jac[b * len]);
    return TO_OK;
}
// grad-constraint_jacobians! (src/abstract_constraint.jl:267-280): H[B][knots][(n+m)^2]; lambda [B][knots][p] or NULL = the current multipliers
int orc_constraint_hessians(orc_handle* h, int con, const double* lambda, double* H) {
    Problem& P = h->P;
    if (con < 0 || con >= (int)P.cons.size()) return fail(h, TO_EINVAL, "constraint index out of range");
    const Constraint& c = P.cons[con];
    const int w = P.n + P.m;
    const size_t len = (size_t)c.nknots();
#pragma omp parallel for schedule(static)
    for (int b = 0; b < P.B; b++)
        for (int k = c.first; k <= c.last; k++) {
            const double* u = (k == P.N) ? ZERO_U : &P.Ub(b)[(k - 1) * P.m];
            const double* lam = lambda ? &lambda[((size_t)b * len + (k - c.first)) * c.p] : &P.lamb(b)[P.con_offset[con] + (size_t)(k - c.first) * c.p];
            con_hess_vec(c, &P.Xb(b)[(k - 1) * P.n], u, lam, &H[((size_t)b * len + (k - c.first)) * w * w]);
        }
    return TO_OK;
}
int orc_constraint_info(orc_handle* h, int con, int32_t* p, int32_t* sense, int32_t* first, int32_t* last) {
    Problem& P = h->P;
    if (con < 0 || con >= (int)P.cons.size()) return fail(h, TO_EINVAL, "constraint index out of range");
    *p = P.cons[con].p; *sense = P.cons[con].sense; *first = P.cons[con].first; *last = P.cons[con].last;
    return TO_OK;
}
int orc_max_violation(orc_handle* h, double* v) {
    Problem& P = h->P;
#pragma omp parallel for schedule(static)
    for (int b = 0; b < P.B; b++) v[b] = max_violation(P, P.Xb(b), P.Ub(b));
    return TO_OK;
}
int orc_merit(orc_handle* h, double* J) {
    Problem& P = h->P;
#pragma omp parallel for schedule(static)
    for (int b = 0; b < P.B; b++) J[b] = merit(P, P.Xb(b), P.Ub(b), P.lamb(b));
    return TO_OK;
}
int orc_al_expansion(orc_handle* h, double* grad, double* hess) {
    Problem& P = h->P; const int nm = P.n + P.m;
#pragma omp parallel for schedule(static)
    for (int b = 0; b < P.B; b++)
        for (int k = 0; k < P.N; k++)
            cost_expansion(P, P.Xb(b), P.Ub(b), P.lamb(b), k, &grad[((size_t)b * P.N + k) * nm], &hess[((size_t)b * P.N + k) * nm * nm]);
    return TO_OK;
}
int orc_projection(int cone, int p, int count, const double* x, double* px) {
    int rc = 0;
    for (int i = 0; i < count; i++) if (projection(cone, &x[(size_t)i * p], p, &px[(size_t)i * p])) rc = TO_ECONE;
    return rc;
}
int orc_grad_projection(int cone, int p, int count, const double* x, double* J) {
    int rc = 0;
    for (int i = 0; i < count; i++) if (grad_projection(cone, &x[(size_t)i * p], p, &J[(size_t)i * p * p])) rc = TO_ECONE;
    return rc;
}
int orc_hess_projection(int cone, int p, int count, const double* x, const double* b, double* H) {
    int rc = 0;
    for (int i = 0; i < count; i++) if (hess_projection(cone, &x[(size_t)i * p], &b[(size_t)i * p], p, &H[(size_t)i * p * p])) rc = TO_ECONE;
    return rc;
}

int orc_backward(orc_handle* h, int32_t* status) {
    Problem& P = h->P;
    P.opts.noise_epoch++;
#pragma omp parallel for schedule(dynamic, 4)
    for (int b = 0; b < P.B; b++) backward_pass(P, b);
    if (status) for (int b = 0; b < P.B; b++) status[b] = P.bp_status[b];
    return TO_OK;
}
int orc_forward(orc_handle* h, double* J, double* alpha) {
    Problem& P = h->P;
    ensure_merit(P);
#pragma omp parallel for schedule(dynamic, 4)
    for (int b = 0; b < P.B; b++) forward_pass(P, b);
    if (J) std::memcpy(J, P.J.data(), sizeof(double) * P.B);
    if (alpha) std::memcpy(alpha, P.alpha.data(), sizeof(double) * P.B);
    return TO_OK;
}
int orc_ilqr_step(orc_handle* h, int iters) { ilqr_step(h->P, iters); return TO_OK; }
int orc_al_update(orc_handle* h) { al_update(h->P); return TO_OK; }
int orc_get_gains(orc_handle* h, double* K, double* d) {
    if (K) std::memcpy(K, h->P.K.data(), sizeof(double) * h->P.K.size());
    if (d) std::memcpy(d, h->P.d.data(), sizeof(double) * h->P.d.size());
    return TO_OK;
}
int orc_get_multipliers(orc_handle* h, int con, double* lam) {
    Problem& P = h->P; const size_t len = (size_t)P.cons[con].nknots() * P.cons[con].p;
    for (int b = 0; b < P.B; b++) std::memcpy(&lam[b * len], P.lamb(b) + P.con_offset[con], sizeof(double) * len);
    return TO_OK;
}
int orc_set_multipliers(orc_handle* h, int con, const double* lam) {
    Problem& P = h->P; const size_t len = (size_t)P.cons[con].nknots() * P.cons[con].p;
    for (int b = 0; b < P.B; b++) std::memcpy(P.lamb(b) + P.con_offset[con], &lam[b * len], sizeof(double) * len);
    P.J_valid = false;
    return TO_OK;
}
int orc_get_penalty(orc_handle* h, int con, double* mu) { *mu = h->P.mu[con]; return TO_OK; }
int orc_set_penalty(orc_handle* h, int con, double mu) { h->P.mu[con] = mu; h->P.J_valid = false; return TO_OK; }
int orc_get_solver_state(orc_handle* h, double* rho, double* dV, double* alpha, int32_t* ls_iters, int32_t* bp_status) {
    Problem& P = h->P;
    if (rho) std::memcpy(rho, P.rho.data(), sizeof(double) * P.B);
    if (dV) std::memcpy(dV, P.dV.data(), sizeof(double) * 2 * P.B);
    if (alpha) std::memcpy(alpha, P.alpha.data(), sizeof(double) * P.B);
    if (ls_iters) for (int b = 0; b < P.B; b++) ls_iters[b] = P.ls_iters[b];
    if (bp_status) for (int b = 0; b < P.B; b++) bp_status[b] = P.bp_status[b];
    return TO_OK;
}

// single-point model evaluation, for KATs (hover, RK4 vs scipy, Jacobian vs finite differences)
int orc_dynamics(int model, int dim, const double* params, int nparams, const double* x, const double* u, double* xdot) {
    ModelParams mp = default_model(model, dim);
    if (params) for (int i = 0; i < nparams && i < 16; i++) mp.p[i] = params[i];
    dynamics<double>(mp, x, u, xdot);
    return TO_OK;
}
int orc_discrete_dynamics(int model, int dim, const double* params, int nparams, const double* x, const double* u, double h, double* xn) {
    ModelParams mp = default_model(model, dim);
    if (params) for (int i = 0; i < nparams && i < 16; i++) mp.p[i] = params[i];
    rk4_step<double>(mp, x, u, h, xn);
    return TO_OK;
}
int orc_discrete_jacobian(int model, int dim, const double* params, int nparams, const double* x, const double* u, double h, double* AB) {
    ModelParams mp = default_model(model, dim);
    if (params) for (int i = 0; i < nparams && i < 16; i++) mp.p[i] = params[i];
    dynamics_jacobian(mp, x, u, h, AB);
    return TO_OK;
}

// ---- Lie-group error state -----------------------------------------------------------------------------------
int orc_error_state_dim(orc_handle* h, int32_t* ne) { *ne = h->P.ne; return TO_OK; }
int orc_state_diff(orc_handle* h, const double* Xbar, double* dx) {
    Problem& P = h->P;
    for (int b = 0; b < P.B; b++)
        for (int k = 0; k < P.N; k++) state_diff(P, &Xbar[((size_t)b * P.N + k) * P.n], &P.Xb(b)[k * P.n], &dx[((size_t)b * P.N + k) * P.ne]);
    return TO_OK;
}
int orc_get_error_dynamics(orc_handle* h, double* ABe) {
    Problem& P = h->P;
    if (P.lie) std::memcpy(ABe, P.ABe.data(), sizeof(double) * P.ABe.size());
    else std::memcpy(ABe, P.AB.data(), sizeof(double) * P.AB.size());
    return TO_OK;
}
int orc_error_expansion(orc_handle* h, double* grad, double* hess) {
    Problem& P = h->P; const int nm = P.n + P.m, nme = P.ne + P.m;
    if (!P.lie) return orc_al_expansion(h, grad, hess);
#pragma omp parallel for schedule(static)
    for (int b = 0; b < P.B; b++) {
        std::vector<double> g(nm), H((size_t)nm * nm);
        for (int k = 0; k < P.N; k++) {
            cost_expansion(P, P.Xb(b), P.Ub(b), P.lamb(b), k, g.data(), H.data());
            error_expansion(P, &P.Xb(b)[k * P.n], g.data(), H.data(), &grad[((size_t)b * P.N + k) * nme], &hess[((size_t)b * P.N + k) * nme * nme]);
        }
    }
    return TO_OK;
}

}  // extern "C"
