// capi.cu -- the C ABI (include/trajopt_b200.h): opaque handle, device memory, descriptor tables, and the
// sequencing of the hot-path kernels.  No compute happens on the host: every compute entry point launches the
// sm_90a kernels of rollout.cu / sweep.cu / riccati.cu / forward.cu on the handle's stream.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/trajopt_b200.h"
#include "frag_layout.cuh"
#include "kernels.h"

namespace {

std::string g_create_error;

struct Scratch {
    void* ptr = nullptr;
    size_t bytes = 0;
};

}  // namespace

struct to_handle {
    DevProblem P{};
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    cudaStream_t stream2 = nullptr;     // high-priority side stream: late line-search trials overlap the next expansion
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr, ev_merit = nullptr, ev_cons = nullptr;
    bool overlap = true;                // TO_NO_OVERLAP=1: keep every kernel on the main stream (profiling under ncu, A/B timing)
    bool side_pending = false;          // stream2 still holds the late line-search trials of the last iteration (ev_join follows them)
    // to_solve: per-instance solve state on the device; the ACTIVE count of an iteration comes back through pinned memory + an event
    SolveDev solve{};
    int* pin_count = nullptr;           // [2] (pinned)
    cudaEvent_t ev_count[2] = {nullptr, nullptr};
    std::string err;
    std::vector<void*> allocs;
    std::vector<DevCost> h_costs;
    std::vector<DevCon> h_cons;
    std::vector<double> h_mu, h_dt;
    std::vector<int> h_cost_index;
    std::vector<DevDyn> h_dyn;    // TO_MODEL_EXPR
    std::vector<int> h_dyn_index;
    DevCost* d_costs = nullptr;
    DevCon* d_cons = nullptr;
    double* d_mu = nullptr;
    double* d_stageX = nullptr;   // dense [B][N][n] staging for get/set
    double* d_stageU = nullptr;
    double* d_viol = nullptr;     // [B]
    double* d_merit2 = nullptr;   // {sum J, max viol}
    int* d_work = nullptr;
    ExpTab* d_exptab = nullptr;   // (frag) AL rows per z entry, rebuilt with the constraint tables / penalties
    // host copies of the per-instance tables, empty until the first per-instance call (commit_rows); each goes to the device whole after every change
    std::vector<double> h_qr;        // linear cost terms (DevProblem::qr), [B][ncost][n+m]
    std::vector<double> h_mparams;   // model parameters (DevProblem::mparams), [B][TO_NPARAM]
    std::vector<double> h_cdata;     // constraint data and Goal values (DevProblem::cdata), [B][ncdata]
    std::vector<double> stage;       // the rows a setter is building, committed by commit_rows (kept to reuse its allocation)
    int* d_fragerr = nullptr;     // sticky error word of that kernel (queue overflow / spin limit), read by to_synchronize
    double* d_fragpool = nullptr; // gains of its speculative regularisation candidates
    int* d_fragq = nullptr;       // work queue of the register-resident Riccati kernel (riccati_frag.cu)
    int* d_err = nullptr;
    Scratch scratch;
    double t0 = 0;
    bool J_valid = false, expanded = false, backward_done = false;
    bool rec_costexp = false;     // (record path) a cost + AL expansion has been written into REC[192, 240) (to_get_expansion_records)
    int64_t launches = 0;
    // phase timing
    bool timing = false;
    struct Ev { cudaEvent_t a, b; int phase; };
    std::vector<Ev> pending;
    std::vector<cudaEvent_t> pool;
    double phase_ms[TO_PHASE_COUNT] = {0};
    int64_t phase_launches[TO_PHASE_COUNT] = {0};
};

namespace {

int fail(to_handle* h, int code, const std::string& msg) {
    if (h) h->err = msg; else g_create_error = msg;
    return code;
}
int cuda_fail(to_handle* h, cudaError_t e, const char* what) {
    return fail(h, e == cudaErrorMemoryAllocation ? TO_ENOMEM : TO_ECUDA, std::string(what) + ": " + cudaGetErrorString(e));
}
#define CU(h, expr)                                                   \
    do {                                                              \
        cudaError_t e__ = (expr);                                     \
        if (e__ != cudaSuccess) return cuda_fail(h, e__, #expr);      \
    } while (0)

template <class T>
int dalloc(to_handle* h, T** p, size_t count) {
    void* q = nullptr;
    cudaError_t e = cudaMalloc(&q, std::max<size_t>(count, 1) * sizeof(T));
    if (e != cudaSuccess) return cuda_fail(h, e, "cudaMalloc");
    h->allocs.push_back(q);
    *p = static_cast<T*>(q);
    return TO_OK;
}

int ensure_scratch(to_handle* h, size_t bytes) {
    if (h->scratch.bytes >= bytes) return TO_OK;
    if (h->scratch.ptr) { cudaStreamSynchronize(h->stream); cudaFree(h->scratch.ptr); h->scratch.ptr = nullptr; h->scratch.bytes = 0; }
    cudaError_t e = cudaMalloc(&h->scratch.ptr, bytes);
    if (e != cudaSuccess) return cuda_fail(h, e, "cudaMalloc(scratch)");
    h->scratch.bytes = bytes;
    return TO_OK;
}

// ExpTab (common.cuh): the Goal / Bound rows acting on each z entry, for the record expansion of the dynamics expansion kernel
int upload_exptab(to_handle* h) {
    if (!h->d_exptab) return TO_OK;
    ExpTab t;
    std::memset(&t, 0, sizeof(t));
    const int nm = h->P.n + h->P.m, n = h->P.n;
    for (int i = 0; i < nm; i++) {
        int nterm = 0;
        for (int k = 0; k < TO_EXP_MAXT; k++) { t.nms[k][i] = -1.0; t.pkx[k][i] = 4095u; t.inst[k][i] = -1; }      // empty knot range
        for (size_t ci = 0; ci < h->h_cons.size(); ci++) {
            const DevCon& con = h->h_cons[ci];
            if (!con.diagonal) continue;
            const double mu = h->h_mu[ci];
            for (int side = 0; side < 2; side++) {
                int row = -1; double sign = 1.0, bound = 0.0; bool eq = false;
                if (con.kind == CON_GOAL) { if (side == 0 && i < n) { row = con.row_max[i]; if (row >= 0) bound = con.a[row]; eq = true; } }
                else if (side == 0) { row = con.row_max[i]; bound = con.a[i]; }
                else { row = con.row_min[i]; bound = con.b[i]; sign = -1.0; }
                if (row < 0) continue;
                if (nterm < TO_EXP_MAXT && con.last >= con.first && con.first < 4095 && con.p < 128) {
                    t.nms[nterm][i] = -mu * sign; t.bound[nterm][i] = bound;
                    t.pkx[nterm][i] = (unsigned)con.first | ((unsigned)(con.last - con.first) << 12) | ((unsigned)con.p << 24) | (eq ? 0x80000000u : 0u);
                    t.pky[nterm][i] = (unsigned)(con.offset + row - con.first * con.p);
                    t.inst[nterm][i] = con.cdoff + (eq ? row : (side ? nm : 0) + i);
                }
                nterm++;
            }
        }
    }
    CU(h, cudaMemcpyAsync(h->d_exptab, &t, sizeof(t), cudaMemcpyHostToDevice, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));   // `t` goes out of scope
    return TO_OK;
}

// set_LQR_goal! (src/cost_functions.jl:245-254): the linear term -M xf of a goal xf (q = -Q xf, r = -R uf), M dim x dim column-major.
// The one place where a goal becomes a linear term: the shared setters and the per-instance ones produce the same bits for the same xf.
void lqr_linear_term(const double* M, int dim, const double* xf, double* out) {
    for (int i = 0; i < dim; i++) { double t = 0; for (int j = 0; j < dim; j++) t += M[j * dim + i] * xf[j]; out[i] = -t; }
}

// Commits the complete rows staged in h->stage as the per-instance table whose host copy is `host` and whose device pointer is `dev`
// (DevProblem::qr / mparams / cdata): the device buffer is allocated on first use, the rows are copied, and only once the device holds them
// do they become the host copy and is the pointer published.  A failed call leaves the table, or its absence, as it was: no kernel reads
// rows the device lacks and no getter reports them.
int commit_rows(to_handle* h, std::vector<double>& host, const double*& dev) {
    std::vector<double>& rows = h->stage;
    double* d = const_cast<double*>(dev);
    if (!d) { int rc = dalloc(h, &d, rows.size()); if (rc) return rc; }
    CU(h, cudaMemcpyAsync(d, rows.data(), sizeof(double) * rows.size(), cudaMemcpyHostToDevice, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));   // the staged rows are the source of the copy
    host.swap(rows);
    dev = d;
    return TO_OK;
}

int upload_tables(to_handle* h) {
    CU(h, cudaMemcpyAsync(h->d_costs, h->h_costs.data(), sizeof(DevCost) * h->h_costs.size(), cudaMemcpyHostToDevice, h->stream));
    if (!h->h_cons.empty()) {
        CU(h, cudaMemcpyAsync(h->d_cons, h->h_cons.data(), sizeof(DevCon) * h->h_cons.size(), cudaMemcpyHostToDevice, h->stream));
        CU(h, cudaMemcpyAsync(h->d_mu, h->h_mu.data(), sizeof(double) * h->h_mu.size(), cudaMemcpyHostToDevice, h->stream));
    }
    CU(h, cudaStreamSynchronize(h->stream));   // the host vectors may change right after
    return upload_exptab(h);
}


// phase timing helpers
struct PhaseScope {
    to_handle* h; int phase; cudaEvent_t a = nullptr, b = nullptr;
    cudaStream_t st;
    PhaseScope(to_handle* h_, int phase_, cudaStream_t st_ = nullptr) : h(h_), phase(phase_), st(st_ ? st_ : h_->stream) {
        if (!h->timing) return;
        auto get = [&]() { cudaEvent_t e; if (!h->pool.empty()) { e = h->pool.back(); h->pool.pop_back(); } else cudaEventCreate(&e); return e; };
        a = get(); b = get();
        cudaEventRecord(a, st);
    }
    ~PhaseScope() {
        if (!h->timing) return;
        cudaEventRecord(b, st);
        h->pending.push_back({a, b, phase});
    }
};

void set_default_options(DevOptions& o) {
    o.bp_reg_increase_factor = 1.6; o.bp_reg_max = 1e8; o.bp_reg_min = 1e-8; o.bp_reg_initial = 0.0; o.bp_reg_fp = 10.0;
    o.ls_lower = 1e-8; o.ls_upper = 10.0; o.ls_iters = 10; o.pad = 0;
    o.max_state_value = 1e8; o.max_control_value = 1e8;
    o.penalty_initial = 1.0; o.penalty_scaling = 10.0; o.penalty_max = 1e8; o.dual_max = 1e8;
}

void model_defaults(int model, int m, int& n_out, int& m_out, double* p) {
    for (int i = 0; i < 16; i++) p[i] = 0;
    switch (model) {
        case TO_MODEL_DOUBLE_INTEGRATOR: n_out = 2 * m; m_out = m; p[0] = 1.0; break;   // p[1] = 1/mass is filled by to_create
        case TO_MODEL_CARTPOLE: n_out = 4; m_out = 1; p[0] = 1.0; p[1] = 0.2; p[2] = 0.5; p[3] = 9.81; break;
        case TO_MODEL_QUADROTOR:
            n_out = 13; m_out = 4; p[0] = 0.5; p[1] = 0.0023; p[2] = 0.0023; p[3] = 0.004; p[4] = 0; p[5] = 0; p[6] = -9.81;
            p[7] = 0.1750; p[8] = 1.0; p[9] = 0.0245; break;
        case TO_MODEL_ACROBOT:
            n_out = 4; m_out = 1; p[0] = 1; p[1] = 1; p[2] = 1; p[3] = 1; p[4] = 1.0 / 12; p[5] = 1.0 / 12; p[6] = 1.0; p[7] = 9.81; break;
        case TO_MODEL_EXPR: n_out = 4; m_out = 2; break;       // recorded programs on the padded dimensions the kernels are instantiated for
        default: n_out = -1; m_out = -1;
    }
}

// The entries of a parameter vector the caller gives (to_spec.params, to_set_model_params), and the names of those the device dynamics
// divide by or build a determinant from (models.cuh): they must be positive.
int model_nparams(int model) {
    switch (model) {
        case TO_MODEL_DOUBLE_INTEGRATOR: return 1;
        case TO_MODEL_CARTPOLE: return 4;
        case TO_MODEL_QUADROTOR: return 10;
        case TO_MODEL_ACROBOT: return 8;
        default: return 0;
    }
}
const char* positive_param_name(int model, int i) {
    static const char* di[] = {"mass"};
    static const char* cp[] = {"mc", "mp", "l"};
    static const char* qr[] = {"mass", "J1", "J2", "J3"};
    static const char* ac[] = {"l1", "l2", "m1", "m2"};
    switch (model) {
        case TO_MODEL_DOUBLE_INTEGRATOR: return i < 1 ? di[i] : nullptr;
        case TO_MODEL_CARTPOLE: return i < 3 ? cp[i] : nullptr;
        case TO_MODEL_QUADROTOR: return i < 4 ? qr[i] : nullptr;
        case TO_MODEL_ACROBOT: return i < 4 ? ac[i] : nullptr;
        default: return nullptr;
    }
}

// The one place where a parameter vector is completed for the device: the reciprocals the dynamics multiply by (models.cuh).  to_create and
// to_set_model_params both go through it, so a per-instance row and a shared vector with the same entries hold the same bits.
void complete_model_params(int model, double* p) {
    if (model == TO_MODEL_DOUBLE_INTEGRATOR) p[1] = 1.0 / p[0];
    if (model == TO_MODEL_QUADROTOR) { p[10] = 1.0 / p[0]; p[11] = 1.0 / p[1]; p[12] = 1.0 / p[2]; p[13] = 1.0 / p[3]; }
}

int build_cost(to_handle* h, const to_cost_spec& tc, int n, int m, DevCost& c) {
    std::memset(&c, 0, sizeof(c));
    if (tc.kind == TO_COST_EXPR) {   // user cost recorded as a program (RD.@autodiff CostFunction)
        if (!tc.prog || tc.prog_len < 1 || tc.prog_len > TO_EXPR_LEN || tc.nconst < 0 || tc.nconst > TO_EXPR_CONST || (tc.nconst > 0 && !tc.consts))
            return fail(h, TO_EINVAL, "expression cost: bad program size");
        c.expr = 1; c.prog_len = tc.prog_len; c.terminal = tc.terminal != 0;
        for (int j = 0; j < tc.prog_len; j++) {
            const int op = tc.prog[3 * j], a = tc.prog[3 * j + 1], b = tc.prog[3 * j + 2];
            const bool bin = op >= TO_OP_ADD && op <= TO_OP_DIV;
            bool ok = op >= 0 && op <= TO_OP_RSUBC;
            if (op == TO_OP_CONST) ok = ok && a >= 0 && a < tc.nconst;
            else if (op == TO_OP_X) ok = ok && a >= 0 && a < n;
            else if (op == TO_OP_U) ok = ok && a >= 0 && a < m;
            else { ok = ok && a >= 0 && a < j; if (bin) ok = ok && b >= 0 && b < j; if (op == TO_OP_POWC || op >= TO_OP_ADDC) ok = ok && b >= 0 && b < tc.nconst; }
            if (!ok) return fail(h, TO_EINVAL, "expression cost: invalid instruction");
            c.prog[3 * j] = op; c.prog[3 * j + 1] = a; c.prog[3 * j + 2] = b;
        }
        for (int j = 0; j < tc.nconst; j++) c.pconst[j] = tc.consts[j];
        return TO_OK;
    }
    if (!tc.Q || !tc.R || !tc.q || !tc.r) return fail(h, TO_EINVAL, "cost: null Q/R/q/r");
    c.diag = (tc.kind == TO_COST_DIAGONAL || tc.kind == TO_COST_DIAGONAL_QUAT); c.terminal = tc.terminal != 0; c.c = tc.c;
    if (tc.kind == TO_COST_DIAGONAL_QUAT) {   // DiagonalQuatCost, src/lie_costs.jl:33-56
        if (!tc.q_ref) return fail(h, TO_EINVAL, "DiagonalQuatCost: null q_ref");
        c.quat = 1; c.w = tc.w;
        for (int i = 0; i < 4; i++) {
            c.q_ref[i] = tc.q_ref[i]; c.q_ind[i] = tc.q_ind ? tc.q_ind[i] - 1 : 3 + i;
            if (c.q_ind[i] < 0 || c.q_ind[i] >= n) return fail(h, TO_EDIM, "DiagonalQuatCost: q_ind outside the state");
        }
    } else if (tc.kind != TO_COST_DIAGONAL && tc.kind != TO_COST_QUADRATIC) return fail(h, TO_EINVAL, "unknown cost kind");
    for (int i = 0; i < n; i++) c.q[i] = tc.q[i];
    for (int i = 0; i < m; i++) c.r[i] = tc.r[i];
    if (c.diag) {
        for (int i = 0; i < n; i++) { c.Qd[i] = tc.Q[i]; c.Q[i * n + i] = tc.Q[i]; }
        for (int i = 0; i < m; i++) { c.Rd[i] = tc.R[i]; c.R[i * m + i] = tc.R[i]; }
        c.zeroH = 1;
    } else {
        for (int i = 0; i < n * n; i++) c.Q[i] = tc.Q[i];
        for (int i = 0; i < m * m; i++) c.R[i] = tc.R[i];
        for (int i = 0; i < n; i++) c.Qd[i] = tc.Q[i * n + i];
        for (int i = 0; i < m; i++) c.Rd[i] = tc.R[i * m + i];
        double hn = 0;
        if (tc.H) for (int i = 0; i < m * n; i++) { c.H[i] = tc.H[i]; hn = std::fmax(hn, std::fabs(tc.H[i])); }
        c.zeroH = (hn == 0.0);   // is_blockdiag(cost) = zeroH, src/cost_functions.jl:445,455
    }
    return TO_OK;
}

// doubles of constraint c in an instance's row of DevProblem::cdata (0: no per-instance data)
int con_row_len(const DevCon& c, int nm) {
    switch (c.kind) {
        case CON_GOAL: return c.p;
        case CON_BOUND: return 2 * nm;
        case CON_LINEAR: return c.p;
        case CON_CIRCLE: return 3 * c.p;
        case CON_SPHERE: return 4 * c.p;
        case CON_NORM: case CON_COLLISION: return 1;
    }
    return 0;
}
// ... as to_constraint_data_len reports it: a Goal's values are set with to_set_goal_values, not to_set_constraint_data
int con_data_len(const DevCon& c, int nm) { return c.kind == CON_GOAL ? 0 : con_row_len(c, nm); }
// the shared data of constraint c in the layout of its row (common.cuh con_data)
void con_shared_row(const DevCon& c, int nm, double* row) {
    const int p = c.p;
    switch (c.kind) {
        case CON_GOAL: std::memcpy(row, c.a, sizeof(double) * p); break;
        case CON_BOUND: std::memcpy(row, c.a, sizeof(double) * nm); std::memcpy(row + nm, c.b, sizeof(double) * nm); break;
        case CON_LINEAR: std::memcpy(row, c.b, sizeof(double) * p); break;
        case CON_CIRCLE: case CON_SPHERE: {
            const bool sph = c.kind == CON_SPHERE;
            std::memcpy(row, c.a, sizeof(double) * p); std::memcpy(row + p, c.b, sizeof(double) * p);
            if (sph) std::memcpy(row + 2 * p, c.c3, sizeof(double) * p);
            std::memcpy(row + (sph ? 3 : 2) * p, c.rad, sizeof(double) * p);
            break;
        }
        case CON_NORM: case CON_COLLISION: row[0] = c.val; break;
    }
}

int build_con(to_handle* h, const to_constraint_spec& tc, int n, int m, int N, DevCon& c) {
    std::memset(&c, 0, sizeof(c));
    const int nm = n + m;
    c.kind = tc.kind; c.first = tc.first; c.last = tc.last; c.flag = tc.flag; c.val = tc.val;
    if (tc.first < 1 || tc.last > N || tc.last < tc.first) return fail(h, TO_EINVAL, "constraint knot range outside 1:N");
    for (int j = 0; j < TO_MAXNM; j++) { c.row_max[j] = -1; c.row_min[j] = -1; }
    switch (tc.kind) {
        case TO_CON_GOAL:
            if (tc.ninds < 1 || tc.ninds > n || !tc.inds || !tc.a) return fail(h, TO_EINVAL, "GoalConstraint: bad inds/xf");
            c.p = tc.ninds; c.sense = CONE_ZERO; c.diagonal = 1; c.ninds = tc.ninds;
            for (int i = 0; i < tc.ninds; i++) {
                const int j = tc.inds[i] - 1;
                if (j < 0 || j >= n) return fail(h, TO_EDIM, "GoalConstraint: index outside the state");
                c.inds[i] = j; c.a[i] = tc.a[i]; c.row_max[j] = i;
            }
            break;
        case TO_CON_BOUND:
            if (!tc.a || !tc.b) return fail(h, TO_EINVAL, "BoundConstraint: null bounds");
            c.sense = CONE_NEGATIVE_ORTHANT; c.diagonal = 1;
            for (int j = 0; j < nm; j++) {
                if (!(tc.a[j] >= tc.b[j])) return fail(h, TO_EINVAL, "Upper bounds must be greater than or equal to lower bounds");   // src/constraints.jl:712
                c.a[j] = tc.a[j]; c.b[j] = tc.b[j];
            }
            for (int j = 0; j < nm; j++) if (std::isfinite(tc.a[j])) { c.row_max[j] = c.n_max; c.a_max[c.n_max++] = j; }
            for (int j = 0; j < nm; j++) if (std::isfinite(tc.b[j])) { c.row_min[j] = c.n_max + c.n_min; c.a_min[c.n_min++] = j; }
            c.p = c.n_max + c.n_min;
            if (c.p == 0) return fail(h, TO_EINVAL, "BoundConstraint without any finite bound");
            break;
        case TO_CON_LINEAR: {
            const int w = tc.flag ? m : n;
            if (tc.p < 1 || tc.p > TO_MAXP || tc.p * w > TO_CON_A || !tc.a || !tc.b) return fail(h, TO_EINVAL, "LinearConstraint: bad size");
            c.p = tc.p; c.sense = tc.sense;
            for (int i = 0; i < tc.p * w; i++) c.a[i] = tc.a[i];
            for (int i = 0; i < tc.p; i++) c.b[i] = tc.b[i];
            break;
        }
        case TO_CON_CIRCLE:
        case TO_CON_SPHERE: {
            const int need = tc.kind == TO_CON_CIRCLE ? 2 : 3;
            if (tc.p < 1 || tc.p > TO_MAXP || !tc.a || !tc.b || !tc.rad || (need == 3 && !tc.c)) return fail(h, TO_EINVAL, "Circle/SphereConstraint: bad size");
            c.p = tc.p; c.sense = CONE_NEGATIVE_ORTHANT;
            for (int i = 0; i < tc.p; i++) { c.a[i] = tc.a[i]; c.b[i] = tc.b[i]; c.rad[i] = tc.rad[i]; if (need == 3) c.c3[i] = tc.c[i]; }
            for (int i = 0; i < need; i++) {
                c.inds[i] = (tc.inds && tc.ninds > i) ? tc.inds[i] - 1 : i;
                if (c.inds[i] < 0 || c.inds[i] >= n) return fail(h, TO_EDIM, "Circle/SphereConstraint: index outside the state");
            }
            break;
        }
        case TO_CON_NORM:
            if (tc.ninds < 1 || tc.ninds > nm || !tc.inds) return fail(h, TO_EINVAL, "NormConstraint: bad inds");
            c.sense = tc.sense; c.ninds = tc.ninds;
            for (int i = 0; i < tc.ninds; i++) {
                c.inds[i] = tc.inds[i] - 1;
                if (c.inds[i] < 0 || c.inds[i] >= nm) return fail(h, TO_EDIM, "NormConstraint: index outside z");
            }
            c.p = (tc.sense == TO_CONE_SECOND_ORDER) ? tc.ninds + 1 : 1;
            if (tc.sense != TO_CONE_SECOND_ORDER && tc.sense != TO_CONE_NEGATIVE_ORTHANT && tc.sense != TO_CONE_ZERO)
                return fail(h, TO_EINVAL, "NormConstraint: sense must be Inequality, Equality or SecondOrderCone");
            break;
        case TO_CON_COLLISION: {
            const int D = tc.ninds / 2;
            if (tc.ninds < 2 || (tc.ninds & 1) || tc.ninds > TO_MAXNM || !tc.inds)
                return fail(h, TO_EDIM, "Position dimensions must be of equal length");   // @assert src/constraints.jl:349
            c.p = 1; c.sense = CONE_NEGATIVE_ORTHANT; c.ninds = tc.ninds; c.val = tc.val;
            for (int i = 0; i < 2 * D; i++) {
                c.inds[i] = tc.inds[i] - 1;
                if (c.inds[i] < 0 || c.inds[i] >= n) return fail(h, TO_EDIM, "CollisionConstraint: index outside the state");
            }
            break;
        }
        case TO_CON_EXPR: {    // user constraint recorded as a program
            const int L = tc.ninds / 3;
            if (!tc.inds || tc.ninds % 3 || L < 1 || L > TO_EXPR_LEN || tc.p < 1 || tc.p > L || tc.p > TO_MAXP || tc.flag < 0 || tc.flag > TO_EXPR_CONST || (tc.flag > 0 && !tc.a))
                return fail(h, TO_EINVAL, "expression constraint: bad program size");
            c.p = tc.p; c.sense = tc.sense; c.prog_len = L; c.ninds = 0;
            if (tc.sense < 0 || tc.sense > CONE_POSITIVE_ORTHANT) return fail(h, TO_EINVAL, "expression constraint: unknown sense");
            for (int j = 0; j < L; j++) {
                const int op = tc.inds[3 * j], a = tc.inds[3 * j + 1], b = tc.inds[3 * j + 2];
                const bool bin = op >= TO_OP_ADD && op <= TO_OP_DIV;
                bool ok = op >= 0 && op <= TO_OP_RSUBC;
                if (op == TO_OP_CONST) ok = ok && a >= 0 && a < tc.flag;
                else if (op == TO_OP_X) ok = ok && a >= 0 && a < n;
                else if (op == TO_OP_U) ok = ok && a >= 0 && a < m;
                else { ok = ok && a >= 0 && a < j; if (bin) ok = ok && b >= 0 && b < j; if (op == TO_OP_POWC || op >= TO_OP_ADDC) ok = ok && b >= 0 && b < tc.flag; }
                if (!ok) return fail(h, TO_EINVAL, "expression constraint: invalid instruction");
                c.prog[3 * j] = op; c.prog[3 * j + 1] = a; c.prog[3 * j + 2] = b;
            }
            for (int j = 0; j < tc.flag; j++) c.pconst[j] = tc.a[j];
            c.flag = 0;
            break;
        }
        case TO_CON_QUATVEC:   // QuatVecEq, src/constraints.jl:938-965
            if (!tc.a || n < 4) return fail(h, TO_EINVAL, "QuatVecEq: null qf");
            c.p = 3; c.sense = CONE_ZERO; c.ninds = 4;
            for (int i = 0; i < 4; i++) {
                c.a[i] = tc.a[i];
                c.inds[i] = (tc.inds && tc.ninds == 4) ? tc.inds[i] - 1 : 3 + i;
                if (c.inds[i] < 0 || c.inds[i] >= n) return fail(h, TO_EDIM, "QuatVecEq: qind outside the state");
            }
            break;
        default: return fail(h, TO_EINVAL, "unknown constraint kind");
    }
    if (c.p > (c.diagonal ? TO_MAXPV : TO_MAXP))
        return fail(h, TO_EINVAL, "constraint output dimension exceeds the library limit (32 rows per knot; 2 (n + m) for Goal / Bound constraints)");
    return TO_OK;
}

}  // namespace

extern "C" {

const char* to_last_error(const to_handle* h) { return h ? h->err.c_str() : g_create_error.c_str(); }

// Every entry point makes the handle's device current for its duration and restores the caller's afterwards: one process may hold
// handles on several GPUs (to_spec.device), and the host application (torch, Julia's CUDA.jl) has its own idea of the current device.
struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(const to_handle* h) {
        if (!h) return;
        int cur = -1;
        if (cudaGetDevice(&cur) == cudaSuccess && cur != h->device) { prev = cur; cudaSetDevice(h->device); }
    }
    ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};
// Every entry point that touches trajectory data on the main stream first joins the side stream (see to_ilqr_step).
static int join_side(to_handle* h) {
    if (h && h->side_pending) {
        h->side_pending = false;
        if (cudaStreamWaitEvent(h->stream, h->ev_join, 0) != cudaSuccess) return fail(h, TO_ECUDA, "cudaStreamWaitEvent");
    }
    return TO_OK;
}
#define JOIN(h) DeviceGuard device_guard__(h); do { int jrc_ = join_side(h); if (jrc_) return jrc_; } while (0)

int to_default_options(to_options* o) {
    if (!o) return TO_EINVAL;
    DevOptions d; set_default_options(d);
    o->bp_reg_increase_factor = d.bp_reg_increase_factor; o->bp_reg_max = d.bp_reg_max; o->bp_reg_min = d.bp_reg_min;
    o->bp_reg_initial = d.bp_reg_initial; o->bp_reg_fp = d.bp_reg_fp;
    o->line_search_lower_bound = d.ls_lower; o->line_search_upper_bound = d.ls_upper; o->iterations_linesearch = d.ls_iters; o->backward_kernel = 0;
    o->max_state_value = d.max_state_value; o->max_control_value = d.max_control_value;
    o->penalty_initial = d.penalty_initial; o->penalty_scaling = d.penalty_scaling; o->penalty_max = d.penalty_max; o->dual_max = d.dual_max;
    return TO_OK;
}

int to_create(const to_spec* s, to_handle** out) {
    if (!s || !out) return fail(nullptr, TO_EINVAL, "null argument");
    *out = nullptr;
    int dev_count = 0;
    cudaError_t ce = cudaGetDeviceCount(&dev_count);
    if (ce != cudaSuccess || dev_count == 0)
        return fail(nullptr, TO_ECUDA, "no CUDA device: this library has no CPU fallback (" + std::string(cudaGetErrorString(ce)) + ")");
    if (s->device < 0 || s->device >= dev_count) return fail(nullptr, TO_EINVAL, "device ordinal out of range");
    int mn = 0, mm = 0; double params[16];
    model_defaults(s->model, s->m, mn, mm, params);
    if (mn < 0) return fail(nullptr, TO_EINVAL, "unknown model id");
    if (s->model == TO_MODEL_DOUBLE_INTEGRATOR && s->m != 1 && s->m != 2) return fail(nullptr, TO_EDIM, "DoubleIntegrator: supported dimensions are 1 and 2");
    std::vector<DevDyn> dyn_tab; std::vector<int> dyn_idx;
    if (s->model == TO_MODEL_EXPR) {
        // Problem(models::Vector, ...) with RD.dims(models) (src/dynamics.jl:15-31): per-knot dimensions, padded to the (n, m) = (4, 2) the kernels exist for
        if (s->n != 4 || s->m != 2) return fail(nullptr, TO_EDIM, "recorded-program models: the padded dimensions must be n = 4, m = 2 (largest per-knot dimensions <= that)");
        if (s->N < 2 || !s->dyn || s->ndyn < 1 || !s->dyn_index || !s->nx || !s->nu) return fail(nullptr, TO_EINVAL, "recorded-program models: null dyn / dyn_index / nx / nu");
        for (int i = 0; i < s->ndyn; i++) {
            const to_dynamics_spec& d = s->dyn[i];
            if (!d.prog || d.prog_len < 1 || d.prog_len > TO_EXPR_LEN || d.nconst < 0 || d.nconst > TO_EXPR_CONST || (d.nconst > 0 && !d.consts) ||
                d.n_in < 1 || d.n_in > 4 || d.m_in < 0 || d.m_in > 2 || d.n_out < 1 || d.n_out > 4 || d.n_out > d.prog_len)
                return fail(nullptr, TO_EINVAL, "recorded-program model: bad program size or dimensions");
            DevDyn dd; std::memset(&dd, 0, sizeof(dd));
            dd.n_in = d.n_in; dd.m_in = d.m_in; dd.n_out = d.n_out; dd.discrete = d.discrete != 0; dd.prog_len = d.prog_len;
            for (int j = 0; j < d.prog_len; j++) {
                const int op = d.prog[3 * j], a = d.prog[3 * j + 1], b = d.prog[3 * j + 2];
                const bool bin = op >= TO_OP_ADD && op <= TO_OP_DIV;
                bool ok = op >= 0 && op <= TO_OP_RSUBC;
                if (op == TO_OP_CONST) ok = ok && a >= 0 && a < d.nconst;
                else if (op == TO_OP_X) ok = ok && a >= 0 && a < d.n_in;
                else if (op == TO_OP_U) ok = ok && a >= 0 && a < d.m_in;
                else { ok = ok && a >= 0 && a < j; if (bin) ok = ok && b >= 0 && b < j; if (op == TO_OP_POWC || op >= TO_OP_ADDC) ok = ok && b >= 0 && b < d.nconst; }
                if (!ok) return fail(nullptr, TO_EINVAL, "recorded-program model: invalid instruction");
                dd.prog[3 * j] = op; dd.prog[3 * j + 1] = a; dd.prog[3 * j + 2] = b;
            }
            for (int j = 0; j < d.nconst; j++) dd.pconst[j] = d.consts[j];
            dyn_tab.push_back(dd);
        }
        for (int k = 0; k < s->N - 1; k++) {
            const int di = s->dyn_index[k];
            if (di < 0 || di >= s->ndyn) return fail(nullptr, TO_EINVAL, "dyn_index out of range");
            const DevDyn& d = dyn_tab[di];
            if (d.n_in != s->nx[k] || d.m_in != s->nu[k])
                return fail(nullptr, TO_EDIM, "Model " + std::to_string(k + 1) + " has state / control dimensions (" + std::to_string(d.n_in) + ", " + std::to_string(d.m_in) +
                            ") but knot " + std::to_string(k + 1) + " has (" + std::to_string(s->nx[k]) + ", " + std::to_string(s->nu[k]) + ").");
            if (d.n_out != s->nx[k + 1])     // src/dynamics.jl:23-28
                return fail(nullptr, TO_EDIM, "Model mismatch at time step " + std::to_string(k + 1) + ". Model " + std::to_string(k + 1) + " has an output dimension of " +
                            std::to_string(d.n_out) + " but model " + std::to_string(k + 2) + " has a state dimension of " + std::to_string(s->nx[k + 1]) + ".");
            dyn_idx.push_back(di);
        }
    }
    if (mn != s->n) return fail(nullptr, TO_EDIM, "Objective state dimensions don't match model.");     // src/problem.jl:67
    if (mm != s->m) return fail(nullptr, TO_EDIM, "Objective control dimensions don't match model.");   // src/problem.jl:68
    if (s->N < 2 || s->B < 1) return fail(nullptr, TO_EINVAL, "need N >= 2 knot points and B >= 1 instances");
    if (!s->dt || !s->costs || !s->cost_index || s->ncost < 1) return fail(nullptr, TO_EINVAL, "null dt / costs / cost_index");
    if (s->ncon < 0 || s->ncon > TO_MAXCON || (s->ncon > 0 && !s->cons)) return fail(nullptr, TO_EINVAL, "too many constraints (max 8) or null list");
    for (int k = 0; k < s->N - 1; k++) if (!(s->dt[k] > 0)) return fail(nullptr, TO_EINVAL, "time steps must be positive");   // tf > t0, src/problem.jl:50
    if (s->error_state && s->model != TO_MODEL_QUADROTOR)
        return fail(nullptr, TO_EINVAL, "error_state: the model has no Lie-group state (only the Quadrotor does)");
    if (s->params) for (int i = 0; i < s->nparams && i < 10; i++) params[i] = s->params[i];
    complete_model_params(s->model, params);

    auto* h = new to_handle();
    h->device = s->device;
    DeviceGuard device_guard(h);        // the caller's current device is restored when to_create returns
    auto bail = [&](int code) { std::string msg = h->err; to_destroy(h); g_create_error = msg; return code; };
    if (cudaSetDevice(s->device) != cudaSuccess) { h->err = "cudaSetDevice failed"; return bail(TO_ECUDA); }
    if (cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess) { h->err = "cudaStreamCreate failed"; return bail(TO_ECUDA); }
    h->own_stream = true;
    {
        int lo = 0, hi = 0;
        cudaDeviceGetStreamPriorityRange(&lo, &hi);
        if (const char* ev = getenv("TO_NO_OVERLAP")) h->overlap = atoi(ev) == 0;
        if (cudaStreamCreateWithPriority(&h->stream2, cudaStreamNonBlocking, hi) != cudaSuccess ||
            cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&h->ev_join, cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&h->ev_merit, cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&h->ev_cons, cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&h->ev_count[0], cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&h->ev_count[1], cudaEventDisableTiming) != cudaSuccess) { h->err = "side stream creation failed"; return bail(TO_ECUDA); }
        if (cudaHostAlloc((void**)&h->pin_count, 2 * sizeof(int), cudaHostAllocDefault) != cudaSuccess) { h->err = "cudaHostAlloc failed"; return bail(TO_ENOMEM); }
    }
    DevProblem& P = h->P;
    P.model = s->model; P.n = mn; P.m = mm; P.N = s->N; P.B = s->B;
    // row stride of [A B]: even (16-byte rows); 20 (= 4 mod 16) for the tensor-MMA Riccati path (n >= 8), see riccati.cu
    P.ldab = (mn >= 8 && mn <= 16 && mn + mm + 1 <= 20) ? 20 : ((mn + mm + 1) & ~1);
    std::memcpy(P.params, params, sizeof(params));
    set_default_options(P.opt);
    h->t0 = s->t0;
    const int n = mn, m = mm, N = s->N, B = s->B;

    h->h_costs.resize(s->ncost);
    P.all_diag_cost = 1;
    for (int i = 0; i < s->ncost; i++) {
        int rc = build_cost(h, s->costs[i], n, m, h->h_costs[i]);
        if (rc) return bail(rc);
        if (!h->h_costs[i].diag) P.all_diag_cost = 0;
        if (h->h_costs[i].quat || h->h_costs[i].expr) { P.all_diag_cost = 0; P.dense_riccati = 1; }   // the fused fast paths assume purely quadratic costs
    }
    P.lie = s->error_state ? 1 : 0; P.qs = 3; P.ne = P.lie ? n - 1 : n;
    if (P.lie) P.dense_riccati = 1;
    {   // compact expansion (lie.cu): error state + DiagonalCost + Goal/Bound constraints only
        bool diag_costs = true;
        for (const auto& c : h->h_costs) if (!c.diag || c.expr || c.quat) diag_costs = false;   // (quaternion costs: generic expansion, until the compact kernel's variant is GPU-tested)
        bool diag_cons = true;
        for (int i = 0; i < s->ncon; i++) if (s->cons[i].kind != TO_CON_GOAL && s->cons[i].kind != TO_CON_BOUND) diag_cons = false;
        P.compact = (P.lie && diag_costs && diag_cons && P.ne == 12 && m == 4) ? 1 : 0;
        // compact problems: [A_e B_e] + expansion as per-knot records for the register-resident Riccati kernel (riccati_frag.cu);
        // TO_NO_FRAG=1 keeps the shared-memory kernel of lie.cu (A/B timing)
        const char* nf = getenv("TO_NO_FRAG");
        P.frag = (P.compact && !(nf && atoi(nf) != 0)) ? 1 : 0;
    }
    if (P.dense_riccati && !P.compact) h->overlap = false;   // generic lie.cu path: every kernel on the main stream
    h->h_cost_index.assign(s->cost_index, s->cost_index + N);
    for (int k = 0; k < N; k++)
        if (h->h_cost_index[k] < 0 || h->h_cost_index[k] >= s->ncost) { h->err = "cost_index out of range"; return bail(TO_EINVAL); }
    h->h_cons.resize(s->ncon);
    P.all_diag_con = 1; P.lambda_len = 0;
    for (int i = 0; i < s->ncon; i++) {
        int rc = build_con(h, s->cons[i], n, m, N, h->h_cons[i]);
        if (rc) return bail(rc);
        h->h_cons[i].offset = P.lambda_len;
        P.lambda_len += (h->h_cons[i].last - h->h_cons[i].first + 1) * h->h_cons[i].p;
        const int clen = con_row_len(h->h_cons[i], n + m);
        h->h_cons[i].cdoff = clen ? P.ncdata : -1; P.ncdata += clen;
        if (!h->h_cons[i].diagonal) P.all_diag_con = 0;
    }
    P.ncost = s->ncost; P.ncon = s->ncon;
    P.max_p_knot = 0; P.max_terms_per_z = 0;
    for (int j = 0; j < n + m; j++) {
        int cnt = 0;
        for (const auto& c : h->h_cons) if (c.diagonal) cnt += (c.row_max[j] >= 0) + (c.kind == CON_BOUND && c.row_min[j] >= 0);
        P.max_terms_per_z = std::max(P.max_terms_per_z, cnt);
    }
    P.max_cons_knot = 0;
    for (int k = 1; k <= N; k++) {
        int pk = 0, nk = 0;
        for (const auto& c : h->h_cons) if (k >= c.first && k <= c.last) { pk += c.p; nk++; }
        P.max_p_knot = std::max(P.max_p_knot, pk);
        P.max_cons_knot = std::max(P.max_cons_knot, nk);
    }
    {   // DevProblem::fwd_compact
        bool cls = N >= 2 && P.all_diag_cost && P.all_diag_con;
        for (int k = 1; k < N - 1; k++) if (h->h_cost_index[k] != h->h_cost_index[0]) cls = false;
        int nbox = 0, ngc = 0;
        for (const auto& c : h->h_cons) {
            if (c.kind == CON_BOUND) {
                bool ubox = c.first == 1 && c.last == N - 1 && c.p == 2 * m;
                for (int j = 0; j < n + m; j++) if ((c.row_max[j] >= 0) != (j >= n) || (c.row_min[j] >= 0) != (j >= n)) ubox = false;
                cls = cls && ubox; nbox++;
            } else if (c.kind == CON_GOAL) {
                cls = cls && c.first == N && c.last == N; ngc++;
            } else cls = false;
        }
        P.fwd_compact = (cls && nbox <= 1 && ngc <= 1) ? 1 : 0;
    }
    h->h_mu.assign(s->ncon, P.opt.penalty_initial);
    h->h_dt.assign(s->dt, s->dt + (N - 1));
    h->h_dyn = dyn_tab; h->h_dyn_index = dyn_idx;

    int rc = TO_OK;
    double* d_dt = nullptr; int* d_ci = nullptr;
    P.strideX = (size_t)B * N * n; P.strideU = (size_t)B * (N - 1) * m;
#define ALLOC(ptr, count) if (!rc) rc = dalloc(h, &(ptr), (size_t)(count))
    ALLOC(d_dt, N - 1); ALLOC(d_ci, N);
    DevDyn* d_dyn = nullptr; int* d_dyni = nullptr;
    if (!h->h_dyn.empty()) { ALLOC(d_dyn, h->h_dyn.size()); ALLOC(d_dyni, N - 1); }
    ALLOC(h->d_costs, s->ncost); ALLOC(h->d_cons, std::max(1, s->ncon)); ALLOC(h->d_mu, std::max(1, s->ncon));
    ALLOC(P.x0, (size_t)B * n); ALLOC(P.X, TO_NBUF * P.strideX); ALLOC(P.U, TO_NBUF * P.strideU); ALLOC(P.cur, B);
    ALLOC(P.AB, (size_t)B * (N - 1) * n * P.ldab); ALLOC(P.K, (size_t)B * (N - 1) * P.ne * m); ALLOC(P.d, (size_t)B * (N - 1) * m);
    if (P.dense_riccati) {
        const size_t nme = P.ne + m;
        ALLOC(P.ABe, (size_t)B * (N - 1) * P.ne * nme); ALLOC(P.EG, (size_t)B * N * nme); ALLOC(P.EH, (size_t)B * N * nme * nme);
        if (P.compact) ALLOC(P.EC, (size_t)B * N * TO_EC_LEN);
        if (P.frag) ALLOC(P.REC, (size_t)B * N * TO_REC_LEN);
    }
    ALLOC(P.lambda, (size_t)B * std::max(1, P.lambda_len));
    ALLOC(P.rho, B); ALLOC(P.drho, B); ALLOC(P.dV, 2 * (size_t)B); ALLOC(P.J, B); ALLOC(P.Jc, B); ALLOC(P.alpha, B);
    ALLOC(P.bp_status, B); ALLOC(P.ls_iters, B); ALLOC(P.accepted, B); ALLOC(P.acc1, B);
    // The later line-search passes can walk a compact list of the late instances (the ones pass 1 did not accept) instead of scanning all, in half-warp
    // CTAs of two instances (forward.cu launch_pass): only CTAs with work stay resident next to the expansion kernels of the main stream.  On the record
    // path (error-state Quadrotor: cost + dynamics expansion on the main stream) that balances the two overlapped chains -- 2.10 vs 2.21 ms per step
    // on one H100; on the other paths the late pass itself is the longer chain and the list makes it longer, so they keep scanning with full warps.
    if (P.frag) { ALLOC(P.late_list, B); ALLOC(P.late_count, 1); }
    ALLOC(h->d_stageX, P.strideX); ALLOC(h->d_stageU, P.strideU); ALLOC(h->d_viol, B); ALLOC(h->d_merit2, 2);
    ALLOC(h->d_work, 1); ALLOC(h->d_err, 1);
    {   // to_solve state (solve.cu)
        SolveDev& S = h->solve;
        ALLOC(S.state, B); ALLOC(S.status, B); ALLOC(S.iter, B); ALLOC(S.outer, B); ALLOC(S.inner, B); ALLOC(S.dj_zero, B);
        ALLOC(S.J_prev, B); ALLOC(S.dJ, B); ALLOC(S.grad, B); ALLOC(S.cmax, B); ALLOC(S.n_active, 1);
    }
    if (P.frag) { ALLOC(h->d_fragq, frag_queue_ints(B)); ALLOC(h->d_fragpool, frag_pool_doubles(B, N)); ALLOC(h->d_fragerr, 1); ALLOC(h->d_exptab, 1); }
#undef ALLOC
    if (rc) return bail(rc);
    P.exptab = h->d_exptab;
    P.dyn = d_dyn; P.dyn_index = d_dyni;
    P.dt = d_dt; P.cost_index = d_ci; P.costs = h->d_costs; P.cons = h->d_cons; P.mu = h->d_mu; P.viol = h->d_viol;
    cudaStream_t st = h->stream;
    bool okc = true;
    okc &= cudaMemcpyAsync(d_dt, h->h_dt.data(), sizeof(double) * (N - 1), cudaMemcpyHostToDevice, st) == cudaSuccess;
    okc &= cudaMemcpyAsync(d_ci, h->h_cost_index.data(), sizeof(int) * N, cudaMemcpyHostToDevice, st) == cudaSuccess;
    if (d_dyn) {
        okc &= cudaMemcpyAsync(d_dyn, h->h_dyn.data(), sizeof(DevDyn) * h->h_dyn.size(), cudaMemcpyHostToDevice, st) == cudaSuccess;
        okc &= cudaMemcpyAsync(d_dyni, h->h_dyn_index.data(), sizeof(int) * (N - 1), cudaMemcpyHostToDevice, st) == cudaSuccess;
    }
    okc &= cudaMemsetAsync(P.x0, 0, sizeof(double) * B * n, st) == cudaSuccess;
    okc &= cudaMemsetAsync(P.X, 0xFF, sizeof(double) * TO_NBUF * P.strideX, st) == cudaSuccess;   // NaN: X0 = NaN until rollout!, src/problem.jl:83
    okc &= cudaMemsetAsync(P.U, 0, sizeof(double) * TO_NBUF * P.strideU, st) == cudaSuccess;      // U0 = 0, src/problem.jl:84
    okc &= cudaMemsetAsync(P.cur, 0, sizeof(int) * B, st) == cudaSuccess;
    okc &= cudaMemsetAsync(P.AB, 0, sizeof(double) * (size_t)B * (N - 1) * n * P.ldab, st) == cudaSuccess;
    okc &= cudaMemsetAsync(P.K, 0, sizeof(double) * (size_t)B * (N - 1) * P.ne * m, st) == cudaSuccess;
    okc &= cudaMemsetAsync(P.d, 0, sizeof(double) * (size_t)B * (N - 1) * m, st) == cudaSuccess;
    okc &= cudaMemsetAsync(P.lambda, 0, sizeof(double) * (size_t)B * std::max(1, P.lambda_len), st) == cudaSuccess;
    okc &= cudaMemsetAsync(P.rho, 0, sizeof(double) * B, st) == cudaSuccess;
    okc &= cudaMemsetAsync(P.drho, 0, sizeof(double) * B, st) == cudaSuccess;
    okc &= cudaMemsetAsync(P.dV, 0, sizeof(double) * 2 * B, st) == cudaSuccess;
    okc &= cudaMemsetAsync(P.J, 0, sizeof(double) * B, st) == cudaSuccess;
    okc &= cudaMemsetAsync(P.Jc, 0, sizeof(double) * B, st) == cudaSuccess;
    okc &= cudaMemsetAsync(P.alpha, 0, sizeof(double) * B, st) == cudaSuccess;
    okc &= cudaMemsetAsync(P.bp_status, 0, sizeof(int) * B, st) == cudaSuccess;
    okc &= cudaMemsetAsync(P.ls_iters, 0, sizeof(int) * B, st) == cudaSuccess;
    okc &= cudaMemsetAsync(P.accepted, 0, sizeof(int) * B, st) == cudaSuccess;
    okc &= cudaMemsetAsync(P.acc1, 0, sizeof(int) * B, st) == cudaSuccess;
    if (h->d_fragerr) okc &= cudaMemsetAsync(h->d_fragerr, 0, sizeof(int), st) == cudaSuccess;
    okc &= cudaMemsetAsync(h->d_err, 0, sizeof(int), st) == cudaSuccess;
    if (!okc) { h->err = std::string("device initialisation failed: ") + cudaGetErrorString(cudaGetLastError()); return bail(TO_ECUDA); }
    rc = upload_tables(h);
    if (rc) return bail(rc);
    if (launch_trivial_columns_full(P, st) != cudaSuccess) { h->err = "k_trivial_columns_full failed"; return bail(TO_ECUDA); }   // closed-form columns of [A B] (rollout.cu SeedList)
    if (P.lie && P.model == MODEL_QUADROTOR) {        // the position / velocity columns of [A_e B_e] are functions of the time steps alone (rollout.cu)
        if (launch_trivial_columns(P, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess) { h->err = "k_trivial_columns failed"; return bail(TO_ECUDA); }
    }
    *out = h;
    return TO_OK;
}

int to_destroy(to_handle* h) {
    if (!h) return TO_OK;
    DeviceGuard device_guard(h);
    if (h->stream) cudaStreamSynchronize(h->stream);
    for (void* p : h->allocs) cudaFree(p);
    if (h->scratch.ptr) cudaFree(h->scratch.ptr);
    for (auto& e : h->pending) { cudaEventDestroy(e.a); cudaEventDestroy(e.b); }
    for (auto e : h->pool) cudaEventDestroy(e);
    if (h->stream2) { cudaStreamSynchronize(h->stream2); cudaStreamDestroy(h->stream2); }
    if (h->ev_fork) cudaEventDestroy(h->ev_fork);
    if (h->ev_join) cudaEventDestroy(h->ev_join);
    if (h->ev_merit) cudaEventDestroy(h->ev_merit);
    if (h->ev_cons) cudaEventDestroy(h->ev_cons);
    for (auto e : h->ev_count) if (e) cudaEventDestroy(e);
    if (h->pin_count) cudaFreeHost(h->pin_count);
    if (h->own_stream && h->stream) cudaStreamDestroy(h->stream);
    delete h;
    return TO_OK;
}

int to_set_options(to_handle* h, const to_options* o) {
    JOIN(h);
    if (!h || !o) return TO_EINVAL;
    if (o->iterations_linesearch < 0 || o->iterations_linesearch > 15) return fail(h, TO_EINVAL, "iterations_linesearch must be in 0..15");
    if (!(o->penalty_initial > 0) || !(o->penalty_scaling > 0)) return fail(h, TO_EINVAL, "penalties must be positive");
    DevOptions& d = h->P.opt;
    // the AL penalties and the regularisation state restart only when THEIR initial values change: setting an unrelated option in the
    // middle of a solve must not discard the penalty schedule
    const bool reset_mu = d.penalty_initial != o->penalty_initial, reset_rho = d.bp_reg_initial != o->bp_reg_initial;
    d.bp_reg_increase_factor = o->bp_reg_increase_factor; d.bp_reg_max = o->bp_reg_max; d.bp_reg_min = o->bp_reg_min;
    d.bp_reg_initial = o->bp_reg_initial; d.bp_reg_fp = o->bp_reg_fp;
    d.ls_lower = o->line_search_lower_bound; d.ls_upper = o->line_search_upper_bound; d.ls_iters = o->iterations_linesearch;
    d.pad = o->backward_kernel;   // kernel choice of launch_backward (0 automatic)
    d.max_state_value = o->max_state_value; d.max_control_value = o->max_control_value;
    d.penalty_initial = o->penalty_initial; d.penalty_scaling = o->penalty_scaling; d.penalty_max = o->penalty_max; d.dual_max = o->dual_max;
    if (reset_mu) for (auto& mu : h->h_mu) mu = d.penalty_initial;
    if (reset_rho) {
        std::vector<double> r(h->P.B, d.bp_reg_initial);
        CU(h, cudaMemcpyAsync(h->P.rho, r.data(), sizeof(double) * h->P.B, cudaMemcpyHostToDevice, h->stream));
        CU(h, cudaMemsetAsync(h->P.drho, 0, sizeof(double) * h->P.B, h->stream));
        CU(h, cudaStreamSynchronize(h->stream));     // `r` goes out of scope
    }
    h->J_valid = false;
    return upload_tables(h);
}

int to_set_stream(to_handle* h, void* cuda_stream) {
    JOIN(h);
    if (!h) return TO_EINVAL;
    CU(h, cudaStreamSynchronize(h->stream));
    if (h->own_stream) { cudaStreamDestroy(h->stream); h->own_stream = false; }
    h->stream = static_cast<cudaStream_t>(cuda_stream);
    return TO_OK;
}
int to_synchronize(to_handle* h) {
    JOIN(h);
    if (!h) return TO_EINVAL;
    CU(h, cudaStreamSynchronize(h->stream));
    if (h->d_fragerr) {     // the Riccati kernel's work queue never hangs the device: it gives up and says so here
        int e = 0;
        CU(h, cudaMemcpy(&e, h->d_fragerr, sizeof(int), cudaMemcpyDeviceToHost));
        if (e) return fail(h, TO_ESTATE, e & 2 ? "backward pass: work queue overflow (results invalid)" : "backward pass: a warp waited for queued work beyond the spin limit (results invalid)");
    }
    return TO_OK;
}
int to_dims(const to_handle* h, int32_t* n, int32_t* m, int32_t* N, int32_t* B) {
    if (!h) return TO_EINVAL;
    if (n) *n = h->P.n; if (m) *m = h->P.m; if (N) *N = h->P.N; if (B) *B = h->P.B;
    return TO_OK;
}
int to_num_constraints(const to_handle* h, int32_t* p_per_knot) {
    if (!h || !p_per_knot) return TO_EINVAL;
    for (int k = 1; k <= h->P.N; k++) {
        int p = 0;
        for (const auto& c : h->h_cons) if (k >= c.first && k <= c.last) p += c.p;
        p_per_knot[k - 1] = p;
    }
    return TO_OK;
}
int to_constraint_info(const to_handle* h, int32_t con, int32_t* p, int32_t* sense, int32_t* first, int32_t* last) {
    if (!h || con < 0 || con >= (int)h->h_cons.size()) return TO_EINVAL;
    const DevCon& c = h->h_cons[con];
    if (p) *p = c.p; if (sense) *sense = c.sense; if (first) *first = c.first; if (last) *last = c.last;
    return TO_OK;
}
// upper_bound / lower_bound by sense, src/abstract_constraint.jl:97-123
int to_bounds(const to_handle* h, int32_t con, double* lower, double* upper) {
    if (!h || con < 0 || con >= (int)h->h_cons.size()) return TO_EINVAL;
    const DevCon& c = h->h_cons[con];
    for (int i = 0; i < c.p; i++) {
        double lo = 0, up = 0;
        switch (c.sense) {
            case CONE_ZERO: lo = 0; up = 0; break;
            case CONE_NEGATIVE_ORTHANT: lo = -INFINITY; up = 0; break;
            case CONE_SECOND_ORDER: lo = -INFINITY; up = INFINITY; break;
            default: lo = -INFINITY; up = INFINITY;
        }
        if (lower) lower[i] = lo;
        if (upper) upper[i] = up;
    }
    return TO_OK;
}

// ---- setters / getters ----------------------------------------------------------------------------------
int to_set_initial_state(to_handle* h, const double* x0) {
    JOIN(h);
    if (!h || !x0) return TO_EINVAL;
    CU(h, cudaMemcpyAsync(h->P.x0, x0, sizeof(double) * (size_t)h->P.B * h->P.n, cudaMemcpyHostToDevice, h->stream));
    h->J_valid = false;
    return TO_OK;
}
int to_set_controls(to_handle* h, const double* U) {
    JOIN(h);
    if (!h || !U) return TO_EINVAL;
    CU(h, cudaMemcpyAsync(h->d_stageU, U, sizeof(double) * h->P.strideU, cudaMemcpyHostToDevice, h->stream));
    CU(h, launch_scatter_traj(h->P, nullptr, h->d_stageU, h->stream)); h->launches++;
    h->J_valid = false; h->expanded = false; h->backward_done = false;
    return TO_OK;
}
int to_set_states(to_handle* h, const double* X) {
    JOIN(h);
    if (!h || !X) return TO_EINVAL;
    CU(h, cudaMemcpyAsync(h->d_stageX, X, sizeof(double) * h->P.strideX, cudaMemcpyHostToDevice, h->stream));
    CU(h, launch_scatter_traj(h->P, h->d_stageX, nullptr, h->stream)); h->launches++;
    h->J_valid = false; h->expanded = false; h->backward_done = false;
    return TO_OK;
}
int to_get_states(to_handle* h, double* X) {
    JOIN(h);
    if (!h || !X) return TO_EINVAL;
    CU(h, launch_gather_traj(h->P, h->d_stageX, nullptr, h->stream)); h->launches++;
    CU(h, cudaMemcpyAsync(X, h->d_stageX, sizeof(double) * h->P.strideX, cudaMemcpyDeviceToHost, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    return TO_OK;
}
int to_get_controls(to_handle* h, double* U) {
    JOIN(h);
    if (!h || !U) return TO_EINVAL;
    CU(h, launch_gather_traj(h->P, nullptr, h->d_stageU, h->stream)); h->launches++;
    CU(h, cudaMemcpyAsync(U, h->d_stageU, sizeof(double) * h->P.strideU, cudaMemcpyDeviceToHost, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    return TO_OK;
}
int to_get_times(to_handle* h, double* t) {
    JOIN(h);
    if (!h || !t) return TO_EINVAL;
    t[0] = h->t0;
    for (int k = 1; k < h->P.N; k++) t[k] = t[k - 1] + h->h_dt[k - 1];
    return TO_OK;
}
int to_set_initial_time(to_handle* h, double t0, double* tf_out) {
    JOIN(h);
    if (!h) return TO_EINVAL;
    h->t0 = t0;
    if (tf_out) { double t = t0; for (double d : h->h_dt) t += d; *tf_out = t; }
    return TO_OK;
}
// ---- per-instance goals (DevProblem::qr, and the Goal rows of DevProblem::cdata) ------------------------------------------------------
// A setter stages the complete new rows of a table in h->stage and commits them (commit_rows).  The first per-instance call creates a table
// from the shared values; later shared calls write through to every row.
static int hybrid_goals(to_handle* h) { return fail(h, TO_EINVAL, "per-instance goals are not supported on hybrid problems"); }
static size_t q_off(const to_handle* h, int b, int cid) { return ((size_t)b * h->P.ncost + cid) * (h->P.n + h->P.m); }
static size_t cd_off(const to_handle* h, int b, const DevCon& c) { return (size_t)b * h->P.ncdata + c.cdoff; }
// h->stage := the rows of the cost-term table, or every instance's shared terms when it does not exist yet
static void stage_qr(to_handle* h) {
    if (h->P.qr) { h->stage = h->h_qr; return; }
    const int B = h->P.B, ncost = h->P.ncost, n = h->P.n, m = h->P.m;
    h->stage.resize((size_t)B * ncost * (n + m));
    for (int b = 0; b < B; b++)
        for (int ci = 0; ci < ncost; ci++) {
            std::memcpy(h->stage.data() + q_off(h, b, ci), h->h_costs[ci].q, sizeof(double) * n);
            std::memcpy(h->stage.data() + q_off(h, b, ci) + n, h->h_costs[ci].r, sizeof(double) * m);
        }
}
// h->stage := the rows of the constraint-data table, or every instance's shared data of every constraint when it does not exist yet
static void stage_cdata(to_handle* h) {
    if (h->P.cdata) { h->stage = h->h_cdata; return; }
    const int nm = h->P.n + h->P.m;
    h->stage.resize((size_t)h->P.B * h->P.ncdata);
    for (int b = 0; b < h->P.B; b++)
        for (const auto& c : h->h_cons)
            if (c.cdoff >= 0) con_shared_row(c, nm, h->stage.data() + cd_off(h, b, c));
}

// set_goal_state! src/problem.jl:294-310 with set_LQR_goal! (q = -Q xf; c untouched) src/cost_functions.jl:245-248
int to_set_goal_state(to_handle* h, const double* xf, int objective, int constraint) {
    JOIN(h);
    if (!h || !xf) return TO_EINVAL;
    const int n = h->P.n;
    if (objective)
        for (auto& c : h->h_costs) lqr_linear_term(c.Q, n, xf, c.q);
    if (constraint)
        for (auto& c : h->h_cons)
            if (c.kind == CON_GOAL) for (int i = 0; i < c.p; i++) c.a[i] = xf[c.inds[i]];
    h->J_valid = false;
    int rc = upload_tables(h); if (rc) return rc;
    // the later call wins: every instance takes the shared goal
    if (objective && h->P.qr) {
        stage_qr(h);
        for (int b = 0; b < h->P.B; b++)
            for (int ci = 0; ci < h->P.ncost; ci++) std::memcpy(h->stage.data() + q_off(h, b, ci), h->h_costs[ci].q, sizeof(double) * n);
        rc = commit_rows(h, h->h_qr, h->P.qr); if (rc) return rc;
    }
    if (constraint && h->P.cdata) {
        stage_cdata(h);
        for (int b = 0; b < h->P.B; b++)
            for (const auto& c : h->h_cons)
                if (c.kind == CON_GOAL) std::memcpy(h->stage.data() + cd_off(h, b, c), c.a, sizeof(double) * c.p);
        rc = commit_rows(h, h->h_cdata, h->P.cdata); if (rc) return rc;
    }
    return TO_OK;
}
// set_goal_state! per instance: xf [B][n]
int to_set_goal_states(to_handle* h, const double* xf, int objective, int constraint) {
    JOIN(h);
    if (!h || !xf) return TO_EINVAL;
    if (h->P.model == MODEL_EXPR) return hybrid_goals(h);
    const int n = h->P.n;
    if (objective) {
        stage_qr(h);
        for (int b = 0; b < h->P.B; b++)
            for (int ci = 0; ci < h->P.ncost; ci++) lqr_linear_term(h->h_costs[ci].Q, n, xf + (size_t)b * n, h->stage.data() + q_off(h, b, ci));
        int rc = commit_rows(h, h->h_qr, h->P.qr); if (rc) return rc;
        h->J_valid = false;
    }
    if (constraint) {
        stage_cdata(h);
        for (int b = 0; b < h->P.B; b++)
            for (const auto& c : h->h_cons)
                if (c.kind == CON_GOAL) for (int i = 0; i < c.p; i++) h->stage[cd_off(h, b, c) + i] = xf[(size_t)b * n + c.inds[i]];
        int rc = commit_rows(h, h->h_cdata, h->P.cdata); if (rc) return rc;
        h->J_valid = false;
    }
    return TO_OK;
}
// update_trajectory! per instance: Xref [B][nref][n], Uref [B][nref][m], one start for the batch
int to_update_trajectories(to_handle* h, const double* Xref, const double* Uref, int32_t nref, int32_t start) {
    JOIN(h);
    if (!h || !Xref || !Uref) return TO_EINVAL;
    const int n = h->P.n, m = h->P.m, N = h->P.N;
    if (start < 1 || start - 1 + N > nref) return fail(h, TO_EDIM, "update_trajectory!: the reference is shorter than start + N - 1");
    if (h->P.model == MODEL_EXPR) return hybrid_goals(h);
    stage_qr(h);
    for (int b = 0; b < h->P.B; b++)
        for (int i = 0; i < N; i++) {                   // set_LQR_goal!(obj[i], state(Z[k]), control(Z[k])) of instance b
            const int cid = h->h_cost_index[i];
            const DevCost& c = h->h_costs[cid];
            double* row = h->stage.data() + q_off(h, b, cid);
            lqr_linear_term(c.Q, n, Xref + ((size_t)b * nref + start - 1 + i) * n, row);
            lqr_linear_term(c.R, m, Uref + ((size_t)b * nref + start - 1 + i) * m, row + n);
        }
    int rc = commit_rows(h, h->h_qr, h->P.qr); if (rc) return rc;
    h->J_valid = false; h->expanded = false; h->backward_done = false;
    return TO_OK;
}
// the linear terms of every cost of every instance: q [B][ncost][n], r [B][ncost][m] (the shared ones broadcast when none are set)
int to_get_cost_terms(to_handle* h, double* q, double* r) {
    JOIN(h);
    if (!h || !q || !r) return TO_EINVAL;
    const int n = h->P.n, m = h->P.m, ncost = h->P.ncost;
    for (int b = 0; b < h->P.B; b++)
        for (int ci = 0; ci < ncost; ci++) {
            const double* sq = h->P.qr ? h->h_qr.data() + q_off(h, b, ci) : h->h_costs[ci].q;
            const double* sr = h->P.qr ? h->h_qr.data() + q_off(h, b, ci) + n : h->h_costs[ci].r;
            std::memcpy(q + ((size_t)b * ncost + ci) * n, sq, sizeof(double) * n);
            std::memcpy(r + ((size_t)b * ncost + ci) * m, sr, sizeof(double) * m);
        }
    return TO_OK;
}
// the values of Goal constraint con of every instance: vals [B][p] (the shared ones broadcast when none are set)
int to_get_goal_values(to_handle* h, int32_t con, double* vals) {
    JOIN(h);
    if (!h || !vals) return TO_EINVAL;
    if (con < 0 || con >= (int)h->h_cons.size() || h->h_cons[con].kind != CON_GOAL) return fail(h, TO_EINVAL, "to_get_goal_values: not a Goal constraint");
    const DevCon& c = h->h_cons[con];
    for (int b = 0; b < h->P.B; b++)
        std::memcpy(vals + (size_t)b * c.p, h->P.cdata ? h->h_cdata.data() + cd_off(h, b, c) : c.a, sizeof(double) * c.p);
    return TO_OK;
}
int to_set_goal_values(to_handle* h, int32_t con, const double* vals) {
    JOIN(h);
    if (!h || !vals) return TO_EINVAL;
    if (con < 0 || con >= (int)h->h_cons.size() || h->h_cons[con].kind != CON_GOAL) return fail(h, TO_EINVAL, "to_set_goal_values: not a Goal constraint");
    if (h->P.model == MODEL_EXPR) return hybrid_goals(h);
    const DevCon& c = h->h_cons[con];
    stage_cdata(h);
    for (int b = 0; b < h->P.B; b++) std::memcpy(h->stage.data() + cd_off(h, b, c), vals + (size_t)b * c.p, sizeof(double) * c.p);
    int rc = commit_rows(h, h->h_cdata, h->P.cdata); if (rc) return rc;
    h->J_valid = false;
    return TO_OK;
}
// set_LQR_goal!(obj[k], ...) per instance with the raw terms: q [B][ncost][n], r [B][ncost][m]
int to_set_cost_terms(to_handle* h, const double* q, const double* r) {
    JOIN(h);
    if (!h || !q || !r) return TO_EINVAL;
    if (h->P.model == MODEL_EXPR) return hybrid_goals(h);
    const int n = h->P.n, m = h->P.m, ncost = h->P.ncost;
    h->stage.resize((size_t)h->P.B * ncost * (n + m));    // every row is written
    for (int b = 0; b < h->P.B; b++)
        for (int ci = 0; ci < ncost; ci++) {
            std::memcpy(h->stage.data() + q_off(h, b, ci), q + ((size_t)b * ncost + ci) * n, sizeof(double) * n);
            std::memcpy(h->stage.data() + q_off(h, b, ci) + n, r + ((size_t)b * ncost + ci) * m, sizeof(double) * m);
        }
    int rc = commit_rows(h, h->h_qr, h->P.qr); if (rc) return rc;
    h->J_valid = false; h->expanded = false; h->backward_done = false;
    return TO_OK;
}

// ---- per-instance model parameters (DevProblem::mparams) ----------------------------------------------------------
// params [B][nparams] in the order of to_spec.params.  The whole batch is checked before anything changes: a refused call leaves the rows
// (or their absence) as they were.  X is not rolled out again (set_initial_state! does not either); the next rollout, expansion, line
// search or solve integrates with the new values.
int to_set_model_params(to_handle* h, const double* params, int32_t nparams) {
    JOIN(h);
    if (!h || !params) return TO_EINVAL;
    const int model = h->P.model, B = h->P.B;
    if (model == MODEL_EXPR) return fail(h, TO_EINVAL, "per-instance model parameters are not supported on hybrid problems (their constants live in the recorded programs)");
    const int np = model_nparams(model);
    if (nparams != np)
        return fail(h, TO_EDIM, "to_set_model_params: the model takes " + std::to_string(np) + " parameters per instance, got " + std::to_string(nparams));
    std::vector<double>& rows = h->stage;
    rows.assign((size_t)B * TO_NPARAM, 0.0);
    for (int b = 0; b < B; b++) {
        double* row = rows.data() + (size_t)b * TO_NPARAM;
        for (int i = 0; i < np; i++) {
            const double v = params[(size_t)b * np + i];
            const char* pos = positive_param_name(model, i);
            if (!std::isfinite(v))
                return fail(h, TO_EINVAL, "to_set_model_params: instance " + std::to_string(b) + ", parameter " + std::to_string(i) + " is not finite");
            if (pos && !(v > 0))
                return fail(h, TO_EINVAL, "to_set_model_params: instance " + std::to_string(b) + ", parameter " + std::to_string(i) + " (" + pos + ") must be positive");
            row[i] = v;
        }
        complete_model_params(model, row);
    }
    int rc = commit_rows(h, h->h_mparams, h->P.mparams); if (rc) return rc;
    h->J_valid = false; h->expanded = false; h->backward_done = false;
    return TO_OK;
}
// params [B][nparams]: every instance's parameters (the shared ones broadcast when none are set)
int to_get_model_params(to_handle* h, double* params) {
    JOIN(h);
    if (!h || !params) return TO_EINVAL;
    const int np = model_nparams(h->P.model);
    if (np == 0) return fail(h, TO_EINVAL, "hybrid problems have no model parameter vector");
    for (int b = 0; b < h->P.B; b++)
        std::memcpy(params + (size_t)b * np, h->P.mparams ? h->h_mparams.data() + (size_t)b * TO_NPARAM : h->P.params, sizeof(double) * np);
    return TO_OK;
}

// ---- per-instance constraint data (DevProblem::cdata) ----------------------------------------------------------
int to_constraint_data_len(const to_handle* h, int32_t con, int32_t* len) {
    if (!h || !len) return TO_EINVAL;
    if (con < 0 || con >= (int)h->h_cons.size()) return TO_EINVAL;
    *len = con_data_len(h->h_cons[con], h->P.n + h->P.m);
    return TO_OK;
}
// data [B][len] of constraint con (the layout of con_shared_row).  The whole batch is checked before anything changes: a refused call leaves the
// table (or its absence) as it was.  The first call creates the table with the shared data of every constraint in every row.
int to_set_constraint_data(to_handle* h, int32_t con, const double* data) {
    JOIN(h);
    if (!h || !data) return TO_EINVAL;
    if (h->P.model == MODEL_EXPR) return fail(h, TO_EINVAL, "per-instance constraint data is not supported on hybrid problems");
    if (con < 0 || con >= (int)h->h_cons.size()) return fail(h, TO_EINVAL, "to_set_constraint_data: no constraint " + std::to_string(con));
    const DevCon& c = h->h_cons[con];
    if (c.kind == CON_GOAL) return fail(h, TO_EINVAL, "to_set_constraint_data: a Goal constraint's values are set with to_set_goal_values");
    const int nm = h->P.n + h->P.m, len = con_data_len(c, nm), B = h->P.B;
    if (len == 0) return fail(h, TO_EINVAL, "to_set_constraint_data: the data of QuatVecEq and recorded (expression) constraints stays shared");
    auto where = [](int b, int j) { return "instance " + std::to_string(b) + ", entry " + std::to_string(j); };
    for (int b = 0; b < B; b++) {
        const double* row = data + (size_t)b * len;
        if (c.kind == CON_BOUND) {   // the rows, and so p and the multiplier layout, stay those of the shared bound
            for (int j = 0; j < 2 * nm; j++) {
                const double v = row[j], s = j < nm ? c.a[j] : c.b[j - nm];
                if (std::isfinite(s) ? !std::isfinite(v) : !(v == s))
                    return fail(h, TO_EINVAL, "to_set_constraint_data: " + where(b, j) + ": BoundConstraint entries must be finite exactly where the shared "
                                              "bound is, with the same infinities");
            }
            for (int j = 0; j < nm; j++)
                if (!(row[j] >= row[nm + j]))
                    return fail(h, TO_EINVAL, "to_set_constraint_data: " + where(b, j) + ": Upper bounds must be greater than or equal to lower bounds");   // src/constraints.jl:712
        } else {
            for (int j = 0; j < len; j++)
                if (!std::isfinite(row[j])) return fail(h, TO_EINVAL, "to_set_constraint_data: " + where(b, j) + " is not finite");
            if (c.kind == CON_NORM && !(row[0] >= 0))
                return fail(h, TO_EINVAL, "to_set_constraint_data: " + where(b, 0) + ": NormConstraint value must be non-negative");   // src/constraints.jl:451
        }
    }
    stage_cdata(h);
    for (int b = 0; b < B; b++) std::memcpy(h->stage.data() + cd_off(h, b, c), data + (size_t)b * len, sizeof(double) * len);
    int rc = commit_rows(h, h->h_cdata, h->P.cdata); if (rc) return rc;
    h->J_valid = false; h->expanded = false; h->backward_done = false;
    return TO_OK;
}
// data [B][len]: constraint con's data of every instance (the shared data broadcast when none is set)
int to_get_constraint_data(to_handle* h, int32_t con, double* data) {
    JOIN(h);
    if (!h || !data) return TO_EINVAL;
    if (con < 0 || con >= (int)h->h_cons.size()) return fail(h, TO_EINVAL, "to_get_constraint_data: no constraint " + std::to_string(con));
    const DevCon& c = h->h_cons[con];
    const int nm = h->P.n + h->P.m, len = con_data_len(c, nm);
    if (len == 0) return fail(h, TO_EINVAL, "to_get_constraint_data: the constraint has no per-instance data here (Goal: to_get_goal_values)");
    std::vector<double> shared(len);
    con_shared_row(c, nm, shared.data());
    for (int b = 0; b < h->P.B; b++)
        std::memcpy(data + (size_t)b * len, h->P.cdata ? h->h_cdata.data() + cd_off(h, b, c) : shared.data(), sizeof(double) * len);
    return TO_OK;
}

// ---- kernel 1 ---------------------------------------------------------------------------------------------
int to_update_trajectory(to_handle* h, const double* Xref, const double* Uref, int32_t nref, int32_t start) {
    JOIN(h);
    if (!h || !Xref || !Uref) return TO_EINVAL;
    const int n = h->P.n, m = h->P.m, N = h->P.N;
    if (start < 1 || start - 1 + N > nref) return fail(h, TO_EDIM, "update_trajectory!: the reference is shorter than start + N - 1");
    for (int i = 0; i < N; i++) {                       // set_LQR_goal!(obj[i], state(Z[k]), control(Z[k]))
        DevCost& c = h->h_costs[h->h_cost_index[i]];
        lqr_linear_term(c.Q, n, Xref + (size_t)(start - 1 + i) * n, c.q);
        lqr_linear_term(c.R, m, Uref + (size_t)(start - 1 + i) * m, c.r);
    }
    h->J_valid = false; h->expanded = false; h->backward_done = false;
    int rc = upload_tables(h); if (rc) return rc;
    if (!h->P.qr) return TO_OK;
    stage_qr(h);
    for (int b = 0; b < h->P.B; b++)                    // the later call wins: every instance takes the shared reference
        for (int i = 0; i < N; i++) {
            const int cid = h->h_cost_index[i];
            std::memcpy(h->stage.data() + q_off(h, b, cid), h->h_costs[cid].q, sizeof(double) * n);
            std::memcpy(h->stage.data() + q_off(h, b, cid) + n, h->h_costs[cid].r, sizeof(double) * m);
        }
    return commit_rows(h, h->h_qr, h->P.qr);
}
int to_shift_trajectory(to_handle* h, int32_t steps) {
    JOIN(h);
    if (!h || steps < 0) return TO_EINVAL;
    if (steps == 0) return TO_OK;
    if (steps > h->P.N - 1) steps = h->P.N - 1;
    CU(h, launch_shift_traj(h->P, steps, h->stream)); h->launches++;
    for (int k = 0; k < steps; k++) h->t0 += h->h_dt[k];
    h->J_valid = false; h->expanded = false; h->backward_done = false;
    return TO_OK;
}
int to_rollout(to_handle* h) {
    JOIN(h);
    if (!h) return TO_EINVAL;
    CU(h, launch_rollout(h->P, h->stream)); h->launches++;
    h->J_valid = false; h->expanded = false; h->backward_done = false;
    return TO_OK;
}
// the records' cost + AL expansion comes from the host-built term table (common.cuh ExpTab) when the Goal / Bound rows fit it:
// <= 3 rows per z entry, knot indices < 4095, < 128 rows per knot; otherwise k_expansion_rec walks the descriptors
static bool rec_fused(const DevProblem& P) { return P.frag && P.max_terms_per_z <= 3 && P.N < 4095 && P.max_p_knot < 128; }
// the record path (k_riccati_frag) unless to_options.backward_kernel forces a shared-memory kernel: 3 generic DFMA kernel on the full
// expansion, 5 tensor kernel on the compact expansion
static bool record_path(const DevProblem& P) { return P.frag && P.opt.pad != 3 && P.opt.pad != 5; }
int to_expand(to_handle* h) {
    JOIN(h);
    if (!h) return TO_EINVAL;
    { PhaseScope ps(h, TO_PHASE_EXPAND); CU(h, launch_expand(h->P, h->stream)); if (h->P.lie) { CU(h, launch_expand_lie(h->P, h->stream)); h->launches++; } }
    h->launches++; h->phase_launches[TO_PHASE_EXPAND]++;
    h->expanded = true; h->backward_done = false;
    return TO_OK;
}
int to_get_dynamics_jacobians(to_handle* h, double* AB) {
    JOIN(h);
    if (!h || !AB) return TO_EINVAL;
    if (!h->expanded) return fail(h, TO_ESTATE, "to_get_dynamics_jacobians before to_expand");
    const size_t cnt = (size_t)h->P.B * (h->P.N - 1) * h->P.n * (h->P.n + h->P.m);
    int rc = ensure_scratch(h, cnt * sizeof(double)); if (rc) return rc;
    CU(h, launch_export_ab(h->P, (double*)h->scratch.ptr, h->stream)); h->launches++;
    CU(h, cudaMemcpyAsync(AB, h->scratch.ptr, cnt * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    return TO_OK;
}

// ---- kernel 2 ---------------------------------------------------------------------------------------------
static int run_to_host(to_handle* h, size_t count, double* host, cudaError_t (*fn)(to_handle*, double*)) {
    int rc = ensure_scratch(h, count * sizeof(double)); if (rc) return rc;
    CU(h, fn(h, (double*)h->scratch.ptr)); h->launches++;
    CU(h, cudaMemcpyAsync(host, h->scratch.ptr, count * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    return TO_OK;
}
int to_cost(to_handle* h, double* J) {
    JOIN(h);
    if (!h || !J) return TO_EINVAL;
    return run_to_host(h, h->P.B, J, [](to_handle* hh, double* d) { return launch_cost(hh->P, d, nullptr, hh->stream); });
}
int to_cost_knots(to_handle* h, double* Jk) {
    JOIN(h);
    if (!h || !Jk) return TO_EINVAL;
    return run_to_host(h, (size_t)h->P.B * h->P.N, Jk, [](to_handle* hh, double* d) { return launch_cost(hh->P, nullptr, d, hh->stream); });
}
int to_cost_gradient(to_handle* h, double* grad) {
    JOIN(h);
    if (!h || !grad) return TO_EINVAL;
    return run_to_host(h, (size_t)h->P.B * h->P.N * (h->P.n + h->P.m), grad, [](to_handle* hh, double* d) { return launch_cost_gradient(hh->P, d, hh->stream); });
}
int to_cost_hessian(to_handle* h, double* hess) {
    JOIN(h);
    if (!h || !hess) return TO_EINVAL;
    const int nm = h->P.n + h->P.m;
    return run_to_host(h, (size_t)h->P.B * h->P.N * nm * nm, hess, [](to_handle* hh, double* d) { return launch_cost_hessian(hh->P, d, hh->stream); });
}
int to_al_expansion(to_handle* h, double* grad, double* hess) {
    JOIN(h);
    if (!h || !grad || !hess) return TO_EINVAL;
    const int nm = h->P.n + h->P.m;
    const size_t ng = (size_t)h->P.B * h->P.N * nm, nh = ng * nm;
    int rc = ensure_scratch(h, (ng + nh) * sizeof(double)); if (rc) return rc;
    double* dg = (double*)h->scratch.ptr; double* dh = dg + ng;
    CU(h, launch_al_expansion(h->P, dg, dh, h->stream)); h->launches++;
    CU(h, cudaMemcpyAsync(grad, dg, ng * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    CU(h, cudaMemcpyAsync(hess, dh, nh * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    return TO_OK;
}
int to_eval_constraints(to_handle* h, int32_t con, double* vals) {
    JOIN(h);
    if (!h || !vals) return TO_EINVAL;
    if (con < 0 || con >= (int)h->h_cons.size()) return fail(h, TO_EINVAL, "constraint index out of range");
    const DevCon& c = h->h_cons[con];
    const size_t cnt = (size_t)h->P.B * (c.last - c.first + 1) * c.p;
    int rc = ensure_scratch(h, cnt * sizeof(double)); if (rc) return rc;
    CU(h, launch_eval_constraints(h->P, con, (double*)h->scratch.ptr, h->stream)); h->launches++;
    CU(h, cudaMemcpyAsync(vals, h->scratch.ptr, cnt * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    return TO_OK;
}
int to_constraint_jacobians(to_handle* h, int32_t con, double* jac) {
    JOIN(h);
    if (!h || !jac) return TO_EINVAL;
    if (con < 0 || con >= (int)h->h_cons.size()) return fail(h, TO_EINVAL, "constraint index out of range");
    const DevCon& c = h->h_cons[con];
    const size_t cnt = (size_t)h->P.B * (c.last - c.first + 1) * c.p * (h->P.n + h->P.m);
    int rc = ensure_scratch(h, cnt * sizeof(double)); if (rc) return rc;
    CU(h, launch_constraint_jacobians(h->P, con, (double*)h->scratch.ptr, h->stream)); h->launches++;
    CU(h, cudaMemcpyAsync(jac, h->scratch.ptr, cnt * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    return TO_OK;
}
int to_constraint_hessians(to_handle* h, int32_t con, const double* lambda, double* H) {
    JOIN(h);
    if (!h || !H) return TO_EINVAL;
    if (con < 0 || con >= (int)h->h_cons.size()) return fail(h, TO_EINVAL, "constraint index out of range");
    const DevCon& c = h->h_cons[con];
    const int len = c.last - c.first + 1, w = h->P.n + h->P.m;
    const size_t nh = (size_t)h->P.B * len * w * w, nl = (size_t)h->P.B * len * c.p;
    int rc = ensure_scratch(h, (nh + nl) * sizeof(double)); if (rc) return rc;
    double* dH = (double*)h->scratch.ptr; double* dl = dH + nh;
    if (lambda) CU(h, cudaMemcpyAsync(dl, lambda, nl * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    CU(h, launch_constraint_hessians(h->P, con, len, lambda ? dl : nullptr, dH, h->stream)); h->launches++;
    CU(h, cudaMemcpyAsync(H, dH, nh * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    return TO_OK;
}
static int ensure_merit(to_handle* h) {
    if (h->J_valid) return TO_OK;
    CU(h, launch_merit(h->P, h->P.J, h->d_viol, h->stream)); h->launches++;
    h->J_valid = true;
    return TO_OK;
}
int to_merit(to_handle* h, double* J) {
    JOIN(h);
    if (!h || !J) return TO_EINVAL;
    int rc = ensure_merit(h); if (rc) return rc;
    CU(h, cudaMemcpyAsync(J, h->P.J, sizeof(double) * h->P.B, cudaMemcpyDeviceToHost, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    return TO_OK;
}
int to_max_violation(to_handle* h, double* v) {
    JOIN(h);
    if (!h || !v) return TO_EINVAL;
    CU(h, launch_merit(h->P, h->P.J, h->d_viol, h->stream)); h->launches++;
    h->J_valid = true;
    CU(h, cudaMemcpyAsync(v, h->d_viol, sizeof(double) * h->P.B, cudaMemcpyDeviceToHost, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    return TO_OK;
}

static int cone_call(to_handle* h, int32_t cone, int32_t p, int32_t count, const double* x, const double* b, double* out, int mode) {
    DeviceGuard device_guard(h);
    if (!h || !x || !out || (mode == 2 && !b)) return TO_EINVAL;
    if (p < 1 || p > TO_MAXP || count < 1) return fail(h, TO_EINVAL, "cone op: p must be in 1..32 and count >= 1");
    if (cone < 0 || cone > CONE_POSITIVE_ORTHANT) return fail(h, TO_EINVAL, "unknown cone");
    const size_t nx = (size_t)count * p, nout = mode == 0 ? nx : nx * p;
    int rc = ensure_scratch(h, (2 * nx + nout) * sizeof(double)); if (rc) return rc;
    double* dx = (double*)h->scratch.ptr; double* db = dx + nx; double* dout = db + nx;
    CU(h, cudaMemcpyAsync(dx, x, nx * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    if (mode == 2) CU(h, cudaMemcpyAsync(db, b, nx * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    CU(h, cudaMemsetAsync(h->d_err, 0, sizeof(int), h->stream));
    if (mode == 0) CU(h, launch_projection(cone, p, count, dx, dout, h->d_err, h->stream));
    else if (mode == 1) CU(h, launch_grad_projection(cone, p, count, dx, dout, h->d_err, h->stream));
    else CU(h, launch_hess_projection(cone, p, count, dx, db, dout, h->d_err, h->stream));
    h->launches++;
    int err = 0;
    CU(h, cudaMemcpyAsync(out, dout, nout * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    CU(h, cudaMemcpyAsync(&err, h->d_err, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    if (err) return fail(h, TO_ECONE, "Invalid second-order cone projection");   // src/cones.jl:91,124
    return TO_OK;
}
int to_projection(to_handle* h, int32_t cone, int32_t p, int32_t count, const double* x, double* px) { return cone_call(h, cone, p, count, x, nullptr, px, 0); }
int to_grad_projection(to_handle* h, int32_t cone, int32_t p, int32_t count, const double* x, double* J) { return cone_call(h, cone, p, count, x, nullptr, J, 1); }
int to_hess_projection(to_handle* h, int32_t cone, int32_t p, int32_t count, const double* x, const double* b, double* H) { return cone_call(h, cone, p, count, x, b, H, 2); }

// ---- kernel 3 + forward pass --------------------------------------------------------------------------------
static int solver_supported(to_handle* h) {
    // Goal / Bound rows are handled lane-resident; any other kind goes through the warp-cooperative general path of
    // k_riccati (DFMA variant) and the pointer-based rollout, which take up to 16 rows per constraint and knot.
    for (const auto& c : h->h_cons)
        if (!c.diagonal && c.p > 16)
            return fail(h, TO_ESTATE, "the solver kernels take at most 16 rows per general (non Goal/Bound) constraint");
    return TO_OK;
}
// lie.cu path: materialise [A_e B_e] and the (error-state) cost + AL expansion of every knot, then the dense Riccati pass
static int materialise_expansion(to_handle* h, double* EG, double* EH) {
    const DevProblem& P = h->P;
    const int nm = P.n + P.m;
    const size_t ng = (size_t)P.B * P.N * nm, nh = ng * nm;
    int rc = ensure_scratch(h, (ng + nh) * sizeof(double)); if (rc) return rc;
    double* gf = (double*)h->scratch.ptr; double* hf = gf + ng;
    CU(h, launch_al_expansion(P, gf, hf, h->stream)); h->launches++;
    CU(h, launch_error_expansion(P, gf, hf, EG, EH, h->stream)); h->launches++;
    return TO_OK;
}
static int do_backward(to_handle* h, bool costexp_done = false) {
    if (record_path(h->P)) {
        if (!costexp_done) {   // cost + AL expansion of every record: always from the current trajectory, multipliers and penalties
            PhaseScope pe(h, TO_PHASE_COSTEXP);
            if (rec_fused(h->P)) CU(h, launch_expansion_rec16(h->P, h->stream, 0));      // 16 lanes per knot, host-built term table
            else CU(h, launch_expansion_rec(h->P, h->stream));                          // more than 3 rows on one z entry: descriptor walk
            h->launches++; h->phase_launches[TO_PHASE_COSTEXP]++;
        }
        h->rec_costexp = true;     // (costexp_done: to_ilqr_step launched it, split or not)
        PhaseScope ps(h, TO_PHASE_BACKWARD);
        CU(h, launch_backward_frag(h->P, h->d_fragq, h->d_fragpool, h->d_fragerr, h->stream));
    } else if (h->P.dense_riccati) {
        PhaseScope ps(h, TO_PHASE_BACKWARD);
        if (h->P.frag) { CU(h, launch_export_abe(h->P, h->stream)); h->launches++; }     // the shared-memory kernels read P.ABe
        DevProblem Q = h->P;
        Q.compact = (h->P.compact && h->P.opt.pad != 3) ? 1 : 0;      // backward_kernel = 3: the generic (DFMA, full expansion) kernel
        if (Q.compact) { CU(h, launch_expansion_compact(Q, h->stream)); h->launches++; }
        else { int rc = materialise_expansion(h, h->P.EG, h->P.EH); if (rc) return rc; }
        if (!Q.lie) { CU(h, launch_error_dynamics(Q, h->stream)); h->launches++; }   // error state: [A_e B_e] comes from k_expand_lie
        CU(h, launch_backward_dense(Q, h->stream));
    } else {
        PhaseScope ps(h, TO_PHASE_BACKWARD); CU(h, launch_backward(h->P, h->d_work, h->stream));
    }
    h->launches++; h->phase_launches[TO_PHASE_BACKWARD]++;
    h->backward_done = true;
    return TO_OK;
}
static int do_forward(to_handle* h) {
    { PhaseScope ps(h, TO_PHASE_FORWARD); CU(h, launch_forward(h->P, h->stream)); }   // trials alpha = 1 .. 1/8
    h->launches++; h->phase_launches[TO_PHASE_FORWARD]++;
    { PhaseScope ps(h, TO_PHASE_LADDER); CU(h, launch_ladder(h->P, h->stream)); }     // remaining trials + commit of failures
    h->launches++; h->phase_launches[TO_PHASE_LADDER]++;

    h->expanded = false; h->backward_done = false;   // the trajectory moved
    return TO_OK;
}
int to_backward(to_handle* h, int32_t* status) {
    JOIN(h);
    if (!h) return TO_EINVAL;
    int rc = solver_supported(h); if (rc) return rc;
    if (!h->expanded) return fail(h, TO_ESTATE, "to_backward before to_expand");
    rc = do_backward(h); if (rc) return rc;
    if (status) {
        CU(h, cudaMemcpyAsync(status, h->P.bp_status, sizeof(int) * h->P.B, cudaMemcpyDeviceToHost, h->stream));
        CU(h, cudaStreamSynchronize(h->stream));
    }
    return TO_OK;
}
int to_forward(to_handle* h, double* J, double* alpha) {
    JOIN(h);
    if (!h) return TO_EINVAL;
    int rc = solver_supported(h); if (rc) return rc;
    if (!h->backward_done) return fail(h, TO_ESTATE, "to_forward before to_backward");
    rc = ensure_merit(h); if (rc) return rc;
    rc = do_forward(h); if (rc) return rc;
    if (J) CU(h, cudaMemcpyAsync(J, h->P.J, sizeof(double) * h->P.B, cudaMemcpyDeviceToHost, h->stream));
    if (alpha) CU(h, cudaMemcpyAsync(alpha, h->P.alpha, sizeof(double) * h->P.B, cudaMemcpyDeviceToHost, h->stream));
    if (J || alpha) CU(h, cudaStreamSynchronize(h->stream));
    return TO_OK;
}
// the ACTIVE count after the iteration's stopping-rule checks -> pinned slot `slot`, event ev_count[slot] (to_solve reads it one iteration later)
static int record_active_count(to_handle* h, const SolveDev& sv, int slot, cudaStream_t st) {
    CU(h, cudaMemcpyAsync(h->pin_count + slot, sv.n_active, sizeof(int), cudaMemcpyDeviceToHost, st));
    CU(h, cudaEventRecord(h->ev_count[slot], st));
    return TO_OK;
}
// One iteration of to_ilqr_step.  Per iteration: E (expansion) -> R (Riccati) -> F pass 1 (alpha = 1..1/8, ~90% of the instances) -> F pass 2 (the rest).
// Pass 2 is latency-bound and touches few instances, so it runs on a high-priority side stream followed by the
// expansion of ITS instances, concurrently with the next iteration's expansion of the instances pass 1 accepted
// (instances never interact); the Riccati pass joins both. The overlap carries across calls (h->side_pending): any
// other entry point joins the side stream first.  So with a pass 2 pending, the expansions of the late instances go on the side stream
// behind it, and the cost expansion (record path) then the dynamics expansion of the pass-1 instances on the main stream; without one,
// the dynamics expansion of every instance on the main stream.
// sv (to_solve): the stopping-rule check of every ACTIVE instance right after its line search -- for the two halves of an overlapped iteration
// on their own streams, before the next iteration's expansion of each -- and the ACTIVE count behind it (record_active_count).
static int ilqr_iteration(to_handle* h, const SolveDev* sv, int slot) {
    // (error state: only [A_e B_e] is needed by the solver kernels -- k_expand_lie; the full [A B] is produced by to_expand on request)
    auto expand = [&](cudaStream_t st, int mode) { return h->P.lie ? launch_expand_lie(h->P, st, mode) : launch_expand(h->P, st, mode); };
    bool costexp_done = false;
    const bool rec = record_path(h->P) && rec_fused(h->P);
    if (h->side_pending) {
        {
            PhaseScope pl(h, TO_PHASE_LATE, h->stream2);
            CU(h, expand(h->stream2, 2)); h->launches++;
            if (rec) { CU(h, launch_expansion_rec16(h->P, h->stream2, 2)); h->launches++; }
        }
        h->phase_launches[TO_PHASE_LATE]++;
        if (rec) {
            { PhaseScope pe(h, TO_PHASE_COSTEXP); CU(h, launch_expansion_rec16(h->P, h->stream, 1)); }
            h->launches++; h->phase_launches[TO_PHASE_COSTEXP]++;
            costexp_done = true;
        }
        CU(h, cudaEventRecord(h->ev_join, h->stream2));
    }
    { PhaseScope ps(h, TO_PHASE_EXPAND); CU(h, expand(h->stream, h->side_pending ? 1 : 0)); }
    h->launches++; h->phase_launches[TO_PHASE_EXPAND]++;
    JOIN(h);
    h->expanded = true;
    int rc = do_backward(h, costexp_done); if (rc) return rc;
    { PhaseScope ps(h, TO_PHASE_FORWARD); CU(h, launch_forward(h->P, h->stream)); }
    h->launches++; h->phase_launches[TO_PHASE_FORWARD]++;
    if (h->overlap) {
        // to_solve: the stopping-rule check of the instances pass 1 accepted (final for this iteration) comes before the fork, so that
        // everything ordered after ev_fork -- the late trials, the side stream's ACTIVE count -- sees its decisions
        if (sv) { CU(h, launch_solve_check(h->P, *sv, 1, h->stream)); h->launches++; }
        CU(h, cudaEventRecord(h->ev_fork, h->stream));
        CU(h, cudaStreamWaitEvent(h->stream2, h->ev_fork, 0));
        { PhaseScope ps(h, TO_PHASE_LADDER, h->stream2); CU(h, launch_ladder(h->P, h->stream2)); }
        if (sv) { CU(h, launch_solve_check(h->P, *sv, 2, h->stream2)); h->launches++; }      // ... the others, before their expansion on the side stream
        if (sv) { int rc2 = record_active_count(h, *sv, slot, h->stream2); if (rc2) return rc2; }
        CU(h, cudaEventRecord(h->ev_join, h->stream2));
        h->side_pending = true;
    } else {
        { PhaseScope ps(h, TO_PHASE_LADDER); CU(h, launch_ladder(h->P, h->stream)); }
        if (sv) {
            CU(h, launch_solve_check(h->P, *sv, 0, h->stream)); h->launches++;
            int rc2 = record_active_count(h, *sv, slot, h->stream); if (rc2) return rc2;
        }
    }
    h->launches++; h->phase_launches[TO_PHASE_LADDER]++;
    h->expanded = false; h->backward_done = false;   // the trajectory moved
    return TO_OK;
}
int to_ilqr_step(to_handle* h, int32_t iters) {
    if (!h || iters < 0) return TO_EINVAL;
    DeviceGuard device_guard(h);
    int rc = solver_supported(h); if (rc) return rc;
    if (!h->J_valid) { rc = join_side(h); if (rc) return rc; }
    rc = ensure_merit(h); if (rc) return rc;
    for (int it = 0; it < iters; it++) { rc = ilqr_iteration(h, nullptr, 0); if (rc) return rc; }
    return TO_OK;
}
int to_al_update(to_handle* h) {
    JOIN(h);
    if (!h) return TO_EINVAL;
    if (h->P.ncon > 0) { CU(h, launch_al_update(h->P, h->stream)); h->launches++; }    // (k_al_update also restarts rho / drho)
    else {
        // no multipliers to update, but the regularisation restarts at bp_reg_initial all the same: Altro's inner solve resets it at
        // the start of every AL iteration, constrained or not
        std::vector<double> r(h->P.B, h->P.opt.bp_reg_initial);
        CU(h, cudaMemcpyAsync(h->P.rho, r.data(), sizeof(double) * h->P.B, cudaMemcpyHostToDevice, h->stream));
        CU(h, cudaMemsetAsync(h->P.drho, 0, sizeof(double) * h->P.B, h->stream));
        CU(h, cudaStreamSynchronize(h->stream));     // `r` goes out of scope
    }
    for (auto& mu : h->h_mu) mu = std::fmin(mu * h->P.opt.penalty_scaling, h->P.opt.penalty_max);
    if (!h->h_mu.empty()) CU(h, cudaMemcpyAsync(h->d_mu, h->h_mu.data(), sizeof(double) * h->h_mu.size(), cudaMemcpyHostToDevice, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    h->J_valid = false;
    return upload_exptab(h);        // the penalties are part of the table
}
int to_get_gains(to_handle* h, double* K, double* d) {
    JOIN(h);
    if (!h) return TO_EINVAL;
    if (K) CU(h, cudaMemcpyAsync(K, h->P.K, sizeof(double) * (size_t)h->P.B * (h->P.N - 1) * h->P.ne * h->P.m, cudaMemcpyDeviceToHost, h->stream));
    if (d) CU(h, cudaMemcpyAsync(d, h->P.d, sizeof(double) * (size_t)h->P.B * (h->P.N - 1) * h->P.m, cudaMemcpyDeviceToHost, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    return TO_OK;
}
// ---- solve to convergence (solve.cu; semantics in include/trajopt_b200.h and DESIGN.md 5d) ----------------------------------------------
int to_default_solve_options(to_solve_options* o) {
    if (!o) return TO_EINVAL;
    o->cost_tolerance = 1e-4; o->cost_tolerance_intermediate = 1e-3;
    o->gradient_tolerance = 10.0; o->gradient_tolerance_intermediate = 1.0;
    o->constraint_tolerance = 1e-6;
    o->iterations = 300; o->iterations_inner = 300; o->iterations_outer = 30; o->dJ_counter_limit = 10;
    return TO_OK;
}
// the solve with P.active set (to_solve clears it on every exit)
static int solve_run(to_handle* h) {
    SolveDev& S = h->solve;
    DevProblem& P = h->P;
    CU(h, launch_solve_init(P, S, h->stream)); h->launches++;      // every instance ACTIVE, rho = bp_reg_initial, counters zero
    CU(h, launch_rollout(P, h->stream)); h->launches++;
    CU(h, launch_merit(P, P.J, h->d_viol, h->stream)); h->launches++;
    h->J_valid = true;
    CU(h, launch_solve_begin(P, S, h->stream)); h->launches++;
    for (;;) {
        // inner loops: iterations are queued without waiting for each other; the ACTIVE count of iteration i - 1 (ordered after both of its
        // checks) is read while iteration i is in the queue, so one iteration in which no instance is ACTIVE (every kernel exits at once)
        // follows the last real one
        int prev = -1;
        for (int it = 0;; it++) {
            const int slot = it & 1;
            int rc = ilqr_iteration(h, &S, slot); if (rc) return rc;
            if (prev >= 0) {
                CU(h, cudaEventSynchronize(h->ev_count[prev]));
                if (h->pin_count[prev] == 0) break;
            }
            prev = slot;
            if (it > S.opt.iterations + 1) return fail(h, TO_ESTATE, "to_solve: an inner loop outlived the iteration cap");
        }
        int rc = join_side(h); if (rc) return rc;
        if (P.ncon == 0) break;                                       // no constraints: the iLQR loop decided every status
        // outer step: the WAITING instances are done or go on; the ones that go on get the dual update, the penalties of the next outer
        // iteration and a fresh merit
        CU(h, launch_solve_outer(P, S, h->stream)); h->launches++;
        CU(h, cudaMemcpyAsync(h->pin_count, S.n_active, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
        CU(h, cudaStreamSynchronize(h->stream));
        if (h->pin_count[0] == 0) break;
        CU(h, launch_al_update(P, h->stream)); h->launches++;        // ACTIVE instances only; also resets their rho / drho
        for (auto& mu : h->h_mu) mu = std::fmin(mu * P.opt.penalty_scaling, P.opt.penalty_max);
        CU(h, cudaMemcpyAsync(h->d_mu, h->h_mu.data(), sizeof(double) * h->h_mu.size(), cudaMemcpyHostToDevice, h->stream));
        CU(h, cudaStreamSynchronize(h->stream));
        rc = upload_exptab(h); if (rc) return rc;                     // the penalties are part of the table
        CU(h, launch_merit(P, P.J, h->d_viol, h->stream)); h->launches++;
        CU(h, launch_solve_begin(P, S, h->stream)); h->launches++;
    }
    return TO_OK;
}
int to_solve(to_handle* h, const to_solve_options* o, int32_t* status, int32_t* iterations, int32_t* iterations_outer, double* cost, double* dJ,
             double* gradient, double* c_max) {
    JOIN(h);
    if (!h || !o) return TO_EINVAL;
    if (!(o->cost_tolerance > 0) || !(o->cost_tolerance_intermediate > 0) || !(o->gradient_tolerance > 0) || !(o->gradient_tolerance_intermediate > 0) ||
        !(o->constraint_tolerance > 0))
        return fail(h, TO_EINVAL, "to_solve: tolerances must be positive");
    if (o->iterations < 1 || o->iterations_inner < 1 || o->iterations_outer < 1 || o->dJ_counter_limit < 0)
        return fail(h, TO_EINVAL, "to_solve: iterations, iterations_inner and iterations_outer must be positive, dJ_counter_limit non-negative");
    int rc = solver_supported(h); if (rc) return rc;
    SolveDev& S = h->solve;
    S.opt = SolveOpts{o->cost_tolerance, o->cost_tolerance_intermediate, o->gradient_tolerance, o->gradient_tolerance_intermediate, o->constraint_tolerance,
                      o->iterations, o->iterations_inner, o->iterations_outer, o->dJ_counter_limit};
    h->P.active = S.state;
    rc = solve_run(h);
    const int jrc = join_side(h);
    h->P.active = nullptr;                 // every other entry point works on every instance again
    h->J_valid = false; h->expanded = false; h->backward_done = false;   // (the merits of the instances that stopped early belong to older penalties)
    if (rc) return rc;
    if (jrc) return jrc;
    const int B = h->P.B;
    if (cost) { rc = run_to_host(h, B, cost, [](to_handle* hh, double* d) { return launch_cost(hh->P, d, nullptr, hh->stream); }); if (rc) return rc; }
    if (status) CU(h, cudaMemcpyAsync(status, S.status, sizeof(int) * B, cudaMemcpyDeviceToHost, h->stream));
    if (iterations) CU(h, cudaMemcpyAsync(iterations, S.iter, sizeof(int) * B, cudaMemcpyDeviceToHost, h->stream));
    if (iterations_outer) CU(h, cudaMemcpyAsync(iterations_outer, S.outer, sizeof(int) * B, cudaMemcpyDeviceToHost, h->stream));
    if (dJ) CU(h, cudaMemcpyAsync(dJ, S.dJ, sizeof(double) * B, cudaMemcpyDeviceToHost, h->stream));
    if (gradient) CU(h, cudaMemcpyAsync(gradient, S.grad, sizeof(double) * B, cudaMemcpyDeviceToHost, h->stream));
    if (c_max) CU(h, cudaMemcpyAsync(c_max, S.cmax, sizeof(double) * B, cudaMemcpyDeviceToHost, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    return TO_OK;
}
// ---- Lie-group error state (lie.cu) ---------------------------------------------------------------------------
int to_backward_algebra(const to_handle* h, int32_t* variant) {
    if (!h || !variant) return TO_EINVAL;
    *variant = record_path(h->P) ? 1 : 0;
    return TO_OK;
}
static_assert(TO_LS_GENERIC == KC_LS_GENERIC && TO_LS_FAST == KC_LS_FAST && TO_LS_COMPACT == KC_LS_COMPACT, "to_linesearch_loop");
static_assert(TO_BK_THREAD == KC_BK_THREAD && TO_BK_WARP_MMA == KC_BK_WARP_MMA && TO_BK_WARP_DFMA == KC_BK_WARP_DFMA && TO_BK_FRAGMENT == KC_BK_FRAGMENT &&
              TO_BK_DENSE_MMA == KC_BK_DENSE_MMA && TO_BK_DENSE_DFMA == KC_BK_DENSE_DFMA, "to_backward_kernel");
int to_kernel_choice(const to_handle* h, int32_t* choice) {
    if (!h || !choice) return TO_EINVAL;
    DeviceGuard device_guard(h);     // the SM count (riccati_small_supported) and the resident warps are those of the handle's device
    const DevProblem& P = h->P;
    const int ls = linesearch_path(P);
    const int bk = record_path(P) ? KC_BK_FRAGMENT : backward_kernel_of(P);   // do_backward
    choice[TO_CHOICE_LINESEARCH] = ls;
    choice[TO_CHOICE_COST_CACHED] = (ls != KC_LS_GENERIC && linesearch_costs_cached(P)) ? 1 : 0;
    choice[TO_CHOICE_BACKWARD] = bk;
    choice[TO_CHOICE_FASTAL] = ((bk == KC_BK_WARP_MMA || bk == KC_BK_WARP_DFMA) && riccati_fastal(P)) ? 1 : 0;
    choice[TO_CHOICE_REC_FUSED] = (record_path(P) && rec_fused(P)) ? 1 : 0;
    choice[TO_CHOICE_LATE_LIST] = P.late_list ? 1 : 0;
    choice[TO_CHOICE_INST_FORWARD] = inst_forward(P) ? 1 : 0;     // launch_pass
    choice[TO_CHOICE_INST_BACKWARD] = inst_backward(P) ? 1 : 0;   // k_riccati, k_riccati_small, k_expansion_rec(16b), k_expansion_compact,
                                                                  // k_al_expansion, k_al_update, k_cost, k_eval_constraints, k_constraint_jacobians
    choice[TO_CHOICE_RESIDENT] = bk == KC_BK_FRAGMENT ? frag_resident_warps() : 0;
    return TO_OK;
}
int to_error_state_dim(const to_handle* h, int32_t* ne) {
    if (!h || !ne) return TO_EINVAL;
    *ne = h->P.ne;
    return TO_OK;
}
int to_state_diff(to_handle* h, const double* Xbar, double* dx) {
    JOIN(h);
    if (!h || !Xbar || !dx) return TO_EINVAL;
    const size_t nin = (size_t)h->P.B * h->P.N * h->P.n, nout = (size_t)h->P.B * h->P.N * h->P.ne;
    int rc = ensure_scratch(h, (nin + nout) * sizeof(double)); if (rc) return rc;
    double* din = (double*)h->scratch.ptr; double* dout = din + nin;
    CU(h, cudaMemcpyAsync(din, Xbar, nin * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    CU(h, launch_state_diff(h->P, din, dout, h->stream)); h->launches++;
    CU(h, cudaMemcpyAsync(dx, dout, nout * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    return TO_OK;
}
int to_get_error_dynamics(to_handle* h, double* ABe) {
    JOIN(h);
    if (!h || !ABe) return TO_EINVAL;
    if (!h->expanded) return fail(h, TO_ESTATE, "to_get_error_dynamics before to_expand");
    if (!h->P.dense_riccati) return to_get_dynamics_jacobians(h, ABe);     // no error state: [A_e B_e] = [A B]
    if (!h->P.lie) { CU(h, launch_error_dynamics(h->P, h->stream)); h->launches++; }   // error state: written by k_expand_lie in to_expand
    else if (h->P.frag) { CU(h, launch_export_abe(h->P, h->stream)); h->launches++; }    // ... as record fragments: back to col-major 12 x 16
    const size_t cnt = (size_t)h->P.B * (h->P.N - 1) * h->P.ne * (h->P.ne + h->P.m);
    CU(h, cudaMemcpyAsync(ABe, h->P.ABe, cnt * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    return TO_OK;
}
int to_error_expansion(to_handle* h, double* grad, double* hess) {
    JOIN(h);
    if (!h || !grad || !hess) return TO_EINVAL;
    if (!h->P.dense_riccati) return to_al_expansion(h, grad, hess);
    int rc = materialise_expansion(h, h->P.EG, h->P.EH); if (rc) return rc;
    const size_t nme = h->P.ne + h->P.m, ng = (size_t)h->P.B * h->P.N * nme;
    CU(h, cudaMemcpyAsync(grad, h->P.EG, ng * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    CU(h, cudaMemcpyAsync(hess, h->P.EH, ng * nme * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    return TO_OK;
}
// diagnostic: the cost + AL expansion as the record path's Riccati kernel reads it, REC[192, 240) of every (instance, knot)
int to_get_expansion_records(to_handle* h, double* out) {
    JOIN(h);
    if (!h || !out) return TO_EINVAL;
    if (!(h->P.frag && h->P.opt.pad != 3 && h->P.opt.pad != 5)) return fail(h, TO_ESTATE, "to_get_expansion_records: the handle is not on the record path");
    if (!h->rec_costexp) return fail(h, TO_ESTATE, "to_get_expansion_records before any backward pass wrote the records' expansion");
    constexpr int W = TO_REC_LEN - TO_REC_G;
    CU(h, cudaMemcpy2DAsync(out, W * sizeof(double), h->P.REC + TO_REC_G, TO_REC_LEN * sizeof(double), W * sizeof(double), (size_t)h->P.B * h->P.N,
                            cudaMemcpyDeviceToHost, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    return TO_OK;
}
static int multipliers_copy(to_handle* h, int32_t con, double* host, bool to_host) {
    JOIN(h);
    if (!h || !host) return TO_EINVAL;
    if (con < 0 || con >= (int)h->h_cons.size()) return fail(h, TO_EINVAL, "constraint index out of range");
    const DevCon& c = h->h_cons[con];
    const size_t len = (size_t)(c.last - c.first + 1) * c.p;
    if (to_host) {
        CU(h, cudaMemcpy2DAsync(host, len * sizeof(double), h->P.lambda + c.offset, (size_t)h->P.lambda_len * sizeof(double), len * sizeof(double), h->P.B, cudaMemcpyDeviceToHost, h->stream));
    } else {
        CU(h, cudaMemcpy2DAsync(h->P.lambda + c.offset, (size_t)h->P.lambda_len * sizeof(double), host, len * sizeof(double), len * sizeof(double), h->P.B, cudaMemcpyHostToDevice, h->stream));
        h->J_valid = false;
    }
    CU(h, cudaStreamSynchronize(h->stream));
    return TO_OK;
}
int to_get_multipliers(to_handle* h, int32_t con, double* lambda) { return multipliers_copy(h, con, lambda, true); }
int to_set_multipliers(to_handle* h, int32_t con, const double* lambda) { return multipliers_copy(h, con, const_cast<double*>(lambda), false); }
int to_get_penalty(to_handle* h, int32_t con, double* mu) {
    JOIN(h);
    if (!h || !mu || con < 0 || con >= (int)h->h_mu.size()) return TO_EINVAL;
    *mu = h->h_mu[con];
    return TO_OK;
}
int to_set_penalty(to_handle* h, int32_t con, double mu) {
    JOIN(h);
    if (!h || con < 0 || con >= (int)h->h_mu.size() || !(mu > 0)) return TO_EINVAL;
    h->h_mu[con] = mu;
    CU(h, cudaMemcpyAsync(h->d_mu, h->h_mu.data(), sizeof(double) * h->h_mu.size(), cudaMemcpyHostToDevice, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    h->J_valid = false;
    return upload_exptab(h);
}
int to_get_solver_state(to_handle* h, double* rho, double* dV, double* alpha, int32_t* ls_iters, int32_t* bp_status) {
    JOIN(h);
    if (!h) return TO_EINVAL;
    const int B = h->P.B;
    if (rho) CU(h, cudaMemcpyAsync(rho, h->P.rho, sizeof(double) * B, cudaMemcpyDeviceToHost, h->stream));
    if (dV) CU(h, cudaMemcpyAsync(dV, h->P.dV, sizeof(double) * 2 * B, cudaMemcpyDeviceToHost, h->stream));
    if (alpha) CU(h, cudaMemcpyAsync(alpha, h->P.alpha, sizeof(double) * B, cudaMemcpyDeviceToHost, h->stream));
    if (ls_iters) CU(h, cudaMemcpyAsync(ls_iters, h->P.ls_iters, sizeof(int) * B, cudaMemcpyDeviceToHost, h->stream));
    if (bp_status) CU(h, cudaMemcpyAsync(bp_status, h->P.bp_status, sizeof(int) * B, cudaMemcpyDeviceToHost, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    return TO_OK;
}

// ---- multi-GPU / measurement plumbing -----------------------------------------------------------------------
int to_reduce_merit(to_handle* h) {
    JOIN(h);
    if (!h) return TO_EINVAL;
    int rc = ensure_merit(h); if (rc) return rc;      // J and viol are kept current by the line search; recomputed only after edits
    CU(h, launch_reduce_merit(h->P, h->d_viol, h->d_merit2, h->stream)); h->launches++;
    return TO_OK;
}
int to_reduce_merit_async(to_handle* h, void* consumer_stream) {
    if (!h) return TO_EINVAL;
    DeviceGuard device_guard(h);
    cudaStream_t cs = (cudaStream_t)consumer_stream;
    cudaStream_t on = h->stream;
    if (h->side_pending && h->J_valid) {
        // the late line-search trials are still in flight on the side stream: reduce behind them, leave the main stream alone
        on = h->stream2;
    } else {
        int jrc = join_side(h); if (jrc) return jrc;
        int rc = ensure_merit(h); if (rc) return rc;
    }
    CU(h, cudaEventRecord(h->ev_cons, cs));                 // the consumer's earlier reads of the buffer come first
    CU(h, cudaStreamWaitEvent(on, h->ev_cons, 0));
    CU(h, launch_reduce_merit(h->P, h->d_viol, h->d_merit2, on)); h->launches++;
    CU(h, cudaEventRecord(h->ev_merit, on));
    if (on == h->stream2) CU(h, cudaEventRecord(h->ev_join, h->stream2));   // later joins cover the reduction too
    CU(h, cudaStreamWaitEvent(cs, h->ev_merit, 0));
    return TO_OK;
}
int to_merit_device_ptr(to_handle* h, void** ptr) {
    if (!h || !ptr) return TO_EINVAL;
    *ptr = h->d_merit2;
    return TO_OK;
}
int to_set_phase_timing(to_handle* h, int enable) {
    if (!h) return TO_EINVAL;
    h->timing = enable != 0;
    return TO_OK;
}
int to_get_phase_times(to_handle* h, double* ms, int64_t* launches, int reset) {
    DeviceGuard device_guard(h);
    if (!h) return TO_EINVAL;
    CU(h, cudaStreamSynchronize(h->stream));
    for (auto& e : h->pending) {
        float t = 0;
        if (cudaEventElapsedTime(&t, e.a, e.b) == cudaSuccess) h->phase_ms[e.phase] += t;
        h->pool.push_back(e.a); h->pool.push_back(e.b);
    }
    h->pending.clear();
    for (int i = 0; i < TO_PHASE_COUNT; i++) {
        if (ms) ms[i] = h->phase_ms[i];
        if (launches) launches[i] = h->phase_launches[i];
        if (reset) { h->phase_ms[i] = 0; h->phase_launches[i] = 0; }
    }
    return TO_OK;
}
int64_t to_launch_count(const to_handle* h) { return h ? h->launches : 0; }
// SURVEY.md 8(d): E=(XU+AB+HES)w, R=(AB+XU+KD+Lambda+HES)w, F=(2XU+KD+Lambda)w+8 ; HES=0 (LQR costs are never materialised)
int to_algorithmic_bytes(const to_handle* h, int64_t* E, int64_t* R, int64_t* F) {
    if (!h) return TO_EINVAL;
    const int64_t n = h->P.n, m = h->P.m, N = h->P.N, w = 8;
    const int64_t ne = h->P.ne;
    const int64_t XU = (n + m) * N, AB = n * (n + m) * (N - 1), KD = m * (ne + 1) * (N - 1), L = h->P.lambda_len;
    // materialised expansion (lie.cu): HES = per-knot gradient + Hessian in the (error) state, [A_e B_e] written once and read once
    const int64_t HES = h->P.dense_riccati ? ((ne + m) * (ne + m) + (ne + m)) * N : 0;
    const int64_t ABe = h->P.dense_riccati ? ne * (ne + m) * (N - 1) : 0;
    if (E) *E = (XU + AB) * w;
    // backward phase of the lie.cu path = expansion kernels + Riccati kernel: the expansion is written once and read once.
    //   compact (error state, diagonal costs, Goal/Bound): XU + L -> EC (40 per knot) ; EC + [A_e B_e] -> K, d
    //   generic: full-state expansion (scratch) -> error-state expansion (HES) ; [A B] -> [A_e B_e] unless k_expand_lie wrote it
    const int64_t EC = (int64_t)TO_EC_LEN * N, HESF = ((n + m) * (n + m) + (n + m)) * N;
    if (R) {
        // record path (riccati_frag.cu): the Riccati kernel is timed alone; its compulsory inputs are [A_e B_e], the trajectory and the
        // multipliers (what the expansion it consumes is made of), its outputs the gains -- SURVEY 8(d)'s R column on the error state
        if (h->P.frag && h->P.opt.pad != 3 && h->P.opt.pad != 5) *R = (ABe + XU + KD + L) * w;
        else if (h->P.compact && h->P.opt.pad != 3) *R = (XU + L + 2 * EC + ABe + KD) * w;
        else if (h->P.dense_riccati) *R = (XU + L + 2 * HESF + 2 * HES + (h->P.lie ? 0 : AB + ABe) + ABe + KD) * w;
        else *R = (AB + XU + KD + L) * w;
    }
    if (E && h->P.lie) *E = (XU + ABe) * w;     // k_expand_lie writes [A_e B_e] only
    if (F) *F = (2 * XU + KD + L) * w + 8;
    return TO_OK;
}

}  // extern "C"
