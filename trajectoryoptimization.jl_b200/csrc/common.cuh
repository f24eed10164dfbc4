// common.cuh -- shared device/host definitions of the H100 (sm_90a) batched trajectory-optimization hot path.
//
// Data layout in HBM (all fp64, instance-major so one instance's per-knot blocks are contiguous and can be
// streamed with 1-D bulk TMA copies by the warp that owns the instance):
//   X   [NBUF][B][N][n]       trajectory ring (cur[b] selects the live buffer; the line search writes the candidate
//   U   [NBUF][B][N-1][m]     of trial j into buffer (cur[b]+1+j) % NBUF and acceptance just moves cur[b])
//   AB  [B][N-1][n][LDAB]     discrete dynamics Jacobian [A B], ROW-major, row stride LDAB = n+m rounded up to
//                             even (16-byte rows for bulk copies / LDS.128); pad column = 0
//   K   [B][N-1][n][m]        feedback gains, m x n column-major (Julia layout)      d [B][N-1][m]
//   lambda [B][lambda_len]    multipliers, per constraint: [knot in range][p]
#pragma once
#include <cuda_runtime.h>
#include <cstdlib>
#include <stdint.h>

#define TO_MAXN 16
#define TO_MAXM 8
#define TO_MAXNM (TO_MAXN + TO_MAXM)
#define TO_MAXCON 8
#define TO_MAXP 32          // rows of one general constraint at one knot (dense Jacobian / cone scratch is sized by it)
#define TO_MAXPV (2 * TO_MAXNM)   // rows of a Goal / Bound constraint: a BoundConstraint with every entry of z bounded on both sides
#define TO_CON_A 256
#define TO_EXPR_LEN 128      // == TO_EXPR_MAXLEN / TO_EXPR_MAXCONST of include/trajopt_b200.h
#define TO_EXPR_CONST 64
#define TO_EC_LEN 40
#define TO_NBUF 9            // trajectory buffers per instance: the live one + 8 line-search candidates

// reference enums (mirrors include/trajopt_b200.h)
enum { MODEL_DOUBLE_INTEGRATOR = 0, MODEL_CARTPOLE = 1, MODEL_QUADROTOR = 2, MODEL_ACROBOT = 3, MODEL_EXPR = 4 };
enum { CONE_ZERO = 0, CONE_NEGATIVE_ORTHANT = 1, CONE_SECOND_ORDER = 2, CONE_IDENTITY = 3, CONE_POSITIVE_ORTHANT = 4 };
enum { RULE_EULER = 1, RULE_RK2 = 2, RULE_RK3 = 3, RULE_RK4 = 4 };   // to_integration
enum { CON_GOAL = 0, CON_BOUND = 1, CON_LINEAR = 2, CON_CIRCLE = 3, CON_SPHERE = 4, CON_NORM = 5, CON_COLLISION = 6, CON_QUATVEC = 7, CON_EXPR = 8 };

// QuadraticCostFunction (reference src/cost_functions.jl:326-347, :417-454); dense storage + diagonal copy
struct DevCost {
    int diag, terminal, zeroH;
    int cwoff;                     // offset of the cost's weights in an instance's row of DevProblem::cw (-1: EXPR, no weights)
    double c;
    double Qd[TO_MAXN], Rd[TO_MAXM];
    double q[TO_MAXN], r[TO_MAXM];
    double Q[TO_MAXN * TO_MAXN];   // n*n col-major (stride n)
    double R[TO_MAXM * TO_MAXM];   // m*m col-major (stride m)
    double H[TO_MAXM * TO_MAXN];   // m*n col-major (stride m)
    // DiagonalQuatCost (reference src/lie_costs.jl:33-95): + w min(1 + q_ref'p, 1 - q_ref'p), p = x[q_ind]
    int quat, q_ind[4], pad2[3];
    double w, q_ref[4];
    // user cost recorded as a straight-line program (to_cost_spec EXPR; reference RD.@autodiff CostFunction, docs/src/costfunction_interface.md:30-50)
    int expr, prog_len, pad3[2];
    int prog[3 * TO_EXPR_LEN];
    double pconst[TO_EXPR_CONST];
};

// AbstractConstraint descriptor (reference src/constraints.jl); `diagonal` constraints (Goal, Bound) have a
// +-1 selector Jacobian and get the fast AL path inside the Riccati / forward kernels.
struct DevCon {
    int kind, first, last, p, sense, offset, ninds, flag;   // first/last: 1-based inclusive knots; offset into lambda
    int diagonal;
    int n_max, n_min;
    int pad;
    int inds[TO_MAXNM];      // GOAL: state index per row (0-based); NORM: indices into z; CIRCLE/SPHERE: xi,yi,zi
    int a_max[TO_MAXNM];     // BOUND: z index of each finite upper bound (row i)        src/constraints.jl:675
    int a_min[TO_MAXNM];     // BOUND: z index of each finite lower bound (row n_max+i)  src/constraints.jl:676
    int row_max[TO_MAXNM];   // BOUND: row of z_j's upper bound or -1 ; GOAL: row of x_j or -1
    int row_min[TO_MAXNM];   // BOUND: row of z_j's lower bound or -1
    double val;
    double a[TO_CON_A];      // GOAL xf[p] | BOUND z_max[n+m] | LINEAR A[p x w] col-major | CIRCLE/SPHERE xc[p]
    double b[TO_MAXP];       // BOUND z_min[n+m] | LINEAR b[p] | yc[p]
    double c3[TO_MAXP];      // SPHERE zc[p]
    double rad[TO_MAXP];
    // CON_EXPR: user constraint recorded as a program (outputs = the last p instructions); to_constraint_spec TO_CON_EXPR
    int prog_len;
    int cdoff;               // GOAL / BOUND / LINEAR / CIRCLE / SPHERE / NORM / COLLISION: offset of its data in an instance's row of DevProblem::cdata
    int pad4[2];
    int prog[3 * TO_EXPR_LEN];
    double pconst[TO_EXPR_CONST];
};

// Table of the Goal / Bound rows acting on each full-state entry z_i (compact problems), built on the host whenever the constraint
// tables or the penalties change, read by the dynamics expansion kernel for the records' cost + AL expansion (rollout.cu).
// One AL term on z_i:  c = sign (z_i - bound);  Goal: equality (always active), Bound: inequality.
#define TO_EXP_MAXT 3
struct ExpTab {
    double nms[TO_EXP_MAXT][TO_MAXNM];      // -mu * sign
    double bound[TO_EXP_MAXT][TO_MAXNM];
    unsigned pkx[TO_EXP_MAXT][TO_MAXNM];    // first knot (12 bits) | last - first (12) | rows p of the constraint (7) | equality (1)
    unsigned pky[TO_EXP_MAXT][TO_MAXNM];    // lambda index of the row at knot 0
    int inst[TO_EXP_MAXT][TO_MAXNM];        // index of the term's bound in an instance's row of DevProblem::cdata; -1: no term
    int con[TO_EXP_MAXT][TO_MAXNM];         // the term's constraint (its penalty in an instance's row of DevProblem::mub); -1: no term
};

// one dynamics model of a hybrid problem (to_dynamics_spec): a recorded program, discretised with the problem's rule, or a discrete jump map
struct DevDyn {
    int n_in, m_in, n_out, discrete;
    int prog_len, pad[3];
    int prog[3 * TO_EXPR_LEN];
    double pconst[TO_EXPR_CONST];
};

struct DevOptions {
    double bp_reg_increase_factor, bp_reg_max, bp_reg_min, bp_reg_initial, bp_reg_fp;
    double ls_lower, ls_upper;
    int ls_iters, backward_kernel;   // to_options.backward_kernel (riccati.cu backward_plan)
    double max_state_value, max_control_value;
    double penalty_initial, penalty_scaling, penalty_max, dual_max;
};

// Everything a kernel needs, passed by value (lives in the kernel parameter / constant bank).
struct DevProblem {
    int model, n, m, N, B;
    int ldab;                 // row stride of AB
    int ncost, ncon, lambda_len;
    int all_diag_cost;        // every cost is a DiagonalCost
    int all_diag_con;         // every constraint is Goal/Bound
    int max_p_knot;           // largest number of constraint rows active at one knot
    int max_terms_per_z;      // largest number of Goal/Bound rows acting on one z entry
    int max_cons_knot;        // largest number of constraints active at one knot
    // Lie-group error state (to_spec.error_state; lie.cu): the solver kernels work on ne = n - 1 dimensions, the quaternion
    // x[qs..qs+3] contributing its 3-dimensional differential.  dense_riccati: the backward pass reads the per-knot expansion
    // (EG, EH) and [A_e B_e] (ABe) materialised in HBM by lie.cu instead of expanding in-kernel (error state, quaternion costs).
    int lie, ne, qs, dense_riccati;
    int compact, frag;        // compact: lie + only DiagonalCost + Goal/Bound constraints: the expansion of a knot is a
                              // gradient, a diagonal and the 3 x 3 attitude block -> EC, 40 doubles per knot instead of EG + EH (272)
                              // frag: compact problems keep [A_e B_e] + expansion as per-knot RECORDS in MMA-fragment order (REC,
                              // frag_layout.cuh) for the register-resident Riccati kernel (riccati_frag.cu); ABe / EC are then only
                              // filled on request (export, the shared-memory kernels forced by to_options.backward_kernel)
    double* EC;               // [B][N][TO_EC_LEN]: g_e(16) | diag(16) | block (0,1),(0,2),(1,2) | pad
    double* REC;              // [B][N][TO_REC_LEN] (frag)
    const ExpTab* exptab;     // (frag) see ExpTab
    const DevDyn* dyn;        // MODEL_EXPR: the models; knot k uses dyn[dyn_index[k]]
    const int* dyn_index;     // [N-1]
    double* ABe;              // [B][N-1][ne+m][ne]   ne x (ne+m) col-major
    double* EG;               // [B][N][ne+m]
    double* EH;               // [B][N][ne+m][ne+m]
    double params[16];
    DevOptions opt;
    const double* dt;         // [N-1]
    const DevCost* costs;     // [ncost]
    const int* cost_index;    // [N]
    const DevCon* cons;       // [ncon]
    const double* mu;         // [ncon] penalties
    double* x0;               // [B][n]
    double* X;                // [NBUF][B][N][n]
    double* U;                // [NBUF][B][N-1][m]
    int* cur;                 // [B] live trajectory buffer (0..NBUF-1)
    double* AB;               // [B][N-1][n][ldab]
    double* K;                // [B][N-1][n][m]
    double* d;                // [B][N-1][m]
    double* lambda;           // [B][lambda_len]
    double* rho;              // [B]
    double* drho;             // [B]
    double* dV;               // [B][2]
    double* J;                // [B] merit of the live trajectory
    double* Jc;               // [B] merit of the candidate
    double* viol;             // [B] max constraint violation of the live trajectory
    double* alpha;            // [B]
    int* bp_status;           // [B]
    int* ls_iters;            // [B]
    int* accepted;            // [B]
    int* acc1;                // [B] accepted by the first line-search pass (read by the overlapped expansion)
    int* late_list;           // [B] the instances pass 1 did not accept, in arrival order (written by pass 1, walked by the later passes)
    int* late_count;          // [1] ... and how many; late_list == nullptr: the later passes scan every instance
    size_t strideX, strideU;  // elements between the two trajectory buffers
    // to_solve (capi.cu): per-instance solve state, SOLVE_ACTIVE / SOLVE_WAITING / SOLVE_DONE.  The per-instance kernels of an iteration
    // skip every instance that is not ACTIVE, so a converged instance keeps the X, U, lambda, K, d, rho, J it stopped with.
    // nullptr outside to_solve: every instance is worked on.
    const int* active;        // [B]
    // Per-instance goals / tracking references (to_set_goal_states, to_update_trajectories, to_set_cost_terms): the linear terms of every
    // cost, per instance.  nullptr until the first per-instance call; every kernel then reads the shared DevCost::q / r.
    const double* qr;         // [B][ncost][n+m]: q | r of cost cid for instance b
    // The line search's compact problem class (forward.cu rollout_compact): one cost on every stage knot and another on the terminal
    // knot, at most one Bound with finite limits on every control and none on the state, on every stage knot, and at most one Goal, on the
    // terminal knot only.  Set at to_create (the structure of the costs and constraints never changes afterwards).
    int fwd_compact;
    // The explicit rule of the discretised dynamics (to_set_integration): TO_EULER .. TO_RK4, TO_RK4 from to_create.  The launchers of every
    // kernel that steps the dynamics dispatch on it (models.cuh TO_DISPATCH_RULE); it fills the padding in front of the next pointer.
    int integration;
    // Per-instance model parameters (to_set_model_params): [B][TO_NPARAM] in the layout of `params`, the host-computed reciprocals included.
    // nullptr until the first per-instance call; every kernel then reads the shared `params`.
    const double* mparams;
    // Per-instance constraint data (to_set_constraint_data, and the Goal values of to_set_goal_values / to_set_goal_states): row b holds, at
    // DevCon::cdoff, the data of every constraint that carries data (see con_data).  nullptr until the first call; every kernel then reads
    // the shared DevCon fields.
    const double* cdata;      // [B][ncdata]
    int ncdata;
    // Per-instance cost weights (to_set_cost_weights): row b holds, at DevCost::cwoff, the weights of every quadratic cost (see cost_data).
    // nullptr until the first call; every kernel then reads the shared DevCost fields.
    int ncw;
    const double* cw;         // [B][ncw]
    // Per-instance AL penalties (to_set_penalties): row b holds the penalty of every constraint for instance b (see penalty).  nullptr until
    // the first call; every kernel then reads the shared `mu`.  Unlike the other tables the device also writes it: k_al_update scales the
    // rows of the instances it updates, and to_solve runs each instance's outer step on the device.
    double* mub;              // [B][ncon]
    // Per-instance time steps (to_set_time_steps): row b holds the N-1 steps of instance b (see time_step).  nullptr until the first call;
    // every kernel then reads the shared `dt`.
    const double* dtb;        // [B][N-1]
};
#define TO_NPARAM 16        // slots of DevProblem::params and of a row of DevProblem::mparams (one 128-byte line)

enum { SOLVE_ACTIVE = 0, SOLVE_WAITING = 1, SOLVE_DONE = 2 };
__host__ __device__ inline bool retired(const DevProblem& P, int b) { return P.active != nullptr && P.active[b] != SOLVE_ACTIVE; }

// Which variant of a kernel family runs: INST = true when a per-instance table the family reads exists.  The only place that decides; every
// launcher and to_kernel_choice ask here.  The line search reads the linear cost terms, the model parameters, the time steps and the
// constraint data; the expansion, backward and sweep kernels the cost terms and the constraint data (none of them reads a time step); the
// dynamics kernels, the closed-form Jacobian columns included, the model parameters and the time steps.
__host__ __device__ inline bool inst_forward(const DevProblem& P) { return P.qr || P.mparams || P.cdata || P.cw || P.mub || P.dtb; }
__host__ __device__ inline bool inst_backward(const DevProblem& P) { return P.qr || P.cdata || P.cw || P.mub; }
__host__ __device__ inline bool inst_dynamics(const DevProblem& P) { return P.mparams || P.dtb; }

// The weights and linear terms of cost cid for instance b: the only place that decides between an instance's rows (DevProblem::cw for the
// weights, DevProblem::qr for the linear terms) and the descriptor, and the only way a kernel reads them.  The cost's structure (diag, zeroH,
// quat, q_ind, q_ref, the program) stays in the descriptor.  An instance's row of cw, at DevCost::cwoff, by kind:
//   DIAGONAL Qd[n] | Rd[m] | c ;  QUADRATIC Q[n*n] | R[m*m] | H[m*n] | c ;  DIAGONAL_QUAT Qd[n] | Rd[m] | c | w.
// So with the diagonal layout entry i of z reads row[i], as it does in the row of qr (q[n] | r[m]).  A diagonal row has no dense Q / R / H
// and a dense one no Qd / Rd: those fields keep the descriptor's, and every reader takes the form the cost's `diag` selects.
// INST = false is the shared path, compiled without a look at the tables; the hot kernels take INST as a template parameter and are launched
// with INST = true only when a table exists.  Every field is a pointer, c and w included, as in ConData: building the view loads nothing.
// `shared`: the descriptor's fields, or a kernel's staged copy of them (the line search's cost cache in shared memory).
struct CostData { const double *Qd, *Rd, *Q, *R, *H, *q, *r, *c, *w; };
template <bool INST>
__device__ __forceinline__ CostData cost_data(const DevProblem& P, int b, int cid, CostData shared) {
    if constexpr (INST) {
        const int n = P.n, m = P.m;
        if (P.qr) { const double* row = P.qr + ((size_t)b * P.ncost + cid) * (n + m); shared.q = row; shared.r = row + n; }
        const DevCost& c = P.costs[cid];
        if (P.cw && c.cwoff >= 0) {
            const double* row = P.cw + (size_t)b * P.ncw + c.cwoff;
            if (c.diag) { shared.Qd = row; shared.Rd = row + n; shared.c = row + n + m; shared.w = row + n + m + 1; }
            else { shared.Q = row; shared.R = row + n * n; shared.H = row + n * n + m * m; shared.c = row + n * n + m * m + m * n; }
        }
    }
    return shared;
}
__device__ __forceinline__ CostData cost_fields(const DevCost& c) { return CostData{c.Qd, c.Rd, c.Q, c.R, c.H, c.q, c.r, &c.c, &c.w}; }
template <bool INST>
__device__ __forceinline__ CostData cost_data(const DevProblem& P, int b, int cid) {
    return cost_data<INST>(P, b, cid, cost_fields(P.costs[cid]));
}
// Doubles of a cost's row of DevProblem::cw (the table above; 0 for a program cost)
__host__ __device__ inline int cost_weights_len(const DevCost& c, int n, int m) {
    if (c.expr) return 0;
    if (c.diag) return n + m + 1 + (c.quat ? 1 : 0);
    return n * n + m * m + m * n + 1;
}
// Model parameter i of instance b: the only place that decides between the rows of DevProblem::mparams and the shared vector.  A value, not a
// pointer: the shared vector lives in the kernel's parameter bank, and a pointer that may point there makes the kernel copy it to local memory.
// The kernels stage an instance's parameters with it (models.cuh stage_model_params) and run the dynamics on the copy.
template <bool INST>
__device__ __forceinline__ double model_param(const DevProblem& P, int b, int i) {
    if constexpr (INST) { if (P.mparams) return P.mparams[(size_t)b * TO_NPARAM + i]; }
    return P.params[i];
}
// The time step of knot k (0-based, k < N-1) for instance b: the only place that decides between an instance's row of DevProblem::dtb and the
// shared steps.  `shared`: P.dt, or a kernel's staged copy of it (the line search's table in shared memory), so that with INST = false a kernel
// reads the address it always read.
template <bool INST>
__device__ __forceinline__ double time_step(const DevProblem& P, int b, int k, const double* shared) {
    if constexpr (INST) { if (P.dtb) return P.dtb[(size_t)b * (P.N - 1) + k]; }
    return shared[k];
}
template <bool INST>
__device__ __forceinline__ double time_step(const DevProblem& P, int b, int k) { return time_step<INST>(P, b, k, P.dt); }
// The AL penalty of constraint ci for instance b: the only place that decides between an instance's row of DevProblem::mub and the shared
// DevProblem::mu, and the only way a kernel reads a penalty.
template <bool INST>
__device__ __forceinline__ double penalty(const DevProblem& P, int b, int ci) {
    if constexpr (INST) { if (P.mub) return P.mub[(size_t)b * P.ncon + ci]; }
    return P.mu[ci];
}
// The data of constraint ci for instance b, in the fields of DevCon it replaces: a (GOAL xf | BOUND z_max | CIRCLE / SPHERE xc), b (BOUND z_min |
// LINEAR b | yc), c3 (zc), rad (CIRCLE / SPHERE r), val (NORM val | COLLISION radius).  LINEAR's A and every other field stay shared.  The only
// place that decides between an instance's row of DevProblem::cdata and the descriptor, and the only way a kernel reads a constraint's data.
// An instance's row of cdata, at DevCon::cdoff: GOAL xf[inds], BOUND z_max[n+m] | z_min[n+m], LINEAR b[p], CIRCLE xc[p] | yc[p] | r[p],
// SPHERE xc[p] | yc[p] | zc[p] | r[p], NORM val, COLLISION radius.
// Every field is a pointer, val included: building the view loads nothing, so with INST = false it is the address arithmetic of reading the
// descriptor in place, and each value is loaded where it is used (a value field would load con.val before the stores that precede its use,
// which may alias it).  `shared`: the descriptor's fields, or a kernel's staged copy of them (the line search's tables in shared memory).
struct ConData { const double *a, *b, *c3, *rad, *val; };
template <bool INST>
__device__ __forceinline__ ConData con_data(const DevProblem& P, int b, int ci, ConData shared) {
    if constexpr (INST) {
        const DevCon& con = P.cons[ci];
        if (P.cdata && con.cdoff >= 0) {
            const double* row = P.cdata + (size_t)b * P.ncdata + con.cdoff;
            switch (con.kind) {
                case CON_GOAL: shared.a = row; break;
                case CON_BOUND: shared.a = row; shared.b = row + P.n + P.m; break;
                case CON_LINEAR: shared.b = row; break;
                case CON_CIRCLE: shared.a = row; shared.b = row + con.p; shared.rad = row + 2 * con.p; break;
                case CON_SPHERE: shared.a = row; shared.b = row + con.p; shared.c3 = row + 2 * con.p; shared.rad = row + 3 * con.p; break;
                case CON_NORM: case CON_COLLISION: shared.val = row; break;
            }
        }
    }
    return shared;
}
template <bool INST>
__device__ __forceinline__ ConData con_data(const DevProblem& P, int b, int ci) {
    const DevCon& con = P.cons[ci];
    return con_data<INST>(P, b, ci, ConData{con.a, con.b, con.c3, con.rad, &con.val});
}

__host__ __device__ inline const double* traj_X(const DevProblem& P, int buf, int b) { return P.X + buf * P.strideX + (size_t)b * P.N * P.n; }
__host__ __device__ inline const double* traj_U(const DevProblem& P, int buf, int b) { return P.U + buf * P.strideU + (size_t)b * (P.N - 1) * P.m; }
__host__ __device__ inline double* traj_Xw(const DevProblem& P, int buf, int b) { return P.X + buf * P.strideX + (size_t)b * P.N * P.n; }
__host__ __device__ inline double* traj_Uw(const DevProblem& P, int buf, int b) { return P.U + buf * P.strideU + (size_t)b * (P.N - 1) * P.m; }

// The receding-horizon shift of instance b by `steps` knots, run by the whole CTA (sweep.cu k_shift_traj, rollout.cu k_mpc_advance): the
// trajectory goes to the next ring buffer, the multipliers shift in place (thread = one row of one constraint, ascending knots: reads
// k+steps, writes k), x0 <- X[steps] (thread i writes x0[i]).  Ends with a barrier and the move of cur[b].
__device__ __forceinline__ void shift_traj_cta(const DevProblem& P, int b, int steps) {
    const int n = P.n, m = P.m, N = P.N;
    const int src = P.cur[b], dst = (src + 1) % TO_NBUF;
    const double* X = traj_X(P, src, b); const double* U = traj_U(P, src, b);
    double* Xn = traj_Xw(P, dst, b); double* Un = traj_Uw(P, dst, b);
    for (int i = threadIdx.x; i < N * n; i += blockDim.x) { int k = i / n + steps; if (k > N - 1) k = N - 1; Xn[i] = X[k * n + i % n]; }
    for (int i = threadIdx.x; i < (N - 1) * m; i += blockDim.x) { int k = i / m + steps; if (k > N - 2) k = N - 2; Un[i] = U[k * m + i % m]; }
    for (int i = threadIdx.x; i < n; i += blockDim.x) { int k = steps < N - 1 ? steps : N - 1; P.x0[(size_t)b * n + i] = X[k * n + i]; }
    double* lam = P.lambda + (size_t)b * P.lambda_len;
    for (int ci = 0; ci < P.ncon; ci++) {
        const DevCon& c = P.cons[ci];
        const int nk = c.last - c.first + 1;
        for (int r = threadIdx.x; r < c.p; r += blockDim.x)
            for (int k = 0; k + steps < nk; k++) lam[c.offset + k * c.p + r] = lam[c.offset + (k + steps) * c.p + r];
    }
    __syncthreads();
    if (threadIdx.x == 0) P.cur[b] = dst;
}

// One process may hold handles on several GPUs (to_spec.device): function attributes and occupancy are per device, so the
// launchers cache their one-time configuration per device ordinal.
#define TO_MAXDEV 64
inline int current_device_slot() { int d = 0; cudaGetDevice(&d); return (d >= 0 && d < TO_MAXDEV) ? d : 0; }

// Altro.jl regularization_update! (restated; see oracle/oracle.hpp reg_increase / reg_decrease)
__host__ __device__ inline void reg_increase(const DevOptions& o, double& rho, double& drho) {
    drho = fmax(drho * o.bp_reg_increase_factor, o.bp_reg_increase_factor);
    rho = fmax(rho * drho, o.bp_reg_min);
}
__host__ __device__ inline void reg_decrease(const DevOptions& o, double& rho, double& drho) {
    drho = fmin(drho / o.bp_reg_increase_factor, 1.0 / o.bp_reg_increase_factor);
    rho = rho * drho * ((rho * drho > o.bp_reg_min) ? 1.0 : 0.0);
}
// The regularisation ladder of a backward pass (Altro backwardpass!), for every backward kernel.
// A failed sweep: raise rho and count the restart; true when rho went past bp_reg_max, where the ladder gives up.
__host__ __device__ inline bool reg_restart(const DevOptions& o, double& rho, double& drho, int& restarts) {
    reg_increase(o, rho, drho);
    restarts++;
    return rho > o.bp_reg_max;
}
// The end of instance b's pass, called by every lane of the instance's warp (the thread kernel passes lane 0): lower rho unless the
// ladder gave up, then lane 0 stores rho, drho and bp_status = the restarts, or -1 when the ladder gave up.  solve.cu and forward.cu
// read bp_status in that encoding.
__device__ inline void reg_finish(const DevProblem& P, int b, double rho, double drho, int restarts, bool failed, int lane) {
    if (!failed) reg_decrease(P.opt, rho, drho);
    if (lane == 0) { P.rho[b] = rho; P.drho[b] = drho; P.bp_status[b] = failed ? -1 : restarts; }
}
