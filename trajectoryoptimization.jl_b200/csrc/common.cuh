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
enum { CON_GOAL = 0, CON_BOUND = 1, CON_LINEAR = 2, CON_CIRCLE = 3, CON_SPHERE = 4, CON_NORM = 5, CON_COLLISION = 6, CON_QUATVEC = 7, CON_EXPR = 8 };

// QuadraticCostFunction (reference src/cost_functions.jl:326-347, :417-454); dense storage + diagonal copy
struct DevCost {
    int diag, terminal, zeroH, pad;
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
};

// one dynamics model of a hybrid problem (to_dynamics_spec): a recorded program, RK4-discretised or a discrete jump map
struct DevDyn {
    int n_in, m_in, n_out, discrete;
    int prog_len, pad[3];
    int prog[3 * TO_EXPR_LEN];
    double pconst[TO_EXPR_CONST];
};

struct DevOptions {
    double bp_reg_increase_factor, bp_reg_max, bp_reg_min, bp_reg_initial, bp_reg_fp;
    double ls_lower, ls_upper;
    int ls_iters, pad;
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
    // Per-instance model parameters (to_set_model_params): [B][TO_NPARAM] in the layout of `params`, the host-computed reciprocals included.
    // nullptr until the first per-instance call; every kernel then reads the shared `params`.
    const double* mparams;
    // Per-instance constraint data (to_set_constraint_data, and the Goal values of to_set_goal_values / to_set_goal_states): row b holds, at
    // DevCon::cdoff, the data of every constraint that carries data (see con_data).  nullptr until the first call; every kernel then reads
    // the shared DevCon fields.
    const double* cdata;      // [B][ncdata]
    int ncdata;
};
#define TO_NPARAM 16        // slots of DevProblem::params and of a row of DevProblem::mparams (one 128-byte line)

enum { SOLVE_ACTIVE = 0, SOLVE_WAITING = 1, SOLVE_DONE = 2 };
__host__ __device__ inline bool retired(const DevProblem& P, int b) { return P.active != nullptr && P.active[b] != SOLVE_ACTIVE; }

// Which variant of a kernel family runs: INST = true when a per-instance table the family reads exists.  The only place that decides; every
// launcher and to_kernel_choice ask here.  The line search reads the linear cost terms, the model parameters and the constraint data; the
// expansion, backward and sweep kernels the cost terms and the constraint data; the dynamics kernels the model parameters alone.
__host__ __device__ inline bool inst_forward(const DevProblem& P) { return P.qr || P.mparams || P.cdata; }
__host__ __device__ inline bool inst_backward(const DevProblem& P) { return P.qr || P.cdata; }
__host__ __device__ inline bool inst_dynamics(const DevProblem& P) { return P.mparams; }

// Linear cost terms of instance b: the only place that decides between the per-instance table and the shared descriptors.
// INST = false is the shared path, compiled without a look at the tables; the hot kernels take INST as a template parameter and are
// launched with INST = true only when the tables exist.
template <bool INST>
__host__ __device__ __forceinline__ const double* inst_q(const DevProblem& P, int b, int cid) {
    if constexpr (INST) { if (P.qr) return P.qr + ((size_t)b * P.ncost + cid) * (P.n + P.m); }
    return P.costs[cid].q;
}
template <bool INST>
__host__ __device__ __forceinline__ const double* inst_r(const DevProblem& P, int b, int cid) {
    if constexpr (INST) { if (P.qr) return P.qr + ((size_t)b * P.ncost + cid) * (P.n + P.m) + P.n; }
    return P.costs[cid].r;
}
// Model parameter i of instance b: the only place that decides between the rows of DevProblem::mparams and the shared vector.  A value, not a
// pointer: the shared vector lives in the kernel's parameter bank, and a pointer that may point there makes the kernel copy it to local memory.
// The kernels stage an instance's parameters with it (models.cuh stage_model_params) and run the dynamics on the copy.
template <bool INST>
__device__ __forceinline__ double model_param(const DevProblem& P, int b, int i) {
    if constexpr (INST) { if (P.mparams) return P.mparams[(size_t)b * TO_NPARAM + i]; }
    return P.params[i];
}
// The data of constraint ci for instance b, in the fields of DevCon it replaces: a (GOAL xf | BOUND z_max | CIRCLE / SPHERE xc), b (BOUND z_min |
// LINEAR b | yc), c3 (zc), rad (CIRCLE / SPHERE r), val (NORM val | COLLISION radius).  LINEAR's A and every other field stay shared.  With
// con_row, the only place that decides between an instance's row of DevProblem::cdata and the descriptor; INST = false returns the descriptor's
// fields.  An instance's row of cdata, at DevCon::cdoff: GOAL xf[inds], BOUND z_max[n+m] | z_min[n+m], LINEAR b[p], CIRCLE xc[p] | yc[p] | r[p],
// SPHERE xc[p] | yc[p] | zc[p] | r[p], NORM val, COLLISION radius.
// con_row: constraint ci's part of instance b's row when the table exists, else `shared`.  For a constraint that carries data (DevCon::cdoff
// >= 0); the Goal read sites take their values with it (con_row<INST>(P, b, ci, con.a)).
template <bool INST>
__host__ __device__ __forceinline__ const double* con_row(const DevProblem& P, int b, int ci, const double* shared) {
    if constexpr (INST) { if (P.cdata) return P.cdata + (size_t)b * P.ncdata + P.cons[ci].cdoff; }
    return shared;
}
struct ConData { const double *a, *b, *c3, *rad; double val; };
template <bool INST>
__device__ __forceinline__ ConData con_data(const DevProblem& P, int b, int ci) {
    const DevCon& con = P.cons[ci];
    ConData d{con.a, con.b, con.c3, con.rad, con.val};
    if constexpr (INST) {
        if (P.cdata && con.cdoff >= 0) {
            const double* row = con_row<true>(P, b, ci, nullptr);
            switch (con.kind) {
                case CON_GOAL: d.a = row; break;
                case CON_BOUND: d.a = row; d.b = row + P.n + P.m; break;
                case CON_LINEAR: d.b = row; break;
                case CON_CIRCLE: d.a = row; d.b = row + con.p; d.rad = row + 2 * con.p; break;
                case CON_SPHERE: d.a = row; d.b = row + con.p; d.c3 = row + 2 * con.p; d.rad = row + 3 * con.p; break;
                case CON_NORM: case CON_COLLISION: d.val = row[0]; break;
            }
        }
    }
    return d;
}

__host__ __device__ inline const double* traj_X(const DevProblem& P, int buf, int b) { return P.X + buf * P.strideX + (size_t)b * P.N * P.n; }
__host__ __device__ inline const double* traj_U(const DevProblem& P, int buf, int b) { return P.U + buf * P.strideU + (size_t)b * (P.N - 1) * P.m; }
__host__ __device__ inline double* traj_Xw(const DevProblem& P, int buf, int b) { return P.X + buf * P.strideX + (size_t)b * P.N * P.n; }
__host__ __device__ inline double* traj_Uw(const DevProblem& P, int buf, int b) { return P.U + buf * P.strideU + (size_t)b * (P.N - 1) * P.m; }

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
