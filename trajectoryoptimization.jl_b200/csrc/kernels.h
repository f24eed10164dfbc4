// kernels.h -- host-side launch wrappers (one per kernel), implemented in the .cu files next to this header.
#pragma once
#include "common.cuh"

// blocks of `threads` threads that cover `total` threads (the grid of a launcher)
inline unsigned nblk(long long total, int threads) { return (unsigned)((total + threads - 1) / threads); }

// kernel 1: batched rollout / dual-number dynamics expansion with the problem's explicit rule           (rollout.cu)
cudaError_t launch_rollout(const DevProblem& P, cudaStream_t s, bool masked = false);   // masked: only the instances P.active marks ACTIVE
cudaError_t launch_expand(const DevProblem& P, cudaStream_t s, int mode = 0);   // mode 1 / 2: only instances with acc1 == 1 / == 0
// The launchers of the kernels that step the dynamics, per explicit rule RULE (to_integration).  rollout.cu and forward.cu are compiled once
// per rule; the object of rule R instantiates these for R alone, and the public launchers (launch_rollout, launch_expand, launch_expand_lie,
// launch_forward, launch_ladder) dispatch on DevProblem::integration.
template <int RULE> cudaError_t launch_rollout_rule(const DevProblem& P, cudaStream_t s, bool masked);
template <int RULE> cudaError_t launch_expand_rule(const DevProblem& P, cudaStream_t s, int mode);
template <int RULE> cudaError_t launch_expand_lie_rule(const DevProblem& P, cudaStream_t s, int mode);
template <int RULE> cudaError_t launch_forward_rule(const DevProblem& P, cudaStream_t s);
template <int RULE> cudaError_t launch_ladder_rule(const DevProblem& P, cudaStream_t s);
// Closed-loop MPC (to_mpc_run): the device copies of the run's inputs, made by to_mpc_setup, and the history the run writes.
struct MpcDev {
    const double* Xref;        // [B][nref][n] or nullptr: no reference window
    const double* Uref;        // [B][nref][m]
    const int* last_knot;      // [ncost]: the last knot that uses each cost (-1: none), the row the host's update_trajectory! writes last
    const double* W;           // [B][nsteps][ne] or nullptr: no disturbance
    const double* plant;       // [B][TO_NPARAM] (the layout of DevProblem::mparams) or nullptr: the planner's parameters
    double* Xcl;               // [B][nsteps+1][n]: row j = the state step j started from, row j+1 = where it ended
    double* Ucl;               // [B][nsteps][m]
    double* Jcl;               // [B][nsteps]: the merit of the plan step j applied
    int nref, nsteps;
    // to_mpc_solve: the solve statistics of step j, [B][nsteps] each (to_mpc_setup writes status -1, 0, 0, NaN: a step to_mpc_run took)
    int* status;
    int* iterations;
    int* iterations_outer;
    double* c_max;
};
cudaError_t launch_mpc_window(const DevProblem& P, const MpcDev& M, int row, cudaStream_t s);   // sweep.cu: the linear terms of reference row `row`
cudaError_t launch_mpc_advance(const DevProblem& P, const MpcDev& M, int j, cudaStream_t s);    // rollout.cu: record, plant step, shift of step j
template <int RULE> cudaError_t launch_mpc_advance_rule(const DevProblem& P, const MpcDev& M, int j, cudaStream_t s);
#define TO_RULE_EXTERN(R)                                                                                   \
    extern template cudaError_t launch_rollout_rule<R>(const DevProblem&, cudaStream_t, bool);            \
    extern template cudaError_t launch_expand_rule<R>(const DevProblem&, cudaStream_t, int);              \
    extern template cudaError_t launch_expand_lie_rule<R>(const DevProblem&, cudaStream_t, int);          \
    extern template cudaError_t launch_forward_rule<R>(const DevProblem&, cudaStream_t);                  \
    extern template cudaError_t launch_ladder_rule<R>(const DevProblem&, cudaStream_t);                   \
    extern template cudaError_t launch_mpc_advance_rule<R>(const DevProblem&, const MpcDev&, int, cudaStream_t);
TO_RULE_EXTERN(1)
TO_RULE_EXTERN(2)
TO_RULE_EXTERN(3)
TO_RULE_EXTERN(4)
#undef TO_RULE_EXTERN
// kernel 2: cost + constraint + AL sweep                                     (sweep.cu)
cudaError_t launch_cost(const DevProblem& P, double* J, double* Jk, cudaStream_t s);
cudaError_t launch_merit(const DevProblem& P, double* J, double* viol, cudaStream_t s);
cudaError_t launch_cost_gradient(const DevProblem& P, double* grad, cudaStream_t s);
cudaError_t launch_cost_hessian(const DevProblem& P, double* hess, cudaStream_t s);
cudaError_t launch_al_expansion(const DevProblem& P, double* grad, double* hess, cudaStream_t s);
cudaError_t launch_eval_constraints(const DevProblem& P, int con, double* vals, cudaStream_t s);
cudaError_t launch_constraint_jacobians(const DevProblem& P, int con, double* jac, cudaStream_t s);
cudaError_t launch_constraint_hessians(const DevProblem& P, int con, int len, const double* lam, double* H, cudaStream_t s);
cudaError_t launch_projection(int cone, int p, int count, const double* x, double* px, int* err, cudaStream_t s);
cudaError_t launch_grad_projection(int cone, int p, int count, const double* x, double* J, int* err, cudaStream_t s);
cudaError_t launch_hess_projection(int cone, int p, int count, const double* x, const double* b, double* H, int* err, cudaStream_t s);
cudaError_t launch_al_update(const DevProblem& P, cudaStream_t s);
cudaError_t launch_reduce_merit(const DevProblem& P, const double* viol, double* out2, cudaStream_t s);
cudaError_t launch_shift_traj(const DevProblem& P, int steps, cudaStream_t s);
cudaError_t launch_gather_traj(const DevProblem& P, double* Xout, double* Uout, cudaStream_t s);
cudaError_t launch_scatter_traj(const DevProblem& P, const double* Xin, const double* Uin, cudaStream_t s);
cudaError_t launch_export_ab(const DevProblem& P, double* ABout, cudaStream_t s);
// Kernel choices made from the problem's shape.  The launchers and the diagnostics (capi.cu) ask the functions below, so each reports what
// the launch does.  The values are those of include/trajopt_b200.h (TO_LS_*, TO_BK_*).
enum { KC_LS_GENERIC = 0, KC_LS_FAST = 1, KC_LS_COMPACT = 2 };
enum { KC_BK_THREAD = 0, KC_BK_WARP_MMA = 1, KC_BK_WARP_DFMA = 2, KC_BK_FRAGMENT = 3, KC_BK_DENSE_MMA = 4, KC_BK_DENSE_DFMA = 5 };
struct BackwardPlan {
    int kernel;   // KC_BK_*: the kernel launch_backward / launch_backward_frag launches
    // where it reads the cost + AL expansion: in k_riccati / k_riccati_small; the records, by k_expansion_rec16b from the term table
    // (common.cuh ExpTab) or by k_expansion_rec walking the descriptors; EC (k_expansion_compact); EG / EH (k_al_expansion + k_error_expansion)
    enum Expansion { IN_KERNEL, REC_TABLE, REC_WALK, COMPACT, MATERIALISED } expansion;
    bool fastal;  // k_riccati holds the AL terms lane-resident
};
BackwardPlan backward_plan(const DevProblem& P);   // riccati.cu: the only place that chooses the backward pass
int linesearch_path(const DevProblem& P);          // forward.cu: the knot loop of the line search (KC_LS_*)
bool linesearch_costs_cached(const DevProblem& P);  // forward.cu: the fast / compact loop reads the costs from shared memory
int frag_resident_warps();                          // riccati_frag.cu: k_riccati_frag warps (= instances) resident at once on this device
// kernel 3: Riccati backward pass                                             (riccati.cu)
cudaError_t launch_backward(const DevProblem& P, const BackwardPlan& plan, int* work_counter, cudaStream_t s);   // every kernel but KC_BK_FRAGMENT
bool riccati_small_supported(const DevProblem& P, bool any_batch);                     // riccati_small.cu: thread-per-instance pass for n <= 4, m <= 2
cudaError_t launch_backward_small(const DevProblem& P, cudaStream_t s);
// Lie-group error state + Riccati pass on a materialised expansion               (lie.cu)
cudaError_t launch_state_diff(const DevProblem& P, const double* Xbar, double* dx, cudaStream_t s);
cudaError_t launch_error_dynamics(const DevProblem& P, cudaStream_t s);
cudaError_t launch_error_expansion(const DevProblem& P, const double* gfull, const double* hfull, double* EG, double* EH, cudaStream_t s);
cudaError_t launch_backward_dense(const DevProblem& P, const BackwardPlan& plan, cudaStream_t s);
cudaError_t launch_expansion_compact(const DevProblem& P, cudaStream_t s);             // EC of every knot (P.compact)
cudaError_t launch_expand_lie(const DevProblem& P, cudaStream_t s, int mode = 0);     // [A_e B_e] straight from the dual-number explicit step (rollout.cu)
// register-resident Riccati pass of the error-state Quadrotor + its record producers   (riccati_frag.cu)
cudaError_t launch_expansion_rec(const DevProblem& P, cudaStream_t s);                 // compact expansion -> REC[192..240) of every knot
cudaError_t launch_expansion_rec16(const DevProblem& P, cudaStream_t s, int mode);               // ... 16-knot blocks per 16-lane group, from the host-built term table (rollout.cu)
// masked (to_solve_queue_tables' refill, with per-slot time steps): only the instances P.active marks ACTIVE
cudaError_t launch_trivial_columns_full(const DevProblem& P, cudaStream_t s, bool masked = false);   // ... of the full-state [A B]
cudaError_t launch_trivial_columns(const DevProblem& P, cudaStream_t s, bool masked = false);        // closed-form position / velocity columns of [A_e B_e], once per problem
cudaError_t launch_export_abe(const DevProblem& P, cudaStream_t s);                    // REC fragments -> ABe (col-major 12 x 16)
size_t frag_queue_ints(int B);
size_t frag_pool_doubles(int B, int N);                                                 // doubles of the speculative candidates' gain pool                                                         // ints of the kernel's work queue (allocated by the handle)
cudaError_t launch_backward_frag(const DevProblem& P, int* queue, double* pool, int* sticky_err, cudaStream_t s);
// forward pass: closed-loop rollout + merit + line search                     (forward.cu)
cudaError_t launch_forward(const DevProblem& P, cudaStream_t s);
cudaError_t launch_ladder(const DevProblem& P, cudaStream_t s);
cudaError_t launch_accept(const DevProblem& P, cudaStream_t s);
// to_solve: per-instance stopping rules (solve.cu).  The options are to_solve_options (include/trajopt_b200.h) field for field.
struct SolveOpts {
    double cost_tolerance, cost_tolerance_intermediate, gradient_tolerance, gradient_tolerance_intermediate, constraint_tolerance;
    int iterations, iterations_inner, iterations_outer, dJ_counter_limit;
};
struct SolveDev {
    SolveOpts opt;
    int* state;        // [B] SOLVE_ACTIVE / SOLVE_WAITING / SOLVE_DONE (DevProblem::active during to_solve)
    int* status;       // [B] to_solve_status
    int* iter;         // [B] iterations, all inner loops together
    int* outer;        // [B] outer (AL) iteration, 1-based
    int* inner;        // [B] iterations of the current inner loop
    int* dj_zero;      // [B] failed line searches in the current inner loop
    double* J_prev;    // [B] merit before the last step
    double* dJ;        // [B] last dJ
    double* grad;      // [B] last gradient (Altro gradient_todorov)
    double* cmax;      // [B] max violation when the last inner loop ended
    int* n_active;     // [1] instances ACTIVE
    // Per-instance penalties (DevProblem::mub): each instance's outer step runs on the device in the iteration in which its inner loop ends.
    // go[half * B + b] == SOLVE_ACTIVE: instance b's inner loop ended in that half of the iteration (0: main stream, 1: side stream) and it
    // goes on to another outer iteration; the outer-step kernels of that half see it as DevProblem::active.  nullptr: the host's outer step.
    int* go;           // [2][B]
};
cudaError_t launch_solve_init(const DevProblem& P, const SolveDev& S, cudaStream_t s);
cudaError_t launch_solve_begin(const DevProblem& P, const SolveDev& S, cudaStream_t s);
cudaError_t launch_solve_check(const DevProblem& P, const SolveDev& S, int mode, cudaStream_t s);   // mode as launch_expand
cudaError_t launch_solve_outer(const DevProblem& P, const SolveDev& S, cudaStream_t s);
cudaError_t launch_solve_restart(const DevProblem& P, const SolveDev& S, int half, cudaStream_t s);
cudaError_t launch_mpc_solve_record(const DevProblem& P, const SolveDev& S, const MpcDev& M, int j, cudaStream_t s);   // row j of the statistics
// to_solve_queue (capi.cu, DESIGN.md 5n): M problems through the B slots of the batch.  A slot whose instance is DONE hands its results to row p
// of the outputs (harvest) and takes the next problem (refill), in the half of the iteration whose check stopped it.
enum { QUEUE_TABLES = 6 };   // the per-instance tables of DevProblem (capi.cu Table)
// One of them as the refill replaces it: problem p's row src + p * stride (stride 0: every problem takes the same row) goes to row b of the
// slot table, [B][w] (nullptr: the slots keep the handle's table)
struct QueueTable {
    const double* src;
    double* slot;
    int stride, w;
};
struct QueueDev {
    int M, U0_shared;
    int* next;               // [1] the next problem to claim
    int* slot;               // [B] the problem in slot b, -1: none
    int* mask;               // [2][B] per half: the slots harvested, then the slots refilled (SOLVE_ACTIVE), as DevProblem::active of the launches after
    double* cost_slot;       // [B] the objective of the harvested slots (k_cost)
    const double* x0;        // [M][n]
    const double* U0;        // [M][N-1][m], or [N-1][m] when U0_shared
    QueueTable tables[QUEUE_TABLES];
    // outputs [M]: to_solve's statistics, and X [M][N][n], U [M][N-1][m] or nullptr
    int *status, *iter, *outer;
    double *cost, *dJ, *grad, *cmax, *X, *U;
};
cudaError_t launch_queue_init(const DevProblem& P, const SolveDev& S, const QueueDev& Q, cudaStream_t s);
cudaError_t launch_queue_harvest(const DevProblem& P, const SolveDev& S, const QueueDev& Q, int half, int mode, cudaStream_t s);   // mode as launch_solve_check
cudaError_t launch_queue_refill(const DevProblem& P, const SolveDev& S, const QueueDev& Q, int half, int mode, cudaStream_t s);
cudaError_t launch_queue_begin(const DevProblem& P, const SolveDev& S, const QueueDev& Q, int half, cudaStream_t s);
