// solve.cu -- the per-instance stopping rules of to_solve (Altro's AL-iLQR `solve!`, restated in DESIGN.md 5d and include/trajopt_b200.h).
//
// The iteration itself is the one to_ilqr_step runs (expansion, backward pass, line search).  These kernels only DECIDE, one thread per
// instance: after an instance's line search, whether its inner (iLQR) loop goes on; when its inner loop has ended, whether it is done or goes
// on to another outer (AL) iteration.  With shared penalties that second decision waits until every inner loop of the batch has ended
// (k_solve_outer), and an instance whose loop has ended is marked WAITING or DONE in SolveDev::state, which is DevProblem::active while
// to_solve runs: every per-instance kernel of the iteration then skips it.  With per-instance penalties k_solve_check decides at once, and an
// instance that goes on stays ACTIVE, flagged in SolveDev::go for the outer step that follows the check on its stream.
#include "../../include/trajopt_b200.h"
#include "kernels.h"

namespace {

// Altro gradient_todorov: mean over the knots of max_i |d_k,i| / (|u_k,i| + 1), with the controls after the step
__device__ double todorov_gradient(const DevProblem& P, int b) {
    const int m = P.m, N = P.N;
    const double* U = traj_U(P, P.cur[b], b);
    const double* d = P.d + (size_t)b * (N - 1) * m;
    double acc = 0.0;
    for (int k = 0; k < N - 1; k++) {
        double g = 0.0;
        for (int i = 0; i < m; i++) g = fmax(g, fabs(d[(size_t)k * m + i]) / (fabs(U[(size_t)k * m + i]) + 1.0));
        acc += g;
    }
    return acc / (N - 1);
}

// the start of instance b's solve: ACTIVE, counters zero, rho restarted (k_solve_init, and k_queue_refill for a slot's new problem)
__device__ __forceinline__ void solve_init_instance(const DevProblem& P, const SolveDev& S, int b) {
    S.state[b] = SOLVE_ACTIVE; S.status[b] = TO_SOLVE_UNSOLVED;
    S.iter[b] = 0; S.outer[b] = 1; S.inner[b] = 0; S.dj_zero[b] = 0;
    S.dJ[b] = 0.0; S.grad[b] = 0.0; S.cmax[b] = 0.0;
    if (S.go) { S.go[b] = SOLVE_DONE; S.go[P.B + b] = SOLVE_DONE; }
    P.rho[b] = P.opt.bp_reg_initial; P.drho[b] = 0.0;      // Altro initialize!: the regularisation restarts
}

__global__ void k_solve_init(const DevProblem P, SolveDev S) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b == 0) *S.n_active = P.B;
    if (b >= P.B) return;
    solve_init_instance(P, S, b);
}

// Altro's outer-loop rules for instance b, whose inner loop has ended with violation S.cmax[b]: its final status, or TO_SOLVE_UNSOLVED when
// it goes on to another outer iteration
__device__ int outer_decision(const SolveDev& S, int b) {
    const SolveOpts& o = S.opt;
    if (S.cmax[b] < o.constraint_tolerance) return TO_SOLVE_SUCCEEDED;
    if (S.iter[b] >= o.iterations) return TO_SOLVE_MAX_ITERATIONS;
    if (S.outer[b] >= o.iterations_outer) return TO_SOLVE_MAX_ITERATIONS_OUTER;
    return TO_SOLVE_UNSOLVED;
}

// start of an inner loop of the ACTIVE instances: J_prev = the merit of the live trajectory (with the current multipliers and penalties)
__global__ void k_solve_begin(const DevProblem P, SolveDev S) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= P.B || S.state[b] != SOLVE_ACTIVE) return;
    S.J_prev[b] = P.J[b]; S.inner[b] = 0; S.dj_zero[b] = 0;
}

// after the line search of instance b.  mode 1 / 2: only the instances the first line-search pass accepted / did not accept (the two halves
// of an overlapped iteration, capi.cu), 0: all.
__global__ void k_solve_check(const DevProblem P, SolveDev S, int mode) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= P.B || S.state[b] != SOLVE_ACTIVE) return;
    if (mode != 0 && (P.acc1[b] != 0) != (mode == 1)) return;
    const SolveOpts& o = S.opt;
    const int iter = ++S.iter[b], inner = ++S.inner[b];
    const bool constrained = P.ncon > 0;
    // Altro set_tolerances!: the intermediate tolerances except in the last allowed outer iteration; no constraints: the plain iLQR loop
    const bool final_tol = !constrained || S.outer[b] >= o.iterations_outer;
    const double ctol = final_tol ? o.cost_tolerance : o.cost_tolerance_intermediate;
    const double gtol = final_tol ? o.gradient_tolerance : o.gradient_tolerance_intermediate;
    int next = SOLVE_ACTIVE, status = TO_SOLVE_UNSOLVED;
    if (P.bp_status[b] < 0) {                      // the backward pass failed at bp_reg_max: terminal
        S.dJ[b] = 0.0;
        next = SOLVE_DONE; status = TO_SOLVE_MAX_REGULARIZATION;
    } else {
        const double J = P.J[b];
        const bool stepped = P.alpha[b] > 0.0;
        const double dJ = stepped ? S.J_prev[b] - J : 0.0;
        if (!stepped) S.dj_zero[b]++;
        S.J_prev[b] = J;
        const double grad = todorov_gradient(P, b);
        S.dJ[b] = dJ; S.grad[b] = grad;
        const bool converged = stepped && dJ >= 0.0 && dJ < ctol && grad < gtol;
        const bool ended = converged || S.dj_zero[b] > o.dJ_counter_limit || iter >= o.iterations || (constrained && inner >= o.iterations_inner);
        if (ended) {
            if (constrained && S.go) {                      // per-instance penalties: the outer rules, now
                S.cmax[b] = P.viol[b];
                status = outer_decision(S, b);
                if (status == TO_SOLVE_UNSOLVED) { S.go[(mode == 2 ? P.B : 0) + b] = SOLVE_ACTIVE; return; }   // the outer step of this half follows
                next = SOLVE_DONE;
            } else if (constrained) next = SOLVE_WAITING;   // the outer step (k_solve_outer) decides
            else { next = SOLVE_DONE; status = converged ? TO_SOLVE_SUCCEEDED : iter >= o.iterations ? TO_SOLVE_MAX_ITERATIONS : TO_SOLVE_UNSOLVED; }
        }
    }
    if (next != SOLVE_ACTIVE) {
        S.cmax[b] = constrained ? P.viol[b] : 0.0;    // max violation of the live trajectory (the line search keeps it current)
        S.status[b] = status;
        S.state[b] = next;
        __threadfence();
        atomicSub(S.n_active, 1);
    }
}

// every inner loop has ended: the WAITING instances are done, or go on to another outer iteration (ACTIVE again)
__global__ void k_solve_outer(const DevProblem P, SolveDev S) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= P.B || S.state[b] != SOLVE_WAITING) return;
    const int status = outer_decision(S, b);
    if (status != TO_SOLVE_UNSOLVED) { S.status[b] = status; S.state[b] = SOLVE_DONE; return; }
    S.outer[b]++;
    S.state[b] = SOLVE_ACTIVE;
    atomicAdd(S.n_active, 1);
}

// per-instance penalties: the end of the outer step of the instances flagged in half `half` of SolveDev::go, after their dual update, penalty
// update and fresh merit (k_al_update and k_cost, launched with go as DevProblem::active): the next inner loop starts, as k_solve_begin starts it
__global__ void k_solve_restart(const DevProblem P, SolveDev S, int half) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= P.B || S.go[half * P.B + b] != SOLVE_ACTIVE) return;
    S.J_prev[b] = P.J[b]; S.inner[b] = 0; S.dj_zero[b] = 0;
    S.outer[b]++;
    S.go[half * P.B + b] = SOLVE_DONE;
}

// ---- to_solve_queue (DESIGN.md 5n): one thread per slot ----
// mode as k_solve_check: the slots of that half of the iteration (1: accepted by the first line-search pass, 2: the others, 0: every slot)
__device__ __forceinline__ bool in_half(const DevProblem& P, int b, int mode) { return mode == 0 || (P.acc1[b] != 0) == (mode == 1); }

// every slot empty and DONE, nothing claimed yet
__global__ void k_queue_init(const DevProblem P, SolveDev S, QueueDev Q) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b == 0) { *S.n_active = 0; *Q.next = 0; }
    if (b >= P.B) return;
    S.state[b] = SOLVE_DONE;
    Q.slot[b] = -1;
    Q.mask[b] = SOLVE_DONE; Q.mask[P.B + b] = SOLVE_DONE;
    if (S.go) { S.go[b] = SOLVE_DONE; S.go[P.B + b] = SOLVE_DONE; }
}

// mask of half `half` := the slots of the half whose problem stopped in this half's check (its objective, k_cost, follows with this mask)
__global__ void k_queue_harvest(const DevProblem P, SolveDev S, QueueDev Q, int half, int mode) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= P.B) return;
    Q.mask[half * P.B + b] = in_half(P, b, mode) && Q.slot[b] >= 0 && S.state[b] == SOLVE_DONE ? SOLVE_ACTIVE : SOLVE_DONE;
}

// The harvested slots hand their statistics, objective and trajectory to their problem's row of the outputs; then every DONE slot of the half
// claims the next problem.  A claimed problem starts as to_solve starts an instance that holds it: x0, U0 in the live buffer, lambda = 0, the
// shared penalties or its own, its rows of the slot tables, k_solve_init's state.  The mask then marks the refilled slots, for their closed-form
// Jacobian columns (with time-step rows), rollout, merit and k_queue_begin.
__global__ void k_queue_refill(const DevProblem P, SolveDev S, QueueDev Q, int half, int mode) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= P.B || !in_half(P, b, mode)) return;
    const int n = P.n, m = P.m, N = P.N;
    int* mask = Q.mask + (size_t)half * P.B + b;
    if (*mask == SOLVE_ACTIVE) {
        const int p = Q.slot[b];
        Q.status[p] = S.status[b]; Q.iter[p] = S.iter[b]; Q.outer[p] = S.outer[b];
        Q.cost[p] = Q.cost_slot[b]; Q.dJ[p] = S.dJ[b]; Q.grad[p] = S.grad[b]; Q.cmax[p] = S.cmax[b];
        if (Q.X) { const double* X = traj_X(P, P.cur[b], b); for (int i = 0; i < N * n; i++) Q.X[(size_t)p * N * n + i] = X[i]; }
        if (Q.U) { const double* U = traj_U(P, P.cur[b], b); for (int i = 0; i < (N - 1) * m; i++) Q.U[(size_t)p * (N - 1) * m + i] = U[i]; }
        Q.slot[b] = -1;
    }
    *mask = SOLVE_DONE;
    if (S.state[b] != SOLVE_DONE || *(volatile int*)Q.next >= Q.M) return;
    const int p = atomicAdd(Q.next, 1);
    if (p >= Q.M) return;
    Q.slot[b] = p;
    for (int i = 0; i < n; i++) P.x0[(size_t)b * n + i] = Q.x0[(size_t)p * n + i];
    const double* U0 = Q.U0 + (Q.U0_shared ? 0 : (size_t)p * (N - 1) * m);
    double* U = traj_Uw(P, P.cur[b], b);
    for (int i = 0; i < (N - 1) * m; i++) U[i] = U0[i];
    for (int i = 0; i < P.lambda_len; i++) P.lambda[(size_t)b * P.lambda_len + i] = 0.0;
#pragma unroll
    for (int t = 0; t < QUEUE_TABLES; t++) {
        const QueueTable& T = Q.tables[t];
        if (T.slot) for (int i = 0; i < T.w; i++) T.slot[(size_t)b * T.w + i] = T.src[(size_t)p * T.stride + i];
    }
    solve_init_instance(P, S, b);
    *mask = SOLVE_ACTIVE;
    __threadfence();
    atomicAdd(S.n_active, 1);
}

// the refilled slots of half `half`, after their rollout and merit: their first inner loop starts, as k_solve_begin starts it
__global__ void k_queue_begin(const DevProblem P, SolveDev S, QueueDev Q, int half) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= P.B || Q.mask[half * P.B + b] != SOLVE_ACTIVE) return;
    S.J_prev[b] = P.J[b]; S.inner[b] = 0; S.dj_zero[b] = 0;
}

// to_mpc_solve: step j's solve statistics of instance b, as to_solve returns them, into row j of the history.  A launch of its own:
// k_mpc_advance's plant step is kept as it is compiled (DESIGN.md 5l)
__global__ void k_mpc_solve_record(const DevProblem P, const SolveDev S, const MpcDev M, int j) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= P.B) return;
    const size_t r = (size_t)b * M.nsteps + j;
    M.status[r] = S.status[b]; M.iterations[r] = S.iter[b]; M.iterations_outer[r] = S.outer[b]; M.c_max[r] = S.cmax[b];
}

}  // namespace

cudaError_t launch_solve_init(const DevProblem& P, const SolveDev& S, cudaStream_t s) {
    k_solve_init<<<nblk(P.B, 128), 128, 0, s>>>(P, S);
    return cudaGetLastError();
}
cudaError_t launch_solve_begin(const DevProblem& P, const SolveDev& S, cudaStream_t s) {
    k_solve_begin<<<nblk(P.B, 128), 128, 0, s>>>(P, S);
    return cudaGetLastError();
}
cudaError_t launch_solve_check(const DevProblem& P, const SolveDev& S, int mode, cudaStream_t s) {
    k_solve_check<<<nblk(P.B, 128), 128, 0, s>>>(P, S, mode);
    return cudaGetLastError();
}
cudaError_t launch_solve_outer(const DevProblem& P, const SolveDev& S, cudaStream_t s) {
    k_solve_outer<<<nblk(P.B, 128), 128, 0, s>>>(P, S);
    return cudaGetLastError();
}
cudaError_t launch_solve_restart(const DevProblem& P, const SolveDev& S, int half, cudaStream_t s) {
    k_solve_restart<<<nblk(P.B, 128), 128, 0, s>>>(P, S, half);
    return cudaGetLastError();
}
cudaError_t launch_mpc_solve_record(const DevProblem& P, const SolveDev& S, const MpcDev& M, int j, cudaStream_t s) {
    k_mpc_solve_record<<<nblk(P.B, 128), 128, 0, s>>>(P, S, M, j);
    return cudaGetLastError();
}
cudaError_t launch_queue_init(const DevProblem& P, const SolveDev& S, const QueueDev& Q, cudaStream_t s) {
    k_queue_init<<<nblk(P.B, 128), 128, 0, s>>>(P, S, Q);
    return cudaGetLastError();
}
cudaError_t launch_queue_harvest(const DevProblem& P, const SolveDev& S, const QueueDev& Q, int half, int mode, cudaStream_t s) {
    k_queue_harvest<<<nblk(P.B, 128), 128, 0, s>>>(P, S, Q, half, mode);
    return cudaGetLastError();
}
cudaError_t launch_queue_refill(const DevProblem& P, const SolveDev& S, const QueueDev& Q, int half, int mode, cudaStream_t s) {
    k_queue_refill<<<nblk(P.B, 128), 128, 0, s>>>(P, S, Q, half, mode);
    return cudaGetLastError();
}
cudaError_t launch_queue_begin(const DevProblem& P, const SolveDev& S, const QueueDev& Q, int half, cudaStream_t s) {
    k_queue_begin<<<nblk(P.B, 128), 128, 0, s>>>(P, S, Q, half);
    return cudaGetLastError();
}
