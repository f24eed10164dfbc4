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

__global__ void k_solve_init(const DevProblem P, SolveDev S) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b == 0) *S.n_active = P.B;
    if (b >= P.B) return;
    S.state[b] = SOLVE_ACTIVE; S.status[b] = TO_SOLVE_UNSOLVED;
    S.iter[b] = 0; S.outer[b] = 1; S.inner[b] = 0; S.dj_zero[b] = 0;
    S.dJ[b] = 0.0; S.grad[b] = 0.0; S.cmax[b] = 0.0;
    if (S.go) { S.go[b] = SOLVE_DONE; S.go[P.B + b] = SOLVE_DONE; }
    P.rho[b] = P.opt.bp_reg_initial; P.drho[b] = 0.0;      // Altro initialize!: the regularisation restarts
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
