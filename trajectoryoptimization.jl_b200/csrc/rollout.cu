// rollout.cu -- kernel 1 of the hot path: batched rollout and dual-number dynamics expansion.
//
//   k_rollout : rollout!(prob)                         reference src/problem.jl:330-340
//               x_1 = x0 ; x_k = step(x_{k-1}, u_{k-1}, dt_{k-1}) with the problem's explicit rule (models.cuh explicit_step).
//               Serial in k, parallel over instances:
//               one thread per instance (the recursion has no intra-instance parallelism worth a warp).
//   k_expand  : RD.jacobian!(ForwardAD) on the discretised dynamics at every knot (no call site inside the
//               reference; shape [A B] = n x (n+m) pinned by test/dynamics_constraints.jl:35,57-62).
//               One thread per (instance, knot, seed direction j): the explicit step is pushed through a
//               Dual<1> whose tangent is the one-hot e_j, i.e. the thread computes column j of [A B] with the
//               partial carried in registers.  Threads of one knot are adjacent, so row i of AB is written by
//               adjacent lanes; the pad columns of a row (LDAB > n+m) are never touched and stay zero.
#include <cstdlib>

#include "costcon.cuh"
#include "frag_layout.cuh"
#include "kernels.h"
#include "models.cuh"

// The kernels that step the dynamics take the explicit rule RULE (DevProblem::integration).  This file is compiled once per rule (Makefile):
// the object built with TO_RULE = 4 (TO_RK4) holds the RK4 instantiations, every kernel that steps no dynamics and the launchers that dispatch on
// the rule; the objects of the other rules hold only their rule's instantiations, so that they compile in parallel.
#ifndef TO_RULE
#define TO_RULE 4
#endif

// One thread integrates one instance; the warp writes its 32 states of a knot through a shared-memory transpose, so that the stores are runs of
// n contiguous doubles per instance (full 32-byte sectors) instead of 32 scattered 8-byte words per instruction.
// INST: the instance's own model parameters (DevProblem::mparams), one shared-memory copy per lane, and time steps (DevProblem::dtb).
// (Copied to registers instead, the parameter-only subexpressions of the dynamics were hoisted out of the knot loop and lost FMA contractions
// the shared kernel has.)
// MASK (to_solve_queue's refill): only the instances P.active marks ACTIVE are written; the others compute a rollout of their own that is not
// stored, so that the knot loop is the one the unmasked kernel runs.  A warp with no instance to write exits.
template <int MODEL, bool INST, int RULE, bool MASK = false>
__global__ void __launch_bounds__(32) k_rollout(const DevProblem P) {
    constexpr int n = ModelDims<MODEL>::n, m = ModelDims<MODEL>::m;
    __shared__ double stage[32 * n];
    __shared__ double* base[32];
    const int lane = threadIdx.x;
    const int b = blockIdx.x * 32 + lane;
    const bool valid = b < P.B && (!MASK || !retired(P, b));
    if constexpr (MASK) { if (!__any_sync(0xffffffffu, valid)) return; }
    const int bc = b < P.B ? b : P.B - 1;                   // (idle lanes of the last warp shadow a real instance and store nothing)
    base[lane] = valid ? traj_Xw(P, P.cur[bc], bc) : nullptr;
    const double* U = traj_U(P, P.cur[bc], bc);
    const double* prm = nullptr;
    if constexpr (INST) {
        __shared__ double prm_s[32][TO_NPARAM];
        stage_model_params<INST>(P, bc, prm_s[lane]);
        prm = prm_s[lane];
    }
    double x[n], u[m], xn[n];
#pragma unroll
    for (int i = 0; i < n; i++) x[i] = P.x0[(size_t)bc * n + i];
    for (int k = 0; k < P.N; k++) {
#pragma unroll
        for (int i = 0; i < n; i++) stage[lane * n + i] = x[i];
        __syncwarp();
#pragma unroll
        for (int j = 0; j < n; j++) {
            const int e = j * 32 + lane, ii = e / n, c = e - ii * n;
            double* Xi = base[ii];
            if (Xi) Xi[(size_t)k * n + c] = stage[e];
        }
        __syncwarp();
        if (k == P.N - 1) break;
#pragma unroll
        for (int i = 0; i < m; i++) u[i] = U[k * m + i];
        explicit_step<MODEL, double, RULE>(model_params<MODEL, INST>(P, prm, k), x, u, time_step<INST>(P, bc, k), xn);
#pragma unroll
        for (int i = 0; i < n; i++) x[i] = xn[i];
    }
}

// to_mpc_run, steps 4-6 of MPC step j, CTA = instance b.  Warp 0 steps the plant: k_rollout's loop over a trajectory of `knots` = 2 knots
// (x0, x+), written as k_rollout writes it -- the parameters staged per lane, the knot count read at run time, the state staged in shared
// memory behind a warp barrier every knot -- so that the compiler hoists and contracts the step's arithmetic as it does in k_rollout, and
// the plant computes k_rollout's bits: explicit_step<MODEL, double, RULE> on model_params<MODEL, INST> (the launcher's view carries the plant's
// rows as DevProblem::mparams) over knot 0's time step.  Every lane steps instance b; lane 0 applies the disturbance, x+ = step(x0, u_j) (+) w_j
// (costcon.cuh state_add), and records x0, x+, u_j = U[0] and the plan's merit J_j.  Then the CTA shifts the plan by one knot
// (shift_traj_cta, k_shift_traj's body), and x+ overwrites the x0 the shift wrote (each thread its own entry): the next step starts from the
// plant.
template <int MODEL, bool INST, int RULE>
__global__ void __launch_bounds__(128) k_mpc_advance(const DevProblem P, const MpcDev M, int j, int knots) {
    constexpr int n = ModelDims<MODEL>::n, m = ModelDims<MODEL>::m;
    __shared__ double xp[n];
    const int b = blockIdx.x;
    if (threadIdx.x < 32) {
        __shared__ double stage[32 * n];
        const int lane = threadIdx.x;
        const double* U = traj_U(P, P.cur[b], b);
        const double* prm = nullptr;
        if constexpr (INST) {
            __shared__ double prm_s[32][TO_NPARAM];
            stage_model_params<INST>(P, b, prm_s[lane]);
            prm = prm_s[lane];
        }
        double x[n], u[m], xn[n];
#pragma unroll
        for (int i = 0; i < n; i++) x[i] = P.x0[(size_t)b * n + i];
        for (int k = 0; k < knots; k++) {
#pragma unroll
            for (int i = 0; i < n; i++) stage[lane * n + i] = x[i];
            __syncwarp();
            if (k == knots - 1) break;
#pragma unroll
            for (int i = 0; i < m; i++) u[i] = U[k * m + i];
            explicit_step<MODEL, double, RULE>(model_params<MODEL, INST>(P, prm, k), x, u, time_step<INST>(P, b, k), xn);
#pragma unroll
            for (int i = 0; i < n; i++) x[i] = xn[i];
        }
        if (lane == 0) {
            if (M.W) state_add(P.lie != 0, n, P.qs, x, M.W + ((size_t)b * M.nsteps + j) * P.ne);
            double* Xh = M.Xcl + ((size_t)b * (M.nsteps + 1) + j) * n;
#pragma unroll
            for (int i = 0; i < n; i++) { Xh[i] = P.x0[(size_t)b * n + i]; Xh[n + i] = x[i]; xp[i] = x[i]; }
#pragma unroll
            for (int i = 0; i < m; i++) M.Ucl[((size_t)b * M.nsteps + j) * m + i] = U[i];
            M.Jcl[(size_t)b * M.nsteps + j] = P.J[b];
        }
    }
    __syncthreads();
    shift_traj_cta(P, b, 1);
    if (threadIdx.x < n) P.x0[(size_t)b * n + threadIdx.x] = xp[threadIdx.x];
}

// Seed pruning (full state).  The position r and the world-frame linear velocity v of the Quadrotor (a RobotDynamics RigidBody) enter the
// dynamics only through rdot = v, so their columns of [A B] are known in closed form -- d x+/d r = e_r, d x+/d v = h e_r + e_v (the weights
// of every explicit rule sum to one, so this holds for Euler, RK2, RK3 and RK4 alike) -- and are written when the problem is created and when
// its time steps change (k_trivial_columns_full); 11 seeds (quaternion, angular velocity, controls) are pushed through the dual-number step
// instead of 17.  Other models: every seed.
template <int MODEL> struct SeedList {
    static constexpr int count = ModelDims<MODEL>::n + ModelDims<MODEL>::m;
    __host__ __device__ static constexpr int seed(int s) { return s; }
    __host__ __device__ static constexpr int ntrivial() { return 0; }
    __host__ __device__ static constexpr int trivial(int) { return 0; }
};
template <> struct SeedList<MODEL_QUADROTOR> {
    static constexpr int count = 11;
    __host__ __device__ static constexpr int seed(int s) { return s < 4 ? 3 + s : 6 + s; }       // 3..6 (q), 10..12 (omega), 13..16 (u)
    __host__ __device__ static constexpr int ntrivial() { return 6; }
    __host__ __device__ static constexpr int trivial(int s) { return s < 3 ? s : 4 + s; }        // 0..2 (r), 7..9 (v)
};

// INST: the instance's own model parameters (DevProblem::mparams), one shared-memory copy per thread (see k_rollout), and time steps
template <int MODEL, int NP, bool INST, int RULE>
__global__ void __launch_bounds__(128) k_expand(const DevProblem P, int mode) {
    constexpr int n = ModelDims<MODEL>::n, m = ModelDims<MODEL>::m, nm = n + m;
    constexpr int NSEED = SeedList<MODEL>::count;
    constexpr int TPK = (NSEED + NP - 1) / NP;     // threads per knot: each carries NP seed directions
    using D = Dual<NP>;
    const int ld = P.ldab;
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)P.B * (P.N - 1) * TPK;
    if (t >= total) return;
    const int s0 = (int)(t % TPK) * NP;            // first seed slot of this thread
    const long long bk = t / TPK;
    const int k = (int)(bk % (P.N - 1));
    const int b = (int)(bk / (P.N - 1));
    if (mode != 0 && (P.acc1[b] != 0) != (mode == 1)) return;     // overlapped expansion: this launch covers the other group
    if (retired(P, b)) return;                                     // to_solve: not ACTIVE
    double* AB = P.AB + ((size_t)b * (P.N - 1) + k) * n * ld;     // pad columns nm..ld-1 stay zero from to_create
    const double* X = traj_X(P, P.cur[b], b) + (size_t)k * n;
    const double* U = traj_U(P, P.cur[b], b) + (size_t)k * m;
    int js[NP];                                    // the z index each seed slot differentiates with respect to (nm = none)
#pragma unroll
    for (int q = 0; q < NP; q++) js[q] = (s0 + q < NSEED) ? SeedList<MODEL>::seed(s0 + q) : nm;
    D x[n], u[m], xn[n];
#pragma unroll
    for (int i = 0; i < n; i++) {
        x[i].v = X[i];
#pragma unroll
        for (int q = 0; q < NP; q++) x[i].d[q] = (i == js[q]) ? 1.0 : 0.0;
    }
#pragma unroll
    for (int i = 0; i < m; i++) {
        u[i].v = U[i];
#pragma unroll
        for (int q = 0; q < NP; q++) u[i].d[q] = (n + i == js[q]) ? 1.0 : 0.0;
    }
    const double* prm = nullptr;
    if constexpr (INST) {
        __shared__ double prm_s[128][TO_NPARAM];
        stage_model_params<INST>(P, b, prm_s[threadIdx.x]);
        prm = prm_s[threadIdx.x];
    }
    explicit_step<MODEL, D, RULE>(model_params<MODEL, INST>(P, prm, k), x, u, time_step<INST>(P, b, k), xn);
#pragma unroll
    for (int i = 0; i < n; i++) {
        if (NP == 2 && js[1] == js[0] + 1 && !(js[0] & 1)) *reinterpret_cast<double2*>(&AB[i * ld + js[0]]) = make_double2(xn[i].d[0], xn[i].d[1]);
        else {
#pragma unroll
            for (int q = 0; q < NP; q++) if (js[q] < nm) AB[i * ld + js[q]] = xn[i].d[q];
        }
    }
}

#if TO_RULE == 4
// the closed-form columns of [A B] (SeedList<MODEL>::trivial): thread = (instance, knot, one of them); run when the problem is created and
// whenever its time steps change (INST: each instance's own, DevProblem::dtb).  MASK (to_solve_queue_tables' refill): only the instances
// P.active marks ACTIVE
template <int MODEL, bool INST, bool MASK = false>
__global__ void __launch_bounds__(128) k_trivial_columns_full(const DevProblem P) {
    constexpr int n = ModelDims<MODEL>::n, NT = SeedList<MODEL>::ntrivial();
    if constexpr (NT > 0) {
        const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
        if (t >= (long long)P.B * (P.N - 1) * NT) return;
        const int jt = SeedList<MODEL>::trivial((int)(t % NT));
        const long long bk = t / NT;
        const int k = (int)(bk % (P.N - 1));
        if constexpr (MASK) { if (retired(P, (int)(bk / (P.N - 1)))) return; }
        double* AB = P.AB + (size_t)bk * n * P.ldab;
        const double h = time_step<INST>(P, (int)(bk / (P.N - 1)), k);
        // x = [r(0..2); q(3..6); v(7..9); omega(10..12)]: d r+/d r = I, d r+/d v = h I, d v+/d v = I
        for (int i = 0; i < n; i++) AB[i * P.ldab + jt] = (i == jt) ? 1.0 : ((jt >= 7 && i == jt - 7) ? h : 0.0);
    }
}
// (a masked launch comes with per-slot time steps, so it has INST instantiations only)
cudaError_t launch_trivial_columns_full(const DevProblem& P, cudaStream_t s, bool masked) {
    if (P.model == MODEL_QUADROTOR) {
        const long long total = (long long)P.B * (P.N - 1) * SeedList<MODEL_QUADROTOR>::ntrivial();
        if (masked) k_trivial_columns_full<MODEL_QUADROTOR, true, true><<<(unsigned)((total + 127) / 128), 128, 0, s>>>(P);
        else if (inst_dynamics(P)) k_trivial_columns_full<MODEL_QUADROTOR, true><<<(unsigned)((total + 127) / 128), 128, 0, s>>>(P);
        else k_trivial_columns_full<MODEL_QUADROTOR, false><<<(unsigned)((total + 127) / 128), 128, 0, s>>>(P);
    }
    return cudaGetLastError();
}

// (g, h) = (lz_i, lzz_ii) of entry i of the full-state z = [x; u] at knot k (0-based): DiagonalCost (RD.gradient!/hessian!, src/cost_functions.jl:137-233)
// + the AL terms of the Goal / Bound rows acting on z_i (src/constraints.jl:55-68, :738-765; projection on the dual cone src/cones.jl:96-145).
// The compact problem class only (P.compact): every cost diagonal, every constraint Goal or Bound, at most TO_EXP_MAXT rows per entry
// (the host-built table P.exptab; walking the constraint descriptors per thread instead adds work comparable to the RK4 itself).
// The bound of term t of z entry i for instance b: its entry of the instance's row of DevProblem::cdata when the table exists, else `shared`
__device__ __forceinline__ double exp_term_bound(const DevProblem& P, const ExpTab& tab, int b, int t, int i, double shared) {
    const int j = __ldg(&tab.inst[t][i]);
    if (P.cdata && j >= 0) return P.cdata[(size_t)b * P.ncdata + j];
    return shared;
}
// -mu sign of term t of z entry i for instance b: with its penalty from the instance's row of DevProblem::mub when the table exists (exact:
// sign = +-1 and `shared` = -mu sign carries it), else `shared`
__device__ __forceinline__ double exp_term_nms(const DevProblem& P, const ExpTab& tab, int b, int t, int i, double shared) {
    const int ci = __ldg(&tab.con[t][i]);
    if (P.mub && ci >= 0) { const double mu = penalty<true>(P, b, ci); return shared < 0.0 ? -mu : mu; }
    return shared;
}
// (INST: the cost weights, linear cost terms, Goal / Bound bounds and penalties of instance b)
template <bool INST>
__device__ __forceinline__ void compact_entry_expansion(const DevProblem& P, const ExpTab& tab, int b, int k, int i, double zi, const double* __restrict__ lam_b, double& g, double& h) {
    const int n = P.n;
    const bool last = (k == P.N - 1);
    const int cid = P.cost_index[k];
    const CostData c = cost_data<INST>(P, b, cid);
    if (i < n) { g = fma(c.Qd[i], zi, c.q[i]); h = c.Qd[i]; }
    else if (last) { g = 0.0; h = 0.0; return; }
    else { g = fma(c.Rd[i - n], zi, c.r[i - n]); h = c.Rd[i - n]; }
#pragma unroll
    for (int t = 0; t < TO_EXP_MAXT; t++) {
        const unsigned px = __ldg(&tab.pkx[t][i]);
        if ((unsigned)(k + 1) - (px & 0xfffu) <= ((px >> 12) & 0xfffu)) {
            double nms = __ldg(&tab.nms[t][i]);
            if constexpr (INST) nms = exp_term_nms(P, tab, b, t, i, nms);
            const double lam = lam_b[(int)(__ldg(&tab.pky[t][i]) + (unsigned)(k + 1) * ((px >> 24) & 0x7fu))];
            double bound = __ldg(&tab.bound[t][i]);
            if constexpr (INST) bound = exp_term_bound(P, tab, b, t, i, bound);
            const double lb = fma(nms, zi - bound, lam);          // lambda - mu c
            if ((px >> 31) || lb <= 0.0) { g += (nms < 0.0) ? -lb : lb; h += fabs(nms); }   // g -= sign lb ; h += mu
        }
    }
}

#endif  // TO_RULE == 4

// Seed pruning.  The position r and the (world-frame) linear velocity v of a RigidBody enter the dynamics only through rdot = v: f does not
// depend on r, and on v only in rdot.  Their columns of the discrete Jacobian are therefore known in closed form -- d x+/d r = e_r and
// d x+/d v = h e_r + e_v (the weights of every explicit rule sum to one) -- and need no dual-number sweep: 10 seeds (attitude, angular
// velocity, controls) are pushed through the step instead of 16, one thread each; the six trivial columns depend on the time steps only.  The materialised P.ABe
// gets them when the problem is created and when its time steps change (k_trivial_columns); k_expand_lie_rec writes them into every record
// block it assembles, and the export of the records (launch_export_abe) carries them to P.ABe on the record path.
__device__ __forceinline__ int lie_seed(int s) { return (int)((0xFEDCBA9543ULL >> (4 * s)) & 15); }       // 3,4,5,9,10,11,12,13,14,15
__device__ __forceinline__ int lie_trivial(int s) { return (int)((0x876210ULL >> (4 * s)) & 15); }        // 0,1,2,6,7,8

// column j of [A_e B_e]_k: the explicit step of knot k pushed through Dual<1> with the seed of error-state coordinate j (attitude: a column of G(q_k)),
// projected on the error state of knot k + 1 with G(q_{k+1})'  (INST: with instance b's parameters, staged in `prm`, and its time step)
template <int MODEL, bool INST, int RULE>
__device__ __forceinline__ void expand_lie_column(const DevProblem& P, const double* prm, int b, int k, int j, const double* __restrict__ X,
                                                  const double* __restrict__ U, double (&col)[ModelDims<MODEL>::n - 1]) {
    constexpr int n = ModelDims<MODEL>::n, m = ModelDims<MODEL>::m, ne = n - 1, qs = 3;
    using D = Dual<1>;
    const double h = time_step<INST>(P, b, k);
    D x[n], u[m], xn[n];
#pragma unroll
    for (int i = 0; i < n; i++) { x[i].v = X[i]; x[i].d[0] = 0.0; }
#pragma unroll
    for (int i = 0; i < m; i++) { u[i].v = U[i]; u[i].d[0] = (ne + i == j) ? 1.0 : 0.0; }
    if (j < qs + 3) {
        const double w = X[qs], qx = X[qs + 1], qy = X[qs + 2], qz = X[qs + 3];
        const int c = j - qs;        // column c of L(q) H: (-x,w,z,-y), (-y,-z,w,x), (-z,y,-x,w)
        x[qs].d[0] = (c == 0) ? -qx : (c == 1) ? -qy : -qz;
        x[qs + 1].d[0] = (c == 0) ? w : (c == 1) ? -qz : qy;
        x[qs + 2].d[0] = (c == 0) ? qz : (c == 1) ? w : -qx;
        x[qs + 3].d[0] = (c == 0) ? -qy : (c == 1) ? qx : w;
    } else if (j < ne) {
#pragma unroll
        for (int i = qs + 4; i < n; i++) x[i].d[0] = (i == j + 1) ? 1.0 : 0.0;
    }
    explicit_step<MODEL, D, RULE>(model_params<MODEL, INST>(P, prm, k), x, u, h, xn);
    const double* q1 = X + n + qs;                                     // attitude of knot k + 1
    const double w1 = q1[0], x1 = q1[1], y1 = q1[2], z1 = q1[3];
#pragma unroll
    for (int i = 0; i < qs; i++) col[i] = xn[i].d[0];
    const double t0 = xn[qs].d[0], t1 = xn[qs + 1].d[0], t2 = xn[qs + 2].d[0], t3 = xn[qs + 3].d[0];
    col[qs] = -x1 * t0 + w1 * t1 + z1 * t2 - y1 * t3;
    col[qs + 1] = -y1 * t0 - z1 * t1 + w1 * t2 + x1 * t3;
    col[qs + 2] = -z1 * t0 + y1 * t1 - x1 * t2 + w1 * t3;
#pragma unroll
    for (int i = qs + 4; i < n; i++) col[i - 1] = xn[i].d[0];
}

#ifndef TO_EXPAND_LIE_MINB
#define TO_EXPAND_LIE_MINB 4      // CTAs per SM the register allocation aims at: 128 registers, 16 warps per SM
#endif
// CTA size: the kernel fills the register file (128 registers x 512 threads), so every CTA of another kernel that becomes resident next to it (the
// late line-search trials on the side stream, 4096 registers each) evicts a whole CTA of this one: 64-thread CTAs lose 1/8 of an SM, not 1/4.
#ifndef TO_EXPAND_LIE_THREADS
#define TO_EXPAND_LIE_THREADS 64
#endif
// INST: the instance's own model parameters (DevProblem::mparams), one shared-memory copy per thread (see k_rollout), and time steps
template <int MODEL, bool INST, int RULE>
__global__ void __launch_bounds__(TO_EXPAND_LIE_THREADS, TO_EXPAND_LIE_MINB * 128 / TO_EXPAND_LIE_THREADS) k_expand_lie(const DevProblem P, int mode) {
    constexpr int n = ModelDims<MODEL>::n, m = ModelDims<MODEL>::m, ne = n - 1, nme = ne + m, NS = 10;
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)P.B * (P.N - 1) * NS;
    if (t >= total) return;
    const int sd = (int)(t % NS);
    const int j = lie_seed(sd);
    const long long bk = t / NS;
    const int k = (int)(bk % (P.N - 1));
    const int b = (int)(bk / (P.N - 1));
    if (mode != 0 && (P.acc1[b] != 0) != (mode == 1)) return;
    if (retired(P, b)) return;                                     // to_solve: not ACTIVE
    const double* X = traj_X(P, P.cur[b], b) + (size_t)k * n;
    const double* U = traj_U(P, P.cur[b], b) + (size_t)k * m;
    const double* prm = nullptr;
    if constexpr (INST) {
        __shared__ double prm_s[TO_EXPAND_LIE_THREADS][TO_NPARAM];
        stage_model_params<INST>(P, b, prm_s[threadIdx.x]);
        prm = prm_s[threadIdx.x];
    }
    double col[ne];
    expand_lie_column<MODEL, INST, RULE>(P, prm, b, k, j, X, U, col);
    double* out = P.ABe + ((size_t)bk * nme + j) * ne;                 // column j of [A_e B_e]: 12 contiguous doubles
#pragma unroll
    for (int e = 0; e < ne; e++) out[e] = col[e];
}

// ---- k_expand_lie_rec: the record path's dynamics expansion ---------------------------------------------------------------------------------
// Stored column by column into the record, each column would be 12 scattered 8-byte stores (one L2 sector operation each), and only 10 of the 16
// columns change: in the record's fragment order a 32-byte sector holds columns {c, c + 8} of two rows, and 4 of the 8 column pairs mix a seed
// column with a closed-form one, so every iteration would write those sectors only partly and the L2 would fill them from DRAM first.
// Here a CTA owns EXPB_KPB consecutive knots of ONE instance (one thread per (knot, seed), the same expand_lie_column as k_expand_lie: the
// blocks are bit-identical to its [A_e B_e]).  Each thread drops its column into a shared-memory image of its knot's 1536-byte [A_e B_e] block; the six seed threads
// sd < 6 of the knot also write one closed-form column each (positions, velocities: 1 on the diagonal, dt[k] at (e, e + 6)), so the image is
// complete, and the CTA writes the images out as whole 128-byte lines with 16-byte stores: no sector of the block is ever partly written.
//   mapping   6 knots x 10 seeds = 60 of 64 threads; at N = 101, 17 CTAs per instance and 8 % of the lanes idle.  The instance test of the
//             overlapped launches (mode 1 / 2) is uniform over the CTA; mode 2 walks the compact late list when there is one (k_linesearch).
//   CTA size  64 threads like k_expand_lie: a CTA of the late line-search trials that becomes resident beside it displaces 1/8 of an SM.
//   image     record order (frag_layout.cuh) with the 16-byte chunks of each 128-byte line permuted by fraglayout::stage_swz: the column
//             stores of a warp spread over the banks, the line stores read every bank once.
// tests/test_expand_staging.py restates the staging map and the write-out in NumPy.
// INST: the instance's own model parameters (DevProblem::mparams), staged in shared memory once per CTA (the CTA's one instance), and time steps
#define EXPB_KPB 6
#define EXPB_T 64
template <int MODEL, bool INST, int RULE>
__global__ void __launch_bounds__(EXPB_T, TO_EXPAND_LIE_MINB * 128 / EXPB_T) k_expand_lie_rec(const DevProblem P, int mode, int nkb) {
    constexpr int n = ModelDims<MODEL>::n, m = ModelDims<MODEL>::m, ne = n - 1, NS = 10;
    static_assert(ne == 12 && m == 4 && EXPB_KPB * NS <= EXPB_T, "record layout of the error-state Quadrotor");
    __shared__ __align__(16) double st[EXPB_KPB][TO_REC_G];
    const int slot = blockIdx.x / nkb, kb = blockIdx.x - slot * nkb;
    int b = slot;
    if (mode == 2 && P.late_list) {                                                    // the instances pass 1 did not accept (acc1[b] == 0)
        if (slot >= *P.late_count) return;
        b = P.late_list[slot];
    } else if (mode != 0 && (P.acc1[b] != 0) != (mode == 1)) return;                   // overlapped iterations: the other launch covers this instance
    if (retired(P, b)) return;                                                         // to_solve: not ACTIVE (uniform over the CTA)
    const int k0 = kb * EXPB_KPB;
    const int nk = (P.N - 1 - k0 < EXPB_KPB) ? P.N - 1 - k0 : EXPB_KPB;
    const int tid = threadIdx.x, kk = tid / NS, sd = tid - kk * NS;
    const double* prm = nullptr;
    if constexpr (INST) {
        __shared__ double prm_s[TO_NPARAM];
        if (tid == 0) stage_model_params<INST>(P, b, prm_s);
        __syncthreads();
        prm = prm_s;
    }
    if (kk < nk) {
        const int k = k0 + kk;
        const int buf = P.cur[b];
        const double* X = traj_X(P, buf, b) + (size_t)k * n;
        const double* U = traj_U(P, buf, b) + (size_t)k * m;
        double* img = st[kk];
        // element (row e, column jj) sits at ab_index(e, 12) | 8 (c & 7) | (c >> 3), c = phys_z(jj) (disjoint bits: ab_index(e, 12) = 64 ks + 2 fc)
        auto put = [&](int jj, const double (&col)[ne]) {
            const int c = (int)((0x6420FDB9E7CA8531ULL >> (4 * jj)) & 15);            // fraglayout::phys_z(jj) as a nibble table
            const int cb = 8 * (c & 7) + (c >> 3);
#pragma unroll
            for (int e = 0; e < ne; e++) img[fraglayout::stage_swz(fraglayout::ab_index(e, 12) | cb, kk)] = col[e];
        };
        double col[ne];
        expand_lie_column<MODEL, INST, RULE>(P, prm, b, k, lie_seed(sd), X, U, col);
        put(lie_seed(sd), col);
        if (sd < 6) {                                                                  // closed-form column jt: d x+/d r = I, d r+/d v = h I, d v+/d v = I
            const int jt = lie_trivial(sd);
            const double h = time_step<INST>(P, b, k);
#pragma unroll
            for (int e = 0; e < ne; e++) col[e] = (e == jt) ? 1.0 : ((jt >= 6 && e == jt - 6) ? h : 0.0);
            put(jt, col);
        }
    }
    __syncthreads();
    // write-out: warp w takes knots w, w + 2, w + 4; lane l the 16-byte chunks l, l + 32, l + 64 of the knot's 96 (4 whole lines per store instruction).
    // Streaming stores: the 629 MB of blocks per iteration (B = 4096, N = 101) cannot stay in the L2 until the Riccati pass reads them; evict-first
    // keeps the line-search trials' operands there (E beside the late trials 0.409-0.410 -> 0.406-0.407 ms on one H100 80GB HBM3, 700 W).
    const int warp = tid >> 5, lane = tid & 31;
    double* recb = P.REC + ((size_t)b * P.N + k0) * TO_REC_LEN;
    for (int q = warp; q < nk; q += EXPB_T / 32) {
        double2* dst = reinterpret_cast<double2*>(recb + (size_t)q * TO_REC_LEN);
        const double2* src = reinterpret_cast<const double2*>(st[q]);
#pragma unroll
        for (int r = 0; r < 3; r++) {
            const int w = lane + 32 * r;
            __stcs(dst + w, src[fraglayout::stage_swz(2 * w, q) >> 1]);
        }
    }
}

#if TO_RULE == 4
// the closed-form columns of [A_e B_e] (positions, velocities): thread = (instance, knot, one of the six); INST: each instance's time steps;
// MASK as k_trivial_columns_full
template <bool INST, bool MASK = false>
__global__ void __launch_bounds__(128) k_trivial_columns(const DevProblem P) {
    constexpr int ne = 12, nme = 16;
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)P.B * (P.N - 1) * 6) return;
    const int sd = (int)(t % 6);
    const long long bk = t / 6;
    const int k = (int)(bk % (P.N - 1));
    if constexpr (MASK) { if (retired(P, (int)(bk / (P.N - 1)))) return; }
    const int jt = lie_trivial(sd);
    const double h = time_step<INST>(P, (int)(bk / (P.N - 1)), k);
    for (int e = 0; e < ne; e++) P.ABe[((size_t)bk * nme + jt) * ne + e] = (e == jt) ? 1.0 : ((jt >= 6 && e == jt - 6) ? h : 0.0);
}
cudaError_t launch_trivial_columns(const DevProblem& P, cudaStream_t s, bool masked) {
    const long long total = (long long)P.B * (P.N - 1) * 6;
    if (P.frag) return cudaSuccess;       // k_expand_lie_rec writes the whole block, closed-form columns included, every time
    if (masked) k_trivial_columns<true, true><<<(unsigned)((total + 127) / 128), 128, 0, s>>>(P);
    else if (inst_dynamics(P)) k_trivial_columns<true><<<(unsigned)((total + 127) / 128), 128, 0, s>>>(P);
    else k_trivial_columns<false><<<(unsigned)((total + 127) / 128), 128, 0, s>>>(P);
    return cudaGetLastError();
}

// ---- k_expansion_rec16b: the cost + AL expansion part of every record (frag_layout.cuh [192, 240)), the terminal knot included ---------------
// Outside the attitude the error-state expansion of a diagonal full-state one is the same entry; the quaternion block is projected from the
// (g, h, q) of q_w..q_z: G'g, G' diag(h) G - (q'g_q) I3 (Altro error_expansion!; lie.cu k_expansion_compact is the one-thread-per-knot version of
// the same numbers).  A light kernel (every load independent) that runs at full occupancy; fused into the FP64-bound k_expand_lie it doubled
// that kernel's time.
// One knot per 16-lane step (lane i = entry i of the full-state z = [x; u]) would spend many instructions per lane and knot on 3 outputs, and wait
// on two-level dependent loads (cur[b] -> X, cost_index[k] -> DevCost): every step would pay for the attitude projection that 3 of its lanes need
// (24 shuffles + ~40 FP64), for the 17th entry u_3 that lane 0 would take in a divergent second call, and for the unpacking of the term table.
// Here a 16-lane group owns a BLOCK of 16 consecutive knots of one instance:
//   phase A   16 steps, lane i < 13 = state entry x_i of one knot: diagonal cost + AL terms -> (g, h); loads (x_i and the multipliers of
//             its <= 3 terms) are issued for 4 knots at a time before the arithmetic; the cost coefficients of the lane are cached in
//             registers while the cost index does not change; lanes 3..6 (the quaternion) leave (g, h, q) in shared memory
//   phase B   lane j projects the attitude block of knot j (G'g, G' diag(h) G - (q'g_q) I3): once per knot instead of once per step
//   phase C   lane j takes the four control entries of knot j (their Bound rows are the AL terms that are active at every knot: in
//             phase A three lanes of sixteen would execute them at every step)
// ~55 instructions per lane and knot.
#ifndef TO_CEXP2_MINB
#define TO_CEXP2_MINB 9
#endif
#ifndef TO_CEXP2_THREADS
#define TO_CEXP2_THREADS 64
#endif
// INST: the linear cost terms, Goal / Bound bounds and penalties of each instance (DevProblem::qr / cdata / mub), a variant of its own so that the shared one stays as it is
template <bool INST>
__global__ void __launch_bounds__(TO_CEXP2_THREADS, TO_CEXP2_MINB) k_expansion_rec16b(const DevProblem P, int mode) {
    constexpr int qs = 3, n = 13, m = 4;
    constexpr int ROW = 49;                                                          // 48 doubles of expansion per knot, padded: lane j works on row j (stride 98 words: conflict-free)
    // the block's 16 x 48 outputs are staged in shared memory and leave as whole 128-byte lines: written entry by entry they are 8-byte
    // stores scattered over the records, and every one of them costs the L2 a 32-byte sector transaction
    __shared__ __align__(16) double stage_s[TO_CEXP2_THREADS / 16][16][ROW];
    const int i = threadIdx.x & 15;
    double (*stage)[ROW] = stage_s[threadIdx.x >> 4];
    const int N = P.N, NB = (N + 15) >> 4;
    const int ngroups = (int)((gridDim.x * blockDim.x) >> 4);
    const ExpTab& tab = *P.exptab;
    unsigned px[TO_EXP_MAXT], py[TO_EXP_MAXT]; double nms[TO_EXP_MAXT], bnd[TO_EXP_MAXT];
#pragma unroll
    for (int t = 0; t < TO_EXP_MAXT; t++) { px[t] = tab.pkx[t][i]; py[t] = tab.pky[t][i]; nms[t] = tab.nms[t][i]; bnd[t] = tab.bound[t][i]; }
    const int e = (i < qs) ? i : i - 1;                                               // error-state coordinate of entry i (controls: 12 + a = i - 1)
    const int pme = (int)((0x6420FDB9E7CA8531ULL >> (4 * (e & 15))) & 15);            // its physical slot
    const bool quat = (i >= qs && i <= qs + 3);
    const unsigned gm = 0xFFFFu << (threadIdx.x & 16);
    const int total = P.B * NB;
    constexpr int G_ = TO_REC_G - TO_REC_G, HD_ = TO_REC_HD - TO_REC_G, HB_ = TO_REC_HB - TO_REC_G;   // offsets inside the staged 48 doubles
    for (int unit = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 4); unit < total; unit += ngroups) {
        const int b = unit / NB, kb = (unit - b * NB) << 4;
        if (mode != 0 && (P.acc1[b] != 0) != (mode == 1)) continue;                   // (uniform over the group)
        if (retired(P, b)) continue;                                                   // to_solve: not ACTIVE
        const int buf = P.cur[b];
        const double* __restrict__ Xb = traj_X(P, buf, b);
        const double* __restrict__ Ub = traj_U(P, buf, b);
        const double* __restrict__ lam_b = P.lambda + (size_t)b * P.lambda_len;
        double* __restrict__ recb = P.REC + ((size_t)b * N + kb) * TO_REC_LEN + TO_REC_G;
        if constexpr (INST) {                                                         // this instance's Goal / Bound bounds and penalties into the lane's terms
#pragma unroll
            for (int t = 0; t < TO_EXP_MAXT; t++) { bnd[t] = exp_term_bound(P, tab, b, t, i, tab.bound[t][i]); nms[t] = exp_term_nms(P, tab, b, t, i, tab.nms[t][i]); }
        }
        const int nk = (N - kb < 16) ? N - kb : 16;
        const int mycid = (i < nk) ? P.cost_index[kb + i] : 0;                        // lane j <-> knot kb + j (phases B, C; broadcast in phase A)
        int ccid = -1; double ca = 0.0, cb = 0.0;                                     // this lane's coefficients (Qd_i, q_i) of cost ccid
        // term t acts on the knots of the block whose bit is set in act[t]; lp[t] = its multiplier at the first knot of the block
        unsigned act[TO_EXP_MAXT]; const double* lp[TO_EXP_MAXT]; int ls[TO_EXP_MAXT];
#pragma unroll
        for (int t = 0; t < TO_EXP_MAXT; t++) {
            const int first = (int)(px[t] & 0xfffu), span = (int)((px[t] >> 12) & 0xfffu);
            int lo = first - 1 - kb, hi = first + span - kb;                          // knots kb + lo .. kb + hi - 1 (0-based) carry the row
            lo = lo < 0 ? 0 : lo; hi = hi > nk ? nk : hi;
            act[t] = (hi > lo && i < n) ? ((0xFFFFu >> (16 - (hi - lo))) << lo) : 0u;
            ls[t] = (int)((px[t] >> 24) & 0x7fu);
            lp[t] = lam_b + (int)(py[t] + (unsigned)(kb + 1) * (unsigned)ls[t]);
        }
        // ---- phase A: the state entries (lanes 0..12) ---------------------------------------------------------------------------------
        const double* __restrict__ zp = Xb + (size_t)kb * n + (i < n ? i : 0);
        for (int k0 = 0; k0 < nk; k0 += 4) {
            double zi[4], lam[4][TO_EXP_MAXT];
            const unsigned a0 = act[0] >> k0, a1 = act[1] >> k0, a2 = act[2] >> k0;
#pragma unroll
            for (int u = 0; u < 4; u++) {
                const int kk = k0 + u;
                zi[u] = 0.0; lam[u][0] = 0.0; lam[u][1] = 0.0; lam[u][2] = 0.0;
                if (kk < nk && i < n) zi[u] = __ldg(zp + kk * n);
                if ((a0 >> u) & 1u) lam[u][0] = __ldg(lp[0] + kk * ls[0]);
                if ((a1 >> u) & 1u) lam[u][1] = __ldg(lp[1] + kk * ls[1]);
                if ((a2 >> u) & 1u) lam[u][2] = __ldg(lp[2] + kk * ls[2]);
            }
#pragma unroll
            for (int u = 0; u < 4; u++) {
                if (k0 + u >= nk) break;                                               // (uniform over the group)
                const int cid = __shfl_sync(gm, mycid, k0 + u, 16);
                if (i < n) {
                    if (cid != ccid) { const CostData c = cost_data<INST>(P, b, cid); ca = c.Qd[i]; cb = c.q[i]; ccid = cid; }
                    double g = fma(ca, zi[u], cb), h = ca;
#pragma unroll
                    for (int t = 0; t < TO_EXP_MAXT; t++) {
                        if ((((t == 0) ? a0 : (t == 1) ? a1 : a2) >> u) & 1u) {
                            const double lb = fma(nms[t], zi[u] - bnd[t], lam[u][t]);   // lambda - mu c
                            if ((px[t] >> 31) || lb <= 0.0) { g += (nms[t] < 0.0) ? -lb : lb; h += fabs(nms[t]); }   // g -= sign lb ; h += mu
                        }
                    }
                    double* row = stage[k0 + u];
                    if (quat) { double* a = row + HB_ + 3 * (i - qs); a[0] = g; a[1] = h; a[2] = zi[u]; }   // (g, h, q) of q_w..q_z wait in Hb[0..11] for phase B
                    else {
                        row[G_ + pme] = g; row[HD_ + pme] = h;
                        if (e == 7) { row[HB_ + 12] = 0.0; row[HB_ + 13] = 0.0; row[HB_ + 14] = 0.0; row[HB_ + 15] = h; }   // p = 14 is row 3 of Hb
                    }
                }
            }
        }
        __syncwarp(gm);
        if (i < nk) {
            double* row = stage[i];
            // ---- phase B: attitude block of knot kb + i ---------------------------------------------------------------------------
            double gq[4], hq[4], q[4];
#pragma unroll
            for (int r = 0; r < 4; r++) { gq[r] = row[HB_ + 3 * r]; hq[r] = row[HB_ + 3 * r + 1]; q[r] = row[HB_ + 3 * r + 2]; }
            // rows of G' = (L(q) H)': (-x,w,z,-y), (-y,-z,w,x), (-z,y,-x,w)
            const double G0[4] = {-q[1], q[0], q[3], -q[2]}, G1[4] = {-q[2], -q[3], q[0], q[1]}, G2[4] = {-q[3], q[2], -q[1], q[0]};
#pragma unroll
            for (int cc = 0; cc < 3; cc++) {
                double gc[4];
#pragma unroll
                for (int r = 0; r < 4; r++) gc[r] = (cc == 0) ? G0[r] : (cc == 1) ? G1[r] : G2[r];
                double qb = 0.0, ge = 0.0, hb0 = 0.0, hb1 = 0.0, hb2 = 0.0;
#pragma unroll
                for (int r = 0; r < 4; r++) {
                    qb += q[r] * gq[r]; ge += gc[r] * gq[r];
                    const double tt = gc[r] * hq[r];
                    hb0 += tt * G0[r]; hb1 += tt * G1[r]; hb2 += tt * G2[r];
                }
                const double hd = ((cc == 0) ? hb0 : (cc == 1) ? hb1 : hb2) - qb;
                const int p = 8 + 2 * cc;                                             // attitude error e = 3 + c sits on p = 8, 10, 12 (frag_layout.cuh)
                row[G_ + p] = ge; row[HD_ + p] = hd;
                row[HB_ + 4 * cc + 0] = (cc == 0) ? hd : hb0;
                row[HB_ + 4 * cc + 1] = (cc == 1) ? hd : hb1;
                row[HB_ + 4 * cc + 2] = (cc == 2) ? hd : hb2;
                row[HB_ + 4 * cc + 3] = 0.0;
            }
            // ---- phase C: the control entries of knot kb + i (coordinate 12 + a, physical slot 2a) ----------------------------------
            const int k = kb + i;
            const CostData c = cost_data<INST>(P, b, mycid);
            const double* cr = c.r;
            double zu[m], lu[m][TO_EXP_MAXT];
#pragma unroll
            for (int a = 0; a < m; a++) {                                             // every load of the phase first
                zu[a] = (k != N - 1) ? __ldg(Ub + (size_t)k * m + a) : 0.0;
#pragma unroll
                for (int t = 0; t < TO_EXP_MAXT; t++) {
                    const unsigned rx = __ldg(&tab.pkx[t][n + a]);
                    lu[a][t] = (k != N - 1 && (unsigned)(k + 1) - (rx & 0xfffu) <= ((rx >> 12) & 0xfffu))
                                   ? __ldg(lam_b + (int)(__ldg(&tab.pky[t][n + a]) + (unsigned)(k + 1) * ((rx >> 24) & 0x7fu))) : 0.0;
                }
            }
#pragma unroll
            for (int a = 0; a < m; a++) {
                double g = 0.0, h = 0.0;
                if (k != N - 1) {
                    g = fma(c.Rd[a], zu[a], cr[a]); h = c.Rd[a];
#pragma unroll
                    for (int t = 0; t < TO_EXP_MAXT; t++) {
                        const unsigned rx = __ldg(&tab.pkx[t][n + a]);
                        if ((unsigned)(k + 1) - (rx & 0xfffu) <= ((rx >> 12) & 0xfffu)) {
                            double rn = __ldg(&tab.nms[t][n + a]);
                            double bd = __ldg(&tab.bound[t][n + a]);
                            if constexpr (INST) { bd = exp_term_bound(P, tab, b, t, n + a, bd); rn = exp_term_nms(P, tab, b, t, n + a, rn); }
                            const double lb = fma(rn, zu[a] - bd, lu[a][t]);
                            if ((rx >> 31) || lb <= 0.0) { g += (rn < 0.0) ? -lb : lb; h += fabs(rn); }
                        }
                    }
                }
                row[G_ + 2 * a] = g; row[HD_ + 2 * a] = h;
            }
        }
        __syncwarp(gm);
        // ---- write-out: 384 contiguous bytes per knot, 16 bytes per lane and store -------------------------------------------------------
        for (int kk = 0; kk < nk; kk++) {
            const double* row = stage[kk];
            double* dst = recb + (size_t)kk * TO_REC_LEN;
            *reinterpret_cast<double2*>(dst + 2 * i) = make_double2(row[2 * i], row[2 * i + 1]);
            if (i < 8) *reinterpret_cast<double2*>(dst + 32 + 2 * i) = make_double2(row[32 + 2 * i], row[33 + 2 * i]);
        }
        __syncwarp(gm);                                                               // the stage is free again
    }
}
cudaError_t launch_expansion_rec16(const DevProblem& P, cudaStream_t s, int mode) {
    int dev = 0, sms = 132; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    // blocks of 16 knots, one 16-lane group each
    const long long units = (long long)P.B * ((P.N + 15) / 16);
    constexpr int GPB = TO_CEXP2_THREADS / 16;                                       // 16-lane groups per CTA
    long long blocks = (units + GPB - 1) / GPB;
    if (blocks < sms) blocks = sms;
    if (inst_backward(P)) k_expansion_rec16b<true><<<(unsigned)blocks, TO_CEXP2_THREADS, 0, s>>>(P, mode);
    else k_expansion_rec16b<false><<<(unsigned)blocks, TO_CEXP2_THREADS, 0, s>>>(P, mode);
    return cudaGetLastError();
}

#endif  // TO_RULE == 4

template <int RULE>
cudaError_t launch_expand_lie_rule(const DevProblem& P, cudaStream_t s, int mode) {
    if (P.model != MODEL_QUADROTOR) return cudaErrorNotSupported;
    const long long total = (long long)P.B * (P.N - 1) * 10;      // 10 dual-number seeds per knot (k_expand_lie: seed pruning)
    static_assert(fraglayout::phys_z(0) == 1 && fraglayout::phys_z(5) == 12 && fraglayout::phys_z(11) == 15 && fraglayout::phys_z(12) == 0 && fraglayout::phys_z(15) == 6, "nibble table of k_expand_lie_rec and k_expansion_rec16b");
    constexpr int T = TO_EXPAND_LIE_THREADS;
    if (P.frag) {
        // one CTA per (instance, block of EXPB_KPB knots); mode 2 with the late list: the first *late_count instance slots carry work
        const int nkb = (P.N - 1 + EXPB_KPB - 1) / EXPB_KPB;
        const unsigned blocks = (unsigned)((long long)P.B * nkb);
        if (inst_dynamics(P)) k_expand_lie_rec<MODEL_QUADROTOR, true, RULE><<<blocks, EXPB_T, 0, s>>>(P, mode, nkb);
        else k_expand_lie_rec<MODEL_QUADROTOR, false, RULE><<<blocks, EXPB_T, 0, s>>>(P, mode, nkb);
    } else if (inst_dynamics(P)) k_expand_lie<MODEL_QUADROTOR, true, RULE><<<(unsigned)((total + T - 1) / T), T, 0, s>>>(P, mode);
    else k_expand_lie<MODEL_QUADROTOR, false, RULE><<<(unsigned)((total + T - 1) / T), T, 0, s>>>(P, mode);
    return cudaGetLastError();
}

// the dynamics kernels read nothing per instance but the model parameters and the time steps: their INST variant runs exactly when a table exists
template <int RULE>
cudaError_t launch_rollout_rule(const DevProblem& P, cudaStream_t s, bool masked) {
    const int threads = 32, blocks = (P.B + threads - 1) / threads;
    if (masked) {
        if (inst_dynamics(P)) { TO_DISPATCH_MODEL(P.model, P.m, (k_rollout<MODEL, true, RULE, true><<<blocks, threads, 0, s>>>(P))); }
        else { TO_DISPATCH_MODEL(P.model, P.m, (k_rollout<MODEL, false, RULE, true><<<blocks, threads, 0, s>>>(P))); }
    } else if (inst_dynamics(P)) { TO_DISPATCH_MODEL(P.model, P.m, (k_rollout<MODEL, true, RULE><<<blocks, threads, 0, s>>>(P))); }
    else { TO_DISPATCH_MODEL(P.model, P.m, (k_rollout<MODEL, false, RULE><<<blocks, threads, 0, s>>>(P))); }
    return cudaGetLastError();
}

template <int MODEL, int NP, int RULE>
static cudaError_t launch_expand_t(const DevProblem& P, cudaStream_t s, int mode) {
    constexpr int TPK = (SeedList<MODEL>::count + NP - 1) / NP;
    const long long total = (long long)P.B * (P.N - 1) * TPK;
    const int threads = 128;
    const unsigned blocks = (unsigned)((total + threads - 1) / threads);
    if (inst_dynamics(P)) k_expand<MODEL, NP, true, RULE><<<blocks, threads, 0, s>>>(P, mode);
    else k_expand<MODEL, NP, false, RULE><<<blocks, threads, 0, s>>>(P, mode);
    return cudaGetLastError();
}

template <int RULE>
cudaError_t launch_expand_rule(const DevProblem& P, cudaStream_t s, int mode) {
    // seeds per thread: 1 (value recomputed per seed) or 2 (value shared by two seeds, more registers)
    static int np = -1;
    if (np < 0) { const char* v = getenv("TO_EXPAND_SEEDS"); np = v ? atoi(v) : 1; }
    cudaError_t e = cudaErrorNotSupported;
    if (np == 2) { TO_DISPATCH_MODEL(P.model, P.m, (e = launch_expand_t<MODEL, 2, RULE>(P, s, mode))); }
    else { TO_DISPATCH_MODEL(P.model, P.m, (e = launch_expand_t<MODEL, 1, RULE>(P, s, mode))); }
    return e;
}

// the plant's parameters: its own rows when to_mpc_setup was given them, else the planner's (per instance when set); the INST variant runs
// exactly when k_rollout's would on a problem holding those rows and the planner's time steps
template <int RULE>
cudaError_t launch_mpc_advance_rule(const DevProblem& P, const MpcDev& M, int j, cudaStream_t s) {
    DevProblem Q = P;
    if (M.plant) Q.mparams = M.plant;
    if (inst_dynamics(Q)) { TO_DISPATCH_MODEL(Q.model, Q.m, (k_mpc_advance<MODEL, true, RULE><<<Q.B, 128, 0, s>>>(Q, M, j, 2))); }
    else { TO_DISPATCH_MODEL(Q.model, Q.m, (k_mpc_advance<MODEL, false, RULE><<<Q.B, 128, 0, s>>>(Q, M, j, 2))); }
    return cudaGetLastError();
}

template cudaError_t launch_expand_lie_rule<TO_RULE>(const DevProblem&, cudaStream_t, int);
template cudaError_t launch_rollout_rule<TO_RULE>(const DevProblem&, cudaStream_t, bool);
template cudaError_t launch_expand_rule<TO_RULE>(const DevProblem&, cudaStream_t, int);
template cudaError_t launch_mpc_advance_rule<TO_RULE>(const DevProblem&, const MpcDev&, int, cudaStream_t);

#if TO_RULE == 4
cudaError_t launch_expand_lie(const DevProblem& P, cudaStream_t s, int mode) {
    cudaError_t e = cudaErrorNotSupported;
    TO_DISPATCH_RULE(P.integration, (e = launch_expand_lie_rule<RULE>(P, s, mode)));
    return e;
}
cudaError_t launch_rollout(const DevProblem& P, cudaStream_t s, bool masked) {
    cudaError_t e = cudaErrorNotSupported;
    TO_DISPATCH_RULE(P.integration, (e = launch_rollout_rule<RULE>(P, s, masked)));
    return e;
}
cudaError_t launch_expand(const DevProblem& P, cudaStream_t s, int mode) {
    cudaError_t e = cudaErrorNotSupported;
    TO_DISPATCH_RULE(P.integration, (e = launch_expand_rule<RULE>(P, s, mode)));
    return e;
}
cudaError_t launch_mpc_advance(const DevProblem& P, const MpcDev& M, int j, cudaStream_t s) {
    cudaError_t e = cudaErrorNotSupported;
    TO_DISPATCH_RULE(P.integration, (e = launch_mpc_advance_rule<RULE>(P, M, j, s)));
    return e;
}
#endif
