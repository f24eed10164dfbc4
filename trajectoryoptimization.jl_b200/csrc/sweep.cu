// sweep.cu -- kernel 2 of the hot path: the cost + constraint + augmented-Lagrangian sweep over all knots of
// all instances, plus the small layout/utility kernels of the C ABI.
//
//   k_cost      : cost!(obj, Z) / cost(obj, Z)              reference src/objective.jl:89-110
//                 per-knot J_k = l_k(x_k,u_k) for all k (independent), then the per-instance sum.  One CTA per
//                 instance; the knot loop is strided over the CTA, the reduction over knots uses warp shuffles.
//   k_merit     : cost + conic AL penalty + max constraint violation per instance (what a solver's line search
//                 and convergence test read); AL building blocks: src/cones.jl, write-up test/socp.jl:52-82.
//   k_eval_constraints / k_constraint_jacobians
//               : evaluate_constraints! / constraint_jacobians!   src/abstract_constraint.jl:200-248
//   k_cost_gradient / k_cost_hessian : RD.gradient! / RD.hessian! over the trajectory  src/cost_functions.jl:137-233
//   k_projection ... : projection! / grad-projection! / hess-projection!  src/cones.jl:96-276
//   k_al_update : dual update lambda <- Pi_{K*}(lambda - mu c)
#include "costcon.cuh"
#include "kernels.h"

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// INST (here and below): per-instance linear cost terms / Goal values, a variant of its own so that the shared one stays as it is
template <bool WITH_AL, bool INST>
__global__ void __launch_bounds__(128) k_cost(const DevProblem P, double* __restrict__ J, double* __restrict__ Jk,
                                              double* __restrict__ viol_out) {
    const int b = blockIdx.x;
    if (retired(P, b)) return;          // to_solve: not ACTIVE (uniform over the CTA)
    const int n = P.n, m = P.m, N = P.N;
    const double* X = traj_X(P, P.cur[b], b);
    const double* U = traj_U(P, P.cur[b], b);
    const double* lam = P.lambda + (size_t)b * P.lambda_len;
    double acc = 0, viol = 0;
    for (int k = threadIdx.x; k < N; k += blockDim.x) {
        const bool last = (k == N - 1);
        double zero_u[TO_MAXM];
        for (int i = 0; i < m; i++) zero_u[i] = 0.0;
        const double* u = last ? zero_u : U + (size_t)k * m;
        const int cid = P.cost_index[k];
        double v = cost_value(P.costs[cid], inst_q<INST>(P, b, cid), inst_r<INST>(P, b, cid), n, m, X + (size_t)k * n, u, !last);
        if (Jk) Jk[(size_t)b * N + k] = v;
        if (WITH_AL) v += al_knot_penalty<INST>(P, k + 1, X + (size_t)k * n, u, lam, viol, b);
        acc += v;
    }
    __shared__ double s_sum[4], s_max[4];
    acc = warp_sum(acc);
    viol = warp_max(viol);
    if ((threadIdx.x & 31) == 0) { s_sum[threadIdx.x >> 5] = acc; s_max[threadIdx.x >> 5] = viol; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0, vm = 0;
        for (int w = 0; w < (blockDim.x >> 5); w++) { t += s_sum[w]; vm = fmax(vm, s_max[w]); }
        if (J) J[b] = t;
        if (viol_out) viol_out[b] = vm;
    }
}

template <bool INST>
__global__ void k_cost_gradient(const DevProblem P, double* __restrict__ grad) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)P.B * P.N) return;
    const int k = (int)(t % P.N), b = (int)(t / P.N);
    const int n = P.n, m = P.m, nm = n + m;
    const bool last = (k == P.N - 1);
    double zero_u[TO_MAXM] = {0};
    const double* x = traj_X(P, P.cur[b], b) + (size_t)k * n;
    const double* u = last ? zero_u : traj_U(P, P.cur[b], b) + (size_t)k * m;
    double g[TO_MAXNM];
    for (int i = 0; i < nm; i++) g[i] = 0;
    const int cid = P.cost_index[k];
    cost_gradient(P.costs[cid], inst_q<INST>(P, b, cid), inst_r<INST>(P, b, cid), n, m, x, u, last, g);
    for (int i = 0; i < nm; i++) grad[t * nm + i] = g[i];
}

__global__ void k_cost_hessian(const DevProblem P, double* __restrict__ hess) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)P.B * P.N) return;
    const int k = (int)(t % P.N), b = (int)(t / P.N);
    const int nm = P.n + P.m;
    const bool last = (k == P.N - 1);
    double zero_u[TO_MAXM] = {0};
    const double* x = traj_X(P, P.cur[b], b) + (size_t)k * P.n;
    const double* u = last ? zero_u : traj_U(P, P.cur[b], b) + (size_t)k * P.m;
    cost_hessian(P.costs[P.cost_index[k]], P.n, P.m, x, u, last, hess + t * nm * nm);
}

template <bool INST>
__global__ void k_al_expansion(const DevProblem P, double* __restrict__ grad, double* __restrict__ hess) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)P.B * P.N) return;
    const int k = (int)(t % P.N), b = (int)(t / P.N);
    const int n = P.n, m = P.m, nm = n + m;
    const bool last = (k == P.N - 1);
    double zero_u[TO_MAXM] = {0};
    const double* x = traj_X(P, P.cur[b], b) + (size_t)k * n;
    const double* u = last ? zero_u : traj_U(P, P.cur[b], b) + (size_t)k * m;
    al_knot_expansion<INST>(P, k, x, u, P.lambda + (size_t)b * P.lambda_len, grad + t * nm, hess + t * nm * nm, b);
}

template <bool INST>
__global__ void k_eval_constraints(const DevProblem P, int ci, double* __restrict__ vals) {
    const DevCon& con = P.cons[ci];
    const int len = con.last - con.first + 1;
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)P.B * len) return;
    const int ki = (int)(t % len), b = (int)(t / len);
    const int k1 = con.first + ki;
    double zero_u[TO_MAXM] = {0};
    const double* x = traj_X(P, P.cur[b], b) + (size_t)(k1 - 1) * P.n;
    const double* u = (k1 == P.N) ? zero_u : traj_U(P, P.cur[b], b) + (size_t)(k1 - 1) * P.m;
    double c[TO_MAXPV];
    con_evaluate_b<INST>(P, con, b, ci, P.n, P.m, x, u, c);
    for (int i = 0; i < con.p; i++) vals[t * con.p + i] = c[i];
}

// lam_in: [B][len][p] or nullptr = the handle's multipliers
__global__ void k_constraint_hessians(const DevProblem P, int ci, const double* __restrict__ lam_in, double* __restrict__ H) {
    const DevCon& con = P.cons[ci];
    const int len = con.last - con.first + 1, w = P.n + P.m;
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)P.B * len) return;
    const int ki = (int)(t % len), b = (int)(t / len);
    const int k1 = con.first + ki;
    double zero_u[TO_MAXM] = {0};
    const double* x = traj_X(P, P.cur[b], b) + (size_t)(k1 - 1) * P.n;
    const double* u = (k1 == P.N) ? zero_u : traj_U(P, P.cur[b], b) + (size_t)(k1 - 1) * P.m;
    const double* lam = lam_in ? lam_in + t * con.p : P.lambda + (size_t)b * P.lambda_len + con.offset + (size_t)ki * con.p;
    con_hess_vec(con, P.n, P.m, x, u, lam, H + t * w * w);
}

template <bool INST>
__global__ void k_constraint_jacobians(const DevProblem P, int ci, double* __restrict__ jac) {
    const DevCon& con = P.cons[ci];
    const int len = con.last - con.first + 1;
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)P.B * len) return;
    const int ki = (int)(t % len), b = (int)(t / len);
    const int k1 = con.first + ki;
    double zero_u[TO_MAXM] = {0};
    const double* x = traj_X(P, P.cur[b], b) + (size_t)(k1 - 1) * P.n;
    const double* u = (k1 == P.N) ? zero_u : traj_U(P, P.cur[b], b) + (size_t)(k1 - 1) * P.m;
    con_jacobian_b<INST>(P, con, b, ci, P.n, P.m, x, u, jac + t * con.p * (P.n + P.m));
}

__global__ void k_projection(int cone, int p, int count, const double* __restrict__ x, double* __restrict__ px, int* err) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= count) return;
    if (cone_projection(cone, x + (size_t)t * p, p, px + (size_t)t * p)) atomicExch(err, 1);
}
__global__ void k_grad_projection(int cone, int p, int count, const double* __restrict__ x, double* __restrict__ J, int* err) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= count) return;
    if (cone_grad_projection(cone, x + (size_t)t * p, p, J + (size_t)t * p * p)) atomicExch(err, 1);
}
__global__ void k_hess_projection(int cone, int p, int count, const double* __restrict__ x, const double* __restrict__ b,
                                  double* __restrict__ H, int* err) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= count) return;
    if (cone_hess_projection(cone, x + (size_t)t * p, b + (size_t)t * p, p, H + (size_t)t * p * p)) atomicExch(err, 1);
}

// dual update: lambda <- clamp(Pi_{K*}(lambda - mu c)); one thread per (instance, constraint, knot)
template <bool INST>
__global__ void k_al_update(const DevProblem P) {
    const int b = blockIdx.x;
    if (retired(P, b)) return;          // to_solve: only the instances that go on to another outer iteration
    double* lam_b = P.lambda + (size_t)b * P.lambda_len;
    const double* X = traj_X(P, P.cur[b], b);
    const double* U = traj_U(P, P.cur[b], b);
    double zero_u[TO_MAXM] = {0};
    for (int ci = 0; ci < P.ncon; ci++) {
        const DevCon& con = P.cons[ci];
        const double mu = P.mu[ci];
        for (int k1 = con.first + threadIdx.x; k1 <= con.last; k1 += blockDim.x) {
            const double* x = X + (size_t)(k1 - 1) * P.n;
            const double* u = (k1 == P.N) ? zero_u : U + (size_t)(k1 - 1) * P.m;
            double c[TO_MAXPV], lbar[TO_MAXPV], lp[TO_MAXPV];
            double* lam = lam_b + con.offset + (size_t)(k1 - con.first) * con.p;
            con_evaluate_b<INST>(P, con, b, ci, P.n, P.m, x, u, c);
            for (int i = 0; i < con.p; i++) lbar[i] = lam[i] - mu * c[i];
            cone_projection(dualcone(con.sense), lbar, con.p, lp);
            for (int i = 0; i < con.p; i++) lam[i] = fmax(-P.opt.dual_max, fmin(P.opt.dual_max, lp[i]));
        }
    }
    if (threadIdx.x == 0) { P.rho[b] = P.opt.bp_reg_initial; P.drho[b] = 0.0; }
}

// {sum_b J_b, max_b viol_b} for the cross-GPU merit all-reduce (SURVEY 8e)
__global__ void __launch_bounds__(1024) k_reduce_merit(int B, const double* __restrict__ J, const double* __restrict__ viol, double* out2) {
    double acc = 0, vm = 0;
    for (int b = threadIdx.x; b < B; b += blockDim.x) { acc += J[b]; if (viol) vm = fmax(vm, viol[b]); }
    __shared__ double s_sum[32], s_max[32];
    acc = warp_sum(acc); vm = warp_max(vm);
    if ((threadIdx.x & 31) == 0) { s_sum[threadIdx.x >> 5] = acc; s_max[threadIdx.x >> 5] = vm; }
    __syncthreads();
    if (threadIdx.x < 32) {
        acc = threadIdx.x < (blockDim.x >> 5) ? s_sum[threadIdx.x] : 0.0;
        vm = threadIdx.x < (blockDim.x >> 5) ? s_max[threadIdx.x] : 0.0;
        acc = warp_sum(acc); vm = warp_max(vm);
        if (threadIdx.x == 0) { out2[0] = acc; out2[1] = vm; }
    }
}

// copy the live trajectory buffer of every instance to/from a dense staging buffer
__global__ void k_gather_traj(const DevProblem P, double* __restrict__ Xout, double* __restrict__ Uout) {
    const int b = blockIdx.x;
    const int nx = P.N * P.n, nu = (P.N - 1) * P.m;
    const double* X = traj_X(P, P.cur[b], b);
    const double* U = traj_U(P, P.cur[b], b);
    if (Xout) for (int i = threadIdx.x; i < nx; i += blockDim.x) Xout[(size_t)b * nx + i] = X[i];
    if (Uout) for (int i = threadIdx.x; i < nu; i += blockDim.x) Uout[(size_t)b * nu + i] = U[i];
}
__global__ void k_scatter_traj(const DevProblem P, const double* __restrict__ Xin, const double* __restrict__ Uin) {
    const int b = blockIdx.x;
    const int nx = P.N * P.n, nu = (P.N - 1) * P.m;
    double* X = traj_Xw(P, P.cur[b], b);
    double* U = traj_Uw(P, P.cur[b], b);
    if (Xin) for (int i = threadIdx.x; i < nx; i += blockDim.x) X[i] = Xin[(size_t)b * nx + i];
    if (Uin) for (int i = threadIdx.x; i < nu; i += blockDim.x) U[i] = Uin[(size_t)b * nu + i];
}
// device AB (row-major, padded rows) -> Julia layout n x (n+m) column-major
__global__ void k_export_ab(const DevProblem P, double* __restrict__ out) {
    const int n = P.n, nm = P.n + P.m, ld = P.ldab;
    const size_t blk = blockIdx.x;   // (b, k) flattened
    const double* AB = P.AB + blk * n * ld;
    for (int e = threadIdx.x; e < n * nm; e += blockDim.x) {
        const int j = e / n, i = e % n;
        out[blk * n * nm + e] = AB[i * ld + j];
    }
}

// ------------------------------------------------------------------------------------------------------
static inline unsigned nblk(long long total, int threads) { return (unsigned)((total + threads - 1) / threads); }

cudaError_t launch_cost(const DevProblem& P, double* J, double* Jk, cudaStream_t s) {
    if (inst_backward(P)) k_cost<false, true><<<P.B, 128, 0, s>>>(P, J, Jk, nullptr);
    else k_cost<false, false><<<P.B, 128, 0, s>>>(P, J, Jk, nullptr);
    return cudaGetLastError();
}
cudaError_t launch_merit(const DevProblem& P, double* J, double* viol, cudaStream_t s) {
    if (inst_backward(P)) k_cost<true, true><<<P.B, 128, 0, s>>>(P, J, nullptr, viol);
    else k_cost<true, false><<<P.B, 128, 0, s>>>(P, J, nullptr, viol);
    return cudaGetLastError();
}
cudaError_t launch_cost_gradient(const DevProblem& P, double* grad, cudaStream_t s) {
    if (inst_backward(P)) k_cost_gradient<true><<<nblk((long long)P.B * P.N, 128), 128, 0, s>>>(P, grad);
    else k_cost_gradient<false><<<nblk((long long)P.B * P.N, 128), 128, 0, s>>>(P, grad);
    return cudaGetLastError();
}
cudaError_t launch_cost_hessian(const DevProblem& P, double* hess, cudaStream_t s) {
    k_cost_hessian<<<nblk((long long)P.B * P.N, 128), 128, 0, s>>>(P, hess);
    return cudaGetLastError();
}
cudaError_t launch_al_expansion(const DevProblem& P, double* grad, double* hess, cudaStream_t s) {
    if (inst_backward(P)) k_al_expansion<true><<<nblk((long long)P.B * P.N, 64), 64, 0, s>>>(P, grad, hess);
    else k_al_expansion<false><<<nblk((long long)P.B * P.N, 64), 64, 0, s>>>(P, grad, hess);
    return cudaGetLastError();
}
cudaError_t launch_eval_constraints(const DevProblem& P, int con, double* vals, cudaStream_t s) {
    // the knot-range length is read on the device; size the grid for the worst case N
    if (inst_backward(P)) k_eval_constraints<true><<<nblk((long long)P.B * P.N, 128), 128, 0, s>>>(P, con, vals);
    else k_eval_constraints<false><<<nblk((long long)P.B * P.N, 128), 128, 0, s>>>(P, con, vals);
    return cudaGetLastError();
}
cudaError_t launch_constraint_hessians(const DevProblem& P, int con, int len, const double* lam, double* H, cudaStream_t s) {
    const long long total = (long long)P.B * len;
    k_constraint_hessians<<<(unsigned)((total + 127) / 128), 128, 0, s>>>(P, con, lam, H);
    return cudaGetLastError();
}
cudaError_t launch_constraint_jacobians(const DevProblem& P, int con, double* jac, cudaStream_t s) {
    if (inst_backward(P)) k_constraint_jacobians<true><<<nblk((long long)P.B * P.N, 128), 128, 0, s>>>(P, con, jac);
    else k_constraint_jacobians<false><<<nblk((long long)P.B * P.N, 128), 128, 0, s>>>(P, con, jac);
    return cudaGetLastError();
}
cudaError_t launch_projection(int cone, int p, int count, const double* x, double* px, int* err, cudaStream_t s) {
    k_projection<<<nblk(count, 128), 128, 0, s>>>(cone, p, count, x, px, err);
    return cudaGetLastError();
}
cudaError_t launch_grad_projection(int cone, int p, int count, const double* x, double* J, int* err, cudaStream_t s) {
    k_grad_projection<<<nblk(count, 128), 128, 0, s>>>(cone, p, count, x, J, err);
    return cudaGetLastError();
}
cudaError_t launch_hess_projection(int cone, int p, int count, const double* x, const double* b, double* H, int* err, cudaStream_t s) {
    k_hess_projection<<<nblk(count, 128), 128, 0, s>>>(cone, p, count, x, b, H, err);
    return cudaGetLastError();
}
cudaError_t launch_al_update(const DevProblem& P, cudaStream_t s) {
    if (inst_backward(P)) k_al_update<true><<<P.B, 128, 0, s>>>(P);
    else k_al_update<false><<<P.B, 128, 0, s>>>(P);
    return cudaGetLastError();
}
cudaError_t launch_reduce_merit(const DevProblem& P, const double* viol, double* out2, cudaStream_t s) {
    k_reduce_merit<<<1, 1024, 0, s>>>(P.B, P.J, viol, out2);
    return cudaGetLastError();
}
// receding-horizon shift (to_shift_trajectory): CTA = instance; the trajectory goes to the next ring buffer, the
// multipliers shift in place (thread = one row of one constraint, ascending knots: reads k+steps, writes k)
__global__ void k_shift_traj(const DevProblem P, int steps) {
    const int b = blockIdx.x, n = P.n, m = P.m, N = P.N;
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
cudaError_t launch_shift_traj(const DevProblem& P, int steps, cudaStream_t s) {
    k_shift_traj<<<P.B, 128, 0, s>>>(P, steps);
    return cudaGetLastError();
}

cudaError_t launch_gather_traj(const DevProblem& P, double* Xout, double* Uout, cudaStream_t s) {
    k_gather_traj<<<P.B, 128, 0, s>>>(P, Xout, Uout);
    return cudaGetLastError();
}
cudaError_t launch_scatter_traj(const DevProblem& P, const double* Xin, const double* Uin, cudaStream_t s) {
    k_scatter_traj<<<P.B, 128, 0, s>>>(P, Xin, Uin);
    return cudaGetLastError();
}
cudaError_t launch_export_ab(const DevProblem& P, double* ABout, cudaStream_t s) {
    k_export_ab<<<(unsigned)((size_t)P.B * (P.N - 1)), 128, 0, s>>>(P, ABout);
    return cudaGetLastError();
}
