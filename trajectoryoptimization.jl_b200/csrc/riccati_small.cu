// riccati_small.cu -- kernel 3 for small models (n <= 4, m <= 2: double integrator, Cartpole, Acrobot).
//
// Same recursion as riccati.cu (Altro.jl backwardpass!, restated in oracle/oracle.hpp `backward_pass`):
//     Qzz = lzz + [A B]' S [A B]      Qz = lz + [A B]' s
//     K = -(Quu + rho I)^-1 Qux       d = -(Quu + rho I)^-1 Qu        (non-PD Quu + rho I -> rho increase + restart)
//     S <- Qxx + W'K, s <- Qx + W'd with W = Qux - rho K              dV += (d'Qu, 1/2 d'Quu d)
// with the cost expansion of RD.gradient!/RD.hessian! (src/cost_functions.jl:137-233) and the AL terms of Goal / Bound
// constraints (src/constraints.jl:55-68, :738-765; projection src/cones.jl:96-145).
//
// Mapping: for these sizes a warp per instance spends its time in shuffles and shared-memory round trips for 4x5
// matrices.  Here ONE THREAD owns an instance: S, [A B]_k,
// T, Q and the gains live in registers with every loop unrolled at compile time, no synchronisation at all.  [A B]_k is a
// contiguous, 32-byte aligned run per thread (full sectors), prefetched one knot ahead into registers and four knots
// ahead into L2 (prefetch.global.L2), K/d are written as they are produced.  The kernel is HBM/latency-bound:
// 240 B and ~250 FMA per instance-knot.
#include <cstddef>

#include "common.cuh"
#include "costcon.cuh"
#include "kernels.h"

namespace {

__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

// cost + AL expansion of knot k0 (0-based) for Goal / Bound constraints: g[nm], H[nm*nm] col-major symmetric
// (INST: with the linear cost terms and Goal values of instance b)
template <int n, int m, bool INST>
__device__ __forceinline__ void expand_knot(const DevProblem& P, int b, int k0, const double* x, const double* u, const double* lam_b,
                                            double (&g)[n + m], double (&H)[(n + m) * (n + m)]) {
    constexpr int nm = n + m;
    const bool last = (k0 == P.N - 1);
    const int cid = P.cost_index[k0];
    const DevCost& cost = P.costs[cid];
#pragma unroll
    for (int i = 0; i < nm; i++) g[i] = 0.0;
    const CostData cd = cost_data<INST>(P, b, cid);
    cost_gradient_quadratic<false>(cost, cd, n, m, x, u, last, g);      // this kernel never sees user (program) costs: launch_backward routes them to lie.cu
    cost_hessian_quadratic<INST>(cost, cd, n, m, last, H);
    double z[nm];
#pragma unroll
    for (int i = 0; i < n; i++) z[i] = x[i];
#pragma unroll
    for (int i = 0; i < m; i++) z[n + i] = last ? 0.0 : u[i];
    const int lim = last ? n : nm;
    for (int ci = 0; ci < P.ncon; ci++) {
        const DevCon& con = P.cons[ci];
        if (k0 + 1 < con.first || k0 + 1 > con.last) continue;
        const double mu = penalty<INST>(P, b, ci);
        const double* lam = lam_b + con.offset + (size_t)(k0 + 1 - con.first) * con.p;
        const ConData cd = con_data<INST>(P, b, ci);
        if (con.kind == CON_GOAL) {
            const double* ga = cd.a;
            for (int r = 0; r < con.p; r++) {
                const int j = con.inds[r];
#pragma unroll
                for (int i = 0; i < n; i++) if (i == j) { const double lb = lam[r] - mu * (x[i] - ga[r]); g[i] -= lb; H[i * nm + i] += mu; }
            }
        } else {   // CON_BOUND: upper block, then lower block
            for (int r = 0; r < con.n_max; r++) {
                const int j = con.a_max[r];
                if (j >= lim) continue;
#pragma unroll
                for (int i = 0; i < nm; i++) if (i == j) { const double lb = lam[r] - mu * (z[i] - cd.a[j]); if (lb <= 0.0) { g[i] -= lb; H[i * nm + i] += mu; } }
            }
            for (int r = 0; r < con.n_min; r++) {
                const int j = con.a_min[r];
                if (j >= lim) continue;
#pragma unroll
                for (int i = 0; i < nm; i++) if (i == j) { const double lb = lam[con.n_max + r] - mu * (cd.b[j] - z[i]); if (lb <= 0.0) { g[i] += lb; H[i * nm + i] += mu; } }
            }
        }
    }
}

template <int N_, int M_, bool INST>
__global__ void __maxnreg__(255) k_riccati_small(const DevProblem P) {
    constexpr int n = N_, m = M_, nm = n + m;
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= P.B || retired(P, b)) return;       // (to_solve: not ACTIVE)
    const int N = P.N, ld = P.ldab;
    const int buf = P.cur[b];
    const double* X = traj_X(P, buf, b);
    const double* U = traj_U(P, buf, b);
    const double* lam_b = P.lambda + (size_t)b * P.lambda_len;
    const double* ABg = P.AB + (size_t)b * (N - 1) * n * ld;
    double* Kg = P.K + (size_t)b * (N - 1) * n * m;
    double* dg = P.d + (size_t)b * (N - 1) * m;
    double rho = P.rho[b], drho = P.drho[b];
    int restarts = 0;
    bool failed = false;

    for (;;) {
        double S[n * n], s[n];   // col-major, kept fully symmetric
        {
            double g[nm], H[nm * nm];
            double xk[n];
#pragma unroll
            for (int i = 0; i < n; i++) xk[i] = X[(size_t)(N - 1) * n + i];
            expand_knot<n, m, INST>(P, b, N - 1, xk, xk, lam_b, g, H);   // u is not read at the terminal knot
#pragma unroll
            for (int j = 0; j < n; j++) {
                s[j] = g[j];
#pragma unroll
                for (int i = 0; i < n; i++) S[j * n + i] = H[j * nm + i];
            }
        }
        double dV1 = 0.0, dV2 = 0.0;
        bool ok = true;
        // [A B] of the first stage knot (row-major n x ld); later knots are loaded one iteration ahead
        double ab[n * nm];
        {
            const double* src = ABg + (size_t)(N - 2) * n * ld;
#pragma unroll
            for (int i = 0; i < n; i++)
#pragma unroll
                for (int j = 0; j < nm; j++) ab[i * nm + j] = src[i * ld + j];
        }
        int k;
        for (k = N - 2; k >= 0; k--) {
            if (k >= 4) { const char* pf = reinterpret_cast<const char*>(ABg + (size_t)(k - 4) * n * ld); prefetch_l2(pf); if (n * ld * 8 > 128) prefetch_l2(pf + 128); }
            double abn[n * nm];
            if (k > 0) {
                const double* src = ABg + (size_t)(k - 1) * n * ld;
#pragma unroll
                for (int i = 0; i < n; i++)
#pragma unroll
                    for (int j = 0; j < nm; j++) abn[i * nm + j] = src[i * ld + j];
            }
            // (a software-pipelined variant that expands knot k-1 at the end of iteration k was tried and not kept: the chain is
            //  bound by the dependent table look-ups of the expansion, not by the latency of x / u / lambda)
            double g[nm], H[nm * nm];
            {
                double xk[n], uk[m];
#pragma unroll
                for (int i = 0; i < n; i++) xk[i] = X[(size_t)k * n + i];
#pragma unroll
                for (int i = 0; i < m; i++) uk[i] = U[(size_t)k * m + i];
                expand_knot<n, m, INST>(P, b, k, xk, uk, lam_b, g, H);
            }
            // T = S [A B] (n x nm), ts = s
            double T[n * nm];
#pragma unroll
            for (int i = 0; i < n; i++)
#pragma unroll
                for (int j = 0; j < nm; j++) {
                    double t = 0.0;
#pragma unroll
                    for (int r = 0; r < n; r++) t = fma(S[r * n + i], ab[r * nm + j], t);
                    T[i * nm + j] = t;
                }
            // Q = H + [A B]' T (lower incl. diagonal, col-major Q[j*nm+i], i >= j) ; q = g + [A B]' s
            double Q[nm * nm], q[nm];
#pragma unroll
            for (int j = 0; j < nm; j++) {
                double t = g[j];
#pragma unroll
                for (int r = 0; r < n; r++) t = fma(ab[r * nm + j], s[r], t);
                q[j] = t;
#pragma unroll
                for (int i = j; i < nm; i++) {
                    double a = H[j * nm + i];
#pragma unroll
                    for (int r = 0; r < n; r++) a = fma(ab[r * nm + i], T[r * nm + j], a);
                    Q[j * nm + i] = a; Q[i * nm + j] = a;
                }
            }
            // gains: (Quu + rho I) [K d] = -[Qux Qu]   (m <= 2: Cholesky by hand)
            double Kc[m * n], dc[m];
            bool pd;
            if constexpr (m == 1) {
                const double p0 = Q[n * nm + n] + rho;
                pd = (p0 > 0.0) && isfinite(p0);
                const double inv = 1.0 / p0;
#pragma unroll
                for (int c = 0; c < n; c++) Kc[c] = -Q[c * nm + n] * inv;
                dc[0] = -q[n] * inv;
            } else {
                const double a = Q[n * nm + n] + rho, bq = Q[n * nm + n + 1], c2 = Q[(n + 1) * nm + n + 1] + rho;
                const double inva = 1.0 / a;
                const double l10 = bq * inva;
                const double d1 = c2 - l10 * bq;
                pd = (a > 0.0) && (d1 > 0.0) && isfinite(a) && isfinite(d1);
                const double invd1 = 1.0 / d1;
#pragma unroll
                for (int c = 0; c <= n; c++) {
                    const double r0 = (c < n) ? Q[c * nm + n] : q[n], r1 = (c < n) ? Q[c * nm + n + 1] : q[n + 1];
                    const double y0 = -r0, y1 = -r1 - l10 * y0;          // forward
                    const double x1 = y1 * invd1, x0 = y0 * inva - l10 * x1;   // diagonal + backward
                    if (c < n) { Kc[c * m] = x0; Kc[c * m + 1] = x1; } else { dc[0] = x0; dc[1] = x1; }
                }
            }
            if (!pd) { ok = false; break; }
#pragma unroll
            for (int c = 0; c < n; c++)
#pragma unroll
                for (int a = 0; a < m; a++) Kg[(size_t)k * n * m + c * m + a] = Kc[c * m + a];
#pragma unroll
            for (int a = 0; a < m; a++) dg[(size_t)k * m + a] = dc[a];
            // expected decrease
#pragma unroll
            for (int a = 0; a < m; a++) {
                dV1 = fma(dc[a], q[n + a], dV1);
                double qd = 0.0;
#pragma unroll
                for (int r = 0; r < m; r++) qd = fma(Q[(n + r) * nm + n + a], dc[r], qd);
                dV2 = fma(0.5 * dc[a], qd, dV2);
            }
            // S <- Qxx + W'K, s <- Qx + W'd with W = Qux - rho K (m x n)
            double W[m * n];
#pragma unroll
            for (int c = 0; c < n; c++)
#pragma unroll
                for (int a = 0; a < m; a++) W[c * m + a] = fma(-rho, Kc[c * m + a], Q[c * nm + n + a]);
#pragma unroll
            for (int j = 0; j < n; j++) {
                double t = q[j];
#pragma unroll
                for (int a = 0; a < m; a++) t = fma(W[j * m + a], dc[a], t);
                s[j] = t;
#pragma unroll
                for (int i = j; i < n; i++) {
                    double v = Q[j * nm + i];
#pragma unroll
                    for (int a = 0; a < m; a++) v = fma(W[i * m + a], Kc[j * m + a], v);
                    S[j * n + i] = v;
                }
            }
#pragma unroll
            for (int j = 0; j < n; j++)
#pragma unroll
                for (int i = j + 1; i < n; i++) S[i * n + j] = S[j * n + i];   // mirror the computed triangle
            if (k > 0) {
#pragma unroll
                for (int i = 0; i < n * nm; i++) ab[i] = abn[i];
            }
        }
        if (ok) { P.dV[2 * b] = dV1; P.dV[2 * b + 1] = dV2; break; }
        if (reg_restart(P.opt, rho, drho, restarts)) { failed = true; break; }
    }
    reg_finish(P, b, rho, drho, restarts, failed, 0);
}

template <int N_, int M_>
cudaError_t launch_small(const DevProblem& P, cudaStream_t s) {
    if (inst_backward(P)) k_riccati_small<N_, M_, true><<<(P.B + 31) / 32, 32, 0, s>>>(P);
    else k_riccati_small<N_, M_, false><<<(P.B + 31) / 32, 32, 0, s>>>(P);
    return cudaGetLastError();
}

}  // namespace

// thread-per-instance Riccati pass: small models with DiagonalCost / QuadraticCost and Goal / Bound constraints.
// Chosen automatically once the batch is larger than one wave of the warp-per-instance kernel (16 one-warp CTAs per SM, riccati.cu):
// up to that the warp kernel runs every instance at once and is faster.  One H100 (132 SMs, 400 W), Riccati pass warp vs thread:
// Cartpole N=101 B=1024 0.126 vs 0.186 ms, B=2048 0.162 vs 0.212, B=3072 0.278 vs 0.215, B=8192 0.596 vs 0.247;
// Acrobot N=201 B=2048 0.531 vs 0.569, B=4096 1.04 vs 0.58.
bool riccati_small_supported(const DevProblem& P, bool any_batch) {
    if (!(P.n <= 4 && P.m <= 2 && P.all_diag_con)) return false;
    if (any_batch) return true;
    static int sms[TO_MAXDEV] = {0};
    const int dev = current_device_slot();
    if (!sms[dev] && cudaDeviceGetAttribute(&sms[dev], cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) sms[dev] = 0;
    return sms[dev] > 0 && P.B > 16 * sms[dev];
}

cudaError_t launch_backward_small(const DevProblem& P, cudaStream_t s) {
    if (P.n == 4 && P.m == 1) return launch_small<4, 1>(P, s);
    if (P.n == 4 && P.m == 2) return launch_small<4, 2>(P, s);
    if (P.n == 2 && P.m == 1) return launch_small<2, 1>(P, s);
    return cudaErrorNotSupported;
}
