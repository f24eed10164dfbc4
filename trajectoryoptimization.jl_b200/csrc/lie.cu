// lie.cu -- Lie-group (quaternion) error state of the solver kernels (SURVEY.md 8 f2) and the Riccati pass that reads a
// MATERIALISED per-knot expansion.
//
// What it stands for.  Altro.jl solves rigid-body problems (RobotZoo.Quadrotor is a RobotDynamics `RigidBody` with a
// `LieState`) on the ERROR STATE: n_e = RD.errstate_dim(model) = 12 instead of n = 13.  Per iteration it builds
//     G_k   = errstate_jacobian(model, x_k) = blkdiag(I3, grad-differential(q_k), I6)            (Rotations.jl: L(q) H, 4 x 3)
//     [A_e B_e]_k = G_{k+1}' [A_k G_k | B_k]                                                     (error_expansion!(D, model, G))
//     E_k.x = G_k' lx ;  E_k.xx = G_k' lxx G_k + grad^2-differential(q_k, lx[q]) = ... - (q'lx[q]) I3 ;  E_k.ux = lux G_k
//                                                                                                (error_expansion!(E, Q, model, Z, G))
// runs the Riccati recursion on those, and feeds dx = RD.state_diff(model, xbar, x) (inverse Cayley map of q^-1 (x) qbar)
// through the gains in the forward pass.  None of that arithmetic is under /root/reference; what the reference holds is the
// constraint-side hook (error_expansion! of constraint Jacobians by G, src/abstract_constraint.jl:282-303), the quaternion cost
// DiagonalQuatCost (src/lie_costs.jl:33-95) and the attitude constraint QuatVecEq (src/constraints.jl:938-965) -- both of the
// latter are evaluated by costcon.cuh.  Restatement + finite-difference checks: oracle/oracle.hpp, tests/test_oracle_lie.py.
//
// Kernels
//   k_state_diff        RD.state_diff of every knot against the live trajectory (C ABI to_state_diff)
//   k_error_dynamics    [A_e B_e] from [A B] (rollout.cu k_expand) -- one thread per (instance, knot, column)
//   k_error_expansion   error-state cost + AL expansion from the full-state one (sweep.cu k_al_expansion) -- one thread per
//                       (instance, knot, column)
//   k_expansion_compact the compact error-state expansion EC of every knot (P.compact) -- one thread per (instance, knot)
//   k_riccati_dense     backward pass, one warp per instance, reading [A_e B_e]_k, E_k from HBM: 3.7 KB per knot instead of the
//                       2 KB of the fused kernel (riccati.cu), in exchange for taking ANY cost / constraint type -- the expansion
//                       is whatever the sweep kernels wrote.  DFMA on shared-memory operands, lane-strided.
//   k_riccati_dense_mma the same pass for n_e = 12, m = 4 on the FP64 tensor cores, on EG / EH or on EC
// Both backward passes take their gain step (LDL' of Quu + rho I, the solves, dV) from gains.cuh, as riccati.cu does.
#include "costcon.cuh"
#include "gains.cuh"
#include "kernels.h"
#include "ptx.cuh"

namespace {

__global__ void k_state_diff(const DevProblem P, const double* __restrict__ Xbar, double* __restrict__ dx) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)P.B * P.N) return;
    const int k = (int)(t % P.N), b = (int)(t / P.N);
    const double* x = traj_X(P, P.cur[b], b) + (size_t)k * P.n;
    double xb[TO_MAXN], xx[TO_MAXN], d[TO_MAXN];
    for (int i = 0; i < P.n; i++) { xb[i] = Xbar[t * P.n + i]; xx[i] = x[i]; }
    state_diff(P.lie != 0, P.n, P.qs, xb, xx, d);
    for (int i = 0; i < P.ne; i++) dx[t * P.ne + i] = d[i];
}

// column e (0 .. ne+m-1) of [A_e B_e]_k.  [A B] is row-major with row stride ldab (common.cuh); the output is col-major ne x (ne+m).
__global__ void __launch_bounds__(128) k_error_dynamics(const DevProblem P) {
    const int n = P.n, m = P.m, ne = P.ne, nme = ne + m, qs = P.qs, ld = P.ldab;
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)P.B * (P.N - 1) * nme) return;
    const int e = (int)(t % nme);
    const long long bk = t / nme;
    const int k = (int)(bk % (P.N - 1)), b = (int)(bk / (P.N - 1));
    const double* AB = P.AB + ((size_t)b * (P.N - 1) + k) * n * ld;
    const double* X = traj_X(P, P.cur[b], b);
    double col[TO_MAXN];                                   // column e of [A G_k | B]  (n entries)
    if (P.lie && e >= qs && e < qs + 3) {
        double G[12]; quat_G(X + (size_t)k * n + qs, G);
        const double* g = &G[(e - qs) * 4];
        for (int i = 0; i < n; i++) {
            double s = 0;
            for (int r = 0; r < 4; r++) s += AB[i * ld + qs + r] * g[r];
            col[i] = s;
        }
    } else {
        const int j = (!P.lie || e < qs) ? e : e + 1;       // full-state column ([A B] columns n.. are B)
        for (int i = 0; i < n; i++) col[i] = AB[i * ld + j];
    }
    double* out = P.ABe + (((size_t)b * (P.N - 1) + k) * nme + e) * ne;
    if (!P.lie) { for (int i = 0; i < n; i++) out[i] = col[i]; return; }
    double G1[12]; quat_G(X + (size_t)(k + 1) * n + qs, G1);
    for (int i = 0; i < qs; i++) out[i] = col[i];
    for (int c = 0; c < 3; c++) {
        double s = 0;
        for (int r = 0; r < 4; r++) s += G1[c * 4 + r] * col[qs + r];
        out[qs + c] = s;
    }
    for (int i = qs + 4; i < n; i++) out[i - 1] = col[i];
}

// column e of the error-state expansion of knot k from the full-state (grad, hess) in `gfull`, `hfull` ([B][N][nm], [B][N][nm][nm])
__global__ void __launch_bounds__(128) k_error_expansion(const DevProblem P, const double* __restrict__ gfull, const double* __restrict__ hfull,
                                                         double* __restrict__ EG, double* __restrict__ EH) {
    const int n = P.n, m = P.m, nm = n + m, ne = P.ne, nme = ne + m, qs = P.qs;
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)P.B * P.N * nme) return;
    const int e = (int)(t % nme);
    const long long bk = t / nme;
    const int k = (int)(bk % P.N), b = (int)(bk / P.N);
    const double* g = gfull + bk * nm;
    const double* H = hfull + bk * nm * nm;
    double* ge = EG + bk * nme;
    double* He = EH + bk * nme * nme + (size_t)e * nme;     // column e
    if (!P.lie) {
        for (int i = 0; i < nm; i++) He[i] = H[e * nm + i];
        ge[e] = g[e];
        return;
    }
    const double* q = traj_X(P, P.cur[b], b) + (size_t)k * n + qs;
    double G[12]; quat_G(q, G);
    double col[TO_MAXNM];                                    // column e of hess * blkdiag(E, I)  (nm entries)
    const bool qcol = (e >= qs && e < qs + 3);
    if (qcol) {
        const double* gq = &G[(e - qs) * 4];
        for (int i = 0; i < nm; i++) {
            double s = 0;
            for (int r = 0; r < 4; r++) s += H[(qs + r) * nm + i] * gq[r];
            col[i] = s;
        }
    } else {
        const int j = e < qs ? e : e + 1;
        for (int i = 0; i < nm; i++) col[i] = H[j * nm + i];
    }
    // rows: blkdiag(E, I)' col
    for (int i = 0; i < qs; i++) He[i] = col[i];
    for (int c = 0; c < 3; c++) {
        double s = 0;
        for (int r = 0; r < 4; r++) s += G[c * 4 + r] * col[qs + r];
        He[qs + c] = s;
    }
    for (int i = qs + 4; i < nm; i++) He[i - 1] = col[i];
    double qb = 0;                                           // grad^2-differential: -(q'g_q) on the attitude diagonal
    for (int r = 0; r < 4; r++) qb += q[r] * g[qs + r];
    if (qcol) {
        He[e] -= qb;
        double s = 0;
        for (int r = 0; r < 4; r++) s += G[(e - qs) * 4 + r] * g[qs + r];
        ge[e] = s;
    } else {
        ge[e] = g[e < qs ? e : e + 1];
    }
}

// Compact error-state expansion (P.compact): one thread per (instance, knot), costcon.cuh compact_expansion stored in logical order
// into EC, 40 doubles per knot (TO_EC_LEN) instead of the 272 of EG + EH.  riccati_frag.cu k_expansion_rec stores the same numbers
// in the record's order for the register-resident kernel.
template <bool INST>   // INST: the linear cost terms and constraint data of each instance
__global__ void __launch_bounds__(128) k_expansion_compact(const DevProblem P) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)P.B * P.N) return;
    const int k = (int)(t % P.N), b = (int)(t / P.N);
    if (retired(P, b)) return;                                     // to_solve: not ACTIVE
    double ge[16], hd[16], b01, b02, b12;
    compact_expansion<INST>(P, b, k, ge, hd, b01, b02, b12);
    double* out = P.EC + t * TO_EC_LEN;
#pragma unroll
    for (int e = 0; e < 16; e++) { out[e] = ge[e]; out[16 + e] = hd[e]; }
    out[32] = b01; out[33] = b02; out[34] = b12;
    for (int e = 35; e < TO_EC_LEN; e++) out[e] = 0.0;
}

// ---- Riccati backward pass on the materialised expansion: one warp per instance ---------------------------------------------
// Same recursion and restart / regularisation rules as riccati.cu (Altro backwardpass!, oracle/oracle.hpp backward_pass).
template <int NR, int M>
struct DenseSmem {
    static constexpr int NME = NR + M;
    double ab[NR * NME];        // [A_e B_e]_k, col-major NR x NME
    double Q[NME * NME];        // E_k.hess, then Qzz (col-major, full)
    double q[NME];              // E_k.grad, then Qz
    double S[NR * NR];          // cost-to-go Hessian (symmetric, full)
    double s[NR];
    double T[NR * NME];         // S [A B]
    double K[M * (NR + 1)];     // [K | d], row a = control
    double W[M * (NR + 1)];     // Qux - rho K | (unused)
};

template <int NR, int M, int WARPS>
__global__ void __launch_bounds__(32 * WARPS) k_riccati_dense(const DevProblem P) {
    using SM = DenseSmem<NR, M>;
    constexpr int NME = NR + M;
    __shared__ SM smem[WARPS];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int b = blockIdx.x * WARPS + warp;
    if (b >= P.B || retired(P, b)) return;       // (to_solve: not ACTIVE)
    SM& sm = smem[warp];
    const int N = P.N;
    const double* ABg = P.ABe + (size_t)b * (N - 1) * NR * NME;
    const double* EGg = P.EG + (size_t)b * N * NME;
    const double* EHg = P.EH + (size_t)b * N * NME * NME;
    double* Kg = P.K + (size_t)b * (N - 1) * NR * M;
    double* dg = P.d + (size_t)b * (N - 1) * M;
    double rho = P.rho[b], drho = P.drho[b];
    int restarts = 0;
    bool failed = false;

    for (;;) {
        // terminal knot: S = E_N.xx, s = E_N.x
        {
            const double* H = EHg + (size_t)(N - 1) * NME * NME;
            for (int e = lane; e < NR * NR; e += 32) sm.S[e] = H[(e / NR) * NME + (e % NR)];
            if (lane < NR) sm.s[lane] = EGg[(size_t)(N - 1) * NME + lane];
        }
        __syncwarp();
        double dV1 = 0.0, dV2 = 0.0;
        bool ok = true;
        for (int k = N - 2; k >= 0; k--) {
            {
                const double* src = ABg + (size_t)k * NR * NME;
                for (int e = lane; e < NR * NME; e += 32) sm.ab[e] = src[e];
                const double* H = EHg + (size_t)k * NME * NME;
                for (int e = lane; e < NME * NME; e += 32) sm.Q[e] = H[e];
                if (lane < NME) sm.q[lane] = EGg[(size_t)k * NME + lane];
            }
            __syncwarp();
            // T = S [A B]
            for (int e = lane; e < NR * NME; e += 32) {
                const int i = e % NR, j = e / NR;
                double t = 0.0;
#pragma unroll
                for (int r = 0; r < NR; r++) t = fma(sm.S[r * NR + i], sm.ab[j * NR + r], t);
                sm.T[e] = t;
            }
            __syncwarp();
            // Qzz = lzz + [A B]' T ; Qz = lz + [A B]' s
            for (int e = lane; e < NME * NME; e += 32) {
                const int i = e % NME, j = e / NME;
                double t = sm.Q[e];
#pragma unroll
                for (int r = 0; r < NR; r++) t = fma(sm.ab[i * NR + r], sm.T[j * NR + r], t);
                sm.Q[e] = t;
            }
            if (lane < NME) {
                double t = sm.q[lane];
#pragma unroll
                for (int r = 0; r < NR; r++) t = fma(sm.ab[lane * NR + r], sm.s[r], t);
                sm.q[lane] = t;
            }
            __syncwarp();
            // gains: LDL' of Quu + rho I (every lane factors the same M x M matrix), one lane per column of [Qux | Qu]
            double Quu[M * (M + 1) / 2], Lf[M * (M + 1) / 2], dj[M];
#pragma unroll
            for (int a = 0; a < M; a++)
#pragma unroll
                for (int c = 0; c <= a; c++) Quu[a * (a + 1) / 2 + c] = 0.5 * (sm.Q[(NR + c) * NME + NR + a] + sm.Q[(NR + a) * NME + NR + c]);
            if (!ldl_factor<M>(Quu, rho, Lf, dj, [](double t) { return 1.0 / t; })) ok = false;   // a division, where the other kernels take rcp_pos
            if (!ok) break;   // uniform across the warp
            if (lane <= NR) {
                const int c = lane;
                double rhs[M], kc[M];
#pragma unroll
                for (int a = 0; a < M; a++) rhs[a] = (c < NR) ? sm.Q[c * NME + NR + a] : sm.q[NR + a];   // Qux[a][c] | Qu[a]
                ldl_solve<M>(Lf, rhs, kc);
#pragma unroll
                for (int a = 0; a < M; a++) { sm.K[a * (NR + 1) + c] = kc[a]; sm.W[a * (NR + 1) + c] = fma(-rho, kc[a], rhs[a]); }
                if (c < NR) {
#pragma unroll
                    for (int a = 0; a < M; a++) Kg[(size_t)k * NR * M + c * M + a] = kc[a];
                } else {
#pragma unroll
                    for (int a = 0; a < M; a++) dg[(size_t)k * M + a] = kc[a];
                    double t1, t2;
                    expected_decrease<M>(Quu, kc, rhs, t1, t2);
                    dV1 += t1; dV2 += t2;
                }
            }
            __syncwarp();
            // S <- Qxx + W'K (symmetrised), s <- Qx + W'd
            for (int e = lane; e < NR * NR; e += 32) {
                const int i = e % NR, j = e / NR;
                if (i > j) continue;
                double v = 0.5 * (sm.Q[j * NME + i] + sm.Q[i * NME + j]);
                double wk = 0.0;
#pragma unroll
                for (int a = 0; a < M; a++) wk += sm.W[a * (NR + 1) + i] * sm.K[a * (NR + 1) + j] + sm.W[a * (NR + 1) + j] * sm.K[a * (NR + 1) + i];
                v = fma(0.5, wk, v);
                sm.S[j * NR + i] = v; sm.S[i * NR + j] = v;
            }
            if (lane < NR) {
                double t = sm.q[lane];
#pragma unroll
                for (int a = 0; a < M; a++) t = fma(sm.W[a * (NR + 1) + lane], sm.K[a * (NR + 1) + NR], t);
                sm.s[lane] = t;
            }
            __syncwarp();
        }
        if (ok) {
            if (lane == NR) { P.dV[2 * b] = dV1; P.dV[2 * b + 1] = dV2; }
            break;
        }
        if (reg_restart(P.opt, rho, drho, restarts)) { failed = true; break; }
        __syncwarp();
    }
    reg_finish(P, b, rho, drho, restarts, failed, lane);
}

// ---- the same pass for n_e = 12, m = 4 on the FP64 tensor cores -----------------------------------------------------------------
// n_e + m = 16 and n_e = 12 tile mma.sync.m8n8k4 (SASS DMMA) exactly: T = S [A B] is 2 x 2 tiles x 3 k-steps, Qzz += [A B]' T the same,
// S <- Qxx + W'K one k-step (k = m = 4) on 2 x 2 tiles: 28 DMMA per knot and no remainder handling (the fused n = 13 kernel of
// riccati.cu needs 39 DMMA + 24 rank-1 DFMA).  Operand layouts are chosen so that every fragment load is two shared-memory
// wavefronts (the minimum for 32 x 8 B): column-major with leading dimension 12 for S, [A B], T (12 = 4 mod 8), 20 for Q, 24 for K / W.
// The next knot's [A_e B_e], E.hess, E.grad are fetched with cp.async (LDGSTS) into the other half of a double buffer while this
// knot computes.
struct MmaSmem {   // one warp; NR = 12, M = 4, NME = 16
    static constexpr int LDQ = 20, LDK = 24;
    double ab[2][12 * 16];      // [A_e B_e]_k col-major ld 12, double buffered
    double Q[2][16 * LDQ];      // E_k.hess -> Qzz, col-major ld 20
    double q[2][16];            // E_k.grad -> Qz
    double S[16 * 12];          // symmetric 12 x 12 (ld 12) + 4 zero pad rows read by the second row tile
    double T[16 * 12];          // S [A B] (12 x 16, ld 12); later the unsymmetrised S update
    double K[4 * LDK];          // [K | d | 0]: row a = control
    double W[4 * LDK];          // Qux - rho K
    double s[12];
    double rec[2][TO_EC_LEN];   // compact expansion of the knot (P.compact), double buffered
};

template <int WARPS, bool COMPACT>
__global__ void __launch_bounds__(32 * WARPS) k_riccati_dense_mma(const DevProblem P) {
    constexpr int NR = 12, M = 4, NME = 16, LDQ = MmaSmem::LDQ, LDK = MmaSmem::LDK;
    extern __shared__ __align__(16) unsigned char dense_smem_raw[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int b = blockIdx.x * WARPS + warp;
    if (b >= P.B || retired(P, b)) return;       // (to_solve: not ACTIVE)
    MmaSmem& sm = reinterpret_cast<MmaSmem*>(dense_smem_raw)[warp];
    const int fr = lane >> 2, fc = lane & 3;      // fragment coordinates: A(8x4) row fr col fc ; B(4x8) row fc col fr ; D(8x8) row fr cols 2fc, 2fc+1
    const int N = P.N;
    const double* ABg = P.ABe + (size_t)b * (N - 1) * NR * NME;
    const double* EGg = COMPACT ? nullptr : P.EG + (size_t)b * N * NME;
    const double* EHg = COMPACT ? nullptr : P.EH + (size_t)b * N * NME * NME;
    const double* ECg = COMPACT ? P.EC + (size_t)b * N * TO_EC_LEN : nullptr;
    double* Kg = P.K + (size_t)b * (N - 1) * NR * M;
    double* dg = P.d + (size_t)b * (N - 1) * M;
    double rho = P.rho[b], drho = P.drho[b];
    int restarts = 0;
    bool failed = false;
    for (int e = lane; e < 16 * 12; e += 32) sm.S[e] = 0.0;
    for (int e = lane; e < 4 * LDK; e += 32) { sm.K[e] = 0.0; sm.W[e] = 0.0; }

    // async copies of knot k into buffer st: [A_e B_e] (96 sixteen-byte chunks) + the expansion (128 + 8 chunks, or the 20 of the compact record)
    auto fetch = [&](int st, int k) {
        const double* srcab = ABg + (size_t)k * NR * NME;
        for (int c = lane; c < 96; c += 32) cp_async16(&sm.ab[st][2 * c], srcab + 2 * c);
        if constexpr (COMPACT) {
            if (lane < TO_EC_LEN / 2) cp_async16(&sm.rec[st][2 * lane], ECg + (size_t)k * TO_EC_LEN + 2 * lane);
        } else {
            const double* srch = EHg + (size_t)k * NME * NME;
            for (int c = lane; c < 128; c += 32) { const int j = c >> 3, i = (c & 7) * 2; cp_async16(&sm.Q[st][j * LDQ + i], srch + j * NME + i); }
            if (lane < 8) cp_async16(&sm.q[st][2 * lane], EGg + (size_t)k * NME + 2 * lane);
        }
    };
    // entry (row, col) of the compact record's Hessian: diagonal + the symmetric 3 x 3 attitude block
    auto rec_h = [&](const double* rec, int row, int col) -> double {
        if (row == col) return rec[16 + row];
        if (row >= 3 && row < 6 && col >= 3 && col < 6) return rec[32 + (row - 3) + (col - 3) - 1];
        return 0.0;
    };

    for (;;) {
        if constexpr (COMPACT) {   // terminal knot: S = E_N.xx, s = E_N.x
            const double* rec = ECg + (size_t)(N - 1) * TO_EC_LEN;
            for (int e = lane; e < NR * NR; e += 32) sm.S[e] = rec_h(rec, e % NR, e / NR);
            if (lane < NR) sm.s[lane] = rec[lane];
        } else {
            const double* H = EHg + (size_t)(N - 1) * NME * NME;
            for (int e = lane; e < NR * NR; e += 32) sm.S[e] = H[(e / NR) * NME + (e % NR)];
            if (lane < NR) sm.s[lane] = EGg[(size_t)(N - 1) * NME + lane];
        }
        fetch(0, N - 2); cp_async_commit();
        __syncwarp();
        double dV1 = 0.0, dV2 = 0.0;
        bool ok = true;
        int st = 0;
        for (int k = N - 2; k >= 0; k--, st ^= 1) {
            if (k > 0) fetch(st ^ 1, k - 1);
            cp_async_commit();
            cp_async_wait<1>();            // this lane's copies of knot k have landed ...
            __syncwarp();                  // ... and everybody else's
            const double* ab = sm.ab[st];
            double* Qs = sm.Q[st];
            double* qs = sm.q[st];
            // fragments of [A B]: B operand of T = S [A B]; the same registers are the A operand ([A B]' rows) of Q += [A B]' T
            double bfr[3][2];
#pragma unroll
            for (int kk = 0; kk < 3; kk++)
#pragma unroll
                for (int t = 0; t < 2; t++) bfr[kk][t] = ab[(8 * t + fr) * 12 + 4 * kk + fc];
            {   // ---- T = S [A B] ----
                double d[2][2][2];
#pragma unroll
                for (int mi = 0; mi < 2; mi++)
#pragma unroll
                    for (int ni = 0; ni < 2; ni++) { d[mi][ni][0] = 0.0; d[mi][ni][1] = 0.0; }
#pragma unroll
                for (int kk = 0; kk < 3; kk++) {
                    double a[2];
#pragma unroll
                    for (int mi = 0; mi < 2; mi++) a[mi] = sm.S[(8 * mi + fr) * 12 + 4 * kk + fc];     // S is symmetric: row-major read
#pragma unroll
                    for (int mi = 0; mi < 2; mi++)
#pragma unroll
                        for (int ni = 0; ni < 2; ni++) dmma(d[mi][ni][0], d[mi][ni][1], a[mi], bfr[kk][ni]);
                }
#pragma unroll
                for (int mi = 0; mi < 2; mi++)
#pragma unroll
                    for (int ni = 0; ni < 2; ni++) {
                        const int row = 8 * mi + fr, col = 8 * ni + 2 * fc;
                        if (row < NR) { sm.T[col * 12 + row] = d[mi][ni][0]; sm.T[(col + 1) * 12 + row] = d[mi][ni][1]; }
                    }
            }
            __syncwarp();
            {   // ---- Qzz = lzz + [A B]' T (all four 8 x 8 tiles), Qz = lz + [A B]' s ----
                double c[2][2][2];
#pragma unroll
                for (int mi = 0; mi < 2; mi++)
#pragma unroll
                    for (int ni = 0; ni < 2; ni++) {
                        const int row = 8 * mi + fr, col = 8 * ni + 2 * fc;
                        if constexpr (COMPACT) { c[mi][ni][0] = rec_h(sm.rec[st], row, col); c[mi][ni][1] = rec_h(sm.rec[st], row, col + 1); }
                        else { c[mi][ni][0] = Qs[col * LDQ + row]; c[mi][ni][1] = Qs[(col + 1) * LDQ + row]; }
                    }
#pragma unroll
                for (int kk = 0; kk < 3; kk++) {
                    double bt[2];
#pragma unroll
                    for (int ni = 0; ni < 2; ni++) bt[ni] = sm.T[(8 * ni + fr) * 12 + 4 * kk + fc];
#pragma unroll
                    for (int mi = 0; mi < 2; mi++)
#pragma unroll
                        for (int ni = 0; ni < 2; ni++) dmma(c[mi][ni][0], c[mi][ni][1], bfr[kk][mi], bt[ni]);
                }
                double qz = 0.0;
                if (lane < NME) {
                    qz = COMPACT ? sm.rec[st][lane] : qs[lane];
#pragma unroll
                    for (int r = 0; r < NR; r++) qz = fma(ab[lane * 12 + r], sm.s[r], qz);
                }
                __syncwarp();              // every lane has read lzz / lz / s before they are overwritten
#pragma unroll
                for (int mi = 0; mi < 2; mi++)
#pragma unroll
                    for (int ni = 0; ni < 2; ni++) {
                        const int row = 8 * mi + fr, col = 8 * ni + 2 * fc;
                        Qs[col * LDQ + row] = c[mi][ni][0]; Qs[(col + 1) * LDQ + row] = c[mi][ni][1];
                    }
                if (lane < NME) qs[lane] = qz;
            }
            __syncwarp();
            // ---- gains: LDL' of Quu + rho I (every lane factors the same 4 x 4 matrix), one lane per column of [Qux | Qu] ----
            double Quu[M * (M + 1) / 2], Lf[M * (M + 1) / 2], dj[M];
#pragma unroll
            for (int a = 0; a < M; a++)
#pragma unroll
                for (int c = 0; c <= a; c++) Quu[a * (a + 1) / 2 + c] = 0.5 * (Qs[(NR + c) * LDQ + NR + a] + Qs[(NR + a) * LDQ + NR + c]);
            if (!ldl_factor<M>(Quu, rho, Lf, dj, rcp_pos)) ok = false;
            if (!ok) break;   // uniform across the warp
            if (lane <= NR) {
                const int c = lane;
                double rhs[M], kc[M];
#pragma unroll
                for (int a = 0; a < M; a++) rhs[a] = (c < NR) ? Qs[c * LDQ + NR + a] : qs[NR + a];   // Qux[a][c] | Qu[a]
                ldl_solve<M>(Lf, rhs, kc);
#pragma unroll
                for (int a = 0; a < M; a++) { sm.K[a * LDK + c] = kc[a]; sm.W[a * LDK + c] = fma(-rho, kc[a], rhs[a]); }
                if (c < NR) {
#pragma unroll
                    for (int a = 0; a < M; a++) Kg[(size_t)k * NR * M + c * M + a] = kc[a];
                } else {
#pragma unroll
                    for (int a = 0; a < M; a++) dg[(size_t)k * M + a] = kc[a];
                    double t1, t2;
                    expected_decrease<M>(Quu, kc, rhs, t1, t2);
                    dV1 += t1; dV2 += t2;
                }
            }
            __syncwarp();
            {   // ---- S <- Qxx + W'K: one DMMA k-step per tile (k = m = 4) on the upper tiles; the off-diagonal tile is mirrored, so S is
                //      symmetric up to the rounding inside the two diagonal tiles (as in riccati.cu) ----
                double af[2], bk[2];
#pragma unroll
                for (int t = 0; t < 2; t++) { af[t] = sm.W[fc * LDK + 8 * t + fr]; bk[t] = sm.K[fc * LDK + 8 * t + fr]; }
#pragma unroll
                for (int mi = 0; mi < 2; mi++)
#pragma unroll
                    for (int ni = mi; ni < 2; ni++) {
                        const int row = 8 * mi + fr, col = 8 * ni + 2 * fc;
                        double a0 = Qs[col * LDQ + row], a1 = Qs[(col + 1) * LDQ + row];
                        dmma(a0, a1, af[mi], bk[ni]);
                        if (row < NR && col < NR) {        // NR is even: col + 1 < NR too
                            sm.S[col * 12 + row] = a0; sm.S[(col + 1) * 12 + row] = a1;
                            if (ni != mi) { sm.S[row * 12 + col] = a0; sm.S[row * 12 + col + 1] = a1; }
                        }
                    }
                if (lane < NR) {
                    double t = qs[lane];
#pragma unroll
                    for (int a = 0; a < M; a++) t = fma(sm.W[a * LDK + lane], sm.K[a * LDK + NR], t);
                    sm.s[lane] = t;
                }
            }
            __syncwarp();
        }
        cp_async_wait<0>();
        __syncwarp();
        if (ok) {
            if (lane == NR) { P.dV[2 * b] = dV1; P.dV[2 * b + 1] = dV2; }
            break;
        }
        if (reg_restart(P.opt, rho, drho, restarts)) { failed = true; break; }
    }
    reg_finish(P, b, rho, drho, restarts, failed, lane);
}

#ifndef TO_DENSE_WARPS
#define TO_DENSE_WARPS 2     // warps (= instances) per CTA of k_riccati_dense_mma; A/B: profiles/build_lie_variants.sh
#endif
cudaError_t launch_dense_mma(const DevProblem& P, bool compact, cudaStream_t s) {
    constexpr int WARPS = TO_DENSE_WARPS;
    const int smem = (int)sizeof(MmaSmem) * WARPS;
    static bool configured[TO_MAXDEV] = {false};
    const int dev = current_device_slot();
    if (!configured[dev]) {
        cudaError_t e = cudaFuncSetAttribute(k_riccati_dense_mma<WARPS, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(k_riccati_dense_mma<WARPS, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e != cudaSuccess) return e;
        configured[dev] = true;
    }
    if (compact) k_riccati_dense_mma<WARPS, true><<<(P.B + WARPS - 1) / WARPS, 32 * WARPS, smem, s>>>(P);
    else k_riccati_dense_mma<WARPS, false><<<(P.B + WARPS - 1) / WARPS, 32 * WARPS, smem, s>>>(P);
    return cudaGetLastError();
}

template <int NR, int M, int WARPS = 4>
cudaError_t launch_dense_t(const DevProblem& P, cudaStream_t s) {
    static_assert(sizeof(DenseSmem<NR, M>) * WARPS <= 48 * 1024, "static shared memory");
    k_riccati_dense<NR, M, WARPS><<<(P.B + WARPS - 1) / WARPS, 32 * WARPS, 0, s>>>(P);
    return cudaGetLastError();
}

}  // namespace

cudaError_t launch_state_diff(const DevProblem& P, const double* Xbar, double* dx, cudaStream_t s) {
    k_state_diff<<<nblk((long long)P.B * P.N, 128), 128, 0, s>>>(P, Xbar, dx);
    return cudaGetLastError();
}
cudaError_t launch_error_dynamics(const DevProblem& P, cudaStream_t s) {
    k_error_dynamics<<<nblk((long long)P.B * (P.N - 1) * (P.ne + P.m), 128), 128, 0, s>>>(P);
    return cudaGetLastError();
}
cudaError_t launch_error_expansion(const DevProblem& P, const double* gfull, const double* hfull, double* EG, double* EH, cudaStream_t s) {
    k_error_expansion<<<nblk((long long)P.B * P.N * (P.ne + P.m), 128), 128, 0, s>>>(P, gfull, hfull, EG, EH);
    return cudaGetLastError();
}
cudaError_t launch_expansion_compact(const DevProblem& P, cudaStream_t s) {
    if (inst_backward(P)) k_expansion_compact<true><<<nblk((long long)P.B * P.N, 128), 128, 0, s>>>(P);
    else k_expansion_compact<false><<<nblk((long long)P.B * P.N, 128), 128, 0, s>>>(P);
    return cudaGetLastError();
}
cudaError_t launch_backward_dense(const DevProblem& P, const BackwardPlan& plan, cudaStream_t s) {
    if (plan.kernel == KC_BK_DENSE_MMA) return launch_dense_mma(P, plan.expansion == BackwardPlan::COMPACT, s);
    if (P.ne == 12 && P.m == 4) return launch_dense_t<12, 4>(P, s);
    if (P.ne == 13 && P.m == 4) return launch_dense_t<13, 4>(P, s);
    if (P.ne == 4 && P.m == 1) return launch_dense_t<4, 1>(P, s);
    if (P.ne == 4 && P.m == 2) return launch_dense_t<4, 2>(P, s);
    if (P.ne == 2 && P.m == 1) return launch_dense_t<2, 1>(P, s);
    // the recorded-program size classes (8, 4) and (16, 8) with a user cost.  (16, 8) takes 220 registers and 15 KB of shared memory per
    // warp: the register file holds 9 such warps per SM, which one-warp CTAs reach and two- or four-warp CTAs do not (8)
    if (P.ne == 8 && P.m == 4) return launch_dense_t<8, 4>(P, s);
    if (P.ne == 16 && P.m == 8) return launch_dense_t<16, 8, 1>(P, s);
    return cudaErrorNotSupported;
}
