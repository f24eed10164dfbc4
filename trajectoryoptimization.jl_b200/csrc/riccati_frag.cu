// riccati_frag.cu -- kernel 3 for the error-state Quadrotor (n_e = 12, m = 4): the Riccati backward pass with the whole
// recursion state resident in FP64 tensor-core fragment registers.
//
// What it computes: Altro.jl backwardpass! on the error state (restated in oracle/oracle.hpp backward_pass; SURVEY.md 8 a14, f2),
// per instance, serial in k = N-1 .. 1, with z = [x_e; u] (16 entries):
//     Qzz = lzz + [A_e B_e]' S [A_e B_e]     Qz = lz + [A_e B_e]' s
//     K = -(Quu + rho I)^-1 Qux   d = -(Quu + rho I)^-1 Qu          (non-PD Quu + rho I -> rho increase + restart)
//     S <- Qxx + W'K   s <- Qx + W'd   with W = Qux - rho K          dV += (d'Qu, 1/2 d'Quu d)
// lzz / lz is the reference's cost expansion (RD.gradient!/hessian!, src/cost_functions.jl:137-233) plus the AL terms of Goal / Bound
// constraints (src/constraints.jl:55-68, :738-765; projection! src/cones.jl:96-145), projected on the error state
// (error_expansion!, intent at src/abstract_constraint.jl:282-303) by k_expansion_rec below.
//
// Mapping (why this kernel exists: the shared-memory kernels spend their time on five smem hand-offs
// per knot and a 47-deep scalar LDL' chain at 4 warps per scheduler):
//   * one warp per instance; z is held in the PHYSICAL order of frag_layout.cuh, chosen so that the D fragments of every
//     mma.sync.m8n8k4.f64 (SASS DMMA) are exactly the A / B fragments of the next one:
//        T' = [A B]' S^      12 DMMA   B operand = the S accumulators of the previous knot (s rides in row 0 of S^)
//        Q^ = H^ + [A B]' T   9 DMMA   B operand = the T' accumulators; column 0 of T' is [A B]'s = Qz - lz for free; tiles (0,0),(1,0),(1,1)
//        [K|W]' = Q^[:,u] [-Minv | I + rho Minv]   2 DMMA   A operand = register 0 of the Q^ tiles (u_a sits on p = 2a);
//                                                  row 0 <- Qu gives d and w_d = Qu - rho d in the same product
//        S^ <- Q^ + W'K      3 DMMA    A / B operands = the two result registers of the previous product (row 0 / column 0 <- Qz give s);
//                                      S^(0,1) = S^(1,0)' by 4 shuffles; the diagonal tiles are symmetrised every 4th knot (the antisymmetric
//                                      part of S is an unstable mode of the recursion)
//     26 DMMA per knot, S / T / Q never leave the register file; per knot the warp touches shared memory for the record
//     (3 LDS.128 + 6 LDS.64), the 4 x 4 Quu (one STS, one LDS burst) and the 10 entries of its inverse.
//   * (Quu + rho I)^-1 by 2 x 2 block elimination (two Newton reciprocals, 20-deep chain instead of the 47 of a scalar LDL'),
//     evaluated by the lower half-warp only (an FP64 instruction of a half-empty warp takes one pipe pass);
//     positive-definiteness = positive leading minors a, det P, s00, det S (the pivots of LDL' are their ratios).
//   * the record of knot k (1920 B: fragments of [A_e B_e] + compact expansion) arrives by ONE 1-D bulk TMA copy (cp.async.bulk +
//     mbarrier, SASS UBLKCP) into a per-warp ring, issued one knot ahead.
//   * 4-warp CTAs; 128 registers x 4 CTAs per SM = 16 resident warps, two nearly full waves of B = 4096 instances on 132 SMs (1.94;
//     TO_FRAG_MINB below).
#include "costcon.cuh"
#include "frag_layout.cuh"
#include "kernels.h"

#ifndef TO_FRAG_STAGES
#define TO_FRAG_STAGES 2
#endif
#ifndef TO_FRAG_WARPS
#define TO_FRAG_WARPS 4
#endif
// Speculation rounds of the regularisation ladder: candidate c belongs to the round [first, next) with first = the largest boundary <= c.
// 0: {1} {2,3} {4..7} {8..15}    1: {1} {2..15}    2: {1..3} {4..15}    3: {1} {2..7} {8..15}    4: {1..7} {8..15}    5: {1..15}
// 2 is the default.
#ifndef TO_FRAG_ROUNDS
#define TO_FRAG_ROUNDS 2
#endif
// CTAs per SM the register allocation aims at.  A full SM does not make the sweeps faster in total: R grows almost in proportion to the
// resident warps beyond 4 per scheduler, so 6 CTAs (80 registers, 24 warps, 180 / 368 B of spills) ran B = 4096 as a full wave of 3168
// sweeps and then 928 more at lone-warp latency.  4 CTAs (128 registers, 16 warps, 12 B of spills) run two nearly full waves of 2112 and
// 1984 sweeps, each faster per sweep.  On one H100 (700 W), k_riccati_frag: BASELINE 0.484 ms (6 CTAs 0.529, 5 CTAs 0.493, 7 CTAs 0.553),
// quadrotor_calm 0.361 ms (6 CTAs 0.450, 5 CTAs 0.399, 7 CTAs 0.473).  A build-time knob (-DTO_FRAG_MINB=6) for variant builds.
#ifndef TO_FRAG_MINB
#define TO_FRAG_MINB 4
#endif
// L2 prefetch distance of the record stream, in knots beyond the shared-memory ring (0 = off).  The ring hides the copy latency while the SM is
// full (28 warps); a LONE warp -- the retry sweeps at the tail of the regularisation ladder, small batches -- waits for every record.
#ifndef TO_FRAG_PF
#define TO_FRAG_PF 0
#endif

namespace {

inline unsigned nblk(long long total, int threads) { return (unsigned)((total + threads - 1) / threads); }

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "DONE:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void bulk_prefetch_l2(const void* src, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ double2 lds128(const double* p) { return *reinterpret_cast<const double2*>(p); }
__device__ __forceinline__ void dmma(double& d0, double& d1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
}
__device__ __forceinline__ int ld_volatile_s32(const int* p) {
    int v;
    asm volatile("ld.volatile.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
// 8 x 8 tile held as D fragments (x0, x1) = X[fr][2fc], X[fr][2fc+1]  ->  its transpose in the same layout: Y[fr][2fc + r] = X[2fc + r][fr]
// sits in lane (2fc + r, fr >> 1), register fr & 1.   src = 8 fc + (fr >> 1) = lane (2fc, fr >> 1).
__device__ __forceinline__ void tile_transpose(double x0, double x1, int src, int odd_row, double& y0, double& y1) {
    const double a0 = __shfl_sync(0xffffffffu, x0, src), a1 = __shfl_sync(0xffffffffu, x1, src);
    const double b0 = __shfl_sync(0xffffffffu, x0, src + 4), b1 = __shfl_sync(0xffffffffu, x1, src + 4);
    y0 = odd_row ? a1 : a0;
    y1 = odd_row ? b1 : b0;
}
// 1/x for a positive finite x: hardware seed + two Newton steps (<= 1 ulp), no IEEE-division slow path on the pivot chain
__device__ __forceinline__ double rcp_pos(double x) {
    double y;
    asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(x));
    double e = fma(-x, y, 1.0);
    y = fma(y, e, y);
    e = fma(-x, y, 1.0);
    return fma(y, e, y);
}

// ---- compact error-state expansion into the record --------------------------------------------------------------------------------
// One thread per (instance, knot).  Full-state expansion of a DiagonalCost + Goal / Bound AL rows is a gradient g and a DIAGONAL h;
// on the error state it is G'g, the same diagonal outside the attitude, and the 3 x 3 block G_q' diag(h_q) G_q - (q'g_q) I3
// (Altro error_expansion!; lie.cu k_expansion_compact computes the same numbers in logical order for the shared-memory kernel).
template <bool INST>   // INST: the linear cost terms and Goal values of each instance
__global__ void __launch_bounds__(128) k_expansion_rec(const DevProblem P) {
    const int n = P.n, m = P.m, nm = n + m, qs = P.qs;
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)P.B * P.N) return;
    const int k = (int)(t % P.N), b = (int)(t / P.N);
    if (retired(P, b)) return;                                     // to_solve: not ACTIVE
    const bool last = (k == P.N - 1);
    const double* xg = traj_X(P, P.cur[b], b) + (size_t)k * n;
    const double* ug = traj_U(P, P.cur[b], b) + (size_t)k * m;
    const double* lam_b = P.lambda + (size_t)b * P.lambda_len;
    double z[TO_MAXNM], g[TO_MAXNM], h[TO_MAXNM];
    for (int i = 0; i < n; i++) z[i] = xg[i];
    for (int a = 0; a < m; a++) z[n + a] = last ? 0.0 : ug[a];
    const int cid = P.cost_index[k];
    const DevCost& c = P.costs[cid];
    const double* cq = inst_q<INST>(P, b, cid); const double* cr = inst_r<INST>(P, b, cid);
    for (int i = 0; i < n; i++) { g[i] = fma(c.Qd[i], z[i], cq[i]); h[i] = c.Qd[i]; }
    for (int a = 0; a < m; a++) { g[n + a] = last ? 0.0 : fma(c.Rd[a], z[n + a], cr[a]); h[n + a] = last ? 0.0 : c.Rd[a]; }
    const int lim = last ? n : nm;
    for (int ci = 0; ci < P.ncon; ci++) {
        const DevCon& con = P.cons[ci];
        if (k + 1 < con.first || k + 1 > con.last) continue;
        const double mu = P.mu[ci];
        const double* lam = lam_b + con.offset + (size_t)(k + 1 - con.first) * con.p;
        const bool eq = (con.kind == CON_GOAL);
        const ConData cd = con_data<INST>(P, b, ci);
        const int nrow = eq ? con.p : con.n_max + con.n_min;
        for (int r = 0; r < nrow; r++) {
            const int j = eq ? con.inds[r] : (r < con.n_max ? con.a_max[r] : con.a_min[r - con.n_max]);
            const bool lower = !eq && r >= con.n_max;
            const double cv = eq ? z[j] - cd.a[r] : (lower ? cd.b[j] - z[j] : z[j] - cd.a[j]);
            const double lb = lam[r] - mu * cv;
            if ((eq || lb <= 0.0) && j < lim) { g[j] -= lower ? -lb : lb; h[j] += mu; }
        }
    }
    double* out = P.REC + t * TO_REC_LEN;
    double G[12]; quat_G(z + qs, G);
    double ge[16], hd[16];
    for (int e = 0; e < qs; e++) { ge[e] = g[e]; hd[e] = h[e]; }
    for (int e = qs + 3; e < n - 1 + m; e++) { ge[e] = g[e + 1]; hd[e] = h[e + 1]; }
    double qb = 0;
    for (int r = 0; r < 4; r++) qb += z[qs + r] * g[qs + r];
    for (int cc = 0; cc < 3; cc++) {
        double s = 0, d = 0;
        for (int r = 0; r < 4; r++) { s += G[cc * 4 + r] * g[qs + r]; d += G[cc * 4 + r] * h[qs + r] * G[cc * 4 + r]; }
        ge[qs + cc] = s; hd[qs + cc] = d - qb;
    }
    double b01 = 0, b02 = 0, b12 = 0;
    for (int r = 0; r < 4; r++) { b01 += G[r] * h[qs + r] * G[4 + r]; b02 += G[r] * h[qs + r] * G[8 + r]; b12 += G[4 + r] * h[qs + r] * G[8 + r]; }
#pragma unroll
    for (int j = 0; j < 16; j++) { out[TO_REC_G + fraglayout::phys_z(j)] = ge[j]; out[TO_REC_HD + fraglayout::phys_z(j)] = hd[j]; }
    // Hb[a][b] = H~[8+2a][8+2b]: a, b = 0..2 the attitude error (e = 3..5), a = 3 is p = 14 (e = 7)
    out[TO_REC_HB + 0] = hd[3]; out[TO_REC_HB + 1] = b01;   out[TO_REC_HB + 2] = b02;    out[TO_REC_HB + 3] = 0.0;
    out[TO_REC_HB + 4] = b01;   out[TO_REC_HB + 5] = hd[4]; out[TO_REC_HB + 6] = b12;    out[TO_REC_HB + 7] = 0.0;
    out[TO_REC_HB + 8] = b02;   out[TO_REC_HB + 9] = b12;   out[TO_REC_HB + 10] = hd[5]; out[TO_REC_HB + 11] = 0.0;
    out[TO_REC_HB + 12] = 0.0;  out[TO_REC_HB + 13] = 0.0;  out[TO_REC_HB + 14] = 0.0;   out[TO_REC_HB + 15] = hd[7];
}

// [A_e B_e] of the record back in the col-major 12 x 16 layout of P.ABe (to_get_error_dynamics, the shared-memory kernels of lie.cu)
__global__ void __launch_bounds__(128) k_export_abe(const DevProblem P) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)P.B * (P.N - 1) * 16) return;
    const int j = (int)(t & 15);
    const long long bk = t >> 4;
    const int k = (int)(bk % (P.N - 1)), b = (int)(bk / (P.N - 1));
    const double* rec = P.REC + ((size_t)b * P.N + k) * TO_REC_LEN;
    double* out = P.ABe + ((size_t)bk * 16 + j) * 12;
    for (int e = 0; e < 12; e++) {
        const int q = fraglayout::phys_x(e);
        const int ks = (q < 8) ? 0 : ((q & 1) ? 2 : 1);
        const int fc = (q < 8) ? (q - 1) / 2 : ((q & 1) ? (q - 9) / 2 : (q - 8) / 2);
        const int c = fraglayout::phys_z(j);
        out[e] = rec[(ks * 32 + 4 * (c & 7) + fc) * 2 + (c >> 3)];
    }
}

// ---- the backward pass ----------------------------------------------------------------------------------------------------------------
template <int STAGES, int WARPS>
struct FragSmem {
    double rec[WARPS][STAGES][TO_REC_LEN];    // per-warp ring of knot records (1920 B = 15 x 128 B each)
    double quu[WARPS][32];                    // [0,16) Quu (row-major 4 x 4) ; [16,27) the 10 entries of its inverse + the PD flag
    uint64_t bar[WARPS][STAGES];
};

// entries of the symmetric inverse in the order they are stored in shared memory
enum { MI_P00 = 0, MI_P01, MI_P11, MI_N00, MI_N01, MI_N10, MI_N11, MI_V00, MI_V01, MI_V11, MI_OK };
__device__ __forceinline__ int minv_slot(int i, int j) {   // slot of Minv[i][j]
    if (i > j) { const int t = i; i = j; j = t; }
    if (j < 2) return i == 0 ? (j == 0 ? MI_P00 : MI_P01) : MI_P11;
    if (i >= 2) return i == 2 ? (j == 2 ? MI_V00 : MI_V01) : MI_V11;
    // i < 2 <= j: Minv[j][i] = n_{j-2, i}
    return (j == 2) ? (i == 0 ? MI_N00 : MI_N01) : (i == 0 ? MI_N10 : MI_N11);
}

template <int STAGES, int WARPS, int MINB>
__global__ void __launch_bounds__(32 * WARPS, MINB) k_riccati_frag(const DevProblem P, int* __restrict__ Qd, double* __restrict__ pool, int nslots, int* __restrict__ sticky_err) {
    using SM = FragSmem<STAGES, WARPS>;
    extern __shared__ __align__(128) unsigned char frag_smem_raw[];
    SM& sm = *reinterpret_cast<SM*>(frag_smem_raw);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int fr = lane >> 2, fc = lane & 3;
    const int N = P.N;
    double* const ring = &sm.rec[warp][0][0];
    double* const quu = sm.quu[warp];
    double* const minv = quu + 16;
    uint64_t* const bar = sm.bar[warp];

    // loop-invariant lane roles
    const bool d00 = (fr == 2 * fc), d01 = (fr == 2 * fc + 1);   // this lane holds a diagonal entry of a diagonal tile in reg 0 / reg 1
    const bool fr_even = (fr & 1) == 0;
    const bool row0 = (fr == 0);
    const int eoff0 = (fr & 1) ? fraglayout::e_of_p(fr) * 4 + fc : -1;          // K[a = fc][e(p = fr)]      (tile row 0: x_e only on odd p)
    const int eoff1 = fraglayout::e_of_p(8 + fr) * 4 + fc;                      // K[a = fc][e(p = 8 + fr)]
    const int mslot = minv_slot(fc, fr >> 1);                                     // this lane's entry Minv[fc][fr >> 1] of the B fragment
    const double bdelta = ((fr & 1) && fc == (fr >> 1)) ? 1.0 : 0.0;
    const int tsrc = 8 * fc + (fr >> 1);          // lane (2 fc, fr >> 1): holder of the transposed entries of this lane's register 0 (register 1: + 4)

    if (lane == 0) {
#pragma unroll
        for (int s = 0; s < STAGES; s++) mbar_init(&bar[s], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncwarp();
    uint32_t phase_bits = 0;

    // ---- work queue (zero / 0xFF / 0x7F-initialised by the launcher) -------------------------------------------------------------------
    //   Qd[0] head   next work index: indices < B are the first sweeps (instance = index), index B + q is slot q of the item list
    //   Qd[1] tail   item slots handed out          Qd[2] nfinal  instances finalised          Qd[3] error flag (spin limit)
    //   cnt[B]   candidates of the instance's current round still running     items[QCAP]  instance * 16 + candidate, -1 = not yet written
    //   best[B]  lowest successful candidate of the round: candidate << 16 | gain-pool slot (0x7f7f7f7f = none)
    //   Qd[4] pool slots handed out.  A candidate that is not the lowest of its round writes its gains to a slot of `pool` (if one is left);
    //   when it wins the round they are copied into place instead of being recomputed by one more sweep.
    // Regularisation ladder (Altro regularization_update!(:increase) after a failed sweep, restart from the terminal knot): the sequence
    // rho_1, rho_2, ... an instance will try is a function of (rho_0, drho_0) alone, so after a failed first sweep the candidates are
    // evaluated SPECULATIVELY IN PARALLEL by whichever warps are idle, in rounds (TO_FRAG_ROUNDS above); the result is the lowest
    // successful candidate = exactly what the sequential loop returns (it stops at its first success), in <= 3 sweep times instead of <= 14.
    const int QCAP = 16 * P.B + 8192;
    int* const q_head = Qd; int* const q_tail = Qd + 1; int* const q_nfinal = Qd + 2; int* const q_err = Qd + 3;
    int* const q_nslot = Qd + 4;
    int* const q_cnt = Qd + 8; int* const q_items = q_cnt + P.B; int* const q_best = q_items + QCAP;
    const size_t slot_stride = (size_t)(P.N - 1) * 52 + 2;       // K (48 per knot), d (4 per knot), dV (2)

    for (;;) {
        int idx = 0;
        if (lane == 0) idx = atomicAdd(q_head, 1);
        idx = __shfl_sync(0xffffffffu, idx, 0);
        int b, cand;
        if (idx < P.B) {
            b = idx; cand = 0;
            if (retired(P, b)) {                    // to_solve: not ACTIVE -- counts as finalised, so the queue still drains at nfinal == B
                if (lane == 0) atomicAdd(q_nfinal, 1);
                continue;
            }
        } else {
            const int qi = idx - P.B;
            int item = -2;
            if (lane == 0) {
                unsigned spins = 0, ns = 128;
                for (;;) {
                    item = (qi < QCAP) ? ld_volatile_s32(q_items + qi) : -1;
                    if (item >= 0) break;
                    if (ld_volatile_s32(q_nfinal) >= P.B) { item = -2; break; }      // every instance is finalised: nothing more will be queued
                    __nanosleep(ns);                                                  // back off: an idle warp must not take issue slots from the running ones
                    if (ns < 4096) ns *= 2;
                    if (++spins > (1u << 18)) { atomicExch(q_err, 1); atomicOr(sticky_err, 1); item = -2; break; }   // ~1 s: never hang the device
                }
            }
            item = __shfl_sync(0xffffffffu, item, 0);
            if (item < 0) break;
            b = item >> 4; cand = item & 15;
        }
        const double* recg = P.REC + (size_t)b * N * TO_REC_LEN;
        double* const Kg = P.K + (size_t)b * (N - 1) * 48;
        double* const dg = P.d + (size_t)b * (N - 1) * 4;
        double* Kdst = Kg; double* ddst = dg;             // where a storing sweep puts its gains (the instance's, or a pool slot)
        const double rho0 = P.rho[b], drho0 = P.drho[b];

        auto issue = [&](int st, int k) {
            if (lane == 0) {
                mbar_expect_tx(&bar[st], TO_REC_LEN * 8);
                bulk_g2s(ring + st * TO_REC_LEN, recg + (size_t)k * TO_REC_LEN, TO_REC_LEN * 8, &bar[st]);
                if (TO_FRAG_PF > 0 && k - TO_FRAG_PF >= 0) bulk_prefetch_l2(recg + (size_t)(k - TO_FRAG_PF) * TO_REC_LEN, TO_REC_LEN * 8);
            }
        };
        // (rho_j, drho_j): j applications of regularization_update!(:increase); returns the first i <= j whose rho exceeds bp_reg_max (the
        // sequential loop gives up there) or 0
        auto ladder = [&](int j, double& rho, double& drho) -> int {
            rho = rho0; drho = drho0;
            for (int i = 1; i <= j; i++) { reg_increase(P.opt, rho, drho); if (rho > P.opt.bp_reg_max) return i; }
            return 0;
        };
        double acc1 = 0.0, acc2 = 0.0;   // lanes (0, fc): sum_k d_a Qu_a, sum_k d_a^2 of the last sweep
        // one sweep N-1 .. 1 with the given rho; store: write the gains; poll: give up when a lower candidate of the round has succeeded
        auto sweep = [&](double rho, bool store, bool poll) -> bool {
#pragma unroll
            for (int s = 0; s < STAGES; s++) { const int k = N - 2 - s; if (k >= 0) issue(s, k); }
            if (TO_FRAG_PF > 1 && lane == 0)       // the knots between the ring and the first per-knot prefetch
                for (int k = N - 2 - STAGES; k > N - 2 - STAGES - (TO_FRAG_PF - 1) && k >= 0; k--) bulk_prefetch_l2(recg + (size_t)k * TO_REC_LEN, TO_REC_LEN * 8);
            // ---- terminal knot: S^ = H^_N with s = g_N in row 0 ---------------------------------------------------------------------
            double S[2][2][2];
            {
                const double* rN = recg + (size_t)(N - 1) * TO_REC_LEN;
                const double hd0 = rN[TO_REC_HD + fr], hd1 = rN[TO_REC_HD + 8 + fr], hb = rN[TO_REC_HB + (fr >> 1) * 4 + fc];
                S[0][0][0] = d00 ? hd0 : 0.0; S[0][0][1] = d01 ? hd0 : 0.0;
                S[0][1][0] = 0.0; S[0][1][1] = 0.0; S[1][0][0] = 0.0; S[1][0][1] = 0.0;
                S[1][1][0] = fr_even ? hb : 0.0; S[1][1][1] = d01 ? hd1 : 0.0;
                if (row0) {
                    S[0][0][0] = rN[TO_REC_G + 2 * fc]; S[0][0][1] = rN[TO_REC_G + 2 * fc + 1];
                    S[0][1][0] = rN[TO_REC_G + 8 + 2 * fc]; S[0][1][1] = rN[TO_REC_G + 9 + 2 * fc];
                }
            }
            acc1 = 0.0; acc2 = 0.0;
            bool ok = true, aborted = false;
            int stage = 0;
            int k;
            for (k = N - 2; k >= 0; k--) {
                const int best_seen = poll ? ld_volatile_s32(q_best + b) : 0x7fffffff;     // consumed at the bottom of the knot
                mbar_wait(&bar[stage], (phase_bits >> stage) & 1u);
                phase_bits ^= (1u << stage);
                const double* r = ring + stage * TO_REC_LEN;
                // fragments of [A_e B_e]_k: abf[ks][mi] = AB[q(ks,fc)][p = 8 mi + fr]
                double abf[3][2];
#pragma unroll
                for (int ks = 0; ks < 3; ks++) { const double2 v = lds128(r + (ks * 32 + lane) * 2); abf[ks][0] = v.x; abf[ks][1] = v.y; }
                // ---- T'[c][j] = sum_q AB[q][c] S^[j][q] ------------------------------------------------------------------------------
                double T[2][2][2];
#pragma unroll
                for (int mi = 0; mi < 2; mi++)
#pragma unroll
                    for (int nj = 0; nj < 2; nj++) { T[mi][nj][0] = 0.0; T[mi][nj][1] = 0.0; }
#pragma unroll
                for (int ks = 0; ks < 3; ks++) {
                    const int ni = (ks == 0) ? 0 : 1, rg = (ks == 1) ? 0 : 1;   // k-step class -> (column tile, register)
#pragma unroll
                    for (int mi = 0; mi < 2; mi++)
#pragma unroll
                        for (int nj = 0; nj < 2; nj++) dmma(T[mi][nj][0], T[mi][nj][1], abf[ks][mi], S[nj][ni][rg]);
                }
                // ---- Q^ = H^ + [A B]' T ; Qz (column form, lanes fc == 0) = g~ + column 0 of T' ----------------------------------------
                double Q[2][2][2];
                {
                    const double hd0 = r[TO_REC_HD + fr], hd1 = r[TO_REC_HD + 8 + fr], hb = r[TO_REC_HB + (fr >> 1) * 4 + fc];
                    Q[0][0][0] = d00 ? hd0 : 0.0; Q[0][0][1] = d01 ? hd0 : 0.0;
                    Q[0][1][0] = 0.0; Q[0][1][1] = 0.0; Q[1][0][0] = 0.0; Q[1][0][1] = 0.0;
                    Q[1][1][0] = fr_even ? hb : 0.0; Q[1][1][1] = d01 ? hd1 : 0.0;
                }
                const double qzc0 = r[TO_REC_G + fr] + T[0][0][0], qzc1 = r[TO_REC_G + 8 + fr] + T[1][0][0];
#pragma unroll
                for (int ks = 0; ks < 3; ks++) {
                    const int ni = (ks == 0) ? 0 : 1, rg = (ks == 1) ? 0 : 1;
                    // the tiles on and below the diagonal: (0,1) is never used, the update leaves S^(0,1) = S^(1,0)'
                    dmma(Q[0][0][0], Q[0][0][1], abf[ks][0], T[0][ni][rg]);
                    dmma(Q[1][0][0], Q[1][0][1], abf[ks][1], T[0][ni][rg]);
                    dmma(Q[1][1][0], Q[1][1][1], abf[ks][1], T[1][ni][rg]);
                }
                // Qz in row form for lanes (0, fc): entries 2fc, 2fc+1 live in lanes (2fc, 0) / (2fc+1, 0)
                const double qx00 = __shfl_sync(0xffffffffu, qzc0, 8 * fc), qx01 = __shfl_sync(0xffffffffu, qzc0, 8 * fc + 4);
                // ---- gains -------------------------------------------------------------------------------------------------------------
                if (fr_even) quu[(fr >> 1) * 4 + fc] = Q[0][0][0];      // Quu[a][b] = Q^[2a][2b] sits in lane (2a, b)
                __syncwarp();
                if (lane < 16) {
                    const double2 r0a = lds128(quu + 0), r0b = lds128(quu + 2), r1b = lds128(quu + 6), r2b = lds128(quu + 10);
                    const double m11 = quu[5], m33 = quu[15];
                    const double a = r0a.x + rho, bq = r0a.y, c = m11 + rho;
                    const double M20 = r0b.x, M30 = r0b.y, M21 = r1b.x, M31 = r1b.y;      // block (2:3, 0:1), upper-triangle copies
                    const double R00 = r2b.x + rho, R01 = r2b.y, R11 = m33 + rho;
                    const double detP = fma(a, c, -bq * bq);
                    const double iP = rcp_pos(detP);
                    const double yt00 = fma(M20, c, -M21 * bq), yt01 = fma(M21, a, -M20 * bq);     // Y~ = Q21 adj(P)
                    const double yt10 = fma(M30, c, -M31 * bq), yt11 = fma(M31, a, -M30 * bq);
                    const double z00 = fma(yt00, M20, yt01 * M21), z01 = fma(yt00, M30, yt01 * M31), z11 = fma(yt10, M30, yt11 * M31);
                    const double s00 = fma(-iP, z00, R00), s01 = fma(-iP, z01, R01), s11 = fma(-iP, z11, R11);   // Schur complement
                    const double detS = fma(s00, s11, -s01 * s01);
                    const double iS = rcp_pos(detS);
                    const double v00 = s11 * iS, v01 = -s01 * iS, v11 = s00 * iS;
                    const double y00 = yt00 * iP, y01 = yt01 * iP, y10 = yt10 * iP, y11 = yt11 * iP;
                    const double n00 = -fma(v00, y00, v01 * y10), n01 = -fma(v00, y01, v01 * y11);
                    const double n10 = -fma(v01, y00, v11 * y10), n11 = -fma(v01, y01, v11 * y11);
                    const double p00 = fma(c, iP, -fma(y00, n00, y10 * n10));
                    const double p01 = fma(-bq, iP, -fma(y00, n01, y10 * n11));
                    const double p11 = fma(a, iP, -fma(y01, n01, y11 * n11));
                    const bool pd = (a > 0.0) && (detP > 0.0) && (s00 > 0.0) && (detS > 0.0) && (detP < 1e300) && (detS < 1e300);
                    if (lane == 0) {
                        *reinterpret_cast<double2*>(minv + MI_P00) = make_double2(p00, p01);
                        *reinterpret_cast<double2*>(minv + MI_P11) = make_double2(p11, n00);
                        *reinterpret_cast<double2*>(minv + MI_N01) = make_double2(n01, n10);
                        *reinterpret_cast<double2*>(minv + MI_N11) = make_double2(n11, v00);
                        *reinterpret_cast<double2*>(minv + MI_V01) = make_double2(v01, v11);
                        minv[MI_OK] = pd ? 1.0 : 0.0;
                    }
                }
                __syncwarp();
                const double Eij = minv[mslot];
                ok = minv[MI_OK] != 0.0;
                if (!ok) break;                       // uniform
                const double bfrag = (fr & 1) ? fma(rho, Eij, bdelta) : -Eij;     // [-Minv | I + rho Minv], columns interleaved
                const double af0 = row0 ? qx00 : Q[0][0][0];                      // row 0 <- Qu (Qu[fc] = Qz[2 fc])
                double k0 = 0.0, w0 = 0.0, k1 = 0.0, w1 = 0.0;
                dmma(k0, w0, af0, bfrag);             // lane (fr, fc): K[fc][p = fr], W[fc][p = fr]; row 0: d[fc], w_d[fc]
                dmma(k1, w1, Q[1][0][0], bfrag);      //                K[fc][p = 8 + fr], W[fc][p = 8 + fr]
                acc1 = fma(k0, af0, acc1); acc2 = fma(k0, k0, acc2);
                if (store) {
                    if (eoff0 >= 0) Kdst[(size_t)k * 48 + eoff0] = k0;
                    Kdst[(size_t)k * 48 + eoff1] = k1;
                    if (row0) ddst[(size_t)k * 4 + fc] = k0;
                }
                // row 0 <- Qz (the product below leaves s = Qx + K'w_d there), column 0 <- Qz (... leaves s = Qx + W'd there: K^[a][0] = d[a])
                if (fc == 0) { Q[0][0][0] = qzc0; Q[1][0][0] = qzc1; }
                if (row0) { Q[0][0][0] = qx00; Q[0][0][1] = qx01; }
                // ---- S^ <- Q^ + W'K on the three tiles; S^(0,1) <- S^(1,0)' ---------------------------------------------------------------
                dmma(Q[0][0][0], Q[0][0][1], w0, k0);
                dmma(Q[1][0][0], Q[1][0][1], w1, k0);
                dmma(Q[1][1][0], Q[1][1][1], w1, k1);
                S[0][0][0] = Q[0][0][0]; S[0][0][1] = Q[0][0][1]; S[1][0][0] = Q[1][0][0]; S[1][0][1] = Q[1][0][1];
                S[1][1][0] = Q[1][1][0]; S[1][1][1] = Q[1][1][1];
                tile_transpose(S[1][0][0], S[1][0][1], tsrc, fr & 1, S[0][1][0], S[0][1][1]);
                // The antisymmetric part of S is an unstable mode of the recursion (it grows by ~1.25 per knot: 1e-16 -> 1e-6 over 100 knots,
                // measured).  The off-diagonal tiles are exact mirrors by construction; the diagonal tiles are averaged
                // with their transposes every 4th knot (growth 2.4 between two averagings).
                if ((k & 3) == 0) {
                    double y0, y1;
                    tile_transpose(S[0][0][0], S[0][0][1], tsrc, fr & 1, y0, y1);
                    S[0][0][0] = 0.5 * (S[0][0][0] + y0); S[0][0][1] = 0.5 * (S[0][0][1] + y1);
                    tile_transpose(S[1][1][0], S[1][1][1], tsrc, fr & 1, y0, y1);
                    S[1][1][0] = 0.5 * (S[1][1][0] + y0); S[1][1][1] = 0.5 * (S[1][1][1] + y1);
                }
                // the record and the Minv slots have been consumed by every lane: refill the ring slot
                __syncwarp();
                if ((best_seen >> 16) < cand) { ok = false; aborted = true; }      // a lower candidate of this round already succeeded: this sweep is moot
                if (aborted) { k--; break; }                                 // (this knot's slot was consumed: same drain as a failure one knot later)
                if (k - STAGES >= 0) issue(stage, k - STAGES);
                stage = (stage + 1 == STAGES) ? 0 : stage + 1;
            }   // knots
            if (!ok) {
                // drain the copies in flight: slot `stage` (knot k of the failure) was consumed, the slots after it hold knots k-1 .. k-STAGES+1
                const int kf = aborted ? k + 1 : k;
                const int outstanding = (kf < STAGES - 1) ? kf : STAGES - 1;
                for (int i = 1; i <= outstanding; i++) {
                    const int st = (stage + i) % STAGES;
                    mbar_wait(&bar[st], (phase_bits >> st) & 1u);
                    phase_bits ^= (1u << st);
                }
                __syncwarp();
            }
            return ok;
        };
        // expected decrease of the sweep this warp just completed (the accumulators live in its registers)
        auto write_dV = [&](double rho, double* dst) {
            acc1 += __shfl_xor_sync(0xffffffffu, acc1, 1); acc1 += __shfl_xor_sync(0xffffffffu, acc1, 2);
            acc2 += __shfl_xor_sync(0xffffffffu, acc2, 1); acc2 += __shfl_xor_sync(0xffffffffu, acc2, 2);
            // 1/2 d'Quu d = -1/2 (d'Qu + rho d'd)   since (Quu + rho I) d = -Qu
            if (lane == 0) { dst[0] = acc1; dst[1] = -0.5 * fma(rho, acc2, acc1); }
        };
        auto finalise = [&](double rho, double drho, int status) {
            if (status >= 0) reg_decrease(P.opt, rho, drho);
            if (lane == 0) {
                P.rho[b] = rho; P.drho[b] = drho; P.bp_status[b] = status;
                __threadfence();
                atomicAdd(q_nfinal, 1);
            }
        };
        // queue the candidates first .. first + n - 1 of instance b
        auto start_round = [&](int first, int n) {
            if (lane == 0) {
                atomicExch(q_cnt + b, n);
                atomicExch(q_best + b, 0x7f7f7f7f);
                __threadfence();
                const int slot = atomicAdd(q_tail, n);
                for (int i = 0; i < n; i++)
                    if (slot + i < QCAP) atomicExch(q_items + slot + i, b * 16 + first + i); else { atomicExch(q_err, 2); atomicOr(sticky_err, 2); }
            }
            __syncwarp();
        };

        double rho, drho;
        const int over = ladder(cand, rho, drho);
        auto round_first = [](int c) {
#if TO_FRAG_ROUNDS == 1
            return c >= 2 ? 2 : 1;
#elif TO_FRAG_ROUNDS == 2
            return c >= 4 ? 4 : 1;
#elif TO_FRAG_ROUNDS == 3
            return c >= 8 ? 8 : (c >= 2 ? 2 : 1);
#elif TO_FRAG_ROUNDS == 4
            return c >= 8 ? 8 : 1;
#elif TO_FRAG_ROUNDS == 5
            return 1;
#else
            int lo = 1; while (2 * lo <= c) lo *= 2; return lo;
#endif
        };
        auto round_next = [](int first) {                                  // first candidate of the following round (16 = none)
#if TO_FRAG_ROUNDS == 1
            return first == 1 ? 2 : 16;
#elif TO_FRAG_ROUNDS == 2
            return first == 1 ? 4 : 16;
#elif TO_FRAG_ROUNDS == 3
            return first == 1 ? 2 : (first == 2 ? 8 : 16);
#elif TO_FRAG_ROUNDS == 4
            return first == 1 ? 8 : 16;
#elif TO_FRAG_ROUNDS == 5
            return 16;
#else
            return 2 * first;
#endif
        };
        const bool first_of_round = cand == 0 || cand == round_first(cand);   // the lowest candidate of a round stores its gains speculatively
        bool ok = false;
        int myslot = 0xFFFF;
        double* dVdst = P.dV + 2 * (size_t)b;
        bool store = first_of_round;
        if (!first_of_round && !over) {        // a speculative candidate: gains into a pool slot, copied into place if it wins its round
            int sl = 0;
            if (lane == 0) sl = atomicAdd(q_nslot, 1);
            sl = __shfl_sync(0xffffffffu, sl, 0);
            if (sl < nslots && sl < 0xFFFF) {
                myslot = sl; store = true;
                Kdst = pool + (size_t)sl * slot_stride; ddst = Kdst + (size_t)(N - 1) * 48; dVdst = Kdst + (size_t)(N - 1) * 52;
            }
        }
        if (cand == 0 || !over) ok = sweep(rho, store, !first_of_round);
        // the lowest candidate of a round stores in place: if it succeeds it IS the winner, its gains and dV are final
        if (ok && store) write_dV(rho, dVdst);
        if (myslot != 0xFFFF) { __threadfence(); __syncwarp(); }      // every lane's pool stores precede lane 0's atomicMin below
        Kdst = Kg; ddst = dg;
        if (cand == 0) {
            if (ok) finalise(rho, drho, 0);
            else start_round(1, round_next(1) - 1);
            continue;
        }
        // a candidate of round [lo, 2 lo): record, and let the last one to finish decide
        const int lo = round_first(cand);
        int last = 0;
        if (lane == 0) {
            if (ok) atomicMin(q_best + b, (cand << 16) | myslot);
            __threadfence();
            last = (atomicSub(q_cnt + b, 1) == 1) ? 1 : 0;
        }
        last = __shfl_sync(0xffffffffu, last, 0);
        if (!last) continue;
        int best = 0;
        if (lane == 0) { best = atomicAdd(q_best + b, 0); __threadfence(); }
        best = __shfl_sync(0xffffffffu, best, 0);
        const int bslot = best & 0xFFFF;
        best >>= 16;
        if (best < 16) {
            ladder(best, rho, drho);
            // gains and dV of the round's lowest candidate (lo) are in place; another winner's are in its pool slot (written before its
            // atomicMin / fence, read here after ours, past L1) -- or, without a slot, recomputed by one more sweep
            if (best != lo) {
                if (bslot != 0xFFFF) {
                    const double* src = pool + (size_t)bslot * slot_stride;
                    for (int i = lane; i < (N - 1) * 48; i += 32) Kg[i] = __ldcg(src + i);
                    for (int i = lane; i < (N - 1) * 4; i += 32) dg[i] = __ldcg(src + (size_t)(N - 1) * 48 + i);
                    if (lane < 2) P.dV[2 * (size_t)b + lane] = __ldcg(src + (size_t)(N - 1) * 52 + lane);
                } else { sweep(rho, true, false); write_dV(rho, P.dV + 2 * (size_t)b); }
            }
            finalise(rho, drho, best);
            continue;
        }
        // nobody succeeded: the sequential loop gives up at the first rho beyond bp_reg_max, else the next round
        const int hi = round_next(lo) - 1;
        const int ov = ladder(hi, rho, drho);
        if (ov) { ladder(ov, rho, drho); finalise(rho, drho, -1); continue; }
        if (hi < 15) { start_round(hi + 1, round_next(hi + 1) - (hi + 1)); continue; }
        // ladder longer than 15 steps (a huge bp_reg_max): finish sequentially in this warp
        int status = -1;
        for (int j = 16; ; j++) {
            reg_increase(P.opt, rho, drho);
            if (rho > P.opt.bp_reg_max) break;
            if (sweep(rho, true, false)) { status = j; write_dV(rho, P.dV + 2 * (size_t)b); break; }
        }
        finalise(rho, drho, status);
    }
}

}  // namespace

cudaError_t launch_expansion_rec(const DevProblem& P, cudaStream_t s) {
    if (inst_backward(P)) k_expansion_rec<true><<<nblk((long long)P.B * P.N, 128), 128, 0, s>>>(P);
    else k_expansion_rec<false><<<nblk((long long)P.B * P.N, 128), 128, 0, s>>>(P);
    return cudaGetLastError();
}
cudaError_t launch_export_abe(const DevProblem& P, cudaStream_t s) {
    k_export_abe<<<nblk((long long)P.B * (P.N - 1) * 16, 128), 128, 0, s>>>(P);
    return cudaGetLastError();
}

size_t frag_queue_ints(int B) { return 8 + (size_t)B + (16 * (size_t)B + 8192) + (size_t)B; }
// gain pool of the speculative candidates: one slot per instance up to 4096, and at most 1 GiB (a candidate without a slot is recomputed if it wins)
int frag_pool_slots(int B, int N) {
    const size_t slot = ((size_t)(N - 1) * 52 + 2) * sizeof(double);
    size_t n = B < 4096 ? B : 4096;
    if (n * slot > ((size_t)1 << 30)) n = ((size_t)1 << 30) / slot;
    return (int)(n < 1 ? 1 : n);
}
size_t frag_pool_doubles(int B, int N) { return (size_t)frag_pool_slots(B, N) * ((size_t)(N - 1) * 52 + 2); }

namespace {
constexpr int FRAG_WARPS = TO_FRAG_WARPS;
// per-device launch configuration (one process may hold handles on several GPUs): the SM count and the CTAs the occupancy API fits per SM
int ctas_per_sm[TO_MAXDEV] = {0}, num_sms[TO_MAXDEV] = {0};
cudaError_t frag_configure(int dev) {
    if (ctas_per_sm[dev]) return cudaSuccess;
    auto kern = k_riccati_frag<TO_FRAG_STAGES, FRAG_WARPS, TO_FRAG_MINB>;
    const int smem = (int)sizeof(FragSmem<TO_FRAG_STAGES, FRAG_WARPS>);
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return e;
    cudaDeviceGetAttribute(&num_sms[dev], cudaDevAttrMultiProcessorCount, dev);
    int c = 0;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&c, kern, 32 * FRAG_WARPS, smem);
    if (e != cudaSuccess) return e;
    ctas_per_sm[dev] = c < 1 ? 1 : c;
    return cudaSuccess;
}
}  // namespace

int frag_resident_warps() {
    const int dev = current_device_slot();
    return frag_configure(dev) == cudaSuccess ? num_sms[dev] * ctas_per_sm[dev] * FRAG_WARPS : 0;
}

cudaError_t launch_backward_frag(const DevProblem& P, int* queue, double* pool, int* sticky_err, cudaStream_t s) {
    constexpr int STAGES = TO_FRAG_STAGES, WARPS = FRAG_WARPS;
    using SM = FragSmem<STAGES, WARPS>;
    auto kern = k_riccati_frag<STAGES, WARPS, TO_FRAG_MINB>;
    const int smem = (int)sizeof(SM);
    const int dev = current_device_slot();
    cudaError_t e = frag_configure(dev);
    if (e != cudaSuccess) return e;
    // queue layout (k_riccati_frag): head, tail, nfinal, error, pool slots, 3 x pad | cnt[B] = 0 | items[16 B + 8192] = -1 | best[B] = 0x7f7f7f7f
    const size_t qcap = 16 * (size_t)P.B + 8192;
    e = cudaMemsetAsync(queue, 0, sizeof(int) * (8 + (size_t)P.B), s);
    if (e == cudaSuccess) e = cudaMemsetAsync(queue + 8 + P.B, 0xFF, sizeof(int) * qcap, s);
    if (e == cudaSuccess) e = cudaMemsetAsync(queue + 8 + P.B + qcap, 0x7F, sizeof(int) * (size_t)P.B, s);
    if (e != cudaSuccess) return e;
    int grid = num_sms[dev] * ctas_per_sm[dev];       // persistent: warps pull work from the queue (all CTAs are co-resident: the
    const int need = (P.B + WARPS - 1) / WARPS;       // waiting warps of the speculative ladder cannot starve the running ones)
    if (grid > need) grid = need;
    kern<<<grid, 32 * WARPS, smem, s>>>(P, queue, pool, pool ? frag_pool_slots(P.B, P.N) : 0, sticky_err);
    return cudaGetLastError();
}
