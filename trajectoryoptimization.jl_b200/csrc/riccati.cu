// riccati.cu -- kernel 3 of the hot path: the dense Riccati backward pass of iLQR for a batch of instances.
//
// What it computes (Altro.jl backwardpass!, which drives the reference's expansions; restated in
// oracle/oracle.hpp `backward_pass`; SURVEY.md 8 a14), per instance, serial in k = N-1 .. 1:
//     Qzz = lzz + [A B]' S [A B]      Qz = lz + [A B]' s          (z = [x;u], lzz/lz = cost + AL expansion)
//     K = -(Quu + rho I)^-1 Qux       d = -(Quu + rho I)^-1 Qu    (non-PD Quu + rho I -> rho increase + restart)
//     S <- Qxx + K'Quu K + K'Qux + Qux'K     s <- Qx + K'Quu d + K'Qu + Qux'd     dV += (d'Qu, 1/2 d'Quu d)
// With W = Qux - rho K the update collapses to S <- Qxx + W'K, s <- Qx + W'd (identical algebra, Quu K = -Qux - rho K).
// The cost expansion consumed here is the reference's RD.gradient!/RD.hessian! (src/cost_functions.jl:137-233)
// plus the AL terms built from projection!/grad-projection! (src/cones.jl:96-145) for Goal/Bound constraints
// (src/constraints.jl:55-68, :738-765), whose Jacobians are +-1 selectors, so both are diagonal in z.
//
// Mapping
//   * one WARP per instance (the recursion is serial in k; B=4096 gives ~28 instances per SM, so intra-instance
//     parallelism has to fill the FP64 pipe).  Persistent one-warp CTAs pull instances from an atomic queue.
//   * [A B]_k (n x LDAB doubles, contiguous per knot thanks to the instance-major layout) is streamed from HBM
//     by 1-D bulk TMA copies (cp.async.bulk + mbarrier complete_tx) into a multi-stage shared-memory ring, issued
//     by lane 0 several knots ahead of use -- this is the dominant HBM traffic of the whole iteration.
//   * T = S [A B] (with s appended as an extra column), then Qzz|Qz = [A B]' T restricted to the upper tiles.
//     n >= 8 (Quadrotor): FP64 tensor-core MMA, mma.sync m8n8k4 (SASS DMMA).  2x2 register micro-blocks with DFMA
//     load the SHARED-MEMORY pipe instead (an LDS.128 takes 4 wavefronts, broadcast or not, i.e. 4 B per lane per
//     cycle; a DFMA needs two fresh operands).  A DMMA moves 256 FMAs with one 8-byte operand per lane per fragment,
//     ~5x fewer wavefronts per FLOP, so the kernel is bound by the FP64 pipe
//     (profiles/microbench/fp64_pipes.cu measures the DMMA and DFMA rates).  K = n is split into n/4 MMA k-steps plus
//     rank-1 DFMA updates for the n%4 remainder; smem row strides are = 4 (mod 16) doubles so that the 8x4 / 4x8
//     fragment loads are bank-conflict free.
//     n < 8 (Cartpole, Acrobot, double integrator): 2x2 register micro-blocks with DFMA (tiles would be >75% padding).
//   * lane i < n+m owns z_i: its cost / AL descriptors live in registers for the whole kernel, and z_i, lambda of the
//     NEXT knot are prefetched while the current knot's products run (global latency off the critical path).
//   * Quu + rho I is m x m (m <= 8): LDL' with reciprocal pivots (no fp64 sqrt / division chain) and the triangular
//     solves are done per right-hand-side column, one lane per column of [Qux Qu], in registers.
#include <cstddef>

#include "costcon.cuh"
#include "kernels.h"

#ifndef TO_RICCATI_STAGES
#define TO_RICCATI_STAGES 2     // depth of the [A B] ring
#endif
#ifndef TO_RICCATI_MINB
#define TO_RICCATI_MINB 16   // one-warp CTAs per SM of the tensor-MMA kernel (A/B: profiles/build_variants.sh)
#endif

// register cap of k_riccati: by default from the CTAs-per-SM target; TO_RICCATI_MAXREG pins it instead (ptxas rounds the
// launch-bounds cap down to 96 for 18 CTAs although 112 fit)
#ifdef TO_RICCATI_MAXREG
#define TO_RICCATI_BOUNDS(MINB) __maxnreg__(TO_RICCATI_MAXREG)
#else
#define TO_RICCATI_BOUNDS(MINB) __launch_bounds__(32, MINB)
#endif

namespace {

__host__ __device__ constexpr int even_up(int v) { return (v + 1) & ~1; }
constexpr int MAXT = 3;   // AL terms per z entry kept in registers (e.g. upper bound + lower bound + goal)

__device__ __forceinline__ double2 lds128(const double* p) { return *reinterpret_cast<const double2*>(p); }
__device__ __forceinline__ void sts128(double* p, double a, double b) { *reinterpret_cast<double2*>(p) = make_double2(a, b); }

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
// 1-D bulk TMA copy global -> shared, completion signalled on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// global load the compiler may not sink towards its use (prefetch of the next knot's operands)
__device__ __forceinline__ double ldg_pinned(const double* p) {
    double v;
    asm volatile("ld.global.nc.f64 %0, [%1];" : "=d"(v) : "l"(p));
    return v;
}

__device__ __forceinline__ int ldg_pinned(const int* p) {
    int v;
    asm volatile("ld.global.nc.s32 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
}

// 1/x for a positive finite pivot: hardware seed (MUFU.RCP64H, >= 20 bits) + two Newton steps -> <= 1 ulp, without
// the rounding / special-case fix-up of __drcp_rn (12 dependent instructions + a branch on the knot's critical chain)
__device__ __forceinline__ double rcp_pivot(double x) {
    double y;
    asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(x));
    double e = fma(-x, y, 1.0);
    y = fma(y, e, y);
    e = fma(-x, y, 1.0);
    return fma(y, e, y);
}

// 2x2 micro-block outer-product accumulate
__device__ __forceinline__ void fma2x2(double (&acc)[4], const double2& a, const double2& b) {
    acc[0] = fma(a.x, b.x, acc[0]);
    acc[1] = fma(a.x, b.y, acc[1]);
    acc[2] = fma(a.y, b.x, acc[2]);
    acc[3] = fma(a.y, b.y, acc[3]);
}

__device__ __forceinline__ void dmma(double& d0, double& d1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
}

template <int N_, int M_, int STAGES, bool MMA>
struct RiccatiSmem {
    static constexpr int NM = N_ + M_;
    static constexpr int NP = even_up(N_);          // padded state dim
    static constexpr int MMA_LD = 20;               // = 4 (mod 16): conflict-free m8n8k4 fragment loads
    static constexpr int LDAB = (N_ >= 8 && N_ <= 16 && NM + 1 <= MMA_LD) ? MMA_LD : even_up(NM);   // row stride of [A B] in HBM == P.ldab (to_create)
    static constexpr int LDABS = LDAB;                            // ... and in shared memory (one bulk copy per knot)
    static constexpr int LDS_ = MMA ? MMA_LD : NP;                // S
    static constexpr int LDT = MMA ? MMA_LD : even_up(NM + 1);    // T / Q: one extra column carries s / Qz
    static constexpr int SROWS = MMA ? 16 : NP;
    static constexpr int TROWS = MMA ? 16 : NP;
    static constexpr int LDK = MMA ? MMA_LD : even_up(N_ + 1);    // K|d row stride
    static constexpr int LDQS = even_up(M_ + 1);    // u / Qz strip of Q (MMA path): columns n..NM
    static constexpr int AB_BYTES = N_ * LDAB * 8;
    static constexpr int AB_STRIDE = (N_ * LDABS * 8 + 127) / 128 * 16;   // doubles, 128-byte aligned stages
    static_assert(!MMA || (N_ <= 16 && NM + 1 <= MMA_LD && N_ >= 8 && M_ <= 4), "MMA path: 8 <= n <= 16, m <= 4, n+m+1 <= 20");
    double ab[STAGES][AB_STRIDE];
    double S[SROWS * LDS_];
    double T[TROWS * LDT + 8];
    double Q[MMA ? 2 : even_up(NM) * LDT + 8];   // full Q only on the DFMA path
    // u / Qz strip of Q, gains K|d and W = Qux - rho K.  MMA path: they overlay T, which is dead once Q sits in the
    // accumulator registers and is rewritten only by the next knot (2.2 KB per warp -> room for 18-20 warps per SM)
    static constexpr int QS_SIZE = (NM + 1) * LDQS, KW_SIZE = 4 * LDK + 8;
    static_assert(!MMA || QS_SIZE + 2 * KW_SIZE <= TROWS * LDT + 8, "overlay does not fit T");
    double QKW[MMA ? 2 : QS_SIZE + 2 * KW_SIZE];
    __device__ __forceinline__ double* qs() { return MMA ? T : QKW; }
    __device__ __forceinline__ double* kk() { return qs() + QS_SIZE; }
    __device__ __forceinline__ double* ww() { return kk() + KW_SIZE; }
    double g[MMA ? 2 : even_up(NM) + 2];   // lz (cost + AL gradient), padded (DFMA path; the MMA path keeps it in lane registers)
    double h[MMA ? 2 : even_up(NM) + 2];   // diag(lzz)
    // lane-indexed table of the Goal / Bound rows acting on z_lane (instance-independent, filled once per warp):
    // keeping it here instead of in registers is what lets the knot loop fit 128 registers without spills
    static constexpr int NMT = even_up(NM);
    double tnms[MAXT][NMT];      // -mu * sign  (sign = +1: c = z - bound, -1: c = bound - z ; mu = |.|)
    double tbound[MAXT][NMT];
    uint2 tpk[MAXT][NMT];        // see pack_term
    // scratch of the general-constraint AL expansion (Linear / Circle / Sphere / Norm incl. SOC), DFMA path only
    static constexpr int GP = MMA ? 1 : 16;         // rows of one general constraint handled by the solver kernels
    double gc[GP], glbar[GP], glp[GP], gD[GP * GP], gjac[GP * (MMA ? 1 : TO_MAXNM)], gtmp[GP * (MMA ? 1 : TO_MAXNM)];
    uint64_t bar[STAGES];
};

// one AL term acting on z_i:  c = sign * (z_i - bound) ;  Goal: equality (always active), Bound: inequality.
// Packed into RiccatiSmem::tnms / tbound / tpk; the packing limits (N < 4095, p < 128) are checked
// by launch_riccati_nm, which otherwise takes the generic (FASTAL = false) expansion.
__device__ __forceinline__ uint2 pack_term(int first, int last, int base, int p, bool eq) {
    // x = first (12 bits) | last - first (12) | p (7) | eq (1) ;  y = lambda index of the row at knot 0 (= base - first p)
    const int span = last >= first ? last - first : 0;
    const int f = last >= first ? first : 4095;              // empty range: never active for knots <= 4094
    return make_uint2((unsigned)f | ((unsigned)span << 12) | ((unsigned)p << 24) | (eq ? 0x80000000u : 0u), (unsigned)(base - f * p));
}

template <int N_, int M_, int STAGES, bool FASTAL, bool MMA, int MINB, int NSLOT, bool INST>
__global__ void TO_RICCATI_BOUNDS(MINB) k_riccati(const DevProblem P, int* __restrict__ work_counter) {
    using SM = RiccatiSmem<N_, M_, STAGES, MMA>;
    constexpr int n = N_, m = M_, NM = SM::NM, LDAB = SM::LDAB, LDT = SM::LDT, NP = SM::NP, LDK = SM::LDK;
    constexpr int LDABS = SM::LDABS, LDS_ = SM::LDS_;
    // MMA tiling: T (n x NM+1) = S (n x n) [A B | s] ; Q (NM x NM+1) upper tiles = [A B]' T
    constexpr int MT = (n + 7) / 8, NT = (NM + 1 + 7) / 8, MQ = (NM + 7) / 8, KS = n / 4, KR = n % 4;
    constexpr int NQT = MQ * NT - MQ * (MQ - 1) / 2;        // upper tiles (mi <= ni)
    constexpr int RBT = NP / 2, CBT = even_up(NM) / 2;       // T blocks: rows of S x column pairs of [A B]
    constexpr int NBT = RBT * CBT;
    constexpr int RT = (NBT + 31) / 32;
    constexpr int RBQ = even_up(NM) / 2, CBQ = even_up(NM + 1) / 2;   // Q blocks (upper: cb >= rb)
    constexpr int NBQ = RBQ * CBQ - RBQ * (RBQ - 1) / 2;
    constexpr int RQ = (NBQ + 31) / 32;
    constexpr int RBS = NP / 2;                              // S blocks (upper)
    constexpr int NBS = RBS * (RBS + 1) / 2;
    constexpr int RS = (NBS + 31) / 32;
    constexpr bool NM_ODD = (NM & 1) != 0;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    SM& sm = *reinterpret_cast<SM*>(smem_raw);
    double* const Qs_ = sm.qs(); double* const K_ = sm.kk(); double* const W_ = sm.ww();
    const int lane = threadIdx.x;
    const int N = P.N;

    // ---- loop-invariant lane -> block assignments (element offsets into the smem matrices) -----------------
    int t_a[RT], t_b[RT], t_o[RT]; bool t_on[RT], t_lastcol[RT];
#pragma unroll
    for (int r = 0; r < RT; r++) {
        int id = lane + 32 * r; t_on[r] = id < NBT; if (!t_on[r]) id = NBT - 1;
        const int rb = id / CBT, cb = id % CBT;
        t_a[r] = 2 * rb; t_b[r] = 2 * cb; t_o[r] = (2 * rb) * LDT + 2 * cb;
        t_lastcol[r] = NM_ODD && (cb == CBT - 1);   // the block's second column is the pad column, where s is stored
    }
    int q_a[RQ], q_b[RQ], q_o[RQ], q_i0[RQ], q_j0[RQ]; bool q_on[RQ], q_diag[RQ];
#pragma unroll
    for (int r = 0; r < RQ; r++) {
        int id = lane + 32 * r; q_on[r] = id < NBQ; if (!q_on[r]) id = NBQ - 1;
        int rb = 0, rem = id;                                  // row rb holds CBQ - rb blocks
        while (rem >= CBQ - rb) { rem -= CBQ - rb; rb++; }
        const int cb = rb + rem;
        q_a[r] = 2 * rb; q_b[r] = 2 * cb; q_o[r] = (2 * rb) * LDT + 2 * cb; q_i0[r] = 2 * rb; q_j0[r] = 2 * cb; q_diag[r] = (rb == cb);
    }
    int s_a[RS], s_b[RS]; bool s_on[RS], s_diag[RS];
#pragma unroll
    for (int r = 0; r < RS; r++) {
        int id = lane + 32 * r; s_on[r] = id < NBS; if (!s_on[r]) id = NBS - 1;
        int rb = 0, rem = id;
        while (rem >= RBS - rb) { rem -= RBS - rb; rb++; }
        s_a[r] = 2 * rb; s_b[r] = 2 * (rb + rem); s_diag[r] = (rem == 0);
    }

    // ---- lane-resident AL terms of z_lane (Goal / Bound constraints) ----------------------------------------
    int tinst[MAXT];   // (INST) index of a term's bound in an instance's row of P.cdata, -1: none
#pragma unroll
    for (int t = 0; t < MAXT; t++) tinst[t] = -1;
    if (FASTAL) {
        if (lane < SM::NMT) {
#pragma unroll
            for (int t = 0; t < MAXT; t++) { sm.tnms[t][lane] = -1.0; sm.tbound[t][lane] = 0.0; sm.tpk[t][lane] = pack_term(1, 0, 0, 0, false); }   // empty range
        }
        int nterm = 0;
        if (lane < NM) {
            for (int ci = 0; ci < P.ncon; ci++) {
                const DevCon& con = P.cons[ci];
                const double mu = P.mu[ci];
                for (int side = 0; side < 2; side++) {
                    int row = -1; double sign = 1.0, bound = 0.0; bool eq = false;
                    if (con.kind == CON_GOAL) { if (side == 0 && lane < n) { row = con.row_max[lane]; if (row >= 0) bound = con.a[row]; eq = true; } }
                    else if (side == 0) { row = con.row_max[lane]; bound = con.a[lane]; }
                    else { row = con.row_min[lane]; bound = con.b[lane]; sign = -1.0; }
                    if (row < 0) continue;
                    if (nterm < MAXT) { sm.tnms[nterm][lane] = -mu * sign; sm.tbound[nterm][lane] = bound; sm.tpk[nterm][lane] = pack_term(con.first, con.last, con.offset + row, con.p, eq); }
                    if (INST && nterm < MAXT) {
                        const int src = con.cdoff + (eq ? row : (side ? n + m : 0) + lane);
#pragma unroll
                        for (int t = 0; t < MAXT; t++) if (t == nterm) tinst[t] = src;
                    }
                    nterm++;
                }
            }
        }
        (void)nterm;   // NSLOT (template) >= the largest per-lane count: launch_riccati_nm picks it from P.max_terms_per_z
    }

    for (int e = lane; e < 4 * LDK + 8; e += 32) { K_[e] = 0.0; W_[e] = 0.0; }   // padding columns stay finite
    if (lane == 0) {
#pragma unroll
        for (int s = 0; s < STAGES; s++) mbar_init(&sm.bar[s], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncwarp();
    uint32_t phase_bits = 0;   // per-stage parity of the next completion to wait for

    for (;;) {
        int b = 0;
        if (lane == 0) b = atomicAdd(work_counter, 1);
        b = __shfl_sync(0xffffffffu, b, 0);
        if (b >= P.B) break;
        if (retired(P, b)) continue;            // to_solve: not ACTIVE
        if constexpr (INST && FASTAL) {         // this instance's Goal / Bound values into the lane-resident terms (read back by this lane only)
            if (lane < NM) {
#pragma unroll
                for (int t = 0; t < MAXT; t++)
                    if (P.cdata && tinst[t] >= 0) sm.tbound[t][lane] = P.cdata[(size_t)b * P.ncdata + tinst[t]];
            }
        }

        const int buf = P.cur[b];
        const double* X = traj_X(P, buf, b);
        const double* U = traj_U(P, buf, b);
        const double* lam_b = P.lambda + (size_t)b * P.lambda_len;
        const double* ABg = P.AB + (size_t)b * (N - 1) * n * LDAB;
        double* Kg = P.K + (size_t)b * (N - 1) * n * m;
        double* dg = P.d + (size_t)b * (N - 1) * m;
        double rho = P.rho[b], drho = P.drho[b];
        int restarts = 0;
        bool failed = false;
        // address of z_lane at knot k (0-based): x part or u part
        const double* zbase = (lane < n) ? (X + lane) : (U + (lane < NM ? lane - n : 0));
        const int zstride = (lane < n) ? n : m;

        // the expansion of one knot for this lane: (gi, hi) = (lz_i, lzz_ii) from z_i and its multipliers
        // (cH, cG) = (Qd_i | Rd_i, q_i | r_i) of this lane's z_i for a DiagonalCost
        // DevCost keeps Qd | Rd | q | r contiguous, so q_i - Qd_i == r_a - Rd_a: one per-lane offset serves H and G
        const int coff = (lane < n) ? (int)offsetof(DevCost, Qd) + 8 * lane : (int)offsetof(DevCost, Rd) + 8 * (lane < NM ? lane - n : 0);
        constexpr int GOFF = (int)(offsetof(DevCost, q) - offsetof(DevCost, Qd));
        static_assert(offsetof(DevCost, r) - offsetof(DevCost, Rd) == offsetof(DevCost, q) - offsetof(DevCost, Qd), "DevCost layout");
        auto cost_coeff_ptr = [&](int cid, bool hess) -> const double* {
            return reinterpret_cast<const double*>(reinterpret_cast<const char*>(P.costs) + (size_t)cid * sizeof(DevCost) + coff + (hess ? 0 : GOFF));
        };
        // cG of cost cid: the instance's own q | r row when INST (same lane -> entry mapping: q_i | r_a sit at i | n + a)
        auto cost_g_ptr = [&](int cid) -> const double* {
            if constexpr (INST) { if (P.qr) return inst_q<true>(P, b, cid) + (lane < NM ? lane : n); }
            return cost_coeff_ptr(cid, false);
        };
        // act: bit t = term slot t is active at the knot, bit 4 + t = it is an equality (computed by load_lams one knot ahead)
        auto expand_fast = [&](double zi, const double (&lam)[MAXT], int act, double cH, double cG, double& gi, double& hi) {
            gi = fma(cH, zi, cG); hi = cH;
#pragma unroll
            for (int t = 0; t < MAXT; t++) {
                if (t < NSLOT && (act & (1 << t))) {
                    const double nms = sm.tnms[t][lane];
                    const double lb = fma(nms, zi - sm.tbound[t][lane], lam[t]);   // lambda - mu c
                    if ((act & (16 << t)) || lb <= 0.0) { gi += (nms < 0.0) ? -lb : lb; hi += fabs(nms); }   // g -= sign lb ; h += mu
                }
            }
        };
        auto load_lams = [&](int k, double (&lam)[MAXT], int& act) {
            act = 0;
#pragma unroll
            for (int t = 0; t < MAXT; t++) {
                lam[t] = 0.0;
                if (t < NSLOT) {
                    const uint2 pk = sm.tpk[t][lane];
                    if ((unsigned)(k + 1) - (pk.x & 0xfffu) <= ((pk.x >> 12) & 0xfffu)) {
                        lam[t] = ldg_pinned(lam_b + (int)(pk.y + (unsigned)(k + 1) * ((pk.x >> 24) & 0x7fu)));
                        act |= (1 << t) | ((pk.x >> 31) << (4 + t));
                    }
                }
            }
        };

        // AL expansion of the non-selector constraints active at knot k1 (1-based): Gauss-Newton terms
        //   grad -= (D cz)' lp ,  hess += mu (D cz)'(D cz)   with D = grad Pi_K*(lambda - mu c), lp = Pi_K*(lambda - mu c)
        // added to [Q | Qz] (stage knots) or to S / s (terminal).  Warp-cooperative slow path; lane 0 evaluates c and cz.
        auto general_constraints = [&](int k1, bool terminal, double& s_lane) {
            if constexpr (!MMA) {
                for (int ci = 0; ci < P.ncon; ci++) {
                    const DevCon& con = P.cons[ci];
                    if (con.diagonal || k1 < con.first || k1 > con.last) continue;
                    const int p = con.p;
                    const double mu = P.mu[ci];
                    const double* lam = lam_b + con.offset + (size_t)(k1 - con.first) * p;
                    const double* xk = X + (size_t)(k1 - 1) * n;
                    if (lane == 0) {
                        double uz[M_];
                        for (int a = 0; a < m; a++) uz[a] = terminal ? 0.0 : U[(size_t)(k1 - 1) * m + a];
                        if constexpr (INST) {
                            const ConData cd = con_data<true>(P, b, ci);
                            con_evaluate(con, cd, n, m, xk, uz, sm.gc);
                            con_jacobian(con, cd, n, m, xk, uz, sm.gjac);
                        } else {
                            con_evaluate(con, n, m, xk, uz, sm.gc);
                            con_jacobian(con, n, m, xk, uz, sm.gjac);
                        }
                    }
                    __syncwarp();
                    if (lane < p) sm.glbar[lane] = lam[lane] - mu * sm.gc[lane];
                    __syncwarp();
                    if (lane == 0) { const int dc = dualcone(con.sense); cone_projection(dc, sm.glbar, p, sm.glp); cone_grad_projection(dc, sm.glbar, p, sm.gD); }
                    __syncwarp();
                    for (int e = lane; e < p * NM; e += 32) {
                        const int i = e % p, j = e / p;
                        double t = 0.0;
                        for (int r = 0; r < p; r++) t = fma(sm.gD[r * p + i], sm.gjac[j * p + r], t);
                        sm.gtmp[j * p + i] = t;
                    }
                    __syncwarp();
                    const int lim = terminal ? n : NM;
                    if (lane < lim) {
                        double gsum = 0.0;
                        for (int i = 0; i < p; i++) gsum = fma(sm.gtmp[lane * p + i], sm.glp[i], gsum);
                        if (terminal) s_lane -= gsum; else sm.Q[lane * LDT + NM] -= gsum;
                    }
                    for (int e = lane; e < lim * lim; e += 32) {
                        const int j = e / lim, j2 = e % lim;
                        if (!terminal && (j >> 1) > (j2 >> 1)) continue;      // Q keeps its upper 2x2 blocks
                        double hs = 0.0;
                        for (int i = 0; i < p; i++) hs = fma(sm.gtmp[j * p + i], sm.gtmp[j2 * p + i], hs);
                        if (terminal) sm.S[j * LDS_ + j2] += mu * hs; else sm.Q[j * LDT + j2] += mu * hs;
                    }
                    __syncwarp();
                }
            }
        };

        // stream [A B]_k into ring slot st with one bulk TMA copy
        auto issue_ab = [&](int st, int k) {
            if (lane == 0) {
                mbar_expect_tx(&sm.bar[st], SM::AB_BYTES);
                bulk_g2s(sm.ab[st], ABg + (size_t)k * n * LDAB, SM::AB_BYTES, &sm.bar[st]);
            }
        };

        for (;;) {   // regularisation restart loop
            // ---- prologue: start streaming the last STAGES knots ----------------------------------------
#pragma unroll
            for (int s = 0; s < STAGES; s++) {
                const int k = N - 2 - s;
                if (k >= 0) issue_ab(s, k);
            }
            // ---- terminal knot: S = lxx_N, s = lx_N (cost + AL) ------------------------------------------
            for (int e = lane; e < SM::SROWS * LDS_; e += 32) sm.S[e] = 0.0;
            __syncwarp();
            double s_reg = 0.0;   // lane i < n holds s_i
            {
                const int cidN = P.cost_index[N - 1];
                const DevCost& cost = P.costs[cidN];
                const double* cq = inst_q<INST>(P, b, cidN);
                if (lane < n) {
                    const int i = lane;
                    const double xi = X[(size_t)(N - 1) * n + i];
                    double gi, hi;
                    if (FASTAL && cost.diag) {
                        double lam[MAXT];
                        int act; load_lams(N - 1, lam, act);
                        expand_fast(xi, lam, act, cost.Qd[lane], cq[lane], gi, hi);
                        sm.S[i * LDS_ + i] = hi;
                    } else {
                        gi = cq[i]; hi = 0.0;
                        if (cost.diag) { gi = fma(cost.Qd[i], xi, gi); hi = cost.Qd[i]; }
                        else {
                            for (int j = 0; j < n; j++) { gi = fma(cost.Q[j * n + i], X[(size_t)(N - 1) * n + j], gi); sm.S[j * LDS_ + i] = cost.Q[j * n + i]; }
                        }
                        for (int ci = 0; ci < P.ncon; ci++) {
                            const DevCon& con = P.cons[ci];
                            if (N < con.first || N > con.last) continue;
                            const double mu = P.mu[ci];
                            const double* lam = lam_b + con.offset + (size_t)(N - con.first) * con.p;
                            if (con.kind == CON_GOAL) {
                                const int row = con.row_max[i];
                                if (row >= 0) { const double lp = lam[row] - mu * (xi - con_row<INST>(P, b, ci, con.a)[row]); gi -= lp; hi += mu; }
                            } else if (con.kind == CON_BOUND) {
                                const double* ba = con.a; const double* bb = con.b;
                                if constexpr (INST) { const ConData cd = con_data<true>(P, b, ci); ba = cd.a; bb = cd.b; }
                                int row = con.row_max[i];
                                if (row >= 0) { const double lb = lam[row] - mu * (xi - ba[i]); if (lb <= 0) { gi -= lb; hi += mu; } }
                                row = con.row_min[i];
                                if (row >= 0) { const double lb = lam[row] - mu * (bb[i] - xi); if (lb <= 0) { gi += lb; hi += mu; } }
                            }
                        }
                        if (cost.diag) sm.S[i * LDS_ + i] = hi; else sm.S[i * LDS_ + i] += hi;
                    }
                    s_reg = gi;
                }
            }
            if (!P.all_diag_con) { __syncwarp(); general_constraints(N, true, s_reg); }
            // operands of the first stage knot
            double z_cur = 0.0, lam_cur[MAXT];
#pragma unroll
            for (int t = 0; t < MAXT; t++) lam_cur[t] = 0.0;
            int act_cur = 0;
            if (lane < NM) { z_cur = zbase[(size_t)(N - 2) * zstride]; if (FASTAL) load_lams(N - 2, lam_cur, act_cur); }
            // software pipeline of the cost coefficients: (cH,cG) of knot k are loaded during knot k+1, its index during knot k+2
            double cH_cur = 0.0, cG_cur = 0.0;
            int cid_next = (N >= 3) ? P.cost_index[N - 3] : 0;
            if (FASTAL && P.all_diag_cost) { const int c0 = P.cost_index[N - 2]; cH_cur = *cost_coeff_ptr(c0, true); cG_cur = *cost_g_ptr(c0); }
            __syncwarp();

            double dV1 = 0.0, dV2 = 0.0;   // accumulated by lane n
            bool ok = true;
            int stage = 0;
            int k;
            double g_reg = 0.0, h_reg = 0.0;
            for (k = N - 2; k >= 0; k--) {
                // ---- prefetch z_i / multipliers of the next knot (k-1); consumed one iteration later -------
                double z_nxt = 0.0, lam_nxt[MAXT];
#pragma unroll
                for (int t = 0; t < MAXT; t++) lam_nxt[t] = 0.0;
                int act_nxt = 0;
                if (k > 0 && lane < NM) { z_nxt = ldg_pinned(zbase + (size_t)(k - 1) * zstride); if (FASTAL) load_lams(k - 1, lam_nxt, act_nxt); }
                double cH_nxt = 0.0, cG_nxt = 0.0;
                int cid_next2 = 0;
                if (FASTAL && P.all_diag_cost && k > 0) {
                    cH_nxt = ldg_pinned(cost_coeff_ptr(cid_next, true)); cG_nxt = ldg_pinned(cost_g_ptr(cid_next));
                    if (k > 1) cid_next2 = ldg_pinned(P.cost_index + (k - 2));
                }
                // ---- cost + AL expansion of knot k: lane i < NM handles z_i (diagonal terms) ------------
                {
                    g_reg = 0.0; h_reg = 0.0;
                    double gi = 0.0, hi = 0.0;
                    if (FASTAL && P.all_diag_cost) {
                        if (lane < NM) expand_fast(z_cur, lam_cur, act_cur, cH_cur, cG_cur, gi, hi);
                    } else if (lane < NM) {
                        const int cidk = P.cost_index[k];
                        const DevCost& cost = P.costs[cidk];
                        const double* cq = inst_q<INST>(P, b, cidk);
                        const double* cr = inst_r<INST>(P, b, cidk);
                        const int i = lane;
                        const double zi = z_cur;
                        if (FASTAL && cost.diag) {
                            expand_fast(zi, lam_cur, act_cur, (i < n) ? cost.Qd[i] : cost.Rd[i - n], (i < n) ? cq[i] : cr[i - n], gi, hi);
                        } else {
                            if (cost.diag) {
                                if (i < n) { gi = fma(cost.Qd[i], zi, cq[i]); hi = cost.Qd[i]; }
                                else { gi = fma(cost.Rd[i - n], zi, cr[i - n]); hi = cost.Rd[i - n]; }
                            } else {
                                if (i < n) {
                                    gi = cq[i];
                                    for (int j = 0; j < n; j++) gi = fma(cost.Q[j * n + i], X[(size_t)k * n + j], gi);
                                    if (!cost.zeroH) for (int a = 0; a < m; a++) gi = fma(cost.H[i * m + a], U[(size_t)k * m + a], gi);
                                } else {
                                    const int a = i - n;
                                    gi = cr[a];
                                    for (int j = 0; j < m; j++) gi = fma(cost.R[j * m + a], U[(size_t)k * m + j], gi);
                                    if (!cost.zeroH) for (int j = 0; j < n; j++) gi = fma(cost.H[j * m + a], X[(size_t)k * n + j], gi);
                                }
                            }
                            for (int ci = 0; ci < P.ncon; ci++) {
                                const DevCon& con = P.cons[ci];
                                if (k + 1 < con.first || k + 1 > con.last) continue;
                                const double mu = P.mu[ci];
                                const double* lam = lam_b + con.offset + (size_t)(k + 1 - con.first) * con.p;
                                if (con.kind == CON_GOAL) {
                                    const int row = (i < n) ? con.row_max[i] : -1;
                                    if (row >= 0) { const double lp = lam[row] - mu * (zi - con_row<INST>(P, b, ci, con.a)[row]); gi -= lp; hi += mu; }
                                } else if (con.kind == CON_BOUND) {
                                    const double* ba = con.a; const double* bb = con.b;
                                    if constexpr (INST) { const ConData cd = con_data<true>(P, b, ci); ba = cd.a; bb = cd.b; }
                                    int row = con.row_max[i];
                                    if (row >= 0) { const double lb = lam[row] - mu * (zi - ba[i]); if (lb <= 0) { gi -= lb; hi += mu; } }
                                    row = con.row_min[i];
                                    if (row >= 0) { const double lb = lam[row] - mu * (bb[i] - zi); if (lb <= 0) { gi += lb; hi += mu; } }
                                }
                            }
                        }
                    }
                    g_reg = gi; h_reg = hi;
                    if constexpr (!MMA) { if (lane < even_up(NM) + 2) { sm.g[lane] = gi; sm.h[lane] = hi; } }
                }
                // ---- wait for [A B]_k in the ring ------------------------------------------------------
                mbar_wait(&sm.bar[stage], (phase_bits >> stage) & 1u);
                phase_bits ^= (1u << stage);
                const double* sAB = sm.ab[stage];

                if constexpr (MMA) {
                    // Tensor-MMA knot (requires DiagonalCost + Goal/Bound: lzz is diagonal and lives in lane registers).
                    // lane's fragment coordinates: A(8x4): row fr, col fc ; B(4x8): row fc, col fr ; D(8x8): row fr, cols 2fc, 2fc+1
                    const int fr = lane >> 2, fc = lane & 3;
                    constexpr int LDQS = SM::LDQS;
                    // fragments of [A B]_k: B operand of T = S [A B], re-used as the A operand of Q = [A B]' T
                    double bfr[KS][NT];
#pragma unroll
                    for (int kk = 0; kk < KS; kk++)
#pragma unroll
                        for (int t = 0; t < NT; t++) bfr[kk][t] = sAB[(4 * kk + fc) * LDABS + 8 * t + fr];
                    // ---- T = S [A B | .] : S is kept as its upper 8x8 tiles, a lower tile is read as the transpose ----
                    {
                        double d[MT][NT][2];
#pragma unroll
                        for (int mi = 0; mi < MT; mi++)
#pragma unroll
                            for (int ni = 0; ni < NT; ni++) { d[mi][ni][0] = 0.0; d[mi][ni][1] = 0.0; }
#pragma unroll
                        for (int kk = 0; kk < KS; kk++) {
                            double a[MT];
#pragma unroll
                            for (int mi = 0; mi < MT; mi++)
                                a[mi] = (mi > (4 * kk) / 8) ? sm.S[(4 * kk + fc) * LDS_ + 8 * mi + fr] : sm.S[(8 * mi + fr) * LDS_ + 4 * kk + fc];
#pragma unroll
                            for (int mi = 0; mi < MT; mi++)
#pragma unroll
                                for (int ni = 0; ni < NT; ni++) dmma(d[mi][ni][0], d[mi][ni][1], a[mi], bfr[kk][ni]);
                        }
#pragma unroll
                        for (int kr = 0; kr < KR; kr++) {
                            const int kx = 4 * KS + kr;
                            double a[MT]; double2 bb[NT];
#pragma unroll
                            for (int mi = 0; mi < MT; mi++)
                                a[mi] = (mi > kx / 8) ? sm.S[kx * LDS_ + 8 * mi + fr] : sm.S[(8 * mi + fr) * LDS_ + kx];
#pragma unroll
                            for (int ni = 0; ni < NT; ni++) bb[ni] = lds128(&sAB[kx * LDABS + 8 * ni + 2 * fc]);
#pragma unroll
                            for (int mi = 0; mi < MT; mi++)
#pragma unroll
                                for (int ni = 0; ni < NT; ni++) { d[mi][ni][0] = fma(a[mi], bb[ni].x, d[mi][ni][0]); d[mi][ni][1] = fma(a[mi], bb[ni].y, d[mi][ni][1]); }
                        }
#pragma unroll
                        for (int mi = 0; mi < MT; mi++)
#pragma unroll
                            for (int ni = 0; ni < NT; ni++) {
                                const int row = 8 * mi + fr, col = 8 * ni + 2 * fc;
                                if (col + 1 < NM) sts128(&sm.T[row * LDT + col], d[mi][ni][0], d[mi][ni][1]);
                                else if (col < NM) sm.T[row * LDT + col] = d[mi][ni][0];      // column NM is reserved for s
                            }
                        if (lane < n) sm.T[lane * LDT + NM] = s_reg;
                    }
                    __syncwarp();
                    // ---- [Qzz | Qz] = [A B]' [T | s] : upper tiles (mi <= ni); tiles with mi,ni < MT become the S accumulators ----
                    double q[NQT][2];
#pragma unroll
                    for (int t = 0; t < NQT; t++) { q[t][0] = 0.0; q[t][1] = 0.0; }
#pragma unroll
                    for (int kk = 0; kk < KS; kk++) {
                        double bf[NT];
#pragma unroll
                        for (int ni = 0; ni < NT; ni++) bf[ni] = sm.T[(4 * kk + fc) * LDT + 8 * ni + fr];
                        int t = 0;
#pragma unroll
                        for (int mi = 0; mi < MQ; mi++)
#pragma unroll
                            for (int ni = mi; ni < NT; ni++, t++) dmma(q[t][0], q[t][1], bfr[kk][mi], bf[ni]);
                    }
#pragma unroll
                    for (int kr = 0; kr < KR; kr++) {
                        const int kx = 4 * KS + kr;
                        double a[MQ]; double2 bb[NT];
#pragma unroll
                        for (int mi = 0; mi < MQ; mi++) a[mi] = sAB[kx * LDABS + 8 * mi + fr];
#pragma unroll
                        for (int ni = 0; ni < NT; ni++) bb[ni] = lds128(&sm.T[kx * LDT + 8 * ni + 2 * fc]);
                        int t = 0;
#pragma unroll
                        for (int mi = 0; mi < MQ; mi++)
#pragma unroll
                            for (int ni = mi; ni < NT; ni++, t++) { q[t][0] = fma(a[mi], bb[ni].x, q[t][0]); q[t][1] = fma(a[mi], bb[ni].y, q[t][1]); }
                    }
                    __syncwarp();     // every lane has read T: the Qz strip below overwrites it (racecheck flags the write-after-read without it)
                    // ---- + [lzz | lz] (lane-resident, fetched by shuffle) ; the u / Qz strip (columns >= n) goes to shared memory ----
                    {
                        double hrow[MQ], grow[MQ];
#pragma unroll
                        for (int mi = 0; mi < MQ; mi++) { hrow[mi] = __shfl_sync(0xffffffffu, h_reg, (8 * mi + fr) & 31); grow[mi] = __shfl_sync(0xffffffffu, g_reg, (8 * mi + fr) & 31); }
                        int t = 0;
#pragma unroll
                        for (int mi = 0; mi < MQ; mi++)
#pragma unroll
                            for (int ni = mi; ni < NT; ni++, t++) {
                                const int row = 8 * mi + fr, col = 8 * ni + 2 * fc;
                                if (row == col) q[t][0] += hrow[mi];
                                if (row == col + 1) q[t][1] += hrow[mi];
                                if (col == NM) q[t][0] += grow[mi];
                                if (col + 1 == NM) q[t][1] += grow[mi];
                                if (row < NM) {
                                    if (col >= n && col <= NM) Qs_[row * LDQS + col - n] = q[t][0];
                                    if (col + 1 >= n && col + 1 <= NM) Qs_[row * LDQS + col + 1 - n] = q[t][1];
                                }
                            }
                    }
                    __syncwarp();
                    if (k - STAGES >= 0) issue_ab(stage, k - STAGES);     // T and the ring slot have been consumed
                    stage = (stage + 1 == STAGES) ? 0 : stage + 1;
                    // ---- gains: LDL' of Quu + rho I, one lane per column of [Qux | Qu]; lanes 0..15 only (half the wavefronts) ----
                    double kc[M_], wc[M_];
#pragma unroll
                    for (int a = 0; a < m; a++) { kc[a] = 0.0; wc[a] = 0.0; }
                    bool okl = true;
                    if (lane < 16) {   // half a warp: FP64 instructions of a half-empty warp take one pipe pass instead of two
                        double Quu[M_ * (M_ + 1) / 2], Lf[M_ * (M_ + 1) / 2], dj[M_];
#pragma unroll
                        for (int a = 0; a < m; a++)
#pragma unroll
                            for (int c = 0; c <= a; c++) Quu[a * (a + 1) / 2 + c] = Qs_[(n + c) * LDQS + a];
#pragma unroll
                        for (int j = 0; j < m; j++) {
                            double t = Quu[j * (j + 1) / 2 + j] + rho;
#pragma unroll
                            for (int r = 0; r < j; r++) t = fma(-Lf[j * (j + 1) / 2 + r] * Lf[j * (j + 1) / 2 + r], dj[r], t);
                            if (!(t > 0.0) || !isfinite(t)) okl = false;
                            dj[j] = t;
                            const double inv = rcp_pivot(t);
                            Lf[j * (j + 1) / 2 + j] = inv;
#pragma unroll
                            for (int i = j + 1; i < m; i++) {
                                double v = Quu[i * (i + 1) / 2 + j];
#pragma unroll
                                for (int r = 0; r < j; r++) v = fma(-Lf[i * (i + 1) / 2 + r] * Lf[j * (j + 1) / 2 + r], dj[r], v);
                                Lf[i * (i + 1) / 2 + j] = v * inv;
                            }
                        }
                        const int c = (lane <= n) ? lane : n;
                        double rhs[M_];
#pragma unroll
                        for (int a = 0; a < m; a++) rhs[a] = (c < n) ? Qs_[c * LDQS + a] : Qs_[(n + a) * LDQS + m];   // Qux[a][c] | Qu[a]
#pragma unroll
                        for (int a = 0; a < m; a++) {
                            double t = -rhs[a];
#pragma unroll
                            for (int r = 0; r < a; r++) t = fma(-Lf[a * (a + 1) / 2 + r], kc[r], t);
                            kc[a] = t;
                        }
#pragma unroll
                        for (int a = 0; a < m; a++) kc[a] *= Lf[a * (a + 1) / 2 + a];
#pragma unroll
                        for (int a = m - 1; a >= 0; a--) {
                            double t = kc[a];
#pragma unroll
                            for (int r = a + 1; r < m; r++) t = fma(-Lf[r * (r + 1) / 2 + a], kc[r], t);
                            kc[a] = t;
                        }
#pragma unroll
                        for (int a = 0; a < m; a++) wc[a] = fma(-rho, kc[a], rhs[a]);   // W = Qux - rho K
                        if (okl) {
                            if (lane <= n) {
#pragma unroll
                                for (int a = 0; a < m; a++) { K_[a * LDK + c] = kc[a]; W_[a * LDK + c] = wc[a]; }
                            }
                            if (lane < n) {
#pragma unroll
                                for (int a = 0; a < m; a++) Kg[(size_t)k * n * m + lane * m + a] = kc[a];
                            } else if (lane == n) {
                                double t1 = 0.0, t2 = 0.0;
#pragma unroll
                                for (int a = 0; a < m; a++) {
                                    dg[(size_t)k * m + a] = kc[a];
                                    t1 = fma(kc[a], rhs[a], t1);
                                    double qd = 0.0;
#pragma unroll
                                    for (int r = 0; r < m; r++) qd = fma((r <= a) ? Quu[a * (a + 1) / 2 + r] : Quu[r * (r + 1) / 2 + a], kc[r], qd);
                                    t2 = fma(0.5 * kc[a], qd, t2);
                                }
                                dV1 += t1; dV2 += t2;
                            }
                        }
                    }
                    ok = __shfl_sync(0xffffffffu, okl ? 1 : 0, 0) != 0;
                    if (!ok) break;
                    __syncwarp();
                    // ---- S <- Qxx + W'K on the tensor cores (one k-step, K = m <= 4), accumulators = the Qxx tiles ----
                    {
                        double af[MT], bk[MT];
#pragma unroll
                        for (int mi = 0; mi < MT; mi++) { af[mi] = (fc < m) ? W_[fc * LDK + 8 * mi + fr] : 0.0; bk[mi] = (fc < m) ? K_[fc * LDK + 8 * mi + fr] : 0.0; }
                        int t = 0;
#pragma unroll
                        for (int mi = 0; mi < MQ; mi++)
#pragma unroll
                            for (int ni = mi; ni < NT; ni++, t++) {
                                if (mi < MT && ni < MT) {
                                    dmma(q[t][0], q[t][1], af[mi], bk[ni]);
                                    sts128(&sm.S[(8 * mi + fr) * LDS_ + 8 * ni + 2 * fc], q[t][0], q[t][1]);
                                }
                            }
                        // s <- Qx + W'd : W column of lane c is in its registers, d comes from lane n
                        double snew = (lane < n) ? Qs_[lane * LDQS + m] : 0.0;
#pragma unroll
                        for (int a = 0; a < m; a++) snew = fma(wc[a], __shfl_sync(0xffffffffu, kc[a], n), snew);
                        s_reg = snew;
                    }
                } else {
                        // ---- T = S [A B]  (2x2 blocks), extra column NM <- s ---------------------------------------
                        {
                            double acc[RT][4];
        #pragma unroll
                            for (int r = 0; r < RT; r++) { acc[r][0] = acc[r][1] = acc[r][2] = acc[r][3] = 0.0; }
        #pragma unroll
                            for (int j = 0; j < n; j++) {
        #pragma unroll
                                for (int r = 0; r < RT; r++) {
                                    const double2 a = lds128(&sm.S[j * LDS_ + t_a[r]]);
                                    const double2 bb = lds128(&sAB[j * LDABS + t_b[r]]);
                                    fma2x2(acc[r], a, bb);
                                }
                            }
        #pragma unroll
                            for (int r = 0; r < RT; r++) {
                                if (t_on[r]) {
                                    if (t_lastcol[r]) { sm.T[t_o[r]] = acc[r][0]; sm.T[t_o[r] + LDT] = acc[r][2]; }   // leave column NM to s
                                    else { sts128(&sm.T[t_o[r]], acc[r][0], acc[r][1]); sts128(&sm.T[t_o[r] + LDT], acc[r][2], acc[r][3]); }
                                }
                            }
                            if (lane < n) sm.T[lane * LDT + NM] = s_reg;
                        }
                        __syncwarp();

                        // ---- [Qzz | Qz] = [A B]' [T | s] + [lzz | lz]  (upper 2x2 blocks) -----------------------
                        {
                            double acc[RQ][4];
        #pragma unroll
                            for (int r = 0; r < RQ; r++) { acc[r][0] = acc[r][1] = acc[r][2] = acc[r][3] = 0.0; }
        #pragma unroll
                            for (int j = 0; j < n; j++) {
        #pragma unroll
                                for (int r = 0; r < RQ; r++) {
                                    const double2 a = lds128(&sAB[j * LDABS + q_a[r]]);
                                    const double2 bb = lds128(&sm.T[j * LDT + q_b[r]]);
                                    fma2x2(acc[r], a, bb);
                                }
                            }
        #pragma unroll
                            for (int r = 0; r < RQ; r++) {
                                const int i0 = q_i0[r], j0 = q_j0[r];
                                const double2 gg = lds128(&sm.g[i0]);
                                if (q_diag[r]) { const double2 hh = lds128(&sm.h[i0]); acc[r][0] += hh.x; acc[r][3] += hh.y; }
                                if (j0 == NM) { acc[r][0] += gg.x; acc[r][2] += gg.y; }
                                if (j0 + 1 == NM) { acc[r][1] += gg.x; acc[r][3] += gg.y; }
                                if (q_on[r]) {
                                    sts128(&sm.Q[q_o[r]], acc[r][0], acc[r][1]);
                                    sts128(&sm.Q[q_o[r] + LDT], acc[r][2], acc[r][3]);
                                }
                            }
                        }
                        __syncwarp();
                    // the stage buffer is free: refill it with the knot STAGES steps ahead
                    if (k - STAGES >= 0) issue_ab(stage, k - STAGES);
                    stage = (stage + 1 == STAGES) ? 0 : stage + 1;

                    // dense cost Hessian (QuadraticCost): add the off-diagonal entries of lzz to the upper part of Q
                    if (!P.all_diag_cost) {
                        const DevCost& cost = P.costs[P.cost_index[k]];
                        if (!cost.diag) {
                            for (int e = lane; e < NM * NM; e += 32) {
                                const int i = e / NM, j = e % NM;     // need (i,j) with block(i) <= block(j)
                                if (i == j || (i >> 1) > (j >> 1)) continue;
                                double v;
                                if (i < n && j < n) v = cost.Q[j * n + i];
                                else if (i >= n && j >= n) v = cost.R[(j - n) * m + (i - n)];
                                else if (i < n) v = cost.zeroH ? 0.0 : cost.H[i * m + (j - n)];   // (x_i, u_a): H[a][i]
                                else v = cost.zeroH ? 0.0 : cost.H[j * m + (i - n)];
                                sm.Q[i * LDT + j] += v;
                            }
                            // diagonal: sm.h carried only the AL part for dense costs -> add Q_ii / R_aa
                            if (lane < NM) sm.Q[lane * LDT + lane] += (lane < n) ? cost.Q[lane * n + lane] : cost.R[(lane - n) * m + (lane - n)];
                            __syncwarp();
                        }
                    }

                    if (!P.all_diag_con) { double dummy = 0.0; general_constraints(k + 1, false, dummy); }

                    // ---- gains: LDL' of Quu + rho I, one lane per column of [Qux | Qu] -------------------------
                    double Quu[M_ * (M_ + 1) / 2];           // packed lower by rows
                    double Lf[M_ * (M_ + 1) / 2];            // unit-lower L (off-diagonal), diagonal slots hold 1/d_j
                    {
    #pragma unroll
                        for (int a = 0; a < m; a++)
    #pragma unroll
                            for (int c = 0; c <= a; c++) Quu[a * (a + 1) / 2 + c] = sm.Q[(n + c) * LDT + (n + a)];   // upper entry (c <= a)
                        double dj[M_];
    #pragma unroll
                        for (int j = 0; j < m; j++) {
                            double t = Quu[j * (j + 1) / 2 + j] + rho;
    #pragma unroll
                            for (int r = 0; r < j; r++) t = fma(-Lf[j * (j + 1) / 2 + r] * Lf[j * (j + 1) / 2 + r], dj[r], t);
                            if (!(t > 0.0) || !isfinite(t)) ok = false;
                            dj[j] = t;
                            const double inv = rcp_pivot(t);
                            Lf[j * (j + 1) / 2 + j] = inv;
    #pragma unroll
                            for (int i = j + 1; i < m; i++) {
                                double v = Quu[i * (i + 1) / 2 + j];
    #pragma unroll
                                for (int r = 0; r < j; r++) v = fma(-Lf[i * (i + 1) / 2 + r] * Lf[j * (j + 1) / 2 + r], dj[r], v);
                                Lf[i * (i + 1) / 2 + j] = v * inv;
                            }
                        }
                    }
                    if (!ok) break;   // uniform across the warp (every lane factors the same matrix)
                    {
                        const int c = (lane <= n) ? lane : n;
                        double rhs[M_], kc[M_];
    #pragma unroll
                        for (int a = 0; a < m; a++) rhs[a] = (c < n) ? sm.Q[c * LDT + (n + a)] : sm.Q[(n + a) * LDT + NM];   // Qux[a][c] | Qu[a]
    #pragma unroll
                        for (int a = 0; a < m; a++) {      // forward: L y = -rhs
                            double t = -rhs[a];
    #pragma unroll
                            for (int r = 0; r < a; r++) t = fma(-Lf[a * (a + 1) / 2 + r], kc[r], t);
                            kc[a] = t;
                        }
    #pragma unroll
                        for (int a = 0; a < m; a++) kc[a] *= Lf[a * (a + 1) / 2 + a];   // D^-1
    #pragma unroll
                        for (int a = m - 1; a >= 0; a--) {  // backward: L' x = y
                            double t = kc[a];
    #pragma unroll
                            for (int r = a + 1; r < m; r++) t = fma(-Lf[r * (r + 1) / 2 + a], kc[r], t);
                            kc[a] = t;
                        }
                        if (lane <= n) {
    #pragma unroll
                            for (int a = 0; a < m; a++) {
                                K_[a * LDK + c] = kc[a];
                                W_[a * LDK + c] = fma(-rho, kc[a], rhs[a]);   // W = Qux - rho K
                            }
                        }
                        if (lane < n) {
    #pragma unroll
                            for (int a = 0; a < m; a++) Kg[(size_t)k * n * m + lane * m + a] = kc[a];
                        } else if (lane == n) {
                            double t1 = 0.0, t2 = 0.0;
    #pragma unroll
                            for (int a = 0; a < m; a++) {
                                dg[(size_t)k * m + a] = kc[a];
                                t1 = fma(kc[a], rhs[a], t1);
                                double qd = 0.0;   // (Quu d)_a
    #pragma unroll
                                for (int r = 0; r < m; r++) qd = fma((r <= a) ? Quu[a * (a + 1) / 2 + r] : Quu[r * (r + 1) / 2 + a], kc[r], qd);
                                t2 = fma(0.5 * kc[a], qd, t2);
                            }
                            dV1 += t1; dV2 += t2;
                        }
                    }
                    __syncwarp();

                    // ---- S <- Qxx + W'K (upper blocks, mirrored) ; s <- Qx + W'd ------------------------------
                    {
                        double acc[RS][4];
    #pragma unroll
                        for (int r = 0; r < RS; r++) {
                            const double2 q0 = lds128(&sm.Q[s_a[r] * LDT + s_b[r]]);
                            const double2 q1 = lds128(&sm.Q[(s_a[r] + 1) * LDT + s_b[r]]);
                            acc[r][0] = q0.x; acc[r][1] = q0.y; acc[r][2] = q1.x; acc[r][3] = q1.y;
                        }
    #pragma unroll
                        for (int a = 0; a < m; a++) {
    #pragma unroll
                            for (int r = 0; r < RS; r++) {
                                const double2 w = lds128(&W_[a * LDK + s_a[r]]);
                                const double2 kk = lds128(&K_[a * LDK + s_b[r]]);
                                fma2x2(acc[r], w, kk);
                            }
                        }
                        double snew = 0.0;
                        if (lane < n) {
                            snew = sm.Q[lane * LDT + NM];
    #pragma unroll
                            for (int a = 0; a < m; a++) snew = fma(W_[a * LDK + lane], K_[a * LDK + n], snew);
                        }
                        s_reg = snew;
    #pragma unroll
                        for (int r = 0; r < RS; r++) {
                            if (!s_on[r]) continue;
                            const int i0 = s_a[r], j0 = s_b[r];
                            if (s_diag[r]) {
                                const double off = 0.5 * (acc[r][1] + acc[r][2]);
                                sts128(&sm.S[i0 * LDS_ + j0], acc[r][0], off);
                                sts128(&sm.S[(i0 + 1) * LDS_ + j0], off, acc[r][3]);
                            } else {
                                sts128(&sm.S[i0 * LDS_ + j0], acc[r][0], acc[r][1]);
                                sts128(&sm.S[(i0 + 1) * LDS_ + j0], acc[r][2], acc[r][3]);
                                sts128(&sm.S[j0 * LDS_ + i0], acc[r][0], acc[r][2]);
                                sts128(&sm.S[(j0 + 1) * LDS_ + i0], acc[r][1], acc[r][3]);
                            }
                        }
                    }
                }
                z_cur = z_nxt; act_cur = act_nxt; cH_cur = cH_nxt; cG_cur = cG_nxt; cid_next = cid_next2;
#pragma unroll
                for (int t = 0; t < MAXT; t++) lam_cur[t] = lam_nxt[t];
                __syncwarp();
            }   // knots

            if (ok) {
                if (lane == n) { P.dV[2 * b] = dV1; P.dV[2 * b + 1] = dV2; }
                break;
            }
            // ---- non-PD Quu at knot k: drain the copies still in flight (knots k-1 .. k-STAGES, already
            //      re-armed), increase rho (Altro regularization_update!(:increase)) and restart ------------
            {
                const int outstanding = (k < STAGES) ? k : STAGES;
                for (int i = 0; i < outstanding; i++) {
                    const int st = (stage + i) % STAGES;
                    mbar_wait(&sm.bar[st], (phase_bits >> st) & 1u);
                    phase_bits ^= (1u << st);
                }
            }
            __syncwarp();
            reg_increase(P.opt, rho, drho);
            restarts++;
            if (rho > P.opt.bp_reg_max) { failed = true; break; }
        }
        if (!failed) reg_decrease(P.opt, rho, drho);
        if (lane == 0) {
            P.rho[b] = rho; P.drho[b] = drho;
            P.bp_status[b] = failed ? -1 : restarts;
        }
        __syncwarp();
    }
}

template <int N_, int M_, bool FASTAL, int STAGES, int MINB, bool MMA, int NSLOT, bool INST>
cudaError_t launch_riccati_v(const DevProblem& P, int* work_counter, cudaStream_t s) {
    using SM = RiccatiSmem<N_, M_, STAGES, MMA>;
    auto kern = k_riccati<N_, M_, STAGES, FASTAL, MMA, MINB, NSLOT, INST>;
    static int ctas_cfg[TO_MAXDEV] = {0}, sms_cfg[TO_MAXDEV] = {0};      // per device (0 = not configured yet)
    const int smem = (int)sizeof(SM);
    const int dev = current_device_slot();
    if (!ctas_cfg[dev]) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e != cudaSuccess) return e;
        cudaDeviceGetAttribute(&sms_cfg[dev], cudaDevAttrMultiProcessorCount, dev);
        int c = 1;
        e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&c, kern, 32, smem);
        if (e != cudaSuccess) return e;
        ctas_cfg[dev] = c < 1 ? 1 : c;
    }
    const int ctas_per_sm = ctas_cfg[dev], num_sms = sms_cfg[dev];
    cudaError_t e = cudaMemsetAsync(work_counter, 0, sizeof(int), s);
    if (e != cudaSuccess) return e;
    int grid = num_sms * ctas_per_sm;     // persistent: a multiple of the SM count, instances pulled from a queue
    if (grid > P.B) grid = P.B;
    kern<<<grid, 32, smem, s>>>(P, work_counter);
    return cudaGetLastError();
}

// INST: per-instance linear cost terms (P.qr) and constraint data (P.cdata), a kernel variant of its own so that the shared one stays as it is
template <int N_, int M_, bool FASTAL, bool INST>
cudaError_t launch_riccati_t(const DevProblem& P, int* work_counter, cudaStream_t s) {
    if constexpr (N_ >= 8 && M_ <= 4) {
        if (backward_kernel_of(P) == KC_BK_WARP_MMA) {   // tensor-MMA kernel: diagonal lzz (DiagonalCost + Goal/Bound)
            // 2-stage ring, 16 one-warp CTAs per SM.  NSLOT stays MAXT (the loop bound of the slot loop).
            return launch_riccati_v<N_, M_, FASTAL, TO_RICCATI_STAGES, TO_RICCATI_MINB, true, MAXT, INST>(P, work_counter, s);
        }
        return launch_riccati_v<N_, M_, FASTAL, 2, 12, false, MAXT, INST>(P, work_counter, s);   // dense costs: DFMA micro-block kernel
    } else {
        return launch_riccati_v<N_, M_, FASTAL, 3, 16, false, MAXT, INST>(P, work_counter, s);
    }
}

template <int N_, int M_>
cudaError_t launch_riccati_nm(const DevProblem& P, int* work_counter, cudaStream_t s) {
    const bool fastal = riccati_fastal(P);
    if (inst_backward(P)) return fastal ? launch_riccati_t<N_, M_, true, true>(P, work_counter, s) : launch_riccati_t<N_, M_, false, true>(P, work_counter, s);
    return fastal ? launch_riccati_t<N_, M_, true, false>(P, work_counter, s) : launch_riccati_t<N_, M_, false, false>(P, work_counter, s);
}

}  // namespace

// the lane-resident AL terms hold at most MAXT rows per z entry (upper + lower bound + goal); knot and row indices are packed in bit fields
bool riccati_fastal(const DevProblem& P) { return P.max_terms_per_z <= MAXT && P.N < 4095 && P.max_p_knot < 128; }

int backward_kernel_of(const DevProblem& P) {
    // lie.cu: error state / quaternion costs (expansion materialised by the caller)
    if (P.dense_riccati) return dense_backward_mma(P) ? KC_BK_DENSE_MMA : KC_BK_DENSE_DFMA;
    // small models: one thread per instance, everything in registers (riccati_small.cu); backward_kernel = 1 forces the warp kernel
    const int choice = P.opt.pad;   // to_options.backward_kernel: 0 automatic, 1 warp kernel, 2 thread kernel where it applies
    if ((choice == 2 && riccati_small_supported(P, true)) || (choice == 0 && riccati_small_supported(P, false))) return KC_BK_THREAD;
    // tensor-MMA k_riccati (n >= 8): diagonal lzz (DiagonalCost + Goal/Bound); otherwise the DFMA micro-block kernel
    return (P.n >= 8 && P.m <= 4 && P.all_diag_cost && P.all_diag_con) ? KC_BK_WARP_MMA : KC_BK_WARP_DFMA;
}

cudaError_t launch_backward(const DevProblem& P, int* work_counter, cudaStream_t s) {
    if (P.dense_riccati) return launch_backward_dense(P, s);
    if (backward_kernel_of(P) == KC_BK_THREAD) return launch_backward_small(P, s);
    if (P.n == 13 && P.m == 4) return launch_riccati_nm<13, 4>(P, work_counter, s);
    if (P.n == 4 && P.m == 1) return launch_riccati_nm<4, 1>(P, work_counter, s);
    if (P.n == 4 && P.m == 2) return launch_riccati_nm<4, 2>(P, work_counter, s);
    if (P.n == 2 && P.m == 1) return launch_riccati_nm<2, 1>(P, work_counter, s);
    return cudaErrorNotSupported;
}
