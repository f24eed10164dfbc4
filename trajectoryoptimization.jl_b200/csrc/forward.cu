#include <cstdlib>
#include <type_traits>
// forward.cu -- the forward pass of iLQR: closed-loop rollout fused with the cost + constraint + AL-penalty
// sweep (kernel 1 without partials + kernel 2), and the per-instance backtracking line search.
//
// What it computes (Altro.jl forwardpass! / rollout!(solver, alpha), restated in oracle/oracle.hpp
// `forward_rollout` / `forward_pass`; it drives the reference's rollout (src/problem.jl:334-340), cost
// (src/objective.jl:89-106) and constraint evaluation (src/abstract_constraint.jl:200-225)):
//     dx = xbar_k - x_k ; ubar_k = u_k + K_k dx + alpha d_k ; xbar_{k+1} = step(xbar_k, ubar_k)  (the problem's explicit rule, models.cuh)
//     J(alpha) = sum_k l_k(xbar_k, ubar_k) + AL penalty ;  z = (J_prev - J) / -(alpha (dV1 + alpha dV2))
//     accept the first alpha in 1, 1/2, ..., 2^-ls_iters with  lower < z <= upper  or  J < J_prev.
// The line search is per instance (no communication, SURVEY.md 8e).
//
// Mapping.  The recursion is serial in k and one rollout has no parallelism worth a warp, so the kernel is
// bound by the LATENCY of the per-knot dependency chain (feedback -> 1 to 4 dynamics evaluations, by rule -> next knot).  Two
// things follow:
//   * backtracking trials are evaluated CONCURRENTLY: a group of G lanes owns one instance and lane j rolls out
//     step size 2^-(trial0+j), writing its candidate into trajectory buffer (cur+1+j) % NBUF.  A ballot picks the
//     first acceptable lane -- exactly the sequential backtracking result -- and acceptance only moves cur[b]
//     (no copy).  Pass 1 (G=4: alpha = 1..1/8) covers ~95% of the instances, pass 2 (G=8) the remaining trials and
//     commits failures (regularisation increase, Altro's bp_reg_fp).
//   * everything off the chain is kept off it: the group's per-knot operands (K_k, d_k, x_k, u_k, lambda_k, ~650 B,
//     identical for all lanes of the group) are prefetched one knot ahead with cp.async (LDGSTS) by the lanes
//     cooperatively into a double-buffered shared-memory stage and read back as broadcasts; cost / constraint
//     descriptors are copied once per CTA into shared memory; x, u live in registers; no fp64 division on the chain.
#include "costcon.cuh"
#include "kernels.h"
#include "models.cuh"
#include "ptx.cuh"

// The explicit rule this object instantiates the line search for (rollout.cu explains the one object per rule); the object of rule 4 (RK4)
// also holds the host functions that do not depend on it and the launchers that dispatch on DevProblem::integration.
#ifndef TO_RULE
#define TO_RULE 4
#endif

namespace {

constexpr int FWD_MAX_COST = 4;    // cost functions cached in shared memory (more -> read from global)
constexpr int FWD_MAX_N = 512;
constexpr int FWD_THREADS = 32;

struct FwdCon {
    int kind, first, last, p, offset;
    unsigned mask_max, mask_min;     // bit j set: z_j has a finite upper / lower bound (Goal: x_j constrained)
    int ubox;                        // Bound with both bounds finite on every control and none on the state: rows are static
    double mu, inv2mu;
    int row_max[TO_MAXNM], row_min[TO_MAXNM];
    double a[TO_MAXNM], b[TO_MAXNM];
};
// the data view (common.cuh con_data) of a staged constraint: its Goal values / Bound limits in shared memory
__device__ __forceinline__ ConData staged(const FwdCon& c) { return ConData{c.a, c.b}; }
struct FwdCost {
    double Qd[TO_MAXN], Rd[TO_MAXM], q[TO_MAXN], r[TO_MAXM], c;
};
// the cost view (common.cuh cost_data) of a cached cost: its diagonal weights, linear terms and c in shared memory
__device__ __forceinline__ CostData staged(const FwdCost& c) { return CostData{c.Qd, c.Rd, nullptr, nullptr, nullptr, c.q, c.r, &c.c, nullptr}; }
struct alignas(16) FwdTab {
    int ncon, ncost_cached, pad0, pad1;
    FwdCon con[TO_MAXCON];
    FwdCost cost[FWD_MAX_COST];
    double dt[FWD_MAX_N];
    int cost_index[FWD_MAX_N];
    int lam_off[FWD_MAX_N][2];       // multipliers to stage for knot k: up to two (offset, count) segments of lambda_b
    int lam_cnt[FWD_MAX_N][2];
};

__device__ inline void load_tables(const DevProblem& P, FwdTab& tab) {
    const int t = threadIdx.x, T = blockDim.x;
    if (t == 0) { tab.ncon = P.ncon; tab.ncost_cached = P.ncost <= FWD_MAX_COST ? P.ncost : 0; }
    for (int ci = 0; ci < P.ncon; ci++) {
        const DevCon& c = P.cons[ci];
        FwdCon& f = tab.con[ci];
        if (t == 0) {
            f.kind = c.kind; f.first = c.first; f.last = c.last; f.p = c.p; f.offset = c.offset;
            f.mu = penalty<false>(P, 0, ci); f.inv2mu = 1.0 / (2.0 * penalty<false>(P, 0, ci));   // the shared penalty (INST: rollout_fast reads each instance's)
            unsigned mx = 0, mn = 0;
            for (int j = 0; j < TO_MAXNM; j++) { if (c.row_max[j] >= 0) mx |= 1u << j; if (c.row_min[j] >= 0) mn |= 1u << j; }
            f.mask_max = mx; f.mask_min = mn;
            const unsigned ubits = ((1u << P.m) - 1u) << P.n;
            f.ubox = (c.kind == CON_BOUND && mx == ubits && mn == ubits) ? 1 : 0;
        }
        for (int j = t; j < TO_MAXNM; j += T) {
            f.row_max[j] = c.row_max[j]; f.row_min[j] = c.row_min[j];
            f.a[j] = c.a[j]; f.b[j] = c.b[j];
        }
    }
    if (P.ncost <= FWD_MAX_COST)
        for (int ci = 0; ci < P.ncost; ci++) {
            const DevCost& c = P.costs[ci];
            FwdCost& f = tab.cost[ci];
            for (int j = t; j < TO_MAXN; j += T) { f.Qd[j] = c.Qd[j]; f.q[j] = c.q[j]; }
            for (int j = t; j < TO_MAXM; j += T) { f.Rd[j] = c.Rd[j]; f.r[j] = c.r[j]; }
            if (t == 0) f.c = c.c;
        }
    for (int k = t; k < P.N && k < FWD_MAX_N; k += T) {
        tab.dt[k] = (k < P.N - 1) ? P.dt[k] : 0.0; tab.cost_index[k] = P.cost_index[k];
        int ns = 0;
        tab.lam_cnt[k][0] = tab.lam_cnt[k][1] = 0; tab.lam_off[k][0] = tab.lam_off[k][1] = 0;
        for (int ci = 0; ci < P.ncon; ci++) {
            const DevCon& c = P.cons[ci];
            if (k + 1 < c.first || k + 1 > c.last) continue;
            if (ns < 2) { tab.lam_off[k][ns] = c.offset + (k + 1 - c.first) * c.p; tab.lam_cnt[k][ns] = c.p; }
            ns++;
        }
    }
    __syncthreads();
}

// The compact problem class (DevProblem::fwd_compact): the stage cost, the control box and the terminal Goal, laid out for the
// straight-line knot loop of rollout_compact.  {coefficient, linear term} pairs are read with one 16-byte load each.
struct alignas(16) FwdCompactTab {
    double2 sx[TO_MAXN];             // stage cost {Qd_i, q_i}
    double2 su[TO_MAXM];             // stage cost {Rd_i, r_i}
    double2 box[TO_MAXM];            // control box {u_max_i, u_min_i}
    double sc, mu, inv2mu, pad0;     // stage cost c; the box's penalty
    int cid, tcid, box_off, box_p;   // stage / terminal cost; the box's multipliers of knot 1 and rows per knot (0: no box)
    int goal_ci, goal_off, goal_p, pad1;   // the Goal (-1: none) and its multipliers
    FwdCost term;                    // terminal cost (Qd, q, c)
    FwdCon goal;                     // the Goal's mu, inv2mu, mask_max, row_max, a
    double dt[FWD_MAX_N];
};
// The per-instance variant's copy of an instance's two costs in the fields of FwdCompactTab, staged for each group by linesearch_pass
struct alignas(16) FwdCompactCost {
    double2 sx[TO_MAXN], su[TO_MAXM];
    double sc, pad;
    FwdCost term;
    double mu, inv2mu, gmu, ginv2mu;     // the instance's penalties of the box and of the Goal, and 1 / (2 mu), as load_compact_tables forms them
};

__device__ inline void load_compact_tables(const DevProblem& P, FwdCompactTab& tab) {
    const int t = threadIdx.x, T = blockDim.x;
    const int cid = P.cost_index[0], tcid = P.cost_index[P.N - 1];
    const DevCost& c = P.costs[cid];
    const DevCost& ct = P.costs[tcid];
    for (int j = t; j < TO_MAXN; j += T) { tab.sx[j] = make_double2(c.Qd[j], c.q[j]); tab.term.Qd[j] = ct.Qd[j]; tab.term.q[j] = ct.q[j]; }
    for (int j = t; j < TO_MAXM; j += T) tab.su[j] = make_double2(c.Rd[j], c.r[j]);
    if (t == 0) {
        tab.sc = c.c; tab.term.c = ct.c; tab.cid = cid; tab.tcid = tcid;
        tab.box_off = tab.box_p = 0; tab.goal_ci = -1; tab.goal_off = tab.goal_p = 0;
    }
    for (int ci = 0; ci < P.ncon; ci++) {
        const DevCon& k = P.cons[ci];
        if (k.kind == CON_BOUND) {   // knots 1..N-1, rows 0..m-1 = upper, m..2m-1 = lower
            for (int j = t; j < P.m; j += T) tab.box[j] = make_double2(k.a[P.n + j], k.b[P.n + j]);
            if (t == 0) { tab.box_off = k.offset; tab.box_p = k.p; tab.mu = penalty<false>(P, 0, ci); tab.inv2mu = 1.0 / (2.0 * penalty<false>(P, 0, ci)); }
        } else {                     // the Goal, knot N
            FwdCon& f = tab.goal;
            if (t == 0) {
                tab.goal_ci = ci; tab.goal_off = k.offset; tab.goal_p = k.p;
                f.mu = penalty<false>(P, 0, ci); f.inv2mu = 1.0 / (2.0 * penalty<false>(P, 0, ci));
                unsigned mx = 0;
                for (int j = 0; j < TO_MAXNM; j++) if (k.row_max[j] >= 0) mx |= 1u << j;
                f.mask_max = mx;
            }
            for (int j = t; j < TO_MAXNM; j += T) { f.row_max[j] = k.row_max[j]; f.a[j] = k.a[j]; }
        }
    }
    for (int k = t; k < P.N - 1; k += T) tab.dt[k] = P.dt[k];
    __syncthreads();
}

// Depth of the operand ring of the closed-loop rollout: knot k + FWD_STAGES - 1 is in flight while knot k is consumed.  One knot ahead
// (2 stages) is the default; deeper rings cost registers and shared memory (TO_FWD_STAGES at build time).
#ifndef TO_FWD_STAGES
#define TO_FWD_STAGES 2
#endif
constexpr int FWD_STAGES = TO_FWD_STAGES;
// knots of candidate trajectory staged in shared memory per lane before the group writes them out (rollout_compact)
constexpr int FWD_OKNOTS = 4;

// shared-memory stage of one knot's operands for the IPB instances of a CTA.
// K_k is stored as 16-byte pairs [pair][IPB][2] (when n*m is even), everything else as 8-byte slots [slot][IPB].
template <int n, int m, int IPB, int NE = n>
struct Stage {
    static constexpr int KSLOTS = NE * m;     // K_k is m x NE (NE = n - 1 on the Lie-group error state)
    static constexpr bool K16 = (KSLOTS % 2) == 0;
    static constexpr int OFF_D = KSLOTS, OFF_U = OFF_D + m, OFF_X = OFF_U + m, OFF_L = OFF_X + n;
    static constexpr int LAM_SLOTS = 2 * (n + m);
    static constexpr int NSLOT = OFF_L + LAM_SLOTS;
    static constexpr int DOUBLES = NSLOT * IPB;          // per stage buffer
    __device__ static __forceinline__ int kidx(int e, int g) { return K16 ? ((e >> 1) * IPB + g) * 2 + (e & 1) : e * IPB + g; }
    __device__ static __forceinline__ int sidx(int slot, int g) { return slot * IPB + g; }
};

// lanes of a group cooperatively issue the async copies of knot k's K_k, d_k, u_k, x_k of instance g (none on the terminal knot)
template <int n, int m, int IPB, int G, int NE>
__device__ __forceinline__ void prefetch_operands(double* base, int g, int l, int k, const double* Kg, const double* dg, const double* X,
                                                  const double* U, int N) {
    using S = Stage<n, m, IPB, NE>;
    if (k < N - 1) {
        const double* Kk = Kg + (size_t)k * NE * m;
        if (S::K16) {
#pragma unroll
            for (int c = 0; c < (S::KSLOTS / 2 + G - 1) / G; c++) {
                const int cc = c * G + l;
                if (cc < S::KSLOTS / 2) cp_async16(base + S::kidx(2 * cc, g), Kk + 2 * cc);
            }
        } else {
#pragma unroll
            for (int c = 0; c < (S::KSLOTS + G - 1) / G; c++) {
                const int cc = c * G + l;
                if (cc < S::KSLOTS) cp_async8(base + S::kidx(cc, g), Kk + cc);
            }
        }
        // d, u, x : 2m + n consecutive 8-byte slots
#pragma unroll
        for (int c = 0; c < (2 * m + n + G - 1) / G; c++) {
            const int s = c * G + l;
            if (s < m) cp_async8(base + S::sidx(S::OFF_D + s, g), dg + (size_t)k * m + s);
            else if (s < 2 * m) cp_async8(base + S::sidx(S::OFF_U + s - m, g), U + (size_t)k * m + (s - m));
            else if (s < 2 * m + n) cp_async8(base + S::sidx(S::OFF_X + s - 2 * m, g), X + (size_t)k * n + (s - 2 * m));
        }
    }
}

// ... and the multipliers of knot k+1 (prefetch_operands + multipliers = one knot of the operand ring)
template <int n, int m, int IPB, int G, int NE>
__device__ __forceinline__ void prefetch_knot(double* base, int g, int l, int k, const double* Kg, const double* dg, const double* X,
                                              const double* U, const double* lam_b, const FwdTab& tab, int N) {
    using S = Stage<n, m, IPB, NE>;
    prefetch_operands<n, m, IPB, G, NE>(base, g, l, k, Kg, dg, X, U, N);
    // multipliers of the (at most two) constraints active at knot k+1, packed in constraint order
    {
        const int c0 = tab.lam_cnt[k][0], c1 = tab.lam_cnt[k][1];
        const double* l0 = lam_b + tab.lam_off[k][0];
        const double* l1 = lam_b + tab.lam_off[k][1];
        for (int i = l; i < c0; i += G) cp_async8(base + S::sidx(S::OFF_L + i, g), l0 + i);
        for (int i = l; i < c1; i += G) cp_async8(base + S::sidx(S::OFF_L + c0 + i, g), l1 + i);
    }
}

// closed-loop rollout of instance b (group g of the CTA) with step size alpha, diagonal costs, Goal/Bound constraints.
// The candidate trajectory goes to buffer `cbuf`.  Returns the merit; `ok` = no blow-up.
// INST: the instance's own linear cost terms and Goal values (DevProblem::qr / goal, read from global memory instead of the CTA's table), and
// time steps (DevProblem::dtb, loaded per knot instead of the table's).
template <int MODEL, int IPB, int G, bool LIE, bool INST, int RULE>
__device__ __forceinline__ double rollout_fast(const DevProblem& P, const FwdTab& tab, double* stage, const double* prm, int b, int g, int l,
                                               unsigned gmask, double alpha, int cbuf, bool& ok, double& viol) {
    constexpr int n = ModelDims<MODEL>::n, m = ModelDims<MODEL>::m, NE = LIE ? n - 1 : n;
    using S = Stage<n, m, IPB, NE>;
    const int N = P.N, buf = P.cur[b];
    const double* X = traj_X(P, buf, b);
    const double* U = traj_U(P, buf, b);
    double* Xc = traj_Xw(P, cbuf, b);
    double* Uc = traj_Uw(P, cbuf, b);
    const double* Kg = P.K + (size_t)b * (N - 1) * NE * m;
    const double* dg = P.d + (size_t)b * (N - 1) * m;
    const double* lam_b = P.lambda + (size_t)b * P.lambda_len;
    double x[n], u[m], xn[n];
    double J = 0.0;
    ok = true; viol = 0.0;
#pragma unroll
    for (int i = 0; i < n; i++) x[i] = P.x0[(size_t)b * n + i];
    constexpr int D = FWD_STAGES - 1;           // prefetch distance in knots
#pragma unroll
    for (int j = 0; j < D; j++) {
        if (j < N) prefetch_knot<n, m, IPB, G, NE>(stage + j * S::DOUBLES, g, l, j, Kg, dg, X, U, lam_b, tab, N);
        cp_async_commit();
    }
    int sb = 0, sp = D;                         // stage of knot k, stage knot k + D goes to (= the one knot k - 1 has just left)
    for (int k = 0; k < N; k++) {
        const bool last = (k == N - 1);
        __syncwarp(gmask);                      // every lane of the group is done reading the stage of knot k-1
        if (k + D < N) prefetch_knot<n, m, IPB, G, NE>(stage + sp * S::DOUBLES, g, l, k + D, Kg, dg, X, U, lam_b, tab, N);
        cp_async_commit();
        cp_async_wait<D>();                     // this lane's copies for knot k have landed ...
        __syncwarp(gmask);                      // ... and so have the other lanes'
        const double* st = stage + sb * S::DOUBLES;
        sb = (sb + 1 == FWD_STAGES) ? 0 : sb + 1; sp = (sp + 1 == FWD_STAGES) ? 0 : sp + 1;
        if (!last) {
#pragma unroll
            for (int a = 0; a < m; a++) u[a] = fma(alpha, st[S::sidx(S::OFF_D + a, g)], st[S::sidx(S::OFF_U + a, g)]);
            double dxe[NE];   // RD.state_diff(xbar_k, x_k): plain difference, or the Cayley error of the attitude (LIE)
            if constexpr (LIE) {
                double xr[n];
#pragma unroll
                for (int i = 0; i < n; i++) xr[i] = st[S::sidx(S::OFF_X + i, g)];
                state_diff(true, n, 3, x, xr, dxe);
            } else {
#pragma unroll
                for (int i = 0; i < n; i++) dxe[i] = x[i] - st[S::sidx(S::OFF_X + i, g)];
            }
#pragma unroll
            for (int i = 0; i < NE; i++) {
                const double dx = dxe[i];
                if (S::K16 && (m % 2 == 0)) {
#pragma unroll
                    for (int a = 0; a < m; a += 2) {
                        const double2 kv = *reinterpret_cast<const double2*>(&st[S::kidx(i * m + a, g)]);
                        u[a] = fma(kv.x, dx, u[a]);
                        u[a + 1] = fma(kv.y, dx, u[a + 1]);
                    }
                } else {
#pragma unroll
                    for (int a = 0; a < m; a++) u[a] = fma(st[S::kidx(i * m + a, g)], dx, u[a]);
                }
            }
#pragma unroll
            for (int a = 0; a < m; a++) if (!(fabs(u[a]) <= P.opt.max_control_value)) ok = false;
        } else {
#pragma unroll
            for (int a = 0; a < m; a++) u[a] = 0.0;
        }
#pragma unroll
        for (int i = 0; i < n; i++) Xc[(size_t)k * n + i] = x[i];
        if (!last) {
#pragma unroll
            for (int a = 0; a < m; a++) Uc[(size_t)k * m + a] = u[a];
        }
        // ---- cost of knot k (DiagonalCost) -------------------------------------------------------------
        {
            const int cid = tab.cost_index[k];
            double a2 = 0.0, l1 = 0.0, cc;
            if (tab.ncost_cached) {
                const CostData c = cost_data<INST>(P, b, cid, staged(tab.cost[cid]));
#pragma unroll
                for (int i = 0; i < n; i++) { a2 = fma(c.Qd[i] * x[i], x[i], a2); l1 = fma(c.q[i], x[i], l1); }
                if (!last) {
#pragma unroll
                    for (int i = 0; i < m; i++) { a2 = fma(c.Rd[i] * u[i], u[i], a2); l1 = fma(c.r[i], u[i], l1); }
                }
                cc = *c.c;
            } else {
                const CostData c = cost_data<INST>(P, b, cid);
#pragma unroll
                for (int i = 0; i < n; i++) { a2 = fma(c.Qd[i] * x[i], x[i], a2); l1 = fma(c.q[i], x[i], l1); }
                if (!last) {
#pragma unroll
                    for (int i = 0; i < m; i++) { a2 = fma(c.Rd[i] * u[i], u[i], a2); l1 = fma(c.r[i], u[i], l1); }
                }
                cc = *c.c;
            }
            J += fma(0.5, a2, l1) + cc;
        }
        // ---- AL penalty of knot k (Goal / Bound): (|Pi_K*(lambda - mu c)|^2 - |lambda|^2) / (2 mu) -------------
        {
            int slot = 0;
            for (int ci = 0; ci < tab.ncon; ci++) {
                const FwdCon& c = tab.con[ci];
                if (k + 1 < c.first || k + 1 > c.last) continue;
                const bool own = INST && P.mub != nullptr;                 // this instance's penalty, with load_tables' operations
                const double mu = own ? penalty<INST>(P, b, ci) : c.mu;
                const int lo = S::OFF_L + slot;
                double a = 0.0, l2 = 0.0;
                if (c.kind == CON_GOAL) {
                    const unsigned mk = c.mask_max;
                    const double* ga = con_data<INST>(P, b, ci, staged(c)).a;
#pragma unroll
                    for (int i = 0; i < n; i++) {
                        if (mk & (1u << i)) {
                            const int row = c.row_max[i];
                            const double lm = st[S::sidx(lo + row, g)];
                            const double cv = x[i] - ga[row];
                            const double lp = fma(-mu, cv, lm);
                            a = fma(lp, lp, a); l2 = fma(lm, lm, l2); viol = fmax(viol, fabs(cv));
                        }
                    }
                } else if (c.ubox) {
                    // u_min <= u <= u_max on every control: rows 0..m-1 = upper, m..2m-1 = lower (src/constraints.jl:738-755)
                    const ConData cd = con_data<INST>(P, b, ci, staged(c));
#pragma unroll
                    for (int i = 0; i < m; i++) {
                        const double lu = st[S::sidx(lo + i, g)], ll = st[S::sidx(lo + m + i, g)];
                        const double cu = u[i] - cd.a[n + i], cl = cd.b[n + i] - u[i];
                        const double pu = fmin(0.0, fma(-mu, cu, lu)), pl = fmin(0.0, fma(-mu, cl, ll));
                        a = fma(pu, pu, a); a = fma(pl, pl, a); l2 = fma(lu, lu, l2); l2 = fma(ll, ll, l2);
                        viol = fmax(viol, fmax(cu, cl));
                    }
                } else {
                    const unsigned mx = c.mask_max, mn = c.mask_min;
                    const ConData cd = con_data<INST>(P, b, ci, staged(c));
                    if ((mx | mn) & ((1u << n) - 1u)) {
#pragma unroll
                        for (int i = 0; i < n; i++) {
                            if (mx & (1u << i)) { const double lm = st[S::sidx(lo + c.row_max[i], g)]; const double cv = x[i] - cd.a[i]; const double lp = fmin(0.0, fma(-mu, cv, lm)); a = fma(lp, lp, a); l2 = fma(lm, lm, l2); viol = fmax(viol, cv); }
                            if (mn & (1u << i)) { const double lm = st[S::sidx(lo + c.row_min[i], g)]; const double cv = cd.b[i] - x[i]; const double lp = fmin(0.0, fma(-mu, cv, lm)); a = fma(lp, lp, a); l2 = fma(lm, lm, l2); viol = fmax(viol, cv); }
                        }
                    }
#pragma unroll
                    for (int i = 0; i < m; i++) {
                        if (mx & (1u << (n + i))) { const double lm = st[S::sidx(lo + c.row_max[n + i], g)]; const double cv = u[i] - cd.a[n + i]; const double lp = fmin(0.0, fma(-mu, cv, lm)); a = fma(lp, lp, a); l2 = fma(lm, lm, l2); viol = fmax(viol, cv); }
                        if (mn & (1u << (n + i))) { const double lm = st[S::sidx(lo + c.row_min[n + i], g)]; const double cv = cd.b[n + i] - u[i]; const double lp = fmin(0.0, fma(-mu, cv, lm)); a = fma(lp, lp, a); l2 = fma(lm, lm, l2); viol = fmax(viol, cv); }
                    }
                }
                J = fma(a - l2, own ? 1.0 / (2.0 * mu) : c.inv2mu, J);
                slot += c.p;
            }
        }
        if (!last) {
            explicit_step<MODEL, double, RULE>(model_params<MODEL, INST>(P, prm, k), x, u, time_step<INST>(P, b, k, tab.dt), xn);
#pragma unroll
            for (int i = 0; i < n; i++) { x[i] = xn[i]; if (!(fabs(xn[i]) <= P.opt.max_state_value)) ok = false; }
            // a blown-up trial keeps integrating (the group stays in lock step); its result is rejected through `ok`
        }
    }
    cp_async_wait<0>();
    return J;
}

// rollout_fast for the compact class, the same FP64 operations on the same operands in the same order, with less work around them:
//   * the terminal knot (no control, no feedback, the Goal) is peeled off, so the knot loop has no `last` tests and no constraint loop:
//     the box is the only constraint of a stage knot, its multipliers of knot k+1 sit at box_off + k p;
//   * the stage cost is a {Qd_i, q_i} pair per 16-byte load instead of two 8-byte loads;
//   * the AL clamp and the violation max are compare-and-select (proofs at the box below);
//   * the candidate trajectory leaves through shared memory: each lane stages FWD_OKNOTS knots of its x and u, then the lanes of the group
//     write each lane's runs together, G consecutive doubles per store instruction.  One lane storing its own 8-byte words sent one L2 write
//     request per word from every lane, and those requests, not the arithmetic, set the pace of the pass (a timing-only build without the
//     candidate stores ran pass 1 in about half the time);
//   * the step writes the next state over the current one (every rule of explicit_step reads x_i for the last time where it writes xn_i), so the loop carries
//     no x <- xn copies.  (Unrolled by two with x / xn swapping roles instead, the loop took 40 more registers and spilled.)
// INST: gbox = the instance's control box {u_max_i, u_min_i} and gcost = its two costs and penalties, staged for the group by linesearch_pass;
// its time steps are loaded per knot (time_step)
template <int MODEL, int IPB, int G, bool LIE, bool INST, int RULE>
__device__ __forceinline__ double rollout_compact(const DevProblem& P, const FwdCompactTab& tab, double* stage, double* ost, const double* prm,
                                                  const double2* gbox, const FwdCompactCost* gcost, int b, int g, int l, unsigned gmask,
                                                  double alpha, int cbuf, bool& ok, double& viol) {
    constexpr int n = ModelDims<MODEL>::n, m = ModelDims<MODEL>::m, NE = LIE ? n - 1 : n;
    using S = Stage<n, m, IPB, NE>;
    const int N = P.N, buf = P.cur[b];
    const double* X = traj_X(P, buf, b);
    const double* U = traj_U(P, buf, b);
    double* Xc = traj_Xw(P, cbuf, b);
    const double* Kg = P.K + (size_t)b * (N - 1) * NE * m;
    const double* dg = P.d + (size_t)b * (N - 1) * m;
    const double* lam_b = P.lambda + (size_t)b * P.lambda_len;
    // ost: the group's output staging, FWD_OKNOTS knots of x then u per lane; lane j's candidate goes to buffer (buf + 1 + j) % TO_NBUF
    constexpr int OX = FWD_OKNOTS * n, OL = FWD_OKNOTS * (n + m);
    double* myx = ost + l * OL;
    double* myu = myx + OX;
    const double2* sx = INST ? gcost->sx : tab.sx;
    const double2* su = INST ? gcost->su : tab.su;
    const double* sc = INST ? &gcost->sc : &tab.sc;
    const FwdCost& term = INST ? gcost->term : tab.term;
    const bool box = tab.box_p != 0;
    double x[n], u[m];
    double J = 0.0;
    ok = true; viol = 0.0;
#pragma unroll
    for (int i = 0; i < n; i++) x[i] = P.x0[(size_t)b * n + i];
    constexpr int D = FWD_STAGES - 1;
    // knot k of the operand ring: K, d, u, x of knot k and the multipliers of knot k+1 (the box's, or the Goal's on the terminal knot)
    auto prefetch = [&](double* base, int k) {
        prefetch_operands<n, m, IPB, G, NE>(base, g, l, k, Kg, dg, X, U, N);
        const bool stg = k < N - 1;
        const int cnt = stg ? tab.box_p : tab.goal_p;
        const double* src = lam_b + (stg ? tab.box_off + k * tab.box_p : tab.goal_off);
        for (int i = l; i < cnt; i += G) cp_async8(base + S::sidx(S::OFF_L + i, g), src + i);
    };
#pragma unroll
    for (int j = 0; j < D; j++) {
        if (j < N) prefetch(stage + j * S::DOUBLES, j);
        cp_async_commit();
    }
    int sb = 0, sp = D;
    auto next_stage = [&](int k) -> const double* {
        __syncwarp(gmask);                      // every lane of the group is done reading the stage of knot k-1
        if (k + D < N) prefetch(stage + sp * S::DOUBLES, k + D);
        cp_async_commit();
        cp_async_wait<D>();                     // this lane's copies for knot k have landed ...
        __syncwarp(gmask);                      // ... and so have the other lanes'
        const double* st = stage + sb * S::DOUBLES;
        sb = (sb + 1 == FWD_STAGES) ? 0 : sb + 1; sp = (sp + 1 == FWD_STAGES) ? 0 : sp + 1;
        return st;
    };
    // stage knot k < N - 1: x_k -> x_{k+1} in place
    auto knot = [&](int k, double* x) {
        const double* st = next_stage(k);
#pragma unroll
        for (int a = 0; a < m; a++) u[a] = fma(alpha, st[S::sidx(S::OFF_D + a, g)], st[S::sidx(S::OFF_U + a, g)]);
        double dxe[NE];
        if constexpr (LIE) {
            double xr[n];
#pragma unroll
            for (int i = 0; i < n; i++) xr[i] = st[S::sidx(S::OFF_X + i, g)];
            state_diff(true, n, 3, x, xr, dxe);
        } else {
#pragma unroll
            for (int i = 0; i < n; i++) dxe[i] = x[i] - st[S::sidx(S::OFF_X + i, g)];
        }
#pragma unroll
        for (int i = 0; i < NE; i++) {
            const double dx = dxe[i];
            if (S::K16 && (m % 2 == 0)) {
#pragma unroll
                for (int a = 0; a < m; a += 2) {
                    const double2 kv = *reinterpret_cast<const double2*>(&st[S::kidx(i * m + a, g)]);
                    u[a] = fma(kv.x, dx, u[a]);
                    u[a + 1] = fma(kv.y, dx, u[a + 1]);
                }
            } else {
#pragma unroll
                for (int a = 0; a < m; a++) u[a] = fma(st[S::kidx(i * m + a, g)], dx, u[a]);
            }
        }
#pragma unroll
        for (int a = 0; a < m; a++) if (!(fabs(u[a]) <= P.opt.max_control_value)) ok = false;
        const int kk = k % FWD_OKNOTS;
#pragma unroll
        for (int i = 0; i < n; i++) myx[kk * n + i] = x[i];
#pragma unroll
        for (int a = 0; a < m; a++) myu[kk * m + a] = u[a];
        if (kk == FWD_OKNOTS - 1 || k == N - 2) {   // group-uniform: write the staged knots k0..k of every lane of the group
            __syncwarp(gmask);
            const int k0 = k - kk, nx = (kk + 1) * n, nu = (kk + 1) * m;
            for (int j = 0; j < G; j++) {
                const int cb = (buf + 1 + j) % TO_NBUF;
                double* xd = traj_Xw(P, cb, b) + (size_t)k0 * n;
                double* ud = traj_Uw(P, cb, b) + (size_t)k0 * m;
                const double* xs = ost + j * OL;
                for (int e = l; e < nx; e += G) xd[e] = xs[e];
                for (int e = l; e < nu; e += G) ud[e] = xs[OX + e];
            }
            // the next knot overwrites the staging only after next_stage's __syncwarp
        }
        {   // stage cost
            double a2 = 0.0, l1 = 0.0;
#pragma unroll
            for (int i = 0; i < n; i++) { const double2 c = sx[i]; a2 = fma(c.x * x[i], x[i], a2); l1 = fma(c.y, x[i], l1); }
#pragma unroll
            for (int i = 0; i < m; i++) { const double2 c = su[i]; a2 = fma(c.x * u[i], u[i], a2); l1 = fma(c.y, u[i], l1); }
            J += fma(0.5, a2, l1) + *sc;
        }
        if (box) {
            // AL penalty of the control box, rollout_fast's ubox branch with two replacements:
            //   pu = fmin(0, v)  ->  v < 0 ? v : 0.  They differ only at v = -0 (fmin gives -0, the select +0; NaN gives 0 in both), and pu
            //     is only used squared in fma(pu, pu, a), whose exact product is +0 either way, so a gets the same bits.
            //   viol = fmax(viol, fmax(cu, cl))  ->  t = cu > cl ? cu : cl ; viol = t > viol ? t : viol.  CUDA's fmax returns the
            //     non-NaN operand and orders -0 below +0 (measured on sm_90a).  viol starts at +0 and so is never NaN or -0.  The bounds
            //     are finite, so cu and cl are both NaN (u is) or neither: both NaN -> t = NaN, and both forms keep viol.  Otherwise t is
            //     fmax(cu, cl) except for cu = +0, cl = -0, where t = -0: then fmax(viol, +0) = viol = the select, as viol >= +0.  For
            //     t != NaN, fmax(viol, t) and the select agree except at viol = +0, t = -0, where both give viol.
            const double mu = INST ? gcost->mu : tab.mu;
            double a = 0.0, l2 = 0.0;
#pragma unroll
            for (int i = 0; i < m; i++) {
                const double lu = st[S::sidx(S::OFF_L + i, g)], ll = st[S::sidx(S::OFF_L + m + i, g)];
                const double2 bx = INST ? gbox[i] : tab.box[i];
                const double cu = u[i] - bx.x, cl = bx.y - u[i];
                const double vu = fma(-mu, cu, lu), vl = fma(-mu, cl, ll);
                const double pu = vu < 0.0 ? vu : 0.0, pl = vl < 0.0 ? vl : 0.0;
                a = fma(pu, pu, a); a = fma(pl, pl, a); l2 = fma(lu, lu, l2); l2 = fma(ll, ll, l2);
                const double t = cu > cl ? cu : cl;
                viol = t > viol ? t : viol;
            }
            J = fma(a - l2, INST ? gcost->inv2mu : tab.inv2mu, J);
        }
        if constexpr (is_recorded<MODEL>) {   // a discrete jump map writes its outputs while it reads its inputs
            double xn[n];
            explicit_step<MODEL, double, RULE>(model_params<MODEL, INST>(P, prm, k), x, u, time_step<INST>(P, b, k, tab.dt), xn);
#pragma unroll
            for (int i = 0; i < n; i++) x[i] = xn[i];
        } else {
            explicit_step<MODEL, double, RULE>(model_params<MODEL, INST>(P, prm, k), x, u, time_step<INST>(P, b, k, tab.dt), x);
        }
#pragma unroll
        for (int i = 0; i < n; i++) if (!(fabs(x[i]) <= P.opt.max_state_value)) ok = false;
        // a blown-up trial keeps integrating (the group stays in lock step); its result is rejected through `ok`
    };
#pragma unroll 1
    for (int k = 0; k < N - 1; k++) knot(k, x);
    {   // terminal knot N - 1: terminal cost and the Goal, as rollout_fast evaluates them on its last knot
        const double* st = next_stage(N - 1);
#pragma unroll
        for (int i = 0; i < n; i++) Xc[(size_t)(N - 1) * n + i] = x[i];
        double a2 = 0.0, l1 = 0.0;
#pragma unroll
        for (int i = 0; i < n; i++) { a2 = fma(term.Qd[i] * x[i], x[i], a2); l1 = fma(term.q[i], x[i], l1); }
        J += fma(0.5, a2, l1) + term.c;
        if (tab.goal_ci >= 0) {
            const FwdCon& c = tab.goal;
            const double mu = INST ? gcost->gmu : c.mu;
            double a = 0.0, l2 = 0.0;
            const unsigned mk = c.mask_max;
            const double* ga = con_data<INST>(P, b, tab.goal_ci, staged(c)).a;
#pragma unroll
            for (int i = 0; i < n; i++) {
                if (mk & (1u << i)) {
                    const int row = c.row_max[i];
                    const double lm = st[S::sidx(S::OFF_L + row, g)];
                    const double cv = x[i] - ga[row];
                    const double lp = fma(-mu, cv, lm);
                    a = fma(lp, lp, a); l2 = fma(lm, lm, l2); viol = fmax(viol, fabs(cv));
                }
            }
            J = fma(a - l2, INST ? gcost->ginv2mu : c.inv2mu, J);
        }
    }
    cp_async_wait<0>();
    return J;
}

// generic path (dense costs or general constraints): pointer-based evaluation, operands read directly from global
template <int MODEL, bool LIE, bool INST, int RULE>
__device__ __forceinline__ double rollout_generic(const DevProblem& P, const double* prm, int b, double alpha, int cbuf, bool& ok, double& viol) {
    constexpr int n = ModelDims<MODEL>::n, m = ModelDims<MODEL>::m, NE = LIE ? n - 1 : n;
    const int N = P.N, buf = P.cur[b];
    const double* X = traj_X(P, buf, b);
    const double* U = traj_U(P, buf, b);
    double* Xc = traj_Xw(P, cbuf, b);
    double* Uc = traj_Uw(P, cbuf, b);
    const double* Kg = P.K + (size_t)b * (N - 1) * NE * m;
    const double* dg = P.d + (size_t)b * (N - 1) * m;
    const double* lam_b = P.lambda + (size_t)b * P.lambda_len;
    double x[n], u[m], xn[n];
    double J = 0.0;
    ok = true; viol = 0.0;
#pragma unroll
    for (int i = 0; i < n; i++) x[i] = P.x0[(size_t)b * n + i];
    for (int k = 0; k < N; k++) {
        const bool last = (k == N - 1);
        if (!last) {
#pragma unroll
            for (int a = 0; a < m; a++) u[a] = fma(alpha, dg[(size_t)k * m + a], U[(size_t)k * m + a]);
            double dxe[NE], xr[n];
#pragma unroll
            for (int i = 0; i < n; i++) xr[i] = X[(size_t)k * n + i];
            state_diff(LIE, n, 3, x, xr, dxe);
#pragma unroll
            for (int i = 0; i < NE; i++) {
                const double dx = dxe[i];
#pragma unroll
                for (int a = 0; a < m; a++) u[a] = fma(Kg[(size_t)k * NE * m + i * m + a], dx, u[a]);
            }
#pragma unroll
            for (int a = 0; a < m; a++) if (!(fabs(u[a]) <= P.opt.max_control_value)) ok = false;
        } else {
#pragma unroll
            for (int a = 0; a < m; a++) u[a] = 0.0;
        }
#pragma unroll
        for (int i = 0; i < n; i++) Xc[(size_t)k * n + i] = x[i];
        if (!last) {
#pragma unroll
            for (int a = 0; a < m; a++) Uc[(size_t)k * m + a] = u[a];
        }
        const int cid = P.cost_index[k];
        J += cost_value(P.costs[cid], cost_data<INST>(P, b, cid), n, m, x, u, !last);
        J += al_knot_penalty<INST>(P, k + 1, x, u, lam_b, viol, b);
        if (!last) {
            // INST: the determinant form the shared kernel compiles to, written out (models.cuh det_sub_square)
            explicit_step<MODEL, double, RULE, INST>(model_params<MODEL, INST>(P, prm, k), x, u, time_step<INST>(P, b, k), xn);
#pragma unroll
            for (int i = 0; i < n; i++) { x[i] = xn[i]; if (!(fabs(xn[i]) <= P.opt.max_state_value)) ok = false; }
            if (!ok) break;
        }
    }
    return J;
}

__device__ __forceinline__ bool ls_accept(const DevProblem& P, double J, double J_prev, double alpha, double dV1, double dV2, bool ok) {
    if (!ok) return false;
    const double expected = -alpha * (dV1 + alpha * dV2);
    const double z = expected > 0.0 ? (J_prev - J) / expected : -1.0;
    return (z > P.opt.ls_lower && z <= P.opt.ls_upper) || (J < J_prev);
}

extern __shared__ __align__(16) unsigned char fwd_smem[];

// rollout of a trial: rollout_generic, rollout_fast or rollout_compact
enum { FWD_GENERIC = 0, FWD_FAST = 1, FWD_COMPACT = 2 };
// the knot loop of the compact class: 1 = rollout_compact; 0 = rollout_fast for it as for every other fast-path problem (A/B builds)
#ifndef TO_FWD_COMPACT
#define TO_FWD_COMPACT 1
#endif

// dynamic shared memory of a line-search CTA: the cached tables, the operand ring and rollout_compact's output staging (the generic path
// uses none of them); the INST variant keeps each group's model parameters behind them (launch_pass_l adds IPB rows of TO_NPARAM)
template <int MODEL, int G, int PATH, int LANES, bool LIE>
__host__ __device__ constexpr size_t ls_smem_bytes() {
    constexpr int n = ModelDims<MODEL>::n, m = ModelDims<MODEL>::m, NE = LIE ? n - 1 : n;
    constexpr int IPB = LANES / G;
    const size_t tab = PATH == FWD_COMPACT ? sizeof(FwdCompactTab) : sizeof(FwdTab);
    const size_t ost = PATH == FWD_COMPACT ? (size_t)LANES * FWD_OKNOTS * (n + m) * sizeof(double) : 0;   // rollout_compact's output staging
    return PATH != FWD_GENERIC ? tab + (size_t)FWD_STAGES * Stage<n, m, IPB, NE>::DOUBLES * sizeof(double) + ost : 0;
}

// One line-search pass: lane l of group g evaluates trial (trial0 + l) of instance b.
//   first_pass : ignore / reset accepted[b];   final_pass : commit failures (no acceptable step size).
template <int MODEL, int G, int PATH, int LANES, bool LIE, bool INST, int RULE>
__device__ __forceinline__ void linesearch_pass(const DevProblem& P, int trial0, int first_pass, int final_pass) {
    constexpr int n = ModelDims<MODEL>::n, m = ModelDims<MODEL>::m, NE = LIE ? n - 1 : n;
    constexpr bool FAST = PATH != FWD_GENERIC;
    // LANES = 16: only half of the warp carries groups.  The pass is a latency-bound FP64 chain at ~4 warps per SM, and
    // an FP64 instruction of a half-empty warp takes one pipe pass instead of two.
    constexpr int IPB = LANES / G;
    using S = Stage<n, m, IPB, NE>;
    using Tab = std::conditional_t<PATH == FWD_COMPACT, FwdCompactTab, FwdTab>;
    Tab* tab = reinterpret_cast<Tab*>(fwd_smem);
    double* stage = reinterpret_cast<double*>(fwd_smem + sizeof(Tab));
    const int g = (threadIdx.x % LANES) / G, l = threadIdx.x % G;
    // pass 1 walks every instance; the later passes walk the list pass 1 left of the instances it did not accept, so that only CTAs with work
    // stay resident next to the kernels of the main stream (a CTA with one late instance of four used to hold its registers for the whole pass)
    int b = blockIdx.x * IPB + g;
    if (!first_pass && P.late_list) b = (b < *P.late_count) ? P.late_list[b] : P.B;
    const unsigned gmask = (G == 32) ? 0xffffffffu : (((1u << G) - 1u) << (g * G));
    // (to_solve: an instance that is not ACTIVE is neither tried, accepted, late-listed nor committed)
    const bool valid = b < P.B && threadIdx.x < LANES && !retired(P, b);
    const int status = valid ? P.bp_status[b] : -1;
    const int was_accepted = (valid && !first_pass) ? P.accepted[b] : 0;
    const bool work = valid && status >= 0 && !was_accepted && trial0 <= P.opt.ls_iters;
    // CTA-uniform: skip the table load when no group of this CTA has work
    const unsigned any = __ballot_sync(0xffffffffu, work);
    if constexpr (PATH == FWD_COMPACT) { if (any) load_compact_tables(P, *tab); }
    else if (FAST && any) load_tables(P, *tab);
    if (!valid) return;
    bool accepted = was_accepted != 0;
    if (work) {
        const int trial = trial0 + l;
        const double alpha = ldexp(1.0, -trial);
        const int cbuf = (P.cur[b] + 1 + l) % TO_NBUF;
        bool ok = false;
        double J, viol = 0.0;
        double* prm = nullptr;
        double2* gbox = nullptr;
        FwdCompactCost* gcost = nullptr;
        if constexpr (INST) {   // the instance's model parameters, one copy per group behind the rest of the CTA's shared memory
            prm = reinterpret_cast<double*>(fwd_smem + ls_smem_bytes<MODEL, G, PATH, LANES, LIE>()) + g * TO_NPARAM;
            if (l == 0) stage_model_params<INST>(P, b, prm);
            if constexpr (PATH == FWD_COMPACT) {   // ... its control box, behind the parameter rows of the CTA's groups, and its two costs
                double2* boxes = reinterpret_cast<double2*>(reinterpret_cast<double*>(fwd_smem + ls_smem_bytes<MODEL, G, PATH, LANES, LIE>()) + IPB * TO_NPARAM);
                gbox = boxes + g * TO_MAXM;
                gcost = reinterpret_cast<FwdCompactCost*>(boxes + IPB * TO_MAXM) + g;
                const CostData c = cost_data<true>(P, b, tab->cid), ct = cost_data<true>(P, b, tab->tcid);
                for (int i = l; i < n; i += G) { gcost->sx[i] = make_double2(c.Qd[i], c.q[i]); gcost->term.Qd[i] = ct.Qd[i]; gcost->term.q[i] = ct.q[i]; }
                for (int i = l; i < m; i += G) gcost->su[i] = make_double2(c.Rd[i], c.r[i]);
                if (l == 0) { gcost->sc = *c.c; gcost->term.c = *ct.c; }
                if (tab->box_p != 0)
                    for (int ci = 0; ci < P.ncon; ci++)
                        if (P.cons[ci].kind == CON_BOUND) {
                            const ConData cd = con_data<true>(P, b, ci);
                            for (int i = l; i < m; i += G) gbox[i] = make_double2(cd.a[n + i], cd.b[n + i]);
                            if (l == 0) { gcost->mu = penalty<true>(P, b, ci); gcost->inv2mu = 1.0 / (2.0 * gcost->mu); }
                        }
                if (l == 0 && tab->goal_ci >= 0) { gcost->gmu = penalty<true>(P, b, tab->goal_ci); gcost->ginv2mu = 1.0 / (2.0 * gcost->gmu); }
            }
            __syncwarp(gmask);
        }
        if constexpr (PATH == FWD_COMPACT) {
            double* ost = stage + FWD_STAGES * S::DOUBLES + (size_t)g * G * FWD_OKNOTS * (n + m);
            J = rollout_compact<MODEL, IPB, G, LIE, INST, RULE>(P, *tab, stage, ost, prm, gbox, gcost, b, g, l, gmask, alpha, cbuf, ok, viol);
        }
        else if (FAST) J = rollout_fast<MODEL, IPB, G, LIE, INST, RULE>(P, *tab, stage, prm, b, g, l, gmask, alpha, cbuf, ok, viol);
        else J = rollout_generic<MODEL, LIE, INST, RULE>(P, prm, b, alpha, cbuf, ok, viol);
        const bool good = (trial <= P.opt.ls_iters) && ls_accept(P, J, P.J[b], alpha, P.dV[2 * b], P.dV[2 * b + 1], ok);
        const unsigned votes = __ballot_sync(gmask, good) & gmask;
        if (votes) {
            const int win = __ffs(votes) - 1 - g * G;
            if (l == win) {
                P.cur[b] = cbuf; P.J[b] = J; P.viol[b] = viol; P.alpha[b] = alpha; P.ls_iters[b] = trial + 1; P.accepted[b] = 1;
            }
            accepted = true;
        }
    }
    if (l == 0 && first_pass) {
        P.acc1[b] = accepted ? 1 : 0;
        if (!accepted && P.late_list) P.late_list[atomicAdd(P.late_count, 1)] = b;
    }
    if (l == 0 && !accepted) {
        if (first_pass) P.accepted[b] = 0;
        if (status < 0) { P.alpha[b] = 0.0; P.ls_iters[b] = 0; }
        else if (final_pass) {   // no acceptable step: keep the trajectory, raise the regularisation (Altro forwardpass!)
            double rho = P.rho[b], drho = P.drho[b];
            reg_increase(P.opt, rho, drho);
            rho += P.opt.bp_reg_fp;
            P.rho[b] = rho; P.drho[b] = drho;
            P.alpha[b] = 0.0; P.ls_iters[b] = P.opt.ls_iters + 1;
        }
    }
    (void)sizeof(S);
}

template <int MODEL, int G, bool FAST, int LANES, bool LIE, bool INST, int RULE>
__global__ void __launch_bounds__(FWD_THREADS) k_linesearch(const DevProblem P, int trial0, int first_pass, int final_pass) {
    linesearch_pass<MODEL, G, FAST ? FWD_FAST : FWD_GENERIC, LANES, LIE, INST, RULE>(P, trial0, first_pass, final_pass);
}

template <int MODEL, int G, int LANES, bool LIE, bool INST, int RULE>
__global__ void __launch_bounds__(FWD_THREADS) k_linesearch_compact(const DevProblem P, int trial0, int first_pass, int final_pass) {
    linesearch_pass<MODEL, G, FWD_COMPACT, LANES, LIE, INST, RULE>(P, trial0, first_pass, final_pass);
}

template <int MODEL, int G, int PATH, int LANES, bool LIE, bool INST, int RULE>
cudaError_t launch_pass_l(const DevProblem& P, int trial0, int first_pass, int final_pass, cudaStream_t s) {
    constexpr int IPB = LANES / G;
    const int blocks = (P.B + IPB - 1) / IPB;
    static_assert(ls_smem_bytes<MODEL, G, PATH, LANES, LIE>() % 16 == 0, "the parameter rows and the staged boxes (double2) follow the tables");
    const size_t smem = ls_smem_bytes<MODEL, G, PATH, LANES, LIE>() + (INST ? (size_t)IPB * TO_NPARAM * sizeof(double) : 0)
                      + (INST && PATH == FWD_COMPACT ? (size_t)IPB * (TO_MAXM * sizeof(double2) + sizeof(FwdCompactCost)) : 0);
    auto kern = [] {
        if constexpr (PATH == FWD_COMPACT) return k_linesearch_compact<MODEL, G, LANES, LIE, INST, RULE>;
        else return k_linesearch<MODEL, G, PATH == FWD_FAST, LANES, LIE, INST, RULE>;
    }();
    static bool configured[TO_MAXDEV] = {false};
    const int dev = current_device_slot();
    if (!configured[dev] && smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
    }
    configured[dev] = true;
    kern<<<blocks, FWD_THREADS, smem, s>>>(P, trial0, first_pass, final_pass);
    return cudaGetLastError();
}

template <int MODEL, int G, int PATH, bool INST, int RULE>
cudaError_t launch_pass_i(const DevProblem& P, int trial0, int first_pass, int final_pass, cudaStream_t s) {
    // lanes of each warp that carry groups: 16 for the first pass (half-warp FP64 instructions take one pipe pass); the later passes
    // use 16 when they walk the compact late list (two-instance CTAs, see to_create) and 32 when they scan all instances.
    const int lanes = first_pass ? 16 : (P.late_list ? 16 : 32);
    if constexpr (MODEL == MODEL_QUADROTOR) {   // Lie-group error state: dx = state_diff(xbar, x), gains m x (n - 1)
        if (P.lie) {
            if (G <= 16 && lanes == 16) return launch_pass_l<MODEL, G, PATH, (G <= 16 ? 16 : 32), true, INST, RULE>(P, trial0, first_pass, final_pass, s);
            return launch_pass_l<MODEL, G, PATH, 32, true, INST, RULE>(P, trial0, first_pass, final_pass, s);
        }
    }
    if (G <= 16 && lanes == 16) return launch_pass_l<MODEL, G, PATH, (G <= 16 ? 16 : 32), false, INST, RULE>(P, trial0, first_pass, final_pass, s);
    return launch_pass_l<MODEL, G, PATH, 32, false, INST, RULE>(P, trial0, first_pass, final_pass, s);
}

// per-instance cost weights / linear cost terms / model parameters / constraint data / penalties / time steps: a kernel variant of its own, so
// that the shared one is the code it has always been.  It serves every per-instance table; each accessor checks its own (cost_data,
// model_param, con_data, penalty, time_step).
template <int MODEL, int G, int PATH, int RULE>
cudaError_t launch_pass(const DevProblem& P, int trial0, int first_pass, int final_pass, cudaStream_t s) {
    if (inst_forward(P)) return launch_pass_i<MODEL, G, PATH, true, RULE>(P, trial0, first_pass, final_pass, s);
    return launch_pass_i<MODEL, G, PATH, false, RULE>(P, trial0, first_pass, final_pass, s);
}

static_assert(FWD_GENERIC == KC_LS_GENERIC && FWD_FAST == KC_LS_FAST && FWD_COMPACT == KC_LS_COMPACT, "kernels.h KC_LS_*");

template <int MODEL, int G, int RULE>
cudaError_t launch_any(const DevProblem& P, int trial0, int first_pass, int final_pass, cudaStream_t s) {
    const int path = linesearch_path(P);
    if constexpr (TO_FWD_COMPACT) { if (path == FWD_COMPACT) return launch_pass<MODEL, G, FWD_COMPACT, RULE>(P, trial0, first_pass, final_pass, s); }
    if (path == FWD_FAST) return launch_pass<MODEL, G, FWD_FAST, RULE>(P, trial0, first_pass, final_pass, s);
    return launch_pass<MODEL, G, FWD_GENERIC, RULE>(P, trial0, first_pass, final_pass, s);
}

}  // namespace

// pass 1: trials 0..3 (alpha = 1, 1/2, 1/4, 1/8), 4 lanes per instance.
// (The alternative, the whole ladder in one 16-lane pass, computes 11x the FLOPs, and its uncoalesced candidate stores load the LSU.)
template <int RULE>
cudaError_t launch_forward_rule(const DevProblem& P, cudaStream_t s) {
    cudaError_t e = cudaErrorNotSupported;
    const int final_pass = P.opt.ls_iters < 4;
    if (P.late_list) { e = cudaMemsetAsync(P.late_count, 0, sizeof(int), s); if (e != cudaSuccess) return e; e = cudaErrorNotSupported; }
    TO_DISPATCH_MODEL(P.model, P.m, (e = launch_any<MODEL, 4, RULE>(P, 0, 1, final_pass, s)));
    return e;
}

// pass 2 (+3 when ls_iters > 11): the remaining trials, 8 lanes per instance; commits failures
template <int RULE>
cudaError_t launch_ladder_rule(const DevProblem& P, cudaStream_t s) {
    cudaError_t e = cudaSuccess;
    for (int trial0 = 4; trial0 <= P.opt.ls_iters && e == cudaSuccess; trial0 += 8) {
        const int final_pass = trial0 + 8 > P.opt.ls_iters;
        TO_DISPATCH_MODEL(P.model, P.m, (e = launch_any<MODEL, 8, RULE>(P, trial0, 0, final_pass, s)));
    }
    return e;
}

template cudaError_t launch_forward_rule<TO_RULE>(const DevProblem&, cudaStream_t);
template cudaError_t launch_ladder_rule<TO_RULE>(const DevProblem&, cudaStream_t);

#if TO_RULE == 4
// load_tables makes the same test on the device
bool linesearch_costs_cached(const DevProblem& P) { return P.ncost <= FWD_MAX_COST; }

// the fast loop (rollout_fast) needs its tables to fit FwdTab: the horizon, 2 (n + m) multipliers and two constraints per knot.  The
// compact loop is the compact class (DevProblem::fwd_compact) inside the fast path, with its costs cached as rollout_fast caches them.
int linesearch_path(const DevProblem& P) {
    const bool fast = P.all_diag_cost && P.all_diag_con && P.N <= FWD_MAX_N && P.max_p_knot <= 2 * (P.n + P.m) && P.max_cons_knot <= 2;
    if (TO_FWD_COMPACT && fast && P.fwd_compact && linesearch_costs_cached(P)) return FWD_COMPACT;
    return fast ? FWD_FAST : FWD_GENERIC;
}

cudaError_t launch_forward(const DevProblem& P, cudaStream_t s) {
    cudaError_t e = cudaErrorNotSupported;
    TO_DISPATCH_RULE(P.integration, (e = launch_forward_rule<RULE>(P, s)));
    return e;
}

cudaError_t launch_ladder(const DevProblem& P, cudaStream_t s) {
    cudaError_t e = cudaErrorNotSupported;
    TO_DISPATCH_RULE(P.integration, (e = launch_ladder_rule<RULE>(P, s)));
    return e;
}

cudaError_t launch_accept(const DevProblem& P, cudaStream_t s) { return cudaSuccess; }   // acceptance is committed inside k_linesearch
#endif
