// gains.cuh -- the gain step of the shared-memory Riccati kernels (riccati.cu k_riccati, lie.cu k_riccati_dense / k_riccati_dense_mma):
//     [K | d] = -(Quu + rho I)^-1 [Qux | Qu]      dV += (d'Qu, 1/2 d'Quu d)
// by an LDL' of the M x M matrix Quu + rho I (M <= 8) held in registers, with reciprocal pivots (no division chain), and one triangular
// solve per right-hand-side column.  Quu and L are packed lower by rows: entry (i, j), j <= i, at i (i + 1) / 2 + j.
// Each kernel loads Quu and the right-hand side from its own shared-memory layout and stores the gains itself; only the arithmetic is here.
#pragma once
#include <cuda_runtime.h>

// Quu + rho I = L D L'.  Lf: the off-diagonal entries of the unit-lower L; its diagonal slots hold 1/D_j = rcp(D_j).  dj: D.
// Returns false when a pivot is not positive and finite (Quu + rho I not positive definite: the caller raises rho and restarts).
template <int M, class Rcp>
__device__ __forceinline__ bool ldl_factor(const double (&Quu)[M * (M + 1) / 2], double rho, double (&Lf)[M * (M + 1) / 2], double (&dj)[M],
                                           Rcp rcp) {
    bool pd = true;
#pragma unroll
    for (int j = 0; j < M; j++) {
        double t = Quu[j * (j + 1) / 2 + j] + rho;
#pragma unroll
        for (int r = 0; r < j; r++) t = fma(-Lf[j * (j + 1) / 2 + r] * Lf[j * (j + 1) / 2 + r], dj[r], t);
        if (!(t > 0.0) || !isfinite(t)) pd = false;
        dj[j] = t;
        const double inv = rcp(t);
        Lf[j * (j + 1) / 2 + j] = inv;
#pragma unroll
        for (int i = j + 1; i < M; i++) {
            double v = Quu[i * (i + 1) / 2 + j];
#pragma unroll
            for (int r = 0; r < j; r++) v = fma(-Lf[i * (i + 1) / 2 + r] * Lf[j * (j + 1) / 2 + r], dj[r], v);
            Lf[i * (i + 1) / 2 + j] = v * inv;
        }
    }
    return pd;
}

// kc = -(Quu + rho I)^-1 rhs from the factor of ldl_factor: one column of [K | d] for the column rhs of [Qux | Qu]
template <int M>
__device__ __forceinline__ void ldl_solve(const double (&Lf)[M * (M + 1) / 2], const double (&rhs)[M], double (&kc)[M]) {
#pragma unroll
    for (int a = 0; a < M; a++) {      // forward: L y = -rhs
        double t = -rhs[a];
#pragma unroll
        for (int r = 0; r < a; r++) t = fma(-Lf[a * (a + 1) / 2 + r], kc[r], t);
        kc[a] = t;
    }
#pragma unroll
    for (int a = 0; a < M; a++) kc[a] *= Lf[a * (a + 1) / 2 + a];   // D^-1
#pragma unroll
    for (int a = M - 1; a >= 0; a--) {  // backward: L' x = y
        double t = kc[a];
#pragma unroll
        for (int r = a + 1; r < M; r++) t = fma(-Lf[r * (r + 1) / 2 + a], kc[r], t);
        kc[a] = t;
    }
}

// the knot's terms of the expected decrease for kc = d, rhs = Qu:  t1 = d'Qu,  t2 = 1/2 d'Quu d
template <int M>
__device__ __forceinline__ void expected_decrease(const double (&Quu)[M * (M + 1) / 2], const double (&kc)[M], const double (&rhs)[M], double& t1,
                                                  double& t2) {
    t1 = 0.0; t2 = 0.0;
#pragma unroll
    for (int a = 0; a < M; a++) {
        t1 = fma(kc[a], rhs[a], t1);
        double qd = 0.0;   // (Quu d)_a
#pragma unroll
        for (int r = 0; r < M; r++) qd = fma((r <= a) ? Quu[a * (a + 1) / 2 + r] : Quu[r * (r + 1) / 2 + a], kc[r], qd);
        t2 = fma(0.5 * kc[a], qd, t2);
    }
}
